"""The bars of tests/test_gpu_kernels.py mean something: on the inputs that test uses, each plausible bug applied to the float64
restatement moves the result by more than ten times the bar a kernel output has to meet. CPU only; a later loosening of the bars
(or of the inputs) that would let such a bug through fails here."""
import numpy as np
import pytest

import kernel_ref as kr
from test_gpu_kernels import (F32, F64, LN_COLUMN_WIDTHS, ln_columns_inputs, ln_mix_inputs, lerp_inputs, ref_wkv6, rng_for, wkv4_inputs,
                              wkv6_inputs)


def assert_caught(r64, r32, bugged):
    moved = kr.error_over_bar(bugged, r64, r32)
    assert moved > 10, moved


@pytest.mark.parametrize("mode,S,T", [("v5.1", 8, 1), ("v5.2", 64, 17), ("v6", 32, 9), ("v6", 128, 63)])
def test_wrong_head_norm_eps_is_caught(mode, S, T):
    d = wkv6_inputs(mode, 3, S, T, rng_for("wkv6", S, mode, T, 3))
    assert_caught(ref_wkv6(d, F64)[0], ref_wkv6(d, F32)[0], ref_wkv6(d, F64, bug="eps")[0])


@pytest.mark.parametrize("mode,S,T", [("v5.2", 16, 7), ("v6", 64, 17), ("v6", 128, 1)])
def test_neighbouring_time_first_is_caught(mode, S, T):
    d = wkv6_inputs(mode, 3, S, T, rng_for("wkv6", S, mode, T, 3))
    assert_caught(ref_wkv6(d, F64)[0], ref_wkv6(d, F32)[0], ref_wkv6(d, F64, bug="tf_neighbour")[0])


def test_neighbouring_time_first_is_caught_in_wkv4():
    d = wkv4_inputs(333, 7, rng_for("wkv4", 333, 7, False), False)
    args = [d[k] for k in ("k", "v", "r", "tf", "td", "aa", "bb", "pp")]
    assert_caught(kr.wkv4(*args, F64)[0], kr.wkv4(*args, F32)[0], kr.wkv4(*args, F64, bug="tf_neighbour")[0])


@pytest.mark.parametrize("mode,S,T", [("v5.1", 8, 9), ("v5.2", 32, 17), ("v6", 64, 63), ("v6", 128, 17)])
def test_dropped_partial_chunk_is_caught(mode, S, T):
    d = wkv6_inputs(mode, 3, S, T, rng_for("wkv6", S, mode, T, 3))
    r64, r32 = ref_wkv6(d, F64), ref_wkv6(d, F32)
    bugged = ref_wkv6(d, F64, bug="drop_tail")
    assert_caught(r64[0], r32[0], bugged[0])
    assert_caught(r64[1], r32[1], bugged[1])


@pytest.mark.parametrize("S,T", [(8, 7), (64, 1), (128, 17)])
def test_per_head_decay_is_caught(S, T):
    d = wkv6_inputs("v5.2", 3, S, T, rng_for("wkv6", S, "v5.2", T, 3))
    assert_caught(ref_wkv6(d, F64)[1], ref_wkv6(d, F32)[1], ref_wkv6(d, F64, bug="per_head_decay")[1])
    if T > 1:       # a token's own output does not see its decay
        assert_caught(ref_wkv6(d, F64)[0], ref_wkv6(d, F32)[0], ref_wkv6(d, F64, bug="per_head_decay")[0])


@pytest.mark.parametrize("C,formula,T", [(64, 0, 2), (2560, 1, 33), (12288, 0, 33)])
def test_token_shift_off_by_one_is_caught(C, formula, T):
    x, w, b, state, coefs = ln_mix_inputs(C, T, 3, rng_for("ln_mix", C, 3, formula, T))
    r64, r32 = kr.ln_mix(x, w, b, state, coefs, formula, F64), kr.ln_mix(x, w, b, state, coefs, formula, F32)
    bugged = kr.ln_mix(x, w, b, state, coefs, formula, F64, bug="shift")
    for j in range(3):
        assert_caught(r64[0][j], r32[0][j], bugged[0][j])


@pytest.mark.parametrize("C", LN_COLUMN_WIDTHS)
@pytest.mark.parametrize("T", [17, 256])
@pytest.mark.parametrize("bug", ["eps", "wb_neighbour", "no_bias", "no_mean", "var_c_minus_1"])
def test_layer_norm_columns_bugs_are_caught(C, T, bug):
    """On the inputs of test_layer_norm_columns_matches_float64 (the ones with a column of variance ~eps, which eps 1e-6 needs)."""
    x, w, b = ln_columns_inputs(C, T, rng_for("ln_columns", C, T))
    r64, r32 = kr.layer_norm_columns(x, w, b, F64), kr.layer_norm_columns(x, w, b, F32)
    assert_caught(r64, r32, kr.layer_norm_columns(x, w, b, F64, bug=bug))


@pytest.mark.parametrize("T,mix,C", [(1, 32, 200), (33, 64, 1000), (8, 30, 200)])
def test_lerp_coefficient_of_wrong_output_is_caught(T, mix, C):
    w2, z, xx, sx, maa = lerp_inputs(C, T, mix, rng_for("lerp", T, mix, C))
    r64, r32 = kr.v6_lerp(w2, z, xx, sx, maa, F64), kr.v6_lerp(w2, z, xx, sx, maa, F32)
    assert_caught(r64[2], r32[2], kr.v6_lerp(w2, z, xx, sx, maa, F64, bug="lerp_j")[2])


# ---- the matrix kernels (tests/test_gpu_gemv.py) -----------------------------------------------------------------------------

def matrix_case(fmt, M, K, T, epi=0, ln=False, tiled=False, seed=0):
    import test_gpu_gemv as tg
    rng = tg.rng_for("bars", fmt, M, K, T, epi, ln, seed)
    xs = tg.inputs([K], T, rng, scale=0.05 if ln else 2.0)
    p = tg.problem(fmt, M, K, T, rng, epi=epi, tiled=tiled)
    if ln:
        tg.with_layernorm(p, xs[0], rng)
    return p, xs


def assert_matrix_bug_caught(p, xs, bug, tc=False):
    import test_gpu_gemv as tg
    r64, r32 = tg.reference(p, xs, F64, tc), tg.reference(p, xs, F32, tc)
    moved = kr.error_over_bar(tg.reference(p, xs, F64, tc, bug=bug), r64, r32, tg.TC_BAR_FACTOR if tc else 4)
    assert moved > 10, (bug, moved)


@pytest.mark.parametrize("fmt,M,K", [("Q5_1", 256, 4096), ("Q4_1", 4096, 160), ("Q4_1", 1000, 32)])
def test_dropped_block_minimum_term_is_caught(fmt, M, K):
    assert_matrix_bug_caught(*matrix_case(fmt, M, K, 1), "drop_min")


@pytest.mark.parametrize("fmt,M,K,T", [("Q5_1", 256, 4096, 1), ("Q4_1", 1000, 32, 1), ("Q5_1", 300, 2048, 3)])
def test_unrounded_activation_sum_is_caught(fmt, M, K, T):
    assert_matrix_bug_caught(*matrix_case(fmt, M, K, T), "s_unrounded")


@pytest.mark.parametrize("epi,tc", [(5, False), (6, False), (5, True), (6, True)])
def test_residual_of_the_neighbouring_row_is_caught(epi, tc):
    assert_matrix_bug_caught(*matrix_case("Q5_1", 300, 2048, 40 if tc else 1, epi, tiled=tc), "res_neighbour", tc)


@pytest.mark.parametrize("tc", [False, True])
def test_gate_of_the_previous_column_is_caught(tc):
    assert_matrix_bug_caught(*matrix_case("Q4_0", 300, 1024, 40 if tc else 3, 6, tiled=tc), "gate_prev_col", tc)


@pytest.mark.parametrize("epi", [7, 8, 9])
@pytest.mark.parametrize("K,tc", [(64, False), (160, False), (256, True)])
def test_bias_of_the_next_row_is_caught(epi, K, tc):
    assert_matrix_bug_caught(*matrix_case("FP16" if tc else "Q5_1", 2048, K, 40 if tc else 1, epi, tiled=tc), "bias_next", tc)


@pytest.mark.parametrize("case,bug", [(2, "ln_eps"), (4, "ln_eps"), (6, "ln_eps"), (0, "ln_no_b"), (2, "ln_no_b"), (4, "ln_no_b"), (6, "ln_no_b")])
def test_layernorm_prologue_bugs_are_caught(case, bug):
    """On the heads of tests/test_gpu_gemv.py: eps 1e-6 instead of 1e-5 on those whose inputs have a small variance (at unit variance
    the difference is invisible), a dropped ln_b on unit-variance and small-variance ones."""
    import test_gpu_gemv as tg
    fmt, V, C, T, _, scale = tg.HEAD_CASES[case]
    V = min(V, 4096)       # the same inputs; fewer rows keep this CPU test short
    p, xs = tg.head_case(fmt, V, C, T, scale)
    assert_matrix_bug_caught(dict(p, M=V, raw=p["raw"][:V * len(p["raw"]) // p["M"]]), xs, bug)


def test_dropped_column_scale_is_caught():
    p, xs = matrix_case("Q5_0", 256, 4096, 48, 5, tiled=True)
    xs[0][:, 3] *= 3.0e5
    assert_matrix_bug_caught(p, xs, "no_colscale", tc=True)


@pytest.mark.parametrize("M", [300, 4096 + 1])
def test_dropped_partial_row_tile_is_caught(M):
    assert_matrix_bug_caught(*matrix_case("Q8_0", M, 256, 33, tiled=True), "drop_last_tile", tc=True)


def test_dropped_last_k_split_is_caught():
    """256 x 4096: two row tiles, each cut over a cluster of 8 CTAs (tests/test_gpu_gemv.py asserts the cut)."""
    import test_gpu_gemv as tg
    p, xs = matrix_case("Q5_0", 256, 4096, 64, tiled=True)
    r64, r32 = (kr.gemm_tc(p["type"], p["raw"], p["M"], xs[0], dt) for dt in (F64, F32))
    bugged = kr.gemm_tc(p["type"], p["raw"], p["M"], xs[0], F64, bug="drop_last_ksplit", ksplit=8)
    assert kr.error_over_bar(bugged, r64, r32, tg.TC_BAR_FACTOR) > 10


@pytest.mark.parametrize("fmt,K", [("Q4_0", 32), ("Q5_0", 96), ("Q8_0", 14336 + 32)])
def test_dropped_odd_trailing_block_is_caught(fmt, K):
    assert_matrix_bug_caught(*matrix_case(fmt, 128, K, 1), "drop_odd_block")
