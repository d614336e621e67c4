"""The bars of tests/test_gpu_kernels.py mean something: on the inputs that test uses, each plausible bug applied to the float64
restatement moves the result by more than ten times the bar a kernel output has to meet. CPU only; a later loosening of the bars
(or of the inputs) that would let such a bug through fails here."""
import numpy as np
import pytest

import kernel_ref as kr
from test_gpu_kernels import F32, F64, ln_mix_inputs, lerp_inputs, ref_wkv6, rng_for, wkv4_inputs, wkv6_inputs


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


@pytest.mark.parametrize("T,mix,C", [(1, 32, 200), (33, 64, 1000), (8, 30, 200)])
def test_lerp_coefficient_of_wrong_output_is_caught(T, mix, C):
    w2, z, xx, sx, maa = lerp_inputs(C, T, mix, rng_for("lerp", T, mix, C))
    r64, r32 = kr.v6_lerp(w2, z, xx, sx, maa, F64), kr.v6_lerp(w2, z, xx, sx, maa, F32)
    assert_caught(r64[2], r32[2], kr.v6_lerp(w2, z, xx, sx, maa, F64, bug="lerp_j")[2])
