"""Per-kernel parity of the eval path's element-wise and recurrent kernels (csrc/kernels/glue.cu, wkv.cu) through the
rwkv_b200_test_* hooks, at every compiled instantiation: head sizes 8-128, LayerNorm widths of 1-16 channels per thread, the decode /
tile-8 / tile-32 lerp kernels with fixed and generic mix, and the batch mode (seq_stride > 0) of the LayerNorm-mix and WKV kernels.

Every output and carried state is compared with the float64 restatement in kernel_ref.py. The bar of one output (of each token
column of an activation) is max(4 x |float32 restatement - float64|, 1e-6 x the output's largest magnitude): tight where fp32 is
accurate, wide only where the operation is ill-conditioned on this input (test_kernel_bars.py checks that plausible bugs land far
outside it). No output may keep a NaN of the 0xFF fill, and no guard element after an output may change. The bit-level contracts
the engine relies on are asserted too: T-token launches equal chained single-token launches, every lerp kernel gives the same bits
for a token, batch columns equal single-sequence launches of the same kernel, and staged columns equal the fp32 output quantised the reference's way,
byte for byte."""
import collections
import zlib

import numpy as np
import pytest

import ggml_file as gf
import kernel_hooks as kh
import kernel_ref as kr

pytestmark = pytest.mark.gpu
F64, F32 = np.float64, np.float32
T_LIST = [1, 7, 8, 9, 16, 17, 63, 128, 512]
HEAD_SIZES = [8, 16, 32, 64, 128]
WKV6_MODES = ["v5.1", "v5.2", "v6"]
STAGE_TYPES = [gf.TYPE_FP32, gf.TYPE_FP16, gf.TYPE_Q5_0, gf.TYPE_Q5_1]     # stage classes F32, F16, Q8_0, Q8_1
WORST = collections.defaultdict(float)


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    for family in sorted(WORST):
        print("\n%-10s worst error / bar = %.3f" % (family, WORST[family]), end="")
    print()


def both(ref):
    """The restatement `ref(dtype)` in float64 and in float32."""
    return ref(F64), ref(F32)


def check(family, name, got, r64, r32):
    """got: the kernel's output; r64 / r32: the same quantity from the float64 / float32 restatement."""
    r64, r32 = np.asarray(r64, F64), np.asarray(r32, F64)
    got = np.asarray(got, F64).reshape(r64.shape)
    assert not np.isnan(got).any(), (family, name, "NaN left in the output")
    ratio = kr.error_over_bar(got, r64, r32)
    WORST[family] = max(WORST[family], ratio)
    assert ratio <= 1, (family, name, ratio, np.abs(got - r64).max())


def guards(o):
    for name, buf in o.items():
        assert buf.guard_intact(), ("write past the end of", name)


def bits(a):
    return np.ascontiguousarray(a).tobytes()


def rng_for(*key):
    return np.random.default_rng(zlib.crc32(repr(key).encode()))


# ---- WKV5 / WKV6 -------------------------------------------------------------------------------------------------------

def wkv6_inputs(mode, H, S, T, rng):
    C = H * S
    r, k, v = (rng.standard_normal((C, T)).astype(F32) * 0.7 for _ in range(3))
    # decays near 1 (exp(-exp(-8))) and near 0 (exp(-exp(3))), so long passes both accumulate and forget
    decay = lambda shape: np.exp(-np.exp(rng.choice([-8.0, -2.0, 0.5, 3.0], size=shape) + 0.1 * rng.standard_normal(shape))).astype(F32)
    if mode == "v5.1":
        td, tf, g, eps = decay(H), rng.standard_normal(H).astype(F32), None, 1e-5
    elif mode == "v5.2":
        td, tf, g, eps = decay(C), rng.standard_normal(C).astype(F32), rng.standard_normal((C, T)).astype(F32), 1e-5
    else:
        td, tf, g, eps = decay((C, T)), rng.standard_normal(C).astype(F32), rng.standard_normal((C, T)).astype(F32), 64e-5
    state = rng.standard_normal(H * S * S).astype(F32)
    lnx_w = (1 + 0.2 * rng.standard_normal(C)).astype(F32)
    lnx_b = (0.2 * rng.standard_normal(C)).astype(F32)
    return dict(r=r, k=k, v=v, td=td, tf=tf, state=state, lnx_w=lnx_w, lnx_b=lnx_b, g=g, eps=eps, H=H, S=S)


def run_wkv6(lib, d, mode, **kw):
    return kh.wkv6(lib, d["r"], d["k"], d["v"], d["td"], d["tf"], d["state"], d["lnx_w"], d["lnx_b"], d["g"], d["eps"], d["H"], d["S"],
                   td_per_token=mode == "v6", per_head=mode == "v5.1", **kw)


def ref_wkv6(d, dt, **kw):
    return kr.wkv6(d["r"], d["k"], d["v"], d["td"], d["tf"], d["state"], d["lnx_w"], d["lnx_b"], d["g"], d["eps"], d["H"], d["S"], dt, **kw)


def wkv6_cases():
    cases = [(S, mode, T, 3 if i % 2 == 0 else 1) for S in HEAD_SIZES for mode in WKV6_MODES for i, T in enumerate(T_LIST)]
    return cases + [(64, mode, T, 64) for mode in WKV6_MODES for T in (1, 17, 128)]


@pytest.mark.parametrize("S,mode,T,H", wkv6_cases())
def test_wkv6_matches_float64(lib, S, mode, T, H):
    d = wkv6_inputs(mode, H, S, T, rng_for("wkv6", S, mode, T, H))
    o = run_wkv6(lib, d, mode)
    guards(o)
    (y64, s64), (y32, s32) = both(lambda dt: ref_wkv6(d, dt))
    check("wkv6", "y", o["y"].cols(H * S), y64, y32)
    check("wkv6", "state", o["state"].value, s64, s32)


def slice_cols(d, t0, t1, keys):
    return {key: (val[:, t0:t1] if key in keys and val is not None else val) for key, val in d.items()}


@pytest.mark.parametrize("S", HEAD_SIZES)
@pytest.mark.parametrize("mode", WKV6_MODES)
def test_wkv6_sequence_equals_chained_tokens(lib, S, mode):
    T = 17
    d = wkv6_inputs(mode, 2, S, T, rng_for("wkv6-chain", S, mode))
    full = run_wkv6(lib, d, mode)
    cols = ("r", "k", "v", "g") + (("td",) if mode == "v6" else ())
    state = d["state"]
    for t in range(T):
        one = run_wkv6(lib, dict(slice_cols(d, t, t + 1, cols), state=state), mode)
        assert bits(one["y"].value) == bits(full["y"].cols(2 * S)[:, t].copy()), t
        state = one["state"].value.copy()
    assert bits(state) == bits(full["state"].value)


@pytest.mark.parametrize("S", HEAD_SIZES)
@pytest.mark.parametrize("mode", WKV6_MODES)
@pytest.mark.parametrize("n_seq", [1, 5, 17])
def test_wkv6_batch_columns_equal_single_launches(lib, S, mode, n_seq):
    H = 3
    SS = H * S * S
    stride = SS + 40
    d = wkv6_inputs(mode, H, S, n_seq, rng_for("wkv6-batch", S, mode, n_seq))
    states = rng_for("wkv6-batch-state", S).standard_normal((n_seq - 1) * stride + SS).astype(F32)
    batch = run_wkv6(lib, dict(d, state=states), mode, n_seq=n_seq, seq_stride=stride)
    guards(batch)
    cols = ("r", "k", "v", "g") + (("td",) if mode == "v6" else ())
    for b in range(n_seq):
        st = states[b * stride:b * stride + SS]
        one = run_wkv6(lib, dict(slice_cols(d, b, b + 1, cols), state=st), mode)
        assert bits(one["y"].value) == bits(batch["y"].cols(H * S)[:, b].copy()), b
        assert bits(one["state"].value) == bits(batch["state"].value[b * stride:b * stride + SS]), b
    # the gaps between the sequences' states are not written
    gaps = np.concatenate([batch["state"].value[b * stride + SS:(b + 1) * stride] for b in range(n_seq - 1)] + [np.zeros(0, F32)])
    assert (gaps.view(np.uint32) == 0xFFFFFFFF).all()


@pytest.mark.parametrize("S", [32, 64, 128])
@pytest.mark.parametrize("q_type", STAGE_TYPES)
def test_wkv6_staged_column(lib, S, q_type):
    d = wkv6_inputs("v6", 3, S, 1, rng_for("wkv6-q", S, q_type))
    o = run_wkv6(lib, d, "v6", q_type=q_type)
    assert bits(o["q"].buf) == bits(kr.staged_column(o["y"].value, q_type, guard=kh.GUARD_BYTES))


# ---- WKV7 --------------------------------------------------------------------------------------------------------------

def wkv7_inputs(H, S, T, rng, vgate):
    C = H * S
    n = lambda *shape: rng.standard_normal(shape).astype(F32)
    sig = lambda x: (1 / (1 + np.exp(-x))).astype(F32)
    d = dict(r=n(C, T), w=np.exp(-0.606531 * sig(2 * n(C, T))).astype(F32), k=n(C, T), v=n(C, T), aa=sig(n(C, T)), g=n(C, T),
             vgate=sig(n(C, T)) if vgate else None, v_first=n(C, T) if vgate else None,
             k_k=(1 + 0.3 * n(C)).astype(F32), k_a=(1 + 0.3 * n(C)).astype(F32), r_k=(0.5 * n(C)).astype(F32),
             lnx_w=(1 + 0.2 * n(C)).astype(F32), lnx_b=(0.2 * n(C)).astype(F32), state=(0.5 * n(H * S * S)).astype(F32), H=H, S=S)
    return d


def run_wkv7(lib, d, **kw):
    return kh.wkv7(lib, d["r"], d["w"], d["k"], d["v"], d["aa"], d["g"], d["vgate"], d["v_first"], d["k_k"], d["k_a"], d["r_k"],
                   d["lnx_w"], d["lnx_b"], d["state"], d["H"], d["S"], **kw)


def ref_wkv7(d, dt):
    return kr.wkv7(d["r"], d["w"], d["k"], d["v"], d["aa"], d["g"], d["vgate"], d["v_first"], d["k_k"], d["k_a"], d["r_k"],
                   d["lnx_w"], d["lnx_b"], d["state"], d["H"], d["S"], dt)


@pytest.mark.parametrize("S", HEAD_SIZES)
@pytest.mark.parametrize("vgate", [False, True])
@pytest.mark.parametrize("T", T_LIST)
def test_wkv7_matches_float64(lib, S, vgate, T):
    H = 3 if T % 2 else 2
    d = wkv7_inputs(H, S, T, rng_for("wkv7", S, vgate, T), vgate)
    o = run_wkv7(lib, d, v_out=T != 8)
    guards(o)
    r64, r32 = both(lambda dt: ref_wkv7(d, dt))
    check("wkv7", "y", o["y"].cols(H * S), r64[0], r32[0])
    check("wkv7", "state", o["state"].value, r64[2], r32[2])
    if "v" in o:
        check("wkv7", "v_out", o["v"].cols(H * S), r64[1], r32[1])


WKV7_COLS = ("r", "w", "k", "v", "aa", "g", "vgate", "v_first")


@pytest.mark.parametrize("S", HEAD_SIZES)
def test_wkv7_sequence_equals_chained_tokens(lib, S):
    T = 17
    d = wkv7_inputs(2, S, T, rng_for("wkv7-chain", S), True)
    full = run_wkv7(lib, d)
    state = d["state"]
    for t in range(T):
        one = run_wkv7(lib, dict(slice_cols(d, t, t + 1, WKV7_COLS), state=state))
        assert bits(one["y"].value) == bits(full["y"].cols(2 * S)[:, t].copy()), t
        assert bits(one["v"].value) == bits(full["v"].cols(2 * S)[:, t].copy()), t
        state = one["state"].value.copy()
    assert bits(state) == bits(full["state"].value)


@pytest.mark.parametrize("S", HEAD_SIZES)
@pytest.mark.parametrize("n_seq", [1, 5, 17])
def test_wkv7_batch_columns_equal_single_launches(lib, S, n_seq):
    H = 2
    SS = H * S * S
    stride = SS + 24
    d = wkv7_inputs(H, S, n_seq, rng_for("wkv7-batch", S, n_seq), n_seq != 5)
    states = rng_for("wkv7-batch-state", S).standard_normal((n_seq - 1) * stride + SS).astype(F32)
    batch = run_wkv7(lib, dict(d, state=states), n_seq=n_seq, seq_stride=stride)
    guards(batch)
    for b in range(n_seq):
        one = run_wkv7(lib, dict(slice_cols(d, b, b + 1, WKV7_COLS), state=states[b * stride:b * stride + SS]))
        assert bits(one["y"].value) == bits(batch["y"].cols(H * S)[:, b].copy()), b
        assert bits(one["v"].value) == bits(batch["v"].cols(H * S)[:, b].copy()), b
        assert bits(one["state"].value) == bits(batch["state"].value[b * stride:b * stride + SS]), b


@pytest.mark.parametrize("S", [32, 64, 128])
@pytest.mark.parametrize("q_type", STAGE_TYPES)
def test_wkv7_staged_column(lib, S, q_type):
    d = wkv7_inputs(3, S, 1, rng_for("wkv7-q", S, q_type), True)
    o = run_wkv7(lib, d, q_type=q_type)
    assert bits(o["q"].buf) == bits(kr.staged_column(o["y"].value, q_type, guard=kh.GUARD_BYTES))


# ---- WKV4 --------------------------------------------------------------------------------------------------------------

def wkv4_inputs(C, T, rng, fresh):
    k = rng.standard_normal((C, T)).astype(F32) * 2
    big = rng.random((C, T)) < 0.3
    k[big] = rng.uniform(-80, 80, big.sum()).astype(F32)           # the max trick of the exponentials has to carry these
    v, r = rng.standard_normal((C, T)).astype(F32), (1 / (1 + np.exp(-rng.standard_normal((C, T))))).astype(F32)
    tf = rng.standard_normal(C).astype(F32)
    td = (-np.exp(rng.choice([-8.0, -1.0, 0.5, 3.0], C))).astype(F32)
    if fresh:                                                     # rwkv_init_state: zeros, pp = -1e30
        aa, bb, pp = np.zeros(C, F32), np.zeros(C, F32), np.full(C, -1e30, F32)
    else:
        aa, bb, pp = rng.standard_normal(C).astype(F32), rng.uniform(0.5, 3, C).astype(F32), (5 * rng.standard_normal(C)).astype(F32)
    return dict(k=k, v=v, r=r, tf=tf, td=td, aa=aa, bb=bb, pp=pp)


def run_wkv4(lib, d, **kw):
    return kh.wkv4(lib, d["k"], d["v"], d["r"], d["tf"], d["td"], d["aa"], d["bb"], d["pp"], **kw)


def ref_wkv4(d, dt):
    return kr.wkv4(d["k"], d["v"], d["r"], d["tf"], d["td"], d["aa"], d["bb"], d["pp"], dt)


@pytest.mark.parametrize("C", [100, 333, 1056, 4160])
@pytest.mark.parametrize("T", [1, 7, 33, 128])
@pytest.mark.parametrize("fresh", [True, False])
def test_wkv4_matches_float64(lib, C, T, fresh):
    d = wkv4_inputs(C, T, rng_for("wkv4", C, T, fresh), fresh)
    o = run_wkv4(lib, d)
    guards(o)
    r64, r32 = both(lambda dt: ref_wkv4(d, dt))
    check("wkv4", "y", o["y"].cols(C), r64[0], r32[0])
    for i, name in enumerate(("aa", "bb", "pp")):
        check("wkv4", name, o[name].value, r64[1 + i], r32[1 + i])


@pytest.mark.parametrize("C", [333, 1056])
@pytest.mark.parametrize("n_seq", [1, 5, 17])
def test_wkv4_batch_columns_equal_single_launches(lib, C, n_seq):
    stride = C + 8
    d = wkv4_inputs(C, n_seq, rng_for("wkv4-batch", C, n_seq), False)
    rng = rng_for("wkv4-batch-state", C)
    n = (n_seq - 1) * stride + C
    st = dict(aa=rng.standard_normal(n).astype(F32), bb=rng.uniform(0.5, 3, n).astype(F32), pp=(5 * rng.standard_normal(n)).astype(F32))
    batch = run_wkv4(lib, dict(d, **st), n_seq=n_seq, seq_stride=stride)
    guards(batch)
    for b in range(n_seq):
        sl = slice(b * stride, b * stride + C)
        one = run_wkv4(lib, dict(slice_cols(d, b, b + 1, ("k", "v", "r")), aa=st["aa"][sl], bb=st["bb"][sl], pp=st["pp"][sl]))
        assert bits(one["y"].value) == bits(batch["y"].cols(C)[:, b].copy()), b
        for name in ("aa", "bb", "pp"):
            assert bits(one[name].value) == bits(batch[name].value[sl]), (b, name)


@pytest.mark.parametrize("q_type", STAGE_TYPES)
def test_wkv4_staged_column(lib, q_type):
    d = wkv4_inputs(1056, 1, rng_for("wkv4-q", q_type), False)
    o = run_wkv4(lib, d, q_type=q_type)
    assert bits(o["q"].buf) == bits(kr.staged_column(o["y"].value, q_type, guard=kh.GUARD_BYTES))


# ---- LayerNorm + token shift + mix -------------------------------------------------------------------------------------

def ln_mix_inputs(C, T, n_out, rng):
    x = rng.standard_normal((C, T)).astype(F32) * 1.5
    # every other token is ill-conditioned for an fp32 LayerNorm, with a well-conditioned token on either side (two of them in a
    # row could hide each other's fp32 error in their difference prev - xx, and with it the bar of the token shift)
    for t in range(1, T):
        if t % 4 == 1:
            x[:, t] = (1e4 + rng.standard_normal(C)).astype(F32)   # large common offset: mean 1e4, std 1
        elif t % 4 == 3:
            x[:, t] = F32(3.7)                                     # constant column: variance 0
    w = (1 + 0.2 * rng.standard_normal(C)).astype(F32)
    b = (0.2 * rng.standard_normal(C)).astype(F32)
    state = rng.standard_normal(C).astype(F32)
    coefs = [rng.random(C).astype(F32) for _ in range(n_out)]
    return x, w, b, state, coefs


@pytest.mark.parametrize("C", [64, 768, 1000, 2048, 2560, 4096, 5120, 8192, 12288])
@pytest.mark.parametrize("n_out", [1, 3, 4, 6])
@pytest.mark.parametrize("formula", [0, 1])
@pytest.mark.parametrize("T", [1, 2, 33])
def test_ln_mix_matches_float64(lib, C, n_out, formula, T):
    x, w, b, state, coefs = ln_mix_inputs(C, T, n_out, rng_for("ln_mix", C, n_out, formula, T))
    with_xs = n_out != 4                                     # out_xx / out_sx are optional
    o = kh.ln_mix(lib, x, w, b, state, coefs, formula, xx=with_xs, sx=with_xs)
    guards(o)
    r64, r32 = both(lambda dt: kr.ln_mix(x, w, b, state, coefs, formula, dt))
    for j in range(n_out):
        check("ln_mix", "out%d" % j, o["out%d" % j].cols(C), r64[0][j], r32[0][j])
    if with_xs:
        check("ln_mix", "xx", o["xx"].cols(C), r64[1], r32[1])
        check("ln_mix", "sx", o["sx"].cols(C), r64[2], r32[2])
    check("ln_mix", "state", o["state"].value, r64[3], r32[3])


@pytest.mark.parametrize("C", [64, 1000, 2560, 5120, 12288])
def test_ln_mix_sequence_equals_chained_tokens(lib, C):
    T = 7
    x, w, b, state, coefs = ln_mix_inputs(C, T, 6, rng_for("ln_mix-chain", C))
    for formula in (0, 1):
        full = kh.ln_mix(lib, x, w, b, state, coefs, formula)
        st = state
        for t in range(T):
            one = kh.ln_mix(lib, x[:, t:t + 1], w, b, st, coefs, formula)
            for key in [k for k in one if k != "state"]:
                assert bits(one[key].value) == bits(full[key].cols(C)[:, t].copy()), (formula, t, key)
            st = one["state"].value.copy()
        assert bits(st) == bits(full["state"].value)


@pytest.mark.parametrize("C", [64, 768, 1000, 2048, 2560, 4096, 5120, 12288])
@pytest.mark.parametrize("n_seq", [1, 5, 17])
@pytest.mark.parametrize("formula", [0, 1])
def test_ln_mix_batch(lib, C, n_seq, formula):
    """Each column equals the single-sequence kernel on that sequence's carry, and matches float64 itself."""
    n_out = 6 if formula else 2
    x, w, b, _, coefs = ln_mix_inputs(C, n_seq, n_out, rng_for("ln_mix-batch", C, n_seq, formula))
    stride = C + 32
    states = rng_for("ln_mix-batch-state", C).standard_normal((n_seq - 1) * stride + C).astype(F32)
    batch = kh.ln_mix(lib, x, w, b, states, coefs, formula, n_seq=n_seq, seq_stride=stride)
    guards(batch)
    for s in range(n_seq):
        carry = states[s * stride:s * stride + C]
        one = kh.ln_mix(lib, x[:, s:s + 1], w, b, carry, coefs, formula)
        for key in [k for k in one if k != "state"]:
            assert bits(one[key].value) == bits(batch[key].cols(C)[:, s].copy()), (s, key)
        assert bits(one["state"].value) == bits(batch["state"].value[s * stride:s * stride + C]), s
        r64, r32 = both(lambda dt: kr.ln_mix(x[:, s:s + 1], w, b, carry, coefs, formula, dt))
        for j in range(n_out):
            check("ln_mix_b", "out%d" % j, batch["out%d" % j].cols(C)[:, s:s + 1], r64[0][j], r32[0][j])
        check("ln_mix_b", "state", batch["state"].value[s * stride:s * stride + C], r64[3], r32[3])


# ---- LayerNorm of columns (the tensor-core head of scoring passes) --------------------------------------------------------

def ln_columns_inputs(C, T, rng):
    """Unit-scale columns and, cycling from the second column on, ones the LayerNorm's conditioning or its eps decides: a large
    common offset over a spread of 1, a variance of the order of eps (1e-5) on an offset of 0.5, and a constant column."""
    x = rng.standard_normal((C, T)).astype(F32) * 1.5
    for t in range(1, T):
        if t % 4 == 1:
            x[:, t] = (1e4 + rng.standard_normal(C)).astype(F32)
        elif t % 4 == 2:
            x[:, t] = (0.5 + 3e-3 * rng.standard_normal(C)).astype(F32)
        elif t % 4 == 3:
            x[:, t] = F32(3.7)
    w = (1 + 0.2 * rng.standard_normal(C)).astype(F32)
    b = (0.2 * rng.standard_normal(C)).astype(F32)
    return x, w, b


LN_COLUMN_WIDTHS = [100, 300, 768, 1000, 1024, 2048, 2560, 4096, 5120]      # the published n_embed and widths off the 256-thread stride


@pytest.mark.parametrize("C", LN_COLUMN_WIDTHS)
@pytest.mark.parametrize("T", [1, 17, 256])
def test_layer_norm_columns_matches_float64(lib, C, T):
    x, w, b = ln_columns_inputs(C, T, rng_for("ln_columns", C, T))
    y = kh.layer_norm_columns(lib, x, w, b)
    assert y.guard_intact(), "write past the end of y"
    check("ln_columns", "y", y.cols(C), *both(lambda dt: kr.layer_norm_columns(x, w, b, dt)))


# ---- v6 lerp -----------------------------------------------------------------------------------------------------------

def lerp_inputs(C, T, mix, rng):
    w2 = (rng.standard_normal((5, C, mix)) / np.sqrt(mix)).astype(F32)
    z = np.tanh(rng.standard_normal((5 * mix, T))).astype(F32)
    xx, sx = rng.standard_normal((C, T)).astype(F32), rng.standard_normal((C, T)).astype(F32)
    maa = rng.random((5, C)).astype(F32)
    return w2, z, xx, sx, maa


@pytest.mark.parametrize("T", [1, 7, 8, 31, 32, 33, 100])
@pytest.mark.parametrize("mix", [32, 64, 48, 96, 30])
@pytest.mark.parametrize("C", [200, 1000])
def test_v6_lerp_matches_float64(lib, T, mix, C):
    w2, z, xx, sx, maa = lerp_inputs(C, T, mix, rng_for("lerp", T, mix, C))
    o = kh.v6_lerp(lib, w2, z, xx, sx, maa)
    guards(o)
    r64, r32 = both(lambda dt: kr.v6_lerp(w2, z, xx, sx, maa, dt))
    for j in range(5):
        check("v6_lerp", "out%d" % j, o["out%d" % j].cols(C), r64[j], r32[j])


@pytest.mark.parametrize("mix", [32, 64, 48, 96, 30, 160])
def test_v6_lerp_kernels_agree_bit_for_bit(lib, mix):
    """A token's outputs are the same bits from the decode kernel (T < 8), the tile-8 kernel (8 <= T < 32) and the tile-32 kernel."""
    C, T = 200, 40
    w2, z, xx, sx, maa = lerp_inputs(C, T, mix, rng_for("lerp-bits", mix))
    t32 = kh.v6_lerp(lib, w2, z, xx, sx, maa)
    t8 = kh.v6_lerp(lib, w2, z[:, :9], xx[:, :9], sx[:, :9], maa)
    for t in range(9):
        one = kh.v6_lerp(lib, w2, z[:, t:t + 1], xx[:, t:t + 1], sx[:, t:t + 1], maa)
        for j in range(5):
            col = bits(one["out%d" % j].value)
            assert col == bits(t8["out%d" % j].cols(C)[:, t].copy()) == bits(t32["out%d" % j].cols(C)[:, t].copy()), (t, j)


@pytest.mark.parametrize("mix", [32, 64, 96])
@pytest.mark.parametrize("q_type", STAGE_TYPES)
def test_v6_lerp_staged_columns(lib, mix, q_type):
    C = 1056
    w2, z, xx, sx, maa = lerp_inputs(C, 1, mix, rng_for("lerp-q", mix, q_type))
    types = [q_type, gf.TYPE_Q5_1, gf.TYPE_FP16, gf.TYPE_Q8_0, gf.TYPE_Q4_1]      # every output its own consumer type
    o = kh.v6_lerp(lib, w2, z, xx, sx, maa, q_types=types)
    guards(o)
    for j in range(5):
        assert bits(o["q%d" % j].buf) == bits(kr.staged_column(o["out%d" % j].value, types[j], guard=kh.GUARD_BYTES)), j


# ---- embedding + ln0 ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("C", [64, 2560, 4096])
@pytest.mark.parametrize("table", ["FP32", "FP16"])
def test_embed_ln0_matches_float64(lib, C, table):
    rng = rng_for("embed", C, table)
    V = 300
    emb = rng.standard_normal((V, C)).astype(F32) * 0.3 + rng.standard_normal((V, 1)).astype(F32)
    emb = emb.astype(np.float16) if table == "FP16" else emb
    w, b = (1 + 0.2 * rng.standard_normal(C)).astype(F32), (0.2 * rng.standard_normal(C)).astype(F32)
    tokens = np.array([0, V - 1, 17, V - 1, 0, 123], np.int32)
    o = kh.embed_ln0(lib, emb, tokens, w, b)
    assert o.guard_intact()
    check("embed_ln0", "x", o.cols(C), *both(lambda dt: kr.embed_ln0(emb.astype(F32), tokens, w, b, dt)))
