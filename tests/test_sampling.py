"""Token sampling. CPU: oracle/sampling_oracle.py reproduces the reference's python/sampling.py draw for draw (golden cases made by
running the reference module, tests/golden/make_sampling_golden.py). GPU: csrc/kernels/sampling.cu against the oracle on the same
logits and the same uniform number."""
import ctypes
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN, model_path

import sampling_oracle as so

CASES = json.load(open(os.path.join(GOLDEN, "sampling_cases.json")))
P_F, P_U = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_uint32)


def make_logits(seed, n_vocab, scale):
    return (np.random.RandomState(seed).standard_normal(n_vocab) * scale).astype(np.float32)


def bias_of(case):
    return {int(k): v for k, v in case["bias"].items()} if case["bias"] else None


def test_oracle_matches_reference_sampling():
    for c in CASES:
        logits = make_logits(c["logits_seed"], c["n_vocab"], c["scale"])
        got = so.sample_logits_u(logits, c["temperature"], c["top_p"], c["u"], bias_of(c))
        assert got == c["token"], c


def test_float64_restatement_holds_the_golden_draws():
    """Every golden draw of the reference module lies in its token's interval of the float64 CDF (so.probs64 / so.cdf64), or within
    eps = 2e-6 * max(1, 1 / T) of its edge where the reference's float32 rounding decides; temperature 0 is the float64 argmax."""
    worst = 0.0
    for c in CASES:
        logits = make_logits(c["logits_seed"], c["n_vocab"], c["scale"])
        p = so.probs64(logits, c["temperature"], c["top_p"], bias_of(c))
        tok = c["token"]
        assert p[tok] > 0, c
        if c["temperature"] == 0.0:
            continue
        cdf = so.cdf64(p)
        eps = 2e-6 * max(1.0, 1.0 / c["temperature"])
        left = cdf[tok - 1] if tok > 0 else 0.0
        err = max(left - c["u"], c["u"] - cdf[tok], 0.0)
        worst = max(worst, err / eps)
        assert err <= eps, (c, left, cdf[tok])
    print("worst distance outside the float64 interval / eps: %.3g" % worst)


def test_oracle_argument_errors():
    with pytest.raises(ValueError):
        so.sample_logits_u(np.zeros(8, np.float32), -1.0, 0.5, 0.1)
    with pytest.raises(ValueError):
        so.sample_logits_u(np.zeros(8, np.float32), 1.0, 1.5, 0.1)


def gpu_sample(lib, logits, temperature, top_p, u, bias=None):
    tok = ctypes.c_uint32(0)
    prob = ctypes.c_float(0)
    ids = vals = None
    n = 0
    if bias:
        n = len(bias)
        ids = (ctypes.c_uint32 * n)(*bias.keys())
        vals = (ctypes.c_float * n)(*bias.values())
    ok = lib.library.rwkv_b200_sample_logits(logits.ctypes.data_as(P_F), logits.size, temperature, top_p, u, ids, vals, n, ctypes.byref(tok), ctypes.byref(prob))
    assert ok
    return int(tok.value), float(prob.value)


@pytest.mark.gpu
def test_gpu_sampling_matches_reference_cases(lib):
    """Every golden case of the reference module, through the kernel. A draw whose u sits within 2e-6 of a CDF edge (float32
    softmax / summation-order noise decides it) may land on the neighbouring token; none of the golden cases should."""
    wrong = []
    for c in CASES:
        logits = make_logits(c["logits_seed"], c["n_vocab"], c["scale"])
        tok, _ = gpu_sample(lib, logits, c["temperature"], c["top_p"], c["u"], bias_of(c))
        if tok != c["token"] and so.boundary_distance(logits, c["temperature"], c["top_p"], c["u"], bias_of(c)) > 2e-6:
            wrong.append((c, tok))
    assert not wrong, wrong[:3]


@pytest.mark.gpu
@pytest.mark.parametrize("n_vocab", [7, 256, 1000, 50277, 65536])
def test_gpu_sampling_sweep(lib, n_vocab):
    rng = np.random.RandomState(n_vocab)
    logits = make_logits(5 + n_vocab, n_vocab, 3.0)
    exact = total = 0
    for temperature, top_p in ((1.0, 0.8), (0.5, 0.3), (1.3, 1.0), (1.0, 0.0), (0.0, 0.5)):
        for _ in range(12):
            u = float(rng.random_sample())
            tok, prob = gpu_sample(lib, logits, temperature, top_p, u)
            want = so.sample_logits_u(logits, temperature, top_p, u)
            assert 0 <= tok < n_vocab
            total += 1
            if tok == want:
                exact += 1
            else:
                assert so.boundary_distance(logits, temperature, top_p, u) <= 2e-6, (temperature, top_p, u, tok, want)
    assert exact >= total - 2


@pytest.mark.gpu
def test_gpu_sample_after_eval_and_errors(pkg, lib):
    m = pkg.RWKVModel(lib, model_path("6v0-3m", "FP32"), thread_count=1)
    try:
        ctx = m._ctx.ptr
        tok = ctypes.c_uint32(0)
        # no logits yet -> error, not garbage
        assert not lib.library.rwkv_b200_sample(ctx, 1.0, 0.8, 0.5, None, None, 0, ctypes.byref(tok))
        logits, state = m.eval(ord("a"), None, use_numpy=True)
        for u in (0.01, 0.37, 0.93):
            assert lib.library.rwkv_b200_sample(ctx, 0.9, 0.7, u, None, None, 0, ctypes.byref(tok))
            assert tok.value == so.sample_logits_u(logits, 0.9, 0.7, u) or so.boundary_distance(logits, 0.9, 0.7, u) <= 2e-6
        assert lib.library.rwkv_b200_sample(ctx, 0.0, 0.7, 0.5, None, None, 0, ctypes.byref(tok)) and tok.value == int(np.argmax(logits))
        assert not lib.library.rwkv_b200_sample(ctx, -1.0, 0.7, 0.5, None, None, 0, ctypes.byref(tok))
        assert not lib.library.rwkv_b200_sample(ctx, 1.0, 1.7, 0.5, None, None, 0, ctypes.byref(tok))
        assert not lib.library.rwkv_b200_sample(ctx, 1.0, 0.7, 1.0, None, None, 0, ctypes.byref(tok))
        # resident generation loop: eval_sample keeps state and logits on the device, 4 bytes come back per token
        lib.library.rwkv_b200_state_load(ctx, None)
        cur, gen = ord("T"), []
        for i in range(8):
            assert lib.library.rwkv_b200_eval_sample(ctx, cur, 0.0, 1.0, 0.5, ctypes.byref(tok))
            gen.append(int(tok.value)); cur = int(tok.value)
        st, want = None, []
        cur = ord("T")
        for i in range(8):
            lg, st = m.eval(cur, st, use_numpy=True)
            cur = int(np.argmax(lg)); want.append(cur)
        assert gen == want
    finally:
        m.free()
