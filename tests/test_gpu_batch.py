"""Batched multi-sequence decode (rwkv_b200_batch_*: the LayerNorm-mix and WKV kernels of csrc/kernels/glue.cu and wkv.cu in
batch mode): B sequences advanced one token each per call must give, per sequence, exactly the bits of that sequence evaluated
alone through rwkv_eval -- the weights are streamed once for the B tokens, nothing else may change. batch_shape_supported (api.cpp)
admits the model shapes these tests cover."""
import ctypes

import numpy as np
import pytest

from conftest import LONG_PROMPT, model_path

pytestmark = pytest.mark.gpu
P_F, P_U = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_uint32)


def alone(lib, ctx, toks, n_state, n_logits, state0=None):
    state = np.zeros(n_state, np.float32) if state0 is None else state0.copy()
    logits = np.zeros(n_logits, np.float32)
    out = []
    for i, t in enumerate(toks):
        sin = None if (i == 0 and state0 is None) else state.ctypes.data_as(P_F)
        assert lib.library.rwkv_eval(ctx.ptr, t, sin, state.ctypes.data_as(P_F), logits.ctypes.data_as(P_F))
        out.append(logits.copy())
    return out, state


def check_batch(lib, path, n_seq, n_steps, vocab_mod=None):
    ctx = lib.rwkv_init_from_file(path, 1, 0)
    batch = None
    try:
        n_state, n_logits = lib.rwkv_get_state_buffer_element_count(ctx), lib.rwkv_get_logits_buffer_element_count(ctx)
        V = vocab_mod or n_logits
        prompts = [[(LONG_PROMPT[(3 * b + i) % len(LONG_PROMPT)] * (b + 1) + 7 * b) % V for i in range(n_steps)] for b in range(n_seq)]
        want = [alone(lib, ctx, p, n_state, n_logits) for p in prompts]
        bptr = lib.library.rwkv_b200_batch_create(ctx.ptr, n_seq)
        assert bptr, "batch_create failed"
        batch = ctypes.c_void_p(bptr)
        assert lib.library.rwkv_b200_batch_size(batch) == n_seq and lib.library.rwkv_b200_batch_size(ctx.ptr) == 0
        lg = np.zeros(n_logits, np.float32)
        st = np.zeros(n_state, np.float32)
        for step in range(n_steps):
            toks = (ctypes.c_uint32 * n_seq)(*[p[step] for p in prompts])
            want_logits = step % 3 != 1 or step == n_steps - 1          # some steps skip the head
            assert lib.library.rwkv_b200_batch_eval(batch, toks, want_logits)
            if want_logits:
                for b in range(n_seq):
                    assert lib.library.rwkv_b200_batch_get_logits(batch, b, lg.ctypes.data_as(P_F))
                    assert lg.tobytes() == want[b][0][step].tobytes(), (path, b, step, np.abs(lg - want[b][0][step]).max())
        for b in range(n_seq):
            assert lib.library.rwkv_b200_batch_get_state(batch, b, st.ctypes.data_as(P_F))
            assert st.tobytes() == want[b][1].tobytes(), (path, b, np.abs(st - want[b][1]).max())
        # hand a host state to one slot, reset another, continue: each sequence still evolves on its own
        if n_seq >= 2:
            assert lib.library.rwkv_b200_batch_set_state(batch, 0, want[1][1].ctypes.data_as(P_F))     # slot 0 continues sequence 1
            assert lib.library.rwkv_b200_batch_set_state(batch, 1, None)                               # slot 1 starts over
            more = [5 % V, 9 % V, 1 % V]
            w0, s0 = alone(lib, ctx, more, n_state, n_logits, state0=want[1][1])
            w1, s1 = alone(lib, ctx, more, n_state, n_logits)
            for t in more:
                toks = (ctypes.c_uint32 * n_seq)(*([t] * n_seq))
                assert lib.library.rwkv_b200_batch_eval(batch, toks, True)
            assert lib.library.rwkv_b200_batch_get_logits(batch, 0, lg.ctypes.data_as(P_F)) and lg.tobytes() == w0[-1].tobytes()
            assert lib.library.rwkv_b200_batch_get_logits(batch, 1, lg.ctypes.data_as(P_F)) and lg.tobytes() == w1[-1].tobytes()
            assert lib.library.rwkv_b200_batch_get_state(batch, 1, st.ctypes.data_as(P_F)) and st.tobytes() == s1.tobytes()
        # the plain entry points refuse a batch context
        assert not lib.library.rwkv_eval(batch, 1, None, st.ctypes.data_as(P_F), None)
    finally:
        if batch:
            lib.library.rwkv_free(batch)
        lib.rwkv_free(ctx)


@pytest.mark.parametrize("ver", ["4v0-660K", "5v1-730K", "5v2-730K", "6v0-3m"])
@pytest.mark.parametrize("fmt", ["FP32", "Q5_1"])
def test_batch_equals_alone_bitwise_fixtures(lib, ver, fmt):
    check_batch(lib, model_path(ver, fmt), n_seq=5, n_steps=9)


def test_batch_of_one_and_odd_sizes(lib):
    for n in (1, 2, 3, 11):
        check_batch(lib, model_path("6v0-3m", "FP16"), n_seq=n, n_steps=4)


@pytest.mark.parametrize("preset,fmt", [("rwkv6-small", "Q5_1"), ("rwkv5-small", "Q8_0"), ("rwkv4-small", "Q4_1"), ("rwkv6-mid", "Q5_1")])
def test_batch_real_head_size(lib, tmp_path, preset, fmt):
    import synthetic_model as sm
    path = str(tmp_path / f"{preset}-{fmt}.bin")
    sm.write_direct(path, preset, fmt, seed=8)
    check_batch(lib, path, n_seq=8, n_steps=5)


@pytest.mark.parametrize("fmt", ["FP32", "FP16", "Q5_1"])
def test_batch_v7_equals_alone_bitwise(lib, fmt):
    """RWKV v7 in a batch context (wkv7 with column t on sequence t's state, v_first per sequence)."""
    check_batch(lib, model_path("7v0-834K", fmt), n_seq=5, n_steps=9)


def test_batch_v7_real_head_size(lib, tmp_path):
    import synthetic_model as sm
    path = str(tmp_path / "rwkv7-small-Q8_0.bin")
    sm.write_direct(path, "rwkv7-small", "Q8_0", seed=8)
    check_batch(lib, path, n_seq=6, n_steps=5)


@pytest.mark.parametrize("preset,fmt,n_seq", [("rwkv6-small", "Q5_1", 16), ("rwkv6-mid", "Q5_1", 24), ("rwkv7-small", "FP16", 16), ("rwkv5-small", "Q4_0", 40)])
def test_large_batches_run_on_the_tensor_cores(lib, tmp_path, preset, fmt, n_seq):
    """From 16 sequences on the layer matrices of a batch pass go through the wgmma kernel (N = sequences padded to 16): per
    sequence the result tracks rwkv_eval of that sequence alone within the bar we hold against the reference for quantised / FP16
    files, and stays there over several steps."""
    import synthetic_model as sm
    path = str(tmp_path / f"{preset}-{fmt}.bin")
    sm.write_direct(path, preset, fmt, seed=8)
    ctx = lib.rwkv_init_from_file(path, 1, 0)
    batch = None
    try:
        n_state, n_logits = lib.rwkv_get_state_buffer_element_count(ctx), lib.rwkv_get_logits_buffer_element_count(ctx)
        n_steps = 6
        prompts = [[(131 * b + 17 * i + 5) % n_logits for i in range(n_steps)] for b in range(n_seq)]
        want = [alone(lib, ctx, p, n_state, n_logits) for p in prompts]
        batch = ctypes.c_void_p(lib.library.rwkv_b200_batch_create(ctx.ptr, n_seq))
        assert batch
        lg = np.zeros(n_logits, np.float32)
        worst = 0.0
        for step in range(n_steps):
            toks = (ctypes.c_uint32 * n_seq)(*[p[step] for p in prompts])
            assert lib.library.rwkv_b200_batch_eval(batch, toks, True)
            for b in range(n_seq):
                assert lib.library.rwkv_b200_batch_get_logits(batch, b, lg.ctypes.data_as(P_F))
                assert np.isfinite(lg).all()
                worst = max(worst, float(np.abs(lg - want[b][0][step]).max()))
        assert worst <= (5e-3 if fmt == "FP16" else 5e-2), (preset, fmt, n_seq, worst)
    finally:
        if batch:
            lib.library.rwkv_free(batch)
        lib.rwkv_free(ctx)


def test_batch_unsupported_and_argument_errors(lib):
    ctx = lib.rwkv_init_from_file(model_path("6v0-3m", "FP32"), 1, 0)
    assert not lib.library.rwkv_b200_batch_create(ctx.ptr, 0)
    assert not lib.library.rwkv_b200_batch_create(ctx.ptr, 100000)
    b = ctypes.c_void_p(lib.library.rwkv_b200_batch_create(ctx.ptr, 2))
    toks = (ctypes.c_uint32 * 2)(1, 100000)
    assert not lib.library.rwkv_b200_batch_eval(b, toks, True)          # token out of range
    buf = np.zeros(lib.rwkv_get_logits_buffer_element_count(ctx), np.float32)
    assert not lib.library.rwkv_b200_batch_get_logits(b, 0, buf.ctypes.data_as(P_F))     # nothing evaluated yet
    assert not lib.library.rwkv_b200_batch_get_logits(b, 5, buf.ctypes.data_as(P_F))
    lib.library.rwkv_free(b)
    lib.rwkv_free(ctx)
