"""Device-side generation without a GPU: the generation step's test hook and the two entry points check their arguments before they
touch a device, and the host restatement of the presence / frequency penalty (tests/generate_ref.py) on fixed cases."""
import ctypes
from collections import Counter

import numpy as np

import generate_ref as gr

ARGS = 1 << 8


def step_args(R=3, V=16, **kw):
    keep = dict(logits=np.zeros((R, V), np.float32), max_tokens=np.array([2] * R, np.uint32), temperature=np.ones(R, np.float32),
                top_p=np.ones(R, np.float32), presence_penalty=np.zeros(R, np.float32), frequency_penalty=np.zeros(R, np.float32),
                u=np.full(R * 2, 0.5), stop_ids=None, step=np.zeros(R, np.uint32), frozen=np.zeros(R, np.uint8), counts=np.zeros((R, V), np.uint32),
                tokens=np.zeros(R * 2, np.uint32), next_tokens=np.zeros(R, np.int32), any_active=np.zeros(1, np.uint32))
    sizes = dict(n_rows=R, n_vocab=V, n_stop=0)
    for k, v in kw.items():
        (sizes if k in sizes else keep)[k] = v
    a = gr.StepArgs(**sizes, **{k: (None if v is None else v.ctypes.data) for k, v in keep.items()})
    return a, keep


def test_generate_step_hook_rejects_bad_arguments_without_a_device(lib):
    nan = np.array([1.0, float("nan"), 1.0], np.float32)
    bad_u = np.full(6, 0.5)
    bad_u[3] = 1.0
    cases = [
        dict(n_rows=0), dict(n_rows=257), dict(n_vocab=0), dict(n_vocab=65537), dict(logits=None), dict(step=None), dict(frozen=None),
        dict(counts=None), dict(tokens=None), dict(next_tokens=None), dict(any_active=None), dict(u=None), dict(max_tokens=None),
        dict(temperature=np.array([1.0, -1.0, 1.0], np.float32)), dict(top_p=np.array([1.0, 1.5, 1.0], np.float32)), dict(top_p=nan),
        dict(presence_penalty=nan), dict(frequency_penalty=np.array([0.0, 0.0, float("inf")], np.float32)), dict(u=bad_u),
        dict(stop_ids=np.array([16], np.uint32), n_stop=1), dict(stop_ids=np.arange(17, dtype=np.uint32), n_stop=17), dict(n_stop=1),
        dict(max_tokens=np.array([0, 0, 0], np.uint32)), dict(max_tokens=np.array([4097, 1, 1], np.uint32), u=np.full(3 * 4097, 0.5)),
        dict(step=np.array([0, 3, 0], np.uint32)),
    ]
    for i, kw in enumerate(cases):
        a, keep = step_args(**kw)
        assert not lib.library.rwkv_b200_test_generate_step(ctypes.byref(a)), (i, kw)
        assert lib.rwkv_get_last_error(None) == ARGS, (i, kw)
    assert not lib.library.rwkv_b200_test_generate_step(None)
    assert lib.rwkv_get_last_error(None) == ARGS


def test_generate_entry_points_reject_a_null_context(lib):
    L = lib.library
    n = ctypes.c_size_t(0)
    toks = (ctypes.c_uint32 * 4)()
    u = (ctypes.c_double * 4)(0.5, 0.5, 0.5, 0.5)
    assert not L.rwkv_b200_generate(None, 4, 1.0, 1.0, 0.0, 0.0, False, u, None, 0, toks, ctypes.byref(n))
    assert lib.rwkv_get_last_error(None) == ARGS
    ng = (ctypes.c_uint32 * 1)()
    assert not L.rwkv_b200_batch_generate(None, (ctypes.c_uint32 * 1)(4), None, None, None, None, None, u, None, 0, toks, ng)
    assert lib.rwkv_get_last_error(None) == ARGS


def test_penalty_bias_fixed_cases():
    counts = Counter({3: 1, 7: 4, 9: 0})
    assert gr.penalty_bias(counts, 0.2, 0.2) == {3: float(-(np.float32(0.2) + np.float32(0.2))), 7: float(-(np.float32(0.2) + np.float32(0.8)))}
    assert gr.penalty_bias(counts, 0.0, 0.0) == {3: -0.0, 7: -0.0}
    assert gr.penalty_bias(Counter(), 1.0, 1.0) == {}
    # the multiply is rounded on its own, not fused with the add
    p, f, c = np.float32(0.1), np.float32(0.3), 3
    b = gr.penalty_bias({5: c}, p, f)[5]
    assert np.float32(b) == -(p + np.float32(np.float32(c) * f))
