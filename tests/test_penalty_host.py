"""Penalty decay, weights and counts without a GPU: the exported prototypes against include/rwkv_b200.h, every refusal the new step
hook and the entry points decide before they touch a device, the buffers the Python wrappers refuse, and the float32 restatement of
the penalty rules (penalty_ref.py) against hand-worked cases."""
import ctypes
import os
import re

import numpy as np
import pytest

import generate_ref as gr
import penalty_ref as pr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = open(os.path.join(ROOT, "include", "rwkv_b200.h")).read()
ERR_ARGS, ERR_CTX_UNSUPPORTED = 1 << 8, (6 << 8) | 9
NAMES = ("rwkv_b200_set_penalty_decay", "rwkv_b200_set_penalty_weights", "rwkv_b200_get_penalty_counts", "rwkv_b200_set_penalty_counts",
         "rwkv_b200_test_generate_step_penalty")
P_F = ctypes.POINTER(ctypes.c_float)


def test_prototypes_match_the_header(lib):
    for name in NAMES:
        assert hasattr(lib.library, name), name
        m = re.search(r"RWKV_API bool " + name + r"\(([^;]*)\);", HDR, re.S)
        assert m, name
        assert len(m.group(1).split(",")) == len(getattr(lib.library, name).argtypes), name


def test_entry_points_refuse_a_null_context(lib):
    L = lib.library
    buf = np.zeros(4, np.float32)
    for call in (lambda: L.rwkv_b200_set_penalty_decay(None, 0, 0.5), lambda: L.rwkv_b200_set_penalty_weights(None, None),
                 lambda: L.rwkv_b200_get_penalty_counts(None, 0, buf.ctypes.data_as(P_F)),
                 lambda: L.rwkv_b200_set_penalty_counts(None, 0, buf.ctypes.data_as(P_F))):
        assert not call()
        assert lib.rwkv_get_last_error(None) == ERR_ARGS


# ---- the step hook's refusals ------------------------------------------------------------------------------------------------------

R, V = 2, 8


def step_call(lib, counts=None, decay=None, weights=None, int_counts=False):
    """rwkv_b200_test_generate_step_penalty (plain family) on R x V logits with the given tables; returns (ok, error flags)."""
    keep = dict(lg=np.zeros((R, V), np.float32), mt=np.full(R, 1, np.uint32), t=np.ones(R, np.float32), p=np.ones(R, np.float32),
                z=np.zeros(R, np.float32), u=np.full(R, 0.5), st=np.zeros(R, np.uint32), fr=np.zeros(R, np.uint8), ic=np.zeros((R, V), np.uint32),
                tk=np.zeros(R, np.uint32), nx=np.zeros(R, np.int32), act=np.zeros(1, np.uint32))
    a = gr.StepArgs(logits=keep["lg"].ctypes.data, n_rows=R, n_vocab=V, max_tokens=keep["mt"].ctypes.data, temperature=keep["t"].ctypes.data,
                    top_p=keep["p"].ctypes.data, presence_penalty=keep["z"].ctypes.data, frequency_penalty=keep["z"].ctypes.data, u=keep["u"].ctypes.data,
                    stop_ids=None, n_stop=0, step=keep["st"].ctypes.data, frozen=keep["fr"].ctypes.data,
                    counts=keep["ic"].ctypes.data if int_counts else None, tokens=keep["tk"].ctypes.data, next_tokens=keep["nx"].ctypes.data,
                    any_active=keep["act"].ctypes.data)
    counts = np.zeros((R, V), np.float32) if counts is None else np.ascontiguousarray(counts, np.float32)
    decay = np.ones(R, np.float32) if decay is None else np.ascontiguousarray(decay, np.float32)
    w = None if weights is None else np.ascontiguousarray(weights, np.float32)
    ok = lib.library.rwkv_b200_test_generate_step_penalty(ctypes.byref(a), 0, None, None, 0, None, None, counts.ctypes.data_as(P_F),
                                                          decay.ctypes.data_as(P_F), None if w is None else w.ctypes.data_as(P_F))
    return ok, lib.rwkv_get_last_error(None)


def with_entry(shape, value, at):
    x = np.ones(shape, np.float32) if len(shape) == 1 else np.zeros(shape, np.float32)
    x[at] = value
    return x


@pytest.mark.parametrize("case", ["decay 0", "decay above 1", "decay NaN", "decay -inf", "count negative", "count NaN", "count inf",
                                  "weight negative", "weight NaN", "weight inf", "integer counts too"])
def test_step_hook_refuses_bad_tables_before_the_device(lib, case):
    kw = {"decay 0": dict(decay=[1.0, 0.0]), "decay above 1": dict(decay=[1.0000001, 1.0]), "decay NaN": dict(decay=[np.nan, 1.0]),
          "decay -inf": dict(decay=[-np.inf, 1.0]),
          "count negative": dict(counts=with_entry((R, V), -1e-30, (1, 7))), "count NaN": dict(counts=with_entry((R, V), np.nan, (0, 0))),
          "count inf": dict(counts=with_entry((R, V), np.inf, (1, 3))),
          "weight negative": dict(weights=with_entry((V,), -0.5, 2)), "weight NaN": dict(weights=with_entry((V,), np.nan, 0)),
          "weight inf": dict(weights=with_entry((V,), np.inf, 7)), "integer counts too": dict(int_counts=True)}[case]
    ok, err = step_call(lib, **kw)
    assert not ok and err == ERR_ARGS, (case, hex(err))


def test_step_hook_accepts_edge_values_up_to_the_device(lib):
    """Decay 1 and a denormal, zero weights, zero and huge counts pass the checks: what stops the call on a machine without a GPU is
    the missing device (with one, the step runs)."""
    counts = with_entry((R, V), 3e38, (0, 1))
    counts[1, 2] = 1e-45
    ok, err = step_call(lib, counts=counts, decay=[1.0, 1e-45], weights=np.zeros(V, np.float32))
    assert ok or err == ERR_CTX_UNSUPPORTED, hex(err)


# ---- the wrappers ---------------------------------------------------------------------------------------------------------------

class FakeLib:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def f(*args):
            self.calls.append((name, args))
            return name.endswith("_logits_len") and 8 or True
        return f


def fake():
    import rwkv_cpp_b200.shared_library as sl
    w = sl.RWKVSharedLibrary.__new__(sl.RWKVSharedLibrary)
    w.library = FakeLib()
    return w, sl.RWKVContext(ctypes.c_void_p(1234))


def test_wrappers_build_the_arguments():
    w, ctx = fake()
    w.rwkv_b200_set_penalty_decay(ctx, 3, 0.996)
    name, args = w.library.calls[-1]
    assert name == "rwkv_b200_set_penalty_decay" and args[1] == 3 and abs(args[2].value - 0.996) < 1e-7
    w.rwkv_b200_set_penalty_weights(ctx, None)
    name, args = w.library.calls[-1]
    assert name == "rwkv_b200_set_penalty_weights" and not ctypes.cast(args[1], ctypes.c_void_p).value
    wt = np.ones(8, np.float32)
    w.rwkv_b200_set_penalty_weights(ctx, wt)
    assert ctypes.cast(w.library.calls[-1][1][1], ctypes.c_void_p).value == wt.ctypes.data
    out = w.rwkv_b200_get_penalty_counts(ctx, 2)
    name, args = w.library.calls[-1]
    assert name == "rwkv_b200_get_penalty_counts" and args[1] == 2 and out.shape == (8,) and out.dtype == np.float32
    assert ctypes.cast(args[2], ctypes.c_void_p).value == out.ctypes.data
    mine = np.zeros(9, np.float32)
    assert w.rwkv_b200_get_penalty_counts(ctx, 0, out=mine) is mine
    c = np.arange(8, dtype=np.float32)
    w.rwkv_b200_set_penalty_counts(ctx, 1, c)
    name, args = w.library.calls[-1]
    assert name == "rwkv_b200_set_penalty_counts" and args[1] == 1 and ctypes.cast(args[2], ctypes.c_void_p).value == c.ctypes.data


@pytest.mark.parametrize("bad", ["float64", "short", "strided", "list", "float16-tensor", "short-tensor", "strided-tensor"])
@pytest.mark.parametrize("call", ["weights", "get", "set"])
def test_wrappers_refuse_buffers_a_table_does_not_fit(bad, call):
    """A buffer the library would read or write past (too short, another dtype, not contiguous, not an array) is refused before the call."""
    import torch
    w, ctx = fake()
    buf = {"float64": np.ones(8, np.float64), "short": np.ones(7, np.float32), "strided": np.ones(16, np.float32)[::2], "list": [1.0] * 8,
           "float16-tensor": torch.ones(8, dtype=torch.float16), "short-tensor": torch.ones(7, dtype=torch.float32),
           "strided-tensor": torch.ones(16, dtype=torch.float32)[::2]}[bad]
    fn = {"weights": lambda b: w.rwkv_b200_set_penalty_weights(ctx, b), "get": lambda b: w.rwkv_b200_get_penalty_counts(ctx, 0, out=b),
          "set": lambda b: w.rwkv_b200_set_penalty_counts(ctx, 0, b)}[call]
    with pytest.raises(ValueError):
        fn(buf)
    assert not any("penalty" in name for name, _ in w.library.calls)
    for ok in (np.ones(9, np.float32)[1:], torch.ones(8, dtype=torch.float32)):     # any float alignment, any length >= n_vocab
        fn(ok)


# ---- the float32 restatement against hand-worked cases --------------------------------------------------------------------------

def test_decay_comes_before_the_add():
    c = np.array([0.0, 1.0, 0.5, 4.0], np.float32)
    got = pr.update(c, 2, 0.5, np.array([1.0, 1.0, 2.0, 1.0], np.float32))
    assert got.tolist() == [0.0, 0.5, 2.25, 2.0]        # 0.5 * 0.5 + 2, not (0.5 + 2) * 0.5
    assert c.tolist() == [0.0, 1.0, 0.5, 4.0]            # a new array


def test_weight_zero_is_never_counted():
    c = np.zeros(4, np.float32)
    w = np.array([1.0, 0.0, 1.0, 1.0], np.float32)
    for tok in (1, 1, 1):
        c = pr.update(c, tok, 0.996, w)
    assert not c.any()
    assert pr.penalty_bias(c, 0.5, 0.5) == {}            # no presence penalty either
    c = pr.update(c, 2, 0.996, w)
    assert pr.penalty_bias(c, 0.5, 0.25) == {2: -0.75}


def test_a_count_that_underflows_is_no_longer_counted():
    tiny = np.float32(2.0 ** -149)                      # the smallest denormal: times 0.5 rounds (to even) to 0
    c = np.array([tiny, 2.0 ** -126, 0.0], np.float32)
    got = pr.update(c, 2, 0.5)
    assert got[0] == 0.0 and got[1] == np.float32(2.0 ** -127) and got[2] == 1.0
    assert sorted(pr.penalty_bias(got, 0.1, 0.1)) == [1, 2]


def test_decay_one_gives_integer_counts_and_the_integer_bias():
    rng = np.random.RandomState(3)
    toks = rng.randint(0, 6, size=200)
    c = np.zeros(6, np.float32)
    from collections import Counter
    ints = Counter()
    for t in toks:
        c = pr.update(c, int(t), 1.0)
        ints[int(t)] += 1
    assert c.tolist() == [float(ints[n]) for n in range(6)]
    assert pr.penalty_bias(c, 0.3, 0.2) == gr.penalty_bias(ints, 0.3, 0.2)


def test_counts_stop_at_two_to_the_24():
    c = np.array([2.0 ** 24], np.float32)
    assert pr.update(c, 0, 1.0)[0] == 2.0 ** 24


def test_bias_rounds_the_multiply_and_the_add_separately():
    c = np.array([0.0, 3.1, 0.7], np.float32)
    p, f = np.float32(0.1), np.float32(0.3)
    assert pr.penalty_bias(c, 0.1, 0.3) == {1: float(-(p + np.float32(np.float32(3.1) * f))), 2: float(-(p + np.float32(np.float32(0.7) * f)))}
    allowed = np.array([True, False, True])
    assert pr.penalty_bias(c, 0.1, 0.3, allowed)[1] == float("-inf")


def test_a_decayed_sequence_matches_the_closed_form_in_float32():
    """Token 0 every step under d: c_k = fl(fl(c_{k-1} * d) + 1), which stays below the geometric limit 1 / (1 - d)."""
    d = np.float32(0.996)
    c = np.zeros(2, np.float32)
    want = np.float32(0)
    for _ in range(3000):
        c = pr.update(c, 0, float(d))
        want = np.float32(np.float32(want * d) + np.float32(1))
    assert c[0] == want and c[1] == 0 and want < 1 / (1 - 0.996)
