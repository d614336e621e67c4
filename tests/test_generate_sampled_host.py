"""Generation with a per-sequence sampler without a GPU: the float64 rules of tests/sampler_ref.py (ties at the k-th value, the cases
that keep everything or only the top tie group, independence of order), the ctypes mirror of struct rwkv_b200_sampler against the
header, the exports, and every refusal of the new entry points that is decided before a device is touched."""
import ctypes
import itertools
import os
import re
import subprocess

import numpy as np
import pytest

import generate_ref as gr
from sampler_ref import kept_mask, sampled_probs64, sampler_bias
from sampling_oracle import probs64

ARGS = 1 << 8
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("rwkv_b200_generate_sampled", "rwkv_b200_batch_generate_sampled", "rwkv_b200_test_generate_step_sampled")


# ---- the float64 rules -----------------------------------------------------------------------------------------------------------

def test_ties_at_the_kth_value_are_all_kept():
    z = np.array([3.0, 2.0, 2.0, 2.0, 1.0, 0.0], np.float32)
    p = probs64(z, 1.0, 1.0)
    assert kept_mask(p, 1.0, top_k=2).tolist() == [True, True, True, True, False, False]
    assert kept_mask(p, 1.0, top_k=1).tolist() == [True] + [False] * 5
    q = sampled_probs64(z, 1.0, 1.0, top_k=3)
    assert (q[:4] > 0).all() and (q[4:] == 0).all() and q[1] == q[2] == q[3]


def test_k_at_or_above_the_positive_count_keeps_everything():
    z = np.array([1.0, 0.5, -np.inf, 0.0, -np.inf], np.float32)
    for k in (3, 4, 5):
        assert np.array_equal(sampled_probs64(z, 0.7, 1.0, top_k=k), probs64(z, 0.7, 1.0))


def test_min_p_one_keeps_only_the_top_tie_group():
    z = np.array([0.0, 2.0, 1.9, 2.0, -1.0], np.float32)
    q = sampled_probs64(z, 1.3, 1.0, min_p=1.0)
    assert (q > 0).tolist() == [False, True, False, True, False] and q[1] == q[3] == 0.5


def test_filters_off_and_temperature_zero_are_the_plain_draw():
    rng = np.random.RandomState(0)
    z = rng.standard_normal(50).astype(np.float32)
    assert np.array_equal(sampled_probs64(z, 0.8, 0.9), probs64(z, 0.8, 0.9))
    assert np.array_equal(sampled_probs64(z, 0.0, 0.5, top_k=3, min_p=0.5), probs64(z, 0.0, 0.5))


def test_the_three_filters_commute():
    """Each filter applied on its own to the same p, in every order, gives the kept set of all three at once."""
    rng = np.random.RandomState(1)
    for _ in range(50):
        z = np.round(rng.standard_normal(40) * 2, 1).astype(np.float32)      # rounding makes ties
        p = probs64(z, 1.0, 1.0)
        top_p, k, mp = rng.choice([0.3, 0.8, 1.0]), int(rng.randint(0, 41)), rng.choice([0.0, 0.05, 0.5])
        one = {"p": kept_mask(p, top_p), "k": kept_mask(p, 1.0, top_k=k), "m": kept_mask(p, 1.0, min_p=mp)}
        want = kept_mask(p, top_p, k, mp)
        for order in itertools.permutations("pkm"):
            got = np.ones(p.size, bool)
            for f in order:
                got &= one[f]
            assert np.array_equal(got, want)
        assert want[np.argmax(p)]


def test_bias_entries_follow_rule_one():
    counts = {1: 2, 2: 1, 4: 3}
    user = {0: 1.5, 1: -0.25, 3: float("-inf"), 4: 2.0}
    allowed = np.array([True, True, True, True, False, True])
    got = sampler_bias(counts, 0.3, 0.2, user, allowed)
    pen = lambda c: np.float32(np.float32(0.3) + np.float32(np.float32(c) * np.float32(0.2)))
    assert got[0] == np.float32(1.5)                                        # uncounted with an entry: the entry
    assert got[1] == np.float32(np.float32(-0.25) - pen(2))                 # counted with an entry: one more rounding
    assert got[2] == -pen(1)                                                # counted without one: as today
    assert got[3] == float("-inf")
    assert got[4] == float("-inf")                                          # not allowed: -inf whatever the count and entry
    assert 5 not in got


# ---- the library -----------------------------------------------------------------------------------------------------------------

def test_sampled_symbols_are_exported_and_declared(lib):
    with open(os.path.join(ROOT, "include", "rwkv_b200.h")) as f:
        header = f.read()
    assert "#define RWKV_B200_LOGIT_BIAS_MAX 1024" in header
    for name in NAMES:
        assert hasattr(lib.library, name), name
        assert getattr(lib.library, name).argtypes is not None, name
        assert re.search(r"RWKV_API [^;]*\b%s\(" % name, header), name


def test_ctypes_sampler_matches_the_header(pkg, tmp_path):
    """Field offsets and size of struct rwkv_b200_sampler from a probe compiled against the header."""
    import rwkv_cpp_b200.shared_library as sl
    fields = [f for f, _ in sl.Sampler._fields_]
    src = tmp_path / "probe.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "rwkv_b200.h"\nint main(void) {\n' +
                   "".join('    printf("%%zu\\n", offsetof(struct rwkv_b200_sampler, %s));\n' % f for f in fields) +
                   '    printf("%zu\\n", sizeof(struct rwkv_b200_sampler));\n    return 0;\n}\n')
    exe = tmp_path / "probe"
    cc = "gcc" if subprocess.run(["which", "gcc"], capture_output=True).returncode == 0 else "g++"
    r = subprocess.run([cc, "-x", "c" if cc == "gcc" else "c++", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [getattr(sl.Sampler, f).offset for f in fields] + [ctypes.sizeof(sl.Sampler)]


def test_sampled_entry_points_reject_a_null_context(lib, pkg):
    import rwkv_cpp_b200.shared_library as sl
    L = lib.library
    calls = []
    fn = sl.RWKV_TOKEN_FN(lambda user, seq, idx, tok: calls.append((seq, idx, tok)) or 0)
    n = ctypes.c_size_t(0)
    toks = (ctypes.c_uint32 * 4)()
    u = (ctypes.c_double * 4)(0.5, 0.5, 0.5, 0.5)
    smp = sl.Sampler(temperature=1.0, top_p=1.0, top_k=5)
    for on_token in (fn, sl.RWKV_TOKEN_FN()):
        for s in (ctypes.byref(smp), None):
            assert not L.rwkv_b200_generate_sampled(None, s, None, None, 4, False, u, None, 0, on_token, None, toks, ctypes.byref(n), None)
            assert lib.rwkv_get_last_error(None) == ARGS
            ng = (ctypes.c_uint32 * 1)()
            assert not L.rwkv_b200_batch_generate_sampled(None, s, None, None, (ctypes.c_uint32 * 1)(4), None, u, None, 0, on_token, None, toks, ng, None)
            assert lib.rwkv_get_last_error(None) == ARGS
    assert calls == []


def hook_args(V, rows=1):
    logits = np.zeros((rows, V), np.float32)
    keep = dict(logits=logits, mt=np.ones(rows, np.uint32), st=np.zeros(rows, np.uint32), fr=np.zeros(rows, np.uint8), cnt=np.zeros((rows, V), np.uint32),
                tk=np.zeros(rows, np.uint32), nx=np.zeros(rows, np.int32), u=np.full(rows, 0.5), act=ctypes.c_uint32(0))
    a = gr.StepArgs(logits=logits.ctypes.data, n_rows=rows, n_vocab=V, max_tokens=keep["mt"].ctypes.data, temperature=None, top_p=None,
                    presence_penalty=None, frequency_penalty=None, u=keep["u"].ctypes.data, stop_ids=None, n_stop=0, step=keep["st"].ctypes.data,
                    frozen=keep["fr"].ctypes.data, counts=keep["cnt"].ctypes.data, tokens=keep["tk"].ctypes.data, next_tokens=keep["nx"].ctypes.data,
                    any_active=ctypes.addressof(keep["act"]))
    return a, keep


def test_step_hook_refuses_bad_samplers_before_the_device(lib, pkg):
    """Every sampler refusal of the contract, decided on the host: NULL samplers, per-row parameters not NULL, top_k > n_vocab, min_p
    NaN or outside [0, 1], too many entries or NULL arrays, a duplicate id, an id >= n_vocab, a NaN or +inf value."""
    import rwkv_cpp_b200.shared_library as sl
    L = lib.library
    V = 8
    a, keep = hook_args(V, 2)
    ids_ok = np.array([1, 3], np.uint32)
    vals_ok = np.array([0.5, -np.inf], np.float32)

    def smp(**kw):
        base = dict(temperature=1.0, top_p=1.0, top_k=0, min_p=0.0, presence_penalty=0.0, frequency_penalty=0.0, n_bias=0, bias_ids=None, bias_values=None)
        base.update(kw)
        return sl.Sampler(**base)

    arrays = []

    def bias(ids, vals):
        ids, vals = np.asarray(ids, np.uint32), np.asarray(vals, np.float32)
        arrays.append((ids, vals))
        return dict(n_bias=len(ids), bias_ids=ids.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32)), bias_values=vals.ctypes.data_as(ctypes.POINTER(ctypes.c_float)))

    assert not L.rwkv_b200_test_generate_step_sampled(ctypes.byref(a), None, None, 0, None, None)
    assert lib.rwkv_get_last_error(None) == ARGS
    ones = np.ones(2, np.float32)
    with_t = gr.StepArgs.from_buffer_copy(a)
    with_t.temperature = ones.ctypes.data
    good = (sl.Sampler * 2)(smp(), smp(**bias(ids_ok, vals_ok)))
    assert not L.rwkv_b200_test_generate_step_sampled(ctypes.byref(with_t), good, None, 0, None, None)
    assert lib.rwkv_get_last_error(None) == ARGS
    big = np.arange(1025, dtype=np.uint32) % V
    bad = [smp(top_k=V + 1), smp(min_p=float("nan")), smp(min_p=-0.01), smp(min_p=1.01), smp(n_bias=1), smp(**bias(big, np.zeros(1025))),
           smp(**bias([2, 5, 2], [0, 0, 0])), smp(**bias([V], [0])), smp(**bias([1], [float("nan")])), smp(**bias([1], [float("inf")]))]
    for s in bad:
        rows = (sl.Sampler * 2)(smp(), s)
        before = {k: v.copy() for k, v in keep.items() if isinstance(v, np.ndarray)}
        assert not L.rwkv_b200_test_generate_step_sampled(ctypes.byref(a), rows, None, 0, None, None)
        assert lib.rwkv_get_last_error(None) == ARGS
        assert all(np.array_equal(before[k], keep[k]) for k in before)
