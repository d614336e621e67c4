"""Beam search without a GPU: the host reference (beam_ref.py) against a brute-force enumeration of every sequence up to length 4 over a
toy Markov model, the exported symbols and ctypes prototypes, the refusals that come before any device call, and the resource usage
of the search kernels in the built library."""
import ctypes
import itertools
import os
import re
import subprocess

import numpy as np
import pytest

import beam_ref as br

ERR_ARGS = 1 << 8
HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "rwkv_b200.h")
V, DEPTH = 5, 4


def toy(seed):
    """Root column and transition logits [V][V] with ties (values on a coarse grid) and a -inf entry, and their float32 log-softmax."""
    rng = np.random.default_rng(seed)
    z = np.round(rng.standard_normal((V + 1, V)) * 2) / 2
    z[rng.integers(0, V + 1), rng.integers(0, V)] = -np.inf
    z = z.astype(np.float32)
    m = z.max(axis=1, keepdims=True)
    lp = ((z - m) - np.log(np.exp((z - m).astype(np.float64)).sum(axis=1, keepdims=True))).astype(np.float32)
    return z, lp        # row V is the root's column, row t the column after token t


def toy_candidates(z, lp, width):
    def cands(h):
        row = V if h is None else h
        return [(int(t), float(lp[row, t])) for t in br.top_order(z[row], 2 * width) if np.isfinite(lp[row, t])]
    return cands


def brute(z, lp, width, stops, length_penalty, n_best):
    """Every sequence up to DEPTH tokens, each decided on its own: at step i a sequence is a candidate when its prefix is live and its
    last token is among the prefix's top 2W with a finite lp; it is reached by the walk when fewer than W candidates that rank before
    it are live and the pool, with the stop candidates that rank before it, holds fewer than W; reached, it is live or (stop id)
    finished. The beam slot of a live sequence is the number of live ones that rank before it."""
    live = {(): (0.0, 0)}           # prefix -> (score, slot)
    pool = []
    for i in range(DEPTH):
        cand = {}
        for s in itertools.product(range(V), repeat=i + 1):
            pre, t = s[:-1], s[-1]
            if pre not in live:
                continue
            row = V if not pre else pre[-1]
            top = [int(x) for x in br.top_order(z[row], 2 * width)]
            if t not in top or not np.isfinite(lp[row, t]):
                continue
            cand[s] = (live[pre][0] + float(lp[row, t]), live[pre][1], top.index(t))
        key = {s: (-c[0], c[1], c[2]) for s, c in cand.items()}
        reached, nxt, added = {}, {}, []
        for s in cand:
            before = [o for o in cand if key[o] < key[s]]
            n_live = sum(1 for o in before if o[-1] not in stops)
            n_fin = len(pool) + sum(1 for o in before if o[-1] in stops)
            if n_live < width and n_fin < width:
                reached[s] = (n_live, key[s])
        for s, (slot, k) in sorted(reached.items(), key=lambda e: e[1][1]):
            if s[-1] in stops:
                added.append((cand[s][0], list(s)))
            else:
                nxt[s] = (cand[s][0], slot)
        pool += added
        live = nxt
        if len(pool) == width or not live:
            break
    ordered = sorted(live.items(), key=lambda e: e[1][1])
    return br.results(pool, [(sc, list(s), None) for s, (sc, _) in ordered], length_penalty, n_best)


@pytest.mark.parametrize("width", [1, 2, 3])
@pytest.mark.parametrize("length_penalty", [0.0, 1.0, -0.5])
@pytest.mark.parametrize("stops", [(), (2,), (0, 4)])
def test_reference_matches_brute_force(width, length_penalty, stops):
    for seed in range(12):
        z, lp = toy(seed)
        pool, live, _ = br.search(None, width, DEPTH, set(stops), toy_candidates(z, lp, width), lambda h, t: t)
        got = br.results(pool, live, length_penalty, width)
        want = brute(z, lp, width, set(stops), length_penalty, width)
        assert got == want, (seed, got, want)


def test_width_one_is_greedy():
    """W = 1 without stops: the argmax path (first index among equal logits), whatever the length penalty."""
    for seed in range(12):
        z, lp = toy(seed)
        pool, live, _ = br.search(None, 1, DEPTH, set(), toy_candidates(z, lp, 1), lambda h, t: t)
        row, path = V, []
        for _ in range(DEPTH):
            row = int(np.argmax(z[row]))
            path.append(row)
        assert not pool and live[0][1] == path, seed


def test_walk_ties_go_to_the_lower_beam_then_the_earlier_position():
    taken, finished = br.walk([[(7, -1.0), (8, -2.0)], [(9, -1.0), (3, -2.0)]], [-1.0, -1.0], 3, 0, {3})
    assert taken == [(0, 7, -2.0), (1, 9, -2.0), (0, 8, -3.0)] and finished == []
    taken, finished = br.walk([[(3, -0.5), (8, -2.0)], [(9, -1.0)]], [-1.0, -1.0], 2, 1, {3})
    assert finished == [(0, 3, -1.5)] and taken == []          # the pool filled: the walk stops


# ---- the library without a device ------------------------------------------------------------------------------------------------

NEW = ("rwkv_b200_beam_search", "rwkv_b200_test_beam_step")


def test_symbols_are_exported_and_prototypes_match_the_header(lib):
    P = ctypes.POINTER
    table = {ctypes.c_void_p: "void *", ctypes.c_size_t: "size_t", ctypes.c_float: "float", P(ctypes.c_uint32): "uint32_t *",
             P(ctypes.c_double): "double *", P(ctypes.c_uint8): "uint8_t *"}
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    for name in NEW:
        assert hasattr(lib.library, name), name
        assert getattr(lib.library, name).restype is ctypes.c_bool
    m = re.search(r"RWKV_API\s+bool\s+rwkv_b200_beam_search\s*\(([^)]*)\)\s*;", text)
    want = [" ".join(p.replace("*", " * ").split()[:-1]).replace("const ", "").replace("struct rwkv_context", "void") for p in m.group(1).split(",")]
    got = [table[a] for a in lib.library.rwkv_b200_beam_search.argtypes]
    assert [" ".join(w.split()) for w in want] == got
    fields = re.search(r"struct rwkv_b200_beam_step_args\s*\{(.*?)\};", text, flags=re.S).group(1)
    names = re.findall(r"\*?\s*(\w+)\s*[,;]", fields)
    import rwkv_cpp_b200.shared_library as sl
    assert [f for f, _ in sl.BeamStepArgs._fields_] == names
    r = subprocess.run(["nm", "-D", "--defined-only", lib.path], capture_output=True, text=True)
    if r.returncode == 0:
        for name in NEW:
            assert re.search(r"\bT " + name + r"\b", r.stdout), name


def test_refusals_before_any_device_call(lib):
    lib.rwkv_set_print_errors(None, False)
    assert not lib.library.rwkv_b200_beam_search(None, 4, 1.0, None, 0, 1, None, None, None, None)
    assert lib.rwkv_get_last_error(None) == ERR_ARGS
    import rwkv_cpp_b200.shared_library as sl
    assert not lib.library.rwkv_b200_test_beam_step(None)
    assert lib.rwkv_get_last_error(None) == ERR_ARGS
    z = np.zeros((1, 8), np.float32)
    sc = np.zeros(1, np.float64)
    outs = [np.zeros(4, np.uint32) for _ in range(6)] + [np.zeros(4, np.float64) for _ in range(2)]
    P_U, P_D = ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_double)
    def args(**kw):
        a = sl.BeamStepArgs(z.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), 2, 8, 1, sc.ctypes.data_as(P_D), 0, None, 0,
                            outs[0].ctypes.data_as(P_U), outs[1].ctypes.data_as(P_U), outs[2].ctypes.data_as(P_U), outs[6].ctypes.data_as(P_D),
                            outs[3].ctypes.data_as(P_U), outs[4].ctypes.data_as(P_U), outs[5].ctypes.data_as(P_U), outs[7].ctypes.data_as(P_D))
        for k, v in kw.items():
            setattr(a, k, v)
        return a
    for bad in (dict(width=0), dict(width=11), dict(n_live=3), dict(n_live=0), dict(n_pool=2), dict(n_vocab=65537), dict(n_stop=17),
                dict(n_stop=1), dict(scores_out=None)):
        a = args(**bad)
        assert not lib.library.rwkv_b200_test_beam_step(ctypes.byref(a)), bad
        assert lib.rwkv_get_last_error(None) == ERR_ARGS, bad
    sc[0] = np.inf
    a = args()
    assert not lib.library.rwkv_b200_test_beam_step(ctypes.byref(a)) and lib.rwkv_get_last_error(None) == ERR_ARGS


def test_search_kernels_do_not_spill(lib):
    r = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-res-usage", lib.path], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    lines = r.stdout.splitlines()
    found = 0
    for i, line in enumerate(lines):
        if "beam_step_kernel" in line or "beam_gather_kernel" in line:
            found += 1
            usage = lines[i + 1]
            assert re.search(r"STACK:0\b", usage), (line, usage)
    assert found == 6, found
