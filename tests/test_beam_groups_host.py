"""Grouped beam search without a GPU: the lockstep reference (beam_groups_ref.py) against a per-group brute-force enumeration over toy
Markov models, the exported symbols and ctypes prototypes, the refusals that come before any device call, and the resource usage of
the grouped search kernels in the built library."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import beam_groups_ref as bg
import beam_ref as br
import test_beam_host as tbh

ERR_ARGS = 1 << 8
HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "rwkv_b200.h")
V = tbh.V

# (max_tokens, length penalty, seed) per group: different roots (toy models), lengths 0 / 1 / 4 and penalties per group
LAYOUTS = {
    1: [(4, 1.0, 0)],
    2: [(4, -0.5, 1), (1, 1.0, 2)],
    3: [(0, 1.0, 3), (4, 0.0, 4), (1, -0.5, 5)],
}


def toy_groups(seeds, width):
    """Handles are (group, row); candidates come from group g's own toy model."""
    models = [tbh.toy(s) for s in seeds]

    def cands(h):
        g, row = h
        z, lp = models[g]
        return tbh.toy_candidates(z, lp, width)(None if row is None else row)
    return models, cands


@pytest.mark.parametrize("G", [1, 2, 3])
@pytest.mark.parametrize("width", [1, 2, 3])
@pytest.mark.parametrize("stops", [(), (2,), (0, 4)])
def test_lockstep_reference_matches_per_group_brute_force(monkeypatch, G, width, stops):
    for base in range(6):
        layout = LAYOUTS[G]
        seeds = [s + 10 * base for _, _, s in layout]
        max_tokens = [m for m, _, _ in layout]
        penalties = [p for _, p, _ in layout]
        models, cands = toy_groups(seeds, width)
        found = bg.search_groups([(g, None) for g in range(G)], width, max_tokens, set(stops), cands,
                                 bg.one_by_one(lambda h, t: (h[0], t)))
        got = bg.results_groups(found, penalties, width)
        for g in range(G):
            if max_tokens[g] == 0:
                assert got[g] == [] and found[g] == ([], [], []), (base, g)
                continue
            monkeypatch.setattr(tbh, "DEPTH", max_tokens[g])
            want = tbh.brute(*models[g], width, set(stops), penalties[g], width)
            assert got[g] == want, (base, g, got[g], want)


def test_a_group_that_ends_early_stops_stepping_while_others_go_on():
    """Group 0 fills its pool at the first step (every candidate a stop id); group 1 runs all four steps. advance_all sees group 0
    only at step 0, and then only with the beams it took (none)."""
    width = 2
    models, cands = toy_groups([7, 8], width)
    z0 = models[0][0]
    stops = set(int(t) for t in br.top_order(z0[V], V))     # every id of group 0's root ends a hypothesis
    seen = []

    def advance_all(moves):
        seen.append([None if m is None else len(m) for m in moves])
        return [None if m is None else [(h[0], t) for h, t in m] for m in moves]
    found = bg.search_groups([(0, None), (1, None)], width, [4, 4], stops, cands, advance_all)
    assert len(found[0][0]) == width and found[0][1] == []
    assert seen[0][0] == 0 and all(s[0] is None for s in seen[1:]), seen
    assert all(s[1] is not None for s in seen)


def test_one_group_is_beam_ref_search():
    for seed in range(6):
        z, lp = tbh.toy(seed)
        pool, live, _ = br.search(None, 3, tbh.DEPTH, {1}, tbh.toy_candidates(z, lp, 3), lambda h, t: t)
        found = bg.search_groups([None], 3, [tbh.DEPTH], {1}, tbh.toy_candidates(z, lp, 3), bg.one_by_one(lambda h, t: t))
        assert found[0][0] == pool and [(s, t) for s, t, _ in found[0][1]] == [(s, t) for s, t, _ in live], seed


# ---- the library without a device ------------------------------------------------------------------------------------------------

NEW = ("rwkv_b200_beam_search_groups", "rwkv_b200_test_beam_step_groups")


def test_symbols_are_exported_and_prototypes_match_the_header(lib):
    P = ctypes.POINTER
    import rwkv_cpp_b200.shared_library as sl
    table = {ctypes.c_void_p: "void *", ctypes.c_size_t: "size_t", ctypes.c_float: "float", P(ctypes.c_uint32): "uint32_t *",
             P(ctypes.c_float): "float *", P(ctypes.c_double): "double *", P(ctypes.c_uint8): "uint8_t *",
             P(sl.BeamStepArgs): "struct rwkv_b200_beam_step_args *"}
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    for name in NEW:
        assert hasattr(lib.library, name), name
        assert getattr(lib.library, name).restype is ctypes.c_bool
        m = re.search(r"RWKV_API\s+bool\s+" + name + r"\s*\(([^)]*)\)\s*;", text)
        want = [" ".join(p.replace("*", " * ").split()[:-1]).replace("const ", "").replace("struct rwkv_context", "void") for p in m.group(1).split(",")]
        got = [table[a] for a in getattr(lib.library, name).argtypes]
        assert [" ".join(w.split()) for w in want] == got, name
    r = subprocess.run(["nm", "-D", "--defined-only", lib.path], capture_output=True, text=True)
    if r.returncode == 0:
        for name in NEW:
            assert re.search(r"\bT " + name + r"\b", r.stdout), name


def step_args(n_live=1, **kw):
    import rwkv_cpp_b200.shared_library as sl
    P_F, P_U, P_D = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_double)
    keep = [np.zeros((max(n_live, 1), 8), np.float32), np.zeros(max(n_live, 1), np.float64)]
    keep += [np.zeros(4, np.uint32) for _ in range(6)] + [np.zeros(4, np.float64) for _ in range(2)]
    a = sl.BeamStepArgs(keep[0].ctypes.data_as(P_F), 2, 8, n_live, keep[1].ctypes.data_as(P_D), 0, None, 0,
                        keep[2].ctypes.data_as(P_U), keep[3].ctypes.data_as(P_U), keep[4].ctypes.data_as(P_U), keep[8].ctypes.data_as(P_D),
                        keep[5].ctypes.data_as(P_U), keep[6].ctypes.data_as(P_U), keep[7].ctypes.data_as(P_U), keep[9].ctypes.data_as(P_D))
    for k, v in kw.items():
        setattr(a, k, v)
    a._keep = keep
    return a


def test_refusals_before_any_device_call(lib):
    import rwkv_cpp_b200.shared_library as sl
    lib.rwkv_set_print_errors(None, False)
    mt, lp = (ctypes.c_uint32 * 2)(4, 4), (ctypes.c_float * 2)(1.0, 1.0)
    assert not lib.library.rwkv_b200_beam_search_groups(None, 2, mt, lp, None, 0, 1, None, None, None, None)
    assert lib.rwkv_get_last_error(None) == ERR_ARGS
    assert not lib.library.rwkv_b200_test_beam_step_groups(None, 1)
    assert lib.rwkv_get_last_error(None) == ERR_ARGS
    good = step_args()
    cases = [([good], 0, "no groups"), ([good, step_args(width=3)], 2, "widths differ"), ([good, step_args(n_vocab=9)], 2, "n_vocab differs"),
             ([good, step_args(n_live=3)], 2, "n_live above the width"), ([good, step_args(n_pool=3)], 2, "n_pool above the width"),
             ([step_args(width=11)], 1, "width 11"), ([step_args(n_vocab=65537)], 1, "n_vocab 65537"), ([good, step_args(n_stop=17)], 2, "17 stops"),
             ([good, step_args(n_stop=1)], 2, "NULL stop ids"), ([good, step_args(scores_out=None)], 2, "NULL output"),
             ([good, step_args(logits=None)], 2, "NULL logits of a running group")]
    for groups, G, what in cases:
        arr = (sl.BeamStepArgs * max(1, len(groups)))(*groups)
        assert not lib.library.rwkv_b200_test_beam_step_groups(arr, G), what
        assert lib.rwkv_get_last_error(None) == ERR_ARGS, what
    bad = step_args()
    bad._keep[1][0] = np.nan
    arr = (sl.BeamStepArgs * 2)(good, bad)
    assert not lib.library.rwkv_b200_test_beam_step_groups(arr, 2) and lib.rwkv_get_last_error(None) == ERR_ARGS


def test_grouped_kernels_do_not_spill(lib):
    r = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-res-usage", lib.path], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    lines = r.stdout.splitlines()
    found = {}
    for i, line in enumerate(lines):
        m = re.search(r"beam_(step|gather|restore)_kernel(ILi(\d+)E)?", line)
        if m and "Function" in line:
            found[(m.group(1), m.group(3))] = lines[i + 1]
    want = {("step", p) for p in ("1", "4", "16", "50", "64")} | {("gather", None), ("restore", None)}
    assert set(found) == want, sorted(found)
    for key, usage in found.items():
        assert re.search(r"STACK:0\b", usage), (key, usage)
