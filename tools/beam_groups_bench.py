"""What many beam searches cost in one grouped call against the same searches run one after another (DESIGN.md 6.8.1). Measurement aid,
not a bench line.

Workload: the synthetic RWKV-6 7B shape at Q5_1 (bench.py's rwkv6-7b:Q5_1 file), width W = 4, 64 tokens without stop ids, G = 1, 2, 4,
8 and 16 searches. Legs, ms per call (one call = all G searches):
  grouped   rwkv_b200_beam_search_groups(G groups, max_tokens 64, length_penalty 1) on a batch context of 4 G sequences: one graph
            launch
  serial    G x rwkv_b200_beam_search(max_tokens 64, length_penalty 1) on a batch context of 4 sequences
  G4/grouped_no_tc   the G = 4 grouped call with rwkv_b200_set_tensor_cores(batch, false)
The legs alternate within every round; the median over the rounds with min / max, per call, per step (the 64 steps of one search) and
as hypotheses per second (G * W * 64 beam-tokens evaluated per call). The card's name and power limit are read in the same run.

    python tools/beam_groups_bench.py [--rounds 5] [--out FILE.json]
"""
import argparse
import ctypes
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import __graft_entry__  # noqa: E402
import bench  # noqa: E402
from ragged_batch_bench import card  # noqa: E402

U32 = ctypes.c_uint32
N, W, GROUPS = 64, 4, (1, 2, 4, 8, 16)


def arr(a, ct):
    return np.ascontiguousarray(a).ctypes.data_as(ctypes.POINTER(ct))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    pkg = __graft_entry__.load_package()
    lib = pkg.load_rwkv_shared_library()
    L = lib.library
    path, _ = bench.workload_file("rwkv6-7b:Q5_1")
    ctx = lib.rwkv_b200_init_from_file_ex(path, 0, 0, -1)
    V = lib.rwkv_get_logits_buffer_element_count(ctx)
    owned = []

    def batch(n, tensor_cores=True):
        b = ctypes.c_void_p(L.rwkv_b200_batch_create(ctx.ptr, n))
        assert b.value
        owned.append(b)
        if not tensor_cores:
            L.rwkv_b200_set_tensor_cores(b, False)
        assert L.rwkv_b200_batch_eval(b, (U32 * n)(*[(7919 * i + 11) % V for i in range(n)]), True)
        return b

    single = batch(W)
    toks1, lens1, scores1 = np.zeros(W * N, np.uint32), np.zeros(W, np.uint32), np.zeros(W, np.float64)

    def serial(G):
        def run():
            for _ in range(G):
                assert L.rwkv_b200_beam_search(single, N, 1.0, None, 0, 1, arr(toks1, U32), arr(lens1, U32), arr(scores1, ctypes.c_double), None)
        return single, run

    def grouped(G, tensor_cores=True):
        b = batch(G * W, tensor_cores)
        mt, lp = np.full(G, N, np.uint32), np.ones(G, np.float32)
        toks, lens, scores = np.zeros(G * N, np.uint32), np.zeros(G, np.uint32), np.zeros(G, np.float64)

        def run():
            assert L.rwkv_b200_beam_search_groups(b, G, arr(mt, U32), arr(lp, ctypes.c_float), None, 0, 1, arr(toks, U32), arr(lens, U32),
                                                  arr(scores, ctypes.c_double), None)
        return b, run

    legs = {}
    for G in GROUPS:
        legs[f"G{G}/grouped"] = grouped(G)
        legs[f"G{G}/serial"] = serial(G)
    legs["G4/grouped_no_tc"] = grouped(4, tensor_cores=False)

    def timed(b, fn):
        assert L.rwkv_b200_synchronize(b)
        t0 = time.perf_counter()
        fn()
        assert L.rwkv_b200_synchronize(b)
        return (time.perf_counter() - t0) * 1e3

    for b, fn in legs.values():        # warm-up: capacity, graph captures, module loads
        timed(b, fn)
    times = {k: [] for k in legs}
    for _ in range(args.rounds):
        for name, (b, fn) in legs.items():
            times[name].append(timed(b, fn))
    for b in owned:
        L.rwkv_free(b)
    lib.rwkv_free(ctx)

    res = {"card": card(), "workload": "rwkv6-7b:Q5_1, W = 4, 64 tokens, no stop ids", "rounds": args.rounds, "legs": {}}
    for name, t in times.items():
        G = int(name[1:name.index("/")])
        med = statistics.median(t)
        res["legs"][name] = {"ms_per_call": round(med, 3), "ms_per_step": round(med / N, 3), "min_max": [round(min(t), 3), round(max(t), 3)],
                             "hypotheses_per_s": round(G * W * N / (med / 1e3), 1)}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
