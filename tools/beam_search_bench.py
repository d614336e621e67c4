"""What a beam search costs on the device against the same search driven from the host (DESIGN.md 6.8). Measurement aid, not a bench line.

Workload: the synthetic RWKV-6 7B shape at Q5_1 (bench.py's rwkv6-7b:Q5_1 file), 64 tokens without stop ids, width W = 2, 4 and 8 (a batch
context of W sequences). Legs, ms per call:
  device    rwkv_b200_beam_search(max_tokens 64, length_penalty 1): one graph launch
  host      the same search over existing calls, per step: W x rwkv_b200_batch_get_logits (a synchronise each), a numpy top-2W per live
            beam and the ranking, the reorder of the beams as W rwkv_b200_batch_get_state into device buffers and W
            rwkv_b200_batch_set_state back (device-pointer copies), and one rwkv_b200_batch_eval with logits
  generate  for scale: rwkv_b200_batch_generate of the W sequences, 64 tokens each at temperature 1
The legs alternate within every round; the median over the rounds with min / max. The card's name and power limit are read in the same run.

    python tools/beam_search_bench.py [--rounds 5] [--out FILE.json]
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
P_F, P_U, P_D = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_double)
N = 64


def arr(a, ct):
    return np.ascontiguousarray(a).ctypes.data_as(ctypes.POINTER(ct))


def main():
    import torch
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
    n_state = lib.rwkv_get_state_buffer_element_count(ctx)
    legs, owned = {}, []
    for W in (2, 4, 8):
        b = ctypes.c_void_p(L.rwkv_b200_batch_create(ctx.ptr, W))
        assert b.value
        owned.append(b)
        assert L.rwkv_b200_batch_eval(b, (U32 * W)(*[(7919 * i + 11) % V for i in range(W)]), True)
        toks, lens, scores = np.zeros(W * N, np.uint32), np.zeros(W, np.uint32), np.zeros(W, np.float64)
        tmp = [torch.empty(n_state, dtype=torch.float32, device="cuda") for _ in range(W)]
        logit = np.zeros(V, np.float32)

        def device(b=b, W=W, toks=toks, lens=lens, scores=scores):
            assert L.rwkv_b200_beam_search(b, N, 1.0, None, 0, 1, arr(toks, U32), arr(lens, U32), arr(scores, ctypes.c_double), None)

        def host(b=b, W=W, tmp=tmp, logit=logit):
            live = [0.0]
            for _ in range(N):
                cands = []
                for k, sc in enumerate(live):
                    assert L.rwkv_b200_batch_get_logits(b, k, logit.ctypes.data_as(P_F))
                    top = np.argpartition(-logit, 2 * W)[:2 * W]
                    m = float(logit.max())
                    lse = m + float(np.log(np.exp(logit.astype(np.float64) - m).sum()))
                    cands += [(sc + float(logit[t]) - lse, k, int(t)) for t in top]
                cands.sort(key=lambda c: -c[0])
                taken = cands[:W]
                for k, (_, parent, _) in enumerate(taken):
                    assert L.rwkv_b200_batch_get_state(b, parent, ctypes.cast(tmp[k].data_ptr(), P_F))
                for k in range(W):
                    assert L.rwkv_b200_batch_set_state(b, k, ctypes.cast(tmp[k].data_ptr(), P_F))
                assert L.rwkv_b200_batch_eval(b, (U32 * W)(*[t for _, _, t in taken]), True)
                live = [s for s, _, _ in taken]
            assert L.rwkv_b200_synchronize(b)

        ones, zeros = np.ones(W, np.float32), np.zeros(W, np.float32)
        us = np.random.RandomState(W).random_sample((W, N))
        out, ng = np.zeros(W * N, np.uint32), np.zeros(W, np.uint32)

        def generate(b=b, W=W, ones=ones, zeros=zeros, us=us, out=out, ng=ng):
            assert L.rwkv_b200_batch_generate(b, arr(np.full(W, N, np.uint32), U32), arr(ones, ctypes.c_float), arr(ones, ctypes.c_float),
                                              arr(zeros, ctypes.c_float), arr(zeros, ctypes.c_float), None, arr(us, ctypes.c_double), None, 0,
                                              arr(out, U32), arr(ng, U32))

        for name, fn in (("device", device), ("host", host), ("generate", generate)):
            def timed(fn=fn, b=b):
                assert L.rwkv_b200_synchronize(b)
                t0 = time.perf_counter()
                fn()
                assert L.rwkv_b200_synchronize(b)
                return (time.perf_counter() - t0) * 1e3
            legs[f"W{W}/{name}"] = timed

    for run in legs.values():        # warm-up: capacity, graph captures, module loads
        run()
    times = {k: [] for k in legs}
    for _ in range(args.rounds):
        for name, run in legs.items():
            times[name].append(run())
    for b in owned:
        L.rwkv_free(b)
    lib.rwkv_free(ctx)

    res = {"card": card(), "workload": "rwkv6-7b:Q5_1, 64 tokens, no stop ids", "rounds": args.rounds, "legs": {}}
    for name, t in times.items():
        res["legs"][name] = {"ms_per_call": round(statistics.median(t), 3), "ms_per_step": round(statistics.median(t) / N, 3),
                             "min_max": [round(min(t), 3), round(max(t), 3)]}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
