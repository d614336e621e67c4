"""What serving several LoRA fine-tunes from one batch context costs (DESIGN.md 6.7.1). Measurement aid, not a bench line.

Workload: the synthetic RWKV-6 7B shape at Q5_1 (bench.py's rwkv6-7b:Q5_1 file). Every adapter puts a seeded rank-16 delta on all 256
layer matrices that take one (att key / value / receptance / gate / output, ffn key / value / receptance of 32 layers), 84 MiB of fp16
A and B; the adapters differ in their seeds. For B = 8 sequences (the multi-column GEMV route) and B = 16 (the tensor-core route), ms
per batch step (one rwkv_b200_batch_eval with logits, graphs on) for:
  base      no adapter
  wide      one adapter attached to the whole batch (rwkv_b200_set_adapter)
  mixed-k   k distinct adapters attached per sequence (rwkv_b200_batch_set_adapter), sequence s on adapter s mod k, k = 2, 4, B
  split-k   the route without per-sequence adapters: k batch contexts of B / k sequences, each with its adapter attached to the whole
            context, stepped in turn (one step = one pass of each)
The legs alternate within every round; the median over the rounds with min / max. Then, on the B = 8 batch with 4 adapters, one
reassignment (sequence 0 to another adapter) followed by a rwkv_b200_batch_generate call of 32 tokens per sequence, against the same
call without the reassignment, alternated the same way. The card's name and power limit are read in the same run.

    python tools/multi_lora_bench.py [--rounds 5] [--steps 64] [--out FILE.json]
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
from lora_bench import adapter_entries  # noqa: E402
from ragged_batch_bench import card  # noqa: E402

U32 = ctypes.c_uint32
RANK = 16
GEN = 32


def arr(a, ct):
    return np.ascontiguousarray(a).ctypes.data_as(ctypes.POINTER(ct))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    pkg = __graft_entry__.load_package()
    lib = pkg.load_rwkv_shared_library()
    L = lib.library
    path, preset = bench.workload_file("rwkv6-7b:Q5_1")
    ctx = lib.rwkv_b200_init_from_file_ex(path, 0, 0, -1)
    V = lib.rwkv_get_logits_buffer_element_count(ctx)
    ads = [lib.rwkv_b200_adapter_create(ctx, adapter_entries(preset, RANK, False, seed=100 + i), 1.0) for i in range(16)]
    delta_bytes = sum(2 * RANK * (K + M) for M, K in [(preset["C"], preset["C"])] * 6 + [(preset["F"], preset["C"]), (preset["C"], preset["F"])]) * preset["L"]

    def batch(n):
        b = ctypes.c_void_p(L.rwkv_b200_batch_create(ctx.ptr, n))
        assert b.value
        return b

    def step_fn(batches):
        toks = [(U32 * L.rwkv_b200_batch_size(b))(*[(7919 * i + 11) % V for i in range(L.rwkv_b200_batch_size(b))]) for b in batches]

        def run(n):
            for b in batches:
                assert L.rwkv_b200_synchronize(b)
            t0 = time.perf_counter()
            for _ in range(n):
                for b, t in zip(batches, toks):
                    assert L.rwkv_b200_batch_eval(b, t, True)
            for b in batches:
                assert L.rwkv_b200_synchronize(b)
            return (time.perf_counter() - t0) * 1e3 / n
        return run

    legs, owned = {}, []
    for B in (8, 16):
        b = batch(B); owned.append(b)
        legs[f"B{B}/base"] = step_fn([b])
        b = batch(B); owned.append(b)
        assert L.rwkv_b200_set_adapter(b, ads[0])
        legs[f"B{B}/wide"] = step_fn([b])
        for k in (2, 4, B):
            b = batch(B); owned.append(b)
            for s in range(B):
                assert L.rwkv_b200_batch_set_adapter(b, s, ads[s % k])
            legs[f"B{B}/mixed-{k}"] = step_fn([b])
            parts = []
            for i in range(k):
                p = batch(B // k); owned.append(p)
                assert L.rwkv_b200_set_adapter(p, ads[i])
                parts.append(p)
            legs[f"B{B}/split-{k}"] = step_fn(parts)

    # reassignment + generate on a B = 8 batch with 4 adapters
    g = batch(8); owned.append(g)
    for s in range(8):
        assert L.rwkv_b200_batch_set_adapter(g, s, ads[s % 4])
    assert L.rwkv_b200_batch_eval(g, (U32 * 8)(*range(8)), True)      # generation draws its first tokens from these logits
    ones, zeros = np.ones(8, np.float32), np.zeros(8, np.float32)
    us = np.random.RandomState(1).random_sample((8, GEN))
    out, ng = np.zeros(8 * GEN, np.uint32), np.zeros(8, np.uint32)
    flip = [0]

    def gen(reassign):
        assert L.rwkv_b200_synchronize(g)
        t0 = time.perf_counter()
        if reassign:
            flip[0] ^= 1
            assert L.rwkv_b200_batch_set_adapter(g, 0, ads[4 + flip[0]])
        assert L.rwkv_b200_batch_generate(g, arr(np.full(8, GEN, np.uint32), U32), arr(ones, ctypes.c_float), arr(ones, ctypes.c_float),
                                          arr(zeros, ctypes.c_float), arr(zeros, ctypes.c_float), None, arr(us, ctypes.c_double), None, 0,
                                          arr(out, U32), arr(ng, U32))
        return (time.perf_counter() - t0) * 1e3
    legs["gen32"] = lambda n: gen(False)
    legs["reassign+gen32"] = lambda n: gen(True)

    for name, run in legs.items():        # warm-up: capacity, graph captures, module loads
        run(4)
        run(4)
    times = {k: [] for k in legs}
    for _ in range(args.rounds):
        for name, run in legs.items():
            if name.startswith("gen32"):
                run(1)                   # the graph of the current assignment
            times[name].append(run(args.steps))
    for b in owned:
        lib.library.rwkv_free(b)
    for a in ads:
        lib.rwkv_b200_adapter_free(a)
    lib.rwkv_free(ctx)

    res = {"card": card(), "workload": "rwkv6-7b:Q5_1, rank-16 deltas on all 256 layer matrices", "rounds": args.rounds, "steps": args.steps,
           "delta_mib_per_adapter": round(delta_bytes / 2 ** 20, 1), "legs": {}}
    for name, t in times.items():
        res["legs"][name] = {"ms": round(statistics.median(t), 4), "min_max": [round(min(t), 4), round(max(t), 4)]}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
