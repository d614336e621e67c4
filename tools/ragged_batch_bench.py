"""Continuous batching at the 7B shape (synthetic RWKV-6-World-7B, Q5_1): one ragged pass of a batch context
(rwkv_b200_batch_eval_ragged) against the routes a caller has without it. Measurement aid (DESIGN.md 6.3), not a bench line.

  admission : (a) one ragged call on a 16-slot batch, counts = 15 x [1] + [128]
              (b) rwkv_b200_batch_eval on a 15-sequence batch + a 128-token rwkv_b200_eval_resident on a single-sequence context
  idle slots: (a) a ragged call with 8 columns on a 32-slot batch (8 active, 24 idle)
              (b) rwkv_b200_batch_eval over all 32 slots

Each step ends in a synchronise and is timed with the host clock; the two legs of a pair alternate step by step, and the result is
the median over rounds. The card's name and power limit are read in the same run.

    python tools/ragged_batch_bench.py [--rounds 7] [--steps 6] [--out FILE.json]
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import __graft_entry__  # noqa: E402
import bench  # noqa: E402

U32 = ctypes.c_uint32


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:          # the numbers are worth little without it: say so in the result
        return "unknown (%s)" % e


def timed(fn, sync):
    t0 = time.perf_counter()
    fn()
    sync()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--spec", default="rwkv6-7b:Q5_1")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    pkg = __graft_entry__.load_package()
    lib = pkg.load_rwkv_shared_library()
    L = lib.library
    path, preset = bench.workload_file(args.spec)
    V = preset["V"]
    ctx = lib.rwkv_b200_init_from_file_ex(path, 0, 0, -1)
    tok = lambda i: (7919 * i + 13) % V

    def batch(n):
        b = ctypes.c_void_p(L.rwkv_b200_batch_create(ctx.ptr, n))
        assert b, "batch_create(%d) failed" % n
        return b

    def ragged(b, counts):
        toks = [tok(i) for i in range(sum(counts))]
        t, c = (U32 * len(toks))(*toks), (U32 * len(counts))(*counts)
        return lambda: L.rwkv_b200_batch_eval_ragged(b, t, c, True) or sys.exit("ragged call failed")

    def batch_eval(b, n):
        t = (U32 * n)(*[tok(i) for i in range(n)])
        return lambda: L.rwkv_b200_batch_eval(b, t, True) or sys.exit("batch_eval failed")

    # admission
    b16, b15 = batch(16), batch(15)
    single = lib.rwkv_b200_init_from_file_ex(path, 0, 0, -1)
    L.rwkv_b200_state_load(single.ptr, None)
    prompt = (U32 * 128)(*[tok(1000 + i) for i in range(128)])
    adm_a = ragged(b16, [1] * 15 + [128])
    dec15 = batch_eval(b15, 15)

    def adm_b():
        dec15()
        assert L.rwkv_b200_eval_resident(single.ptr, prompt, 128, True, None)

    def sync_adm_b():
        L.rwkv_b200_synchronize(b15)
        L.rwkv_b200_synchronize(single.ptr)

    # idle slots
    b32r, b32 = batch(32), batch(32)
    idle_a = ragged(b32r, [1, 0, 0, 0] * 8)
    idle_b = batch_eval(b32, 32)

    legs = {
        "admission_ragged": (adm_a, lambda: L.rwkv_b200_synchronize(b16)),
        "admission_batch_plus_single": (adm_b, sync_adm_b),
        "idle_ragged_8_of_32": (idle_a, lambda: L.rwkv_b200_synchronize(b32r)),
        "idle_batch_eval_32": (idle_b, lambda: L.rwkv_b200_synchronize(b32)),
    }
    pairs = [("admission_ragged", "admission_batch_plus_single"), ("idle_ragged_8_of_32", "idle_batch_eval_32")]
    for fn, sync in legs.values():         # warm-up: module loads, capacity growth, graph capture of the single-token passes
        for _ in range(3):
            fn()
        sync()
    samples = {k: [] for k in legs}
    for _ in range(args.rounds):
        for a, b in pairs:
            ta, tb = [], []
            for _ in range(args.steps):
                ta.append(timed(*legs[a]))
                tb.append(timed(*legs[b]))
            samples[a].append(statistics.median(ta) * 1e3)
            samples[b].append(statistics.median(tb) * 1e3)
    res = {"card": card(), "spec": args.spec, "rounds": args.rounds, "steps_per_round": args.steps,
           "ms_median": {k: round(statistics.median(v), 3) for k, v in samples.items()},
           "ms_min_max": {k: [round(min(v), 3), round(max(v), 3)] for k, v in samples.items()}}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    for b in (b16, b15, b32r, b32):
        L.rwkv_free(b)
    lib.rwkv_free(single)
    lib.rwkv_free(ctx)


if __name__ == "__main__":
    main()
