"""Cost of picking every sequence's next token in a batch context at the 7B shape, in ms per step for B = 1, 4, 16, 64:
  (a) rwkv_b200_batch_eval alone;
  (b) rwkv_b200_batch_eval_sample: the pass, then one launch of the batched sampling kernel; B token ids come back;
  (c) rwkv_b200_batch_eval, then B x rwkv_b200_batch_get_logits (n_vocab floats each, each call synchronises) and a host draw per
      sequence (oracle/sampling_oracle.py, the numpy restatement of the reference's python/sampling.py): the route without (b).
(b) - (a) and (c) - (a) are what choosing the tokens costs. The three legs alternate in rounds so that drift on a shared card
spreads over all of them; each leg reports its median round. Measurement aid (DESIGN.md 6.2), not a bench line.

    python tools/batch_sample_bench.py [preset:format] [--steps N] [--rounds R]
"""
import argparse
import ctypes
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tools")); sys.path.insert(0, os.path.join(ROOT, "oracle"))
import __graft_entry__, bench  # noqa: E402
import sampling_oracle as so  # noqa: E402

P_F, P_U, P_D = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_double)


def card():
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip() if r.returncode == 0 else "unknown (nvidia-smi failed)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("workload", nargs="?", default="rwkv6-7b:Q5_1")
    ap.add_argument("--steps", type=int, default=12, help="timed steps per leg and round (each ends with a synchronise)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sizes", default="1,4,16,64")
    args = ap.parse_args()
    pkg = __graft_entry__.load_package()
    lib = pkg.load_rwkv_shared_library()
    L = lib.library
    path, preset = bench.workload_file(args.workload)
    ctx = lib.rwkv_b200_init_from_file_ex(path, 0, 0, -1)
    V = preset["V"]
    print(f"{args.workload}, n_vocab {V}; card: {card()}")
    print(f"{'B':>4} {'(a) eval':>10} {'(b) eval_sample':>16} {'(c) eval+host':>14} {'(b)-(a)':>9} {'(c)-(a)':>9}   ms per step, median of {args.rounds} rounds x {args.steps} steps")
    for B in (int(s) for s in args.sizes.split(",")):
        b = ctypes.c_void_p(L.rwkv_b200_batch_create(ctx.ptr, B))
        assert b, f"batch_create failed for B = {B}"
        toks = np.array([(7919 * i + 11) % V for i in range(B)], np.uint32)
        temp = np.full(B, 1.0, np.float32)
        top_p = np.full(B, 0.8, np.float32)
        rng = np.random.RandomState(B)
        out = np.zeros(B, np.uint32)
        lg = np.zeros(V, np.float32)
        tp, fp, tpp, op = toks.ctypes.data_as(P_U), temp.ctypes.data_as(P_F), top_p.ctypes.data_as(P_F), out.ctypes.data_as(P_U)

        def leg_a():
            assert L.rwkv_b200_batch_eval(b, tp, True)

        def leg_b():
            u = rng.random_sample(B)
            assert L.rwkv_b200_batch_eval_sample(b, tp, fp, tpp, u.ctypes.data_as(P_D), op)

        def leg_c():
            u = rng.random_sample(B)
            assert L.rwkv_b200_batch_eval(b, tp, True)
            for s in range(B):
                assert L.rwkv_b200_batch_get_logits(b, s, lg.ctypes.data_as(P_F))
                out[s] = so.sample_logits_u(lg, 1.0, 0.8, u[s])

        legs = {"a": leg_a, "b": leg_b, "c": leg_c}
        for fn in legs.values():            # warm-up: module loads, first allocations, pinned buffers
            for _ in range(4):
                fn()
        L.rwkv_b200_synchronize(b)
        times = {k: [] for k in legs}
        for _ in range(args.rounds):
            for k, fn in legs.items():
                t0 = time.perf_counter()
                for _ in range(args.steps):
                    fn()
                L.rwkv_b200_synchronize(b)
                times[k].append((time.perf_counter() - t0) / args.steps * 1e3)
        m = {k: float(np.median(v)) for k, v in times.items()}
        print(f"{B:>4} {m['a']:>10.3f} {m['b']:>16.3f} {m['c']:>14.3f} {m['b'] - m['a']:>9.3f} {m['c'] - m['a']:>9.3f}"
              f"   rounds a {['%.3f' % t for t in times['a']]} b {['%.3f' % t for t in times['b']]} c {['%.3f' % t for t in times['c']]}")
        L.rwkv_free(b)
    lib.rwkv_free(ctx)


if __name__ == "__main__":
    main()
