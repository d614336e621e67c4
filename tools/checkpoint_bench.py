"""What checkpoints inside passes cost (DESIGN.md 6.9). Measurement aid, not a bench line.

Workload: the synthetic RWKV-6 7B shape at Q5_1 (bench.py's rwkv6-7b:Q5_1 file). Legs, ms per call:
  a  rwkv_b200_eval_resident of 2048 tokens
  b  the same call through rwkv_b200_eval_checkpoints with a checkpoint every 256 tokens (copies after each pass)
  c  a checkpoint every 64 tokens into device buffers (three of every four written by the kernels)
  d  the same into pinned host buffers
  e  the route without checkpoints inside passes: 32 calls of 64 tokens, each followed by rwkv_b200_state_store into a device buffer
  f  admission (DESIGN.md 6.3) on a batch of 16: 15 sequences decoding one token and one 128-token prompt in one ragged pass, plain
     (f_plain), with a checkpoint at token 64 of the prompt (f_checkpoint), and cut into two ragged passes at token 64 with
     rwkv_b200_batch_get_state into a device buffer in between (f_two_passes)
Every leg calls the library directly with argument arrays built once, before the timed rounds, so that the differences between the
legs are GPU work and copies, not host-side argument building. The legs alternate within every round; the median over the rounds with
min / max. The card's name and power limit are read in the same run.

    python tools/checkpoint_bench.py [--rounds 5] [--out FILE.json]
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

P_U32, P_F = ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_float)
T = 2048


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
    V, n = lib.rwkv_get_n_vocab(ctx), lib.rwkv_get_state_len(ctx)
    toks = np.ascontiguousarray(np.random.default_rng(0).integers(0, V, T), np.uint32)
    every256, every64 = list(range(255, T, 256)), list(range(63, T, 64))
    dev = [torch.empty(n, dtype=torch.float32, device="cuda:0") for _ in every64]
    pinned = [torch.empty(n, dtype=torch.float32).pin_memory() for _ in every64]

    def resident():
        assert L.rwkv_b200_eval_resident(ctx.ptr, toks.ctypes.data_as(P_U32), T, True, None) and L.rwkv_b200_synchronize(ctx.ptr)

    Checkpoint = pkg.shared_library.Checkpoint

    def entries(pairs, out):
        arr = (Checkpoint * len(pairs))()
        for i, (seq, pos) in enumerate(pairs):
            arr[i] = Checkpoint(seq, pos, ctypes.cast(out[i].data_ptr(), P_F))
        return arr

    cp_every256, cp_every64_dev, cp_every64_pinned = (entries([(0, p) for p in every256], dev), entries([(0, p) for p in every64], dev),
                                                      entries([(0, p) for p in every64], pinned))

    def checkpoints(arr):
        assert L.rwkv_b200_eval_checkpoints(ctx.ptr, toks.ctypes.data_as(P_U32), T, True, None, arr, len(arr))

    def cut_calls():
        for k in range(T // 64):
            assert L.rwkv_b200_eval_resident(ctx.ptr, toks[64 * k:].ctypes.data_as(P_U32), 64, k == T // 64 - 1, None)
            assert L.rwkv_b200_state_store(ctx.ptr, ctypes.cast(dev[k].data_ptr(), P_F))

    B = 16
    batch = L.rwkv_b200_batch_create(ctx.ptr, B)
    assert batch
    prompt = [int(t) for t in toks[:128]]
    decode = [int(t) for t in toks[200:215]]
    counts = [1] * 15 + [128]

    def u32(x):
        return np.ascontiguousarray(x, np.uint32)

    admit_toks, admit_counts = u32(decode + prompt), u32(counts)
    first_toks, first_counts, second_toks, second_counts = u32(decode + prompt[:64]), u32([1] * 15 + [64]), u32(prompt[64:]), u32([0] * 15 + [64])
    cp_admit = entries([(15, 63)], dev)

    def ragged(tk, cn):
        assert L.rwkv_b200_batch_eval_ragged(batch, tk.ctypes.data_as(P_U32), cn.ctypes.data_as(P_U32), True)

    def f_plain():
        ragged(admit_toks, admit_counts)
        assert L.rwkv_b200_synchronize(batch)

    def f_checkpoint():
        assert L.rwkv_b200_batch_eval_ragged_checkpoints(batch, admit_toks.ctypes.data_as(P_U32), admit_counts.ctypes.data_as(P_U32), True,
                                                         cp_admit, 1)

    def f_two_passes():
        ragged(first_toks, first_counts)
        assert L.rwkv_b200_batch_get_state(batch, 15, ctypes.cast(dev[0].data_ptr(), P_F))
        ragged(second_toks, second_counts)
        assert L.rwkv_b200_synchronize(batch)

    legs = {"a_resident": resident, "b_every256": lambda: checkpoints(cp_every256), "c_every64_device": lambda: checkpoints(cp_every64_dev),
            "d_every64_pinned": lambda: checkpoints(cp_every64_pinned), "e_64_token_calls": cut_calls,
            "f_plain": f_plain, "f_checkpoint": f_checkpoint, "f_two_passes": f_two_passes}
    times = {k: [] for k in legs}
    for fn in legs.values():     # warm-up: every shape, buffer and pinned destination
        fn()
    for _ in range(args.rounds):
        for k, fn in legs.items():
            t0 = time.perf_counter()
            fn()
            times[k].append((time.perf_counter() - t0) * 1e3)
    res = {"card": card(), "workload": "rwkv6-7b:Q5_1, 2048-token prompt; admission: 15 decoding + 128-token prompt", "rounds": args.rounds,
           "checkpoint_mb": round(n * 4 / 1e6, 1), "legs": {}}
    for k, t in times.items():
        res["legs"][k] = {"ms": round(statistics.median(t), 3), "min_max": [round(min(t), 3), round(max(t), 3)]}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    L.rwkv_free(batch)
    lib.rwkv_free(ctx)


if __name__ == "__main__":
    main()
