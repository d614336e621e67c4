"""Throughput of scoring a known text on one GPU, at the synthetic 7B shape with Q5_1 layers and an FP16 head (bench.py's workload).

    python tools/score_bench.py [--tokens 2048] [--rounds 5] [--serial-tokens 256]

Legs, in tokens/s, alternated round by round (median and min-max over the rounds):
  (a) score      rwkv_b200_score in calls of 256 tokens, every position with a target;
  (b) layers     rwkv_b200_eval_resident of the same 256-token windows without logits: the floor the layers set;
  (c) per_token  the route without scoring: rwkv_b200_eval_resident one token at a time with the logits copied to the host and a
                 numpy float64 log-softmax per token (over --serial-tokens tokens).
Plus the head's share of one 256-token scoring pass from the in-kernel timeline: LayerNorm + GEMM (with its fp16 conversion) + scoring
kernel, in microseconds, next to the whole pass. The card's name and power limit are read in the same run and printed with the numbers.
The model file goes to the temporary directory.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
P_F, P_U = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_uint32)
WINDOW = 256


def card():
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip() if r.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=2048)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--serial-tokens", type=int, default=256)
    ap.add_argument("--preset", default="rwkv6-7b")
    args = ap.parse_args()
    import __graft_entry__
    import synthetic_model as sm
    lib = __graft_entry__.load_package().load_rwkv_shared_library()
    L = lib.library
    path = os.path.join(tempfile.gettempdir(), f"score-bench-{args.preset}-Q5_1.bin")
    if not os.path.exists(path):
        sm.write_direct(path, args.preset, "Q5_1", seed=1)
    ctx = lib.rwkv_init_from_file(path, 1, 0)
    V = lib.rwkv_get_logits_buffer_element_count(ctx)
    toks = np.ascontiguousarray(sm.synthetic_tokens(args.tokens + 1, V), np.uint32)
    lp = np.empty(WINDOW, np.float32)

    def leg_score():
        assert L.rwkv_b200_state_load(ctx.ptr, None)
        t0 = time.perf_counter()
        for off in range(0, args.tokens, WINDOW):
            n = min(WINDOW, args.tokens - off)
            assert L.rwkv_b200_score(ctx.ptr, toks[off:].ctypes.data_as(P_U), toks[off + 1:].ctypes.data_as(P_U), n, lp.ctypes.data_as(P_F), None)
        return args.tokens / (time.perf_counter() - t0)

    def leg_layers():
        assert L.rwkv_b200_state_load(ctx.ptr, None)
        assert L.rwkv_b200_synchronize(ctx.ptr)
        t0 = time.perf_counter()
        for off in range(0, args.tokens, WINDOW):
            n = min(WINDOW, args.tokens - off)
            assert L.rwkv_b200_eval_resident(ctx.ptr, toks[off:].ctypes.data_as(P_U), n, False, None)
        assert L.rwkv_b200_synchronize(ctx.ptr)
        return args.tokens / (time.perf_counter() - t0)

    logits = np.empty(V, np.float32)

    def leg_per_token():
        assert L.rwkv_b200_state_load(ctx.ptr, None)
        n = args.serial_tokens
        t0 = time.perf_counter()
        total = 0.0
        for i in range(n):
            assert L.rwkv_b200_eval_resident(ctx.ptr, toks[i:].ctypes.data_as(P_U), 1, True, logits.ctypes.data_as(P_F))
            z = logits.astype(np.float64)
            m = z.max()
            total += z[toks[i + 1]] - m - np.log(np.exp(z - m).sum())
        return n / (time.perf_counter() - t0)

    legs = {"score": leg_score, "layers": leg_layers, "per_token": leg_per_token}
    for f in legs.values():
        f()                                   # warm-up: modules, the head's tile-major copy, buffers
    rates = {k: [] for k in legs}
    for _ in range(args.rounds):
        for k, f in legs.items():
            rates[k].append(f())

    # head share of one 256-token scoring pass (in-kernel timeline, a run of its own)
    N = 1024
    st, en = (ctypes.c_double * N)(), (ctypes.c_double * N)()
    names = ctypes.create_string_buffer(32 * N)
    assert L.rwkv_b200_trace_enable(ctx.ptr)
    assert L.rwkv_b200_score(ctx.ptr, toks.ctypes.data_as(P_U), toks[1:].ctypes.data_as(P_U), WINDOW, lp.ctypes.data_as(P_F), None)
    n = L.rwkv_b200_trace_read(ctx.ptr, st, en, ctypes.cast(names, ctypes.c_void_p), N)
    L.rwkv_b200_trace_disable(ctx.ptr)
    recs = [(names.raw[32 * i:32 * i + 32].split(b"\0")[0].decode(), st[i], en[i]) for i in range(n)]
    head = {name: round(e - s, 1) for name, s, e in recs[-4:]}
    pass_us = max(e for _, _, e in recs) - min(s for _, s, _ in recs)
    lib.rwkv_free(ctx)

    out = {"card": card(), "preset": args.preset, "weights": "Q5_1 layers, FP16 head", "tokens": args.tokens, "rounds": args.rounds,
           "serial_tokens": args.serial_tokens}
    for k, v in rates.items():
        out[k + "_tok_s"] = {"median": round(statistics.median(v), 1), "min": round(min(v), 1), "max": round(max(v), 1)}
    out["head_us"] = head
    out["head_total_us"] = round(sum(head.values()), 1)
    out["score_pass_us"] = round(pass_us, 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
