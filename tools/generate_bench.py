"""Device-side generation against the host-driven loop it replaces (DESIGN.md 6.4). Measurement aid, not a bench line.

  7b-b1    : synthetic RWKV-6-World-7B Q5_1, one sequence: 256 x rwkv_b200_eval_sample (token fed back by the host) against one
             rwkv_b200_generate(max_tokens = 256)
  169m-b1  : the rwkv4-169m:Q5_1 workload, the same two legs
  7b-b16   : the 7B shape, a 16-sequence batch: 256 x rwkv_b200_batch_eval_sample against one rwkv_b200_batch_generate(256 each)

Both legs draw with temperature 1 and top_p 0.8, without penalties or stop ids, so both run exactly 256 passes. A leg is timed with
the host clock around work that ends in a synchronise; the two legs of a case alternate, and the result is the median over rounds
in milliseconds per generated token. The card's name and power limit are read in the same run.

    python tools/generate_bench.py [--rounds 5] [--tokens 256] [--out FILE.json]
"""
import argparse
import ctypes
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import __graft_entry__  # noqa: E402
import bench  # noqa: E402
from ragged_batch_bench import card  # noqa: E402

U32, F32, F64, U8 = ctypes.c_uint32, ctypes.c_float, ctypes.c_double, ctypes.c_uint8
TEMPERATURE, TOP_P = 1.0, 0.8


def uniforms(n, seed):
    state = seed
    out = []
    for _ in range(n):     # a fixed sequence in [0, 1) without numpy's global state
        state = (state * 6364136223846793005 + 1442695040888963407) % (1 << 64)
        out.append((state >> 11) / float(1 << 53))
    return out


def single_legs(lib, path, n_tok):
    L = lib.library
    ctx = lib.rwkv_b200_init_from_file_ex(path, 0, 0, -1)
    us = uniforms(n_tok, 1)
    u_arr = (F64 * n_tok)(*us)
    toks = (U32 * n_tok)()
    n = ctypes.c_size_t(0)

    def reset():
        assert L.rwkv_b200_state_load(ctx.ptr, None)
        assert L.rwkv_b200_eval_resident(ctx.ptr, (U32 * 1)(11), 1, True, None)
        assert L.rwkv_b200_synchronize(ctx.ptr)

    def host():
        tok = ctypes.c_uint32(11)
        for i in range(n_tok):
            assert L.rwkv_b200_eval_sample(ctx.ptr, tok.value, TEMPERATURE, TOP_P, us[i], ctypes.byref(tok))

    def device():
        assert L.rwkv_b200_generate(ctx.ptr, n_tok, TEMPERATURE, TOP_P, 0.0, 0.0, False, u_arr, None, 0, toks, ctypes.byref(n)) and n.value == n_tok

    return ctx, reset, host, device


def batch_legs(lib, path, n_tok, B):
    L = lib.library
    base = lib.rwkv_b200_init_from_file_ex(path, 0, 0, -1)
    bt = ctypes.c_void_p(L.rwkv_b200_batch_create(base.ptr, B))
    assert bt
    us = [uniforms(n_tok, 100 + b) for b in range(B)]
    temps, top_ps, zeros = (F32 * B)(*[TEMPERATURE] * B), (F32 * B)(*[TOP_P] * B), (F32 * B)()
    budgets = (U32 * B)(*[n_tok] * B)
    u_arr = (F64 * (B * n_tok))(*[u for row in us for u in row])
    toks, ng = (U32 * (B * n_tok))(), (U32 * B)()
    out = (U32 * B)()

    def reset():
        for b in range(B):
            assert L.rwkv_b200_batch_set_state(bt, b, None)
        assert L.rwkv_b200_batch_eval(bt, (U32 * B)(*[11 + b for b in range(B)]), True)
        assert L.rwkv_b200_synchronize(bt)

    def host():
        cur = (U32 * B)(*[11 + b for b in range(B)])
        for i in range(n_tok):
            step_u = (F64 * B)(*[us[b][i] for b in range(B)])
            assert L.rwkv_b200_batch_eval_sample(bt, cur, temps, top_ps, step_u, out)
            ctypes.memmove(cur, out, 4 * B)

    def device():
        assert L.rwkv_b200_batch_generate(bt, budgets, temps, top_ps, zeros, zeros, None, u_arr, None, 0, toks, ng)
        assert all(ng[b] == n_tok for b in range(B))

    def free():
        L.rwkv_free(bt)
        lib.rwkv_free(base)

    return free, reset, host, device


def measure(reset, host, device, rounds, n_tok):
    for leg in (host, device):          # warm-up: module loads, capacity growth, graph captures
        reset()
        leg()
    samples = {"host_loop": [], "generate": []}
    for _ in range(rounds):
        for name, leg in (("host_loop", host), ("generate", device)):
            reset()
            t0 = time.perf_counter()
            leg()                       # both legs end in a synchronise (the last token is read back)
            samples[name].append((time.perf_counter() - t0) * 1e3 / n_tok)
    res = {k: round(statistics.median(v), 4) for k, v in samples.items()}
    res["min_max"] = {k: [round(min(v), 4), round(max(v), 4)] for k, v in samples.items()}
    res["speedup"] = round(res["host_loop"] / res["generate"], 3)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--tokens", type=int, default=256)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    pkg = __graft_entry__.load_package()
    lib = pkg.load_rwkv_shared_library()
    results = {"card": card(), "tokens_per_leg": args.tokens, "rounds": args.rounds, "unit": "ms per generated token (per step for the batch)"}
    path7b, _ = bench.workload_file("rwkv6-7b:Q5_1")
    path169m, _ = bench.workload_file("rwkv4-169m:Q5_1")
    for name, path in (("7b-b1", path7b), ("169m-b1", path169m)):
        ctx, reset, host, device = single_legs(lib, path, args.tokens)
        results[name] = measure(reset, host, device, args.rounds, args.tokens)
        lib.rwkv_free(ctx)
    free, reset, host, device = batch_legs(lib, path7b, args.tokens, 16)
    results["7b-b16"] = measure(reset, host, device, args.rounds, args.tokens)
    free()
    line = json.dumps(results)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
