"""Streaming generation against the blocking call (DESIGN.md 6.4). Measurement aid, not a bench line.

  169m-b1 / 7b-b1 : rwkv4-169m:Q5_1 and the synthetic RWKV-6-World-7B Q5_1, one sequence: rwkv_b200_generate_stream with a callback
                    that returns 0 at once against rwkv_b200_generate, both max_tokens = 256
  7b-b16          : the 7B shape, a 16-sequence batch: rwkv_b200_batch_generate_stream against rwkv_b200_batch_generate (256 each)
  first_token     : 7B, one sequence: time from the call to the first callback, against the time of the whole blocking call
  sleep_*         : 7B, one sequence: ms per token when the callback sleeps 0.1 / 0.5 / 2 ms before it returns 0

Every leg draws with temperature 1 and top_p 0.8, without penalties or stop ids, so every leg runs exactly 256 passes. A leg is timed
with the host clock around the call, which returns after a synchronise; the legs of a case alternate, and the result is the median
over rounds in milliseconds per generated token (per step for the batch). The card's name and power limit are read in the same run.

    python tools/generate_stream_bench.py [--rounds 5] [--tokens 256] [--out FILE.json]
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
from generate_bench import uniforms  # noqa: E402
from ragged_batch_bench import card  # noqa: E402

U32, F32, F64 = ctypes.c_uint32, ctypes.c_float, ctypes.c_double
TEMPERATURE, TOP_P = 1.0, 0.8


def callback(sleep_s=0.0, first=None):
    """An on_token that returns 0, after sleeping sleep_s; `first`, a one-element list, receives the clock of the first call."""
    from rwkv_cpp_b200.shared_library import RWKV_TOKEN_FN

    def on_token(user, seq, idx, tok):
        if first is not None and not first[0]:
            first[0] = time.perf_counter()
        if sleep_s:
            t_end = time.perf_counter() + sleep_s      # a spin: time.sleep's granularity is too coarse at 0.1 ms
            while time.perf_counter() < t_end:
                pass
        return 0
    return RWKV_TOKEN_FN(on_token)


def single_legs(lib, path, n_tok):
    L = lib.library
    ctx = lib.rwkv_b200_init_from_file_ex(path, 0, 0, -1)
    u_arr = (F64 * n_tok)(*uniforms(n_tok, 1))
    toks = (U32 * n_tok)()
    n = ctypes.c_size_t(0)

    def reset():
        assert L.rwkv_b200_state_load(ctx.ptr, None)
        assert L.rwkv_b200_eval_resident(ctx.ptr, (U32 * 1)(11), 1, True, None)
        assert L.rwkv_b200_synchronize(ctx.ptr)

    def blocking():
        assert L.rwkv_b200_generate(ctx.ptr, n_tok, TEMPERATURE, TOP_P, 0.0, 0.0, False, u_arr, None, 0, toks, ctypes.byref(n)) and n.value == n_tok

    def streaming(fn):
        def leg():
            assert L.rwkv_b200_generate_stream(ctx.ptr, n_tok, TEMPERATURE, TOP_P, 0.0, 0.0, False, u_arr, None, 0, fn, None, toks,
                                               ctypes.byref(n)) and n.value == n_tok
        return leg

    return ctx, reset, blocking, streaming


def batch_legs(lib, path, n_tok, B):
    L = lib.library
    base = lib.rwkv_b200_init_from_file_ex(path, 0, 0, -1)
    bt = ctypes.c_void_p(L.rwkv_b200_batch_create(base.ptr, B))
    assert bt
    temps, top_ps, zeros = (F32 * B)(*[TEMPERATURE] * B), (F32 * B)(*[TOP_P] * B), (F32 * B)()
    budgets = (U32 * B)(*[n_tok] * B)
    u_arr = (F64 * (B * n_tok))(*[u for b in range(B) for u in uniforms(n_tok, 100 + b)])
    toks, ng = (U32 * (B * n_tok))(), (U32 * B)()
    fn = callback()

    def reset():
        for b in range(B):
            assert L.rwkv_b200_batch_set_state(bt, b, None)
        assert L.rwkv_b200_batch_eval(bt, (U32 * B)(*[11 + b for b in range(B)]), True)
        assert L.rwkv_b200_synchronize(bt)

    def blocking():
        assert L.rwkv_b200_batch_generate(bt, budgets, temps, top_ps, zeros, zeros, None, u_arr, None, 0, toks, ng)
        assert all(ng[b] == n_tok for b in range(B))

    def streaming():
        assert L.rwkv_b200_batch_generate_stream(bt, budgets, temps, top_ps, zeros, zeros, None, u_arr, None, 0, fn, None, toks, ng)
        assert all(ng[b] == n_tok for b in range(B))

    def free():
        L.rwkv_free(bt)
        lib.rwkv_free(base)

    return free, reset, blocking, streaming


def measure(reset, legs, rounds, n_tok):
    """legs: {name: fn}; median ms per token of each over `rounds` alternating rounds, with min / max."""
    for leg in legs.values():       # warm-up: module loads, capacity growth, graph captures
        reset()
        leg()
    samples = {k: [] for k in legs}
    for _ in range(rounds):
        for name, leg in legs.items():
            reset()
            t0 = time.perf_counter()
            leg()
            samples[name].append((time.perf_counter() - t0) * 1e3 / n_tok)
    res = {k: round(statistics.median(v), 4) for k, v in samples.items()}
    res["min_max"] = {k: [round(min(v), 4), round(max(v), 4)] for k, v in samples.items()}
    return res


def first_token(reset, blocking, streaming, rounds):
    """Median ms from the call to the first callback, and of the whole blocking call, alternating."""
    first = [0.0]
    leg = streaming(callback(first=first))
    reset()
    leg()
    to_first, whole = [], []
    for _ in range(rounds):
        reset()
        first[0] = 0.0
        t0 = time.perf_counter()
        leg()
        to_first.append((first[0] - t0) * 1e3)
        reset()
        t0 = time.perf_counter()
        blocking()
        whole.append((time.perf_counter() - t0) * 1e3)
    return {"first_callback_ms": round(statistics.median(to_first), 3), "blocking_call_ms": round(statistics.median(whole), 3),
            "min_max": {"first_callback_ms": [round(min(to_first), 3), round(max(to_first), 3)], "blocking_call_ms": [round(min(whole), 3), round(max(whole), 3)]}}


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
    ctx, reset, blocking, streaming = single_legs(lib, path169m, args.tokens)
    results["169m-b1"] = measure(reset, {"generate": blocking, "generate_stream": streaming(callback())}, args.rounds, args.tokens)
    lib.rwkv_free(ctx)
    ctx, reset, blocking, streaming = single_legs(lib, path7b, args.tokens)
    results["7b-b1"] = measure(reset, {"generate": blocking, "generate_stream": streaming(callback())}, args.rounds, args.tokens)
    results["first_token"] = first_token(reset, blocking, streaming, args.rounds)
    results["sleep"] = measure(reset, {"generate": blocking, **{"sleep_%gms" % ms: streaming(callback(ms / 1e3)) for ms in (0.1, 0.5, 2.0)}},
                               args.rounds, args.tokens)
    lib.rwkv_free(ctx)
    free, reset, blocking, streaming = batch_legs(lib, path7b, args.tokens, 16)
    results["7b-b16"] = measure(reset, {"generate": blocking, "generate_stream": streaming}, args.rounds, args.tokens)
    free()
    line = json.dumps(results)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
