"""Penalty decay in device-side generation (DESIGN.md 6.4.5). Measurement aid, not a bench line.

  7b-b1    : synthetic RWKV-6-World-7B Q5_1 (n_vocab 65536), one sequence: rwkv_b200_generate(max_tokens = 256) with decay 1 against
             decay 0.996 and a weight table
  7b-b16   : the 7B shape, a 16-sequence batch: rwkv_b200_batch_generate(256 each), the same two legs

Both legs draw with temperature 1, top_p 0.8, presence and frequency penalty 0.3, without stop ids, so both run exactly 256 passes.
A leg is timed with the host clock around a call, which ends in a synchronise; the two legs of a case alternate, and the result is
the median over rounds in milliseconds per generated token (per step for the batch). The card's name and power limit are read in the
same run.

    python tools/penalty_bench.py [--rounds 5] [--tokens 256] [--out FILE.json]
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
from generate_bench import uniforms  # noqa: E402
from ragged_batch_bench import card  # noqa: E402

U32, F32, F64 = ctypes.c_uint32, ctypes.c_float, ctypes.c_double
TEMPERATURE, TOP_P, PENALTY, DECAY = 1.0, 0.8, 0.3, 0.996


def legs(lib, ctx, B, n_tok, weights):
    """reset, and the call with decay 1 / with decay 0.996 and the weights, on ctx (B = 0: a single-sequence context)."""
    L = lib.library
    rows = max(B, 1)
    us = [u for b in range(rows) for u in uniforms(n_tok, 100 + b)]
    u_arr = (F64 * len(us))(*us)
    toks, ng = (U32 * (rows * n_tok))(), (U32 * rows)()
    budgets = (U32 * rows)(*[n_tok] * rows)
    temps, top_ps, pens = (F32 * rows)(*[TEMPERATURE] * rows), (F32 * rows)(*[TOP_P] * rows), (F32 * rows)(*[PENALTY] * rows)
    n = ctypes.c_size_t(0)

    def reset():
        if B:
            for b in range(B):
                assert L.rwkv_b200_batch_set_state(ctx, b, None)
            assert L.rwkv_b200_batch_eval(ctx, (U32 * B)(*[11 + b for b in range(B)]), True)
        else:
            assert L.rwkv_b200_state_load(ctx, None)
            assert L.rwkv_b200_eval_resident(ctx, (U32 * 1)(11), 1, True, None)
        assert L.rwkv_b200_synchronize(ctx)

    def run():
        if B:
            assert L.rwkv_b200_batch_generate(ctx, budgets, temps, top_ps, pens, pens, None, u_arr, None, 0, toks, ng)
            assert all(ng[b] == n_tok for b in range(B))
        else:
            assert L.rwkv_b200_generate(ctx, n_tok, TEMPERATURE, TOP_P, PENALTY, PENALTY, False, u_arr, None, 0, toks, ctypes.byref(n))
            assert n.value == n_tok

    def set_decay(d, w):
        for b in range(rows):
            assert L.rwkv_b200_set_penalty_decay(ctx, b, d)
        assert L.rwkv_b200_set_penalty_weights(ctx, w)

    def plain():
        set_decay(1.0, None)
        run()

    def decayed():
        set_decay(DECAY, weights.ctypes.data_as(ctypes.POINTER(F32)))
        run()

    return reset, plain, decayed


def measure(reset, plain, decayed, rounds, n_tok):
    for leg in (plain, decayed):        # warm-up: module loads, buffers, graph captures
        reset()
        leg()
    samples = {"decay_1": [], "decay_0.996": []}
    for _ in range(rounds):
        for name, leg in (("decay_1", plain), ("decay_0.996", decayed)):
            reset()
            t0 = time.perf_counter()
            leg()
            samples[name].append((time.perf_counter() - t0) * 1e3 / n_tok)
    res = {k: round(statistics.median(v), 4) for k, v in samples.items()}
    res["min_max"] = {k: [round(min(v), 4), round(max(v), 4)] for k, v in samples.items()}
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
    base = lib.rwkv_b200_init_from_file_ex(path7b, 0, 0, -1)
    V = lib.rwkv_get_logits_len(base)
    weights = np.random.RandomState(0).choice(np.array([0.0, 1.0], np.float32), V).astype(np.float32)
    results["7b-b1"] = measure(*legs(lib, base.ptr, 0, args.tokens, weights), args.rounds, args.tokens)
    bt = ctypes.c_void_p(lib.library.rwkv_b200_batch_create(base.ptr, 16))
    assert bt
    results["7b-b16"] = measure(*legs(lib, bt, 16, args.tokens, weights), args.rounds, args.tokens)
    lib.library.rwkv_free(bt)
    lib.rwkv_free(base)
    line = json.dumps(results)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
