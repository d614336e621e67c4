"""What reporting log-probabilities costs device-side generation (DESIGN.md 6.4.3). Measurement aid, not a bench line.

Workloads: the synthetic rwkv4-169m Q5_1 (n_vocab 50277) and the synthetic RWKV-6 7B shape Q5_1 (n_vocab 65536), each as one sequence
and as a 16-sequence batch, max_tokens = 256 per leg. The legs:
  generate     rwkv_b200_generate / rwkv_b200_batch_generate
  lp_top0      rwkv_b200_generate_logprobs / rwkv_b200_batch_generate_logprobs with top_n 0 (logprobs and sample probs)
  lp_top5      ... with top_n 5
  lp_top20     ... with top_n 20
  host_route   per token: rwkv_b200_eval_sample (batch: rwkv_b200_batch_eval_sample), the logits to the host (rwkv_b200_stage_logits /
               rwkv_b200_batch_get_logits), a numpy log-softmax and an argpartition for the top 5

Every leg draws with temperature 1 and top_p 0.8, without penalties or stop ids, so every leg runs exactly 256 passes. A leg is timed
with the host clock around the call, which returns after a synchronise; the legs of a case alternate, and the result is the median
over rounds in milliseconds per generated token (per step for a batch) with min / max. The card's name and power limit are read in the
same run.

    python tools/generate_logprobs_bench.py [--rounds 5] [--tokens 256] [--out FILE.json]
"""
import argparse
import ctypes
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import __graft_entry__  # noqa: E402
import bench  # noqa: E402
from generate_bench import uniforms  # noqa: E402
from generate_stream_bench import measure  # noqa: E402
from ragged_batch_bench import card  # noqa: E402

U32, F32, F64 = ctypes.c_uint32, ctypes.c_float, ctypes.c_double
TEMPERATURE, TOP_P = 1.0, 0.8
HOST_TOP = 5


def host_logprobs(z, tok):
    z = z.astype(np.float64)
    m = z.max()
    lse = m + np.log(np.exp(z - m).sum())
    top = np.argpartition(-z, HOST_TOP)[:HOST_TOP]
    return z[tok] - lse, top[np.argsort(-z[top])], z[top] - lse


def legs_for(lib, path, n_tok, B):
    from rwkv_cpp_b200.shared_library import RWKV_TOKEN_FN, Logprobs
    L = lib.library
    base = lib.rwkv_b200_init_from_file_ex(path, 0, 0, -1)
    V = lib.rwkv_get_logits_buffer_element_count(base)
    rows = max(B, 1)
    null_fn = RWKV_TOKEN_FN()
    bt = ctypes.c_void_p(L.rwkv_b200_batch_create(base.ptr, B)) if B else None
    if B:
        assert bt
    toks, ng, n = (U32 * (rows * n_tok))(), (U32 * rows)(), ctypes.c_size_t(0)
    u_rows = [uniforms(n_tok, 100 + b) for b in range(rows)]
    u_arr = (F64 * (rows * n_tok))(*[u for r in u_rows for u in r])
    temps, top_ps, zeros = (F32 * rows)(*[TEMPERATURE] * rows), (F32 * rows)(*[TOP_P] * rows), (F32 * rows)()
    budgets = (U32 * rows)(*[n_tok] * rows)
    outs = {k: (np.zeros(rows * n_tok, np.float32), np.zeros(rows * n_tok, np.float32), np.zeros(rows * n_tok * max(k, 1), np.uint32),
                np.zeros(rows * n_tok * max(k, 1), np.float32)) for k in (0, 5, 20)}
    P_F, P_U = ctypes.POINTER(F32), ctypes.POINTER(U32)
    reqs = {k: Logprobs(top_n=k, logprobs=o[0].ctypes.data_as(P_F), sample_probs=o[1].ctypes.data_as(P_F),
                        top_ids=o[2].ctypes.data_as(P_U) if k else None, top_logprobs=o[3].ctypes.data_as(P_F) if k else None) for k, o in outs.items()}
    logits = np.zeros(V, np.float32)

    def reset():
        if B:
            for b in range(B):
                assert L.rwkv_b200_batch_set_state(bt, b, None)
            assert L.rwkv_b200_batch_eval(bt, (U32 * B)(*[11 + b for b in range(B)]), True)
            assert L.rwkv_b200_synchronize(bt)
        else:
            assert L.rwkv_b200_state_load(base.ptr, None)
            assert L.rwkv_b200_eval_resident(base.ptr, (U32 * 1)(11), 1, True, None)
            assert L.rwkv_b200_synchronize(base.ptr)

    def generate():
        if B:
            assert L.rwkv_b200_batch_generate(bt, budgets, temps, top_ps, zeros, zeros, None, u_arr, None, 0, toks, ng)
            assert all(ng[b] == n_tok for b in range(B))
        else:
            assert L.rwkv_b200_generate(base.ptr, n_tok, TEMPERATURE, TOP_P, 0.0, 0.0, False, u_arr, None, 0, toks, ctypes.byref(n)) and n.value == n_tok

    def logprobs(k):
        def leg(arrays=outs[k]):        # the request holds raw pointers: the leg keeps its arrays alive
            if B:
                assert L.rwkv_b200_batch_generate_logprobs(bt, None, None, budgets, temps, top_ps, zeros, zeros, None, u_arr, None, 0, null_fn, None, toks, ng,
                                                           ctypes.byref(reqs[k]))
                assert all(ng[b] == n_tok for b in range(B))
            else:
                assert L.rwkv_b200_generate_logprobs(base.ptr, None, None, n_tok, TEMPERATURE, TOP_P, 0.0, 0.0, False, u_arr, None, 0, null_fn, None, toks,
                                                     ctypes.byref(n), ctypes.byref(reqs[k])) and n.value == n_tok
        return leg

    def host_route():
        if B:
            cur = (U32 * B)(*[11 + b for b in range(B)])
            out = (U32 * B)()
            for i in range(n_tok):
                us = (F64 * B)(*[u_rows[b][i] for b in range(B)])
                assert L.rwkv_b200_batch_eval_sample(bt, cur, temps, top_ps, us, out)
                for b in range(B):
                    assert L.rwkv_b200_batch_get_logits(bt, b, logits.ctypes.data_as(P_F))
                    host_logprobs(logits, out[b])
                cur = out
                out = (U32 * B)()
        else:
            tok, nxt = 11, U32(0)
            for i in range(n_tok):
                assert L.rwkv_b200_eval_sample(base.ptr, tok, TEMPERATURE, TOP_P, u_rows[0][i], ctypes.byref(nxt))
                assert L.rwkv_b200_stage_logits(base.ptr, logits.ctypes.data_as(P_F), None)
                host_logprobs(logits, nxt.value)
                tok = nxt.value

    def free():
        if B:
            L.rwkv_free(bt)
        lib.rwkv_free(base)

    return free, reset, {"generate": generate, "lp_top0": logprobs(0), "lp_top5": logprobs(5), "lp_top20": logprobs(20), "host_route": host_route}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--tokens", type=int, default=256)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    pkg = __graft_entry__.load_package()
    lib = pkg.load_rwkv_shared_library()
    results = {"card": card(), "tokens_per_leg": args.tokens, "rounds": args.rounds, "unit": "ms per generated token (per step for a batch)"}
    for spec, name in [("rwkv4-169m:Q5_1", "169m"), ("rwkv6-7b:Q5_1", "7b")]:
        path, _ = bench.workload_file(spec)
        for B in (0, 16):
            free, reset, legs = legs_for(lib, path, args.tokens, B)
            results[f"{name}-b{max(B, 1)}"] = measure(reset, legs, args.rounds, args.tokens)
            free()
            print(json.dumps({f"{name}-b{max(B, 1)}": results[f"{name}-b{max(B, 1)}"]}), flush=True)
    line = json.dumps(results)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
