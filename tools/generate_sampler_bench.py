"""What top_k, min_p and a logit bias cost device-side generation (DESIGN.md 6.4.4). Measurement aid, not a bench line.

Workloads: the synthetic rwkv4-169m Q5_1 (n_vocab 50277) and the synthetic RWKV-6 7B shape Q5_1 (n_vocab 65536), each as one sequence
and as a 16-sequence batch, max_tokens = 256 per leg. The legs:
  generate     rwkv_b200_generate / rwkv_b200_batch_generate
  sampled_off  rwkv_b200_generate_sampled / rwkv_b200_batch_generate_sampled with top_k 0, min_p 0 and no bias entries
  top_k40      ... with top_k 40
  min_p05      ... with min_p 0.05
  all          ... with top_k 40, min_p 0.05 and 300 bias entries (boosts, cuts and bans)
  host_top_k   per token: rwkv_b200_eval_resident (batch: rwkv_b200_batch_eval), the logits to the host (rwkv_b200_stage_logits /
               rwkv_b200_batch_get_logits) and a numpy top-k 40 draw (argpartition, softmax over the 40, inverse CDF)

Every leg draws with temperature 1 and top_p 0.8, without penalties or stop ids, so every leg runs exactly 256 passes. A leg is timed
with the host clock around the call, which returns after a synchronise; the legs of a case alternate, and the result is the median
over rounds in milliseconds per generated token (per step for a batch) with min / max. The card's name and power limit are read in the
same run.

    python tools/generate_sampler_bench.py [--rounds 5] [--tokens 256] [--out FILE.json]
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
TEMPERATURE, TOP_P, TOP_K, MIN_P, N_BIAS = 1.0, 0.8, 40, 0.05, 300


def host_top_k(z, u):
    """A top-k draw on the host: the TOP_K largest logits, their softmax, and the inverse CDF at u."""
    top = np.argpartition(-z, TOP_K)[:TOP_K]
    top = top[np.argsort(-z[top])]
    e = np.exp(z[top].astype(np.float64) - z[top[0]])
    cdf = np.cumsum(e)
    return int(top[min(int(np.searchsorted(cdf / cdf[-1], u, side="right")), TOP_K - 1)])


def legs_for(lib, path, n_tok, B):
    from rwkv_cpp_b200.shared_library import RWKV_TOKEN_FN, Sampler
    L = lib.library
    base = lib.rwkv_b200_init_from_file_ex(path, 0, 0, -1)
    V = lib.rwkv_get_logits_buffer_element_count(base)
    L.rwkv_set_print_errors(base.ptr, True)
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
    rng = np.random.RandomState(0)
    bias_ids = rng.choice(V, size=N_BIAS, replace=False).astype(np.uint32)
    bias_vals = np.where(rng.rand(N_BIAS) < 0.1, -np.inf, rng.standard_normal(N_BIAS)).astype(np.float32)
    P_F, P_U = ctypes.POINTER(F32), ctypes.POINTER(U32)

    def sampler(top_k=0, min_p=0.0, bias=False):
        s = Sampler(temperature=TEMPERATURE, top_p=TOP_P, top_k=top_k, min_p=min_p)
        if bias:
            s.n_bias, s.bias_ids, s.bias_values = N_BIAS, bias_ids.ctypes.data_as(P_U), bias_vals.ctypes.data_as(P_F)
        return (Sampler * rows)(*[s] * rows)
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

    def sampled(smp):
        def leg(arrays=(bias_ids, bias_vals)):      # the sampler holds raw pointers: the leg keeps its arrays alive
            if B:
                ok = L.rwkv_b200_batch_generate_sampled(bt, smp, None, None, budgets, None, u_arr, None, 0, null_fn, None, toks, ng, None)
                assert ok and all(ng[b] == n_tok for b in range(B)), (ok, list(ng), L.rwkv_get_last_error(bt))
            else:
                ok = L.rwkv_b200_generate_sampled(base.ptr, smp, None, None, n_tok, False, u_arr, None, 0, null_fn, None, toks, ctypes.byref(n), None)
                assert ok and n.value == n_tok, (ok, n.value, hex(lib.rwkv_get_last_error(base)))
        return leg

    def host_route():
        if B:
            for i in range(n_tok):
                cur = []
                for b in range(B):
                    assert L.rwkv_b200_batch_get_logits(bt, b, logits.ctypes.data_as(P_F))
                    cur.append(host_top_k(logits, u_rows[b][i]))
                assert L.rwkv_b200_batch_eval(bt, (U32 * B)(*cur), True)
        else:
            for i in range(n_tok):
                assert L.rwkv_b200_stage_logits(base.ptr, logits.ctypes.data_as(P_F), None)
                tok = host_top_k(logits, u_rows[0][i])
                assert L.rwkv_b200_eval_resident(base.ptr, (U32 * 1)(tok), 1, True, None)

    def free():
        if B:
            L.rwkv_free(bt)
        lib.rwkv_free(base)

    return free, reset, {"generate": generate, "sampled_off": sampled(sampler()), "top_k40": sampled(sampler(top_k=TOP_K)),
                         "min_p05": sampled(sampler(min_p=MIN_P)), "all": sampled(sampler(TOP_K, MIN_P, True)), "host_top_k": host_route}


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
