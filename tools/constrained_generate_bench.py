"""Constrained generation against the unconstrained loop and the host loop a caller needs without it (DESIGN.md 6.4.2). Measurement
aid, not a bench line.

  7b-b1  : the synthetic RWKV-6-World-7B Q5_1 (n_vocab 65536), one sequence, max_tokens = 256 per leg:
             generate      rwkv_b200_generate
             all_allowed   rwkv_b200_generate_constrained with a one-state automaton that allows every token
             sparse_256    rwkv_b200_generate_constrained with a seeded 256-state automaton allowing ~10 % of the tokens per state
             host_loop     per token: a -inf bias list over the forbidden tokens + penalties, rwkv_b200_sample, rwkv_b200_eval_resident
  7b-b16 : the same shape, a 16-sequence batch: rwkv_b200_batch_generate against rwkv_b200_batch_generate_constrained with the
           256-state automaton on every sequence

Every leg draws with temperature 1 and top_p 0.8, without penalties or stop ids, and every state of the automata allows some
token, so every leg runs exactly 256 passes. A leg is timed with the host clock around the call, which returns after a
synchronise; the legs of a case alternate, and the result is the median over rounds in milliseconds per generated token (per step
for the batch) with min / max. The card's name and power limit are read in the same run.

    python tools/constrained_generate_bench.py [--rounds 5] [--tokens 256] [--out FILE.json]
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

U16, U32, F32, F64 = ctypes.c_uint16, ctypes.c_uint32, ctypes.c_float, ctypes.c_double
TEMPERATURE, TOP_P = 1.0, 0.8
DEAD = 0xFFFF


def sparse_table(n_states, n_vocab, share, seed):
    """A seeded automaton: each token allowed in a state with probability `share`, to a random state; every state allows one."""
    rng = np.random.RandomState(seed)
    table = np.where(rng.rand(n_states, n_vocab) < share, rng.randint(0, n_states, size=(n_states, n_vocab)), DEAD).astype(np.uint16)
    table[np.arange(n_states), rng.randint(0, n_vocab, size=n_states)] = rng.randint(0, n_states, size=n_states)
    return np.ascontiguousarray(table)


def automaton(lib, ctx_ptr, table):
    a = lib.library.rwkv_b200_automaton_create(ctx_ptr, table.ctypes.data_as(ctypes.POINTER(U16)), table.shape[0])
    assert a
    return a


def single_legs(lib, path, n_tok):
    from rwkv_cpp_b200.shared_library import RWKV_TOKEN_FN
    L = lib.library
    ctx = lib.rwkv_b200_init_from_file_ex(path, 0, 0, -1)
    V = lib.rwkv_get_logits_buffer_element_count(ctx)
    us = uniforms(n_tok, 1)
    u_arr = (F64 * n_tok)(*us)
    toks = (U32 * n_tok)()
    n = ctypes.c_size_t(0)
    sparse = sparse_table(256, V, 0.1, 7)
    a_all, a_sparse = automaton(lib, ctx.ptr, np.zeros((1, V), np.uint16)), automaton(lib, ctx.ptr, sparse)
    null_fn = RWKV_TOKEN_FN()
    dead_ids = [np.nonzero(sparse[s] == DEAD)[0].astype(np.uint32) for s in range(sparse.shape[0])]

    def reset():
        assert L.rwkv_b200_state_load(ctx.ptr, None)
        assert L.rwkv_b200_eval_resident(ctx.ptr, (U32 * 1)(11), 1, True, None)
        assert L.rwkv_b200_synchronize(ctx.ptr)

    def generate():
        assert L.rwkv_b200_generate(ctx.ptr, n_tok, TEMPERATURE, TOP_P, 0.0, 0.0, False, u_arr, None, 0, toks, ctypes.byref(n)) and n.value == n_tok

    def constrained(a):
        def leg():
            st = U32(0)
            assert L.rwkv_b200_generate_constrained(ctx.ptr, a, ctypes.byref(st), n_tok, TEMPERATURE, TOP_P, 0.0, 0.0, False, u_arr, None, 0, null_fn, None,
                                                    toks, ctypes.byref(n)) and n.value == n_tok
        return leg

    def host_loop():
        st, tok = 0, U32(0)
        one = (U32 * 1)()
        for i in range(n_tok):
            ids = dead_ids[st]
            vals = np.full(len(ids), -np.inf, np.float32)
            assert L.rwkv_b200_sample(ctx.ptr, TEMPERATURE, TOP_P, us[i], ids.ctypes.data_as(ctypes.POINTER(U32)), vals.ctypes.data_as(ctypes.POINTER(F32)),
                                      len(ids), ctypes.byref(tok))
            st = int(sparse[st, tok.value])
            one[0] = tok.value
            assert L.rwkv_b200_eval_resident(ctx.ptr, one, 1, True, None)
        assert L.rwkv_b200_synchronize(ctx.ptr)

    def free():
        L.rwkv_b200_automaton_free(a_all)
        L.rwkv_b200_automaton_free(a_sparse)
        lib.rwkv_free(ctx)

    return free, reset, {"generate": generate, "all_allowed": constrained(a_all), "sparse_256": constrained(a_sparse), "host_loop": host_loop}


def batch_legs(lib, path, n_tok, B):
    from rwkv_cpp_b200.shared_library import RWKV_TOKEN_FN
    L = lib.library
    base = lib.rwkv_b200_init_from_file_ex(path, 0, 0, -1)
    V = lib.rwkv_get_logits_buffer_element_count(base)
    bt = ctypes.c_void_p(L.rwkv_b200_batch_create(base.ptr, B))
    assert bt
    a_sparse = automaton(lib, base.ptr, sparse_table(256, V, 0.1, 7))
    automata = (ctypes.c_void_p * B)(*[a_sparse] * B)
    temps, top_ps, zeros = (F32 * B)(*[TEMPERATURE] * B), (F32 * B)(*[TOP_P] * B), (F32 * B)()
    budgets = (U32 * B)(*[n_tok] * B)
    u_arr = (F64 * (B * n_tok))(*[u for b in range(B) for u in uniforms(n_tok, 100 + b)])
    toks, ng = (U32 * (B * n_tok))(), (U32 * B)()
    null_fn = RWKV_TOKEN_FN()

    def reset():
        for b in range(B):
            assert L.rwkv_b200_batch_set_state(bt, b, None)
        assert L.rwkv_b200_batch_eval(bt, (U32 * B)(*[11 + b for b in range(B)]), True)
        assert L.rwkv_b200_synchronize(bt)

    def generate():
        assert L.rwkv_b200_batch_generate(bt, budgets, temps, top_ps, zeros, zeros, None, u_arr, None, 0, toks, ng)
        assert all(ng[b] == n_tok for b in range(B))

    def constrained():
        states = (U32 * B)()
        assert L.rwkv_b200_batch_generate_constrained(bt, automata, states, budgets, temps, top_ps, zeros, zeros, None, u_arr, None, 0, null_fn, None,
                                                      toks, ng)
        assert all(ng[b] == n_tok for b in range(B))

    def free():
        L.rwkv_b200_automaton_free(a_sparse)
        L.rwkv_free(bt)
        lib.rwkv_free(base)

    return free, reset, {"generate": generate, "sparse_256": constrained}


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
    free, reset, legs = single_legs(lib, path7b, args.tokens)
    results["7b-b1"] = measure(reset, legs, args.rounds, args.tokens)
    free()
    free, reset, legs = batch_legs(lib, path7b, args.tokens, 16)
    results["7b-b16"] = measure(reset, legs, args.rounds, args.tokens)
    free()
    line = json.dumps(results)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
