"""Everything a context allocates goes with it: a clone and a batch context that build every lazily allocated set (bounce buffers,
scoring, sampling, generation of every kind, traces, profiling records, adapter scratch, ragged maps, beam search), an adapter and an
automaton, created and freed round after round, leave the device's free memory where the first round left it. Pinned host memory is
not visible here."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
P_F, P_U, P_U8, P_D, P16 = (ctypes.POINTER(t) for t in (ctypes.c_float, ctypes.c_uint32, ctypes.c_uint8, ctypes.c_double, ctypes.c_uint16))
B = 4                         # sequences of the batch context: beam searches of 1 x 4 and 2 x 2
DEFAULT_BOUNCE_MIN = 4 << 20  # engine.cu: g_bounce_min_bytes


def ptr(a, t):
    return a.ctypes.data_as(t)


def exercise(lib, base, toks, V, C):
    """One round: a clone and a batch context build every set, then they, an adapter and an automaton are freed."""
    import rwkv_cpp_b200.shared_library as sl
    L = lib.library
    clone = lib.rwkv_clone_context(base, 1)
    c = clone.ptr
    batch = sl.RWKVContext(L.rwkv_b200_batch_create(c, B))
    adapter = automaton = None
    try:
        assert batch.ptr
        u = np.full(8, 0.5, np.float64)
        out, n = np.zeros(8, np.uint32), ctypes.c_size_t()
        no_fn, go_on = sl.RWKV_TOKEN_FN(), sl.RWKV_TOKEN_FN(lambda user, seq, i, tok: 0)

        # the overlapped eval with pageable (numpy) state in and out: copy streams, bounce buffers and their helper threads
        L.rwkv_b200_set_overlap(c, True)
        n_state = lib.rwkv_get_state_len(clone)
        s0, s1, logits = np.zeros(n_state, np.float32), np.zeros(n_state, np.float32), np.zeros(V, np.float32)
        lib.rwkv_eval(clone, int(toks[0]), None, s0.ctypes.data, logits.ctypes.data)
        lib.rwkv_eval(clone, int(toks[1]), s0.ctypes.data, s1.ctypes.data, logits.ctypes.data)
        # scoring on the GEMV head (8 tokens) and on the tensor-core head (40)
        for k in (8, 40):
            lp, g = np.zeros(k, np.float32), np.zeros(k, np.uint8)
            assert L.rwkv_b200_score(c, ptr(toks[:k], P_U), ptr(toks[1:k + 1], P_U), k, ptr(lp, P_F), ptr(g, P_U8))
        tok, ids, vals = ctypes.c_uint32(), np.array([3], np.uint32), np.array([1.0], np.float32)
        assert L.rwkv_b200_sample(c, 1.0, 1.0, 0.5, ptr(ids, P_U), ptr(vals, P_F), 1, ctypes.byref(tok))
        # blocking, streaming, constrained, logprob (streaming: the ring too) and sampled generation
        assert L.rwkv_b200_generate(c, 4, 1.0, 1.0, 0.0, 0.0, False, ptr(u, P_D), None, 0, ptr(out, P_U), ctypes.byref(n))
        assert L.rwkv_b200_generate_stream(c, 4, 1.0, 1.0, 0.0, 0.0, False, ptr(u, P_D), None, 0, go_on, None, ptr(out, P_U), ctypes.byref(n))
        table = np.zeros(V, np.uint16)                # one state that allows every token
        automaton = L.rwkv_b200_automaton_create(c, ptr(table, P16), 1)
        assert automaton
        st = np.zeros(1, np.uint32)
        assert L.rwkv_b200_generate_constrained(c, automaton, ptr(st, P_U), 4, 1.0, 1.0, 0.0, 0.0, False, ptr(u, P_D), None, 0, no_fn, None,
                                                ptr(out, P_U), ctypes.byref(n))
        lps, top_ids, top_lps = np.zeros(4, np.float32), np.zeros(8, np.uint32), np.zeros(8, np.float32)
        req = sl.Logprobs(top_n=2, logprobs=ptr(lps, P_F), top_ids=ptr(top_ids, P_U), top_logprobs=ptr(top_lps, P_F), sample_probs=None)
        assert L.rwkv_b200_generate_logprobs(c, None, None, 4, 1.0, 1.0, 0.0, 0.0, False, ptr(u, P_D), None, 0, go_on, None, ptr(out, P_U),
                                             ctypes.byref(n), ctypes.byref(req))
        smp = sl.Sampler(temperature=1.0, top_p=1.0, top_k=8, min_p=0.0, presence_penalty=0.0, frequency_penalty=0.0, n_bias=1,
                         bias_ids=ptr(ids, P_U), bias_values=ptr(vals, P_F))
        assert L.rwkv_b200_generate_sampled(c, ctypes.byref(smp), None, None, 4, False, ptr(u, P_D), None, 0, no_fn, None, ptr(out, P_U),
                                            ctypes.byref(n), None)
        # the trace buffer, profiling records, and the scratch of an adapter attached, used and detached
        assert L.rwkv_b200_trace_enable(c)
        assert L.rwkv_b200_eval_resident(c, ptr(toks[:1], P_U), 1, True, None)
        L.rwkv_b200_trace_disable(c)
        assert L.rwkv_b200_profile_pass(c, ptr(toks[:1], P_U), 1, True, ctypes.byref(sl.ProfileResult()))
        rng = np.random.default_rng(0)
        a = (rng.standard_normal((2, C)) * C ** -0.5).astype(np.float32)
        b = (rng.standard_normal((C, 2)) * 0.05).astype(np.float32)
        adapter = lib.rwkv_b200_adapter_create(clone, [("blocks.0.att.key.weight", 2, a, b, None)], 1.0)
        lib.rwkv_b200_set_adapter(clone, adapter)
        assert L.rwkv_b200_eval_resident(c, ptr(toks[:1], P_U), 1, True, None)
        lib.rwkv_b200_set_adapter(clone, None)

        # the batch: ragged eval and score (20 columns: the tensor-core head), biased sampling, generation, beam search at two group counts
        bt = batch.ptr
        counts = np.array([3, 0, 2, 1], np.uint32)
        assert L.rwkv_b200_batch_eval_ragged(bt, ptr(toks[:6], P_U), ptr(counts, P_U), True)
        counts = np.array([8, 4, 0, 8], np.uint32)
        lp, g = np.zeros(20, np.float32), np.zeros(20, np.uint8)
        assert L.rwkv_b200_batch_score_ragged(bt, ptr(toks[:20], P_U), ptr(counts, P_U), ptr(toks[1:21], P_U), ptr(lp, P_F), ptr(g, P_U8))
        ones, half = np.ones(B, np.float32), np.full(B, 0.5, np.float64)
        offsets, bias_ids, bias_vals = np.array([0, 1, 1, 1, 2], np.uint32), np.array([5, 9], np.uint32), np.array([1.0, -1.0], np.float32)
        drawn = np.zeros(B, np.uint32)
        assert L.rwkv_b200_batch_sample(bt, ptr(ones, P_F), ptr(ones, P_F), ptr(half, P_D), ptr(offsets, P_U), ptr(bias_ids, P_U),
                                        ptr(bias_vals, P_F), ptr(drawn, P_U))
        zeros, mt, us = np.zeros(B, np.float32), np.full(B, 3, np.uint32), np.full(B * 3, 0.5, np.float64)
        gen, ng = np.zeros(B * 3, np.uint32), np.zeros(B, np.uint32)
        assert L.rwkv_b200_batch_generate(bt, ptr(mt, P_U), ptr(ones, P_F), ptr(ones, P_F), ptr(zeros, P_F), ptr(zeros, P_F), None, ptr(us, P_D),
                                          None, 0, ptr(gen, P_U), ptr(ng, P_U))
        lib.rwkv_b200_beam_search_groups(batch, 1, [4], [1.0])
        lib.rwkv_b200_beam_search_groups(batch, 2, [6, 3], [1.0, 0.5])
    finally:
        if batch.ptr:
            lib.rwkv_free(batch)
        lib.rwkv_free(clone)
        if adapter:
            lib.rwkv_b200_adapter_free(adapter)
        if automaton:
            L.rwkv_b200_automaton_free(automaton)


def test_freed_contexts_give_back_their_device_memory(lib, tmp_path):
    """Round 1 also loads the kernels' modules and builds the model's tile-major head, which live as long as the process and the
    model; every later round must end within 4 MiB of where round 1 ended."""
    import torch
    import synthetic_model as sm
    path = str(tmp_path / "rwkv5-1b5-Q5_1.bin")
    sm.write_direct(path, "rwkv5-1b5", "Q5_1", seed=11)
    p = sm.PRESETS["rwkv5-1b5"]
    toks = np.ascontiguousarray(sm.synthetic_tokens(64, p["V"]), np.uint32)
    torch.cuda.mem_get_info(0)                        # torch's own set-up happens before the first round, not between rounds
    base = lib.rwkv_init_from_file(path, 1)           # holds the model between rounds
    lib.library.rwkv_b200_set_bounce_min_bytes(0)
    try:
        free = []
        for _ in range(4):
            exercise(lib, base, toks, p["V"], p["C"])
            free.append(torch.cuda.mem_get_info(0)[0])
        drift = [free[0] - f for f in free[1:]]
        assert all(abs(d) <= 4 << 20 for d in drift), drift
    finally:
        lib.library.rwkv_b200_set_bounce_min_bytes(DEFAULT_BOUNCE_MIN)
        lib.rwkv_free(base)
