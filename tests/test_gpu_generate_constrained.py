"""Constrained generation (rwkv_b200_generate_constrained / rwkv_b200_batch_generate_constrained, the table-mask step kernels of
csrc/kernels/sampling.cu): the whole loop must give, byte for byte, the tokens, state, logits and automaton state of the host loop a
caller needs without it -- rwkv_b200_sample with -inf on every token the automaton's state does not allow (in place of the penalty)
plus rwkv_b200_eval_resident -- and an automaton that allows everything must give the bytes of the unconstrained calls. The tiny
fixtures' vocabulary is the 256 bytes, so the byte DFAs of tests/byte_dfa.py are token automata."""
import ctypes
from collections import Counter

import numpy as np
import pytest

import byte_dfa as bd
import generate_ref as gr
import sampling_oracle as so
from conftest import LONG_PROMPT, model_path
from generate_ref import P_D, P_F, P_U
from test_gpu_generate import ERR_ARGS, ERR_CTX, ERR_UNSUPPORTED, P_U8, Batch, Pair, bias_arrays, f32, generate, logits, ptr, state
from test_gpu_generate_stream import NULL_FN, Recorder, generate_stream

P16 = ctypes.POINTER(ctypes.c_uint16)
NONE = 0xFFFFFFFF


class Automaton:
    def __init__(self, lib, ctx_ptr, table):
        self.lib, self.table = lib, np.ascontiguousarray(table, np.uint16)
        self.ptr = lib.library.rwkv_b200_automaton_create(ctx_ptr, self.table.ctypes.data_as(P16), self.table.shape[0])
        assert self.ptr, lib.rwkv_get_last_error(None)

    def free(self):
        self.lib.library.rwkv_b200_automaton_free(self.ptr)


def all_allowed(n_vocab):
    return np.zeros((1, n_vocab), np.uint16)


def mask_bias(row, counts, presence, frequency):
    bias = gr.penalty_bias(counts, presence, frequency)
    for t in np.nonzero(row == bd.DEAD)[0]:
        bias[int(t)] = float("-inf")
    return bias


def host_constrained(lib, ctx_ptr, table, st, max_tokens, temperature, top_p, presence, frequency, us, stops=(), counts=None):
    """The host loop: returns (tokens, final state)."""
    counts = Counter() if counts is None else counts
    out = []
    for i in range(max_tokens):
        row = table[st]
        if not (row != bd.DEAD).any():
            break
        tok = gr.sample(lib, ctx_ptr, temperature, top_p, us[i], mask_bias(row, counts, presence, frequency))
        out.append(tok)
        if tok in stops:
            break
        counts[tok] += 1
        gr.eval_token(lib, ctx_ptr, tok)
        if row[tok] != bd.DEAD:
            st = int(row[tok])
    return out, st


def gen_constrained(lib, ctx_ptr, auto_ptr, st, max_tokens, temperature, top_p, presence, frequency, us, stops=(), keep=False, rec=None, st_ptr=True):
    toks = np.zeros(max(max_tokens, 1), np.uint32)
    n = ctypes.c_size_t(0)
    s = np.array([st], np.uint32)
    sp = np.array(stops, np.uint32) if len(stops) else None
    ok = lib.library.rwkv_b200_generate_constrained(ctx_ptr, auto_ptr, s.ctypes.data_as(P_U) if st_ptr else None, max_tokens, temperature, top_p, presence,
                                                    frequency, keep, ptr(np.asarray(us, np.float64), P_D), ptr(sp, P_U), len(stops),
                                                    rec.fn if rec else NULL_FN, None, ptr(toks, P_U), ctypes.byref(n))
    return ok, [int(t) for t in toks[:n.value]], int(s[0])


def batch_constrained(bt, automata, states, max_tokens, temps, top_ps, pres, freq, us, stops=(), keep=None, rec=None):
    n = max(max_tokens)
    toks = np.zeros(bt.n * max(n, 1), np.uint32)
    ng = np.zeros(bt.n, np.uint32)
    st = np.array(states, np.uint32)
    arr = (ctypes.c_void_p * bt.n)(*[a.ptr if a else None for a in automata])
    sp = np.array(stops, np.uint32) if len(stops) else None
    ok = bt.lib.library.rwkv_b200_batch_generate_constrained(
        bt.ptr, arr, ptr(st, P_U), ptr(np.asarray(max_tokens, np.uint32), P_U), ptr(f32(temps), P_F), ptr(f32(top_ps), P_F), ptr(f32(pres), P_F),
        ptr(f32(freq), P_F), ptr(None if keep is None else np.asarray(keep, np.uint8), P_U8), ptr(np.ascontiguousarray(us, np.float64), P_D), ptr(sp, P_U),
        len(stops), rec.fn if rec else NULL_FN, None, ptr(toks, P_U), ptr(ng, P_U))
    return ok, [[int(t) for t in toks[b * n:b * n + ng[b]]] for b in range(bt.n)], [int(x) for x in st]


def check_text(dfa, toks, start, end, stops=()):
    """The generated text is a prefix the DFA accepts from `start`, ending in state `end`; a full match when it ended in a dead end."""
    text = [t for t in toks if t not in stops]
    assert dfa.walk(text, start) == end, (toks, start, end)
    if dfa.dead_end(end) and start == 0:
        assert dfa.fullmatch(bytes(text)), bytes(text)


# ---- 1. the step hook ------------------------------------------------------------------------------------------------------------

def hook_constrained(lib, logits, table, states, max_tokens, temps, top_ps, pres, freq, us, stops, step, frozen, counts, tokens):
    R, V = logits.shape
    step, frozen, counts, tokens = np.array(step, np.uint32), np.array(frozen, np.uint8), counts.copy(), tokens.copy()
    nxt, any_active = np.zeros(R, np.int32), ctypes.c_uint32(7)
    st = np.array(stops, np.uint32) if len(stops) else None
    mt, t, p, pr, fr, u = (np.asarray(max_tokens, np.uint32), f32(temps), f32(top_ps), f32(pres), f32(freq), np.ascontiguousarray(us, np.float64))
    s = np.array(states, np.uint32)
    a = gr.StepArgs(logits=logits.ctypes.data, n_rows=R, n_vocab=V, max_tokens=mt.ctypes.data, temperature=t.ctypes.data, top_p=p.ctypes.data,
                    presence_penalty=pr.ctypes.data, frequency_penalty=fr.ctypes.data, u=u.ctypes.data, stop_ids=None if st is None else st.ctypes.data,
                    n_stop=len(stops), step=step.ctypes.data, frozen=frozen.ctypes.data, counts=counts.ctypes.data, tokens=tokens.ctypes.data,
                    next_tokens=nxt.ctypes.data, any_active=ctypes.addressof(any_active))
    ok = lib.library.rwkv_b200_test_generate_step_constrained(ctypes.byref(a), table.ctypes.data_as(P16), table.shape[0], s.ctypes.data_as(P_U))
    return ok, step, frozen, counts, tokens, nxt, any_active.value, [int(x) for x in s]


@pytest.mark.gpu
@pytest.mark.parametrize("V", [7, 1000, 16384, 50277, 65536])
def test_constrained_step_hook(lib, V):
    """One step at every instantiation. Rows: unconstrained, three constrained states (one allows a single token), a dead-end state,
    a row whose draw is a stop id, a frozen row, a row at its budget. Each drawing row is bit for bit rwkv_b200_sample_logits_batch
    with the -inf + penalty bias lists, and the oracle's draw away from knife edges."""
    rng = np.random.RandomState(V + 3)
    n_states = 5
    table = np.where(rng.rand(n_states, V) < 0.1, rng.randint(0, n_states, size=(n_states, V)), bd.DEAD).astype(np.uint16)
    table[0, rng.randint(V)] = 1                  # every state but 3 allows something; state 2 allows exactly one token
    table[1, rng.randint(V)] = 2
    table[2] = bd.DEAD
    table[2, V // 2] = 4
    table[3] = bd.DEAD                            # a dead end
    table[4, 0] = 0
    R = 8
    logits = (rng.standard_normal((R, V)) * 3.0).astype(np.float32)
    states = [NONE, 0, 1, 2, 3, 4, 0, 1]
    max_tokens = [3, 3, 4, 2, 5, 3, 2, 3]
    step = [1, 0, 2, 0, 1, 1, 0, 3]
    frozen = [0, 0, 0, 0, 0, 0, 1, 0]
    temps, top_ps = [1.0, 0.8, 0.0, 1.0, 1.0, 1.3, 1.0, 1.0], [0.9, 1.0, 1.0, 0.5, 1.0, 0.0, 1.0, 1.0]
    pres, freq = [0.2, 0.0, 0.5, 1.0, 0.3, 0.1, 0.0, 0.2], [0.2, 0.7, 0.0, 1.5, 0.1, 0.2, 0.0, 0.0]
    n = max(max_tokens)
    us = rng.random_sample((R, n))
    counts = np.zeros((R, V), np.uint32)
    for b in range(R):
        ids = rng.choice(V, size=min(5, V), replace=False)
        counts[b, ids] = rng.randint(0, 4, size=len(ids))
    tokens = np.full((R, n), 5, np.uint32)
    live = lambda b: states[b] == NONE or (table[states[b]] != bd.DEAD).any()
    drawing = [b for b in range(R) if not frozen[b] and step[b] < max_tokens[b] and live(b)]
    cnt = lambda b: {i: int(c) for i, c in enumerate(counts[b]) if c}
    biases = [None if b not in drawing else gr.penalty_bias(cnt(b), pres[b], freq[b]) if states[b] == NONE else mask_bias(table[states[b]], cnt(b), pres[b], freq[b])
              for b in range(R)]
    off, ids, vals = bias_arrays(biases)
    ref = np.zeros(R, np.uint32)
    u_now = np.array([us[b][min(step[b], n - 1)] for b in range(R)])
    assert lib.library.rwkv_b200_sample_logits_batch(ptr(logits, P_F), R, V, ptr(f32(temps), P_F), ptr(f32(top_ps), P_F), ptr(u_now, P_D), ptr(off, P_U),
                                                      ptr(ids, P_U), ptr(vals, P_F), ptr(ref, P_U), None)
    stops = [int(ref[5])]                         # row 5 draws a stop id, which its state allows
    ok, s2, f2, c2, t2, nxt, any_active, st2 = hook_constrained(lib, logits, table, states, max_tokens, temps, top_ps, pres, freq, us, stops, step, frozen,
                                                                counts, tokens)
    assert ok
    drawn = [int(ref[b]) if b in drawing else None for b in range(R)]
    # the bookkeeping: a dead-end row freezes without drawing, as a row at its budget does
    want_step, want_frozen = list(step), list(frozen)
    for b in range(R):
        if frozen[b]:
            continue
        if step[b] == max_tokens[b] or not live(b):
            want_frozen[b] = 1
            continue
        want_step[b] += 1
        if drawn[b] in stops:
            want_frozen[b] = 1
    assert list(s2) == want_step and list(f2) == want_frozen and any_active == int(any(not f for f in want_frozen))
    want_counts, want_tokens, want_states = counts.copy(), tokens.copy(), list(states)
    for b in drawing:
        want_tokens[b, step[b]] = drawn[b]
        if states[b] != NONE:
            assert table[states[b], drawn[b]] != bd.DEAD, b        # the draw is one the state allows
        if drawn[b] in stops:
            continue                                               # a stop id does not advance the state
        want_counts[b, drawn[b]] += 1
        if states[b] != NONE:
            want_states[b] = int(table[states[b], drawn[b]])
    assert np.array_equal(t2, want_tokens) and np.array_equal(c2, want_counts)
    assert st2 == want_states
    assert list(nxt) == [drawn[b] if not want_frozen[b] else 0 for b in range(R)]
    assert drawn[3] == V // 2
    # the oracle, away from knife-edge draws
    compared = 0
    for b in drawing:
        if so.boundary_distance(logits[b], temps[b], top_ps[b], u_now[b], biases[b]) > 1e-6:
            assert so.sample_logits_u(logits[b], temps[b], top_ps[b], u_now[b], biases[b]) == drawn[b], b
            compared += 1
    assert compared >= 3


# ---- 2. whole models against the host loop ---------------------------------------------------------------------------------------

CASES = [  # max_tokens, temperature, top_p, presence, frequency
    (12, 0.0, 1.0, 0.0, 0.0),
    (12, 1.0, 0.9, 0.0, 0.0),
    (11, 1.0, 1.0, 0.3, 0.4),
    (5, 0.7, 0.8, 0.2, 0.2),
]


@pytest.mark.gpu
@pytest.mark.parametrize("ver", ["4v0-660K", "5v1-730K", "5v2-730K", "6v0-3m", "7v0-834K"])
@pytest.mark.parametrize("fmt", ["FP32", "Q5_1"])
def test_generate_constrained_equals_host_loop(lib, ver, fmt):
    ctx = lib.rwkv_init_from_file(model_path(ver, fmt), 1, 0)
    pair = Pair(lib, ctx)
    num, words = bd.ByteDFA(bd.NUMBER), bd.ByteDFA(bd.WORDS, eos=0)
    a_num, a_words = Automaton(lib, ctx.ptr, num.next), Automaton(lib, ctx.ptr, words.next)
    try:
        L = lib.library
        rng = np.random.RandomState(sum(map(ord, ver + fmt)) + 1)
        prompt = LONG_PROMPT[:5]
        ended = 0
        for dfa, auto, stops in [(num, a_num, ()), (words, a_words, (0,))]:
            for case in CASES:
                mt, t, p, pres, freq = case
                us = rng.random_sample(mt)
                pair.prime(prompt)
                want, want_st = host_constrained(lib, pair.host.ptr, dfa.next, 0, mt, t, p, pres, freq, us, stops)
                ok, got, got_st = gen_constrained(lib, pair.dev.ptr, auto.ptr, 0, mt, t, p, pres, freq, us, stops)
                assert ok and got == want and got_st == want_st, (case, stops, got, want)
                pair.same((case, stops))
                check_text(dfa, got, 0, got_st, stops)
                if stops and got and got[-1] in stops:
                    assert dfa.accepting[got_st]
                ended += dfa.dead_end(got_st) or bool(stops and got and got[-1] in stops)
                # the state buffers after an odd or even number of passes: later calls still follow the host loop
                tok_h, tok_d = ctypes.c_uint32(0), ctypes.c_uint32(0)
                u = float(rng.random_sample())
                assert L.rwkv_b200_eval_sample(pair.host.ptr, 17, 1.0, 0.9, u, ctypes.byref(tok_h))
                assert L.rwkv_b200_eval_sample(pair.dev.ptr, 17, 1.0, 0.9, u, ctypes.byref(tok_d))
                assert tok_h.value == tok_d.value, case
                pair.same(("after", case))
        assert ended >= 2, "no sequence reached the end of its pattern"
    finally:
        a_num.free()
        a_words.free()
        pair.free()
        lib.rwkv_free(ctx)


# ---- 3. an automaton that allows everything --------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("ver,fmt", [("6v0-3m", "Q5_1"), ("7v0-834K", "FP32"), ("4v0-660K", "FP32")])
def test_all_allowed_automaton_equals_generate(lib, ver, fmt):
    """Blocking and streaming, with penalties and a stop id; a following keep_counts call of the plain generate agrees as well."""
    ctx = lib.rwkv_init_from_file(model_path(ver, fmt), 1, 0)
    pair = Pair(lib, ctx)
    auto = Automaton(lib, ctx.ptr, all_allowed(pair.n_vocab))
    try:
        rng = np.random.RandomState(11)
        prompt = LONG_PROMPT[:4]
        for streaming in (False, True):
            for mt, t, p, pres, freq in [(9, 1.0, 0.9, 0.2, 0.3), (8, 0.0, 1.0, 0.5, 0.5), (7, 1.3, 0.6, 0.0, 0.0)]:
                us = rng.random_sample(mt)
                pair.prime(prompt)
                ok, free_run = generate(lib, pair.host.ptr, mt, t, p, pres, freq, us)
                assert ok
                stops = (free_run[4],) if mt == 7 else ()     # a stop id hit mid-way
                pair.prime(prompt)
                ok, want = generate(lib, pair.host.ptr, mt, t, p, pres, freq, us, stops)
                assert ok and (not stops or want[-1] == stops[0])
                rec = Recorder() if streaming else None
                ok, got, st = gen_constrained(lib, pair.dev.ptr, auto.ptr, 0, mt, t, p, pres, freq, us, stops, rec=rec)
                assert ok and got == want and st == 0, (streaming, mt)
                if rec:
                    assert rec.delivered(0) == got
                pair.same((streaming, mt))
                follow = rng.random_sample(4)
                ok, want = generate(lib, pair.host.ptr, 4, 1.0, 1.0, pres, freq, follow, keep=True)
                ok2, got = generate(lib, pair.dev.ptr, 4, 1.0, 1.0, pres, freq, follow, keep=True)
                assert ok and ok2 and got == want, ("follow-up", streaming, mt)
                pair.same(("follow-up", streaming, mt))
    finally:
        auto.free()
        pair.free()
        lib.rwkv_free(ctx)


# ---- 4. batches ------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("ver,fmt", [("6v0-3m", "FP32"), ("7v0-834K", "Q5_1")])
def test_batch_constrained_rows_equal_each_sequence_alone(lib, ver, fmt):
    """B = 4: two automata, a NULL row, a budget of 0 and a dead start state; each row equals its sequence alone in a single
    context (the NULL row: rwkv_b200_generate), state, logits and automaton state included. The automaton of row 2 was created from
    a clone: it serves every context of the model."""
    ctx = lib.rwkv_init_from_file(model_path(ver, fmt), 1, 0)
    alone = lib.rwkv_clone_context(ctx, 1)
    num, words = bd.ByteDFA(bd.NUMBER), bd.ByteDFA(bd.WORDS, eos=0)
    a_num, a_words = Automaton(lib, ctx.ptr, num.next), Automaton(lib, alone.ptr, words.next)
    dead = num.walk(b"7;")
    bt = Batch(lib, ctx, 4)
    try:
        n_state, n_vocab = lib.rwkv_get_state_buffer_element_count(ctx), lib.rwkv_get_logits_buffer_element_count(ctx)
        rng = np.random.RandomState(4)
        automata = [a_num, None, a_words, a_num]
        dfas = [num, None, words, num]
        states = [0, 0, 0, dead]
        max_tokens = [10, 6, 0, 5]
        prompts = [[(37 * b + 5 * i + 3) % n_vocab for i in range(2)] for b in range(4)]
        bt.prime(prompts)
        before = [(bt.state(b, n_state).tobytes(), bt.logits(b, n_vocab).tobytes()) for b in range(4)]
        temps, top_ps, pres, freq = [1.0, 0.7, 0.0, 1.0], [0.9, 1.0, 1.0, 0.8], [0.2, 0.0, 0.3, 0.1], [0.3, 0.2, 0.1, 0.0]
        us = rng.random_sample((4, max(max_tokens)))
        ok, got, st = batch_constrained(bt, automata, states, max_tokens, temps, top_ps, pres, freq, us, (0,))
        assert ok
        for b in (2, 3):      # budget 0, dead start state: nothing generated, nothing changed
            assert got[b] == [] and st[b] == states[b]
            assert (bt.state(b, n_state).tobytes(), bt.logits(b, n_vocab).tobytes()) == before[b], b
        for b in (0, 1):
            assert lib.library.rwkv_b200_state_load(alone.ptr, None)
            for t in prompts[b]:
                gr.eval_token(lib, alone.ptr, t)
            if automata[b]:
                ok, want, want_st = gen_constrained(lib, alone.ptr, automata[b].ptr, states[b], max_tokens[b], temps[b], top_ps[b], pres[b], freq[b], us[b], (0,))
            else:
                (ok, want), want_st = generate(lib, alone.ptr, max_tokens[b], temps[b], top_ps[b], pres[b], freq[b], us[b], (0,)), states[b]
            assert ok and got[b] == want and st[b] == want_st, (b, got[b], want)
            assert bt.state(b, n_state).tobytes() == state(lib, alone.ptr, n_state).tobytes(), b
            assert bt.logits(b, n_vocab).tobytes() == logits(lib, alone.ptr, n_vocab).tobytes(), b
        check_text(num, got[0], 0, st[0], (0,))
    finally:
        bt.free()
        a_num.free()
        a_words.free()
        lib.rwkv_free(alone)
        lib.rwkv_free(ctx)


@pytest.mark.gpu
def test_batch_16_constrained_and_null_rows(lib):
    """B = 16 (the tensor-core path): constrained rows satisfy their patterns, NULL rows equal rwkv_b200_batch_generate."""
    ctx = lib.rwkv_init_from_file(model_path("6v0-3m", "Q5_1"), 1, 0)
    num, words = bd.ByteDFA(bd.NUMBER), bd.ByteDFA(bd.WORDS, eos=0)
    a_num, a_words = Automaton(lib, ctx.ptr, num.next), Automaton(lib, ctx.ptr, words.next)
    B = 16
    bc, bp = Batch(lib, ctx, B), Batch(lib, ctx, B)
    try:
        n_state, n_vocab = lib.rwkv_get_state_buffer_element_count(ctx), lib.rwkv_get_logits_buffer_element_count(ctx)
        rng = np.random.RandomState(16)
        automata = [(a_num, None, a_words, None)[b % 4] for b in range(B)]
        dfas = [(num, None, words, None)[b % 4] for b in range(B)]
        max_tokens = [(12, 8, 10, 0, 5)[b % 5] for b in range(B)]
        temps = [(0.0, 0.7, 1.0, 1.3)[b % 4] for b in range(B)]
        top_ps = [(1.0, 0.6, 0.9, 0.25)[b % 4] for b in range(B)]
        pres = [(0.0, 0.2, 0.5)[b % 3] for b in range(B)]
        freq = [(0.0, 0.2, 0.1, 0.4)[b % 4] for b in range(B)]
        us = rng.random_sample((B, max(max_tokens)))
        prompts = [[(37 * b + 5 * i + 3) % n_vocab for i in range(2)] for b in range(B)]
        bc.prime(prompts)
        bp.prime(prompts)
        ok, got, st = batch_constrained(bc, automata, [0] * B, max_tokens, temps, top_ps, pres, freq, us, (0,))
        ok2, want = bp.generate(max_tokens, temps, top_ps, pres, freq, us, (0,))
        assert ok and ok2
        for b in range(B):
            if automata[b] is None:
                assert got[b] == want[b] and st[b] == 0, b
                assert bc.state(b, n_state).tobytes() == bp.state(b, n_state).tobytes(), b
                assert bc.logits(b, n_vocab).tobytes() == bp.logits(b, n_vocab).tobytes(), b
            else:
                check_text(dfas[b], got[b], 0, st[b], (0,))
                assert len(got[b]) <= max_tokens[b]
    finally:
        bc.free()
        bp.free()
        a_num.free()
        a_words.free()
        lib.rwkv_free(ctx)


# ---- 5. streaming ----------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_constrained_stream_ends_after_token_j(lib):
    """A callback that ends the sequence after token j equals max_tokens = j + 1, automaton state included, single and batch."""
    ctx = lib.rwkv_init_from_file(model_path("6v0-3m", "FP32"), 1, 0)
    pair = Pair(lib, ctx)
    words = bd.ByteDFA(bd.WORDS, eos=0)
    auto = Automaton(lib, ctx.ptr, words.next)
    bh = bs = None
    try:
        rng = np.random.RandomState(5)
        prompt = LONG_PROMPT[:4]
        mt = 9
        for j in (0, 1, 4):
            us = rng.random_sample(mt)
            pair.prime(prompt)
            ok, want, want_st = gen_constrained(lib, pair.host.ptr, auto.ptr, 0, j + 1, 1.0, 0.9, 0.2, 0.3, us[:j + 1])
            assert ok
            rec = Recorder(stop_at={0: j})
            ok, got, st = gen_constrained(lib, pair.dev.ptr, auto.ptr, 0, mt, 1.0, 0.9, 0.2, 0.3, us, rec=rec)
            assert ok and got == want and st == want_st, j
            assert rec.delivered(0) == got
            pair.same(("stop", j))
        B = 4
        n_state, n_vocab = pair.n_state, pair.n_vocab
        bh, bs = Batch(lib, ctx, B), Batch(lib, ctx, B)
        prompts = [[(37 * b + 5 * i + 3) % n_vocab for i in range(2)] for b in range(B)]
        ends = [2, None, 0, 5]
        max_tokens = [8, 6, 7, 9]
        budgets = [m if e is None else e + 1 for e, m in zip(ends, max_tokens)]
        us = rng.random_sample((B, max(max_tokens)))
        automata = [auto, None, auto, auto]
        args = ([1.0] * B, [0.9] * B, [0.1] * B, [0.2] * B)
        bh.prime(prompts)
        bs.prime(prompts)
        ok, want, want_st = batch_constrained(bh, automata, [0] * B, budgets, *args, us[:, :max(budgets)])
        rec = Recorder(stop_at={b: e for b, e in enumerate(ends) if e is not None})
        ok2, got, st = batch_constrained(bs, automata, [0] * B, max_tokens, *args, us, rec=rec)
        assert ok and ok2 and got == want and st == want_st
        for b in range(B):
            assert rec.delivered(b) == got[b], b
            assert bs.state(b, n_state).tobytes() == bh.state(b, n_state).tobytes(), b
            assert bs.logits(b, n_vocab).tobytes() == bh.logits(b, n_vocab).tobytes(), b
    finally:
        for bt in (bh, bs):
            if bt:
                bt.free()
        auto.free()
        pair.free()
        lib.rwkv_free(ctx)


@pytest.mark.gpu
def test_constrained_stream_refuses_reentry(lib):
    ctx = lib.rwkv_init_from_file(model_path("6v0-3m", "FP32"), 1, 0)
    pair = Pair(lib, ctx)
    num = bd.ByteDFA(bd.NUMBER)
    auto = Automaton(lib, ctx.ptr, num.next)
    try:
        L = lib.library
        dev = pair.dev.ptr
        results = []

        def inner(seq, idx, tok):
            if idx == 1:
                ok, _, s = gen_constrained(lib, dev, auto.ptr, 0, 2, 1.0, 1.0, 0.0, 0.0, np.full(2, 0.5))
                results.append((ok, int(L.rwkv_get_last_error(dev)), s))

        us = np.random.RandomState(9).random_sample(8)
        pair.prime(LONG_PROMPT[:3])
        ok, want, want_st = gen_constrained(lib, pair.host.ptr, auto.ptr, 0, 8, 1.0, 0.9, 0.2, 0.2, us)
        rec = Recorder(inner=inner)
        ok2, got, st = gen_constrained(lib, dev, auto.ptr, 0, 8, 1.0, 0.9, 0.2, 0.2, us, rec=rec)
        assert ok and ok2 and got == want and st == want_st and len(got) >= 2
        assert results == [(False, ERR_CTX | ERR_UNSUPPORTED, 0)]
        pair.same("re-entry")
    finally:
        auto.free()
        pair.free()
        lib.rwkv_free(ctx)


# ---- 6. windows ------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("ver,fmt", [("5v2-730K", "Q5_1"), ("7v0-834K", "FP32")])
def test_constrained_windows_equal_one_call(lib, ver, fmt):
    """Two calls passing the automaton state and the counts on (keep_counts, the same u) equal one call over the whole window."""
    ctx = lib.rwkv_init_from_file(model_path(ver, fmt), 1, 0)
    pair = Pair(lib, ctx)
    words = bd.ByteDFA(bd.WORDS, eos=0)
    auto = Automaton(lib, ctx.ptr, words.next)
    try:
        rng = np.random.RandomState(6)
        for split in (1, 3, 5):
            us = rng.random_sample(12)
            pair.prime(LONG_PROMPT[:5])
            ok, whole, whole_st = gen_constrained(lib, pair.host.ptr, auto.ptr, 0, 12, 1.0, 1.0, 0.3, 0.5, us, (0,))
            ok1, first, st = gen_constrained(lib, pair.dev.ptr, auto.ptr, 0, split, 1.0, 1.0, 0.3, 0.5, us[:split], (0,))
            assert ok and ok1
            if first and first[-1] == 0:
                assert first == whole
                continue
            ok2, second, st = gen_constrained(lib, pair.dev.ptr, auto.ptr, st, 12 - split, 1.0, 1.0, 0.3, 0.5, us[split:], (0,), keep=True)
            assert ok2 and first + second == whole and st == whole_st, split
            pair.same(("windows", split))
    finally:
        auto.free()
        pair.free()
        lib.rwkv_free(ctx)


# ---- 7. refusals change nothing --------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_constrained_rejections_change_nothing(lib):
    ctx = lib.rwkv_init_from_file(model_path("6v0-3m", "FP32"), 1, 0)
    other_model = lib.rwkv_init_from_file(model_path("5v2-730K", "FP32"), 1, 0)
    pair = Pair(lib, ctx)
    num = bd.ByteDFA(bd.NUMBER)
    auto = Automaton(lib, ctx.ptr, num.next)
    foreign = Automaton(lib, other_model.ptr, num.next)
    bt = None
    try:
        L = lib.library
        V = pair.n_vocab
        err = lambda p: L.rwkv_get_last_error(p)
        pair.prime(LONG_PROMPT[:4])
        us = np.random.RandomState(3).random_sample(12)
        counts = Counter()
        want, want_st = host_constrained(lib, pair.host.ptr, num.next, 0, 2, 1.0, 1.0, 0.4, 0.4, us[:2], counts=counts)
        ok, got, st = gen_constrained(lib, pair.dev.ptr, auto.ptr, 0, 2, 1.0, 1.0, 0.4, 0.4, us[:2])
        assert ok and got == want and st == want_st and not num.dead_end(st)
        before = (state(lib, pair.dev.ptr, pair.n_state).tobytes(), logits(lib, pair.dev.ptr, V).tobytes())
        dev = pair.dev.ptr
        rec = Recorder()
        for streaming in (False, True):
            r = rec if streaming else None
            for kw, flags in [(dict(st=num.n_states), ERR_ARGS), (dict(auto_ptr=foreign.ptr), ERR_ARGS), (dict(st_ptr=False), ERR_ARGS),
                              (dict(auto_ptr=None), ERR_ARGS), (dict(temperature=-1.0), ERR_ARGS), (dict(max_tokens=0), ERR_ARGS)]:
                a = dict(auto_ptr=auto.ptr, st=st, max_tokens=7, temperature=1.0, st_ptr=True, **{})
                a.update(kw)
                ok, _, st_after = gen_constrained(lib, dev, a["auto_ptr"], a["st"], a["max_tokens"], a["temperature"], 1.0, 0.4, 0.4, us[2:9], keep=True,
                                                  rec=r, st_ptr=a["st_ptr"])
                assert not ok and err(dev) == flags, kw
                assert st_after == a["st"], kw
        # table entries out of range, an empty table, a stage of a pipeline
        bad = num.next.copy()
        bad[1, 7] = num.n_states
        assert not L.rwkv_b200_automaton_create(ctx.ptr, bad.ctypes.data_as(P16), num.n_states) and lib.rwkv_get_last_error(None) == ERR_ARGS
        assert not L.rwkv_b200_automaton_create(ctx.ptr, bad.ctypes.data_as(P16), 0) and lib.rwkv_get_last_error(None) == ERR_ARGS
        stage = lib.rwkv_b200_init_from_file_ex(model_path("6v0-3m", "FP32"), 0, 0, 1)
        assert not L.rwkv_b200_automaton_create(stage.ptr, num.next.ctypes.data_as(P16), num.n_states)
        assert lib.rwkv_get_last_error(None) == ERR_CTX | ERR_UNSUPPORTED
        ok, _, s = gen_constrained(lib, stage.ptr, auto.ptr, 0, 3, 1.0, 1.0, 0.0, 0.0, us[:3])
        assert not ok and err(stage.ptr) == ERR_CTX | ERR_UNSUPPORTED and s == 0
        lib.rwkv_free(stage)
        # the wrong context kinds
        bt = Batch(lib, ctx, 2)
        ok, _, s = gen_constrained(lib, bt.ptr, auto.ptr, 0, 3, 1.0, 1.0, 0.0, 0.0, us[:3])
        assert not ok and err(bt.ptr) == ERR_CTX | ERR_UNSUPPORTED
        single = Batch.__new__(Batch)
        single.lib, single.n, single.ptr = lib, 1, dev
        ok, _, s = batch_constrained(single, [auto], [st], [3], [1.0], [1.0], [0.0], [0.0], us[None, :3])
        assert not ok and err(dev) == ERR_CTX | ERR_UNSUPPORTED and s == [st]
        ok, _, s = batch_constrained(bt, [auto, foreign], [0, 0], [3, 3], [1.0] * 2, [1.0] * 2, [0.0] * 2, [0.0] * 2, np.full((2, 3), 0.5))
        assert not ok and err(bt.ptr) == ERR_ARGS and s == [0, 0]
        ok, _, s = batch_constrained(bt, [None, auto], [0, num.n_states], [3, 3], [1.0] * 2, [1.0] * 2, [0.0] * 2, [0.0] * 2, np.full((2, 3), 0.5))
        assert not ok and err(bt.ptr) == ERR_ARGS and s == [0, num.n_states]
        assert rec.calls == []
        assert (state(lib, dev, pair.n_state).tobytes(), logits(lib, dev, V).tobytes()) == before
        # the counts are unchanged too: continuing equals the host loop continuing from its counts
        want, want_st = host_constrained(lib, pair.host.ptr, num.next, st, 7, 1.0, 1.0, 0.4, 0.4, us[2:9], counts=counts)
        ok, got, st2 = gen_constrained(lib, dev, auto.ptr, st, 7, 1.0, 1.0, 0.4, 0.4, us[2:9], keep=True)
        assert ok and got == want and st2 == want_st
        pair.same("after rejections")
    finally:
        if bt:
            bt.free()
        auto.free()
        foreign.free()
        pair.free()
        lib.rwkv_free(other_model)
        lib.rwkv_free(ctx)


@pytest.mark.gpu
def test_automaton_from_a_device_table(lib):
    """A table in device memory is checked and uploaded as a host table is."""
    import torch
    ctx = lib.rwkv_init_from_file(model_path("6v0-3m", "FP32"), 1, 0)
    pair = Pair(lib, ctx)
    num = bd.ByteDFA(bd.NUMBER)
    host_auto = Automaton(lib, ctx.ptr, num.next)
    try:
        dev_table = torch.from_numpy(num.next.astype(np.int16)).cuda()
        dptr = ctypes.cast(ctypes.c_void_p(dev_table.data_ptr()), P16)
        dev_auto = lib.library.rwkv_b200_automaton_create(ctx.ptr, dptr, num.n_states)
        assert dev_auto
        bad = dev_table.clone()
        bad[2, 9] = num.n_states
        assert not lib.library.rwkv_b200_automaton_create(ctx.ptr, ctypes.cast(ctypes.c_void_p(bad.data_ptr()), P16), num.n_states)
        assert lib.rwkv_get_last_error(None) == ERR_ARGS
        us = np.random.RandomState(2).random_sample(12)
        pair.prime(LONG_PROMPT[:4])
        ok, want, want_st = gen_constrained(lib, pair.host.ptr, host_auto.ptr, 0, 12, 1.0, 0.9, 0.1, 0.1, us)
        ok2, got, st = gen_constrained(lib, pair.dev.ptr, dev_auto, 0, 12, 1.0, 0.9, 0.1, 0.1, us)
        assert ok and ok2 and got == want and st == want_st
        pair.same("device table")
        lib.library.rwkv_b200_automaton_free(dev_auto)
    finally:
        host_auto.free()
        pair.free()
        lib.rwkv_free(ctx)
