"""Constrained generation without a GPU: the new entry points are exported and declared, they reject a NULL context before they touch
a device, and the byte-level DFA builder of the GPU tests agrees with re.fullmatch."""
import ctypes
import os
import re

import numpy as np

import byte_dfa as bd

ARGS = 1 << 8
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("rwkv_b200_automaton_create", "rwkv_b200_automaton_free", "rwkv_b200_generate_constrained", "rwkv_b200_batch_generate_constrained",
         "rwkv_b200_test_generate_step_constrained")


def test_constrained_symbols_are_exported_and_declared(lib):
    with open(os.path.join(ROOT, "include", "rwkv_b200.h")) as f:
        header = f.read()
    assert "#define RWKV_B200_AUTOMATON_DEAD 0xFFFF" in header
    for name in NAMES:
        assert hasattr(lib.library, name), name
        assert getattr(lib.library, name).argtypes is not None, name
        assert re.search(r"RWKV_API [^;]*\b%s\(" % name, header), name


def test_constrained_entry_points_reject_a_null_context(lib, pkg):
    import rwkv_cpp_b200.shared_library as sl
    L = lib.library
    calls = []
    fn = sl.RWKV_TOKEN_FN(lambda user, seq, idx, tok: calls.append((seq, idx, tok)) or 0)
    n = ctypes.c_size_t(0)
    toks = (ctypes.c_uint32 * 4)()
    u = (ctypes.c_double * 4)(0.5, 0.5, 0.5, 0.5)
    state = (ctypes.c_uint32 * 1)(0)
    table = (ctypes.c_uint16 * 256)(*([0] * 256))
    assert not L.rwkv_b200_automaton_create(None, table, 1)
    assert lib.rwkv_get_last_error(None) == ARGS
    L.rwkv_b200_automaton_free(None)
    for on_token in (fn, sl.RWKV_TOKEN_FN()):
        assert not L.rwkv_b200_generate_constrained(None, None, state, 4, 1.0, 1.0, 0.0, 0.0, False, u, None, 0, on_token, None, toks, ctypes.byref(n))
        assert lib.rwkv_get_last_error(None) == ARGS
        ng = (ctypes.c_uint32 * 1)()
        automata = (ctypes.c_void_p * 1)()
        assert not L.rwkv_b200_batch_generate_constrained(None, automata, state, (ctypes.c_uint32 * 1)(4), None, None, None, None, None, u, None, 0,
                                                          on_token, None, toks, ng)
        assert lib.rwkv_get_last_error(None) == ARGS
    assert calls == [] and state[0] == 0


def test_constrained_step_hook_checks_its_table_first(lib):
    """A table entry out of range, a state out of range and a NULL table are refused before any device is touched."""
    import generate_ref as gr
    L = lib.library
    V = 8
    logits = np.zeros(V, np.float32)
    mt, st, fr, cnt, tk, nx = (np.array([1], np.uint32), np.zeros(1, np.uint32), np.zeros(1, np.uint8), np.zeros(V, np.uint32), np.zeros(1, np.uint32),
                               np.zeros(1, np.int32))
    ones, zero, u = np.ones(1, np.float32), np.zeros(1, np.float32), np.full(1, 0.5)
    act = ctypes.c_uint32(0)
    a = gr.StepArgs(logits=logits.ctypes.data, n_rows=1, n_vocab=V, max_tokens=mt.ctypes.data, temperature=ones.ctypes.data, top_p=ones.ctypes.data,
                    presence_penalty=zero.ctypes.data, frequency_penalty=zero.ctypes.data, u=u.ctypes.data, stop_ids=None, n_stop=0, step=st.ctypes.data,
                    frozen=fr.ctypes.data, counts=cnt.ctypes.data, tokens=tk.ctypes.data, next_tokens=nx.ctypes.data, any_active=ctypes.addressof(act))
    P16, P32 = ctypes.POINTER(ctypes.c_uint16), ctypes.POINTER(ctypes.c_uint32)
    good = np.zeros((2, V), np.uint16)
    bad = good.copy()
    bad[1, 3] = 2
    for table, n_states, state in [(bad, 2, 0), (good, 2, 2), (good, 0, 0), (None, 2, 0), (np.full((1, V), 1, np.uint16), 1, 0)]:
        states = np.array([state], np.uint32)
        tp = None if table is None else table.ctypes.data_as(P16)
        assert not L.rwkv_b200_test_generate_step_constrained(ctypes.byref(a), tp, n_states, states.ctypes.data_as(P32))
        assert lib.rwkv_get_last_error(None) == ARGS
        assert states[0] == state


def sample_strings(seed, n=4000):
    rng = np.random.RandomState(seed)
    alphabet = b"-0123456789.;,abcz x"
    out = [b"", b"-", b"0;", b"-12.5;", b"1234.56;", b"12345;", b"1.;", b"1.234;", b"--1;", b"abc", b"ab,cd,ef", b"ab,cd,ef,gh", b"abcdef", b"a,"]
    for _ in range(n):
        k = rng.randint(0, 12)
        out.append(bytes(alphabet[i] for i in rng.randint(0, len(alphabet), size=k)))
        if rng.rand() < 0.5:    # strings close to a match
            d = "".join(rng.choice(list("0123456789"), size=rng.randint(1, 6)))
            out.append(("-" * rng.randint(0, 2) + d + ("." + d[:rng.randint(0, 3)]) * rng.randint(0, 2) + ";" * rng.randint(0, 2)).encode())
    return out


def test_byte_dfa_matches_re():
    for pattern, regex, eos in [(bd.NUMBER, bd.NUMBER_RE, None), (bd.WORDS, bd.WORDS_RE, 0)]:
        dfa = bd.ByteDFA(pattern, eos=eos)
        assert dfa.next.shape == (dfa.n_states, 256) and dfa.next.dtype == np.uint16
        assert ((dfa.next < dfa.n_states) | (dfa.next == bd.DEAD)).all()
        full = prefix = 0
        for s in sample_strings(len(regex)):
            want = re.fullmatch(regex, s) is not None
            assert dfa.fullmatch(s) == want, (regex, s)
            # a prefix the DFA accepts can still be completed to a match; one it refuses cannot
            if dfa.prefix_ok(s):
                prefix += 1
                assert any(re.fullmatch(regex, s + t) for t in (b"", b";", b"0;", b".0;", b"a", b"0"))
            full += want
        assert full > 50 and prefix > 100
        if eos is not None:     # the end of text id is allowed exactly in the accepting states, and does not move the state
            for st in range(dfa.n_states):
                assert (dfa.next[st, eos] != bd.DEAD) == dfa.accepting[st]
                assert dfa.next[st, eos] in (bd.DEAD, st)
    num = bd.ByteDFA(bd.NUMBER)
    end = num.walk(b"12;")
    assert end is not None and num.dead_end(end) and num.accepting[end]
    assert not num.dead_end(0) and not num.accepting[0]
