"""Penalty decay, penalty weights and the penalty counts of device-side generation (rwkv_b200_set_penalty_decay and its neighbours,
include/rwkv_b200.h) against the host loop of rwkv_b200_sample + rwkv_b200_eval_resident / rwkv_b200_batch_eval with the float32
restatement of penalty_ref.py, bit for bit:
1. decay 1 and no weights give every family the bits of an untouched context, and integer counts;
2. decay 0.996 with a weight table that has zeros: every family, single contexts and batches of 4 and of 16 with the tensor cores off;
3. two windows with keep_counts equal one call; 4. a streaming stop and frozen batch rows do not decay;
5. counts set before a call, and a sequence moved to another slot with its state and counts, through every kind of buffer;
6. refused calls change nothing; 7. beam search leaves the counts alone; 8. the step at every vocabulary width of the step kernel."""
import ctypes

import numpy as np
import pytest

from conftest import LONG_PROMPT, model_path
import generate_ref as gr
import penalty_ref as pr
from generate_ref import P_F, P_U
from test_gpu_generate import Batch, Pair, generate
from test_gpu_generate_constrained import Automaton, batch_constrained, gen_constrained
from test_gpu_generate_logprobs import Out, batch_logprobs, gen_logprobs
from test_gpu_generate_sampled import Smp, batch_sampled, gen_sampled, sample_logits
from test_gpu_generate_stream import Recorder, batch_generate_stream, generate_stream
from test_gpu_sampling_edges import VOCABS

pytestmark = pytest.mark.gpu

ERR_ARGS, ERR_CTX_UNSUPPORTED = 1 << 8, (6 << 8) | 9
FAMILIES = ("plain", "stream", "constrained", "logprobs", "sampled")
DEAD = 0xFFFF
DECAY = 0.996


def weights_of(V, seed):
    """A weight table with zeros: 0, 0.5, 1 or 2 per token."""
    return np.random.RandomState(seed).choice(np.array([0.0, 0.5, 1.0, 2.0], np.float32), V).astype(np.float32)


def forbidden_of(V, seed):
    """The automaton of the constrained family: state 0 forbids these tokens and loops on every other one."""
    return np.random.RandomState(seed).choice(V, max(1, V // 50), replace=False)


def allow_table(V, forbidden):
    t = np.zeros((1, V), np.uint16)
    t[0, forbidden] = DEAD
    return t


USER = {3: 1.5, 7: -0.5, 40: 2.0}      # the sampled family's user bias entries


class Single:
    """One family's generate call on a single-sequence context, and what its host loop needs to know about the family."""

    def __init__(self, lib, ctx_ptr, family, V):
        self.lib, self.family, self.V = lib, family, V
        self.allowed = None
        self.auto = None
        if family == "constrained":
            forbidden = forbidden_of(V, 5)
            self.auto = Automaton(lib, ctx_ptr, allow_table(V, forbidden))
            self.allowed = np.ones(V, bool)
            self.allowed[forbidden] = False
        self.user = USER if family == "sampled" else None

    def run(self, ctx_ptr, mt, T, top_p, pres, freq, us, stops=(), keep=False, rec=None):
        L, f = self.lib, self.family
        if f == "plain":
            return generate(L, ctx_ptr, mt, T, top_p, pres, freq, us, stops, keep=keep)
        if f == "stream":
            return generate_stream(L, ctx_ptr, mt, T, top_p, pres, freq, us, stops, keep=keep, rec=rec or Recorder())
        if f == "constrained":
            ok, toks, _ = gen_constrained(L, ctx_ptr, self.auto.ptr, 0, mt, T, top_p, pres, freq, us, stops, keep=keep)
            return ok, toks
        if f == "logprobs":
            ok, toks, _ = gen_logprobs(L, ctx_ptr, Out(1, mt, 2), mt, T, top_p, pres, freq, us, stops, keep=keep)
            return ok, toks
        ok, toks, _ = gen_sampled(L, ctx_ptr, Smp(T, top_p, pres=pres, freq=freq, bias=self.user), mt, us, stops, keep=keep)
        return ok, toks

    def host(self, ctx_ptr, mt, T, top_p, pres, freq, us, stops=(), counts=None, decay=1.0, weights=None):
        return pr.host_generate(self.lib, ctx_ptr, self.V, mt, T, top_p, pres, freq, us, stops, counts, decay, weights, self.allowed, self.user)

    def free(self):
        if self.auto:
            self.auto.free()


def counts_of(lib, ctx, seq=0):
    return lib.rwkv_b200_get_penalty_counts(ctx, seq)


class Raw:
    def __init__(self, ptr):
        self.ptr = ptr


def open_pair(lib, ver="6v0-3m", fmt="Q5_1"):
    ctx = lib.rwkv_init_from_file(model_path(ver, fmt), 1, 0)
    return ctx, Pair(lib, ctx)


# ---- 1 and 2: the families on single contexts -------------------------------------------------------------------------------------

@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("ver,fmt", [("6v0-3m", "Q5_1"), ("7v0-834K", "FP32")])
def test_single_context_families(lib, family, ver, fmt):
    ctx, pair = open_pair(lib, ver, fmt)
    V = pair.n_vocab
    fam = Single(lib, ctx.ptr, family, V)
    third = lib.rwkv_clone_context(ctx, 1)
    try:
        rng = np.random.RandomState(sum(map(ord, family + ver)))
        prompt = LONG_PROMPT[:6]
        stops = ()
        for mt, T, top_p, pres, freq in [(9, 1.0, 0.9, 0.3, 0.4), (8, 0.0, 1.0, 0.5, 0.5), (7, 0.8, 1.0, 0.2, 0.6)]:
            us = rng.random_sample(mt)
            # 1. decay 1 and no weights, after both were set to something else: the bits of an untouched context, integer counts
            lib.rwkv_b200_set_penalty_decay(pair.dev, 0, 0.5)
            lib.rwkv_b200_set_penalty_weights(pair.dev, weights_of(V, 1))
            lib.rwkv_b200_set_penalty_decay(pair.dev, 0, 1.0)
            lib.rwkv_b200_set_penalty_weights(pair.dev, None)
            pair.prime(prompt)
            prime_raw(lib, third.ptr, prompt)
            want, want_counts = fam.host(pair.host.ptr, mt, T, top_p, pres, freq, us, stops)
            ok, got = fam.run(pair.dev.ptr, mt, T, top_p, pres, freq, us, stops)
            ok3, got3 = fam.run(third.ptr, mt, T, top_p, pres, freq, us, stops)
            assert ok and ok3 and got == want == got3, (family, mt)
            pair.same(("decay 1", family, mt))
            assert state_bytes(lib, third.ptr, pair.n_state) == state_bytes(lib, pair.dev.ptr, pair.n_state)
            c = counts_of(lib, pair.dev)
            assert np.array_equal(c, want_counts) and np.array_equal(c, np.round(c)), family
            assert np.array_equal(counts_of(lib, third), c)
            # 2. decay 0.996 and a weight table with zeros
            w = weights_of(V, mt)
            lib.rwkv_b200_set_penalty_decay(pair.dev, 0, DECAY)
            lib.rwkv_b200_set_penalty_weights(pair.dev, w)
            pair.prime(prompt)
            want, want_counts = fam.host(pair.host.ptr, mt, T, top_p, pres, freq, us, stops, decay=DECAY, weights=w)
            ok, got = fam.run(pair.dev.ptr, mt, T, top_p, pres, freq, us, stops)
            assert ok and got == want, (family, mt, "decay")
            pair.same(("decay", family, mt))
            assert counts_of(lib, pair.dev).tobytes() == want_counts.tobytes(), (family, mt)
            if len(want) > 3:
                stops = (want[3],)    # the next case stops on a token of this one, where it comes
        # 3. windows: two calls of k tokens with keep_counts give the bits of one call of 2k
        us = rng.random_sample(12)
        pair.prime(prompt)
        ok, whole = fam.run(pair.dev.ptr, 12, 1.0, 1.0, 0.4, 0.4, us)
        whole_counts = counts_of(lib, pair.dev)
        whole_state = state_bytes(lib, pair.dev.ptr, pair.n_state)
        pair.prime(prompt)
        ok1, first = fam.run(pair.dev.ptr, 6, 1.0, 1.0, 0.4, 0.4, us[:6])
        ok2, second = fam.run(pair.dev.ptr, 6, 1.0, 1.0, 0.4, 0.4, us[6:], keep=True)
        assert ok and ok1 and ok2 and first + second == whole
        assert counts_of(lib, pair.dev).tobytes() == whole_counts.tobytes()
        assert state_bytes(lib, pair.dev.ptr, pair.n_state) == whole_state
    finally:
        fam.free()
        lib.rwkv_free(third)
        pair.free()
        lib.rwkv_free(ctx)


def prime_raw(lib, ctx_ptr, prompt):
    assert lib.library.rwkv_b200_state_load(ctx_ptr, None)
    assert lib.library.rwkv_b200_eval_resident(ctx_ptr, np.asarray(prompt, np.uint32).ctypes.data_as(P_U), len(prompt), True, None)


def state_bytes(lib, ctx_ptr, n):
    st = np.zeros(n, np.float32)
    assert lib.library.rwkv_b200_state_store(ctx_ptr, st.ctypes.data_as(P_F))
    return st.tobytes()


# ---- 2 on batches --------------------------------------------------------------------------------------------------------------

def batch_host(bt, n_state, V, max_tokens, temps, top_ps, pres, freq, us, stops, decay, weights, allowed=None, user=None, counts=None):
    """The batch loop on the host: rwkv_b200_batch_sample with row_bias + rwkv_b200_batch_eval, a stopped sequence put back after each
    pass; the counts follow penalty_ref.update for every evaluated token. Returns (tokens, counts, saved state and logits)."""
    B = bt.n
    counts = [np.zeros(V, np.float32) for _ in range(B)] if counts is None else [c.copy() for c in counts]
    step, frozen, out, saved = [0] * B, [False] * B, [[] for _ in range(B)], {}

    def freeze(b):
        frozen[b] = True
        saved[b] = (bt.state(b, n_state), bt.logits(b, V))

    while True:
        for b in range(B):
            if not frozen[b] and step[b] == max_tokens[b]:
                freeze(b)
        active = [b for b in range(B) if not frozen[b]]
        if not active:
            break
        toks = bt.sample(temps, top_ps, [us[b][step[b]] if not frozen[b] else 0.5 for b in range(B)],
                         [pr.row_bias(counts[b], pres[b], freq[b], allowed, user) if not frozen[b] else None for b in range(B)])
        inputs = [0] * B
        for b in active:
            out[b].append(toks[b])
            step[b] += 1
            if toks[b] in stops:
                freeze(b)
            else:
                counts[b] = pr.update(counts[b], toks[b], decay[b], weights)
                inputs[b] = toks[b]
        if all(frozen):
            break
        assert bt.eval(inputs)
        for b in range(B):
            if frozen[b]:
                assert bt.lib.library.rwkv_b200_batch_set_state(bt.ptr, b, saved[b][0].ctypes.data_as(P_F))
    return out, counts, saved


def batch_run(family, bt, auto, max_tokens, temps, top_ps, pres, freq, us, stops, keep=None, rec=None):
    B = bt.n
    if family == "plain":
        return bt.generate(max_tokens, temps, top_ps, pres, freq, us, stops, keep=keep)
    if family == "stream":
        return batch_generate_stream(bt, max_tokens, temps, top_ps, pres, freq, us, stops, rec or Recorder(), keep=keep)
    if family == "constrained":
        ok, toks, _ = batch_constrained(bt, [auto] * B, [0] * B, max_tokens, temps, top_ps, pres, freq, us, stops, keep=keep)
        return ok, toks
    if family == "logprobs":
        assert keep is None
        return batch_logprobs(bt, Out(B, max(max_tokens), 2), max_tokens, temps, top_ps, pres, freq, us, stops)
    smps = [Smp(temps[b], top_ps[b], pres=pres[b], freq=freq[b], bias=USER) for b in range(B)]
    ok, toks, _ = batch_sampled(bt, smps, max_tokens, us, stops, keep=keep)
    return ok, toks


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("B", [4, 16])
def test_batch_families(lib, family, B):
    """Budgets differ per sequence (one 0), so that frozen rows sit beside rows that go on decaying; every sequence has its own decay
    (1 for one of them); a stop id taken from the free run ends some rows mid-way. B = 16 runs with the tensor cores off."""
    ctx = lib.rwkv_init_from_file(model_path("6v0-3m", "Q5_1"), 1, 0)
    host, dev = Batch(lib, ctx, B), Batch(lib, ctx, B)
    V, n_state = lib.rwkv_get_logits_len(ctx), lib.rwkv_get_state_len(ctx)
    auto = Automaton(lib, ctx.ptr, allow_table(V, forbidden_of(V, 9))) if family == "constrained" else None
    allowed = None
    if auto:
        allowed = np.ones(V, bool)
        allowed[forbidden_of(V, 9)] = False
    user = USER if family == "sampled" else None
    try:
        if B >= 16:
            for bt in (host, dev):
                L = lib.library
                L.rwkv_b200_set_tensor_cores(bt.ptr, False)
        rng = np.random.RandomState(B + len(family))
        prompts = [[int(t) for t in rng.randint(0, 256, 4)] for _ in range(B)]
        max_tokens = [int(x) for x in rng.randint(3, 10, B)]
        max_tokens[1] = 0
        temps = [float(x) for x in rng.choice([0.0, 0.7, 1.0], B)]
        top_ps = [float(x) for x in rng.choice([0.8, 1.0], B)]
        pres, freq = [float(x) for x in rng.uniform(0, 0.6, B)], [float(x) for x in rng.uniform(0, 0.6, B)]
        decay = [float(np.float32(x)) for x in rng.choice([DECAY, 0.9, 0.5], B)]
        decay[2] = 1.0
        w = weights_of(V, B)
        us = rng.random_sample((B, max(max_tokens)))
        for b in range(B):
            lib.rwkv_b200_set_penalty_decay(Raw(dev.ptr), b, decay[b])
        lib.rwkv_b200_set_penalty_weights(Raw(dev.ptr), w)
        stops = ()
        for round_ in range(2):
            host.prime(prompts)
            dev.prime(prompts)
            want, want_counts, saved = batch_host(host, n_state, V, max_tokens, temps, top_ps, pres, freq, us, stops, decay, w, allowed, user)
            ok, got = batch_run(family, dev, auto, max_tokens, temps, top_ps, pres, freq, us, stops)
            assert ok and got == want, (family, round_)
            for b in range(B):
                assert counts_of(lib, Raw(dev.ptr), b).tobytes() == want_counts[b].tobytes(), (family, round_, b)
                if max_tokens[b]:
                    st, lg = saved[b]
                    assert dev.state(b, n_state).tobytes() == st.tobytes(), (family, b)
                    assert dev.logits(b, V).tobytes() == lg.tobytes(), (family, b)
            if round_ == 0:       # the second round stops on a token of the longest row of the first, where it comes
                long_row = max(range(B), key=lambda b: len(want[b]))
                stops = (want[long_row][2],)
    finally:
        if auto:
            auto.free()
        host.free()
        dev.free()
        lib.rwkv_free(ctx)


def test_batch_windows_and_frozen_rows(lib):
    """Two windows with keep_counts equal one call of both budgets; a row whose budget is spent keeps its counts while the others decay."""
    ctx = lib.rwkv_init_from_file(model_path("5v2-730K", "Q5_1"), 1, 0)
    bt = Batch(lib, ctx, 4)
    V = lib.rwkv_get_logits_len(ctx)
    try:
        rng = np.random.RandomState(7)
        prompts = [[int(t) for t in rng.randint(0, 256, 3)] for _ in range(4)]
        for b in range(4):
            lib.rwkv_b200_set_penalty_decay(Raw(bt.ptr), b, 0.9)
        lib.rwkv_b200_set_penalty_weights(Raw(bt.ptr), weights_of(V, 3))
        us = rng.random_sample((4, 10))
        T, P, pres, freq = [1.0] * 4, [1.0] * 4, [0.4] * 4, [0.4] * 4
        bt.prime(prompts)
        ok, whole = bt.generate([10, 2, 10, 10], T, P, pres, freq, us, ())
        whole_counts = [counts_of(lib, Raw(bt.ptr), b) for b in range(4)]
        bt.prime(prompts)
        ok1, first = bt.generate([5, 2, 5, 5], T, P, pres, freq, us[:, :5], ())
        row1 = counts_of(lib, Raw(bt.ptr), 1)
        ok2, second = bt.generate([5, 0, 5, 5], T, P, pres, freq, us[:, 5:], (), keep=[1, 1, 1, 1])
        assert ok and ok1 and ok2
        assert [a + b for a, b in zip(first, second)] == whole
        for b in range(4):
            assert counts_of(lib, Raw(bt.ptr), b).tobytes() == whole_counts[b].tobytes(), b
        assert counts_of(lib, Raw(bt.ptr), 1).tobytes() == row1.tobytes()
    finally:
        bt.free()
        lib.rwkv_free(ctx)


# ---- 4. streaming stops ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("j", [0, 3, 6])
def test_stream_stop_has_the_counts_of_the_shorter_call(lib, j):
    ctx, pair = open_pair(lib)
    try:
        w = weights_of(pair.n_vocab, 11)
        for c in (pair.host, pair.dev):
            lib.rwkv_b200_set_penalty_decay(c, 0, DECAY)
            lib.rwkv_b200_set_penalty_weights(c, w)
        us = np.random.RandomState(j).random_sample(10)
        pair.prime(LONG_PROMPT[:4])
        ok, want = generate(lib, pair.host.ptr, j + 1, 1.0, 1.0, 0.3, 0.3, us)
        rec = Recorder(stop_at={0: j})
        ok2, got = generate_stream(lib, pair.dev.ptr, 10, 1.0, 1.0, 0.3, 0.3, us, rec=rec)
        assert ok and ok2 and got == want
        assert counts_of(lib, pair.dev).tobytes() == counts_of(lib, pair.host).tobytes()
        pair.same(("stream stop", j))
    finally:
        pair.free()
        lib.rwkv_free(ctx)


# ---- 5. setting counts, moving a sequence ------------------------------------------------------------------------------------------

def buffer(kind, values):
    """values (float32, n_vocab) in a buffer of `kind`, and how to pass it: (object for the wrappers, address for the C call)."""
    import torch
    if kind == "host":
        a = np.array(values, np.float32)
        return a, a.ctypes.data
    if kind == "pinned":
        t = torch.from_numpy(np.array(values, np.float32)).pin_memory()
        return t, t.data_ptr()
    t = torch.from_numpy(np.array(values, np.float32)).cuda()
    torch.cuda.synchronize()
    return t, t.data_ptr()


def to_numpy(buf):
    return buf.cpu().numpy() if hasattr(buf, "cpu") else np.asarray(buf)


def set_counts(lib, ctx_ptr, seq, kind, values):
    buf, addr = buffer(kind, values)
    if kind == "device":     # the C call with a raw device pointer
        assert lib.library.rwkv_b200_set_penalty_counts(ctx_ptr, seq, ctypes.cast(addr, P_F)), lib.rwkv_get_last_error(Raw(ctx_ptr))
    else:
        lib.rwkv_b200_set_penalty_counts(Raw(ctx_ptr), seq, buf)


def get_counts(lib, ctx_ptr, seq, kind, V):
    buf, addr = buffer(kind, np.full(V, 7.0, np.float32))
    if kind == "device":
        assert lib.library.rwkv_b200_get_penalty_counts(ctx_ptr, seq, ctypes.cast(addr, P_F))
    else:
        assert lib.rwkv_b200_get_penalty_counts(Raw(ctx_ptr), seq, out=buf) is buf
    return to_numpy(buf)


@pytest.mark.parametrize("kind", ["host", "pinned", "device", "tensor"])
def test_set_counts_then_keep_counts_and_move_a_sequence(lib, kind):
    ctx, pair = open_pair(lib)
    V, n_state = pair.n_vocab, pair.n_state
    fresh = lib.rwkv_clone_context(ctx, 1)
    x, y = Batch(lib, ctx, 4), Batch(lib, ctx, 4)
    try:
        # a context that never generated reads zeros and allocates nothing
        assert not get_counts(lib, fresh.ptr, 0, kind, V).any()
        rng = np.random.RandomState(5)
        seed = np.zeros(V, np.float32)
        seed[rng.choice(V, 40, replace=False)] = rng.uniform(0, 3, 40).astype(np.float32)
        seed[5] = 1e-45
        set_counts(lib, fresh.ptr, 0, kind, seed)
        assert get_counts(lib, fresh.ptr, 0, kind, V).tobytes() == seed.tobytes()
        lib.rwkv_free(fresh)
        fresh = None
        for c in (pair.host, pair.dev):
            lib.rwkv_b200_set_penalty_decay(c, 0, DECAY)
        us = rng.random_sample(8)
        pair.prime(LONG_PROMPT[:5])
        want, want_counts = pr.host_generate(lib, pair.host.ptr, V, 8, 1.0, 1.0, 0.5, 0.5, us, counts=seed, decay=DECAY)
        set_counts(lib, pair.dev.ptr, 0, kind, seed)
        ok, got = generate(lib, pair.dev.ptr, 8, 1.0, 1.0, 0.5, 0.5, us, keep=True)
        assert ok and got == want
        assert get_counts(lib, pair.dev.ptr, 0, kind, V).tobytes() == want_counts.tobytes()
        pair.same("seeded")
        # move sequence 1 of x to slot 3 of y with its state and counts: the continuation is that of x's sequence 1
        prompts = [[int(t) for t in rng.randint(0, 256, 3)] for _ in range(4)]
        for bt in (x, y):
            for b in range(4):
                lib.rwkv_b200_set_penalty_decay(Raw(bt.ptr), b, 0.9)
        x.prime(prompts)
        y.prime(prompts[::-1])
        us = rng.random_sample((4, 6))
        ok, _ = x.generate([6] * 4, [1.0] * 4, [1.0] * 4, [0.4] * 4, [0.4] * 4, us, ())
        assert ok
        assert lib.library.rwkv_b200_batch_set_state(y.ptr, 3, x.state(1, n_state).ctypes.data_as(P_F))
        set_counts(lib, y.ptr, 3, kind, get_counts(lib, x.ptr, 1, kind, V))
        feed = [11, 12, 13, 14]
        assert x.eval(feed)
        assert y.eval([0, 0, 0, 12])
        us2 = rng.random_sample((4, 7))
        ok1, cont_x = x.generate([7] * 4, [1.0] * 4, [1.0] * 4, [0.4] * 4, [0.4] * 4, us2, (), keep=[1] * 4)
        us_y = us2.copy()
        us_y[3] = us2[1]
        ok2, cont_y = y.generate([7] * 4, [1.0] * 4, [1.0] * 4, [0.4] * 4, [0.4] * 4, us_y, (), keep=[1] * 4)
        assert ok1 and ok2 and cont_y[3] == cont_x[1]
        assert get_counts(lib, y.ptr, 3, kind, V).tobytes() == get_counts(lib, x.ptr, 1, kind, V).tobytes()
        assert y.state(3, n_state).tobytes() == x.state(1, n_state).tobytes()
    finally:
        if fresh:
            lib.rwkv_free(fresh)
        x.free()
        y.free()
        pair.free()
        lib.rwkv_free(ctx)


# ---- 6. refusals ----------------------------------------------------------------------------------------------------------------

def test_refusals_change_nothing(lib):
    """Every refusal of the four calls, from outside and from inside a streaming callback, on a context that runs beside an identical
    one: afterwards both give the same bits, so the refusals changed no state, logits, counts, decay or weights."""
    ctx, pair = open_pair(lib)
    V, n_state = pair.n_vocab, pair.n_state
    L = lib.library
    bt = Batch(lib, ctx, 2)
    try:
        pair.prime(LONG_PROMPT[:4])
        us = np.random.RandomState(1).random_sample(6)
        for c in (pair.host, pair.dev):
            ok, _ = generate(lib, c.ptr, 6, 1.0, 1.0, 0.3, 0.3, us)
            assert ok
        dev, err = pair.dev.ptr, (lambda: lib.rwkv_get_last_error(pair.dev))

        def unchanged(what):
            pair.same(what)
            assert counts_of(lib, pair.dev).tobytes() == counts_of(lib, pair.host).tobytes(), what

        for d in (0.0, -0.5, 1.0000001, float("nan"), float("inf")):
            assert not L.rwkv_b200_set_penalty_decay(dev, 0, d) and err() == ERR_ARGS, d
        assert not L.rwkv_b200_set_penalty_decay(dev, 1, 0.5) and err() == ERR_ARGS
        assert not L.rwkv_b200_set_penalty_decay(bt.ptr, 2, 0.5) and lib.rwkv_get_last_error(Raw(bt.ptr)) == ERR_ARGS
        out = np.zeros(V, np.float32)
        assert not L.rwkv_b200_get_penalty_counts(dev, 1, out.ctypes.data_as(P_F)) and err() == ERR_ARGS
        assert not L.rwkv_b200_get_penalty_counts(dev, 0, None) and err() == ERR_ARGS
        for bad in (-1.0, float("nan"), float("inf"), -float("inf")):
            t = np.zeros(V, np.float32)
            t[V - 1] = bad
            assert not L.rwkv_b200_set_penalty_counts(dev, 0, t.ctypes.data_as(P_F)) and err() == ERR_ARGS, bad
            assert not L.rwkv_b200_set_penalty_weights(dev, t.ctypes.data_as(P_F)) and err() == ERR_ARGS, bad
            unchanged(("table", bad))
        assert not L.rwkv_b200_set_penalty_counts(dev, 1, np.zeros(V, np.float32).ctypes.data_as(P_F)) and err() == ERR_ARGS
        assert not L.rwkv_b200_set_penalty_counts(dev, 0, None) and err() == ERR_ARGS
        unchanged("sequence")
        # from inside a streaming callback: refused; the stream gives what the blocking call on the twin gives
        errs = []

        def inner(seq, idx, tok):
            t = np.ones(V, np.float32)
            errs.append((L.rwkv_b200_set_penalty_decay(dev, 0, 0.5), err()))
            errs.append((L.rwkv_b200_set_penalty_weights(dev, t.ctypes.data_as(P_F)), err()))
            errs.append((L.rwkv_b200_get_penalty_counts(dev, 0, t.ctypes.data_as(P_F)), err()))
            errs.append((L.rwkv_b200_set_penalty_counts(dev, 0, t.ctypes.data_as(P_F)), err()))

        us = np.random.RandomState(3).random_sample(4)
        ok, want = generate(lib, pair.host.ptr, 4, 1.0, 1.0, 0.3, 0.3, us, keep=True)
        ok2, got = generate_stream(lib, dev, 4, 1.0, 1.0, 0.3, 0.3, us, keep=True, rec=Recorder(inner=inner))
        assert ok and ok2 and got == want
        assert errs and all(e == (False, ERR_CTX_UNSUPPORTED) for e in errs), errs
        unchanged("streaming callback")
        # a context of some layers only (a pipeline stage) generates nothing and has no penalties
        stage = L.rwkv_b200_init_from_file_ex(model_path("6v0-3m", "Q5_1").encode(), 0, 0, 1)
        assert stage
        try:
            assert not L.rwkv_b200_set_penalty_decay(stage, 0, 0.5) and lib.rwkv_get_last_error(Raw(stage)) == ERR_CTX_UNSUPPORTED
            assert not L.rwkv_b200_get_penalty_counts(stage, 0, out.ctypes.data_as(P_F)) and lib.rwkv_get_last_error(Raw(stage)) == ERR_CTX_UNSUPPORTED
        finally:
            L.rwkv_free(stage)
    finally:
        bt.free()
        pair.free()
        lib.rwkv_free(ctx)


# ---- 7. beam search -------------------------------------------------------------------------------------------------------------

def test_beam_search_leaves_the_counts(lib):
    ctx = lib.rwkv_init_from_file(model_path("6v0-3m", "Q5_1"), 1, 0)
    bt = Batch(lib, ctx, 4)
    V = lib.rwkv_get_logits_len(ctx)
    try:
        rng = np.random.RandomState(4)
        tables = []
        for b in range(4):
            t = np.zeros(V, np.float32)
            t[rng.choice(V, 20, replace=False)] = rng.uniform(0.1, 4, 20).astype(np.float32)
            lib.rwkv_b200_set_penalty_counts(Raw(bt.ptr), b, t)
            tables.append(t)
        bt.prime([[1, 2, 3]] * 4)
        lib.rwkv_b200_beam_search(Raw(bt.ptr), 5, 1.0, (), 2)
        for b in range(4):
            assert counts_of(lib, Raw(bt.ptr), b).tobytes() == tables[b].tobytes(), b
    finally:
        bt.free()
        lib.rwkv_free(ctx)


# ---- 8. the step at every vocabulary width ----------------------------------------------------------------------------------------

def step(lib, family, z, T, top_p, pres, freq, us, counts, decay, w, stops=(), table=None, user=None):
    """One step of the penalty hook over rows z [R, V] (step 0 of 1); returns (tokens, counts after)."""
    import rwkv_cpp_b200.shared_library as sl
    R, V = z.shape
    keep = dict(lg=np.ascontiguousarray(z, np.float32), mt=np.ones(R, np.uint32), t=np.full(R, T, np.float32), p=np.full(R, top_p, np.float32),
                pr=np.full(R, pres, np.float32), fq=np.full(R, freq, np.float32), u=np.ascontiguousarray(us, np.float64), st=np.zeros(R, np.uint32),
                fr=np.zeros(R, np.uint8), tk=np.zeros(R, np.uint32), nx=np.zeros(R, np.int32), act=np.zeros(1, np.uint32),
                stop=np.array(stops or [0], np.uint32))
    sampled = family == "sampled"
    a = gr.StepArgs(logits=keep["lg"].ctypes.data, n_rows=R, n_vocab=V, max_tokens=keep["mt"].ctypes.data,
                    temperature=None if sampled else keep["t"].ctypes.data, top_p=None if sampled else keep["p"].ctypes.data,
                    presence_penalty=None if sampled else keep["pr"].ctypes.data, frequency_penalty=None if sampled else keep["fq"].ctypes.data,
                    u=keep["u"].ctypes.data, stop_ids=keep["stop"].ctypes.data if stops else None, n_stop=len(stops), step=keep["st"].ctypes.data,
                    frozen=keep["fr"].ctypes.data, counts=None, tokens=keep["tk"].ctypes.data, next_tokens=keep["nx"].ctypes.data,
                    any_active=keep["act"].ctypes.data)
    fam = {"plain": 0, "constrained": 1, "logprobs": 2, "sampled": 3}[family]
    smps = [Smp(T, top_p, pres=pres, freq=freq, bias=user) for _ in range(R)] if sampled else None
    arr = (sl.Sampler * R)(*[s.struct() for s in smps]) if sampled else None
    out = Out(R, 1, 2) if family == "logprobs" else None
    lps = out.struct() if out else None
    states = np.zeros(R, np.uint32) if table is not None else None
    c = np.ascontiguousarray(counts, np.float32).copy()
    d = np.ascontiguousarray(decay, np.float32)
    wt = None if w is None else np.ascontiguousarray(w, np.float32)
    assert lib.library.rwkv_b200_test_generate_step_penalty(
        ctypes.byref(a), fam, arr, None if table is None else table.ctypes.data_as(ctypes.POINTER(ctypes.c_uint16)), 0 if table is None else table.shape[0],
        None if states is None else states.ctypes.data_as(P_U), ctypes.byref(lps) if lps else None, c.ctypes.data_as(P_F), d.ctypes.data_as(P_F),
        None if wt is None else wt.ctypes.data_as(P_F)), hex(lib.rwkv_get_last_error(None))
    return [int(t) for t in keep["tk"]], c


@pytest.mark.parametrize("V", sorted(set(VOCABS) - {1, 2}))
@pytest.mark.parametrize("family", ["plain", "constrained", "logprobs", "sampled"])
def test_step_at_every_width(lib, V, family):
    """Rows with counts on both sides of every thread boundary and at V - 1, decays 1, 0.996 and 0.5 and a denormal count, weights with
    zeros, a row whose draw is a stop id: each draw is rwkv_b200_sample_logits with the bias of rule 1, each count follows rule 3."""
    rng = np.random.RandomState(V)
    R = 4
    z = (rng.standard_normal((R, V)) * 2).astype(np.float32)
    counts = np.zeros((R, V), np.float32)
    for b in range(R):
        idx = np.unique(np.concatenate([rng.choice(V, min(V, 30), replace=False), [0, V - 1, min(V - 1, 1023), min(V - 1, 1024)]]))
        counts[b, idx] = rng.uniform(0, 5, idx.size).astype(np.float32)
        counts[b, idx[0]] = 1e-45
    decay = np.array([1.0, DECAY, 0.5, DECAY], np.float32)
    w = weights_of(V, V + 1)
    table, allowed = None, None
    if family == "constrained":
        forbidden = forbidden_of(V, V)
        table = allow_table(V, forbidden)
        allowed = np.ones(V, bool)
        allowed[forbidden] = False
    user = {0: 0.5, V - 1: -0.25} if family == "sampled" else None
    T, top_p, pres, freq = 0.9, 0.95, 0.4, 0.3
    us = rng.random_sample(R)
    want = [sample_logits(lib, z[b], T, top_p, us[b], pr.row_bias(counts[b], pres, freq, allowed, user))[0] for b in range(R)]
    stops = (want[3],)     # row 3 draws a stop id: reported, its counts stay
    toks, got = step(lib, family, z, T, top_p, pres, freq, us, counts, decay, w, stops, table, user)
    assert toks == want, (V, family)
    for b in range(R):
        exp = counts[b] if toks[b] in stops else pr.update(counts[b], toks[b], float(decay[b]), w)
        assert got[b].tobytes() == exp.tobytes(), (V, family, b)
