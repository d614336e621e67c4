"""Every generation step kernel at every vocabulary width it is compiled for (csrc/kernels/sampling.cu: PER = 1, 4, 16, 50 and 64
tokens per thread), the streaming kernels included.

1. The four blocking step families (rwkv_b200_test_generate_step, _constrained, _logprobs, _sampled) at every vocabulary of
   test_gpu_sampling_edges.VOCABS, on rows built to put the deciding entries where the layouts change hands: index 0, V - 1 next to
   the pads, both sides of a thread of the draw's blocked layout (tid * PER + j) and of the stride layout (tid + k * 1024) of the
   top-N selection and score_column. Each draw is held to float64 (sampling_oracle.probs64, sampler_ref, the ambiguity rules of
   test_gpu_generate_sampled.oracle_check, check_entry of test_gpu_generate_logprobs), and the step bookkeeping to its restatement.
2. The four streaming families (rwkv_b200_test_generate_step_streaming) on the same rows give the bits of their blocking twins, and
   publish, record and freeze as the streaming loop's host thread expects.
3. Whole synthetic models at the published vocabularies (50277, 16384, 65536): each streaming generate call gives the bytes of its
   blocking twin, which gives the bytes of the host loop; batch contexts of 4 and 256 sequences with per-sequence samplers.
4. The last test lists every *sample_kernel instantiation of the library and fails unless this module launched it."""
import ctypes
import re
import shutil
import subprocess

import numpy as np
import pytest

import byte_dfa as bd
import generate_ref as gr
from generate_ref import P_F, P_U
from sampler_ref import sampled_probs64, sampler_bias
from test_gpu_batch_sampling import hook_batch
from test_gpu_generate import Batch, Pair, generate
from test_gpu_generate_constrained import NONE, P16, Automaton, gen_constrained, host_constrained
from test_gpu_generate_logprobs import TOP_MAX, Out, check_entry, column_valid, gen_logprobs, top_ref
from test_gpu_generate_sampled import Smp, batch_same, batch_sampled, gen_sampled, hook, oracle_check, sample_logits
from test_gpu_generate_stream import Recorder, generate_stream
from test_gpu_sampling_edges import VOCABS, per_of

pytestmark = pytest.mark.gpu

FAMILIES = ("plain", "constrained", "logprobs", "sampled")
KERNEL = {"plain": "generate_sample_kernel", "constrained": "generate_constrained_sample_kernel", "logprobs": "generate_logprob_sample_kernel",
          "sampled": "generate_sampled_sample_kernel"}
GENERATE_MAX = 4096
RECORD = 2 + 2 * TOP_MAX          # words of a ring record: log-probability, sample probability, top ids, top log-probabilities
MARK = 0xA5A5A5A5                 # what the mapped words hold before a call
LAUNCHED = set()                  # (kernel, PER) of every launch this module made


def kernel_name(family, stream):
    k = KERNEL[family]
    return k.replace("generate_", "generate_stream_", 1) if stream else k


# ---- rows ------------------------------------------------------------------------------------------------------------------------

class Row:
    """One row of a step: logits, sampler, counts, automaton state, position in its loop. `target`: the token the draw must give."""

    def __init__(self, z, T=1.0, top_p=1.0, pres=0.0, freq=0.0, counts=None, state=NONE, step=0, max_tokens=2, frozen=0, top_k=0, min_p=0.0,
                 bias=None, u=0.5, target=None):
        self.z = np.asarray(z, np.float32)
        self.smp = Smp(T, top_p, top_k=top_k, min_p=min_p, pres=pres, freq=freq, bias=bias)
        self.counts, self.state, self.step, self.max_tokens, self.frozen = dict(counts or {}), state, step, max_tokens, frozen
        self.u, self.target = u, target


def allowed_of(table, state):
    return None if table is None or state == NONE else table[state] != bd.DEAD


def row_bias(row, table):
    return sampler_bias(row.counts, row.smp.pres, row.smp.freq, row.smp.bias, allowed_of(table, row.state))


def mid_u(row, table, tok):
    """The float64 CDF midpoint of tok under row's distribution: a draw with it is unambiguous and must give tok."""
    s = row.smp
    p = sampled_probs64(row.z, s.T, s.top_p, s.top_k, s.min_p, row_bias(row, table))
    cdf = np.cumsum(p)
    cdf /= cdf[-1]
    assert p[tok] > 1e-3, (tok, p[tok])
    return ((cdf[tok - 1] if tok else 0.0) + cdf[tok]) / 2


def aim(row, table, tok):
    row.u, row.target = mid_u(row, table, tok), tok
    return row


def boundaries(V):
    """Entries on both sides of a thread of the draw's blocked layout and of the 1024-strided top-N / score layout, 0 and V - 1."""
    per = per_of(V)
    last = (V - 1) // per * per                        # first entry of the last thread that holds any
    pos = {0, V - 1, per - 1, per, last - 1, last, 1023, 1024, 1024 * (V // 2048) - 1, 1024 * (V // 2048), V // 2}
    return sorted(p for p in pos if 0 <= p < V)


def automaton(V):
    """State 0 allows everything (-> 0); 1 allows only V - 1 (-> 0); 2 only the entries of the last thread (-> 2); 3 nothing."""
    last = (V - 1) // per_of(V) * per_of(V)
    t = np.full((4, V), bd.DEAD, np.uint16)
    t[0] = 0
    t[1, V - 1] = 0
    t[2, last:] = 2
    return t


def common_rows(V, rng, table):
    """Rows every family draws with its filters off; steps 0 and 1 so that the streaming gate runs."""
    rows = []
    for i, pos in enumerate(boundaries(V)):
        z = (rng.standard_normal(V) * 2).astype(np.float32)
        z[pos] = z.max() + 1
        rows.append(Row(z, T=0.0, pres=0.3, freq=0.2, counts={int(rng.randint(V)): 1}, target=pos, step=i % 2))
        z = rng.standard_normal(V).astype(np.float32)
        z[pos] = z.max() + 12
        rows.append(aim(Row(z, T=(1.0, 0.7)[i % 2], top_p=(1.0, 0.9)[i % 2], step=(i + 1) % 2), table, pos))
    z = (rng.standard_normal(V) * 2).astype(np.float32)
    z[0] = z[V - 1] = z.max() + 1
    rows.append(Row(z, T=0.0, target=0))                                              # T = 0, the maximum tied between 0 and V - 1
    last = (V - 1) // per_of(V) * per_of(V)
    for pos in (V - 1, last):                                                         # all -inf but one
        z = np.full(V, -np.inf, np.float32)
        z[pos] = 0.5
        rows.append(Row(z, T=0.8, u=rng.random_sample(), target=pos, step=1))
    z = rng.standard_normal(V).astype(np.float32)
    z[V // 2] = np.nan
    rows.append(Row(z, u=rng.random_sample()))
    z = rng.standard_normal(V).astype(np.float32)
    z[V - 1] = np.inf
    rows.append(Row(z, T=0.7, u=rng.random_sample(), step=1))
    z = rng.standard_normal(V).astype(np.float32)                                     # penalties on the ids next to the pads
    z[V - 1] = z.max() + 1
    cnt = {V - 1: 3, max(V - 2, 0): 1}
    rows.append(Row(z, T=0.9, pres=0.5, freq=0.7, counts=cnt, u=rng.random_sample()))
    rows.append(Row(z, T=0.0, pres=0.5, freq=0.7, counts=cnt, step=1))
    z = rng.standard_normal(V).astype(np.float32)                                     # equal top logits across threads and warps
    for p in boundaries(V) + [31, 32, 63, 64]:
        if p < V:
            z[p] = 5.0
    rows.append(Row(z, u=rng.random_sample()))
    z = np.full(V, -1.0, np.float32)                                                  # -0 / +0 decide the top-N tail
    zeros = sorted(set(boundaries(V)) | set(int(x) for x in rng.choice(V, size=min(V, 30), replace=False)))
    for j, p in enumerate(zeros):
        z[p] = -0.0 if j % 2 else 0.0
    ones = [int(x) for x in rng.choice(V, size=min(V, 3), replace=False)]
    z[ones] = 1.0
    rows.append(Row(z, T=1.3, u=rng.random_sample(), step=1))
    if V > 1:                                                                         # automaton states, stop id V - 1 below
        rows.append(Row(rng.standard_normal(V), state=1, u=rng.random_sample(), target=V - 1))
        rows.append(Row(rng.standard_normal(V) * 3, T=0.7, state=2, u=rng.random_sample(), counts={V - 1: 2}, pres=0.4, step=1))
        rows.append(Row(rng.standard_normal(V), state=3))                            # a dead end freezes the row before it draws
        rows.append(Row(rng.standard_normal(V) * 2, T=0.9, top_p=0.6, state=0, u=rng.random_sample(), step=1))
    rows.append(Row(rng.standard_normal(V), frozen=1, step=1))                       # frozen: nothing happens
    rows.append(Row(rng.standard_normal(V), step=2, max_tokens=2))                   # budget spent: freezes
    for r in rows:
        if r.state != NONE and table is None:
            r.state = NONE
    return rows


def filter_rows(V, rng, table):
    """Rows of the sampled family with top_k, min_p and user bias on."""
    per, rows = per_of(V), []
    last = (V - 1) // per * per
    z = rng.standard_normal(V).astype(np.float32)
    z[V - 1] = z.max() + 3
    rows.append(aim(Row(z, top_k=1), table, V - 1))
    for a, b in ((last - 1, last), (1023, 1024), (per - 1, per)):
        if 0 < a and b < V - 1:                           # the top_k-th probability tied across a thread of either layout
            z = rng.standard_normal(V).astype(np.float32)
            m = z.max()
            z[V - 1], z[a], z[b] = m + 3, m + 2, m + 2
            rows.append(aim(Row(z, top_k=2, step=1), table, b))
            rows.append(Row(z, T=0.6, top_k=2, u=rng.random_sample()))
    for k in sorted({max(V - 1, 1), V}):
        rows.append(Row(rng.standard_normal(V) * 4, T=1.2, top_k=k, u=rng.random_sample()))
        rows.append(Row(rng.standard_normal(V) * 4, T=0.8, top_p=0.9, top_k=k, u=rng.random_sample(), step=1))
    if V > 1:
        z = rng.standard_normal(V).astype(np.float32)
        z[0] = z[V - 1] = z.max() + 1
        rows.append(aim(Row(z, min_p=1.0), table, V - 1))                  # tied maxima at both ends, nothing else kept
        rows.append(aim(Row(z, min_p=1.0, step=1), table, 0))
    rows.append(Row(rng.standard_normal(V) * 3, T=0.9, min_p=1e-30, u=rng.random_sample()))
    z = rng.standard_normal(V).astype(np.float32)
    rows.append(aim(Row(z, top_k=min(V, 3), bias={V - 1: 15.0}), table, V - 1))    # a user bias next to the pads
    z = rng.standard_normal(V).astype(np.float32)
    hi = int(np.argmax(z))
    rows.append(Row(z, T=1.1, top_k=min(V, 5), min_p=0.05, pres=0.3, freq=0.2, counts={V - 1: 2, hi: 1},
                    bias={hi: -np.inf, V - 1: 2.5, 0: 1.0} if V > 2 else {hi: 1.0}, u=rng.random_sample(), step=1))
    if table is not None and V > 1:
        rows.append(Row(rng.standard_normal(V), top_k=2, min_p=0.01, state=2, bias={V - 1: -3.0}, u=rng.random_sample()))
    return rows


# ---- one step --------------------------------------------------------------------------------------------------------------------

class Step:
    """The inputs and outputs of one hook call over `rows`."""

    def __init__(self, rows, V, table, stops, top_n):
        R = len(rows)
        self.rows, self.V, self.table, self.stops, self.top_n = rows, V, table, tuple(stops), top_n
        self.n = n = max(r.max_tokens for r in rows)
        self.z = np.ascontiguousarray([r.z for r in rows], np.float32)
        self.mt = np.array([r.max_tokens for r in rows], np.uint32)
        self.params = [np.array([getattr(r.smp, k) for r in rows], np.float32) for k in ("T", "top_p", "pres", "freq")]
        self.u = np.zeros((R, n), np.float64)
        for b, r in enumerate(rows):
            self.u[b, min(r.step, n - 1)] = r.u
        self.step = np.array([r.step for r in rows], np.uint32)
        self.frozen = np.array([r.frozen for r in rows], np.uint8)
        self.counts = np.zeros((R, V), np.uint32)
        for b, r in enumerate(rows):
            for t, c in r.counts.items():
                self.counts[b, t] = c
        self.tokens = np.zeros((R, n), np.uint32)
        self.nxt = np.full(R, -7, np.int32)
        self.act = ctypes.c_uint32(7)
        self.states = np.array([r.state for r in rows], np.uint32) if table is not None else None
        self.st = np.array(stops, np.uint32) if len(stops) else None
        self.out = None
        self.published = self.stream_tokens = self.ring = self.timed_out = None

    def args(self, sampled):
        t, p, pr, fr = [None if sampled else a.ctypes.data for a in self.params]
        return gr.StepArgs(logits=self.z.ctypes.data, n_rows=len(self.rows), n_vocab=self.V, max_tokens=self.mt.ctypes.data, temperature=t, top_p=p,
                           presence_penalty=pr, frequency_penalty=fr, u=self.u.ctypes.data, stop_ids=None if self.st is None else self.st.ctypes.data,
                           n_stop=len(self.stops), step=self.step.ctypes.data, frozen=self.frozen.ctypes.data, counts=self.counts.ctypes.data,
                           tokens=self.tokens.ctypes.data, next_tokens=self.nxt.ctypes.data, any_active=ctypes.addressof(self.act))

    def samplers(self):
        import rwkv_cpp_b200.shared_library as sl
        return (sl.Sampler * len(self.rows))(*[r.smp.struct() for r in self.rows])

    def result(self):
        return (self.step.tobytes(), self.frozen.tobytes(), self.counts.tobytes(), self.tokens.tobytes(), self.nxt.tobytes(), self.act.value,
                None if self.states is None else self.states.tobytes())


def run(lib, family, rows, V, table=None, stops=(), top_n=0, stream=False, acked=None, lp=True):
    """One step of `family` over rows (blocking, or streaming with the acked words given); returns the Step."""
    s = Step(rows, V, table, stops, top_n)
    R = len(rows)
    sampled = family == "sampled"
    a = s.args(sampled)
    tp = None if table is None or family == "plain" else table.ctypes.data_as(P16)
    ns = 0 if tp is None else table.shape[0]
    sp = None if s.states is None or tp is None else s.states.ctypes.data_as(P_U)
    if family in ("logprobs", "sampled") and lp:
        s.out = Out(R, s.n, top_n)
    lps = ctypes.byref(s.out.struct()) if s.out is not None else None
    L = lib.library
    if stream:
        s.published = np.full(R, MARK, np.uint32)
        s.stream_tokens = np.full((R, GENERATE_MAX), MARK, np.uint32)
        s.ring = np.full((R, 2, RECORD), MARK, np.uint32) if s.out is not None else None
        s.timed_out = np.full(1, MARK, np.uint32)
        s.acked = np.ascontiguousarray(acked, np.uint32)
        ok = L.rwkv_b200_test_generate_step_streaming(ctypes.byref(a), FAMILIES.index(family), s.samplers() if sampled else None, tp, ns, sp, lps,
                                                      s.acked.ctypes.data_as(P_U), s.published.ctypes.data_as(P_U), s.stream_tokens.ctypes.data_as(P_U),
                                                      None if s.ring is None else s.ring.ctypes.data_as(P_U), s.timed_out.ctypes.data_as(P_U))
    elif family == "plain":
        ok = L.rwkv_b200_test_generate_step(ctypes.byref(a))
    elif family == "constrained":
        ok = L.rwkv_b200_test_generate_step_constrained(ctypes.byref(a), tp, ns, sp)
    elif family == "logprobs":
        ok = L.rwkv_b200_test_generate_step_logprobs(ctypes.byref(a), tp, ns, sp, lps)
    else:
        ok = L.rwkv_b200_test_generate_step_sampled(ctypes.byref(a), s.samplers(), tp, ns, sp, lps)
    assert ok, (family, stream, lib.rwkv_get_last_error(None))
    LAUNCHED.add((kernel_name(family, stream), per_of(V)))
    return s


def acked_words(rows, stop_rows=()):
    """Every row's previous token acknowledged; the rows of stop_rows also ask to stop."""
    return [(r.step << 1) | (1 if b in stop_rows else 0) for b, r in enumerate(rows)]


# ---- checks (pure numpy: tests/test_generate_vocab_host.py feeds them planted bugs) --------------------------------------------------

def expected_bookkeeping(rows, table, stops, drawn, stop_rows=()):
    """(step, frozen, counts delta {b: tok}, next tokens, states, any_active) after one step in which row b drew drawn[b]."""
    step, frozen, nxt, states, counted = [], [], [], [], {}
    for b, r in enumerate(rows):
        st, fr, nx, state = r.step, r.frozen, 0, r.state
        if not fr and (st == r.max_tokens or dead_end(table, state) or b in stop_rows):
            fr = 1
        elif not fr:
            tok = drawn[b]
            st += 1
            if tok in stops:
                fr = 1
            else:
                counted[b] = tok
                nx = tok
                if table is not None and state != NONE and table[state][tok] != bd.DEAD:
                    state = int(table[state][tok])
        step.append(st); frozen.append(fr); nxt.append(nx); states.append(state)
    return step, frozen, counted, nxt, states, int(any(not f for f in frozen))


def dead_end(table, state):
    return table is not None and state != NONE and not (table[state] != bd.DEAD).any()


def draws(rows, table):
    """The rows that draw in this step (before any stop request)."""
    return [b for b, r in enumerate(rows) if not r.frozen and r.step < r.max_tokens and not dead_end(table, r.state)]


def check_bookkeeping(s, stop_rows=()):
    rows = s.rows
    drawn = {b: int(s.tokens[b, rows[b].step]) for b in draws(rows, s.table) if b not in stop_rows}
    step, frozen, counted, nxt, states, active = expected_bookkeeping(rows, s.table, s.stops, drawn, stop_rows)
    assert list(s.step) == step and list(s.frozen) == frozen and list(s.nxt) == nxt and s.act.value == active
    if s.states is not None:
        assert [int(x) for x in s.states] == states
    for b, r in enumerate(rows):
        want = np.zeros(s.V, np.uint32)
        for t, c in r.counts.items():
            want[t] = c
        if b in counted:
            want[counted[b]] += 1
        assert (s.counts[b] == want).all(), b
        others = np.ones(s.n, bool)
        if b in drawn:
            others[r.step] = False
        assert (s.tokens[b, others] == 0).all(), b


def check_draw(row, table, tok, prob):
    """One draw against float64: the first maximum at T = 0; otherwise oracle_check, and the target when one was aimed at."""
    bias = row_bias(row, table)
    if row.target is not None:
        assert tok == row.target, (tok, row.target)
    if row.smp.T == 0.0:
        zb = row.z.copy()
        for t, v in bias.items():
            zb[t] = np.float32(zb[t] + np.float32(v))
        assert tok == int(np.argmax(zb)) and prob == 1.0, (tok, int(np.argmax(zb)), prob)
        return "argmax"
    return oracle_check(row.z, row.smp, bias, row.u, tok, prob)


def check_top(z, ids):
    assert list(ids) == top_ref(z, len(ids)), (list(ids), top_ref(z, len(ids)))


def check_ring(ring, published, stream_tokens, b, step, tok, lp, prob, top_ids, top_lps):
    """Row b published token `step`: its mapped token word, its count and exactly its record in slot step % 2."""
    assert stream_tokens[b, step] == tok and published[b] == step + 1, (b, step)
    if ring is None:
        return
    rec = ring[b, step % 2]
    k = len(top_ids)
    assert rec[0] == np.float32(lp).view(np.uint32) and rec[1] == np.float32(prob).view(np.uint32), (b, step)
    assert (rec[2:2 + k] == np.asarray(top_ids, np.uint32)).all() and (rec[2 + TOP_MAX:2 + TOP_MAX + k] == np.asarray(top_lps, np.float32).view(np.uint32)).all()
    assert (rec[2 + k:2 + TOP_MAX] == MARK).all() and (rec[2 + TOP_MAX + k:] == MARK).all() and (ring[b, 1 - step % 2] == MARK).all(), (b, step)


# ---- 1. the blocking families against float64 ------------------------------------------------------------------------------------

def vocab_case(V):
    rng = np.random.RandomState(V)
    table = automaton(V) if V > 1 else None
    stops = (V - 1,) if V > 1 else ()
    return common_rows(V, rng, table), filter_rows(V, rng, table), table, stops


def check_family_draws(lib, s):
    """Every drawing row of a logprobs or sampled step: the draw against float64, the sampling probability, the log-probability and
    top-N entries against rwkv_b200_score_logits and float64."""
    done = []
    for b in draws(s.rows, s.table):
        r, tok = s.rows[b], int(s.tokens[b, s.rows[b].step])
        if not column_valid(r.z):      # a NaN or +inf: bit for bit what rwkv_b200_sample_logits draws from the same bias list
            t, p = sample_logits(lib, r.z, r.smp.T, r.smp.top_p, r.u, row_bias(r, s.table))
            LAUNCHED.add(("sample_kernel", per_of(s.V)))
            assert tok == t and s.out.sample_probs[b, r.step].tobytes() == p.tobytes(), b
        else:
            done.append(check_draw(r, s.table, tok, s.out.sample_probs[b, r.step]))
        check_entry(lib, r.z, tok, s.out, b, r.step)
    return done


@pytest.mark.parametrize("V", VOCABS)
def test_blocking_step_families(lib, V):
    common, filtered, table, stops = vocab_case(V)
    lp = {n: run(lib, "logprobs", common, V, table, stops, top_n=min(n, V)) for n in (1, 5, TOP_MAX)}
    full = lp[TOP_MAX]
    check_bookkeeping(full)
    done = check_family_draws(lib, full)
    assert done.count("edge") <= len(done) // 2, done
    for n in (1, 5):        # a shorter top-N is the prefix of the longer one, and nothing else moves
        k = min(n, V)
        assert lp[n].result() == full.result()
        assert lp[n].out.top_ids[:, :, :k].tobytes() == full.out.top_ids[:, :, :k].tobytes()
        assert lp[n].out.top_logprobs[:, :, :k].tobytes() == full.out.top_logprobs[:, :, :k].tobytes()
        assert lp[n].out.logprobs.tobytes() == full.out.logprobs.tobytes() and lp[n].out.sample_probs.tobytes() == full.out.sample_probs.tobytes()
    if table is not None:
        assert run(lib, "constrained", common, V, table, stops).result() == full.result()
    # the plain family has no automaton: its rows are the unconstrained ones, which the constrained kernels draw alike
    free = [r for r in common if r.state == NONE]
    plain = run(lib, "plain", free, V, None, stops)
    ref = run(lib, "logprobs", free, V, None, stops, top_n=min(5, V))
    assert plain.result() == ref.result()
    # the sampled family with its filters off gives the logprobs family's bits, with and without log-probabilities
    off = run(lib, "sampled", common, V, table, stops, top_n=min(TOP_MAX, V))
    assert off.result() == full.result()
    for f in ("logprobs", "sample_probs", "top_ids", "top_logprobs"):
        assert getattr(off.out, f).tobytes() == getattr(full.out, f).tobytes(), f
    assert run(lib, "sampled", common, V, table, stops, lp=False).result() == full.result()
    # and with them on, float64
    on = run(lib, "sampled", filtered, V, table, stops, top_n=min(5, V))
    check_bookkeeping(on)
    done = check_family_draws(lib, on)
    assert "checked" in done or V == 1, done
    assert run(lib, "sampled", filtered, V, table, stops, lp=False).result() == on.result()
    # the single-row and batched sampling kernels at this PER as well
    z = np.ascontiguousarray([common[1].z, common[-4].z])
    ok, toks, probs = hook_batch(lib, z, [1.0, 0.7], [1.0, 0.9], [0.3, 0.8])
    assert ok
    LAUNCHED.add(("batch_sample_kernel", per_of(V)))
    for b in range(2):
        t, p = sample_logits(lib, z[b], [1.0, 0.7][b], [1.0, 0.9][b], [0.3, 0.8][b], {})
        assert toks[b] == t and probs[b].tobytes() == p.tobytes()
    LAUNCHED.add(("sample_kernel", per_of(V)))


# ---- 2. the streaming families equal their blocking twins ------------------------------------------------------------------------

def check_stream_twin(s, blocking, stop_rows):
    """s (streaming) against its blocking twin: every row that drew carries the same bits and published them; a row asked to stop
    froze without drawing."""
    assert s.timed_out[0] == 0
    rows = s.rows
    check_bookkeeping(s, stop_rows)
    for b, r in enumerate(rows):
        if b in stop_rows:
            assert s.published[b] == MARK and (s.stream_tokens[b] == MARK).all() and s.nxt[b] == 0 and s.frozen[b] == 1
            if s.ring is not None:
                assert (s.ring[b] == MARK).all()
            continue
        for name in ("step", "frozen", "nxt"):
            assert getattr(s, name)[b] == getattr(blocking, name)[b], (name, b)
        assert s.counts[b].tobytes() == blocking.counts[b].tobytes() and s.tokens[b].tobytes() == blocking.tokens[b].tobytes(), b
        if s.states is not None:
            assert s.states[b] == blocking.states[b], b
        if b not in draws(rows, s.table):
            assert s.published[b] == MARK and (s.stream_tokens[b] == MARK).all() and (s.ring is None or (s.ring[b] == MARK).all()), b
            continue
        tok, i = int(s.tokens[b, r.step]), r.step
        others = np.arange(GENERATE_MAX) != i
        assert (s.stream_tokens[b, others] == MARK).all(), b
        if s.out is None:
            check_ring(None, s.published, s.stream_tokens, b, i, tok, None, None, [], [])
            continue
        for f in ("logprobs", "sample_probs", "top_ids", "top_logprobs"):
            assert getattr(s.out, f)[b].tobytes() == getattr(blocking.out, f)[b].tobytes(), (f, b)
        k = s.out.top_n
        check_ring(s.ring, s.published, s.stream_tokens, b, i, tok, s.out.logprobs[b, i], s.out.sample_probs[b, i], s.out.top_ids[b, i, :k],
                   s.out.top_logprobs[b, i, :k])


@pytest.mark.parametrize("V", VOCABS)
def test_streaming_step_families(lib, V):
    common, filtered, table, stops = vocab_case(V)
    # one row at step 1 asks to stop: it draws in the blocking twin and freezes here
    stop_rows = {next(b for b, r in enumerate(common) if r.step == 1 and not r.frozen and r.step < r.max_tokens and r.state == NONE)}
    acked = acked_words(common, stop_rows)
    free = [r for r in common if r.state == NONE]
    free_stop = {free.index(common[b]) for b in stop_rows}
    cases = [("plain", free, None, 0, free_stop), ("logprobs", common, table, TOP_MAX, stop_rows), ("sampled", common, table, 5, stop_rows),
             ("sampled", filtered, table, TOP_MAX, set())]
    if table is not None:
        cases.append(("constrained", common, table, 0, stop_rows))
    for family, rows, tbl, top_n, stop in cases:
        top_n = min(top_n, V)
        blocking = run(lib, family, rows, V, tbl, stops, top_n=top_n)
        s = run(lib, family, rows, V, tbl, stops, top_n=top_n, stream=True, acked=acked_words(rows, stop))
        check_stream_twin(s, blocking, stop)
    s = run(lib, "sampled", common, V, table, stops, stream=True, acked=acked, lp=False)       # no log-probabilities: no ring
    check_stream_twin(s, run(lib, "sampled", common, V, table, stops, lp=False), stop_rows)


def random_rows(V, R, rng, table):
    rows = []
    for b in range(R):
        z = rng.standard_normal(V) * (1 + b % 5)
        smp = dict(T=[0.0, 0.5, 1.0, 1.4][b % 4], top_p=[1.0, 0.9, 0.5][b % 3], pres=0.2 * (b % 2), freq=0.1 * (b % 3))
        cnt = {int(t): int(rng.randint(1, 3)) for t in rng.choice(V, size=4, replace=False)}
        rows.append(Row(z, counts=cnt, state=[NONE, 0, 2][b % 3], step=b % 3, max_tokens=3, u=rng.random_sample(),
                        top_k=[0, 40, 1000][b % 3], min_p=[0.0, 0.02][b % 2], bias={int(rng.randint(V)): 2.0, V - 1: -1.0}, **smp))
    return rows


def test_256_rows_at_65536(lib):
    """One launch of every family with the largest batch at the largest vocabulary, blocking against float64 and streaming against
    blocking."""
    V, R = 65536, 256
    rng = np.random.RandomState(256)
    table = automaton(V)
    rows = random_rows(V, R, rng, table)
    plain_rows = [Row(r.z, r.smp.T, r.smp.top_p, r.smp.pres, r.smp.freq, r.counts, NONE, r.step, r.max_tokens, u=r.u) for r in rows]
    for r in rows[::2]:
        r.smp = Smp(r.smp.T, r.smp.top_p, pres=r.smp.pres, freq=r.smp.freq)       # half of them with the filters off
    acked = acked_words(rows)
    on = run(lib, "sampled", rows, V, table, (V - 1,), top_n=5)
    check_bookkeeping(on)
    done = check_family_draws(lib, on)
    assert done.count("edge") <= len(done) // 2, done
    check_stream_twin(run(lib, "sampled", rows, V, table, (V - 1,), top_n=5, stream=True, acked=acked), on, set())
    lp = run(lib, "logprobs", rows, V, table, (V - 1,), top_n=TOP_MAX)
    check_bookkeeping(lp)
    check_stream_twin(run(lib, "logprobs", rows, V, table, (V - 1,), top_n=TOP_MAX, stream=True, acked=acked), lp, set())
    for b in range(0, R, 2):
        assert on.tokens[b].tobytes() == lp.tokens[b].tobytes() and on.out.sample_probs[b].tobytes() == lp.out.sample_probs[b].tobytes(), b
    cons = run(lib, "constrained", rows, V, table, (V - 1,))
    assert cons.result() == lp.result()
    check_stream_twin(run(lib, "constrained", rows, V, table, (V - 1,), stream=True, acked=acked), cons, set())
    plain = run(lib, "plain", plain_rows, V, None, (V - 1,))
    check_stream_twin(run(lib, "plain", plain_rows, V, None, (V - 1,), stream=True, acked=acked_words(plain_rows)), plain, set())
    for b in range(R):
        if rows[b].state == NONE:
            assert plain.tokens[b].tobytes() == lp.tokens[b].tobytes() and plain.counts[b].tobytes() == lp.counts[b].tobytes(), b


# ---- 3. whole models at the published vocabularies -------------------------------------------------------------------------------

MODELS = {   # one-file synthetic models of small width at the vocabularies of the published models
    "v4": dict(arch=(4, 0), C=256, F=1024, L=2, V=50277, out_scale=0.1),
    "v5.2": dict(arch=(5, 2), C=256, F=896, L=2, V=16384, S=64, out_scale=0.1),
    "v6": dict(arch=(6, 0), C=256, F=896, L=2, V=65536, S=64, mix=32, decay=64, out_scale=0.1, lora_fan_in=True),
    "v7": dict(arch=(7, 0), C=256, F=1024, L=2, V=65536, S=64, lora_w=32, lora_a=32, lora_v=16, lora_g=64, out_scale=0.1, lora_fan_in=True),
}
ON = Smp(1.1, 0.95, top_k=40, min_p=0.02, pres=0.3, freq=0.2, bias={10: 2.0, 65535 % 16384: -np.inf, 50276: 1.5})


@pytest.fixture(scope="module")
def model_files(tmp_path_factory):
    import synthetic_model as sm
    d = tmp_path_factory.mktemp("vocab_models")
    paths = {}
    for name, preset in MODELS.items():
        paths[name] = str(d / f"{name}.bin")
        sm.write_direct(paths[name], preset, "FP16", seed=5)
    return paths


def model_automaton(V):
    """State 0 allows the even ids (-> 1), state 1 the odd ids above V / 2 (-> 0)."""
    t = np.full((2, V), bd.DEAD, np.uint16)
    t[0, 0::2] = 1
    t[1, V // 2 + 1::2] = 0
    return t


@pytest.mark.parametrize("name", list(MODELS))
def test_whole_model_streaming_equals_blocking(lib, model_files, name):
    ctx = lib.rwkv_init_from_file(model_files[name], 1, 0)
    pair = Pair(lib, ctx)
    V = pair.n_vocab
    assert V == MODELS[name]["V"]
    prompt = [(7919 * i) % V for i in range(4)]
    rng = np.random.RandomState(V)
    smp = Smp(ON.T, ON.top_p, top_k=ON.top_k, min_p=ON.min_p, pres=ON.pres, freq=ON.freq, bias={k % V: v for k, v in ON.bias.items()})
    mt = 8
    try:
        us = rng.random_sample(mt)
        # blocking generate = the host loop; streaming = blocking
        pair.prime(prompt)
        want = gr.host_generate(lib, pair.host.ptr, mt, 1.0, 0.9, 0.2, 0.1, us)
        ok, got = generate(lib, pair.dev.ptr, mt, 1.0, 0.9, 0.2, 0.1, us)
        assert ok and got == want
        pair.same((name, "generate"))
        pair.prime(prompt)
        rec = Recorder()
        ok, streamed = generate_stream(lib, pair.host.ptr, mt, 1.0, 0.9, 0.2, 0.1, us, rec=rec)
        assert ok and streamed == want and rec.delivered(0) == want
        ok, _ = generate(lib, pair.dev.ptr, mt, 1.0, 0.9, 0.2, 0.1, us)
        pair.same((name, "stream"))
        # constrained
        table = model_automaton(V)
        auto = Automaton(lib, ctx.ptr, table)
        try:
            pair.prime(prompt)
            want, st_want = host_constrained(lib, pair.host.ptr, table, 0, mt, 0.8, 1.0, 0.1, 0.1, us)
            ok, got, st = gen_constrained(lib, pair.dev.ptr, auto.ptr, 0, mt, 0.8, 1.0, 0.1, 0.1, us)
            assert ok and got == want and st == st_want
            pair.same((name, "constrained"))
            pair.prime(prompt)
            ok, streamed, st2 = gen_constrained(lib, pair.host.ptr, auto.ptr, 0, mt, 0.8, 1.0, 0.1, 0.1, us, rec=Recorder())
            ok2, _, _ = gen_constrained(lib, pair.dev.ptr, auto.ptr, 0, mt, 0.8, 1.0, 0.1, 0.1, us)
            assert ok and ok2 and streamed == want and st2 == st_want
            pair.same((name, "constrained stream"))
            # log-probabilities, with the automaton
            pair.prime(prompt)
            o1, o2 = Out(1, mt, TOP_MAX), Out(1, mt, TOP_MAX)
            ok, want, st1 = gen_logprobs(lib, pair.host.ptr, o1, mt, 1.0, 1.0, 0.2, 0.2, us, auto=auto)
            ok2, got, st2 = gen_logprobs(lib, pair.dev.ptr, o2, mt, 1.0, 1.0, 0.2, 0.2, us, auto=auto, rec=Recorder())
            assert ok and ok2 and got == want and st1 == st2
            for f in ("logprobs", "sample_probs", "top_ids", "top_logprobs"):
                assert getattr(o1, f).tobytes() == getattr(o2, f).tobytes(), f
            pair.same((name, "logprobs stream"))
        finally:
            auto.free()
        # sampled with the filters on: the host loop of the step hook, blocking, streaming
        pair.prime(prompt)
        counts = np.zeros((1, V), np.uint32)
        want = []
        for i in range(mt):
            z = np.zeros(V, np.float32)
            assert lib.library.rwkv_b200_stage_logits(pair.host.ptr, z.ctypes.data_as(P_F), None)
            (tok,), counts, _ = hook(lib, z[None, :], [smp], [us[i]], counts)
            want.append(tok)
            gr.eval_token(lib, pair.host.ptr, tok)
        ok, got, _ = gen_sampled(lib, pair.dev.ptr, smp, mt, us)
        assert ok and got == want
        pair.same((name, "sampled"))
        pair.prime(prompt)
        o1, o2 = Out(1, mt, 5), Out(1, mt, 5)
        ok, got1, _ = gen_sampled(lib, pair.host.ptr, smp, mt, us, out=o1)
        ok2, got2, _ = gen_sampled(lib, pair.dev.ptr, smp, mt, us, out=o2, rec=Recorder())
        assert ok and ok2 and got1 == got2 == want
        for f in ("logprobs", "sample_probs", "top_ids", "top_logprobs"):
            assert getattr(o1, f).tobytes() == getattr(o2, f).tobytes(), f
        pair.same((name, "sampled stream"))
        LAUNCHED.update((kernel_name(f, s), per_of(V)) for f in FAMILIES for s in (False, True))      # every call above ran its step kernel
    finally:
        pair.free()
        lib.rwkv_free(ctx)


@pytest.mark.parametrize("B", [4, 256])
def test_batch_streaming_at_65536(lib, model_files, B):
    """Per-sequence samplers, callbacks that end sequences after different tokens: each sequence equals the blocking call whose
    budget ends there; at B = 4 the blocking call also equals the host loop of the step hook and rwkv_b200_batch_eval."""
    ctx = lib.rwkv_init_from_file(model_files["v6"], 1, 0)
    n_state, V = lib.rwkv_get_state_buffer_element_count(ctx), lib.rwkv_get_logits_buffer_element_count(ctx)
    b1, b2 = Batch(lib, ctx, B), Batch(lib, ctx, B)
    rng = np.random.RandomState(B)
    mt = 6
    prompts = [[(7919 * (i + 3 * b)) % V for i in range(3)] for b in range(B)]
    smps = [Smp([0.0, 0.8, 1.0, 1.3][b % 4], [1.0, 0.9][b % 2], top_k=[0, 40, 2][b % 3], min_p=[0.0, 0.03][b % 2], pres=0.2, freq=0.1 * (b % 3),
                bias={int(rng.randint(V)): 3.0, V - 1: 1.0}) for b in range(B)]
    try:
        us = rng.random_sample((B, mt))
        stop_at = {b: b % (mt + 1) for b in range(B) if b % (mt + 1) < mt}
        b1.prime(prompts); b2.prime(prompts)
        rec = Recorder(stop_at=stop_at)
        ok, streamed, _ = batch_sampled(b2, smps, [mt] * B, us, rec=rec)
        assert ok
        budgets = [stop_at[b] + 1 if b in stop_at else mt for b in range(B)]
        ok, want, _ = batch_sampled(b1, smps, budgets, us[:, :max(budgets)])       # u is [B][largest budget]
        assert ok and streamed == want
        for b in range(B):
            assert rec.delivered(b) == want[b] and len(want[b]) == budgets[b], b
        batch_same(b1, b2, n_state, V, "stream")
        if B == 4:
            b1.prime(prompts); b2.prime(prompts)
            counts = np.zeros((B, V), np.uint32)
            loop = [[] for _ in range(B)]
            for i in range(mt):
                z = np.array([b1.logits(b, V) for b in range(B)])
                toks, counts, _ = hook(lib, z, smps, us[:, i], counts)
                for b in range(B):
                    loop[b].append(toks[b])
                assert b1.eval(toks)
            ok, got, _ = batch_sampled(b2, smps, [mt] * B, us)
            assert ok and got == loop
            batch_same(b1, b2, n_state, V, "host loop")
    finally:
        b1.free(); b2.free()
        lib.rwkv_free(ctx)


# ---- 4. every compiled instantiation was launched above --------------------------------------------------------------------------

def library_sample_kernels(path):
    """(kernel, PER) of every *sample_kernel symbol in the library (cuobjdump)."""
    r = subprocess.run(["cuobjdump", "--dump-resource-usage", path], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    found = set()
    for name in re.findall(r"Function ([^:\s]+):", r.stdout):
        if m := re.search(r"([a-z_]*sample_kernel)ILi(\d+)E", name):
            found.add((m[1], int(m[2])))
    return found


def test_every_compiled_sample_kernel_was_launched(lib):
    """Runs after the tests above: the ten step and sampling kernel families at PER 1, 4, 16, 50 and 64 were each launched by this
    module. A new instantiation fails here until a test reaches it."""
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    compiled = library_sample_kernels(lib.path)
    assert len(compiled) == 10 * 5, sorted(compiled)
    assert compiled <= LAUNCHED, sorted(compiled - LAUNCHED)
    print("\n%d of %d *sample_kernel instantiations launched" % (len(compiled & LAUNCHED), len(compiled)))
