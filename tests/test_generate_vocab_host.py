"""CPU-only checks for tests/test_gpu_generate_vocab.py: the streaming step hook refuses bad arguments before it touches a device, and
the module's checks catch the bugs they are there for. Each bar feeds a check a numpy restatement of the kernel's arithmetic, once as
sampling.cu does it (the check passes) and once with one planted bug (the check must fail)."""
import ctypes

import numpy as np
import pytest

from sampling_oracle import probs64
from test_gpu_generate_vocab import (FAMILIES, GENERATE_MAX, MARK, RECORD, TOP_MAX, Row, Step, aim, automaton, check_draw, check_ring, check_top,
                                     common_rows, per_of)
from generate_ref import P_U
from test_gpu_generate_constrained import P16

ARGS = 1 << 8
AUTO = object()      # a Call argument left as the valid call has it


# ---- the hook's refusals ---------------------------------------------------------------------------------------------------------

class Call:
    """A streaming hook call over rows of vocabulary 8, valid unless a test breaks it."""

    def __init__(self, family, rows=None, V=8):
        self.family, self.V = family, V
        self.rows = rows or [Row(np.zeros(V), step=0), Row(np.zeros(V), step=1, max_tokens=3)]
        self.table = automaton(V) if family in ("constrained", "logprobs", "sampled") else None
        self.s = Step(self.rows, V, self.table, (), 0)
        self.acked = np.array([r.step << 1 for r in self.rows], np.uint32)
        R = len(self.rows)
        self.published, self.tokens = np.zeros(R, np.uint32), np.zeros((R, GENERATE_MAX), np.uint32)
        self.ring, self.timed_out = np.zeros((R, 2, RECORD), np.uint32), np.zeros(1, np.uint32)
        self.logprobs = np.zeros((R, self.s.n), np.float32)

    def __call__(self, lib, family=None, samplers=AUTO, table=AUTO, lp=AUTO, args=AUTO, **null):
        import rwkv_cpp_b200.shared_library as sl
        family = self.family if family is None else family
        fid = FAMILIES.index(family) if isinstance(family, str) else family
        sampled = family == "sampled"
        a = self.s.args(sampled) if args is AUTO else args
        smp = (sl.Sampler * len(self.rows))(*[r.smp.struct() for r in self.rows]) if samplers is AUTO and sampled else (None if samplers is AUTO else samplers)
        tbl = self.table if table is AUTO else table
        st = np.array([r.state for r in self.rows], np.uint32)
        lps = sl.Logprobs(top_n=0, logprobs=self.logprobs.ctypes.data_as(ctypes.POINTER(ctypes.c_float))) if lp is AUTO and family == "logprobs" else \
            (None if lp is AUTO else lp)
        words = {k: getattr(self, k).ctypes.data_as(P_U) for k in ("acked", "published", "tokens", "ring", "timed_out")}
        words.update(null)
        ok = lib.library.rwkv_b200_test_generate_step_streaming(
            None if a is None else ctypes.byref(a), fid, smp, None if tbl is None else tbl.ctypes.data_as(P16), 0 if tbl is None else tbl.shape[0],
            st.ctypes.data_as(P_U), None if lps is None else ctypes.byref(lps), words["acked"], words["published"], words["tokens"],
            words["ring"] if lps is not None else None, words["timed_out"])
        return bool(ok), lib.rwkv_get_last_error(None)


def refused(lib, call, **kw):
    ok, flags = call(lib, **kw)
    return not ok and flags == ARGS


@pytest.mark.parametrize("family", FAMILIES)
def test_streaming_hook_refuses_bad_arguments_without_a_device(lib, family):
    c = Call(family)
    ok, flags = c(lib)       # the valid call gets past every argument check: on a machine without a device it fails for that alone
    assert ok or flags != ARGS, flags
    waiting = Call(family)
    waiting.acked[1] = 0                                                     # row 1 would wait for its token 0 to be acknowledged
    assert refused(lib, waiting)
    for word in ("acked", "published", "tokens", "timed_out"):
        assert refused(lib, c, **{word: None}), word
    if family == "logprobs":
        assert refused(lib, c, ring=None)
        assert refused(lib, c, lp=None)
    for bad in (-1, 4):
        assert refused(lib, c, family=bad), bad
    if family == "sampled":
        assert refused(lib, c, samplers=None)
    else:
        import rwkv_cpp_b200.shared_library as sl
        assert refused(lib, c, samplers=(sl.Sampler * 2)())
    if family == "constrained":
        assert refused(lib, c, table=None)
    if family == "plain":
        assert refused(lib, c, table=automaton(8))
    # the checks it shares with the blocking hooks
    for field, value in (("n_rows", 0), ("n_rows", 257), ("n_vocab", 0), ("n_vocab", 65537), ("counts", None), ("step", None)):
        a = c.s.args(family == "sampled")
        setattr(a, field, value)
        assert refused(lib, c, args=a), field
    assert refused(lib, c, args=None)
    late = Call(family, [Row(np.zeros(8), step=3, max_tokens=2)])            # step above max_tokens
    assert refused(lib, late)


def test_rows_that_do_not_draw_need_no_acknowledgement(lib):
    """Frozen rows, spent budgets and dead automaton states never reach the gate, so their acked words are not checked."""
    rows = [Row(np.zeros(8), step=1, max_tokens=3, frozen=1), Row(np.zeros(8), step=2, max_tokens=2), Row(np.zeros(8), step=1, max_tokens=3, state=3),
            Row(np.zeros(8), step=0)]
    c = Call("constrained", rows)
    c.acked[:] = 0
    ok, flags = c(lib)
    assert ok or flags != ARGS, flags


# ---- bars: numpy restatements with one planted bug each ----------------------------------------------------------------------------

def keep_threshold(p, V, top_k, pads_counted=False):
    """KeepFilter::threshold over the 1024 * PER register slots: the largest probability t with at least top_k entries >= t. The pad
    slots past n_vocab hold 0, below every threshold the bisection tries; the bug counts them as entries >= t."""
    pads = 1024 * per_of(V) - V
    need = top_k - (pads if pads_counted else 0)
    return float(np.sort(p)[::-1][max(need, 1) - 1])


def restated_filtered_draw(row, bug=None):
    """The draw of the sampled kernel (T = 1, top-p off, no bias) in float64: the top_k filter, then the inverse CDF over the kept mass."""
    p = probs64(row.z, 1.0, 1.0)
    V = p.size
    q = np.where(p >= keep_threshold(p, V, row.smp.top_k, bug == "pads"), p, 0.0)
    q /= q.sum()
    tok = int(np.argmax(np.cumsum(q) > row.u))
    return tok, np.float32(q[tok])


def test_kth_threshold_counting_pads_is_caught():
    V = 1025                                      # PER 4: 3071 pad slots, whole threads of them
    rng = np.random.RandomState(1)
    z = rng.standard_normal(V).astype(np.float32)
    m = z.max()
    z[V - 1], z[512], z[3] = m + 2.0, m + 1.9, m + 1.8
    row = aim(Row(z, top_k=3), None, 3)
    check_draw(row, None, *restated_filtered_draw(row))
    with pytest.raises(AssertionError):
        check_draw(row, None, *restated_filtered_draw(row, "pads"))


def restated_top(z, n, larger_id_first=False):
    """The top-N selection's order: the larger logit first, then (as top_key's ~id makes it) the smaller id; the bug reverses the ids."""
    z = np.asarray(z, np.float64)
    ids = np.arange(len(z))
    return [int(i) for i in np.lexsort((-ids if larger_id_first else ids, -z))[:n]]


@pytest.mark.parametrize("V", [1025, 4097, 65536])
def test_top_n_by_larger_id_is_caught(V):
    rows = common_rows(V, np.random.RandomState(V), None)
    ties = [r for r in rows if (r.z == 5.0).sum() > 3][0].z              # equal top logits across threads and warps
    zeros = [r for r in rows if (r.z == -1.0).sum() > V // 2][0].z       # -0 / +0 deciding the tail
    for z in (ties, zeros):
        for n in (1, 5, TOP_MAX):
            check_top(z, restated_top(z, n))
        with pytest.raises(AssertionError):
            check_top(z, restated_top(z, TOP_MAX, larger_id_first=True))


def restated_draw(p, u, per, shift=0):
    """sample_row's inverse CDF over the blocked layout: thread t holds slots t * PER + j and reports id t * PER + j. The bug loads
    slot t * PER + j + 1, one entry past the block at its last j (and none of its first)."""
    slots = np.zeros(1024 * per + 1)
    slots[:p.size] = p
    w = slots[shift:shift + 1024 * per]
    c = np.cumsum(w) / w.sum()
    i = int(np.argmax((c > u) & (w > 0)))
    return i, np.float32(w[i] / w.sum())


@pytest.mark.parametrize("V", [1025, 16385, 50277, 65536])
def test_draw_reading_past_its_block_is_caught(V):
    per = per_of(V)
    rng = np.random.RandomState(V)
    z = rng.standard_normal(V).astype(np.float32)
    d = per * (V // per // 2)                     # the first entry of a thread in the middle
    z[d] = z.max() + 12
    row = aim(Row(z), None, d)
    p = probs64(row.z, 1.0, 1.0)
    check_draw(row, None, *restated_draw(p, row.u, per))
    with pytest.raises(AssertionError):
        check_draw(row, None, *restated_draw(p, row.u, per, shift=1))


def test_ring_record_in_the_wrong_slot_is_caught():
    R, step, b, tok = 3, 5, 1, 77
    ids, lps = [77, 3, 9], np.array([-0.1, -2.5, -3.0], np.float32)
    published, stream_tokens = np.full(R, MARK, np.uint32), np.full((R, GENERATE_MAX), MARK, np.uint32)
    published[b], stream_tokens[b, step] = step + 1, tok
    for slot, caught in ((step % 2, False), ((step + 1) % 2, True)):
        ring = np.full((R, 2, RECORD), MARK, np.uint32)
        rec = ring[b, slot]
        rec[0], rec[1] = np.float32(-0.1).view(np.uint32), np.float32(0.8).view(np.uint32)
        rec[2:2 + 3], rec[2 + TOP_MAX:2 + TOP_MAX + 3] = ids, lps.view(np.uint32)
        if caught:
            with pytest.raises(AssertionError):
                check_ring(ring, published, stream_tokens, b, step, tok, -0.1, 0.8, ids, lps)
        else:
            check_ring(ring, published, stream_tokens, b, step, tok, -0.1, 0.8, ids, lps)
