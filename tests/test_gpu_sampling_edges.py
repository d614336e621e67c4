"""The sampling kernel (csrc/kernels/sampling.cu, through rwkv_b200_sample_logits_batch with probs_out) against the float64
restatement of the draw (oracle/sampling_oracle.py: probs64 / cdf64) at the edges where the kernel can go wrong: n_vocab on both
sides of every PER switch, -inf logits on whole threads and warps, u at both ends of [0, 1), tiny temperatures, exact ties and
bias lists. Every draw must satisfy

  I1 (no tolerance)  the drawn token's float64 probability is > 0;
  I2                 cdf64[tok - 1] - eps <= u < cdf64[tok] + eps, eps = 2e-6 * max(1, 1 / T);
  I3                 prob_out is within a relative 1e-5 * max(1, 1 / T) of the float64 probability, plus what float32 cannot hold
                     near its smallest numbers (check_draw);
  I4                 at T = 0 the token is the first maximum of the float32 logits + bias and prob_out is 1;
  I5                 for one row and sorted u, the drawn tokens never decrease.

The float32 and float64 kept sets of top-p differ only where top_p sits within rounding of a tie group's cumulative mass, so every
top_p is first moved away from those boundaries (adjust_top_p; the moves are printed)."""
import collections
import ctypes

import numpy as np
import pytest

import generate_ref as gr
import sampling_oracle as so
from conftest import model_path
from test_gpu_batch_sampling import ERR_ARGS, P_D, P_F, P_U, bias_arrays, f32, hook_batch, ptr
from test_gpu_generate import hook_step
from test_gpu_generate_constrained import hook_constrained

VOCABS = [1, 2, 1023, 1024, 1025, 4095, 4096, 4097, 16383, 16384, 16385, 50277, 51200, 51201, 65535, 65536]
TEMPS = [0.0, 0.01, 0.1, 0.5, 1.0, 1.7, 8.0]
TOP_PS = [0.0, 1e-7, 0.05, 0.5, 0.95, 1.0]
EDGE_US = [0.0, 2.0 ** -53, 0.25, 0.5, 1 - 2.0 ** -40, 1 - 2.0 ** -52, 1 - 2.0 ** -53]
MAX_ROWS = 256
TOP_P_MARGIN = 1e-4
WORST = collections.defaultdict(float)      # family -> worst |u - nearest edge of the token's interval| / eps (I2) over draws
WORST_P = collections.defaultdict(float)    # family -> worst relative prob_out error / bar (I3)
MOVES = []


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    for family in sorted(WORST):
        print("\n%-18s worst I2 error / eps = %.3f   worst I3 error / bar = %.3f" % (family, WORST[family], WORST_P[family]), end="")
    print("\n%d top_p moves, largest %s" % (len(MOVES), max(MOVES, key=lambda m: abs(m[-1] - m[-2])) if MOVES else None))


def per_of(n_vocab):
    """Tokens per thread of the kernel instantiation serving n_vocab (sampling.cu: launch_sample_batch)."""
    per = -(-n_vocab // 1024)
    return 1 if per <= 1 else 4 if per <= 4 else 16 if per <= 16 else 50 if per <= 50 else 64


def eps_of(t):
    return 2e-6 * max(1.0, 1.0 / t) if t > 0 else 0.0


# ---- logit families ----------------------------------------------------------------------------------------------------------------

def _gauss(sigma):
    return lambda rng, V: ((rng.standard_normal(V) * sigma).astype(np.float32), None)


def _dead(fraction, sigma=8.0):
    def make(rng, V):
        x = (rng.standard_normal(V) * sigma).astype(np.float32)
        if fraction is None:                             # all but one token
            keep = rng.randint(V)
            x[np.arange(V) != keep] = -np.inf
        else:
            x[rng.rand(V) < fraction] = -np.inf
        return _alive(rng, x), None
    return make


def _tail(n):
    def make(rng, V):
        x = (rng.standard_normal(V) * 3.0).astype(np.float32)
        x[max(1, V - n):] = -np.inf
        return x, None
    return make


def _runs(warps):
    """-inf on about half of the aligned runs of PER tokens (whole threads) or of 32 * PER tokens (whole warps), the last run
    always among them."""
    def make(rng, V):
        x = (rng.standard_normal(V) * 3.0).astype(np.float32)
        run = per_of(V) * (32 if warps else 1)
        starts = list(range(0, V, run))
        for s in starts[1:]:
            if s == starts[-1] or rng.rand() < 0.5:
                x[s:s + run] = -np.inf
        return x, None
    return make


def _alive(rng, x):
    if not np.isfinite(x).any():
        x[rng.randint(x.size)] = 0.0
    return x


def _ints(rng, V):
    return rng.randint(-4, 5, size=V).astype(np.float32), None


def _dominant(rng, V):
    x = rng.standard_normal(V).astype(np.float32)
    x[rng.randint(V)] += 12.0
    return x, None


def _bias(rng, V):
    """-inf and +-30 entries, ids 0 and V - 1 among them; at least one token keeps a finite logit."""
    x = (rng.standard_normal(V) * 3.0).astype(np.float32)
    if V == 1:
        return x, {0: -30.0}
    bias = {0: -np.inf, V - 1: 30.0} if rng.rand() < 0.5 else {0: 30.0, V - 1: -np.inf}
    for k in rng.choice(np.arange(1, V - 1), size=min(V - 2, 24), replace=False):
        bias[int(k)] = float(rng.choice([-np.inf, -30.0, 30.0, 1.5]))
    return x, bias


FAMILIES = {
    "gauss0.05": _gauss(0.05), "gauss1": _gauss(1.0), "gauss3": _gauss(3.0), "gauss10": _gauss(10.0), "gauss30": _gauss(30.0),
    "ints": _ints, "dominant": _dominant, "dead50%": _dead(0.5), "dead99%": _dead(0.99), "dead-all-but-one": _dead(None),
    "dead-tail1": _tail(1), "dead-tail37": _tail(37), "dead-tail1029": _tail(1029), "dead-threads": _runs(False),
    "dead-warps": _runs(True), "bias": _bias,
}


# ---- the float64 side --------------------------------------------------------------------------------------------------------------

def adjust_top_p(vals, cum, top_p):
    """top_p moved at least TOP_P_MARGIN away from every tie-group boundary of the float64 cumulative mass (or into the middle of its
    gap where boundaries are closer than twice that), and onto a group whose probability is apart from the next group's by more
    than float32 rounding, so that the float32 and the float64 rules keep the same tokens. 0 and 1 mean no cut and stay."""
    if top_p in (0.0, 1.0) or len(vals) == 0:
        return top_p
    lo = np.concatenate([[0.0], cum[:-1]])                 # group k is kept last for top_p in [lo[k], cum[k])
    apart = np.append(vals[:-1] > vals[1:] * (1 + 1e-5), True)
    best = None
    for k in np.nonzero(apart)[0]:
        m = min(TOP_P_MARGIN, (cum[k] - lo[k]) / 4)
        a, b = (lo[k] + m if k > 0 else 0.0), cum[k] - m   # top_p just above 0 is no boundary: group 0 is always kept
        if b <= a:
            continue
        cand = float(np.float32(min(max(top_p, a), b)))
        if not (a <= cand <= b):
            continue
        if best is None or abs(cand - top_p) < abs(best - top_p):
            best = cand
        if cand == np.float32(top_p):
            break
    assert best is not None
    if best != np.float32(top_p):
        MOVES.append((len(vals), top_p, best))
    return best


class Row:
    """One row of logits (+ bias) with its float64 distributions cached per (T, top_p)."""

    def __init__(self, family, V, logits, bias):
        self.family, self.V, self.logits, self.bias = family, V, logits, bias
        self.vals, self.cum = so.top_p_boundaries(logits, bias)
        self.cache = {}

    def top_p(self, top_p):
        return adjust_top_p(self.vals, self.cum, top_p)

    def probs(self, t, top_p):
        key = (t, top_p)
        if key not in self.cache:
            p = so.probs64(self.logits, t, top_p, self.bias)
            self.cache[key] = (p, so.cdf64(p))
        return self.cache[key]

    def float32_resolution(self, t, top_p):
        """How far float32's absolute resolution of the softmax probabilities q (2^-149) can move the tempered CDF: every kept
        token's mass is uncertain by a relative 2^-149 / (q T). Zero for all practical purposes unless tokens with q near float32's
        subnormal range are kept at a large T, as with sigma 30 logits at T = 8."""
        key = ("resolution", t, top_p)
        if key not in self.cache:
            p, q = self.probs(t, top_p)[0], self.probs(1.0, 1.0)[0]
            kept = p > 0
            self.cache[key] = float(np.sum(p[kept] * 2.0 ** -149 / (q[kept] * t)))
        return self.cache[key]


def check_draw(row, t, top_p, u, tok, prob):
    """I1 - I4 for one draw; returns a message or None."""
    V, tok, prob = row.V, int(tok), float(prob)
    if not 0 <= tok < V:
        return "token %d out of range" % tok
    if t == 0.0:
        x = row.logits.copy()
        for k, v in (row.bias or {}).items():
            x[k] = np.float32(x[k] + np.float32(v))
        want = int(np.argmax(x))
        return None if tok == want and prob == 1.0 else "T = 0 drew %d (prob %r), argmax %d" % (tok, prob, want)
    p, cdf = row.probs(t, top_p)
    if not p[tok] > 0 and not so.probs64(row.logits, t, top_p, row.bias, float32_range=False)[tok] > 0:
        return "I1: token %d has float64 probability 0 (prob_out %r)" % (tok, prob)
    eps = eps_of(t) + row.float32_resolution(t, top_p)
    left = cdf[tok - 1] if tok > 0 else 0.0
    err = max(left - u, u - cdf[tok], 0.0)
    WORST[row.family] = max(WORST[row.family], err / eps)
    if err > 0 and not (left - eps <= u < cdf[tok] + eps):
        return "I2: u = %r outside [%r, %r) of token %d by %.3g (eps %.3g)" % (u, left, cdf[tok], tok, err, eps)
    # float32 holds the softmax probability q and prob_out itself to no better than 2^-149 absolute; tempering turns the first into a
    # relative error of 2^-149 / (q T), for this token and, summed, for the normaliser (float32_resolution). These terms matter only
    # for probabilities near or below float32's normal range.
    q = row.probs(1.0, 1.0)[0][tok]
    bar = (1e-5 * max(1.0, 1.0 / t) + row.float32_resolution(t, top_p)) * p[tok] + 2.0 ** -149 * (1.0 + p[tok] / (q * t))
    err = abs(prob - p[tok])
    WORST_P[row.family] = max(WORST_P[row.family], err / bar)
    if err > bar:
        return "I3: prob_out %r against float64 %r (error %.3g, bar %.3g)" % (prob, p[tok], err, bar)
    return None


def run_draws(lib, draws):
    """draws: [(row, T, top_p, u)] -> failure messages. Up to MAX_ROWS rows per launch."""
    bad = []
    for i in range(0, len(draws), MAX_ROWS):
        chunk = draws[i:i + MAX_ROWS]
        V = chunk[0][0].V
        assert all(d[0].V == V for d in chunk)
        ok, toks, probs = hook_batch(lib, np.stack([d[0].logits for d in chunk]), [d[1] for d in chunk], [d[2] for d in chunk],
                                     [d[3] for d in chunk], [d[0].bias for d in chunk])
        assert ok
        for (row, t, top_p, u), tok, prob in zip(chunk, toks, probs):
            msg = check_draw(row, t, top_p, u, tok, prob)
            if msg:
                bad.append((row.family, V, t, top_p, u, msg))
    return bad


# ---- 1. the grid -------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_draws_against_float64(lib):
    """Every n_vocab with every family; for each, every (T, top_p) pair, with u rotating over EDGE_US and three random values so
    that at every n_vocab every pair meets every u. Then I5: one row per n_vocab drawn at 256 sorted u."""
    rng = np.random.RandomState(20261016)
    bad = []
    for V in VOCABS:
        draws = []
        for f, (name, make) in enumerate(FAMILIES.items()):
            logits, bias = make(rng, V)
            row = Row(name, V, logits, bias)
            us = EDGE_US + list(rng.random_sample(3))
            for i, (t, tp) in enumerate((t, tp) for t in TEMPS for tp in TOP_PS):
                draws.append((row, t, row.top_p(tp), us[(i + f) % len(us)]))
        bad += run_draws(lib, draws)
        # I5: sorted u on one row with dead threads, including both ends
        row = Row("monotone", V, *_runs(False)(rng, V))
        us = np.sort(np.concatenate([EDGE_US, rng.random_sample(MAX_ROWS - len(EDGE_US))]))
        ok, toks, probs = hook_batch(lib, np.stack([row.logits] * MAX_ROWS), [1.0] * MAX_ROWS, [1.0] * MAX_ROWS, us)
        assert ok
        assert (np.diff(toks.astype(np.int64)) >= 0).all(), (V, toks)
        bad += [(row.family, V, 1.0, 1.0, u, m) for u, tok, prob in zip(us, toks, probs) for m in [check_draw(row, 1.0, 1.0, u, tok, prob)] if m]
    assert not bad, "%d bad draws, first: %s" % (len(bad), bad[:5])


# ---- 2. the kernel's own CDF edges -------------------------------------------------------------------------------------------------

def bits(x):
    return int(np.float64(x).view(np.int64))


def from_bits(b):
    return float(np.int64(b).view(np.float64))


def sparse_row(rng, V):
    """About 11 tokens with mass (logits within a factor of e^2 of each other), separated by -inf runs that cross thread and warp
    boundaries: the last token of a thread, the first of a later warp, neighbours, and -inf on V - 1 and on the last whole thread."""
    per = per_of(V)
    last_thread = (V - 1) // per * per
    cands = sorted({per - 1, per, 2 * per + 1, 32 * per - 1, 32 * per, 33 * per + per // 2, 64 * per + 3, V // 2, V // 2 + 1,
                    last_thread - 32 * per, last_thread - 1} & set(range(0, max(1, last_thread))))
    x = np.full(V, -np.inf, np.float32)
    x[cands] = rng.uniform(-1.0, 1.0, len(cands)).astype(np.float32)
    return x, cands


@pytest.mark.gpu
@pytest.mark.parametrize("V", [1000, 4096, 16385, 50277, 65536])
def test_kernel_cdf_edges(lib, V):
    """For every pair (a, b) of consecutive tokens with mass: the kernel's own edge between them, found by a 256-ary search over
    doubles, lies within eps of the float64 edge, and the 256 doubles around it draw only a or b, in order, with prob_out > 0. The
    256 doubles just below 1 draw the last token with mass."""
    rng = np.random.RandomState(V)
    logits, tokens = sparse_row(rng, V)
    assert len(tokens) >= 8
    row = Row("edges", V, logits, None)
    p, cdf = row.probs(1.0, 1.0)
    stacked = np.stack([logits] * MAX_ROWS)

    def draw(us):
        ok, toks, probs = hook_batch(lib, stacked[:len(us)], [1.0] * len(us), [1.0] * len(us), us)
        assert ok
        return toks.astype(np.int64), probs

    bad = []
    for a, b in zip(tokens[:-1], tokens[1:]):
        half = 0.25 * min(p[a], p[b])
        lo, hi = bits(cdf[a] - half), bits(cdf[a] + half)          # draws a at lo, b at hi
        while hi - lo > 1:
            probes = sorted({lo + (hi - lo) * k // 256 for k in range(1, 256)} - {lo, hi})
            toks, _ = draw([from_bits(q) for q in probes])
            assert set(toks) <= {a, b}, (a, b, set(toks))
            right = [q for q, t in zip(probes, toks) if t == b]
            left = [q for q, t in zip(probes, toks) if t == a]
            if left and right:
                assert max(left) < min(right), (a, b)
            lo = max(left) if left else lo
            hi = min(right) if right else hi
        edge = from_bits(hi)
        if abs(edge - cdf[a]) > eps_of(1.0):
            bad.append((a, b, "edge %r against float64 %r" % (edge, cdf[a])))
        us = [from_bits(q) for q in range(hi - 128, hi + 128)]
        toks, probs = draw(us)
        if not (set(toks) <= {a, b} and (np.diff(toks) >= 0).all() and (probs > 0).all()):
            bad.append((a, b, "around the edge: tokens %s, prob_out min %r" % (sorted(set(toks)), probs.min())))
    us = [from_bits(bits(1.0) - k) for k in range(MAX_ROWS, 0, -1)]
    toks, probs = draw(us)
    if not ((toks == tokens[-1]).all() and (probs > 0).all()):
        bad.append(("u -> 1", sorted(set(toks)), tokens[-1], float(probs.min())))
    assert not bad, bad


# ---- 3. tempering ------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_tempered_masses_do_not_underflow(lib):
    """T = 0.01, 0.03, 0.1 on near-uniform rows (sigma 0.01, where every p^(1/T) is below float32's range) and on rows whose largest
    probability is about 1e-3: I1 - I3 against float64, for u across [0, 1)."""
    rng = np.random.RandomState(7)
    V = 65536
    draws = []
    for kind in ("uniform", "pmax1e-3"):
        for t in (0.01, 0.03, 0.1):
            x = (rng.standard_normal(V) * 0.01).astype(np.float32)
            if kind == "pmax1e-3":
                x[rng.choice(V, 4, replace=False)] += np.float32(np.log(1e-3 * V / 4))
            row = Row("temper-" + kind, V, x, None)
            for tp in (1.0, 0.5):
                for u in EDGE_US + list(rng.random_sample(13)):
                    draws.append((row, t, row.top_p(tp), u))
    bad = run_draws(lib, draws)
    assert not bad, "%d bad draws, first: %s" % (len(bad), bad[:5])


# ---- 4. the generate step ----------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("V", [1000, 4097, 16385, 51200, 65536])
def test_constrained_step_never_draws_a_dead_token(lib, V):
    """The constrained step kernel with logits of sigma 8 and a state that allows a sparse set, V - 1 and the last whole thread
    dead: the token is allowed, the state moves along the table and the token's count goes up, for u at both ends and between.
    Rows with presence and frequency penalties through the unconstrained step satisfy I1 and I2."""
    rng = np.random.RandomState(V + 11)
    per = per_of(V)
    table = np.full((2, V), 0xFFFF, np.uint16)
    allowed = np.nonzero(rng.rand(V) < 0.05)[0]
    allowed = allowed[allowed < (V - 1) // per * per]
    table[0, allowed] = rng.randint(0, 2, len(allowed))
    table[1] = 0
    R = 64
    us = np.array((EDGE_US + [1 - 2.0 ** -52, 1 - 2.0 ** -53] * 4 + list(rng.random_sample(R)))[:R], np.float64)
    logits = (rng.standard_normal((R, V)) * 8.0).astype(np.float32)
    temps = [(1.0, 0.7, 1.7, 0.1)[b % 4] for b in range(R)]
    top_ps = [(1.0, 0.0, 1.0, 0.95, 1.0)[b % 5] for b in range(R)]
    zeros = [0.0] * R
    counts = np.zeros((R, V), np.uint32)
    ok, step, frozen, c2, toks, nxt, _, states = hook_constrained(lib, logits, table, [0] * R, [1] * R, temps, top_ps, zeros, zeros,
                                                                   us.reshape(R, 1), [], [0] * R, [0] * R, counts, np.zeros((R, 1), np.uint32))
    assert ok
    for b in range(R):
        tok = int(toks[b, 0])
        assert table[0, tok] != 0xFFFF, (b, tok, us[b], temps[b], top_ps[b])
        assert states[b] == int(table[0, tok]) and c2[b, tok] == 1 and c2[b].sum() == 1, b
    # penalties: the step's bias is -(presence + count * frequency) in float32 on every counted token
    pres, freq = [(0.0, 0.5, 3.0)[b % 3] for b in range(R)], [(1.5, 0.0, 0.25)[b % 3] for b in range(R)]
    counts = np.zeros((R, V), np.uint32)
    rows = []
    for b in range(R):
        ids = rng.choice(V, size=min(V, 200), replace=False)
        counts[b, ids] = rng.randint(1, 40, len(ids))
        rows.append(Row("penalties", V, logits[b], gr.penalty_bias({int(i): int(counts[b, i]) for i in ids}, pres[b], freq[b])))
    top_ps = [row.top_p(tp) for row, tp in zip(rows, top_ps)]
    ok, _, _, _, toks, _, _ = hook_step(lib, logits, [1] * R, temps, top_ps, pres, freq, us.reshape(R, 1), [], [0] * R, [0] * R, counts,
                                        np.zeros((R, 1), np.uint32))
    assert ok
    bad = []
    for b, row in enumerate(rows):
        p, cdf = row.probs(temps[b], top_ps[b])
        tok, eps = int(toks[b, 0]), eps_of(temps[b]) + row.float32_resolution(temps[b], top_ps[b])
        left = cdf[tok - 1] if tok > 0 else 0.0
        if not (p[tok] > 0 and left - eps <= us[b] < cdf[tok] + eps):
            bad.append((b, tok, us[b], p[tok], left, cdf[tok]))
    assert not bad, bad


# ---- 5. duplicate bias ids ---------------------------------------------------------------------------------------------------------

def test_duplicate_bias_ids_are_rejected_by_the_hooks(lib):
    """Both kernel hooks check their bias lists before they touch a device (passes without one): a duplicate id within a row, and
    for the single-row hook an id >= n_vocab, is RWKV_ERROR_ARGS. The same id in two different rows is no error."""
    V = 64
    logits = np.zeros(V, np.float32)
    tok, prob = ctypes.c_uint32(0), ctypes.c_float(0)

    def single(ids):
        n = len(ids)
        return lib.library.rwkv_b200_sample_logits(ptr(logits, P_F), V, 1.0, 1.0, 0.5, (ctypes.c_uint32 * n)(*ids), (ctypes.c_float * n)(*[1.0] * n), n,
                                                   ctypes.byref(tok), ctypes.byref(prob))

    for ids in ([3, 3], [0, 5, 9, 5], [V - 1, 2, V - 1], [V], [1, V + 7], [0xFFFFFFFF]):
        assert not single(ids), ids
        assert lib.rwkv_get_last_error(None) == ERR_ARGS, ids
    rows = np.zeros((3, V), np.float32)
    for off, ids in (([0, 2, 2, 3], [4, 4, 1]), ([0, 1, 4, 4], [7, 1, 2, 1]), ([0, 0, 0, 2], [V - 1, V - 1])):
        ok, _, _ = hook_batch_raw(lib, rows, off, ids)
        assert not ok and lib.rwkv_get_last_error(None) == ERR_ARGS, (off, ids)
    ok, _, _ = hook_batch_raw(lib, rows, [0, 2, 3, 5], [4, 1, 4, 1, 4])      # the same ids in different rows
    assert ok or lib.rwkv_get_last_error(None) != ERR_ARGS


def hook_batch_raw(lib, rows, off, ids):
    n_rows, V = rows.shape
    off, ids = np.array(off, np.uint32), np.array(ids, np.uint32)
    vals = np.ones(len(ids), np.float32)
    toks, probs = np.zeros(n_rows, np.uint32), np.zeros(n_rows, np.float32)
    one = lambda x: np.full(n_rows, x, np.float32)
    ok = lib.library.rwkv_b200_sample_logits_batch(ptr(rows, P_F), n_rows, V, ptr(one(1.0), P_F), ptr(one(1.0), P_F),
                                                   ptr(np.full(n_rows, 0.5), P_D), ptr(off, P_U), ptr(ids, P_U), ptr(vals, P_F), ptr(toks, P_U),
                                                   ptr(probs, P_F))
    return ok, toks, probs


@pytest.mark.gpu
def test_duplicate_bias_ids_rejected_by_the_context_calls(lib):
    """rwkv_b200_sample and rwkv_b200_batch_sample refuse a row that names a token twice; the refused call changes nothing, so the
    next valid call draws what it draws without it."""
    ctx = lib.rwkv_init_from_file(model_path("6v0-3m", "FP32"), 1, 0)
    batch = None
    try:
        assert lib.library.rwkv_b200_eval_resident(ctx.ptr, ptr(np.array([ord("a")], np.uint32), P_U), 1, True, None)
        tok = ctypes.c_uint32(0)

        def sample(bias):
            ids, vals, n = gr.bias_list(bias) if isinstance(bias, dict) else ((ctypes.c_uint32 * len(bias))(*[k for k, _ in bias]),
                                                                               (ctypes.c_float * len(bias))(*[v for _, v in bias]), len(bias))
            return lib.library.rwkv_b200_sample(ctx.ptr, 1.0, 0.9, 0.6, ids, vals, n, ctypes.byref(tok)), int(tok.value)

        ok, first = sample({5: 2.0, 9: -1.0})
        assert ok
        assert not sample([(5, 2.0), (9, -1.0), (5, 2.0)])[0]
        assert lib.library.rwkv_get_last_error(ctx.ptr) == ERR_ARGS
        assert sample({5: 2.0, 9: -1.0}) == (True, first)
        B = 3
        batch = ctypes.c_void_p(lib.library.rwkv_b200_batch_create(ctx.ptr, B))
        assert batch
        assert lib.library.rwkv_b200_batch_eval(batch, ptr(np.array([1, 2, 3], np.uint32), P_U), True)
        T, P, U = f32([1.0] * B), f32([0.9] * B), np.array([0.3, 0.6, 0.9])
        out = np.zeros(B, np.uint32)

        def bsample(off, ids):
            vals = np.ones(len(ids), np.float32)
            return lib.library.rwkv_b200_batch_sample(batch, ptr(T, P_F), ptr(P, P_F), ptr(U, P_D), ptr(np.array(off, np.uint32), P_U),
                                                      ptr(np.array(ids, np.uint32), P_U), ptr(vals, P_F), ptr(out, P_U))

        assert bsample([0, 2, 3, 5], [4, 1, 4, 1, 4])
        want = out.copy()
        assert not bsample([0, 2, 3, 5], [4, 1, 4, 1, 1])
        assert lib.library.rwkv_get_last_error(batch) == ERR_ARGS
        out[:] = 0
        assert bsample([0, 2, 3, 5], [4, 1, 4, 1, 4]) and np.array_equal(out, want)
    finally:
        if batch:
            lib.library.rwkv_free(batch)
        lib.rwkv_free(ctx)
