"""TEST INFRASTRUCTURE. Seeded interleavings of every entry point on one context, replayed serially on a shadow.

The engine keeps host-side state that no single-feature test observes: the state_a / state_b swap and `phase`, the CUDA graphs keyed
by them, the scratch that ensure_capacity reallocates, logits_valid, the penalty count tables, automaton states. DESIGN section 3
makes a cheap exact reference possible: below 32 tokens per pass (16 columns in a batch context), or with the tensor cores off at any
length, every route gives the bytes of feeding the same tokens one at a time through rwkv_eval. So `step(state, token)` on a separate
plain context predicts the exact bytes after any sequence of calls.

A schedule is a list of (kind, parameters) and prints as a Python literal that run_schedule accepts back. run_schedule applies each op
to a driver (LibDriver: the ctypes library; ToyDriver: a numpy toy engine that can be given one defect) and to a Shadow, then compares
everything the op returned and audits the context. The Shadow's only arithmetic is driver.step, driver.sample_logits on its own logits
and the loop bookkeeping of generate_ref.py; it never calls the entry points under test."""
import ctypes
import hashlib
import random
from collections import Counter

import numpy as np

import byte_dfa as bd
import generate_ref as gr

ERR_ARGS, ERR_CTX, ERR_UNSUPPORTED = 1 << 8, 6 << 8, 9            # include/rwkv.h
P_F, P_U, P_D = gr.P_F, gr.P_U, gr.P_D
P_U8, P_U16 = ctypes.POINTER(ctypes.c_uint8), ctypes.POINTER(ctypes.c_uint16)
TOKEN_FN = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_uint32)
BOUNCE_DEFAULT = 4 << 20
TC_MIN_SINGLE, TC_MIN_BATCH = 32, 16                               # columns from which a pass takes the tensor cores

SINGLE_KINDS = ["eval", "eval_sequence", "eval_chunks", "state_load", "state_store", "eval_resident", "sample", "eval_sample", "generate",
                "generate_stream", "generate_constrained", "clone", "toggle", "profile_pass", "time_resident", "rejected"]
BATCH_KINDS = ["batch_eval", "batch_eval_ragged", "batch_set_state", "batch_get_state", "batch_get_logits", "batch_sample", "batch_eval_sample",
               "batch_generate", "batch_generate_stream", "batch_generate_constrained", "toggle", "rejected"]
# a batch of 16 takes the tensor cores in every pass: a loop whose tokens feed back cannot be replayed, so those kinds stay out
BATCH16_KINDS = [k for k in BATCH_KINDS if "generate" not in k]

# 3 .. 6 state automata over the byte vocabulary; ";" ends AB and NUM in a state that allows nothing
DFAS = {
    "ab": [bd.cls("ab", 1, 3), bd.cls(";")],
    "num": [bd.cls(bd.digits(), 1, 2), bd.cls(";")],
    "any": [bd.cls(bytes(range(256)), 1, 1), bd.cls(bytes(range(128)), 0, 1), bd.cls(bytes(range(256)), 1, 1)],
}


def dfa_table(name, n_vocab):
    return bd.ByteDFA(DFAS[name], n_vocab=n_vocab).next


# ---- schedules ---------------------------------------------------------------------------------------------------------------------

def de_bruijn_pairs(k):
    """A cyclic sequence of length k * k over 0 .. k - 1 in which every ordered pair (self pairs included) occurs once."""
    a, seq = [0] * (2 * k), []

    def db(t, p):
        if t > 2:
            if 2 % p == 0:
                seq.extend(a[1:p + 1])
            return
        a[t] = a[t - p]
        db(t + 1, p)
        for j in range(a[t - p] + 1, k):
            a[t] = j
            db(t + 1, t)
    db(1, 1)
    return seq


def kind_order(seed, kinds, n_ops):
    """The kinds of a schedule: a window of the pair cycle (consecutive seeds take consecutive windows, so ceil(K * K / (window - 1))
    seeds cover every ordered pair), then every kind the window missed."""
    K = len(kinds)
    cyc = de_bruijn_pairs(K)
    perm = list(range(K))
    random.Random(K).shuffle(perm)
    window = max(n_ops - K, 2)
    start = (seed * (window - 1)) % (K * K)
    order = [kinds[perm[cyc[(start + i) % (K * K)]]] for i in range(window)]
    order += [k for k in kinds if k not in order]
    rng = random.Random(seed)
    while len(order) < n_ops:
        order.append(rng.choice(kinds))
    return order


def seeds_for_all_pairs(kinds, n_ops):
    K = len(kinds)
    return -(-K * K // (max(n_ops - K, 2) - 1))


def _toks(rng, n):
    return [rng.randrange(256) for _ in range(n)]


def _mem(rng, device=True):
    return rng.choice(["pageable", "pinned", "device"] if device else ["pageable", "pinned"])


def _state_choice(rng):
    return rng.choice(["cur", "cur", "fresh", ("rewind", rng.randrange(8))])


def _draw(rng):
    return dict(temperature=rng.choice([0.0, 0.7, 1.0, 1.5]), top_p=rng.choice([0.0, 0.5, 0.9, 1.0]), u=rng.random())


def _bias(rng):
    n = rng.choice([0, 3, 40])
    return [(i, round(rng.uniform(-4, 4), 3)) for i in rng.sample(range(256), n)]


def _gen(rng, stream, constrained):
    n = rng.randrange(1, 10)
    g = dict(max_tokens=n, temperature=rng.choice([0.0, 0.7, 1.0, 1.5]), top_p=rng.choice([0.0, 0.5, 0.9, 1.0]),
             presence=rng.choice([0.0, 0.0, 0.4]), frequency=rng.choice([0.0, 0.0, 0.3]), keep=rng.random() < 0.5,
             us=[rng.random() for _ in range(n)], stop_ranks=rng.sample(range(4), rng.randrange(3)))
    if stream:
        g["end"] = rng.choice([None, 0, 1, n - 1])
    if constrained:
        g["dfa"] = rng.choice(sorted(DFAS))
        g["dfa_state"] = rng.choice(["carry", "carry", "reset", "dead"])
        g["end"] = rng.choice([None, 0, 1, n - 1]) if rng.random() < 0.5 else "blocking"
    return g


def _batch_gen(rng, B, stream, constrained):
    mt = [rng.choice([0, 0, 1, 2, 3, 5, 8, 9]) for _ in range(B)]
    if max(mt) == 0:
        mt[rng.randrange(B)] = 3
    n = max(mt)
    g = dict(max_tokens=mt, temperature=[rng.choice([0.0, 0.7, 1.0, 1.5]) for _ in range(B)], top_p=[rng.choice([0.0, 0.5, 0.9, 1.0]) for _ in range(B)],
             presence=[rng.choice([0.0, 0.4]) for _ in range(B)], frequency=[rng.choice([0.0, 0.3]) for _ in range(B)],
             keep=None if rng.random() < 0.25 else [rng.randrange(2) for _ in range(B)], us=[[rng.random() for _ in range(n)] for _ in range(B)],
             stop_ranks=rng.sample(range(4), rng.randrange(3)))
    if stream:
        g["end"] = [rng.choice([None, 0, 1, max(m - 1, 0)]) for m in mt]
    if constrained:
        g["dfa"] = [rng.choice(sorted(DFAS) + [None]) for _ in range(B)]
        g["dfa_state"] = [rng.choice(["carry", "carry", "reset", "dead"]) for _ in range(B)]
        g["end"] = [rng.choice([None, 0, 1, max(m - 1, 0)]) for m in mt] if rng.random() < 0.5 else "blocking"
    return g


def draw_params(kind, rng, large=False, tc_toggle=True, B=0):
    small_n, big_n = [1, 2, 7, 31], [32, 70, 256, 300]
    n = rng.choice(small_n + big_n if large else small_n)
    toggles = ["graphs", "overlap", "bounce", "trace_enable", "trace_disable"] + (["tensor_cores"] if tc_toggle else [])
    if kind == "eval":
        return dict(token=rng.randrange(256), state=_state_choice(rng), out=rng.random() < 0.7, logits=rng.random() < 0.7, mem=_mem(rng))
    if kind == "eval_sequence":
        return dict(tokens=_toks(rng, n), state=_state_choice(rng), out=rng.random() < 0.7, logits=rng.random() < 0.7, mem=_mem(rng))
    if kind == "eval_chunks":
        return dict(tokens=_toks(rng, rng.randrange(1, 91)), chunk=rng.choice([1, 7, 31, 64] if large else [1, 7, 31]), state=_state_choice(rng),
                    out=rng.random() < 0.7, logits=rng.random() < 0.7, mem=_mem(rng))
    if kind == "state_load":
        return dict(state=_state_choice(rng), mem=_mem(rng, False))
    if kind == "state_store":
        return dict(mem=_mem(rng, False))
    if kind == "eval_resident":
        return dict(tokens=_toks(rng, n), want=rng.random() < 0.7, fetch=rng.random() < 0.4, mem=_mem(rng, False))
    if kind == "sample":
        return dict(_draw(rng), bias=_bias(rng))
    if kind == "eval_sample":
        return dict(_draw(rng), token=rng.randrange(256))
    if kind in ("generate", "generate_stream", "generate_constrained"):
        return _gen(rng, kind == "generate_stream", kind == "generate_constrained")
    if kind == "clone":
        return dict(then=rng.choice(["clone", "parent", "both", "free_parent"]), state=_state_choice(rng), token=rng.randrange(256))
    if kind == "toggle":
        return dict(what=rng.choice(toggles), value=rng.random() < 0.5)
    if kind == "profile_pass":
        return dict(tokens=_toks(rng, rng.choice([1, 5])), want=rng.random() < 0.7)
    if kind == "time_resident":
        per, steps, warm = rng.choice([1, 5]), rng.randrange(1, 4), rng.randrange(2)
        return dict(tokens=_toks(rng, per * (steps + warm)), per=per, steps=steps, warm=warm, want=rng.random() < 0.7)
    if kind == "rejected":
        single = ["token_range", "no_head", "dup_bias", "u_one", "max_tokens_zero", "wrong_kind"]
        return dict(what=rng.choice(["token_range", "no_head", "dup_bias", "u_one", "ragged_sum", "wrong_kind"] if B else single))
    # batch kinds
    if kind == "batch_eval":
        return dict(tokens=_toks(rng, B), want=rng.random() < 0.7)
    if kind == "batch_eval_ragged":
        top = 256 if large else 15
        shape = rng.choice(["lone", "zeros", "all"])
        counts = [0] * B
        if shape == "lone":
            counts[rng.randrange(B)] = rng.randrange(1, top + 1) if large and rng.random() < 0.5 else rng.randrange(1, 16)
        else:
            budget = rng.randrange(B, top + 1) if large and rng.random() < 0.5 else rng.randrange(1, 16)
            for _ in range(budget):
                counts[rng.randrange(B)] += 1
            if shape == "zeros" and B > 1:
                counts[rng.randrange(B)] = 0
            if sum(counts) == 0:
                counts[0] = 1
        return dict(counts=counts, tokens=_toks(rng, sum(counts)), want=rng.random() < 0.7)
    if kind == "batch_set_state":
        return dict(seq=rng.randrange(B), state=rng.choice(["fresh", ("rewind", rng.randrange(8)), ("row", rng.randrange(B))]), mem=_mem(rng))
    if kind in ("batch_get_state", "batch_get_logits"):
        return dict(seq=rng.randrange(B), mem=_mem(rng))
    if kind == "batch_sample":
        d = [_draw(rng) for _ in range(B)]
        return dict(temperature=[x["temperature"] for x in d], top_p=[x["top_p"] for x in d], u=[x["u"] for x in d],
                    bias=None if rng.random() < 0.3 else [_bias(rng) for _ in range(B)])
    if kind == "batch_eval_sample":
        d = [_draw(rng) for _ in range(B)]
        return dict(tokens=_toks(rng, B), temperature=[x["temperature"] for x in d], top_p=[x["top_p"] for x in d], u=[x["u"] for x in d])
    if kind in ("batch_generate", "batch_generate_stream", "batch_generate_constrained"):
        return _batch_gen(rng, B, kind == "batch_generate_stream", kind == "batch_generate_constrained")
    raise ValueError(kind)


def make_schedule(seed, kinds, n_ops, **opts):
    """Deterministic: the kinds from kind_order, the parameters from random.Random(seed). opts: large (passes that take the tensor
    cores), tc_toggle (whether set_tensor_cores may be toggled), B (sequences of a batch context)."""
    rng = random.Random(seed * 7919 + len(kinds))
    return [(k, draw_params(k, rng, **opts)) for k in kind_order(seed, kinds, n_ops)]


def pairs_of(schedule):
    return {(a[0], b[0]) for a, b in zip(schedule, schedule[1:])}


# ---- the shadow --------------------------------------------------------------------------------------------------------------------

class Seq:
    """What the shadow holds per sequence."""

    def __init__(self, state, logits):
        self.state, self.logits, self.counts, self.history = state, logits, Counter(), []


class Shadow:
    def __init__(self, drv, n_seq=1):
        self.drv, self.V, self.fresh = drv, drv.n_vocab, drv.init_state().tobytes()
        self.seqs = [Seq(self.fresh, np.zeros(self.V, np.float32)) for _ in range(n_seq)]
        self.valid, self.tc, self.tracing = False, True, False
        self.auto = [None] * n_seq          # (dfa name, state) after the sequence's last constrained call

    def advance(self, b, tokens, want_logits):
        s = self.seqs[b]
        lg = None
        for t in tokens:
            s.state, lg = self.drv.step(s.state, int(t))
            s.history.append(int(t))
        if want_logits and lg is not None:
            s.logits = lg

    def set_state(self, b, state, history):
        self.seqs[b].state, self.seqs[b].history = state, list(history)

    def stops(self, b, ranks):
        order = np.argsort(-self.seqs[b].logits.astype(np.float64), kind="stable")
        return [int(order[r]) for r in ranks]

    def generate(self, b, max_tokens, temperature, top_p, presence, frequency, keep, us, stops, end=None, table=None, st=0):
        """The loop of rwkv_b200_generate* for one sequence: (tokens, automaton state, [(index, token)] delivered)."""
        s = self.seqs[b]
        if not keep:
            s.counts = Counter()
        out = []
        for i in range(max_tokens):
            bias = gr.penalty_bias(s.counts, presence, frequency)
            if table is not None:
                row = table[st]
                if not (row != bd.DEAD).any():
                    break
                for t in np.nonzero(row == bd.DEAD)[0]:
                    bias[int(t)] = float("-inf")
            tok = self.drv.sample_logits(s.logits, temperature, top_p, us[i], bias)
            out.append(tok)
            if tok in stops:
                break
            s.counts[tok] += 1
            self.advance(b, [tok], True)
            if table is not None:
                st = int(table[st][tok])
            if end is not None and i == end:
                break
        return out, st


# ---- running a schedule ------------------------------------------------------------------------------------------------------------

class Mismatch(AssertionError):
    pass


def check(cond, what, *detail):
    if not cond:
        raise Mismatch(f"{what} {detail if detail else ''}")


def same(got, want, what):
    check(got is not None and np.asarray(got).tobytes() == np.asarray(want).tobytes(), f"{what} differs from the serial replay")


def refused(drv, h, ok, flags, what):
    check(not ok, f"{what} must be refused")
    got = drv.last_error(h)
    check(got == flags, f"{what}: error flags", hex(got), hex(flags))


class Ctx:
    def __init__(self, handle, shadow):
        self.h, self.sh, self.recorded = handle, shadow, []


class Runner:
    """Applies ops to the driver and the shadow. tol: (max-abs bar for a pass on the tensor cores) or None when no such pass may occur."""

    def __init__(self, drv, B=0, tol=None, tc=True):
        self.drv, self.B, self.tol, self.tc = drv, B, tol, tc
        self.stats = dict(ops=Counter(), pairs=set(), graph_ops=0, rebases=0)
        self.root = drv.new_context()
        self.handles, self.tables = [self.root], {}
        if B:
            self.cur = Ctx(drv.batch_create(self.root, B), Shadow(drv, B))
            self.handles.append(self.cur.h)
        else:
            self.cur = Ctx(self.root, Shadow(drv))
            drv.state_load(self.root, None, "pageable")
        self.created(self.cur)
        self.other, self.alternate, self.bounce = None, 0, False

    def created(self, c):
        """tc False: the schedule runs with the tensor cores off, so every context it makes has them switched off."""
        if not self.tc:
            self.drv.toggle(c.h, "tensor_cores", False)
            c.sh.tc = False

    def close(self):
        if self.bounce:
            self.drv.toggle(self.cur.h, "bounce", False)
        for h in self.handles:
            self.drv.free(h)
        self.drv.free_tables()

    def free(self, h):
        self.handles.remove(h)
        self.drv.free(h)

    def table(self, name):
        if name not in self.tables:
            self.tables[name] = dfa_table(name, self.drv.n_vocab)
        return self.tables[name]

    def dead_state(self, name):
        t = self.table(name)
        return next(s for s in range(t.shape[0]) if not (t[s] != bd.DEAD).any())

    # -- helpers
    def resolve(self, c, choice, b=0):
        """(state bytes, history) of a state choice; None state = NULL = fresh."""
        if choice == "cur":
            return c.sh.seqs[b].state, c.sh.seqs[b].history
        if choice == "fresh" or not c.recorded:
            return None, []
        if choice[0] == "row":
            return c.sh.seqs[choice[1]].state, c.sh.seqs[choice[1]].history
        return c.recorded[choice[1] % len(c.recorded)]

    def inexact(self, c, columns):
        return c.sh.tc and columns >= (TC_MIN_BATCH if self.B else TC_MIN_SINGLE)

    def near(self, got, want, what):
        check(self.tol is not None, f"{what}: a pass took the tensor cores in a schedule that must stay bit-exact")
        g, w = (np.frombuffer(np.asarray(x).tobytes(), np.float32).astype(np.float64) for x in (got, want))
        # the bars are those of logits; a state is held to the same bar relative to its largest entry (WKV sums grow with the prompt)
        d, bar = float(np.abs(g - w).max()), self.tol * (max(1.0, float(np.abs(w).max())) if what.startswith("state") else 1.0)
        check(np.isfinite(g).all() and d <= bar, f"{what} is {d:.3g} from the serial replay, bar {bar:g}")

    def rebase(self, c):
        """After a pass on the tensor cores: within the bar of the replay, then the shadow adopts the bytes the context holds."""
        for b, s in enumerate(c.sh.seqs):
            st = self.drv.batch_get_state(c.h, b, "pageable") if self.B else self.drv.state_store(c.h, "pageable")
            self.near(st, np.frombuffer(s.state, np.float32), f"state of sequence {b}")
            s.state = st.tobytes()
            if c.sh.valid:
                lg = self.drv.batch_get_logits(c.h, b, "pageable")[1] if self.B else self.drv.raw_logits(c.h)
                self.near(lg, s.logits, f"logits of sequence {b}")
                s.logits = lg
        self.stats["rebases"] += 1

    def audit(self, c):
        drv, sh = self.drv, c.sh
        for b, s in enumerate(sh.seqs):
            st = drv.batch_get_state(c.h, b, "pageable") if self.B else drv.state_store(c.h, "pageable")
            same(st, np.frombuffer(s.state, np.float32), f"audit: resident state of sequence {b}")
        if self.B:
            for b, s in enumerate(sh.seqs):
                ok, lg = drv.batch_get_logits(c.h, b, "pageable")
                if sh.valid:
                    check(ok, "audit: batch_get_logits with valid logits")
                    same(lg, s.logits, f"audit: logits column {b}")
                else:
                    refused(drv, c.h, ok, ERR_ARGS, "audit: batch_get_logits while the logits are not valid")
        else:
            for temperature, u in ((0.0, 0.0), (1.0, 0.37)):
                ok, tok = drv.sample(c.h, temperature, 0.9, u, {})
                if sh.valid:
                    check(ok and tok == drv.sample_logits(sh.seqs[0].logits, temperature, 0.9, u, {}), "audit: sample from the current logits", tok)
                else:
                    refused(drv, c.h, ok, ERR_ARGS, "audit: sample while the logits are not valid")
        drv.release()

    # -- single-sequence ops
    def host_eval(self, c, p, tokens, call, max_pass):
        state, hist = self.resolve(c, p["state"])
        ok, st_out, lg_out = call(c.h, state, p["out"], p["logits"], p["mem"])
        check(ok, "the call failed", hex(self.drv.last_error(c.h)))
        c.sh.set_state(0, c.sh.fresh if state is None else state, hist)
        c.sh.advance(0, tokens, p["logits"])
        c.sh.valid = p["logits"]
        if self.inexact(c, max_pass):
            if p["out"]:
                self.near(st_out, np.frombuffer(c.sh.seqs[0].state, np.float32), "state_out")
            if p["logits"]:
                self.near(lg_out, c.sh.seqs[0].logits, "logits_out")
            self.rebase(c)
            if p["out"]:
                same(st_out, np.frombuffer(c.sh.seqs[0].state, np.float32), "state_out against the resident state")
            if p["logits"]:
                same(lg_out, c.sh.seqs[0].logits, "logits_out against the resident logits")
        else:
            if p["out"]:
                same(st_out, np.frombuffer(c.sh.seqs[0].state, np.float32), "state_out")
            if p["logits"]:
                same(lg_out, c.sh.seqs[0].logits, "logits_out")
        if p["out"]:
            c.recorded.append((c.sh.seqs[0].state, list(c.sh.seqs[0].history)))

    def op_eval(self, c, p):
        self.host_eval(c, p, [p["token"]], lambda h, s, o, l, m: self.drv.eval(h, p["token"], s, o, l, m), 1)

    def op_eval_sequence(self, c, p):
        self.host_eval(c, p, p["tokens"], lambda h, s, o, l, m: self.drv.eval_sequence(h, p["tokens"], s, o, l, m), min(len(p["tokens"]), 256))

    def op_eval_chunks(self, c, p):
        self.host_eval(c, p, p["tokens"], lambda h, s, o, l, m: self.drv.eval_chunks(h, p["tokens"], p["chunk"], s, o, l, m),
                       min(len(p["tokens"]), p["chunk"]))

    def op_state_load(self, c, p):
        state, hist = self.resolve(c, p["state"])
        check(self.drv.state_load(c.h, state, p["mem"]), "state_load failed")
        c.sh.set_state(0, c.sh.fresh if state is None else state, hist)

    def op_state_store(self, c, p):
        st = self.drv.state_store(c.h, p["mem"])
        same(st, np.frombuffer(c.sh.seqs[0].state, np.float32), "state_store")
        c.recorded.append((c.sh.seqs[0].state, list(c.sh.seqs[0].history)))

    def resident(self, c, tokens, want, got_logits=None):
        c.sh.advance(0, tokens, want)
        c.sh.valid = want
        if self.inexact(c, min(len(tokens), 256)):
            self.rebase(c)
        if got_logits is not None:
            same(got_logits, c.sh.seqs[0].logits, "logits_out")

    def op_eval_resident(self, c, p):
        ok, lg = self.drv.eval_resident(c.h, p["tokens"], p["want"], p["fetch"], p["mem"])
        check(ok, "eval_resident failed", hex(self.drv.last_error(c.h)))
        self.resident(c, p["tokens"], p["want"] or p["fetch"], lg if p["fetch"] else None)

    def op_sample(self, c, p):
        ok, tok = self.drv.sample(c.h, p["temperature"], p["top_p"], p["u"], dict(p["bias"]))
        if not c.sh.valid:
            return refused(self.drv, c.h, ok, ERR_ARGS, "sample after a pass that skipped the head")
        check(ok and tok == self.drv.sample_logits(c.sh.seqs[0].logits, p["temperature"], p["top_p"], p["u"], dict(p["bias"])), "sampled token", tok)

    def op_eval_sample(self, c, p):
        ok, tok = self.drv.eval_sample(c.h, p["token"], p["temperature"], p["top_p"], p["u"])
        check(ok, "eval_sample failed")
        self.resident(c, [p["token"]], True)
        check(tok == self.drv.sample_logits(c.sh.seqs[0].logits, p["temperature"], p["top_p"], p["u"], {}), "sampled token", tok)

    def gen_args(self, c, p, b, constrained):
        """Per-sequence arguments resolved against the shadow: (automaton name, table, start state)."""
        name = (p["dfa"][b] if self.B else p["dfa"]) if constrained else None
        if name is None:
            return None, None, 0
        mode = p["dfa_state"][b] if self.B else p["dfa_state"]
        prev = c.sh.auto[b]
        st = self.dead_state(name) if mode == "dead" else prev[1] if mode == "carry" and prev and prev[0] == name else 0
        return name, self.table(name), st

    def op_generate(self, c, p, kind="generate"):
        sh = c.sh
        constrained = kind == "generate_constrained"
        name, table, st = self.gen_args(c, p, 0, constrained)
        stops = sh.stops(0, p["stop_ranks"]) if sh.valid else []
        end = p.get("end")
        stream = kind == "generate_stream" or (constrained and end != "blocking")
        end = None if end == "blocking" else end
        res = self.drv.generate(c.h, dict(p, stops=stops, stream=stream, end=end, dfa=name, dfa_state=st))
        if not sh.valid:
            return refused(self.drv, c.h, res["ok"], ERR_ARGS, f"{kind} after a pass that skipped the head")
        check(res["ok"], f"{kind} failed", hex(self.drv.last_error(c.h)))
        want, st2 = sh.generate(0, p["max_tokens"], p["temperature"], p["top_p"], p["presence"], p["frequency"], p["keep"], p["us"], stops,
                                end if stream else None, table, st)
        check(res["tokens"] == want, "tokens / n_generated", res["tokens"], want)
        if stream:
            check(res["log"] == [(0, i, t) for i, t in enumerate(want)], "callback log", res["log"])
        if constrained:
            check(res["dfa_state"] == st2, "automaton state", res["dfa_state"], st2)
            sh.auto[0] = (name, st2)

    def op_generate_stream(self, c, p):
        self.op_generate(c, p, "generate_stream")

    def op_generate_constrained(self, c, p):
        self.op_generate(c, p, "generate_constrained")

    def op_clone(self, c, p):
        """rwkv_clone_context gives a new context of the same model: no logits, zero counts, and a state that is whatever the first
        load or rwkv_eval* gives it -- so the op loads one."""
        drv = self.drv
        if self.other:
            self.free(self.other.h)
            self.other, self.alternate = None, 0
        clone = Ctx(drv.clone(c.h), Shadow(drv))
        self.handles.append(clone.h)
        self.created(clone)
        state, hist = self.resolve(c, p["state"])
        check(drv.state_load(clone.h, state, "pageable"), "state_load of the clone failed")
        clone.sh.set_state(0, clone.sh.fresh if state is None else state, hist)
        clone.recorded = list(c.recorded)
        self.audit(clone)
        # its penalty counts start from zero whatever the parent has counted: a bias of +30 on every counted token would win a greedy draw
        self.op_eval_resident(clone, dict(tokens=[p["token"]], want=True, fetch=False, mem="pageable"))
        self.op_generate(clone, dict(max_tokens=1, temperature=0.0, top_p=1.0, presence=-30.0, frequency=0.0, keep=True, us=[0.5], stop_ranks=[]))
        self.audit(clone)
        if p["then"] == "free_parent":
            self.free(c.h)
            self.cur = clone
        elif p["then"] == "clone":
            self.cur, self.other = clone, c
        else:
            self.other = clone
            self.alternate = 6 if p["then"] == "both" else 0

    def op_toggle(self, c, p):
        what, value = p["what"], p["value"]
        if what == "trace_disable" and c.sh.tracing:
            check(self.drv.trace_read(c.h) >= 0, "trace_read failed")
        self.drv.toggle(c.h, what, value)
        if what == "tensor_cores":
            c.sh.tc = value
        if what == "bounce":
            self.bounce = value
        if what in ("trace_enable", "trace_disable"):
            c.sh.tracing = what == "trace_enable"

    def op_profile_pass(self, c, p):
        check(self.drv.profile_pass(c.h, p["tokens"], p["want"]), "profile_pass failed")
        self.resident(c, p["tokens"], p["want"])

    def op_time_resident(self, c, p):
        check(self.drv.time_resident(c.h, p["tokens"], p["per"], p["steps"], p["warm"], p["want"]) >= 0.0, "time_resident failed")
        self.resident(c, p["tokens"], p["want"])

    def op_rejected(self, c, p):
        drv, what, V = self.drv, p["what"], self.drv.n_vocab
        if what == "no_head":       # a legitimate pass without the head, after which every draw is refused
            if self.B:
                check(drv.batch_eval(c.h, [1] * self.B, False), "batch_eval failed")
                c.sh.valid = False
                self.batch_pass(c, [[1]] * self.B, False, self.B)
            else:
                check(drv.eval_resident(c.h, [1], False, False, "pageable")[0], "eval_resident failed")
                c.sh.advance(0, [1], False)
            c.sh.valid = False
            if self.B:
                refused(drv, c.h, drv.batch_sample(c.h, [1.0] * self.B, [1.0] * self.B, [0.5] * self.B, None)[0], ERR_ARGS, "batch_sample without logits")
                g = dict(max_tokens=[1] * self.B, temperature=[1.0] * self.B, top_p=[1.0] * self.B, presence=[0.0] * self.B, frequency=[0.0] * self.B,
                         keep=None, us=[[0.5]] * self.B, stops=[], stream=False, end=None, dfa=None, dfa_state=None)
                refused(drv, c.h, drv.batch_generate(c.h, g)["ok"], ERR_ARGS, "batch_generate without logits")
            else:
                refused(drv, c.h, drv.sample(c.h, 1.0, 1.0, 0.5, {})[0], ERR_ARGS, "sample without logits")
                g = dict(max_tokens=1, temperature=1.0, top_p=1.0, presence=0.0, frequency=0.0, keep=True, us=[0.5], stops=[], stream=False, end=None,
                         dfa=None, dfa_state=0)
                refused(drv, c.h, drv.generate(c.h, g)["ok"], ERR_ARGS, "generate without logits")
        elif what == "token_range":
            if self.B:
                refused(drv, c.h, drv.batch_eval(c.h, [0] * (self.B - 1) + [V], True), ERR_ARGS, "batch_eval of a token >= n_vocab")
                refused(drv, c.h, drv.batch_eval_ragged(c.h, [V], [1] + [0] * (self.B - 1), True), ERR_ARGS, "ragged pass of a token >= n_vocab")
            else:
                refused(drv, c.h, drv.eval(c.h, V, None, True, True, "pageable")[0], ERR_ARGS, "rwkv_eval of a token >= n_vocab")
                refused(drv, c.h, drv.eval_resident(c.h, [3, V], True, False, "pageable")[0], ERR_ARGS, "eval_resident of a token >= n_vocab")
        elif what == "dup_bias":
            if self.B:
                ok = drv.batch_sample(c.h, [1.0] * self.B, [1.0] * self.B, [0.5] * self.B, [[(7, 1.0), (7, 2.0)]] + [[]] * (self.B - 1))[0]
            else:
                ok = drv.sample(c.h, 1.0, 1.0, 0.5, [(7, 1.0), (7, 2.0)])[0]
            refused(drv, c.h, ok, ERR_ARGS, "a bias list that names a token twice")
        elif what == "u_one":
            ok = drv.batch_sample(c.h, [1.0] * self.B, [1.0] * self.B, [0.5] * (self.B - 1) + [1.0], None)[0] if self.B else drv.sample(c.h, 1.0, 1.0, 1.0, {})[0]
            refused(drv, c.h, ok, ERR_ARGS, "u = 1")
        elif what == "max_tokens_zero":
            g = dict(max_tokens=0, temperature=1.0, top_p=1.0, presence=0.0, frequency=0.0, keep=False, us=[0.5], stops=[], stream=False, end=None,
                     dfa=None, dfa_state=0)
            refused(drv, c.h, drv.generate(c.h, g)["ok"], ERR_ARGS, "generate with max_tokens = 0")
        elif what == "ragged_sum":
            refused(drv, c.h, drv.batch_eval_ragged(c.h, [], [0] * self.B, True), ERR_ARGS, "a ragged pass of no tokens")
        elif what == "wrong_kind":
            if self.B:
                refused(drv, c.h, drv.eval_resident(c.h, [1], True, False, "pageable")[0], ERR_CTX | ERR_UNSUPPORTED, "eval_resident on a batch context")
            else:
                refused(drv, c.h, drv.batch_eval_ragged(c.h, [1], [1], True), ERR_CTX | ERR_UNSUPPORTED, "a ragged pass on a single-sequence context")

    # -- batch ops
    def batch_pass(self, c, per_seq, want, columns):
        for b, toks in enumerate(per_seq):
            c.sh.advance(b, toks, want)
        if self.inexact(c, columns):
            self.rebase(c)

    def op_batch_eval(self, c, p):
        check(self.drv.batch_eval(c.h, p["tokens"], p["want"]), "batch_eval failed")
        c.sh.valid = p["want"]
        self.batch_pass(c, [[t] for t in p["tokens"]], p["want"], self.B)

    def split(self, p):
        out, i = [], 0
        for n in p["counts"]:
            out.append(p["tokens"][i:i + n])
            i += n
        return out

    def op_batch_eval_ragged(self, c, p):
        check(self.drv.batch_eval_ragged(c.h, p["tokens"], p["counts"], p["want"]), "batch_eval_ragged failed", hex(self.drv.last_error(c.h)))
        c.sh.valid = c.sh.valid or p["want"]        # idle columns keep what they held
        self.batch_pass(c, self.split(p), p["want"], sum(p["counts"]))

    def op_batch_set_state(self, c, p):
        state, hist = self.resolve(c, p["state"], p["seq"])
        check(self.drv.batch_set_state(c.h, p["seq"], state, p["mem"]), "batch_set_state failed")
        c.sh.set_state(p["seq"], c.sh.fresh if state is None else state, hist)

    def op_batch_get_state(self, c, p):
        s = c.sh.seqs[p["seq"]]
        same(self.drv.batch_get_state(c.h, p["seq"], p["mem"]), np.frombuffer(s.state, np.float32), "batch_get_state")
        c.recorded.append((s.state, list(s.history)))

    def op_batch_get_logits(self, c, p):
        ok, lg = self.drv.batch_get_logits(c.h, p["seq"], p["mem"])
        if not c.sh.valid:
            return refused(self.drv, c.h, ok, ERR_ARGS, "batch_get_logits after a pass that skipped the head")
        check(ok, "batch_get_logits failed")
        same(lg, c.sh.seqs[p["seq"]].logits, "batch_get_logits")

    def want_draws(self, c, p, bias):
        return [self.drv.sample_logits(c.sh.seqs[b].logits, p["temperature"][b], p["top_p"][b], p["u"][b], dict(bias[b]) if bias else {}) for b in range(self.B)]

    def op_batch_sample(self, c, p):
        ok, toks = self.drv.batch_sample(c.h, p["temperature"], p["top_p"], p["u"], p["bias"])
        if not c.sh.valid:
            return refused(self.drv, c.h, ok, ERR_ARGS, "batch_sample after a pass that skipped the head")
        check(ok and toks == self.want_draws(c, p, p["bias"]), "sampled tokens", toks)

    def op_batch_eval_sample(self, c, p):
        ok, toks = self.drv.batch_eval_sample(c.h, p["tokens"], p["temperature"], p["top_p"], p["u"])
        check(ok, "batch_eval_sample failed")
        c.sh.valid = True
        self.batch_pass(c, [[t] for t in p["tokens"]], True, self.B)
        check(toks == self.want_draws(c, p, None), "sampled tokens", toks)

    def op_batch_generate(self, c, p, kind="batch_generate"):
        sh, B = c.sh, self.B
        constrained = kind == "batch_generate_constrained"
        auto = [self.gen_args(c, p, b, constrained) for b in range(B)]
        stops = sh.stops(0, p["stop_ranks"]) if sh.valid else []
        end = p.get("end")
        stream = kind == "batch_generate_stream" or (constrained and end != "blocking")
        end = [None] * B if end in (None, "blocking") else end
        res = self.drv.batch_generate(c.h, dict(p, stops=stops, stream=stream, end=end, dfa=[a[0] for a in auto] if constrained else None,
                                                dfa_state=[a[2] for a in auto]))
        if not sh.valid:
            return refused(self.drv, c.h, res["ok"], ERR_ARGS, f"{kind} after a pass that skipped the head")
        check(res["ok"], f"{kind} failed", hex(self.drv.last_error(c.h)))
        for b in range(B):
            keep = bool(p["keep"][b]) if p["keep"] else False
            want, st2 = sh.generate(b, p["max_tokens"][b], p["temperature"][b], p["top_p"][b], p["presence"][b], p["frequency"][b], keep, p["us"][b], stops,
                                    end[b] if stream else None, auto[b][1], auto[b][2])
            check(res["tokens"][b] == want, f"tokens / n_generated of sequence {b}", res["tokens"][b], want)
            if stream:
                check([e for e in res["log"] if e[0] == b] == [(b, i, t) for i, t in enumerate(want)], f"callback log of sequence {b}", res["log"])
            if auto[b][0] is not None:
                check(res["dfa_state"][b] == st2, f"automaton state of sequence {b}", res["dfa_state"][b], st2)
                sh.auto[b] = (auto[b][0], st2)

    def op_batch_generate_stream(self, c, p):
        self.op_batch_generate(c, p, "batch_generate_stream")

    def op_batch_generate_constrained(self, c, p):
        self.op_batch_generate(c, p, "batch_generate_constrained")

    def run_op(self, kind, p):
        c = self.cur
        before = self.drv.graph_launches()
        getattr(self, "op_" + kind)(c, p)
        if self.drv.graph_launches() > before:
            self.stats["graph_ops"] += 1
        self.audit(self.cur)
        if self.other and (self.alternate > 0):
            self.alternate -= 1
            self.cur, self.other = self.other, self.cur


def run_schedule(drv, schedule, *, B=0, tol=None, tc=True, label="", seed=None, where=__file__, on_end=None):
    """Runs the schedule; a mismatch raises AssertionError naming the file, the seed, the failing op and the literal that replays it.
    Returns the run's statistics. on_end(runner) runs before the contexts are freed."""
    r = Runner(drv, B, tol, tc)
    try:
        prev = None
        for i, (kind, p) in enumerate(schedule):
            try:
                r.run_op(kind, p)
            except AssertionError as e:
                raise AssertionError(f"{where}: {label} seed {seed}: op {i} ({kind}) failed: {e}\nreplay with run_schedule(driver, {schedule[:i + 1]!r})") from None
            r.stats["ops"][kind] += 1
            if prev is not None:
                r.stats["pairs"].add((prev, kind))
            prev = kind
        if on_end:
            on_end(r)
    finally:
        r.close()
    return r.stats


# ---- the toy driver ----------------------------------------------------------------------------------------------------------------

TOY_V, TOY_S = 256, 16
DEFECTS = ["parity", "stale_graph", "idle_state", "frozen_logits", "keep_counts", "stop_advances", "valid_sticky", "profile_noop", "clone_counts"]


def toy_step(state, token):
    h = hashlib.blake2b(state + bytes([token & 255, token >> 8]), digest_size=8).digest()
    rng = np.random.RandomState(int.from_bytes(h[:4], "little"))
    return rng.standard_normal(TOY_S).astype(np.float32).tobytes(), (rng.standard_normal(TOY_V) * 3).astype(np.float32)


def toy_sample(logits, temperature, top_p, u, bias):
    x = logits.astype(np.float64)
    for i, v in dict(bias).items():
        x[i] += v
    if not np.isfinite(x).any():
        return 0
    p = np.exp(x - x[np.isfinite(x)].max())
    p[~np.isfinite(x)] = 0
    p /= p.sum()
    if temperature == 0:
        return int(np.argmax(p))
    if 0 < top_p < 1:
        srt = np.sort(p)[::-1]
        p[p < srt[int(np.argmax(np.cumsum(srt) >= top_p))]] = 0
    if temperature != 1:
        p = (p / p.max()) ** (1.0 / temperature)
    cdf = np.cumsum(p / p.sum())
    return int(np.nonzero(p)[0][np.searchsorted(cdf[np.nonzero(p)[0]], u, "right").clip(0, np.count_nonzero(p) - 1)])


class _ToyCtx:
    def __init__(self, n):
        fresh = np.zeros(TOY_S, np.float32).tobytes()
        self.n, self.state, self.before = n, [fresh] * n, [fresh] * n
        self.logits = [np.zeros(TOY_V, np.float32) for _ in range(n)]
        self.valid, self.counts, self.err = False, [Counter() for _ in range(n)], 0
        self.capacity, self.uses, self.captured, self.stale = 0, 0, None, False


class ToyDriver:
    """A toy recurrent model (state and logits from a hash of state and token) under the engine's bookkeeping written the obvious
    way. defect: one of DEFECTS breaks one rule."""
    n_vocab = TOY_V

    def __init__(self, defect=None):
        assert defect is None or defect in DEFECTS
        self.defect, self.batch = defect, {}

    def init_state(self):
        return np.zeros(TOY_S, np.float32)

    def step(self, state, token):
        return toy_step(state, token)

    def sample_logits(self, logits, temperature, top_p, u, bias):
        return toy_sample(logits, temperature, top_p, u, bias)

    def graph_launches(self):
        return 0

    def release(self):
        pass

    def free_tables(self):
        pass

    def new_context(self):
        return _ToyCtx(1)

    def clone(self, c):
        n = _ToyCtx(1)
        if self.defect == "clone_counts":
            n.counts = c.counts
        return n

    def batch_create(self, c, B):
        return _ToyCtx(B)

    def free(self, c):
        c.state = None

    def last_error(self, c):
        e, c.err = c.err, 0
        return e

    def _fail(self, c, flags):
        c.err = flags
        return False

    def _pass(self, c, per_seq, want):
        """One pass: sequence b advances per_seq[b] tokens."""
        T = sum(len(t) for t in per_seq)
        if T > c.capacity:
            c.capacity = T
            if self.defect == "stale_graph" and c.captured is not None:
                c.stale = True
            else:
                c.uses, c.captured = 0, None
        if c.n == 1 and T == 1:
            if c.stale:
                per_seq = [[c.captured]]
            elif c.captured is None:
                c.uses += 1
                if c.uses >= 2:
                    c.captured = per_seq[0][0]
        for b, toks in enumerate(per_seq):
            if not toks:
                if self.defect == "idle_state":
                    c.state[b], c.before[b] = c.before[b], c.state[b]
                continue
            c.before[b] = c.state[b]
            for t in toks:
                c.state[b], lg = toy_step(c.state[b], t)
            if want:
                c.logits[b] = lg
        return True

    def _valid(self, c, want):
        if not (self.defect == "valid_sticky" and c.valid and not want):
            c.valid = want

    def _range(self, c, tokens):
        return all(0 <= t < TOY_V for t in tokens) or self._fail(c, ERR_ARGS)

    def _host(self, c, tokens, chunk, state, out, logits):
        if c.n != 1:
            return self._fail(c, ERR_CTX | ERR_UNSUPPORTED), None, None
        if not self._range(c, tokens):
            return False, None, None
        c.state[0] = self.init_state().tobytes() if state is None else state
        for i in range(0, len(tokens), chunk):
            self._pass(c, [tokens[i:i + chunk]], logits and i + chunk >= len(tokens))
        self._valid(c, logits)
        return True, np.frombuffer(c.state[0], np.float32) if out else None, c.logits[0].copy() if logits else None

    def eval(self, c, token, state, out, logits, mem):
        return self._host(c, [token], 1, state, out, logits)

    def eval_sequence(self, c, tokens, state, out, logits, mem):
        return self._host(c, tokens, 256, state, out, logits)

    def eval_chunks(self, c, tokens, chunk, state, out, logits, mem):
        return self._host(c, tokens, chunk, state, out, logits)

    def state_load(self, c, state, mem):
        c.state[0] = self.init_state().tobytes() if state is None else state
        return True

    def state_store(self, c, mem):
        return np.frombuffer(c.state[0], np.float32)

    def raw_logits(self, c):
        return c.logits[0].copy()

    def eval_resident(self, c, tokens, want, fetch, mem):
        if c.n != 1:
            return self._fail(c, ERR_CTX | ERR_UNSUPPORTED), None
        if not self._range(c, tokens):
            return False, None
        for i in range(0, len(tokens), 256):
            self._pass(c, [tokens[i:i + 256]], (want or fetch) and i + 256 >= len(tokens))
        self._valid(c, want or fetch)
        return True, c.logits[0].copy() if fetch else None

    def _draw_ok(self, c, temperature, top_p, u, bias):
        ids = [i for i, _ in (bias.items() if isinstance(bias, dict) else bias)]
        return temperature >= 0 and 0 <= top_p <= 1 and 0 <= u < 1 and len(set(ids)) == len(ids) and all(i < TOY_V for i in ids)

    def sample(self, c, temperature, top_p, u, bias):
        if not self._draw_ok(c, temperature, top_p, u, bias) or not c.valid:
            return self._fail(c, ERR_ARGS), None
        return True, toy_sample(c.logits[0], temperature, top_p, u, bias)

    def eval_sample(self, c, token, temperature, top_p, u):
        ok, _ = self.eval_resident(c, [token], True, False, None)
        return self.sample(c, temperature, top_p, u, {}) if ok else (False, None)

    def _loop(self, c, rows, g, tables):
        """The generation loop over `rows`; per row the arguments are g[...][b] (already per row)."""
        n = len(rows)
        if not c.valid:
            return dict(ok=self._fail(c, ERR_ARGS))
        for b in rows:
            if not (g["keep"][b] and self.defect != "keep_counts"):
                c.counts[b] = Counter()
        step, frozen, out, log, st = [0] * n, [False] * n, [[] for _ in rows], [], list(g["dfa_state"])
        passes = 0
        while True:
            nxt = {}
            for b in rows:
                if frozen[b]:
                    continue
                row = tables[b][st[b]] if tables[b] is not None else None
                if step[b] == g["max_tokens"][b] or (row is not None and not (row != bd.DEAD).any()):
                    frozen[b] = True
                    continue
                bias = gr.penalty_bias(c.counts[b], g["presence"][b], g["frequency"][b])
                if row is not None:
                    for t in np.nonzero(row == bd.DEAD)[0]:
                        bias[int(t)] = float("-inf")
                tok = toy_sample(c.logits[b], g["temperature"][b], g["top_p"][b], g["us"][b][step[b]], bias)
                out[b].append(tok)
                log.append((b, step[b], tok))
                step[b] += 1
                if tok in g["stops"]:
                    frozen[b] = True
                    if self.defect == "stop_advances" and row is not None and row[tok] != bd.DEAD:
                        st[b] = int(row[tok])
                    continue
                c.counts[b][tok] += 1
                nxt[b] = tok
                if row is not None:
                    st[b] = int(row[tok])
                if g["stream"] and g["end"][b] is not None and g["end"][b] == step[b] - 1:
                    frozen[b] = True
            if not nxt:
                break
            passes += 1
            for b in rows:
                if b in nxt:
                    c.before[b] = c.state[b]
                    c.state[b], c.logits[b] = toy_step(c.state[b], nxt[b])
                elif self.defect == "frozen_logits":
                    c.logits[b] = toy_step(c.state[b], 0)[1]
        if self.defect == "parity" and passes % 2 == 1:
            c.state = list(c.before)
        if g["stream"]:
            log.sort(key=lambda e: e[1])       # tokens arrive step by step
        return dict(ok=True, tokens=out, log=log, dfa_state=st)

    def generate(self, c, g):
        if c.n != 1:
            return dict(ok=self._fail(c, ERR_CTX | ERR_UNSUPPORTED))
        if not 1 <= g["max_tokens"] <= 4096:
            return dict(ok=self._fail(c, ERR_ARGS))
        table = dfa_table(g["dfa"], TOY_V) if g["dfa"] else None
        per_row = {k: [g[k]] for k in ("max_tokens", "temperature", "top_p", "presence", "frequency", "keep", "us", "end", "dfa_state")}
        r = self._loop(c, [0], dict(per_row, stops=g["stops"], stream=g["stream"]), [table])
        return dict(r, tokens=r["tokens"][0], dfa_state=r["dfa_state"][0]) if r["ok"] else r

    # batch
    def _batch(self, c):
        return c.n > 1 or self._fail(c, ERR_CTX | ERR_UNSUPPORTED)

    def batch_eval(self, c, tokens, want):
        if not self._batch(c) or not self._range(c, tokens):
            return False
        self._pass(c, [[t] for t in tokens], want)
        self._valid(c, want)
        return True

    def batch_eval_ragged(self, c, tokens, counts, want):
        if not self._batch(c):
            return False
        if not 1 <= sum(counts) <= 256 or not self._range(c, tokens):
            return self._fail(c, ERR_ARGS)
        per, i = [], 0
        for n in counts:
            per.append(tokens[i:i + n])
            i += n
        self._pass(c, per, want)
        self._valid(c, c.valid or want)
        return True

    def batch_set_state(self, c, seq, state, mem):
        c.state[seq] = self.init_state().tobytes() if state is None else state
        return True

    def batch_get_state(self, c, seq, mem):
        return np.frombuffer(c.state[seq], np.float32)

    def batch_get_logits(self, c, seq, mem):
        if not c.valid:
            return self._fail(c, ERR_ARGS), None
        return True, c.logits[seq].copy()

    def batch_sample(self, c, temperature, top_p, u, bias):
        if not all(self._draw_ok(c, temperature[b], top_p[b], u[b], bias[b] if bias else {}) for b in range(c.n)) or not c.valid:
            return self._fail(c, ERR_ARGS), None
        return True, [toy_sample(c.logits[b], temperature[b], top_p[b], u[b], dict(bias[b]) if bias else {}) for b in range(c.n)]

    def batch_eval_sample(self, c, tokens, temperature, top_p, u):
        return self.batch_sample(c, temperature, top_p, u, None) if self.batch_eval(c, tokens, True) else (False, None)

    def batch_generate(self, c, g):
        if not self._batch(c):
            return dict(ok=False)
        tables = [dfa_table(d, TOY_V) if d else None for d in (g["dfa"] or [None] * c.n)]
        return self._loop(c, list(range(c.n)), dict(g, keep=g["keep"] or [0] * c.n), tables)

    def toggle(self, c, what, value):
        pass

    def trace_read(self, c):
        return 0

    def profile_pass(self, c, tokens, want):
        return True if self.defect == "profile_noop" else self.eval_resident(c, tokens, want, False, None)[0]

    def time_resident(self, c, tokens, per, steps, warm, want):
        for i in range(0, len(tokens), per):
            self.eval_resident(c, tokens[i:i + per], want, False, None)
        return 0.0


# ---- the library driver ------------------------------------------------------------------------------------------------------------

class _Buf:
    """n floats of pageable (numpy), pinned or device (torch) memory."""

    def __init__(self, n, mem, init=None):
        a = np.zeros(n, np.float32) if init is None else np.frombuffer(init, np.float32).copy()
        if mem == "pageable":
            self.a, self.t, self.addr = a, None, a.ctypes.data
        else:
            import torch
            t = torch.from_numpy(a)
            self.t = t.pin_memory() if mem == "pinned" else t.cuda()
            if mem == "device":
                torch.cuda.synchronize()
            self.addr = self.t.data_ptr()

    def ptr(self):
        return ctypes.cast(self.addr, P_F)

    def get(self):
        return self.a.copy() if self.t is None else self.t.cpu().numpy().copy()


def _u32(xs):
    return (ctypes.c_uint32 * max(len(xs), 1))(*xs)


def _f32(xs):
    return (ctypes.c_float * len(xs))(*xs)


class LibDriver:
    """The ctypes library on one model file. step() runs on a context of its own rwkv_init_from_file with graphs, overlap and tensor
    cores off and pageable buffers."""

    def __init__(self, lib, path):
        self.lib, self.L, self.path = lib, lib.library, path
        self.ref = lib.rwkv_init_from_file(path, 1, 0)
        for f in (self.L.rwkv_b200_set_graphs, self.L.rwkv_b200_set_tensor_cores, self.L.rwkv_b200_set_overlap):
            f(self.ref.ptr, False)
        self.n_vocab = lib.rwkv_get_logits_buffer_element_count(self.ref)
        self.n_state = lib.rwkv_get_state_buffer_element_count(self.ref)
        self.memo, self.memo_bytes, self.live, self.autos = {}, 0, [], {}

    def close(self):
        self.free_tables()
        self.lib.rwkv_free(self.ref)

    def init_state(self):
        st = np.zeros(self.n_state, np.float32)
        self.lib.rwkv_init_state(self.ref, st.ctypes.data)
        return st

    def step(self, state, token):
        key = (hashlib.blake2b(state, digest_size=16).digest(), token)
        if key not in self.memo:
            s_in, s_out, lg = np.frombuffer(state, np.float32), np.zeros(self.n_state, np.float32), np.zeros(self.n_vocab, np.float32)
            assert self.L.rwkv_eval(self.ref.ptr, token, s_in.ctypes.data_as(P_F), s_out.ctypes.data_as(P_F), lg.ctypes.data_as(P_F))
            if self.memo_bytes > 256 << 20:
                self.memo, self.memo_bytes = {}, 0
            self.memo[key] = (s_out.tobytes(), lg)
            self.memo_bytes += 4 * (self.n_state + self.n_vocab)
        return self.memo[key]

    def sample_logits(self, logits, temperature, top_p, u, bias):
        ids, vals, n = gr.bias_list(dict(bias))
        tok = ctypes.c_uint32(0)
        assert self.L.rwkv_b200_sample_logits(logits.ctypes.data_as(P_F), self.n_vocab, temperature, top_p, float(u), ids, vals, n, ctypes.byref(tok), None)
        return int(tok.value)

    def graph_launches(self):
        return int(self.L.rwkv_b200_graph_launch_count())

    def release(self):
        self.live = []

    def new_context(self):
        return self.lib.rwkv_init_from_file(self.path, 1, 0)

    def clone(self, c):
        return self.lib.rwkv_clone_context(c, 1)

    def batch_create(self, c, B):
        p = self.L.rwkv_b200_batch_create(c.ptr, B)
        assert p
        return type(c)(p)

    def free(self, c):
        self.lib.rwkv_free(c)

    def last_error(self, c):
        return int(self.lib.rwkv_get_last_error(c))

    def _in(self, state, mem):
        if state is None:
            return None
        b = _Buf(self.n_state, mem, state)
        self.live.append(b)
        return b.ptr()

    def _host(self, call, state, out, logits, mem):
        s_out, lg = _Buf(self.n_state, mem) if out else None, _Buf(self.n_vocab, mem) if logits else None
        ok = call(self._in(state, mem), s_out.ptr() if out else None, lg.ptr() if logits else None)
        return ok, s_out.get() if ok and out else None, lg.get() if ok and logits else None

    def eval(self, c, token, state, out, logits, mem):
        return self._host(lambda s, o, l: self.L.rwkv_eval(c.ptr, token, s, o, l), state, out, logits, mem)

    def eval_sequence(self, c, tokens, state, out, logits, mem):
        return self._host(lambda s, o, l: self.L.rwkv_eval_sequence(c.ptr, _u32(tokens), len(tokens), s, o, l), state, out, logits, mem)

    def eval_chunks(self, c, tokens, chunk, state, out, logits, mem):
        return self._host(lambda s, o, l: self.L.rwkv_eval_sequence_in_chunks(c.ptr, _u32(tokens), len(tokens), chunk, s, o, l), state, out, logits, mem)

    def state_load(self, c, state, mem):
        return self.L.rwkv_b200_state_load(c.ptr, self._in(state, mem))

    def state_store(self, c, mem):
        b = _Buf(self.n_state, mem)
        assert self.L.rwkv_b200_state_store(c.ptr, b.ptr())
        return b.get()

    def raw_logits(self, c):
        lg = np.zeros(self.n_vocab, np.float32)
        assert self.L.rwkv_b200_stage_logits(c.ptr, lg.ctypes.data_as(P_F), None)
        return lg

    def eval_resident(self, c, tokens, want, fetch, mem):
        lg = _Buf(self.n_vocab, mem) if fetch else None
        ok = self.L.rwkv_b200_eval_resident(c.ptr, _u32(tokens), len(tokens), want, lg.ptr() if fetch else None)
        return ok, lg.get() if ok and fetch else None

    def sample(self, c, temperature, top_p, u, bias):
        pairs = list(bias.items()) if isinstance(bias, dict) else list(bias)
        tok = ctypes.c_uint32(0)
        ok = self.L.rwkv_b200_sample(c.ptr, temperature, top_p, float(u), _u32([i for i, _ in pairs]) if pairs else None,
                                     _f32([v for _, v in pairs]) if pairs else None, len(pairs), ctypes.byref(tok))
        return ok, int(tok.value)

    def eval_sample(self, c, token, temperature, top_p, u):
        tok = ctypes.c_uint32(0)
        ok = self.L.rwkv_b200_eval_sample(c.ptr, token, temperature, top_p, float(u), ctypes.byref(tok))
        return ok, int(tok.value)

    def automaton(self, c, name):
        if name not in self.autos:
            table = np.ascontiguousarray(dfa_table(name, self.n_vocab), np.uint16)
            p = self.L.rwkv_b200_automaton_create(c.ptr, table.ctypes.data_as(P_U16), table.shape[0])
            assert p
            self.autos[name] = p
        return self.autos[name]

    def free_tables(self):
        for p in self.autos.values():
            self.L.rwkv_b200_automaton_free(p)
        self.autos = {}

    def _recorder(self, ends):
        log = []

        def on_token(user, seq, index, token):
            log.append((int(seq), int(index), int(token)))
            return 1 if ends[seq] is not None and index == ends[seq] else 0
        return log, TOKEN_FN(on_token)

    def keep_flag(self, g):          # what the call is given as keep_counts; the teeth tests override it
        return g["keep"]

    def generate(self, c, g):
        n = max(g["max_tokens"], 1)
        toks, ng, st = np.zeros(n, np.uint32), ctypes.c_size_t(0), np.array([g["dfa_state"] or 0], np.uint32)
        us = np.ascontiguousarray(g["us"] + [0.5] * (n - len(g["us"])), np.float64)
        log, fn = self._recorder([g["end"]])
        args = (g["max_tokens"], g["temperature"], g["top_p"], g["presence"], g["frequency"], self.keep_flag(g), us.ctypes.data_as(P_D),
                _u32(g["stops"]) if g["stops"] else None, len(g["stops"]))
        tail = (toks.ctypes.data_as(P_U), ctypes.byref(ng))
        if g["dfa"]:
            ok = self.L.rwkv_b200_generate_constrained(c.ptr, self.automaton(c, g["dfa"]), st.ctypes.data_as(P_U), *args, fn if g["stream"] else TOKEN_FN(), None, *tail)
        elif g["stream"]:
            ok = self.L.rwkv_b200_generate_stream(c.ptr, *args, fn, None, *tail)
        else:
            ok = self.L.rwkv_b200_generate(c.ptr, *args, *tail)
        return dict(ok=ok, tokens=[int(t) for t in toks[:ng.value]], log=log, dfa_state=int(st[0]))

    # batch
    def batch_eval(self, c, tokens, want):
        return self.L.rwkv_b200_batch_eval(c.ptr, _u32(tokens), want)

    def ragged_tokens(self, tokens, counts):      # the token array a ragged call is given; the teeth tests override it
        return tokens

    def batch_eval_ragged(self, c, tokens, counts, want):
        return self.L.rwkv_b200_batch_eval_ragged(c.ptr, _u32(self.ragged_tokens(tokens, counts)), _u32(counts), want)

    def batch_set_state(self, c, seq, state, mem):
        return self.L.rwkv_b200_batch_set_state(c.ptr, seq, self._in(state, mem))

    def batch_get_state(self, c, seq, mem):
        b = _Buf(self.n_state, mem)
        assert self.L.rwkv_b200_batch_get_state(c.ptr, seq, b.ptr())
        return b.get()

    def batch_get_logits(self, c, seq, mem):
        b = _Buf(self.n_vocab, mem)
        ok = self.L.rwkv_b200_batch_get_logits(c.ptr, seq, b.ptr())
        return ok, b.get() if ok else None

    def batch_sample(self, c, temperature, top_p, u, bias):
        B = len(u)
        out = (ctypes.c_uint32 * B)()
        off = ids = vals = None
        if bias is not None:
            flat = [e for row in bias for e in row]
            offs = [0]
            for row in bias:
                offs.append(offs[-1] + len(row))
            off, ids, vals = _u32(offs), _u32([i for i, _ in flat]), _f32([v for _, v in flat] or [0.0])
        ok = self.L.rwkv_b200_batch_sample(c.ptr, _f32(temperature), _f32(top_p), (ctypes.c_double * B)(*u), off, ids, vals, out)
        return ok, [int(t) for t in out]

    def batch_eval_sample(self, c, tokens, temperature, top_p, u):
        B = len(u)
        out = (ctypes.c_uint32 * B)()
        ok = self.L.rwkv_b200_batch_eval_sample(c.ptr, _u32(tokens), _f32(temperature), _f32(top_p), (ctypes.c_double * B)(*u), out)
        return ok, [int(t) for t in out]

    def batch_generate(self, c, g):
        B = len(g["max_tokens"])
        n = max(max(g["max_tokens"]), 1)
        toks, ng = np.zeros(B * n, np.uint32), np.zeros(B, np.uint32)
        us = np.ascontiguousarray([list(r[:n]) + [0.5] * (n - len(r[:n])) for r in g["us"]], np.float64)
        st = np.array([s or 0 for s in g["dfa_state"]] if g["dfa_state"] else [0] * B, np.uint32)
        keep = self.keep_flag(g)
        keep = None if keep is None else np.asarray(keep, np.uint8)
        log, fn = self._recorder(g["end"] or [None] * B)
        args = (_u32(g["max_tokens"]), _f32(g["temperature"]), _f32(g["top_p"]), _f32(g["presence"]), _f32(g["frequency"]),
                None if keep is None else keep.ctypes.data_as(P_U8), us.ctypes.data_as(P_D), _u32(g["stops"]) if g["stops"] else None, len(g["stops"]))
        tail = (toks.ctypes.data_as(P_U), ng.ctypes.data_as(P_U))
        if g["dfa"]:
            autos = (ctypes.c_void_p * B)(*[self.automaton(c, d) if d else None for d in g["dfa"]])
            ok = self.L.rwkv_b200_batch_generate_constrained(c.ptr, autos, st.ctypes.data_as(P_U), *args, fn if g["stream"] else TOKEN_FN(), None, *tail)
        elif g["stream"]:
            ok = self.L.rwkv_b200_batch_generate_stream(c.ptr, *args, fn, None, *tail)
        else:
            ok = self.L.rwkv_b200_batch_generate(c.ptr, *args, *tail)
        return dict(ok=ok, tokens=[[int(t) for t in toks[b * n:b * n + ng[b]]] for b in range(B)], log=log, dfa_state=[int(s) for s in st])

    def toggle(self, c, what, value):
        L = self.L
        if what == "graphs":
            L.rwkv_b200_set_graphs(c.ptr, value)
        elif what == "tensor_cores":
            L.rwkv_b200_set_tensor_cores(c.ptr, value)
        elif what == "overlap":
            L.rwkv_b200_set_overlap(c.ptr, value)
        elif what == "bounce":
            L.rwkv_b200_set_bounce_min_bytes(0 if value else BOUNCE_DEFAULT)
        elif what == "trace_enable":
            assert L.rwkv_b200_trace_enable(c.ptr)
        elif what == "trace_disable":
            L.rwkv_b200_trace_disable(c.ptr)

    def trace_read(self, c):
        start, end, names = (ctypes.c_double * 1024)(), (ctypes.c_double * 1024)(), ctypes.create_string_buffer(1024 * 32)
        return self.L.rwkv_b200_trace_read(c.ptr, start, end, names, 1024)

    def profile_pass(self, c, tokens, want):
        from importlib import import_module
        prof = import_module(type(self.lib).__module__).ProfileResult()
        return self.L.rwkv_b200_profile_pass(c.ptr, _u32(tokens), len(tokens), want, ctypes.byref(prof))

    def time_resident(self, c, tokens, per, steps, warm, want):
        return self.L.rwkv_b200_time_resident(c.ptr, _u32(tokens), per, steps, warm, want)
