"""TEST INFRASTRUCTURE. A small byte-level DFA builder for the constrained-generation tests: the tiny fixtures' vocabulary is the 256
bytes, so a byte automaton is a token automaton. A pattern is a list of items, each a character class repeated lo..hi times,
cls(chars, lo, hi), or a group of items repeated lo..hi times, group([...], lo, hi). It is compiled through an NFA with epsilon moves
and the subset construction into the dense table of rwkv_b200_automaton_create: next[s, t] is the state after byte t, DEAD where t is
not allowed. State 0 is the start state."""
import numpy as np

DEAD = 0xFFFF


def cls(chars, lo=1, hi=1):
    return ("cls", frozenset(chars.encode() if isinstance(chars, str) else chars), lo, hi)


def group(items, lo=0, hi=1):
    return ("group", items, lo, hi)


def digits():
    return "0123456789"


class _NFA:
    def __init__(self):
        self.eps, self.moves = [], []      # per state: [targets], [(byte set, target)]

    def new(self):
        self.eps.append([])
        self.moves.append([])
        return len(self.eps) - 1

    def seq(self, items, start):
        for it in items:
            start = self.repeat(it, start)
        return start

    def once(self, it, start):
        if it[0] == "cls":
            end = self.new()
            self.moves[start].append((it[1], end))
            return end
        return self.seq(it[1], start)

    def repeat(self, it, start):
        lo, hi = it[2], it[3]
        for _ in range(lo):
            start = self.once(it, start)
        ends = [start]
        for _ in range(hi - lo):
            start = self.once(it, start)
            ends.append(start)
        end = self.new()
        for e in ends:
            self.eps[e].append(end)
        return end

    def closure(self, states):
        out, todo = set(states), list(states)
        while todo:
            for t in self.eps[todo.pop()]:
                if t not in out:
                    out.add(t)
                    todo.append(t)
        return frozenset(out)


class ByteDFA:
    """next: [n_states, n_vocab] uint16; accepting: [n_states] bool. eos (a token id) is allowed in accepting states only, as a
    self-loop (a stop id does not advance the state)."""

    def __init__(self, pattern, n_vocab=256, eos=None):
        nfa = _NFA()
        start = nfa.new()
        final = nfa.seq(pattern, start)
        sets, index, rows, accepting = [nfa.closure([start])], {}, [], []
        index[sets[0]] = 0
        i = 0
        while i < len(sets):
            cur = sets[i]
            row = np.full(n_vocab, DEAD, np.uint16)
            for byte in range(min(n_vocab, 256)):
                tgt = nfa.closure([t for s in cur for chars, t in nfa.moves[s] if byte in chars])
                if not tgt:
                    continue
                if tgt not in index:
                    index[tgt] = len(sets)
                    sets.append(tgt)
                row[byte] = index[tgt]
            accepting.append(final in cur)
            if eos is not None and accepting[-1]:
                row[eos] = i
            rows.append(row)
            i += 1
        self.next = np.ascontiguousarray(np.stack(rows))
        self.accepting = np.array(accepting)
        self.eos = eos

    @property
    def n_states(self):
        return self.next.shape[0]

    def walk(self, tokens, state=0):
        """The state after `tokens` (a stop id eos does not move it), or None where a token is not allowed."""
        for t in tokens:
            nxt = int(self.next[state, t])
            if nxt == DEAD:
                return None
            state = nxt
        return state

    def fullmatch(self, text: bytes):
        s = self.walk(text)
        return s is not None and bool(self.accepting[s])

    def prefix_ok(self, text: bytes):
        return self.walk(text) is not None

    def dead_end(self, state):
        return not (self.next[state] != DEAD).any()


# -?[0-9]{1,4}(\.[0-9]{1,2})?;  -- a number and a ';' after which nothing is allowed
NUMBER = [cls("-", 0, 1), cls(digits(), 1, 4), group([cls("."), cls(digits(), 1, 2)], 0, 1), cls(";")]
NUMBER_RE = rb"-?[0-9]{1,4}(\.[0-9]{1,2})?;"
# [a-z]{1,5}(,[a-z]{1,5}){0,2}  -- up to three short words; with eos, the end of text token ends it in an accepting state
WORDS = [cls("abcdefghijklmnopqrstuvwxyz", 1, 5), group([cls(","), cls("abcdefghijklmnopqrstuvwxyz", 1, 5)], 0, 2)]
WORDS_RE = rb"[a-z]{1,5}(,[a-z]{1,5}){0,2}"
