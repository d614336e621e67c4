"""TEST INFRASTRUCTURE. Beam search (rwkv_b200_beam_search, rules 1-6 of its header comment) restated on the host for
tests/test_beam_host.py and tests/test_gpu_beam.py. The search itself (walk, search, results) knows nothing of models: a caller hands
it the candidates of a beam and a way to advance one. model_candidates / ModelBeams drive it over existing entry points only: one
single-sequence context with rwkv_b200_state_load / rwkv_b200_eval_resident / rwkv_b200_state_store per hypothesis step, and
rwkv_b200_score_logits for every log-probability."""
import ctypes

import numpy as np

P_F, P_U, P_D = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_double)


def top_order(z, n):
    """The first n ids of column z in the order of the logprob calls' top entries: larger logit first, smaller id first among equals."""
    z = np.asarray(z, np.float32)
    return np.lexsort((np.arange(len(z)), -z))[:n]


def walk(cands, scores, width, n_pool, stops):
    """One step's ranking and walk (rule 3). cands[b] = [(token, lp)] of live beam b in top-2W order, non-finite lp already dropped;
    scores[b] its score. Returns (taken, finished), each [(parent beam, token, score)] in the order taken."""
    ranked = sorted(((scores[b] + float(lp), b, j, t) for b, cs in enumerate(cands) for j, (t, lp) in enumerate(cs)),
                    key=lambda r: (-r[0], r[1], r[2]))
    taken, finished = [], []
    for sc, b, _, t in ranked:
        if len(taken) == width or n_pool + len(finished) == width:
            break
        (finished if t in stops else taken).append((b, t, sc))
    return taken, finished


def search(root, width, max_tokens, stops, candidates, advance):
    """Rules 3 and 6. candidates(handle) -> [(token, lp)]; advance(handle, token) -> the handle after that token. Returns the pool
    [(score, tokens)] in the order added and the live beams [(score, tokens, handle)] of the last step in slot order, and the live
    beams of the last step that took any (their handles are what the slots hold afterwards)."""
    live, pool, last_taken = [(0.0, [], root)], [], []
    for _ in range(max_tokens):
        taken, finished = walk([candidates(h) for _, _, h in live], [s for s, _, _ in live], width, len(pool), stops)
        pool += [(sc, live[b][1] + [t]) for b, t, sc in finished]
        live = [(sc, live[b][1] + [t], advance(live[b][2], t)) for b, t, sc in taken]
        if live:
            last_taken = live
        if len(pool) == width or not live:
            break
    return pool, live, last_taken


def results(pool, live, length_penalty, n_best):
    """Rules 4 and 5: [(tokens, score, finished)] of the n_best best hypotheses (fewer when fewer exist)."""
    hyps = [(toks, s, True) for s, toks in pool] + [(toks, s, False) for s, toks, _ in live]
    lp = float(np.float32(length_penalty))
    norm = [s / float(len(toks)) ** lp for toks, s, _ in hyps]
    order = sorted(range(len(hyps)), key=lambda i: -norm[i])
    return [hyps[i] for i in order[:n_best]]


# ---- over a model, through existing entry points ----------------------------------------------------------------------------------

def score_logits(lib, z, ids):
    """rwkv_b200_score_logits of column z for each target in ids."""
    n = len(ids)
    if n == 0:
        return np.zeros(0, np.float32)
    rows = np.ascontiguousarray(np.tile(np.asarray(z, np.float32), (n, 1)))
    tg = np.ascontiguousarray(ids, np.uint32)
    out = np.zeros(n, np.float32)
    assert lib.library.rwkv_b200_score_logits(rows.ctypes.data_as(P_F), n, rows.shape[1], tg.ctypes.data_as(P_U), out.ctypes.data_as(P_F), None)
    return out


def model_candidates(lib, z, width):
    ids = top_order(z, 2 * width)
    lps = score_logits(lib, z, ids)
    return [(int(t), float(l)) for t, l in zip(ids, lps) if np.isfinite(l)]


class ModelBeams:
    """Handles are (state, logits) numpy pairs; advance evaluates one token on a single-sequence context from the handle's state."""

    def __init__(self, lib, ctx_ptr, n_state, n_vocab):
        self.lib, self.ptr, self.n_state, self.n_vocab = lib, ctx_ptr, n_state, n_vocab

    def candidates(self, width):
        return lambda h: model_candidates(self.lib, h[1], width)

    def advance(self, h, tok):
        L = self.lib.library
        st = np.ascontiguousarray(h[0], np.float32)
        assert L.rwkv_b200_state_load(self.ptr, st.ctypes.data_as(P_F))
        assert L.rwkv_b200_eval_resident(self.ptr, (ctypes.c_uint32 * 1)(tok), 1, True, None)
        out, lg = np.zeros(self.n_state, np.float32), np.zeros(self.n_vocab, np.float32)
        assert L.rwkv_b200_state_store(self.ptr, out.ctypes.data_as(P_F))
        assert L.rwkv_b200_stage_logits(self.ptr, lg.ctypes.data_as(P_F), None)
        return out, lg

    def search(self, root, width, max_tokens, length_penalty, stops, n_best):
        """(results, live beams of the last step that took any) from root = (state, logits)."""
        pool, live, last = search(root, width, max_tokens, set(stops), self.candidates(width), self.advance)
        return results(pool, live, length_penalty, n_best), last
