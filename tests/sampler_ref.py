"""TEST INFRASTRUCTURE. Float64 restatement of one draw of rwkv_b200_generate_sampled (include/rwkv_b200.h, rules 1-5): the bias entries
of a row from its automaton state, penalty counts and user bias (rule 1, float32 as the kernel rounds them), and the distribution the
draw samples from after top-p, top_k, min_p and temperature (rules 2-5). oracle/sampling_oracle.probs64 is the same computation without
top_k / min_p; sampled_probs64 with both off returns its result."""
import numpy as np

from sampling_oracle import probs64


def sampler_bias(counts, presence, frequency, user=None, allowed=None):
    """{token: entry} of rule 1. counts: {token: count}; user: {token: value}; allowed: bool array of the state's tokens, or None."""
    p, f = np.float32(presence), np.float32(frequency)
    out = {}
    ids = set(int(n) for n, c in counts.items() if c > 0) | set(int(n) for n in (user or {}))
    for n in sorted(ids):
        if allowed is not None and not allowed[n]:
            continue
        c = counts.get(n, 0)
        pen = np.float32(p + np.float32(np.float32(c) * f))
        if user and n in user:
            out[n] = float(np.float32(np.float32(user[n]) - pen)) if c > 0 else float(np.float32(user[n]))
        else:
            out[n] = float(-pen)
    if allowed is not None:
        for n in np.nonzero(~np.asarray(allowed, bool))[0]:
            out[int(n)] = float("-inf")
    return out


def kept_mask(p, top_p, top_k=0, min_p=0.0):
    """Rule 4 on probabilities p (zeros for tokens without mass): the top-p cutoff of sampling.py:42-45, the top_k-th largest entry
    counted with multiplicity, and min_p * max(p). Each threshold is computed from the same p."""
    p = np.asarray(p, np.float64)
    keep = np.ones(p.size, bool)
    tp = 1.0 if top_p == 0.0 else float(top_p)
    if tp < 1.0:
        sp = np.sort(p)[::-1]
        keep &= p >= sp[np.argmax(np.cumsum(sp) > tp)]
    if top_k:
        keep &= p >= np.sort(p)[::-1][int(top_k) - 1]
    if min_p:
        keep &= p >= float(min_p) * p.max()
    return keep


def sampled_probs64(logits, temperature, top_p, top_k=0, min_p=0.0, bias=None):
    """The float64 distribution of a draw with entries `bias` (sampler_bias), rules 2-5. Temperature 0 gives the one-hot of the first
    maximum whatever top_k and min_p are."""
    if temperature == 0.0 or (top_k == 0 and min_p == 0.0):
        return probs64(logits, temperature, top_p, bias)
    p = probs64(logits, 1.0, 1.0, bias)
    p = np.where(kept_mask(p, top_p, top_k, min_p), p, 0.0)
    if temperature != 1.0:
        kept = p > 0
        lp = np.full(p.size, -np.inf)
        lp[kept] = np.log(p[kept])
        p = np.exp((lp - lp[kept].max()) / float(temperature))
    return p / p.sum()
