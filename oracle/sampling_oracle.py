"""TEST INFRASTRUCTURE (only tests/ may import this). CPU restatement of the reference's token sampling
(python/sampling.py:10-52) with the one random draw made explicit: `u` replaces the uniform number numpy.random.choice takes
from the global RandomState (legacy RandomState.choice with p: cdf = p.cumsum(); cdf /= cdf[-1]; idx = cdf.searchsorted(u, 'right')).
Pinned by tests/golden/sampling_cases.json, produced by running the reference module itself (tests/golden/make_sampling_golden.py)."""
import numpy as np


def softmax(x: np.ndarray) -> np.ndarray:                      # sampling.py:5-8 (float32 throughout for float32 logits)
    x = x - x.max(axis=-1, keepdims=True)
    e = np.exp(x)
    return e / e.sum(axis=-1, keepdims=True)


def sample_probs_u(probs: np.ndarray, temperature: float, top_p: float, u: float, logit_bias=None) -> int:
    if not (0.0 <= temperature):                               # :20-23
        raise ValueError("temperature")
    if not (0.0 <= top_p <= 1.0):
        raise ValueError("top_p")
    probs = probs.copy()
    if top_p == 0.0:                                           # :25-26
        top_p = 1.0
    if logit_bias:                                             # :28-37
        logits = np.log(probs)
        ids, values = zip(*logit_bias.items())
        logits[list(ids)] += values
        logits -= logits.max(axis=-1, keepdims=True)
        probs = np.exp(logits) / np.sum(np.exp(logits))
    if temperature == 0.0:                                     # :39-40
        return int(np.argmax(probs))
    if top_p < 1.0:                                            # :42-45
        sorted_probs = np.sort(probs)[::-1]
        cumulative = np.cumsum(sorted_probs)
        cutoff = float(sorted_probs[np.argmax(cumulative > top_p)])
        probs[probs < cutoff] = 0
    if temperature != 1.0:                                     # :47-48
        probs = np.power(probs, 1.0 / temperature)
    probs = probs / np.sum(probs)                              # :50
    cdf = probs.astype(np.float64).cumsum()                    # :52 numpy.random.choice(a, p=probs)
    cdf /= cdf[-1]
    return int(cdf.searchsorted(u, side="right"))


def sample_logits_u(logits: np.ndarray, temperature: float, top_p: float, u: float, logit_bias=None) -> int:   # :10-16
    return sample_probs_u(softmax(np.asarray(logits, dtype=np.float32).copy()), temperature, top_p, u, logit_bias)


def probs64(logits: np.ndarray, temperature: float, top_p: float, logit_bias=None, float32_range: bool = True) -> np.ndarray:
    """Each token's probability in float64 after bias, top-p and temperature: what the draw samples from, computed without the
    float32 rounding of the reference and the kernel. The biased logit is the float32 sum logits + bias, as the C API defines it;
    -inf becomes probability 0. With float32_range, so does a softmax probability below 2^-150, which the reference's float32
    softmax rounds to 0 (at T = 8 such tokens would otherwise hold whole percents of the mass). Top-p is the rule of
    sampling.py:42-45, keeping whole tie groups; tempering is exp((log p - log p_max) / T) over the kept tokens. temperature 0
    gives the one-hot of the first maximum."""
    x = np.asarray(logits, dtype=np.float32).copy()
    if logit_bias:
        for k, v in logit_bias.items():
            x[k] = np.float32(x[k] + np.float32(v))
    if temperature == 0.0:
        out = np.zeros(x.size)
        out[int(np.argmax(x))] = 1.0
        return out
    x = x.astype(np.float64)
    e = np.exp(x - x.max())
    p = e / e.sum()
    if float32_range:
        p[p < 2.0 ** -150] = 0.0
    tp = 1.0 if top_p == 0.0 else float(top_p)
    if tp < 1.0:
        sp = np.sort(p)[::-1]
        cutoff = sp[np.argmax(np.cumsum(sp) > tp)]
        p = np.where(p >= cutoff, p, 0.0)
    if temperature != 1.0:
        kept = p > 0
        lp = np.full(p.size, -np.inf)
        lp[kept] = np.log(p[kept])
        p = np.exp((lp - lp[kept].max()) / float(temperature))
    return p / p.sum()


def cdf64(probs: np.ndarray) -> np.ndarray:
    """The float64 CDF of probs64: token t owns [cdf[t - 1], cdf[t])."""
    c = np.cumsum(probs)
    return c / c[-1]


def top_p_boundaries(logits: np.ndarray, logit_bias=None) -> tuple:
    """(values, cumulative) of the float64 probabilities' tie groups, largest first: top_p in [cumulative[k - 1], cumulative[k])
    keeps groups 0 .. k."""
    p = probs64(logits, 1.0, 1.0, logit_bias)
    vals, counts = np.unique(p[p > 0], return_counts=True)
    vals, counts = vals[::-1], counts[::-1]
    return vals, np.cumsum(vals * counts)


def boundary_distance(logits: np.ndarray, temperature: float, top_p: float, u: float, logit_bias=None) -> float:
    """How far u is from the nearest edge of the chosen token's CDF interval (tests skip knife-edge draws)."""
    probs = softmax(np.asarray(logits, dtype=np.float32).copy())
    if temperature == 0.0:
        s = np.sort(probs)
        return float(s[-1] - s[-2])
    p = probs.copy()
    if logit_bias:
        lg = np.log(p); ids, values = zip(*logit_bias.items()); lg[list(ids)] += values; lg -= lg.max(); p = np.exp(lg) / np.sum(np.exp(lg))
    tp = 1.0 if top_p == 0.0 else top_p
    if tp < 1.0:
        sp = np.sort(p)[::-1]; cutoff = float(sp[np.argmax(np.cumsum(sp) > tp)]); p[p < cutoff] = 0
    if temperature != 1.0:
        p = np.power(p, 1.0 / temperature)
    p = p / p.sum()
    cdf = p.astype(np.float64).cumsum(); cdf /= cdf[-1]
    return float(np.min(np.abs(cdf - u)))
