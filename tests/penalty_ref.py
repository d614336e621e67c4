"""TEST INFRASTRUCTURE. The penalty rules of device-side generation (include/rwkv_b200.h, rwkv_b200_set_penalty_decay) restated in
float32 numpy beside generate_ref.py: the bias of a float count table (rule 1), the update after an evaluated token (rule 3: decay
every count, then add the token's weight), and the host loop of rwkv_b200_sample + rwkv_b200_eval_resident that follows them."""
import numpy as np

import generate_ref as gr
from sampler_ref import sampler_bias


def penalty_bias(counts, presence, frequency, allowed=None):
    """{token: bias} for every counted token (count != 0): -(presence + c * frequency) in float32, the multiply and the add rounded
    separately. With `allowed` (a bool mask of the automaton state), a token it does not allow takes -inf whatever its count."""
    c = np.asarray(counts, np.float32)
    p, f = np.float32(presence), np.float32(frequency)
    ids = np.flatnonzero(c != 0)
    bias = {int(n): float(-(p + c[n] * f)) for n in ids}
    if allowed is not None:
        for n in np.flatnonzero(~np.asarray(allowed, bool)):
            bias[int(n)] = float("-inf")
    return dict(sorted(bias.items()))


def update(counts, tok, decay, weights=None):
    """The counts after evaluated token tok: every count times decay, then counts[tok] + weights[tok] (1 without a table), each
    rounded to float32 (with denormals). Returns a new array."""
    c = np.asarray(counts, np.float32)
    if decay != 1.0:
        c = c * np.float32(decay)
    else:
        c = c.copy()
    w = np.float32(1.0) if weights is None else np.float32(weights[tok])
    c[tok] = c[tok] + w
    return c


def row_bias(counts, presence, frequency, allowed=None, user=None):
    """The bias list of one draw: penalty_bias, or with a sampler's user entries the sampled family's rule (sampler_ref.sampler_bias)."""
    if not user:
        return penalty_bias(counts, presence, frequency, allowed)
    c = np.asarray(counts, np.float32)
    return sampler_bias({int(n): c[n] for n in np.flatnonzero(c != 0)}, presence, frequency, user, allowed)


def host_generate(lib, ctx_ptr, n_vocab, max_tokens, temperature, top_p, presence, frequency, us, stops=(), counts=None, decay=1.0,
                  weights=None, allowed=None, user=None):
    """The loop driven from the host under the penalty rules, one rwkv_b200_sample (bias from the float counts, row_bias) +
    rwkv_b200_eval_resident per evaluated token. Returns (tokens written, counts after)."""
    counts = np.zeros(n_vocab, np.float32) if counts is None else np.asarray(counts, np.float32).copy()
    out = []
    for i in range(max_tokens):
        tok = gr.sample(lib, ctx_ptr, temperature, top_p, us[i], row_bias(counts, presence, frequency, allowed, user))
        out.append(tok)
        if tok in stops:
            break
        counts = update(counts, tok, decay, weights)
        gr.eval_token(lib, ctx_ptr, tok)
    return out, counts
