"""TEST INFRASTRUCTURE. The generation loop of the reference's scripts restated on the host for tests/test_*generate*.py: the
presence / frequency penalty of python/chat_with_bot.py:244-247 as a float32 logit bias, and the per-step bookkeeping (budget, stop
ids, counts) of :249-260 and python/generate_completions.py:60-67."""
import ctypes
from collections import Counter

import numpy as np

P_F, P_U, P_D = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_double)


def penalty_bias(counts, presence, frequency):
    """{token: bias} for every counted token: -(presence + count * frequency) in float32, the multiply and the add rounded
    separately (chat_with_bot.py:246-247: logits[n] -= presence_penalty + occurrence[n] * frequency_penalty)."""
    p, f = np.float32(presence), np.float32(frequency)
    return {int(n): float(-(p + np.float32(c) * f)) for n, c in sorted(counts.items()) if c > 0}


def bias_list(bias):
    n = len(bias)
    if not n:
        return None, None, 0
    return (ctypes.c_uint32 * n)(*bias.keys()), (ctypes.c_float * n)(*bias.values()), n


def sample(lib, ctx_ptr, temperature, top_p, u, bias):
    ids, vals, n = bias_list(bias)
    tok = ctypes.c_uint32(0)
    assert lib.library.rwkv_b200_sample(ctx_ptr, temperature, top_p, float(u), ids, vals, n, ctypes.byref(tok))
    return int(tok.value)


def eval_token(lib, ctx_ptr, tok):
    assert lib.library.rwkv_b200_eval_resident(ctx_ptr, (ctypes.c_uint32 * 1)(tok), 1, True, None)


def host_generate(lib, ctx_ptr, max_tokens, temperature, top_p, presence, frequency, us, stops=(), counts=None):
    """The loop driven from the host, one rwkv_b200_sample (bias from the counts) + rwkv_b200_eval_resident per token.
    Returns the tokens written; `counts` (a Counter) is updated in place."""
    counts = Counter() if counts is None else counts
    out = []
    for i in range(max_tokens):
        tok = sample(lib, ctx_ptr, temperature, top_p, us[i], penalty_bias(counts, presence, frequency))
        out.append(tok)
        if tok in stops:
            break
        counts[tok] += 1
        eval_token(lib, ctx_ptr, tok)
    return out


def step_flags(max_tokens, step, frozen, drawn, stops):
    """One step's bookkeeping for rows whose draws are `drawn` (None where a row does not draw): (step, frozen, active)."""
    new_step, new_frozen = list(step), list(frozen)
    for b in range(len(step)):
        if frozen[b]:
            continue
        if step[b] == max_tokens[b]:
            new_frozen[b] = 1
            continue
        new_step[b] = step[b] + 1
        if drawn[b] in stops:
            new_frozen[b] = 1
    return new_step, new_frozen, any(not f for f in new_frozen)


class StepArgs(ctypes.Structure):   # include/rwkv_b200.h: struct rwkv_b200_generate_step_args
    _fields_ = [("logits", ctypes.c_void_p), ("n_rows", ctypes.c_size_t), ("n_vocab", ctypes.c_size_t)] + \
               [(n, ctypes.c_void_p) for n in ("max_tokens", "temperature", "top_p", "presence_penalty", "frequency_penalty", "u", "stop_ids")] + \
               [("n_stop", ctypes.c_size_t)] + [(n, ctypes.c_void_p) for n in ("step", "frozen", "counts", "tokens", "next_tokens", "any_active")]
