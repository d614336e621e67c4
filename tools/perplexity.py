"""Perplexity of a model on a token stream, scored on the GPU.

    python tools/perplexity.py MODEL.bin TOKENS ignore_first_n_tokens [token_limit]

The loop of the reference's python/measure_pexplexity.py (the same arguments, the same loss and perplexity lines), but every window of
256 tokens is one rwkv_b200_score call: the log-probabilities of the next tokens are computed on the device, and no logits cross PCIe.
Tokenizers are out of scope here: TOKENS is a file of token ids, whitespace- or comma-separated text, or a .npy array.
Loss is the cross entropy of tokens[i + 1] after tokens[0 .. i]; perplexity is exp of the average loss over the positions i with
i + 1 >= ignore_first_n_tokens (all of them when it is 0).
"""
import argparse
import ctypes
import math
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WINDOW = 256
P_F, P_U = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_uint32)


def read_tokens(path):
    if path.endswith(".npy"):
        return [int(t) for t in np.load(path).reshape(-1)]
    return [int(t) for t in open(path).read().replace(",", " ").split()]


def score_losses(lib, ctx, tokens, window=WINDOW, on_window=None):
    """Loss of tokens[i + 1] after tokens[0 .. i] for i < len(tokens) - 1, from a fresh state, in windows of `window` tokens. A window's
    last target is the first token of the next window."""
    L = lib.library
    run = len(tokens) - 1
    losses = np.empty(run, np.float64)
    if not L.rwkv_b200_state_load(ctx.ptr, None):
        raise ValueError("rwkv_b200_state_load failed")
    for off in range(0, run, window):
        n = min(window, run - off)
        toks = np.ascontiguousarray(tokens[off:off + n], np.uint32)
        targets = np.ascontiguousarray(tokens[off + 1:off + n + 1], np.uint32)
        lp = np.empty(n, np.float32)
        if not L.rwkv_b200_score(ctx.ptr, toks.ctypes.data_as(P_U), targets.ctypes.data_as(P_U), n, lp.ctypes.data_as(P_F), None):
            raise ValueError(f"rwkv_b200_score failed (error flags 0x{L.rwkv_get_last_error(ctx.ptr):x})")
        losses[off:off + n] = -lp.astype(np.float64)
        if on_window:
            on_window(off + n, losses[:off + n])
    return losses


def counted(n, ignore_first_n):
    return [i for i in range(n) if ignore_first_n == 0 or i + 1 >= ignore_first_n]


def average(losses, ignore_first_n):
    """(average loss, perplexity) over the counted positions, as measure_pexplexity.py counts them."""
    keep = counted(len(losses), ignore_first_n)
    loss = float(np.mean(losses[keep]))
    return loss, math.exp(loss)


def format_loss_with_perplexity(loss, ppl):
    return f"loss [{loss:.3f}], perplexity {ppl:.3f}"


def main():
    ap = argparse.ArgumentParser(description="Measure perplexity of an RWKV model on a file of token ids")
    ap.add_argument("model_path")
    ap.add_argument("tokens_path")
    ap.add_argument("ignore_first_n_tokens", type=int)
    ap.add_argument("token_limit", nargs="?", type=int, default=-1)
    args = ap.parse_args()

    sys.path.insert(0, ROOT)
    import __graft_entry__
    lib = __graft_entry__.load_package().load_rwkv_shared_library()
    print("Loading model")
    ctx = lib.rwkv_init_from_file(args.model_path, 1, 0)
    print("Loading tokens")
    tokens = read_tokens(args.tokens_path)
    token_count = len(tokens)
    print(f"{token_count} tokens in the text")
    if not (args.token_limit == -1 or args.token_limit > 0):
        raise ValueError("Invalid token_limit")
    if args.token_limit != -1 and token_count > args.token_limit:
        tokens, token_count = tokens[:args.token_limit], args.token_limit
        print(f"Text was limited to {args.token_limit} tokens")
    if not (token_count - args.ignore_first_n_tokens > 1):
        raise ValueError("Need at least 2 tokens for evaluation")
    run_count = token_count - 1
    start = time.time()

    def progress(done, so_far):
        keep = counted(done, args.ignore_first_n_tokens)
        duration = time.time() - start
        remaining = int((run_count - done) * duration / done)
        line = f"Token #{done - 1}/{token_count}, {int(100.0 * (done - 1) / token_count)}%, ETA {remaining // 60} m {remaining % 60} s"
        if keep:
            line += ", averages so far: " + format_loss_with_perplexity(*average(so_far, args.ignore_first_n_tokens))
        print(line)

    losses = score_losses(lib, ctx, tokens, on_window=progress)
    loss, ppl = average(losses, args.ignore_first_n_tokens)
    elapsed = time.time() - start
    lib.rwkv_free(ctx)
    print()
    print(f"Model: {os.path.basename(args.model_path)}, data: {os.path.basename(args.tokens_path)} with {token_count} tokens, "
          f"skipped {args.ignore_first_n_tokens} tokens, averages: {format_loss_with_perplexity(loss, ppl)}, "
          f"latency {elapsed * 1000 / run_count:.3f} ms per token")


if __name__ == "__main__":
    main()
