"""What a LoRA adapter costs (DESIGN.md 6.7). Measurement aid, not a bench line.

Workload: the synthetic RWKV-6 7B shape at Q5_1 (bench.py's rwkv6-7b:Q5_1 file), one sequence. Adapters put a seeded low-rank delta on
every matrix that takes one (att key / value / receptance / gate / output, ffn key / value / receptance of all 32 layers) at rank 8,
16 and 64; the "+vec" adapters also replace every layer's ln1 / ln2 weights and ffn time_maa_k. The legs:
  base        no adapter. A LoRA merged offline into the FP16 master and re-quantized to Q5_1 (the only route without adapters) is a
              file of the base's shapes and types: it runs these launches over these bytes, so this leg stands for it; no merged
              file is built or timed.
  r8 .. r64   the adapter of that rank attached; "+vec" with the replaced vectors
For each leg: decode ms per token (256 single-token passes through rwkv_b200_eval_resident, graphs on, host clock around the passes
and a synchronise) and prefill tokens/s (passes of 128 tokens), alternating the legs over the rounds; the median with min / max.
Launches per step: the records of one single-token pass in the in-kernel timeline (rwkv_b200_trace_*), one per launch, with the
microseconds the lora_shrink / lora_expand launches span, in a run of their own after the timed rounds; and the library's kernel
launch counter across the same kind of pass. The card's name and power limit are read in the same run.

    python tools/lora_bench.py [--rounds 5] [--tokens 256] [--out FILE.json]
"""
import argparse
import ctypes
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import __graft_entry__  # noqa: E402
import bench  # noqa: E402
from ragged_batch_bench import card  # noqa: E402

U32 = ctypes.c_uint32
PREFILL = 128
TARGETS = ("att.key.weight", "att.value.weight", "att.receptance.weight", "att.gate.weight", "att.output.weight",
           "ffn.key.weight", "ffn.value.weight", "ffn.receptance.weight")


def adapter_entries(p, rank, vectors, seed=0):
    """Entries for every delta target of the preset's layers; matrices of one shape share their seeded A and B (the cost does not
    depend on the values)."""
    C, F, L = p["C"], p["F"], p["L"]
    rng = np.random.default_rng(seed)
    shapes = {"ffn.key.weight": (F, C), "ffn.value.weight": (C, F)}
    ab = {}
    out = []
    for i in range(L):
        for t in TARGETS:
            M, K = shapes.get(t, (C, C))
            if (M, K) not in ab:
                ab[(M, K)] = ((rng.standard_normal((rank, K)) * K ** -0.5).astype(np.float32), (rng.standard_normal((M, rank)) * 0.01).astype(np.float32))
            a, b = ab[(M, K)]
            out.append((f"blocks.{i}.{t}", rank, a, b, None))
        if vectors:
            for v in ("ln1.weight", "ln2.weight", "ffn.time_maa_k"):
                out.append((f"blocks.{i}.{v}", 0, None, None, (1.0 + rng.standard_normal(C) * 0.01).astype(np.float32)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--tokens", type=int, default=256)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    pkg = __graft_entry__.load_package()
    lib = pkg.load_rwkv_shared_library()
    L = lib.library
    path, preset = bench.workload_file("rwkv6-7b:Q5_1")
    ctx = lib.rwkv_b200_init_from_file_ex(path, 0, 0, -1)
    V = lib.rwkv_get_logits_buffer_element_count(ctx)
    adapters = {"base": None}
    for rank in (8, 16, 64):
        for vec in (False, True):
            adapters[f"r{rank}" + ("+vec" if vec else "")] = lib.rwkv_b200_adapter_create(ctx, adapter_entries(preset, rank, vec), 1.0)
    toks = [(7919 * i + 11) % V for i in range(max(args.tokens, PREFILL))]
    prefill = (U32 * PREFILL)(*toks[:PREFILL])

    def decode():
        assert L.rwkv_b200_state_load(ctx.ptr, None)
        assert L.rwkv_b200_synchronize(ctx.ptr)
        t0 = time.perf_counter()
        for t in toks[:args.tokens]:
            assert L.rwkv_b200_eval_resident(ctx.ptr, (U32 * 1)(t), 1, True, None)
        assert L.rwkv_b200_synchronize(ctx.ptr)
        return (time.perf_counter() - t0) * 1e3 / args.tokens

    def prefill_rate(n=4):
        assert L.rwkv_b200_state_load(ctx.ptr, None)
        assert L.rwkv_b200_synchronize(ctx.ptr)
        t0 = time.perf_counter()
        for _ in range(n):
            assert L.rwkv_b200_eval_resident(ctx.ptr, prefill, PREFILL, True, None)
        assert L.rwkv_b200_synchronize(ctx.ptr)
        return n * PREFILL / (time.perf_counter() - t0)

    launches, dec, pre = {}, {k: [] for k in adapters}, {k: [] for k in adapters}
    for name, ad in adapters.items():      # warm-up: module loads, capacity growth, graph captures; and the launch count
        lib.rwkv_b200_set_adapter(ctx, ad)
        decode()
        prefill_rate(1)
        before = L.rwkv_b200_kernel_launch_count()
        assert L.rwkv_b200_eval_resident(ctx.ptr, (U32 * 1)(toks[0]), 1, True, None)
        assert L.rwkv_b200_synchronize(ctx.ptr)
        launches[name] = int(L.rwkv_b200_kernel_launch_count() - before)
    for _ in range(args.rounds):
        for name, ad in adapters.items():
            lib.rwkv_b200_set_adapter(ctx, ad)
            decode()                        # re-capture the single-token graphs outside the timed window
            dec[name].append(decode())
            pre[name].append(prefill_rate())
    traced = {}
    n_rec = 1024
    st, en = (ctypes.c_double * n_rec)(), (ctypes.c_double * n_rec)()
    names = ctypes.create_string_buffer(32 * n_rec)
    assert L.rwkv_b200_trace_enable(ctx.ptr)
    for name, ad in adapters.items():
        lib.rwkv_b200_set_adapter(ctx, ad)
        assert L.rwkv_b200_state_load(ctx.ptr, None)
        for t in toks[:4]:                 # eager, capture, replays; each read re-arms the records, so the last is one graph replay
            assert L.rwkv_b200_eval_resident(ctx.ptr, (U32 * 1)(t), 1, True, None)
            n = L.rwkv_b200_trace_read(ctx.ptr, st, en, ctypes.cast(names, ctypes.c_void_p), n_rec)
        kinds = [names.raw[32 * i:32 * i + 32].split(b"\0")[0].decode() for i in range(n)]
        lora_us = sum(en[i] - st[i] for i in range(n) if kinds[i].startswith("lora_"))
        traced[name] = {"records": n, "lora_records": sum(k.startswith("lora_") for k in kinds), "lora_us": round(lora_us, 1),
                        "step_span_us": round(max(en[i] for i in range(n)) - min(st[i] for i in range(n)), 1)}
    L.rwkv_b200_trace_disable(ctx.ptr)
    lib.rwkv_b200_set_adapter(ctx, None)
    for ad in adapters.values():
        if ad:
            lib.rwkv_b200_adapter_free(ad)
    lib.rwkv_free(ctx)

    base = statistics.median(dec["base"])
    res = {"card": card(), "workload": "rwkv6-7b:Q5_1, one sequence", "rounds": args.rounds, "decode_tokens": args.tokens,
           "prefill_tokens_per_pass": PREFILL, "legs": {}}
    for name in adapters:
        d, p = statistics.median(dec[name]), statistics.median(pre[name])
        res["legs"][name] = {"decode_ms_per_token": round(d, 4), "decode_min_max": [round(min(dec[name]), 4), round(max(dec[name]), 4)],
                             "decode_tokens_per_s": round(1e3 / d, 1), "decode_vs_base": round(d / base, 4),
                             "prefill_tokens_per_s": round(p, 1), "prefill_min_max": [round(min(pre[name]), 1), round(max(pre[name]), 1)],
                             "launches_per_step": launches[name], "trace": traced[name]}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
