"""Synthetic RWKV model files in the rwkv.cpp ggml format (SURVEY.md Appendix E).

No checkpoints are reachable offline, so the benchmark and the large-shape parity tests run on
random-init weights of the exact architectures: same tensor names, shapes, per-tensor dtypes and
value ranges as converted checkpoints, loadable by BOTH this engine and the reference library.

Two paths:
  * write_master(...)      FP16/FP32 master file (numpy), then quantise with rwkv_quantize_model_file;
  * write_direct(...)      quant blocks are generated directly (random nibbles, per-block fp16 scales
                           chosen so that weights have std ~ 1/sqrt(fan_in)); this is how the 7B-shape
                           files are made in seconds instead of minutes.
"""
import os
import sys

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(_ROOT, "oracle"))
import ggml_file as gf  # noqa: E402

# name -> (arch_major, arch_minor, C, F, L, V, head_size, extras)
PRESETS = {
    # BASELINE.json configs / north star
    # out_scale: factor on the two matrices that write into the residual stream (att.output, ffn.value). With 1.0 every block adds a
    # vector as large as the stream itself and a 24-32 layer random network is chaotic: the unmodified reference then differs from
    # ITSELF (AVX2 vs AVX-512 build, same file) by 2.1 in the logits of the 2.9B FP16 shape after one token (tools/ref_self_spread.py),
    # so no end-to-end comparison means anything. Trained checkpoints are nothing like that (RWKV initialises both matrices to zero);
    # 0.1 keeps the residual stream embedding-dominated, as in a trained model, and rounding flips stay local.
    # lora_fan_in: LoRA matrices (v6 time_maa / time_decay, v7 w/a/v/g pairs) get std 0.5/sqrt(fan_in) instead of a flat 0.05, which
    # at n_embed = 4096 drives every tanh / sigmoid of the data-dependent mixes into saturation (pre-activations of std 3.2).
    "rwkv4-169m": dict(arch=(4, 0), C=768, F=3072, L=12, V=50277, out_scale=0.1),
    "rwkv5-1b5": dict(arch=(5, 2), C=2048, F=7168, L=24, V=65536, S=64, out_scale=0.1),
    "rwkv6-7b": dict(arch=(6, 0), C=4096, F=14336, L=32, V=65536, S=64, mix=64, decay=128, out_scale=0.1, lora_fan_in=True),
    "rwkv7-2b9": dict(arch=(7, 0), C=2560, F=10240, L=32, V=65536, S=64, lora_w=96, lora_a=96, lora_v=64, lora_g=320, out_scale=0.1, lora_fan_in=True),
    # small shapes for parity tests (head size 64 like real models)
    "rwkv4-small": dict(arch=(4, 0), C=256, F=1024, L=3, V=1000, out_scale=0.1),
    "rwkv5.1-small": dict(arch=(5, 1), C=256, F=896, L=3, V=1000, S=64, out_scale=0.1),
    "rwkv5-small": dict(arch=(5, 2), C=256, F=896, L=3, V=1000, S=64, out_scale=0.1),
    "rwkv6-small": dict(arch=(6, 0), C=512, F=1792, L=4, V=2000, S=64, mix=32, decay=64, out_scale=0.1, lora_fan_in=True),
    "rwkv6-mid": dict(arch=(6, 0), C=2048, F=7168, L=2, V=4000, S=64, mix=32, decay=64, out_scale=0.1, lora_fan_in=True),      # ffn rows split over 2 warps
    "rwkv6-wide": dict(arch=(6, 0), C=4096, F=14336, L=1, V=2000, S=64, mix=64, decay=128, out_scale=0.1, lora_fan_in=True),   # one layer of the 7B shape
    "rwkv7-small": dict(arch=(7, 0), C=512, F=2048, L=4, V=2000, S=64, lora_w=64, lora_a=64, lora_v=32, lora_g=128, out_scale=0.1, lora_fan_in=True),
}


def _f16(a):
    return np.ascontiguousarray(a, dtype=np.float32).astype(np.float16)


def _vec(a):
    return gf.TYPE_FP32, np.ascontiguousarray(a, dtype=np.float32)


class _Spec:
    """Walks the tensor table of one architecture and yields (name, kind, ggml_ne, generator-args)."""

    def __init__(self, p):
        self.p = p
        self.major, self.minor = p["arch"]

    def tensors(self):
        p = self.p
        C, F, L, V = p["C"], p["F"], p["L"], p["V"]
        S = p.get("S", 0)
        H = C // S if S else 0
        yield "emb.weight", "emb", (C, V), None
        yield "blocks.0.ln0.weight", "ln_w", (C,), None
        yield "blocks.0.ln0.bias", "ln_b", (C,), None
        for i in range(L):
            b = "blocks.%d." % i
            for ln in ("ln1", "ln2"):
                yield b + ln + ".weight", "ln_w", (C,), None
                yield b + ln + ".bias", "ln_b", (C,), None
            if self.major == 4:
                for n in ("k", "v", "r"):
                    yield b + "att.time_mix_" + n, "u01", (C,), None
                yield b + "att.time_first", "n03", (C,), None
                yield b + "att.time_decay", "v4decay", (C,), None
                for n in ("key", "value", "receptance", "output"):
                    yield b + "att.%s.weight" % n, "mat", (C, C), None
            elif self.major == 5:
                names = ("k", "v", "r") + (("g",) if self.minor >= 2 else ())
                for n in names:
                    yield b + "att.time_mix_" + n, "u01", (C,), None
                if self.minor >= 2:
                    yield b + "att.time_faaaa", "n01", (1, S, H), None
                    yield b + "att.time_decay", "v5decay", (1, S, H), None
                else:
                    yield b + "att.time_first", "v51first", (1, 1, H), None
                    yield b + "att.time_decay", "v5decay", (1, 1, H), None
                mats = ("key", "value", "receptance", "output") + (("gate",) if self.minor >= 2 else ())
                for n in mats:
                    yield b + "att.%s.weight" % n, "mat", (C, C), None
                yield b + "att.ln_x.weight", "ln_w", (C,), None
                yield b + "att.ln_x.bias", "ln_b", (C,), None
            elif self.major == 6:
                mix, dec = p["mix"], p["decay"]
                for n in ("x", "w", "k", "v", "r", "g"):
                    yield b + "att.time_maa_" + n, "u01", (C,), None
                yield b + "att.time_maa_w1", "lora", (C, 5 * mix), None
                yield b + "att.time_maa_w2", "lora_f32", (mix, C, 5), None
                yield b + "att.time_decay", "v6decay", (1, S, H), None
                yield b + "att.time_decay_w1", "lora", (C, dec), None
                yield b + "att.time_decay_w2", "lora", (dec, C), None
                yield b + "att.time_faaaa", "n01", (1, S, H), None
                for n in ("receptance", "key", "value", "output", "gate"):
                    yield b + "att.%s.weight" % n, "mat", (C, C), None
                yield b + "att.ln_x.weight", "ln_w", (C,), None
                yield b + "att.ln_x.bias", "ln_b", (C,), None
            else:
                yield b + "att.x_rwkvag", "u01", (C, 1, 6), None
                for n, r in (("w", p["lora_w"]), ("a", p["lora_a"]), ("v", p["lora_v"]), ("g", p["lora_g"])):
                    if n == "v" and i == 0:
                        continue
                    yield b + "att.%s1" % n, "lora_keep", (C, r), None
                    yield b + "att.%s2" % n, "lora_keep", (r, C), None
                    if n != "g":
                        yield b + "att.%s0" % n, "n01", (C, 1, 1), None
                yield b + "att.k_k", "u01", (C, 1, 1), None
                yield b + "att.k_a", "u01", (C, 1, 1), None
                yield b + "att.r_k", "n01", (S, H), None
                for n in ("receptance", "key", "value", "output"):
                    yield b + "att.%s.weight" % n, "mat", (C, C), None
                yield b + "att.ln_x.weight", "ln_w", (C,), None
                yield b + "att.ln_x.bias", "ln_b", (C,), None
            # channel mixing
            if self.major == 7:
                yield b + "ffn.x_k", "u01", (C, 1, 1), None
            elif self.major == 6:
                yield b + "ffn.time_maa_k", "u01", (C,), None
                yield b + "ffn.time_maa_r", "u01", (C,), None
            else:
                yield b + "ffn.time_mix_k", "u01", (C,), None
                yield b + "ffn.time_mix_r", "u01", (C,), None
            yield b + "ffn.key.weight", "mat", (C, F), None
            yield b + "ffn.value.weight", "mat", (F, C), None
            if self.major != 7:
                yield b + "ffn.receptance.weight", "mat", (C, C), None
        yield "ln_out.weight", "ln_w", (C,), None
        yield "ln_out.bias", "ln_b", (C,), None
        yield "head.weight", "head", (C, V), None


def _small_values(kind, ne, rng):
    n = int(np.prod(ne))
    if kind == "ln_w":
        return 1.0 + 0.1 * rng.standard_normal(n)
    if kind == "ln_b":
        return 0.1 * rng.standard_normal(n)
    if kind == "u01":
        return rng.uniform(0.0, 1.0, n)
    if kind == "n01":
        return 0.1 * rng.standard_normal(n)
    if kind == "n03":
        return 0.3 * rng.standard_normal(n)
    if kind == "v4decay":
        return -np.exp(rng.uniform(-5.0, 1.0, n))
    if kind == "v5decay":
        return np.exp(-np.exp(rng.uniform(-6.0, -1.0, n)))
    if kind == "v51first":
        return np.exp(0.3 * rng.standard_normal(n))
    if kind == "v6decay":
        return rng.uniform(-6.0, -1.0, n)
    raise ValueError(kind)


def _mat_std(p, name, ne):
    """std of a 2-D weight: 1/sqrt(fan_in), damped by the preset's out_scale for the matrices that write into the residual stream."""
    s = 1.0 / np.sqrt(ne[0])
    if name.endswith(("att.output.weight", "ffn.value.weight")):
        s *= p.get("out_scale", 1.0)
    return s


def _lora_std(p, ne):
    return 0.5 / np.sqrt(ne[0]) if p.get("lora_fan_in") else 0.05


def _dense(ne, rng, scale):
    """[M, K] float32 (ggml ne = (K, M))."""
    K, M = ne[0], int(np.prod(ne[1:]))
    return (rng.standard_normal((M, K), dtype=np.float32) * np.float32(scale))


def write_master(path, preset, dtype="FP16", seed=0):
    """FP16 (or FP32) master file; 2-D weights N(0,1)/sqrt(fan_in), LoRA 0.01*N, emb 0.1*N."""
    p = PRESETS[preset] if isinstance(preset, str) else preset
    rng = np.random.default_rng(seed)
    wide = gf.TYPE_FP16 if dtype == "FP16" else gf.TYPE_FP32
    conv = _f16 if dtype == "FP16" else (lambda a: np.ascontiguousarray(a, dtype=np.float32))

    def gen():
        for name, kind, ne, _ in _Spec(p).tensors():
            if kind in ("mat", "head"):
                yield name, wide, ne, conv(_dense(ne, rng, _mat_std(p, name, ne)))
            elif kind == "emb":
                yield name, wide, ne, conv(_dense(ne, rng, 0.1))
            elif kind in ("lora", "lora_keep"):
                # v6 LoRA matrices keep FP32 even in FP16 files (names contain `.time_`); v7's become FP16
                t = gf.TYPE_FP32 if (kind == "lora" or dtype != "FP16") else gf.TYPE_FP16
                a = _dense(ne, rng, _lora_std(p, ne))
                yield name, t, ne, (a if t == gf.TYPE_FP32 else _f16(a))
            elif kind == "lora_f32":
                yield name, gf.TYPE_FP32, ne, (_lora_std(p, ne) * rng.standard_normal(int(np.prod(ne)))).astype(np.float32)
            else:
                t, a = _vec(_small_values(kind, ne, rng))
                yield name, t, ne, a

    gf.write_model_file(path, p["V"], p["C"], p["L"], wide, gen(), version=101)
    return p


_QINFO = {  # fmt -> (type id, block bytes, offset of qs, qs bytes, has_qh, has_min, integer std)
    "Q4_0": (gf.TYPE_Q4_0, 18, 2, 16, False, False, 4.61), "Q4_1": (gf.TYPE_Q4_1, 20, 4, 16, False, True, 4.61),
    "Q5_0": (gf.TYPE_Q5_0, 22, 6, 16, True, False, 9.23), "Q5_1": (gf.TYPE_Q5_1, 24, 8, 16, True, True, 9.23),
    "Q8_0": (gf.TYPE_Q8_0, 34, 2, 32, False, False, 73.6),
}


# Q4_K / Q5_K super-blocks: random levels and 6-bit scales / mins; d, dmin fp16 chosen so weights have std ~ target_std.
_KQINFO = {"Q4_K": (13, 144, 15), "Q5_K": (14, 176, 31)}


def _write_kquant_file(path, n_vocab, n_embed, n_layer, data_type, tensors):
    """The file layout of ggml_file.write_model_file, for files that hold Q4_K / Q5_K records (ggml_file reads the legacy formats only)."""
    import struct
    per_elem = {t: bb / 256 for t, bb, _ in _KQINFO.values()}
    with open(path, "wb") as f:
        f.write(struct.pack("<6I", gf.RWKV_FILE_MAGIC, 101, n_vocab, n_embed, n_layer, data_type))
        for name, dtype, ne, raw in tensors:
            key = name.encode("utf-8")
            f.write(struct.pack("<3I", len(ne), len(key), dtype))
            f.write(struct.pack("<%dI" % len(ne), *ne))
            f.write(key)
            raw = np.ascontiguousarray(raw).view(np.uint8).reshape(-1)
            want = int(np.prod(ne) * per_elem[dtype]) if dtype in per_elem else gf.tensor_nbytes(dtype, ne)
            assert raw.size == want, (name, raw.size, want)
            f.write(raw.tobytes())


def _random_kquant(fmt, ne, rng, target_std):
    """The quantizer's per-tensor rule: rows that are not whole 256-weight super-blocks fall back to Q5_0 (Q4_K) / Q5_1 (Q5_K)."""
    K, M = ne[0], int(np.prod(ne[1:]))
    if K % 256:
        return _random_blocks("Q5_0" if fmt == "Q4_K" else "Q5_1", ne, rng, target_std)
    tid, bb, lev = _KQINFO[fmt]
    nb = M * (K // 256)
    b = rng.integers(0, 256, size=(nb, bb), dtype=np.uint8)
    # level std ~ lev/sqrt(12), mean scale ~ 32: d*32*lev/sqrt(12) ~ 2 target_std; the min removes the mean
    d = (2.0 * target_std * np.sqrt(12) / (32 * lev) * rng.uniform(0.8, 1.2, nb)).astype(np.float16)
    dmin = (target_std * rng.uniform(0.8, 1.2, nb) / 32).astype(np.float16)
    b[:, 0:2] = d.view(np.uint8).reshape(nb, 2)
    b[:, 2:4] = dmin.view(np.uint8).reshape(nb, 2)
    return tid, b.reshape(-1)


def _random_blocks(fmt, ne, rng, target_std):
    if fmt in _KQINFO:
        return _random_kquant(fmt, ne, rng, target_std)
    tid, bb, qoff, qbytes, has_qh, has_min, istd = _QINFO[fmt]
    K, M = ne[0], int(np.prod(ne[1:]))
    nb = M * (K // 32)
    blocks = rng.integers(0, 256, size=(nb, bb), dtype=np.uint8)
    d = (target_std / istd) * rng.uniform(0.6, 1.4, nb).astype(np.float32)
    blocks[:, 0:2] = d.astype(np.float16).view(np.uint8).reshape(nb, 2)
    if has_min:
        centre = 7.5 if fmt == "Q4_1" else 15.5
        m = (-centre * d * rng.uniform(0.9, 1.1, nb)).astype(np.float32)
        blocks[:, 2:4] = m.astype(np.float16).view(np.uint8).reshape(nb, 2)
    if fmt == "Q8_0":  # avoid -128, which quantize_row_q8_0 never emits
        q = blocks[:, 2:34].view(np.int8)
        q[q == -128] = -127
    return tid, blocks.reshape(-1)


def write_direct(path, preset, fmt, seed=0):
    """Quantised file generated block-by-block (no FP16 master, no quantiser pass). Which tensors are quantised
    follows rwkv_quantize.inc:1-13,133-140: 2-D, not emb/head, not the v7 LoRA / r_k tensors."""
    p = PRESETS[preset] if isinstance(preset, str) else preset
    rng = np.random.default_rng(seed)
    quant = fmt in _QINFO or fmt in _KQINFO

    def gen():
        for name, kind, ne, _ in _Spec(p).tensors():
            if kind == "mat":
                if quant:
                    t, raw = _random_blocks(fmt, ne, rng, _mat_std(p, name, ne))
                    yield name, t, ne, raw
                else:
                    a = _dense(ne, rng, _mat_std(p, name, ne))
                    yield name, (gf.TYPE_FP16 if fmt == "FP16" else gf.TYPE_FP32), ne, (_f16(a) if fmt == "FP16" else a)
            elif kind == "lora":
                if quant:
                    t, raw = _random_blocks(fmt, ne, rng, _lora_std(p, ne))
                    yield name, t, ne, raw
                else:
                    yield name, gf.TYPE_FP32, ne, _dense(ne, rng, _lora_std(p, ne))
            elif kind == "lora_keep":
                a = _dense(ne, rng, _lora_std(p, ne))
                yield name, (gf.TYPE_FP32 if fmt == "FP32" else gf.TYPE_FP16), ne, (a if fmt == "FP32" else _f16(a))
            elif kind == "lora_f32":
                yield name, gf.TYPE_FP32, ne, (_lora_std(p, ne) * rng.standard_normal(int(np.prod(ne)))).astype(np.float32)
            elif kind in ("emb", "head"):
                a = _dense(ne, rng, 0.1 if kind == "emb" else 1.0 / np.sqrt(ne[0]))
                yield name, (gf.TYPE_FP32 if fmt == "FP32" else gf.TYPE_FP16), ne, (a if fmt == "FP32" else _f16(a))
            else:
                t, a = _vec(_small_values(kind, ne, rng))
                yield name, t, ne, a

    if fmt in _KQINFO:
        _write_kquant_file(path, p["V"], p["C"], p["L"], _KQINFO[fmt][0], gen())
    else:
        gf.write_model_file(path, p["V"], p["C"], p["L"], gf.TYPE_IDS[fmt], gen(), version=101)
    return p


def synthetic_tokens(n, n_vocab):
    """Deterministic token stream used by every benchmark leg: t_i = (7919*i) mod V (BASELINE.md section 4)."""
    return [(7919 * i) % n_vocab for i in range(n)]


if __name__ == "__main__":
    import argparse
    import time
    ap = argparse.ArgumentParser()
    ap.add_argument("preset")
    ap.add_argument("fmt")
    ap.add_argument("out")
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    t0 = time.time()
    write_direct(a.out, a.preset, a.fmt, a.seed)
    print("wrote %s (%.1f MB) in %.1fs" % (a.out, os.path.getsize(a.out) / 1e6, time.time() - t0))
