"""Generates tests/golden/kquant_ref.json and kquant_ref.npz: what the compiled reference (oracle/ref_lib.py) does with Q4_K / Q5_K.

For every preset below, a synthetic FP16 master (tools/synthetic_model.write_master, seed 1) is quantised by the reference to Q4_K and
Q5_K. The JSON keeps the SHA-256 of each output and the presets; the npz keeps the reference's logits after PROMPT_LEN tokens.

Where a tensor's rows are not whole 256-weight super-blocks (rwkv5-small's ffn.value, rwkv6-small's decay LoRA), the reference's
flat quantisation straddles rows and its output cannot be evaluated. This library writes such tensors as Q5_0 (for Q4_K) / Q5_1 (for
Q5_K) instead; the golden for those presets is the splice of two reference runs -- its K-quant bytes for the tensors whose rows are
whole super-blocks, its Q5_0 / Q5_1 bytes for the rest -- and its logits are the reference's on that splice.

    python tests/golden/make_kquant_ref.py
"""
import hashlib
import json
import os
import struct
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

PRESETS = {
    "v4": dict(arch=[4, 0], C=256, F=1024, L=2, V=300, out_scale=0.1),
    "v5.1": dict(arch=[5, 1], C=256, F=1024, L=2, V=300, S=64, out_scale=0.1),
    "v5.2": dict(arch=[5, 2], C=256, F=1024, L=2, V=300, S=64, out_scale=0.1),
    "v6": dict(arch=[6, 0], C=512, F=1792, L=2, V=300, S=64, mix=32, decay=256, out_scale=0.1, lora_fan_in=True),
    "v7": dict(arch=[7, 0], C=512, F=2048, L=2, V=300, S=64, lora_w=64, lora_a=64, lora_v=32, lora_g=128, out_scale=0.1, lora_fan_in=True),
    # fallback cases: rows that are not whole super-blocks
    "rwkv5-small": dict(arch=[5, 2], C=256, F=896, L=2, V=300, S=64, out_scale=0.1),
    "rwkv6-small": dict(arch=[6, 0], C=512, F=1792, L=2, V=300, S=64, mix=32, decay=64, out_scale=0.1, lora_fan_in=True),
}
FALLBACK = {"Q4_K": "Q5_0", "Q5_K": "Q5_1"}
BLOCK = {0: (1, 4), 1: (1, 2), 2: (32, 18), 3: (32, 20), 7: (32, 22), 8: (32, 24), 9: (32, 34), 13: (256, 144), 14: (256, 176)}
TYPE_ID = {"Q4_K": 13, "Q5_K": 14}
SEED = 1
PROMPT_LEN = 40


def prompt(n_vocab):
    return [(7919 * i + 11) % n_vocab for i in range(PROMPT_LEN)]


def read_records(path):
    """(header bytes, [(ne0, record bytes)]) of an rwkv.cpp model file, for any type in BLOCK."""
    buf = open(path, "rb").read()
    recs, off = [], 24
    while off < len(buf):
        dims, klen, dt = struct.unpack_from("<3I", buf, off)
        ne = struct.unpack_from("<%dI" % dims, buf, off + 12)
        blck, size = BLOCK[dt]
        n = size * int(np.prod(ne)) // blck
        end = off + 12 + 4 * dims + klen + n
        recs.append((ne[0], buf[off:end]))
        off = end
    return buf[:24], recs


def splice(kq_path, legacy_path, out_path):
    head, kq = read_records(kq_path)
    _, legacy = read_records(legacy_path)
    with open(out_path, "wb") as f:
        f.write(head)
        for (ne0, a), (_, b) in zip(kq, legacy):
            f.write(a if ne0 % 256 == 0 or a == b else b)


def sha256(path):
    return hashlib.sha256(open(path, "rb").read()).hexdigest()


def main():
    import ctypes
    import ref_lib
    import synthetic_model as sm
    ref = ref_lib.load_reference_library()
    out = {"seed": SEED, "prompt_len": PROMPT_LEN, "presets": PRESETS, "sha256": {}}
    logits = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, p in PRESETS.items():
            master = os.path.join(tmp, name + ".bin")
            sm.write_master(master, dict(p, arch=tuple(p["arch"])), "FP16", seed=SEED)
            for fmt in ("Q4_K", "Q5_K"):
                path = os.path.join(tmp, "%s-%s.bin" % (name, fmt))
                assert ref.rwkv_quantize_model_file(master.encode(), path.encode(), fmt.encode())
                if any(ne0 % 256 for ne0, r in read_records(path)[1] if struct.unpack_from("<3I", r)[2] == TYPE_ID[fmt]):
                    legacy = os.path.join(tmp, "%s-%s.bin" % (name, FALLBACK[fmt]))
                    assert ref.rwkv_quantize_model_file(master.encode(), legacy.encode(), FALLBACK[fmt].encode())
                    spliced = path + ".splice"
                    splice(path, legacy, spliced)
                    path = spliced
                out["sha256"]["%s:%s" % (name, fmt)] = sha256(path)
                ctx = ref.rwkv_init_from_file(path.encode(), 1, 0)
                assert ctx
                n_state, n_logits = ref.rwkv_get_state_len(ctx), ref.rwkv_get_logits_len(ctx)
                state = np.zeros(n_state, np.float32)
                lg = np.zeros(n_logits, np.float32)
                toks = (ctypes.c_uint32 * PROMPT_LEN)(*prompt(p["V"]))
                PF = ctypes.POINTER(ctypes.c_float)
                assert ref.rwkv_eval_sequence(ctx, toks, PROMPT_LEN, None, state.ctypes.data_as(PF), lg.ctypes.data_as(PF))
                ref.rwkv_free(ctx)
                logits["%s:%s" % (name, fmt)] = lg
                print(name, fmt, out["sha256"]["%s:%s" % (name, fmt)][:16], float(np.abs(lg).max()))
    here = os.path.dirname(os.path.abspath(__file__))
    with open(os.path.join(here, "kquant_ref.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    np.savez_compressed(os.path.join(here, "kquant_ref.npz"), **logits)


if __name__ == "__main__":
    main()
