"""Single-token passes of a v6 context fold two LoRA matrices into their neighbouring launches (engine.cu v6_lora_fold): maa_w1 into
the LayerNorm-mix launch (glue.cu v6_prologue_kernel) and decay_w2 into the WKV launch (wkv.cu wkv6_kernel<64, false, DW2>). Passes of
more than one token and batch contexts keep the separate GEMV launches, so a model evaluated token by token must give the same bits as
the same tokens in chunks of < 32 tokens and as the same sequence inside a batch context."""
import ctypes
import sys
import os

import numpy as np
import pytest

from test_gpu_batch import check_batch

pytestmark = pytest.mark.gpu
P_F, P_U = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_uint32)
FORMATS = ["FP32", "FP16", "Q4_0", "Q4_1", "Q5_0", "Q5_1", "Q8_0"]
N_TOKENS = 12


def traced_names(lib, ctx, tok):
    L = lib.library
    N = 1024
    st, en = (ctypes.c_double * N)(), (ctypes.c_double * N)()
    names = ctypes.create_string_buffer(32 * N)
    assert L.rwkv_b200_trace_enable(ctx.ptr)
    arr = (ctypes.c_uint32 * 1)(tok)
    assert L.rwkv_b200_eval_resident(ctx.ptr, arr, 1, True, None)
    n = L.rwkv_b200_trace_read(ctx.ptr, st, en, ctypes.cast(names, ctypes.c_void_p), N)
    L.rwkv_b200_trace_disable(ctx.ptr)
    return [names.raw[32 * i:32 * i + 32].split(b"\0")[0].decode() for i in range(n)]


@pytest.mark.parametrize("preset", ["rwkv6-small", "rwkv6-mid", "rwkv6-wide"])
@pytest.mark.parametrize("fmt", FORMATS)
def test_v6_fold_serial_equals_chunks_and_batch(lib, tmp_path, preset, fmt):
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    import synthetic_model as sm
    path = str(tmp_path / f"{preset}-{fmt}.bin")
    sm.write_direct(path, preset, fmt, seed=5)
    ctx = lib.rwkv_init_from_file(path, 1, 0)
    try:
        L = lib.library
        n_state, n_logits = lib.rwkv_get_state_buffer_element_count(ctx), lib.rwkv_get_logits_buffer_element_count(ctx)
        toks = [(7 * i + 3) % n_logits for i in range(N_TOKENS)]
        state = np.zeros(n_state, np.float32)
        logits = np.zeros(n_logits, np.float32)
        for i, t in enumerate(toks):
            assert L.rwkv_eval(ctx.ptr, t, None if i == 0 else state.ctypes.data_as(P_F), state.ctypes.data_as(P_F), logits.ctypes.data_as(P_F))
        arr = (ctypes.c_uint32 * N_TOKENS)(*toks)
        for chunk in (2, 8, 31):
            st2, lg2 = np.zeros(n_state, np.float32), np.zeros(n_logits, np.float32)
            assert L.rwkv_eval_sequence_in_chunks(ctx.ptr, arr, N_TOKENS, chunk, None, st2.ctypes.data_as(P_F), lg2.ctypes.data_as(P_F))
            assert st2.tobytes() == state.tobytes(), (preset, fmt, chunk, np.abs(st2 - state).max())
            assert lg2.tobytes() == logits.tobytes(), (preset, fmt, chunk, np.abs(lg2 - logits).max())
        # the single-token path takes the fold wherever the streaming GEMV gives maa_w1 one warp per row (row pitch <= 3.5 KB): one
        # v6_prologue launch per layer and no separate ln_mix for the time mixing; elsewhere the separate launches
        names = traced_names(lib, ctx, toks[0])
        n_layer, C = sm.PRESETS[preset]["L"], sm.PRESETS[preset]["C"]
        folded = not ((C >= 2048 and fmt in ("FP16", "FP32")) or (C >= 4096 and fmt == "Q8_0"))
        assert names.count("v6_prologue") == (n_layer if folded else 0), names
        assert names.count("ln_mix") == (n_layer if folded else 2 * n_layer), names
    finally:
        lib.rwkv_free(ctx)
    for n_seq in (1, 5):
        check_batch(lib, path, n_seq=n_seq, n_steps=5)


# ---- each fused kernel against the two launches it replaces, through the kernel test hooks ------------------------------------
import re
import subprocess

import ggml_file as gf
import kernel_hooks as kh
from test_gpu_gemv import random_raw
from test_v6_fold_host import V6PrologueArgs, Wkv6DecayArgs

LAUNCHED = set()      # ("prologue", PER, type) / ("wkv6_decay", type) reached by the tests below
SIZES = [512, 1536, 2048, 3072, 4096]     # PER 1 / 2 / 2 / 4 / 4 of ln_mix_body; 1536 and 3072 reach F16 at PER 2 and Q8_0 at PER 4


def per_of(C):
    per = (C + 1023) // 1024
    return 1 if per <= 1 else 2 if per <= 2 else 4


def vec(rng, *shape, scale=1.0):
    return (rng.standard_normal(shape) * scale).astype(np.float32)


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("C", SIZES)
@pytest.mark.parametrize("mix", [32, 64])
def test_v6_prologue_equals_ln_mix_then_gemv(lib, fmt, C, mix):
    tid = gf.TYPE_IDS[fmt]
    M1 = 5 * mix
    if not lib.library.rwkv_b200_v6_lora_fold_supported(C, 64, tid, mix, gf.TYPE_IDS["Q5_1"], 64):
        pytest.skip("this shape keeps the separate launches")
    rng = np.random.default_rng(C * 7 + mix + tid)
    x, lw, lb, st, coef = vec(rng, C, 1, scale=3.0), 1 + vec(rng, C, scale=0.1), vec(rng, C, scale=0.1), vec(rng, C), rng.uniform(0, 1, C).astype(np.float32)
    _, raw = random_raw(fmt, M1, C)
    ref = kh.ln_mix(lib, x, lw, lb, st, [coef], 1)
    (y_ref,), _ = kh.gemv_batch(lib, 1, [dict(type=tid, K=C, M=M1, raw=raw, epi=3)], [ref["out0"].cols(C)])
    i = kh.Inputs()
    o = {k: kh.Out(n) for k, n in (("state", C), ("xx", C), ("sx", C), ("y1", M1))}
    a = V6PrologueArgs(x=i(x[:, 0]), ln_w=i(lw), ln_b=i(lb), state_in=i(st), coef=i(coef), state_out=o["state"].ptr, out_xx=o["xx"].ptr,
                       out_sx=o["sx"].ptr, w1=i.keep.append(raw) or raw.ctypes.data, w1_type=tid, M1=M1, y1=o["y1"].ptr, C=C)
    kh._call(lib, lib.library.rwkv_b200_test_v6_prologue, a)
    for k, r in (("state", ref["state"]), ("xx", ref["xx"]), ("sx", ref["sx"]), ("y1", y_ref)):
        assert o[k].guard_intact(), k
        assert o[k].value.tobytes() == r.value.tobytes(), (k, np.abs(o[k].value - r.value).max())
    LAUNCHED.add(("prologue", per_of(C), tid))


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("C", SIZES)
@pytest.mark.parametrize("decay", [64, 128])
def test_wkv6_decay_equals_gemv_then_wkv6(lib, fmt, C, decay):
    tid = gf.TYPE_IDS[fmt]
    assert lib.library.rwkv_b200_v6_lora_fold_supported(512, 64, gf.TYPE_IDS["Q5_1"], 32, tid, decay)
    rng = np.random.default_rng(C * 3 + decay + tid)
    H = C // 64
    r, k, v, g = vec(rng, C, 1), vec(rng, C, 1), vec(rng, C, 1), vec(rng, C, 1)
    tf, lw, lb, st = vec(rng, C, scale=0.3), 1 + vec(rng, C, scale=0.1), vec(rng, C, scale=0.1), vec(rng, C * 64)
    lora1, td_bias = np.tanh(vec(rng, decay, 1)), vec(rng, C, scale=0.5) - 1.0
    _, raw = random_raw(fmt, C, decay)
    (w,), _ = kh.gemv_batch(lib, 1, [dict(type=tid, K=decay, M=C, raw=raw, epi=7, bias=td_bias)], [lora1])
    ref = kh.wkv6(lib, r, k, v, w.cols(C), tf, st, lw, lb, g, 64e-5, H, 64, True, False)
    i = kh.Inputs()
    o = {"state": kh.Out(st.size), "y": kh.Out(C)}
    i.keep.append(raw)
    a = Wkv6DecayArgs(r=i(r[:, 0]), k=i(k[:, 0]), v=i(v[:, 0]), tf=i(tf), state_in=i(st), state_out=o["state"].ptr, lnx_w=i(lw), lnx_b=i(lb),
                      g=i(g[:, 0]), y=o["y"].ptr, eps=64e-5, H=H, w2=raw.ctypes.data, w2_type=tid, K2=decay, lora1=i(lora1[:, 0]), td_bias=i(td_bias))
    kh._call(lib, lib.library.rwkv_b200_test_wkv6_decay, a)
    for key in ("state", "y"):
        assert o[key].guard_intact(), key
        assert o[key].value.tobytes() == ref[key].value.tobytes(), (key, np.abs(o[key].value - ref[key].value).max())
    LAUNCHED.add(("wkv6_decay", tid))


def test_every_fused_instantiation_was_launched(lib):
    """Runs after the tests above: every v6_prologue_kernel<PER, TYPE> and wkv6_kernel<64, false, DW2> in the library was reached."""
    r = subprocess.run(["cuobjdump", "--dump-resource-usage", lib.path], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    compiled = set()
    for name in re.findall(r"Function ([^:\s]+):", r.stdout):
        if m := re.search(r"v6_prologue_kernelILi(\d+)ELi(\d+)EE", name):
            compiled.add(("prologue", int(m[1]), int(m[2])))
        elif m := re.search(r"wkv6_kernelILi64ELb0ELi(\d+)EE", name):
            compiled.add(("wkv6_decay", int(m[1])))
    assert len(compiled) == 18 + 7, sorted(compiled)
    assert compiled <= LAUNCHED, sorted(compiled - LAUNCHED)
