"""The v6 LoRA fold without a GPU: which layer shapes take it (rwkv_b200_v6_lora_fold_supported, the predicate engine.cu routes
single-token passes by) and the argument checks of the two fused kernels' test hooks, which reject bad arguments before they touch
a device."""
import ctypes

import numpy as np
import pytest

import ggml_file as gf

ARGS = 1 << 8
T = gf.TYPE_IDS
VP = ctypes.c_void_p


class V6PrologueArgs(ctypes.Structure):
    _fields_ = [("x", VP), ("ln_w", VP), ("ln_b", VP), ("state_in", VP), ("coef", VP), ("state_out", VP), ("out_xx", VP), ("out_sx", VP),
                ("w1", VP), ("w1_type", ctypes.c_int), ("M1", ctypes.c_int), ("y1", VP), ("C", ctypes.c_int)]


class Wkv6DecayArgs(ctypes.Structure):
    _fields_ = [("r", VP), ("k", VP), ("v", VP), ("tf", VP), ("state_in", VP), ("state_out", VP), ("lnx_w", VP), ("lnx_b", VP), ("g", VP),
                ("y", VP), ("eps", ctypes.c_float), ("H", ctypes.c_int), ("w2", VP), ("w2_type", ctypes.c_int), ("K2", ctypes.c_int),
                ("lora1", VP), ("td_bias", VP), ("q_out", VP), ("q_type", ctypes.c_int)]


@pytest.mark.parametrize("C,S,w1,mix,w2,decay,want", [
    (4096, 64, "Q5_1", 64, "Q5_1", 128, True),     # the 7B decode path
    (4096, 64, "Q4_0", 64, "Q4_0", 128, True),
    (4096, 64, "Q8_0", 64, "Q8_0", 128, False),    # maa_w1 rows of 4352 bytes: the streaming plan splits them over two warps
    (3072, 64, "Q8_0", 64, "Q8_0", 64, True),
    (2048, 64, "FP16", 32, "FP32", 64, False),     # F16 rows of 4096 bytes: two warps
    (1536, 64, "FP16", 32, "FP32", 64, True),
    (512, 64, "FP32", 32, "FP32", 64, True),
    (1024, 64, "FP32", 32, "FP32", 64, False),     # F32 rows of 4096 bytes
    (512, 64, "Q5_1", 32, "FP32", 128, True),
    (512, 64, "Q5_1", 32, "FP32", 256, False),     # decay rank above 128
    (512, 32, "Q5_1", 32, "Q5_1", 64, False),      # head size 32
    (5120, 64, "Q5_1", 64, "Q5_1", 128, False),    # n_embed above 4096
    (4096, 64, "Q5_1", 64, "Q5_1", 48, False),     # decay rank not a whole number of blocks
])
def test_v6_lora_fold_predicate(lib, C, S, w1, mix, w2, decay, want):
    assert lib.library.rwkv_b200_v6_lora_fold_supported(C, S, T[w1], mix, T[w2], decay) is want


def test_v6_fold_hooks_reject_invalid_arguments(lib):
    buf = np.zeros(1 << 20, np.float32)
    p = buf.ctypes.data

    def prologue(**kw):
        a = V6PrologueArgs(x=p, ln_w=p, ln_b=p, state_in=p, coef=p, state_out=p, out_xx=p, out_sx=p, w1=p, w1_type=T["Q5_1"], M1=160, y1=p, C=512)
        for k, v in kw.items():
            setattr(a, k, v)
        return lib.library.rwkv_b200_test_v6_prologue(ctypes.byref(a))

    def wkv(**kw):
        a = Wkv6DecayArgs(r=p, k=p, v=p, tf=p, state_in=p, state_out=p, lnx_w=p, lnx_b=p, y=p, eps=64e-5, H=8, w2=p, w2_type=T["Q5_1"], K2=64,
                          lora1=p, td_bias=p)
        for k, v in kw.items():
            setattr(a, k, v)
        return lib.library.rwkv_b200_test_wkv6_decay(ctypes.byref(a))

    cases = [
        lambda: prologue(x=None),                        # a missing input
        lambda: prologue(y1=None),                       # a missing output
        lambda: prologue(M1=0),                          # no rows
        lambda: prologue(C=5120),                        # n_embed above 4096
        lambda: prologue(C=4096, w1_type=T["Q8_0"]),     # rows the streaming plan splits over two warps
        lambda: prologue(C=2048, w1_type=T["FP32"]),
        lambda: prologue(C=48),                          # not a whole number of blocks
        lambda: prologue(w1_type=5),                     # removed format Q4_2
        lambda: wkv(lora1=None),                         # a missing input
        lambda: wkv(y=None),                             # a missing output
        lambda: wkv(H=0),                                # no head
        lambda: wkv(H=65),                               # n_embed above 4096
        lambda: wkv(K2=256),                             # decay rank above 128
        lambda: wkv(K2=48),                              # not a whole number of blocks
        lambda: wkv(w2_type=5),                          # removed format Q4_2
        lambda: wkv(q_out=p, q_type=5),                  # a staged column for a type without a stage class
    ]
    for i, call in enumerate(cases):
        assert not call(), i
        assert lib.rwkv_get_last_error(None) == ARGS, i
