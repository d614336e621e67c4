"""LoRA adapters without a GPU: lora.py's mapping of RWKV-LM-LoRA / RWKV-PEFT checkpoint keys to model tensors and its converter
rewrites, the C structure's layout, the argument checks that refuse before any device call, and the float64 restatement the GPU
tests hold the kernels to."""
import ctypes
import os

import numpy as np
import pytest

import lora_ref as lr
from ggml_file import read_model_file

ERR_ARGS = 1 << 8
KINDS = ["v4", "v5.1", "v5.2", "v6", "v7"]


@pytest.fixture(scope="module")
def lora(pkg):
    from rwkv_cpp_b200 import lora
    return lora


def entries_by_name(entries):
    return {e[0]: e for e in entries}


@pytest.mark.parametrize("kind", KINDS)
def test_checkpoint_entries_place_every_key(lora, kind):
    import synthetic_checkpoint as sc
    sd = sc.make_lora_state_dict(kind, rank=4, seed=2)
    arch = sc.SHAPES[kind]["arch"]
    entries, scale = lora.checkpoint_entries(sd, arch, lora_alpha=8, scale=0.5)
    assert scale == 8 / 4 * 0.5
    got = entries_by_name(entries)
    for key, t in sd.items():
        name, part = lora._lora_part(key)
        if name:
            e = got[name]
            assert e[1] == 4 and e[4] is None
            want = e[2] if part == "lora_A" else e[3]
            assert np.array_equal(want, t.numpy())
        elif ".att.x_" in key:
            assert f"blocks.{key.split('.')[1]}.att.x_rwkvag" in got
        else:
            assert got[key][1] == 0 and got[key][2] is None
    # every delta lands on a matrix that takes one, under its file name
    for name, rank, *_ in entries:
        if rank:
            assert lr.is_delta_target(name), name


@pytest.mark.parametrize("kind", KINDS)
def test_replacements_take_the_converters_rewrites(lora, tmp_path, kind):
    """A replaced parameter reaches the library as the converter writes it: convert the base with the replacements in place and
    compare every replaced tensor's file values with the entry."""
    import synthetic_checkpoint as sc
    from rwkv_cpp_b200 import convert_pytorch_to_ggml as conv
    base = sc.make_state_dict(kind, seed=0)
    sd = sc.make_lora_state_dict(kind, rank=4, seed=3)
    entries, _ = lora.checkpoint_entries(sd, sc.SHAPES[kind]["arch"], lora_alpha=4)
    full = dict(base)
    for k, t in sd.items():
        if lora._lora_part(k)[0] is None:
            full[k] = t
    path = str(tmp_path / "m.bin")
    conv.write_state_dict(full, path, "FP32")
    tensors = read_model_file(path).tensors
    n = 0
    for name, rank, a, b, values in entries:
        if rank == 0:
            want = lr.tensor_f32(tensors[name])
            assert values.dtype == np.float32 and values.tobytes() == want.tobytes(), name
            n += 1
    assert n > 0


def test_checkpoint_errors(lora):
    import torch
    a, b = torch.zeros(4, 8), torch.zeros(16, 4)
    with pytest.raises(ValueError, match="must both be present"):
        lora.checkpoint_entries({"blocks.0.att.key.lora_A": a}, (4, 0), 8)
    with pytest.raises(ValueError, match="low-rank pair"):
        lora.checkpoint_entries({"blocks.0.att.key.lora_A": a, "blocks.0.att.key.lora_B": torch.zeros(16, 3)}, (4, 0), 8)
    with pytest.raises(ValueError, match="different ranks"):
        lora.checkpoint_entries({"blocks.0.att.key.lora_A": a, "blocks.0.att.key.lora_B": b,
                                 "blocks.0.ffn.key.lora_A.weight": torch.zeros(2, 8), "blocks.0.ffn.key.lora_B.weight": torch.zeros(16, 2)}, (4, 0), 8)
    with pytest.raises(ValueError, match="x_rwkvag"):
        lora.checkpoint_entries({"blocks.0.att.x_r": torch.zeros(1, 1, 8)}, (7, 0), 8)


def test_peft_and_lora_lm_key_names(lora):
    assert lora._lora_part("blocks.3.att.key.lora_A") == ("blocks.3.att.key.weight", "lora_A")
    assert lora._lora_part("blocks.3.ffn.value.lora_B.weight") == ("blocks.3.ffn.value.weight", "lora_B")
    assert lora._lora_part("blocks.3.ln1.weight") == (None, None)


def test_struct_layout_matches_the_header(pkg):
    sl = pkg.shared_library
    assert ctypes.sizeof(sl.AdapterTensor) == 40
    assert [f[0] for f in sl.AdapterTensor._fields_] == ["name", "rank", "a", "b", "values"]
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "rwkv_b200.h")).read()
    body = header[header.index("struct rwkv_b200_adapter_tensor {"):]
    body = body[:body.index("};")]
    assert [l.split(";")[0].split()[-1].lstrip("*") for l in body.splitlines()[1:] if ";" in l] == ["name", "rank", "a", "b", "values"]


def test_refusals_before_any_device_call(lib):
    lib.rwkv_set_print_errors(None, False)
    try:
        assert not lib.library.rwkv_b200_adapter_create(None, None, 0, ctypes.c_float(1.0))
        assert lib.rwkv_get_last_error(None) == ERR_ARGS
        assert lib.library.rwkv_b200_adapter_free(None)
        x = np.zeros(64, np.float32)
        P = ctypes.POINTER(ctypes.c_float)
        p = x.ctypes.data_as(P)
        args = dict(K=8, M=8, T=1, rank=1, scale=1.0, epi=0)
        for bad in (dict(T=0), dict(T=257), dict(rank=0), dict(rank=257), dict(K=0), dict(M=0), dict(epi=3), dict(epi=7), dict(epi=6)):
            a = dict(args, **bad)
            gate = p if bad.get("epi") != 6 else None
            assert not lib.library.rwkv_b200_test_lora(a["K"], a["M"], a["T"], a["rank"], ctypes.c_float(a["scale"]), a["epi"], p, p, p, p, gate, p, p), bad
            assert lib.rwkv_get_last_error(None) == ERR_ARGS, bad
        assert not lib.library.rwkv_b200_test_lora(8, 8, 1, 1, ctypes.c_float(1.0), 0, None, p, p, p, None, p, p)
        assert lib.rwkv_get_last_error(None) == ERR_ARGS
    finally:
        lib.rwkv_set_print_errors(None, True)


def test_reference_restatement():
    """lora_ref.lora_ref: rounds A and B to fp16 and applies the epilogue after the delta (or adds it to the base's output)."""
    rng = np.random.default_rng(0)
    a, b = rng.standard_normal((3, 5)).astype(np.float32), rng.standard_normal((4, 3)).astype(np.float32)
    x, z, g = rng.standard_normal((5, 2)), rng.standard_normal((4, 2)), rng.random((4, 2))
    a16 = a.astype(np.float16).astype(np.float64)
    b16 = b.astype(np.float16).astype(np.float64)
    d = 0.5 * (b16 @ (a16 @ x))
    u, y = lr.lora_ref(a, b, x, z, None, 0.5, lr.EPI_SIGMOID)
    assert np.allclose(u, a16 @ x) and np.allclose(y, 1 / (1 + np.exp(-(z + d))))
    assert np.allclose(lr.lora_ref(a, b, x, z, g, 0.5, lr.EPI_MUL_ADD)[1], z + g * d)
    assert np.allclose(lr.lora_ref(a, b, x, z, None, 0.5, lr.EPI_RELU_SQR)[1], np.maximum(z + d, 0) ** 2)


def test_merged_file_applies_deltas_and_replacements(tmp_path):
    from conftest import model_path
    src = model_path("4v0-660K", "FP32")
    entries = lr.make_entries(src, 2, 1, vectors=True)
    dst = str(tmp_path / "m.bin")
    lr.merged_file(src, dst, entries, 0.25)
    a, m = read_model_file(src).tensors, read_model_file(dst).tensors
    assert list(a) == list(m)
    for name, rank, A, B, values in entries:
        if rank:
            M, K = lr.matrix_shape(a[name])
            want = (lr.tensor_f32(a[name]).astype(np.float64).reshape(M, K) + 0.25 * lr.f16(B) @ lr.f16(A)).astype(np.float32)
            assert lr.tensor_f32(m[name]).tobytes() == want.tobytes()
        else:
            assert lr.tensor_f32(m[name]).tobytes() == values.tobytes()
    assert any(e[1] == 0 for e in entries) and any(e[1] for e in entries)


def test_encode_rows_without_a_device(lib):
    """rwkv_b200_test_encode_rows: F32 copied, F16 rounded to nearest even as numpy rounds, Q5_1 as rwkv_quantize_model_file's blocks
    (24 bytes per 32 values); bad arguments refused."""
    rng = np.random.default_rng(1)
    x = rng.standard_normal(2 * 64).astype(np.float32)
    P = ctypes.POINTER(ctypes.c_float)
    for dtype, nbytes, want in ((0, 4 * x.size, x.tobytes()), (1, 2 * x.size, x.astype(np.float16).tobytes()), (8, 24 * x.size // 32, None)):
        out = np.zeros(nbytes, np.uint8)
        assert lib.library.rwkv_b200_test_encode_rows(dtype, x.ctypes.data_as(P), 2, 64, out.ctypes.data_as(ctypes.c_void_p))
        if want is not None:
            assert out.tobytes() == want
        else:   # the oracle's dequantisation of the blocks lands within a quantisation step of x
            import rwkv_oracle
            back = rwkv_oracle.dequantize(8, out, x.size)
            assert np.abs(back - x).max() < (x.max() - x.min()) / 31
    lib.rwkv_set_print_errors(None, False)
    try:
        out = np.zeros(256, np.uint8)
        assert not lib.library.rwkv_b200_test_encode_rows(8, x.ctypes.data_as(P), 1, 33, out.ctypes.data_as(ctypes.c_void_p))
        assert lib.rwkv_get_last_error(None) == ERR_ARGS
        assert not lib.library.rwkv_b200_test_encode_rows(0, None, 1, 8, out.ctypes.data_as(ctypes.c_void_p))
        assert lib.rwkv_get_last_error(None) == ERR_ARGS
    finally:
        lib.rwkv_set_print_errors(None, True)
