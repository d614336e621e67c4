"""Q4_K / Q5_K without a GPU: the quantizer against the compiled reference's bytes, the loader's rules, the routing predicates."""
import ctypes
import hashlib
import struct

import numpy as np
import pytest

from conftest import model_path
import kquant_ref as kr

ERR = dict(ARGS=1 << 8, MODEL_PARAMS=4 << 8, DATA_TYPE=8, UNSUPPORTED=9)
G = kr.golden()


@pytest.fixture(scope="module")
def quantized(lib, tmp_path_factory):
    """preset:fmt -> path of this library's quantisation of the seeded FP16 master."""
    tmp = tmp_path_factory.mktemp("kquant")
    lib.rwkv_set_print_errors(None, False)
    out = {}
    for name, p in G["presets"].items():
        master = tmp / (name + ".bin")
        kr.write_master(master, p, G["seed"])
        for fmt in ("Q4_K", "Q5_K"):
            path = tmp / ("%s-%s.bin" % (name, fmt))
            lib.rwkv_quantize_model_file(str(master), str(path), fmt)
            out["%s:%s" % (name, fmt)] = path
    return out


@pytest.mark.parametrize("key", sorted(G["sha256"]))
def test_quantizer_matches_the_reference(quantized, key):
    # well-formed presets: the reference's own bytes; rwkv5-small / rwkv6-small: its K-quant bytes where rows are whole super-blocks
    # and its Q5_0 / Q5_1 bytes elsewhere (tests/golden/make_kquant_ref.py)
    assert hashlib.sha256(quantized[key].read_bytes()).hexdigest() == G["sha256"][key]


def _records(path):
    buf = path.read_bytes()
    off, out = 24, []
    while off < len(buf):
        dims, klen, dt = struct.unpack_from("<3I", buf, off)
        ne = struct.unpack_from("<%dI" % dims, buf, off + 12)
        name = buf[off + 12 + 4 * dims:off + 12 + 4 * dims + klen].decode()
        n = int(np.prod(ne))
        nbytes = {0: 4 * n, 1: 2 * n, 7: 22 * n // 32, 8: 24 * n // 32, 13: 144 * n // 256, 14: 176 * n // 256}[dt]
        out.append((name, dt, ne, off, nbytes))
        off += 12 + 4 * dims + klen + nbytes
    return buf, out


@pytest.mark.parametrize("fmt", ["Q4_K", "Q5_K"])
def test_fallback_keeps_the_requested_header_type(quantized, fmt):
    buf, recs = _records(quantized["rwkv6-small:" + fmt])
    assert struct.unpack_from("<I", buf, 20)[0] == kr.TYPE_ID[fmt]
    types = {name: dt for name, dt, _, _, _ in recs}
    assert types["blocks.0.att.time_decay_w2"] == (7 if fmt == "Q4_K" else 8)
    assert types["blocks.0.att.key.weight"] == kr.TYPE_ID[fmt]


@pytest.mark.parametrize("fmt", ["Q4_K", "Q5_K"])
def test_inspect_kquant_file(lib, quantized, fmt):
    path = quantized["v6:" + fmt]
    info = lib.rwkv_b200_inspect_file(str(path))
    buf, recs = _records(path)
    # the record sizes above come from 144 / 176 bytes per 256 weights, independently of the library's dtype_block_bytes
    assert info.n_tensors == len(recs) and info.file_size == len(buf) and info.data_type == kr.TYPE_ID[fmt]
    assert info.bytes_per_token == sum(nb // ne[1] if name == "emb.weight" else nb for name, _, ne, _, nb in recs) + 8 * info.state_len
    types = {name: dt for name, dt, _, _, _ in recs}
    for i in range(2):
        for m in ("key", "value", "receptance", "gate", "output"):
            assert types["blocks.%d.att.%s.weight" % (i, m)] == kr.TYPE_ID[fmt]
        for m in ("key", "value", "receptance"):
            assert types["blocks.%d.ffn.%s.weight" % (i, m)] == kr.TYPE_ID[fmt]
        assert types["blocks.%d.att.time_decay_w2" % i] == kr.TYPE_ID[fmt]          # decay rank 256: whole super-blocks
    assert types["emb.weight"] == types["head.weight"] == 1


def _inspect(lib, path):
    from rwkv_cpp_b200.shared_library import FileInfo
    ok = lib.library.rwkv_b200_inspect_file(str(path).encode(), ctypes.byref(FileInfo()))
    return ok, lib.rwkv_get_last_error(None)


def test_loader_refusals(lib, quantized, tmp_path):
    lib.rwkv_set_print_errors(None, False)
    buf, recs = _records(quantized["v4:Q4_K"])
    assert _inspect(lib, quantized["v4:Q4_K"]) == (True, 0)
    # emb.weight / head.weight in a K-quant type (rows of C = 256: the shape is fine, the tensor is not)
    for name in ("emb.weight", "head.weight"):
        _, dt, ne, off, _ = next(r for r in recs if r[0] == name)
        p = tmp_path / ("kq-" + name)
        p.write_bytes(buf[:off + 8] + struct.pack("<I", 13) + buf[off + 12:])
        assert _inspect(lib, p) == (False, ERR["MODEL_PARAMS"] | ERR["UNSUPPORTED"]), name
    # a K-quant tensor with rows of 128 or 64 weights
    q = open(model_path("4v0-660K", "Q5_1"), "rb").read()
    for ne0 in (128, 64):
        p = tmp_path / ("row%d.bin" % ne0)
        p.write_bytes(q[:24] + struct.pack("<3I", 2, 3, 14) + struct.pack("<2I", ne0, 4) + b"abc" + bytes(176))
        assert _inspect(lib, p) == (False, ERR["MODEL_PARAMS"] | ERR["UNSUPPORTED"]), ne0
    # the other K-quant ids and Q8_1 stay refused
    first = 24
    for dt in (10, 11, 12, 15, 16):
        p = tmp_path / ("id%d.bin" % dt)
        p.write_bytes(buf[:first + 8] + struct.pack("<I", dt) + buf[first + 12:])
        assert _inspect(lib, p) == (False, ERR["MODEL_PARAMS"] | ERR["UNSUPPORTED"]), dt


def test_quantizer_refuses_the_other_kquants(lib, quantized, tmp_path):
    lib.rwkv_set_print_errors(None, False)
    master = tmp_path / "m.bin"
    kr.write_master(master, G["presets"]["v4"], 0)
    for fmt in ("Q2_K", "Q3_K", "Q6_K", "Q8_K", "Q8_1"):
        assert not lib.library.rwkv_quantize_model_file(str(master).encode(), str(tmp_path / "o.bin").encode(), fmt.encode())
        assert lib.rwkv_get_last_error(None) == ERR["ARGS"] | ERR["DATA_TYPE"], fmt


def test_v6_fold_is_not_taken_for_kquant_matrices(lib):
    fold = lib.library.rwkv_b200_v6_lora_fold_supported
    fold.restype = ctypes.c_bool
    assert fold(4096, 64, 8, 64, 8, 128)                 # Q5_1: folded
    for kq in (13, 14):
        assert not fold(4096, 64, kq, 64, 8, 128)
        assert not fold(4096, 64, 8, 64, kq, 256)


def test_hooks_reject_partial_super_blocks_before_the_device(lib):
    lib.rwkv_set_print_errors(None, False)
    PF = ctypes.POINTER(ctypes.c_float)
    x, y, w = np.zeros(512, np.float32), np.zeros(512, np.float32), np.zeros(4096, np.uint8)
    for tid in (13, 14):
        assert not lib.library.rwkv_b200_matvec(tid, 128, 4, 1, w.ctypes.data, x.ctypes.data_as(PF), y.ctypes.data_as(PF), 0)
        assert lib.rwkv_get_last_error(None) == ERR["ARGS"]
