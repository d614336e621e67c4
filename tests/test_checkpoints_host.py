"""Checkpoints without a GPU: the exported prototypes and struct layout against include/rwkv_b200.h, every refusal of the entries that
needs no device (through the argument-check hook and a NULL context), and the arguments the Python wrappers build."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = open(os.path.join(ROOT, "include", "rwkv_b200.h")).read()
ERR_ARGS = 1 << 8


def test_prototypes_and_struct_layout_match_the_header(lib, pkg):
    sl = pkg.shared_library
    for name in ("rwkv_b200_eval_checkpoints", "rwkv_b200_batch_eval_ragged_checkpoints", "rwkv_b200_test_checkpoint_args"):
        assert hasattr(lib.library, name), name
        m = re.search(r"RWKV_API bool " + name + r"\(([^;]*)\);", HDR, re.S)
        assert m, name
        assert len(m.group(1).split(",")) == len(getattr(lib.library, name).argtypes), name
    body = re.search(r"struct rwkv_b200_checkpoint \{(.*?)\};", HDR, re.S).group(1)
    assert re.findall(r"(\w+);", re.sub(r"/\*.*?\*/", "", body)) == [f for f, _ in sl.Checkpoint._fields_]
    assert ctypes.sizeof(sl.Checkpoint) == 16 and sl.Checkpoint.position.offset == 4 and sl.Checkpoint.state_out.offset == 8


def entries(pkg, items):
    sl = pkg.shared_library
    arr = (sl.Checkpoint * max(1, len(items)))()
    for i, (s, p, a) in enumerate(items):
        arr[i] = sl.Checkpoint(s, p, ctypes.cast(a, ctypes.POINTER(ctypes.c_float)))
    return arr


N = 100   # floats per state in these checks


@pytest.mark.parametrize("counts,items,ok", [
    ([10], [(0, 0, 4096), (0, 9, 8192)], True),
    ([10], [], True),
    ([10], [(0, 3, 4096), (0, 3, 8192)], False),                # repeated
    ([10], [(0, 4, 4096), (0, 3, 8192)], False),                # out of order
    ([10], [(0, 10, 4096)], False),                             # position out of range
    ([10], [(1, 0, 4096)], False),                              # sequence out of range (single context: 0 only)
    ([10], [(0, 1, 0)], False),                                 # NULL state_out
    ([10], [(0, 1, 4096), (0, 2, 4096 + 4 * N - 4)], False),    # overlapping destinations
    ([10], [(0, 1, 4096 + 4 * N), (0, 2, 4096)], True),         # adjacent, listed out of address order
    ([3, 0, 5], [(0, 2, 4096), (2, 0, 8192), (2, 4, 12288)], True),
    ([3, 0, 5], [(1, 0, 4096)], False),                         # an idle sequence has no position
    ([3, 0, 5], [(2, 1, 4096), (0, 2, 8192)], False),           # (sequence, position) out of order
])
def test_argument_refusals(lib, pkg, counts, items, ok):
    c = np.ascontiguousarray(counts, np.uint32)
    arr = entries(pkg, items)
    got = lib.library.rwkv_b200_test_checkpoint_args(len(counts), c.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32)), N, arr, len(items))
    assert got == ok
    assert lib.rwkv_get_last_error(None) == (0 if ok else ERR_ARGS)


def test_null_cp_and_null_context(lib, pkg):
    c = np.ascontiguousarray([10], np.uint32)
    P = ctypes.POINTER(ctypes.c_uint32)
    assert not lib.library.rwkv_b200_test_checkpoint_args(1, c.ctypes.data_as(P), N, None, 2)
    assert lib.rwkv_get_last_error(None) == ERR_ARGS
    assert lib.library.rwkv_b200_test_checkpoint_args(1, c.ctypes.data_as(P), N, None, 0)
    arr = entries(pkg, [(0, 1, 4096)])
    assert not lib.library.rwkv_b200_eval_checkpoints(None, c.ctypes.data_as(P), 1, False, None, arr, 1)
    assert lib.rwkv_get_last_error(None) == ERR_ARGS
    assert not lib.library.rwkv_b200_batch_eval_ragged_checkpoints(None, c.ctypes.data_as(P), c.ctypes.data_as(P), False, arr, 1)
    assert lib.rwkv_get_last_error(None) == ERR_ARGS


class FakeLib:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def f(*args):
            self.calls.append((name, args))
            return name.endswith("_state_len") and 8 or True
        return f


def test_wrappers_build_the_arguments(pkg):
    sl = pkg.shared_library
    w = sl.RWKVSharedLibrary.__new__(sl.RWKVSharedLibrary)
    w.library = FakeLib()
    ctx = sl.RWKVContext(ctypes.c_void_p(1234))
    out = w.rwkv_b200_eval_checkpoints(ctx, [5, 6, 7], [0, 2], want_logits=True)
    name, args = w.library.calls[-1]
    assert name == "rwkv_b200_eval_checkpoints" and out.shape == (2, 8) and out.dtype == np.float32
    assert list(args[1]) == [5, 6, 7] and args[2] == 3 and args[3] is True and args[6] == 2
    assert [(args[5][i].sequence, args[5][i].position) for i in range(2)] == [(0, 0), (0, 2)]
    assert [ctypes.cast(args[5][i].state_out, ctypes.c_void_p).value for i in range(2)] == [out[0].ctypes.data, out[1].ctypes.data]
    mine = [np.empty(8, np.float32), np.empty(8, np.float32)]
    res = w.rwkv_b200_batch_eval_ragged_checkpoints(ctx, [1, 2, 3], [2, 0, 1], [(0, 1), (2, 0)], out=mine)
    name, args = w.library.calls[-1]
    assert name == "rwkv_b200_batch_eval_ragged_checkpoints" and res is mine
    assert list(args[2]) == [2, 0, 1] and args[5] == 2
    assert [(args[4][i].sequence, args[4][i].position) for i in range(2)] == [(0, 1), (2, 0)]
    assert [ctypes.cast(args[4][i].state_out, ctypes.c_void_p).value for i in range(2)] == [m.ctypes.data for m in mine]
    with pytest.raises(ValueError):
        w.rwkv_b200_eval_checkpoints(ctx, [1], [0], out=[])


@pytest.mark.parametrize("bad", ["float64", "short", "strided", "float16-tensor", "short-tensor", "strided-tensor"])
def test_wrappers_refuse_buffers_a_state_does_not_fit(pkg, bad):
    """A buffer the library would write past (too short, another dtype, not contiguous) is refused before the call."""
    import torch
    sl = pkg.shared_library
    w = sl.RWKVSharedLibrary.__new__(sl.RWKVSharedLibrary)
    w.library = FakeLib()
    ctx = sl.RWKVContext(ctypes.c_void_p(1234))
    buf = {"float64": np.empty(8, np.float64), "short": np.empty(7, np.float32), "strided": np.empty(16, np.float32)[::2],
           "float16-tensor": torch.empty(8, dtype=torch.float16), "short-tensor": torch.empty(7, dtype=torch.float32),
           "strided-tensor": torch.empty(16, dtype=torch.float32)[::2]}[bad]
    with pytest.raises(ValueError):
        w.rwkv_b200_eval_checkpoints(ctx, [1, 2], [0], out=[buf])
    assert not any(name == "rwkv_b200_eval_checkpoints" for name, _ in w.library.calls)
    ok = [np.empty(9, np.float32)[1:], torch.empty(8, dtype=torch.float32)]     # any float alignment, any length >= state_len
    w.rwkv_b200_eval_checkpoints(ctx, [1, 2], [0, 1], out=ok)
