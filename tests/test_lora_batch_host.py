"""Per-sequence adapters of batch contexts without a GPU: the exported symbols, the ctypes prototypes against the header, the refusals
that come before any device call, and the resource usage of the grouped shrink and expand kernels in the built library."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

ERR_ARGS = 1 << 8
HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "rwkv_b200.h")
NEW = ("rwkv_b200_batch_set_adapter", "rwkv_b200_test_lora_columns")


def prototype(name):
    """The parameter types of `name` in the header, as a list of normalised C type strings."""
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    m = re.search(r"RWKV_API\s+bool\s+" + name + r"\s*\(([^)]*)\)\s*;", text)
    assert m, name
    out = []
    for p in m.group(1).split(","):
        words = p.replace("*", " * ").split()
        out.append(" ".join(words[:-1]))      # drop the parameter name
    return out


def ctype_of(c):
    """The C type string a ctypes argtype stands for."""
    P = ctypes.POINTER
    table = {ctypes.c_void_p: "void *", ctypes.c_size_t: "size_t", ctypes.c_int: "int", P(ctypes.c_float): "float *", P(ctypes.c_int): "int *",
             P(P(ctypes.c_float)): "float * *"}
    return table[c]


def test_symbols_are_exported(lib):
    for name in NEW:
        assert hasattr(lib.library, name), name
    r = subprocess.run(["nm", "-D", "--defined-only", lib.path], capture_output=True, text=True)
    if r.returncode == 0:
        for name in NEW:
            assert re.search(r"\bT " + name + r"\b", r.stdout), name


def test_ctypes_prototypes_match_the_header(lib):
    for name in NEW:
        c_types = prototype(name)
        argtypes = getattr(lib.library, name).argtypes
        assert len(argtypes) == len(c_types), name
        assert getattr(lib.library, name).restype is ctypes.c_bool
        for c, a in zip(c_types, argtypes):
            want = c.replace("const ", "").replace("struct rwkv_context", "void").replace("struct rwkv_b200_adapter", "void")
            assert ctype_of(a) == " ".join(want.split()), (name, c, a)


def test_refusals_before_any_device_call(lib):
    lib.rwkv_set_print_errors(None, False)
    try:
        assert not lib.library.rwkv_b200_batch_set_adapter(None, 0, None)
        assert lib.rwkv_get_last_error(None) == ERR_ARGS
        assert not lib.library.rwkv_b200_batch_set_adapter(None, 3, 12345)
        assert lib.rwkv_get_last_error(None) == ERR_ARGS
        x = np.zeros(64, np.float32)
        p = x.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
        PP = ctypes.POINTER(ctypes.c_float) * 2
        ab = PP(p, p)
        PI = ctypes.POINTER(ctypes.c_int)
        ranks, cols = np.array([1, 2], np.int32), np.array([0, -1, 1], np.int32)
        args = dict(K=8, M=8, T=3, n=2, ranks=ranks, cols=cols, epi=0)

        def call(a, A=ab, B=ab, gate=p):
            return lib.library.rwkv_b200_test_lora_columns(a["K"], a["M"], a["T"], a["n"], a["ranks"].ctypes.data_as(PI), p, A, B,
                                                            a["cols"].ctypes.data_as(PI), a["epi"], p, p, gate, p, p)
        bads = [dict(T=0), dict(T=257), dict(K=0), dict(M=0), dict(n=0), dict(n=32), dict(epi=3), dict(epi=7), dict(epi=6),
                dict(ranks=np.array([0, 2], np.int32)), dict(ranks=np.array([1, 257], np.int32)),
                dict(cols=np.array([0, -2, 1], np.int32)), dict(cols=np.array([0, 2, 1], np.int32))]
        for bad in bads:
            a = dict(args, **bad)
            assert not call(a, gate=None if bad.get("epi") == 6 else p), bad
            assert lib.rwkv_get_last_error(None) == ERR_ARGS, bad
        assert not call(args, A=None)
        assert not call(args, B=PP(p, None))
        assert lib.rwkv_get_last_error(None) == ERR_ARGS
    finally:
        lib.rwkv_set_print_errors(None, True)


def test_grouped_kernels_do_not_spill(lib):
    """The shrink and expand kernels reach their columns through the group's list; that must not cost them local memory."""
    r = subprocess.run(["cuobjdump", "--dump-resource-usage", lib.path], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("cuobjdump not available")
    found = {n: (int(reg), int(st)) for n, reg, st in re.findall(r"Function ([^:\s]+):\s*\n\s*REG:(\d+) STACK:(\d+)", r.stdout)
             if "lora_shrink_kernel" in n or "lora_expand_kernel" in n}
    assert len(found) == 2, found
    for name, (reg, stack) in found.items():
        assert stack == 0 and reg <= 128, (name, reg, stack)
