"""Generation with log-probabilities without a GPU: the ctypes mirror of struct rwkv_b200_logprobs matches the header's layout, the new
entry points are exported and declared and reject a NULL context before they touch a device, the float64 top-N reference of the GPU
tests orders ties, -0 and -inf as the contract says, and the new step kernels are built with the resources the existing checks allow."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from test_gpu_generate_logprobs import NO_TARGET, top_ref

ARGS = 1 << 8
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("rwkv_b200_generate_logprobs", "rwkv_b200_batch_generate_logprobs", "rwkv_b200_test_generate_step_logprobs")


def test_logprob_symbols_are_exported_and_declared(lib):
    with open(os.path.join(ROOT, "include", "rwkv_b200.h")) as f:
        header = f.read()
    assert "#define RWKV_B200_TOP_LOGPROBS_MAX 20" in header
    for name in NAMES:
        assert hasattr(lib.library, name), name
        assert getattr(lib.library, name).argtypes is not None, name
        assert re.search(r"RWKV_API [^;]*\b%s\(" % name, header), name


def test_ctypes_struct_matches_the_header(pkg, tmp_path):
    """Field offsets and size of struct rwkv_b200_logprobs from a probe compiled against the header."""
    import rwkv_cpp_b200.shared_library as sl
    fields = [f for f, _ in sl.Logprobs._fields_]
    src = tmp_path / "probe.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "rwkv_b200.h"\nint main(void) {\n' +
                   "".join('    printf("%%zu\\n", offsetof(struct rwkv_b200_logprobs, %s));\n' % f for f in fields) +
                   '    printf("%zu\\n", sizeof(struct rwkv_b200_logprobs));\n    return 0;\n}\n')
    exe = tmp_path / "probe"
    cc = "gcc" if subprocess.run(["which", "gcc"], capture_output=True).returncode == 0 else "g++"
    r = subprocess.run([cc, "-x", "c" if cc == "gcc" else "c++", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [getattr(sl.Logprobs, f).offset for f in fields] + [ctypes.sizeof(sl.Logprobs)]


def test_logprob_entry_points_reject_a_null_context(lib, pkg):
    import rwkv_cpp_b200.shared_library as sl
    L = lib.library
    calls = []
    fn = sl.RWKV_TOKEN_FN(lambda user, seq, idx, tok: calls.append((seq, idx, tok)) or 0)
    n = ctypes.c_size_t(0)
    toks = (ctypes.c_uint32 * 4)()
    u = (ctypes.c_double * 4)(0.5, 0.5, 0.5, 0.5)
    lps = (ctypes.c_float * 4)()
    lp = sl.Logprobs(top_n=0, logprobs=lps)
    for on_token in (fn, sl.RWKV_TOKEN_FN()):
        assert not L.rwkv_b200_generate_logprobs(None, None, None, 4, 1.0, 1.0, 0.0, 0.0, False, u, None, 0, on_token, None, toks, ctypes.byref(n),
                                                 ctypes.byref(lp))
        assert lib.rwkv_get_last_error(None) == ARGS
        ng = (ctypes.c_uint32 * 1)()
        assert not L.rwkv_b200_batch_generate_logprobs(None, None, None, (ctypes.c_uint32 * 1)(4), None, None, None, None, None, u, None, 0,
                                                       on_token, None, toks, ng, ctypes.byref(lp))
        assert lib.rwkv_get_last_error(None) == ARGS
    assert calls == []


def test_step_hook_checks_the_request_first(lib, pkg):
    """A NULL request, NULL logprobs, top_n above 20 or n_vocab and NULL top arrays are refused before any device is touched."""
    import generate_ref as gr
    import rwkv_cpp_b200.shared_library as sl
    V = 8
    logits = np.zeros(V, np.float32)
    mt, st, fr, cnt, tk, nx = (np.array([1], np.uint32), np.zeros(1, np.uint32), np.zeros(1, np.uint8), np.zeros(V, np.uint32), np.zeros(1, np.uint32),
                               np.zeros(1, np.int32))
    ones, zero, u = np.ones(1, np.float32), np.zeros(1, np.float32), np.full(1, 0.5)
    act = ctypes.c_uint32(0)
    a = gr.StepArgs(logits=logits.ctypes.data, n_rows=1, n_vocab=V, max_tokens=mt.ctypes.data, temperature=ones.ctypes.data, top_p=ones.ctypes.data,
                    presence_penalty=zero.ctypes.data, frequency_penalty=zero.ctypes.data, u=u.ctypes.data, stop_ids=None, n_stop=0, step=st.ctypes.data,
                    frozen=fr.ctypes.data, counts=cnt.ctypes.data, tokens=tk.ctypes.data, next_tokens=nx.ctypes.data, any_active=ctypes.addressof(act))
    lps, tl = (ctypes.c_float * 32)(), (ctypes.c_float * 32)()
    ti = (ctypes.c_uint32 * 32)()
    for lp in [None, sl.Logprobs(top_n=0), sl.Logprobs(top_n=21, logprobs=lps, top_ids=ti, top_logprobs=tl),
               sl.Logprobs(top_n=9, logprobs=lps, top_ids=ti, top_logprobs=tl), sl.Logprobs(top_n=2, logprobs=lps, top_logprobs=tl),
               sl.Logprobs(top_n=2, logprobs=lps, top_ids=ti)]:
        assert not lib.library.rwkv_b200_test_generate_step_logprobs(ctypes.byref(a), None, 0, None, ctypes.byref(lp) if lp else None)
        assert lib.rwkv_get_last_error(None) == ARGS
        assert st[0] == 0


def test_top_reference_orders_ties_and_minus_inf():
    inf = np.inf
    assert top_ref([1.0, 3.0, 3.0, 2.0], 3) == [1, 2, 3]                  # equal logits: the smaller id first
    assert top_ref([0.0, -0.0, 0.0, -1.0], 3) == [0, 1, 2]                # -0 equals +0
    assert top_ref([-inf, 2.0, -inf, -inf], 3) == [1, 0, 2]              # -inf only when fewer finite entries than top_n, by id
    assert top_ref([5.0, 5.0, 5.0, 5.0, 4.0], 2) == [0, 1]                # a tie across the boundary keeps the smaller ids
    assert top_ref([1.0, np.nan, 2.0], 2) == [NO_TARGET] * 2              # NaN, +inf and nothing finite: no ids
    assert top_ref([1.0, inf, 2.0], 1) == [NO_TARGET]
    assert top_ref([-inf, -inf], 2) == [NO_TARGET] * 2
    assert top_ref([7.0], 1) == [0]


def test_logprob_kernels_are_built_within_the_resource_checks(lib):
    """Ten new step kernels (two families at the five PER instantiations), named *sample_kernel as test_no_kernel_spills_its_parameters
    expects of the 1024-thread step kernels, each within 64 registers and a stack frame no larger than 512 bytes."""
    r = subprocess.run(["cuobjdump", "--dump-resource-usage", lib.path], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("cuobjdump not available")
    found = re.findall(r"Function (\S*(?:generate_logprob|generate_stream_logprob)_sample_kernel\S*):\s*REG:(\d+) STACK:(\d+)", r.stdout)
    assert len(found) == 10, found
    for name, reg, stack in found:
        assert int(reg) <= 64 and int(stack) <= 512, (name, reg, stack)
