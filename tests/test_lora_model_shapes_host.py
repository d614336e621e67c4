"""The adapted-batch table of tests/test_gpu_lora_model_shapes.py without a GPU: it agrees with the delta targets of adapter.cpp and the
batches engine.cu builds, rwkv_b200_test_lora_gemv_batch refuses bad arguments before touching a device, and each plausible defect of
an adapted batch, planted into the float64 restatement, fails the check of part A."""
import ctypes
import os
import re

import numpy as np
import pytest

import kernel_hooks as kh
import kernel_ref as kr
import lora_ref as lr
import test_gpu_gemv as tg
import test_gpu_lora_model_shapes as lms
import test_gpu_model_shapes as ms

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "rwkv.cpp_b200", "csrc")
ERR_ARGS = 1 << 8
EPI_NAMES = {"EPI_NONE": kr.EPI_NONE, "EPI_SIGMOID": kr.EPI_SIGMOID, "EPI_SILU": kr.EPI_SILU, "EPI_RELU_SQR": kr.EPI_RELU_SQR,
             "EPI_ADD": kr.EPI_ADD, "EPI_MUL_ADD": kr.EPI_MUL_ADD}

# (tensor, epilogue) of the adapted problems of each batch, per architecture
ADAPTED = {
    4: {"att": [("att.receptance.weight", kr.EPI_SIGMOID), ("att.key.weight", 0), ("att.value.weight", 0)]},
    5: {"att": [("att.receptance.weight", 0), ("att.key.weight", 0), ("att.value.weight", 0), ("att.gate.weight", kr.EPI_SILU)]},
    6: {"att": [("att.receptance.weight", 0), ("att.key.weight", 0), ("att.value.weight", 0), ("att.gate.weight", kr.EPI_SILU)]},
    7: {"lora_first": [("att.receptance.weight", 0), ("att.key.weight", 0), ("att.value.weight", 0)]},
}
for a in (4, 5, 6, 7):
    ADAPTED[a].update(ffn_kr=[("ffn.key.weight", kr.EPI_RELU_SQR)] + ([("ffn.receptance.weight", kr.EPI_SIGMOID)] if a != 7 else []),
                      ffn_value=[("ffn.value.weight", kr.EPI_ADD if a == 7 else kr.EPI_MUL_ADD)], att_output=[("att.output.weight", kr.EPI_ADD)])


def field(target):
    """The Layer field of a delta target: att.key.weight -> att_key."""
    return target[:-len(".weight")].replace(".", "_")


def test_delta_targets_match_adapter_cpp():
    src = open(os.path.join(CSRC, "adapter.cpp")).read()
    body = re.search(r"bool delta_target\(.*?\{(.*?)\n\}", src, re.S).group(1)
    assert set(re.findall(r"&L\.(\w+)", body)) == {field(t) for t in lr.DELTA_TARGETS}


def test_adapted_table_matches_engine_cu():
    """Per architecture, the adapted problems of every batch of the table; and every (matrix, epilogue) engine.cu adds for a delta
    target is one of the table, and the other way round."""
    for s in ms.SHAPES:
        got = {b: [(t, epi) for t, _, _, _, epi in spec if t in lr.DELTA_TARGETS] for b, spec in lms.adapted_batches(s).items()}
        assert got == ADAPTED[s.arch[0]], s.name
    src = open(os.path.join(CSRC, "engine.cu")).read()
    calls = set()
    for name, args in re.findall(r"b\.add\(L\.(\w+),([^;]*)\);", src):
        if name in {field(t) for t in lr.DELTA_TARGETS}:
            epis = re.findall(r"EPI_\w+", args) or ["EPI_NONE"]
            calls |= {(name, EPI_NAMES[e]) for e in epis}
    table = {(field(t), epi) for a in ADAPTED.values() for spec in a.values() for t, epi in spec}
    assert calls == table, (sorted(calls - table), sorted(table - calls))


def test_hook_refusals_come_before_the_device(lib):
    """Bad arguments give RWKV_ERROR_ARGS whether or not a device exists."""
    s = ms.BY_NAME["rwkv5-0b4"]
    spec = lms.adapted_batches(s)["att"]
    rng = np.random.default_rng(0)
    probs, xs = ms.build(s, "Q5_1", "att", 3, rng)
    good = lms.layout("mixed", spec, 3, 8, rng)

    def refused(edit, T=3):
        i = kh.Inputs()
        a, _, _ = kh.lora_args(T, probs, xs, "engine", s.C, s.F, *good, i)
        edit(a)
        assert not lib.library.rwkv_b200_test_lora_gemv_batch(ctypes.byref(a))
        assert lib.rwkv_get_last_error(None) == ERR_ARGS

    def set_(path, value):
        def edit(a):
            obj = a
            for k in path[:-1]:
                obj = getattr(obj, k) if isinstance(k, str) else obj[k]
            if isinstance(path[-1], str):
                setattr(obj, path[-1], value)
            else:
                obj[path[-1]] = value
        return edit
    lib.rwkv_set_print_errors(None, False)
    try:
        assert not lib.library.rwkv_b200_test_lora_gemv_batch(None)
        assert lib.rwkv_get_last_error(None) == ERR_ARGS
        for path, value in [(("n_embed",), 0), (("n_ffn",), -1), (("n_adapters",), 0), (("n_adapters",), 32), (("n_deltas",), 32),
                            (("d", 0, "rank"), 0), (("d", 0, "rank"), 257), (("d", 0, "K"), s.C + 32), (("d", 0, "M"), 7),
                            (("d", 1, "a"), None), (("d", 1, "b"), None), (("delta_of", 0, 0), len(good[0])),
                            (("delta_of", 0, 3), 0), (("delta_of", 4, 0), 0), (("delta_of", 0, 0), -2), (("col_adapter", 1), 3),
                            (("col_adapter", 1), -2), (("col_adapter", 3), 0), (("base", "T"), 0), (("base", "n"), 9)]:
            refused(set_(path, value))
    finally:
        lib.rwkv_set_print_errors(None, True)


# ---- planted bugs -------------------------------------------------------------------------------------------------------------------

def case(shape, batch, T=5, fmt="Q5_1"):
    s = ms.BY_NAME[shape]
    spec = lms.adapted_batches(s)[batch]
    rng = tg.rng_for("lora-host", shape, batch)
    probs, xs = ms.build(s, fmt, batch, T, rng)
    return spec, probs, xs, lms.layout("mixed", spec, T, 16, rng)


def caught(spec, probs, xs, lay, bug):
    """Whether part A's check fails on some problem of the batch when the kernel's output is the float64 restatement with `bug`
    planted; the float32 restatement without it must pass."""
    deltas, delta_of, cols = lay
    fails, prev = 0, None
    for j, p in enumerate(probs):
        rows = np.sort(tg.rng_for("lora-host-rows", j).choice(p["M"], min(p["M"], 96), replace=False))
        sub = ms.row_subset(p, rows)
        r64, base64, _ = lms.adapted_reference(p, sub, rows, xs, np.float64, False, deltas, delta_of[j], cols)
        r32, _, _ = lms.adapted_reference(p, sub, rows, xs, np.float32, False, deltas, delta_of[j], cols)
        bad, _, _ = lms.adapted_reference(p, sub, rows, xs, np.float64, False, deltas, delta_of[j], cols, bug=bug, prev_base=prev)
        mag = lms.magnitude(p, sub, rows, xs, base64, deltas, delta_of[j], cols)
        lms.check_adapted("host", (bug, j), r32, r64, r32, 4, mag)
        if not any(k >= 0 for k in delta_of[j]):
            prev = None
            continue
        try:
            lms.check_adapted("host", (bug, j), bad, r64, r32, 4, mag)
        except AssertionError:
            fails += 1
        prev = base64 if p["epi"] not in lms.RESIDUAL else None
    return fails > 0


@pytest.mark.parametrize("bug,shape,batch", [
    ("delta_after_epilogue", "rwkv4-169m", "ffn_kr"),      # relu^2 and sigmoid
    ("delta_after_epilogue", "rwkv5-0b4", "att"),          # silu of the gate
    ("b_fp32", "rwkv6-1b6", "att"),
    ("ungated", "rwkv5-0b4", "ffn_value"),
    ("neighbour_adapter", "rwkv7-0b1", "lora_first"),
    ("neighbour_adapter", "rwkv4-169m", "att_output"),
    ("z_offset", "rwkv5-0b4", "att"),
])
def test_planted_bugs_fail_the_check(bug, shape, batch):
    assert caught(*case(shape, batch), bug), bug
