"""Scoring without a GPU: the argument checks of rwkv_b200_score_logits (made before any device is touched), and the loss bookkeeping of
tools/perplexity.py against the loop of the reference's measure_pexplexity.py."""
import ctypes
import math
import os

import numpy as np

from conftest import ROOT

P_F, P_U, P_U8 = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_uint8)
NO = 0xFFFFFFFF


def test_score_logits_refuses_bad_arguments_before_the_device(lib):
    L = lib.library
    logits = np.zeros((3, 10), np.float32)
    lp, g = np.full(3, 5.0, np.float32), np.full(3, 9, np.uint8)

    def refused(lg, rows, V, targets, out):
        t = None if targets is None else np.ascontiguousarray(targets, np.uint32).ctypes.data_as(P_U)
        assert not L.rwkv_b200_score_logits(None if lg is None else lg.ctypes.data_as(P_F), rows, V, t,
                                            None if out is None else out.ctypes.data_as(P_F), g.ctypes.data_as(P_U8))
        assert lib.rwkv_get_last_error(None) == 1 << 8     # RWKV_ERROR_ARGS

    refused(None, 3, 10, [0, 1, 2], lp)
    refused(logits, 3, 10, None, lp)
    refused(logits, 3, 10, [0, 1, 2], None)
    refused(logits, 0, 10, [0, 1, 2], lp)
    refused(logits, 3, 10, [0, 10, 2], lp)                  # a target >= n_vocab
    refused(np.zeros((1, 65537), np.float32), 1, 65537, [0], lp)
    assert (lp == 5.0).all() and (g == 9).all()
    assert lib.library.rwkv_b200_score_logits.argtypes is not None
    import rwkv_cpp_b200.shared_library as sl
    assert sl.SCORE_NO_TARGET == NO


def reference_loop(losses, ignore):
    """measure_pexplexity.py's accounting: position i counts when ignore == 0 or i + 1 >= ignore; float32 running sum."""
    s, n = np.float32(0), 0
    for i, x in enumerate(losses):
        if ignore == 0 or i + 1 >= ignore:
            s += np.float32(x)
            n += 1
    return float(s / n)


def test_perplexity_accounting_matches_the_reference_loop(tmp_path):
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import perplexity
    losses = np.random.default_rng(3).uniform(0.5, 6.0, 300)
    for ignore in (0, 1, 2, 17, 299):
        loss, ppl = perplexity.average(losses, ignore)
        assert abs(loss - reference_loop(losses, ignore)) <= 1e-5 * loss
        assert ppl == math.exp(loss)
    (tmp_path / "a.txt").write_text("1 2,3\n4")
    np.save(tmp_path / "b.npy", np.array([[5, 6], [7, 8]]))
    assert perplexity.read_tokens(str(tmp_path / "a.txt")) == [1, 2, 3, 4]
    assert perplexity.read_tokens(str(tmp_path / "b.npy")) == [5, 6, 7, 8]
