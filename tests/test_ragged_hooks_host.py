"""The ragged kernel hooks (rwkv_b200_test_*_ragged) check every argument before they touch a device: on a machine without a GPU a
bad call fails with RWKV_ERROR_ARGS alone, not with the missing-device error."""
import ctypes

import numpy as np
import pytest

import kernel_hooks as kh

ARGS = 1 << 8


def call(lib, fn, args, counts, n_seq=None):
    c = None if counts is None else (ctypes.c_uint32 * len(counts))(*counts)
    ok = getattr(lib.library, fn)(None if args is None else ctypes.byref(args), c, ctypes.c_size_t(len(counts or []) if n_seq is None else n_seq))
    return bool(ok), lib.rwkv_get_last_error(None)


def buffers(n):
    return np.zeros(n, np.float32)


def ln_mix_args(C, T, n_seq, stride, keep):
    keep.append(buffers(C * T * 8 + (n_seq + 1) * stride + C))
    p = keep[-1].ctypes.data
    a = kh.LnMixArgs(x=p, ln_w=p, ln_b=p, state_in=p, state_out=p, C=C, T=T, formula=0, n_out=1, n_seq=n_seq, seq_stride=stride)
    a.coef[0], a.out[0] = p, p
    return a


def wkv6_args(H, S, T, n_seq, stride, keep):
    keep.append(buffers(1))
    p = keep[-1].ctypes.data
    return kh.Wkv6Args(r=p, k=p, v=p, td=p, tf=p, td_per_token=1, state_in=p, state_out=p, lnx_w=p, lnx_b=p, y=p, eps=1e-5, H=H, S=S, T=T,
                       n_seq=n_seq, seq_stride=stride)


def wkv7_args(H, S, T, n_seq, stride, keep):
    keep.append(buffers(1))
    p = keep[-1].ctypes.data
    return kh.Wkv7Args(r=p, w=p, k=p, v=p, a=p, g=p, k_k=p, k_a=p, r_k=p, lnx_w=p, lnx_b=p, state_in=p, state_out=p, y=p, H=H, S=S, T=T,
                       n_seq=n_seq, seq_stride=stride)


def wkv4_args(C, T, n_seq, stride, keep):
    keep.append(buffers(1))
    p = keep[-1].ctypes.data
    return kh.Wkv4Args(k=p, v=p, r=p, time_first=p, time_decay=p, aa_in=p, bb_in=p, pp_in=p, aa_out=p, bb_out=p, pp_out=p, y=p, C=C, T=T,
                       n_seq=n_seq, seq_stride=stride)


def bad_calls(make, fn, per_seq):
    """(args, counts, n_seq) triples that must be refused, built around a valid call with counts [2, 0, 3]."""
    keep = []
    good = [2, 0, 3]
    return keep, [
        (make(5, 3, per_seq, keep), None, 3),                          # NULL counts
        (None, good, 3),                                               # NULL args
        (make(5, 3, per_seq, keep), good, 0),                          # no sequences
        (make(5, 3, per_seq, keep), [0] * 257, 257),                   # more than 256 sequences
        (make(4, 3, per_seq, keep), good, 3),                          # T is not the sum of the counts
        (make(5, 2, per_seq, keep), good, 3),                          # the struct's n_seq disagrees
        (make(5, 3, per_seq - 4, keep), good, 3),                      # states overlap
        (make(0, 3, per_seq, keep), [0, 0, 0], 3),                     # no tokens at all
    ]


@pytest.mark.parametrize("kind", ["ln_mix", "wkv4", "wkv6", "wkv7"])
def test_ragged_hooks_reject_bad_arguments_without_a_device(lib, kind):
    C, H, S = 64, 2, 16
    makers = {
        "ln_mix": (lambda T, n, st, k: ln_mix_args(C, T, n, st, k), C),
        "wkv4": (lambda T, n, st, k: wkv4_args(C, T, n, st, k), C),
        "wkv6": (lambda T, n, st, k: wkv6_args(H, S, T, n, st, k), H * S * S),
        "wkv7": (lambda T, n, st, k: wkv7_args(H, S, T, n, st, k), H * S * S),
    }
    make, per_seq = makers[kind]
    fn = "rwkv_b200_test_%s_ragged" % kind
    keep, cases = bad_calls(make, fn, per_seq)
    for i, (args, counts, n_seq) in enumerate(cases):
        ok, flags = call(lib, fn, args, counts, n_seq)
        assert not ok and flags == ARGS, (kind, i, flags)
    # staged columns are single-sequence only
    if kind != "ln_mix":
        args = make(5, 3, per_seq, keep)
        args.q_out = keep[0].ctypes.data
        ok, flags = call(lib, fn, args, [2, 0, 3])
        assert not ok and flags == ARGS, kind
    if kind == "wkv6":
        ok, flags = call(lib, fn, make(5, 3, per_seq + 2, keep), [2, 0, 3])       # the state moves in float4s
        assert not ok and flags == ARGS
