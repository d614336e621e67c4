"""Streaming generation without a GPU: both entry points reject a NULL context before they touch a device, and the ctypes
declaration of the callback type matches rwkv_b200_token_fn."""
import ctypes

ARGS = 1 << 8


def test_generate_stream_entry_points_reject_a_null_context(lib, pkg):
    import rwkv_cpp_b200.shared_library as sl
    L = lib.library
    calls = []
    fn = sl.RWKV_TOKEN_FN(lambda user, seq, idx, tok: calls.append((seq, idx, tok)) or 0)
    n = ctypes.c_size_t(0)
    toks = (ctypes.c_uint32 * 4)()
    u = (ctypes.c_double * 4)(0.5, 0.5, 0.5, 0.5)
    assert not L.rwkv_b200_generate_stream(None, 4, 1.0, 1.0, 0.0, 0.0, False, u, None, 0, fn, None, toks, ctypes.byref(n))
    assert lib.rwkv_get_last_error(None) == ARGS
    ng = (ctypes.c_uint32 * 1)()
    assert not L.rwkv_b200_batch_generate_stream(None, (ctypes.c_uint32 * 1)(4), None, None, None, None, None, u, None, 0, fn, None, toks, ng)
    assert lib.rwkv_get_last_error(None) == ARGS
    assert calls == []
