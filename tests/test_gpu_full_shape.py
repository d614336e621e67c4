"""BASELINE.json's configurations at their FULL shapes against the UNMODIFIED reference.

tests/golden/ref_full_shape.npz holds what the compiled reference (oracle/_ref) computed on the seeded synthetic files of
tools/synthetic_model.py (tests/golden/make_ref_full_shape.py, run in the build container): logits of the last token and a
strided sample of the final state for n single-token evaluations and for one rwkv_eval_sequence_in_chunks call (chunk 128).
The GPU box regenerates the same files from the same seeds and the CUDA path, called through the C ABI, must land within the
bars of the tiny fixtures: 5e-3 max-abs for FP16 files, 5e-2 for quantised ones (DESIGN.md section 3 explains why they are
not tighter: the reference differs from itself by 1.5e-3 / 8.3e-3 between its AVX2 and AVX-512 builds) -- logits here have
|max| 4.3 .. 4.9. The chunk cases run the wgmma prefill path (>= 32 tokens): this is where it is pinned to the reference.
Plus the size-independent invariants the reference's tests pin (serial == sequence == chunked bit for bit below the
tensor-core threshold, logits on / off, clone, overlapped state copies)."""
import ctypes
import os

import numpy as np
import pytest

from conftest import GOLDEN

pytestmark = pytest.mark.gpu
P_F = ctypes.POINTER(ctypes.c_float)
STATE_STRIDE = 1009
TOL = {"FP16": 5e-3, "Q": 5e-2}
# name -> (preset, format, seed)          (the same table as tests/golden/make_ref_full_shape.py)
CASES = {
    "rwkv4-169m:Q5_1": ("rwkv4-169m", "Q5_1", 3),
    "rwkv5-1b5:Q4_0": ("rwkv5-1b5", "Q4_0", 3),
    "rwkv7-2b9:FP16": ("rwkv7-2b9", "FP16", 3),
    "rwkv6-7b:Q8_0": ("rwkv6-7b", "Q8_0", 1),
    "rwkv6-7b:Q5_1": ("rwkv6-7b", "Q5_1", 1),
}


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "ref_full_shape.npz"))


@pytest.fixture(scope="module")
def synth(tmp_path_factory):
    import synthetic_model as sm
    d = tmp_path_factory.mktemp("full_shape")
    made = {}

    def get(name):
        if name not in made:
            preset, fmt, seed = CASES[name]
            shared = os.path.join(os.environ.get("RWKV_B200_BENCH_DIR", "/tmp/rwkv_b200_bench"), f"{preset}-{fmt}-seed{seed}.bin")
            if os.path.isfile(shared):                # bench.py's cache: the same generator, the same seed
                made[name] = shared
            else:
                path = str(d / f"{preset}-{fmt}.bin")
                sm.write_direct(path, preset, fmt, seed=seed)
                made[name] = path
        return made[name]
    return get


def eval_serial(lib, ctx, toks, n_state, n_logits, logits_every=1):
    state = np.zeros(n_state, np.float32)
    logits = np.zeros(n_logits, np.float32)
    for i, t in enumerate(toks):
        want = (i + 1) % logits_every == 0 or i == len(toks) - 1
        assert lib.library.rwkv_eval(ctx.ptr, int(t), None if i == 0 else state.ctypes.data_as(P_F), state.ctypes.data_as(P_F), logits.ctypes.data_as(P_F) if want else None)
    return logits, state


def tol_of(name):
    return TOL["FP16"] if name.endswith("FP16") else TOL["Q"]


@pytest.mark.parametrize("name", list(CASES))
def test_decode_matches_reference(lib, synth, golden, name):
    """n single-token rwkv_eval calls from a fresh state == the compiled reference on the same file and tokens."""
    ctx = lib.rwkv_init_from_file(synth(name), 1, 0)
    try:
        n_state, n_logits = lib.rwkv_get_state_buffer_element_count(ctx), lib.rwkv_get_logits_buffer_element_count(ctx)
        toks = golden[f"{name}/decode_tokens"]
        logits, state = eval_serial(lib, ctx, toks, n_state, n_logits)
        want = golden[f"{name}/decode_logits"]
        err = float(np.abs(logits - want).max())
        serr = float(np.abs(state[::STATE_STRIDE] - golden[f"{name}/decode_state_sample"]).max())
        print(f"{name}: decode max|ours - reference| logits {err:.3e} (|ref|max {np.abs(want).max():.2f}), state sample {serr:.3e}")
        assert np.isfinite(logits).all() and err <= tol_of(name), err
        assert serr <= 20 * tol_of(name), serr
        # sequence mode over the same tokens: bit-identical to serial below the tensor-core threshold
        if len(toks) < 32:
            arr = (ctypes.c_uint32 * len(toks))(*[int(t) for t in toks])
            s2, l2 = np.zeros(n_state, np.float32), np.zeros(n_logits, np.float32)
            assert lib.library.rwkv_eval_sequence(ctx.ptr, arr, len(toks), None, s2.ctypes.data_as(P_F), l2.ctypes.data_as(P_F))
            assert s2.tobytes() == state.tobytes() and l2.tobytes() == logits.tobytes()
    finally:
        lib.rwkv_free(ctx)


@pytest.mark.parametrize("name", [n for n in CASES if n in ("rwkv4-169m:Q5_1", "rwkv5-1b5:Q4_0", "rwkv6-7b:Q5_1")])
def test_chunked_prefill_matches_reference(lib, synth, golden, name):
    """One rwkv_eval_sequence_in_chunks call (chunk = 128: BASELINE.json config 2 and the headline prefill) == the compiled
    reference; the >= 32-token passes run the wgmma kernel. With the tensor cores off the same call must equal serial
    evaluation bit for bit (the reference's own contract, tests/test_eval_sequence_in_chunks.c:54)."""
    ctx = lib.rwkv_init_from_file(synth(name), 1, 0)
    try:
        n_state, n_logits = lib.rwkv_get_state_buffer_element_count(ctx), lib.rwkv_get_logits_buffer_element_count(ctx)
        toks = [int(t) for t in golden[f"{name}/chunk_tokens"]]
        arr = (ctypes.c_uint32 * len(toks))(*toks)
        want = golden[f"{name}/chunk_logits"]
        s, l = np.zeros(n_state, np.float32), np.zeros(n_logits, np.float32)
        assert lib.library.rwkv_eval_sequence_in_chunks(ctx.ptr, arr, len(toks), 128, None, s.ctypes.data_as(P_F), l.ctypes.data_as(P_F))
        err = float(np.abs(l - want).max())
        serr = float(np.abs(s[::STATE_STRIDE] - golden[f"{name}/chunk_state_sample"]).max())
        print(f"{name}: {len(toks)}-token chunk (tensor cores) max|ours - reference| logits {err:.3e}, state sample {serr:.3e}")
        assert np.isfinite(l).all() and np.isfinite(s).all()
        assert err <= tol_of(name), err
        assert serr <= 20 * tol_of(name), serr
        lib.library.rwkv_b200_set_tensor_cores(ctx.ptr, False)
        s0, l0 = np.zeros(n_state, np.float32), np.zeros(n_logits, np.float32)
        assert lib.library.rwkv_eval_sequence_in_chunks(ctx.ptr, arr, len(toks), 128, None, s0.ctypes.data_as(P_F), l0.ctypes.data_as(P_F))
        l1, s1 = eval_serial(lib, ctx, toks, n_state, n_logits, logits_every=10 ** 6)
        assert s0.tobytes() == s1.tobytes() and l0.tobytes() == l1.tobytes()
        err0 = float(np.abs(l0 - want).max())
        print(f"{name}: same chunk on the batch-invariant path: logits {err0:.3e}; tensor-core vs batch-invariant {float(np.abs(l - l0).max()):.3e}")
        assert err0 <= tol_of(name), err0
    finally:
        lib.rwkv_free(ctx)


@pytest.mark.parametrize("name", ["rwkv4-169m:Q5_1", "rwkv5-1b5:Q4_0", "rwkv7-2b9:FP16"])
def test_full_shape_invariants(lib, synth, name):
    import synthetic_model as sm
    ctx = lib.rwkv_init_from_file(synth(name), 1, 0)
    try:
        n_state, n_logits = lib.rwkv_get_state_buffer_element_count(ctx), lib.rwkv_get_logits_buffer_element_count(ctx)
        toks = sm.synthetic_tokens(24, n_logits)
        arr = (ctypes.c_uint32 * len(toks))(*toks)
        lib.library.rwkv_b200_set_overlap(ctx.ptr, False)
        logits, state = eval_serial(lib, ctx, toks, n_state, n_logits)
        assert np.isfinite(logits).all() and np.isfinite(state).all() and logits.std() > 0
        s2, l2 = np.zeros(n_state, np.float32), np.zeros(n_logits, np.float32)
        assert lib.library.rwkv_eval_sequence(ctx.ptr, arr, len(toks), None, s2.ctypes.data_as(P_F), l2.ctypes.data_as(P_F))
        assert s2.tobytes() == state.tobytes() and l2.tobytes() == logits.tobytes()
        for chunk in (1, 5, 10):
            s3, l3 = np.zeros(n_state, np.float32), np.zeros(n_logits, np.float32)
            assert lib.library.rwkv_eval_sequence_in_chunks(ctx.ptr, arr, len(toks), chunk, None, s3.ctypes.data_as(P_F), l3.ctypes.data_as(P_F))
            assert s3.tobytes() == state.tobytes() and l3.tobytes() == logits.tobytes(), chunk
        l4, s4 = eval_serial(lib, ctx, toks, n_state, n_logits, logits_every=4)     # logits only every 4th token
        assert s4.tobytes() == state.tobytes() and l4.tobytes() == logits.tobytes()
        l5, s5 = eval_serial(lib, ctx, toks[:10], n_state, n_logits)                # a clone picks the sequence up in the middle
        clone = lib.rwkv_clone_context(ctx, 1)
        for t in toks[10:]:
            assert lib.library.rwkv_eval(clone.ptr, t, s5.ctypes.data_as(P_F), s5.ctypes.data_as(P_F), l5.ctypes.data_as(P_F))
        lib.rwkv_free(clone)
        assert s5.tobytes() == state.tobytes() and l5.tobytes() == logits.tobytes()
        lib.library.rwkv_b200_set_overlap(ctx.ptr, True)                            # host state copied per layer group (the default)
        l6, s6 = eval_serial(lib, ctx, toks, n_state, n_logits)
        assert s6.tobytes() == state.tobytes() and l6.tobytes() == logits.tobytes()
    finally:
        lib.rwkv_free(ctx)
