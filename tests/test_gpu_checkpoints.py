"""Checkpoints (rwkv_b200_eval_checkpoints, rwkv_b200_batch_eval_ragged_checkpoints): the state after chosen tokens of a pass.

Where passes are bit-identical to serial evaluation (tensor cores off, or passes that never take them) every checkpoint must equal the
state after rwkv_eval of its prefix, bit for bit. Everywhere, asking for checkpoints must change nothing else: resident state, logits and
the kernel launch count equal the plain call's, bit for bit.
"""
import ctypes

import numpy as np
import pytest

from conftest import VERSIONS, model_path

pytestmark = pytest.mark.gpu

P_F = ctypes.POINTER(ctypes.c_float)
P_U = ctypes.POINTER(ctypes.c_uint32)
ERR_ARGS, ERR_CTX_UNSUPPORTED = 1 << 8, (6 << 8) | 9
POSITIONS = [0, 1, 7, 8, 9, 31, 32, 255, 256, 299]    # both sides of a wkv6 chunk and of a two-token trip, a pass end, the last token
STATE_BAR = 1.5e-1                                    # test_gpu_interleave.py's bar for passes on the tensor cores, relative to max(1, |state|)


def fp(a):
    return a.ctypes.data_as(P_F)


def u32(x):
    return np.ascontiguousarray(x, np.uint32)


def tokens_for(n, V, seed=0):
    return [int(t) for t in np.random.default_rng(seed).integers(0, V, n)]


class Ctx:
    def __init__(self, lib, path, tc=True):
        self.lib, self.L = lib, lib.library
        self.c = lib.rwkv_init_from_file(path, 1)
        self.n = lib.rwkv_get_state_len(self.c)
        self.V = lib.rwkv_get_n_vocab(self.c)
        self.L.rwkv_b200_set_tensor_cores(self.c.ptr, tc)
        self.load()        # a new context's resident state is undefined until it is loaded

    def state(self):
        s = np.empty(self.n, np.float32)
        assert self.L.rwkv_b200_state_store(self.c.ptr, fp(s))
        return s

    def load(self, s=None):
        assert self.L.rwkv_b200_state_load(self.c.ptr, fp(s) if s is not None else None)

    def plain(self, toks, want=True):
        logits = np.empty(self.V, np.float32)
        arr = u32(toks)
        assert self.L.rwkv_b200_eval_resident(self.c.ptr, arr.ctypes.data_as(P_U), len(toks), want, fp(logits) if want else None)
        return logits

    def checkpoints(self, toks, positions, want=True, out=None):
        logits = np.empty(self.V, np.float32)
        cps = self.lib.rwkv_b200_eval_checkpoints(self.c, toks, positions, want, out, logits.ctypes.data if want else 0)
        return cps, logits

    def close(self):
        self.lib.rwkv_free(self.c)


def serial_states(lib, path, toks, positions, base=None, adapter=None):
    """The state after rwkv_eval of tokens[0 .. p], one token at a time, for every p of positions; with an adapter, on a clone of the
    context `base` (whose model the adapter belongs to) with the adapter attached."""
    if adapter is None:
        c = Ctx(lib, path)
    else:
        c = Ctx.__new__(Ctx)
        c.lib, c.L, c.n, c.V = lib, lib.library, base.n, base.V
        c.c = lib.rwkv_clone_context(base.c, 1)
        lib.rwkv_b200_set_adapter(c.c, adapter)
    st, out, logits, res = None, np.empty(c.n, np.float32), np.empty(c.V, np.float32), {}
    for i, t in enumerate(toks[:max(positions) + 1]):
        assert c.L.rwkv_eval(c.c.ptr, t, fp(st) if st is not None else None, fp(out), fp(logits))
        st = out.copy()
        if i in positions:
            res[i] = st
    c.close()
    return res


def assert_bits(got, want, what):
    assert got.tobytes() == want.tobytes(), f"{what}: max |diff| {float(np.abs(got - want).max())}"


def q4k_file(tmp_path_factory):
    import synthetic_model as sm
    path = str(tmp_path_factory.mktemp("cp") / "rwkv6-small-Q4_K.bin")
    sm.write_direct(path, "rwkv6-small", "Q4_K", seed=5)
    return path


FILES = [(v, f) for v in VERSIONS for f in ("FP32", "Q5_1")] + [("6v0-3m", "FP16")]


@pytest.fixture(scope="module")
def q4k(tmp_path_factory):
    return q4k_file(tmp_path_factory)


@pytest.mark.parametrize("ver,fmt", FILES + [("Q4_K", None)], ids=[f"{v}-{f}" for v, f in FILES] + ["synthetic-Q4_K"])
def test_serial_bits_with_tensor_cores_off(lib, q4k, ver, fmt):
    path = q4k if ver == "Q4_K" else model_path(ver, fmt)
    c = Ctx(lib, path, tc=False)
    toks = tokens_for(300, c.V, 1)
    short = [0, 1, 7, 8, 9, 30]
    want = serial_states(lib, path, toks, POSITIONS + short)
    cps, _ = c.checkpoints(toks, POSITIONS)
    for i, p in enumerate(POSITIONS):
        assert_bits(cps[i], want[p], f"{ver} {fmt} position {p}")
    assert_bits(c.state(), want[299], "resident state")
    # with the tensor cores on, passes below 32 tokens stay on the bit-exact route
    c.L.rwkv_b200_set_tensor_cores(c.c.ptr, True)
    c.load()
    cps, _ = c.checkpoints(toks[:31], short)
    for i, p in enumerate(short):
        assert_bits(cps[i], want[p], f"{ver} {fmt} tc on, 31 tokens, position {p}")
    c.close()


@pytest.mark.parametrize("ver,fmt", [("4v0-660K", "Q5_1"), ("5v2-730K", "Q5_1"), ("6v0-3m", "Q5_1"), ("7v0-834K", "FP16"), ("Q4_K", None)])
@pytest.mark.parametrize("n", [70, 300])
def test_nothing_else_moves_with_tensor_cores_on(lib, q4k, ver, fmt, n):
    path = q4k if ver == "Q4_K" else model_path(ver, fmt)
    a, b = Ctx(lib, path), Ctx(lib, path)
    toks = tokens_for(n, a.V, 2)
    pos = [p for p in POSITIONS if p < n - 1] + [n - 1]
    k0 = lib.library.rwkv_b200_kernel_launch_count()
    want_logits = a.plain(toks)
    k1 = lib.library.rwkv_b200_kernel_launch_count()
    cps, logits = b.checkpoints(toks, pos)
    k2 = lib.library.rwkv_b200_kernel_launch_count()
    assert k2 - k1 == k1 - k0, "checkpoints changed the number of kernel launches"
    assert_bits(logits, want_logits, "logits")
    assert_bits(b.state(), a.state(), "resident state")
    assert_bits(cps[-1], b.state(), "the last checkpoint against rwkv_b200_state_store")
    serial = serial_states(lib, path, toks, pos)
    for i, p in enumerate(pos):
        w = serial[p]
        d, bar = float(np.abs(cps[i] - w).max()), STATE_BAR * max(1.0, float(np.abs(w).max()))
        assert d <= bar, f"position {p}: {d} > {bar}"
    a.close(), b.close()


@pytest.mark.parametrize("ver,fmt", [("6v0-3m", "Q5_1"), ("7v0-834K", "FP32"), ("4v0-660K", "FP32")])
def test_round_trip(lib, ver, fmt):
    """A checkpoint loaded into a context, or put into another batch slot, continues as the uninterrupted call (tensor cores off)."""
    path = model_path(ver, fmt)
    full, part = Ctx(lib, path, tc=False), Ctx(lib, path, tc=False)
    toks = tokens_for(300, full.V, 3)
    want_logits = full.plain(toks)
    want_state = full.state()
    cps, _ = part.checkpoints(toks, [100])
    part.load(cps[0])
    logits = part.plain(toks[101:])
    assert_bits(logits, want_logits, "logits after state_load")
    assert_bits(part.state(), want_state, "state after state_load")
    B = 3
    batch = lib.library.rwkv_b200_batch_create(full.c.ptr, B)
    assert batch
    lib.library.rwkv_b200_set_tensor_cores(batch, False)
    assert lib.library.rwkv_b200_batch_set_state(batch, 2, fp(cps[0]))
    rest = u32(toks[101:])
    counts = u32([0, 0, len(rest)])
    assert lib.library.rwkv_b200_batch_eval_ragged(batch, rest.ctypes.data_as(P_U), counts.ctypes.data_as(P_U), True)
    st, lg = np.empty(full.n, np.float32), np.empty(full.V, np.float32)
    assert lib.library.rwkv_b200_batch_get_state(batch, 2, fp(st)) and lib.library.rwkv_b200_batch_get_logits(batch, 2, fp(lg))
    assert_bits(st, want_state, "state after batch_set_state")
    assert_bits(lg, want_logits, "logits after batch_set_state")
    lib.library.rwkv_free(batch)
    full.close(), part.close()


class Batch:
    def __init__(self, lib, base, B, tc):
        self.lib, self.L, self.B = lib, lib.library, B
        self.b = self.L.rwkv_b200_batch_create(base.c.ptr, B)
        assert self.b
        self.ctx = type(base.c)(self.b)
        self.L.rwkv_b200_set_tensor_cores(self.b, tc)
        self.n, self.V = base.n, base.V

    def ragged(self, toks, counts):
        t, c = u32(toks if len(toks) else [0]), u32(counts)
        assert self.L.rwkv_b200_batch_eval_ragged(self.b, t.ctypes.data_as(P_U), c.ctypes.data_as(P_U), True)

    def states(self):
        out = np.empty((self.B, self.n), np.float32)
        for s in range(self.B):
            assert self.L.rwkv_b200_batch_get_state(self.b, s, fp(out[s]))
        return out

    def logits(self):
        out = np.empty((self.B, self.V), np.float32)
        for s in range(self.B):
            assert self.L.rwkv_b200_batch_get_logits(self.b, s, fp(out[s]))
        return out


# the counts of four consecutive calls: decoding sequences, prompts and an idle slot; sums 7, 21, 8 and 31, on both sides of 16
RAGGED_CALLS = [[2, 3, 0, 1, 1], [3, 12, 0, 5, 1], [1, 4, 0, 2, 1], [1, 20, 0, 9, 1]]


def ragged_checkpoints(counts):
    cps = []
    for s, n in enumerate(counts):
        for p in sorted({0, n // 2, n - 1}):
            if n and p < n:
                cps.append((s, p))
    return cps


def make_adapter(lib, base, seed):
    ctx = base.c
    C = lib.rwkv_get_n_embed(ctx)
    rng = np.random.default_rng(seed)
    a = rng.standard_normal((2, C)).astype(np.float32) * 0.1
    b = rng.standard_normal((C, 2)).astype(np.float32) * 0.1
    return lib.rwkv_b200_adapter_create(ctx, [("blocks.0.att.key.weight", 2, a, b, None), ("blocks.0.att.output.weight", 2, a, b, None)], 1.0)


@pytest.mark.parametrize("tc", [False, True], ids=["tc-off", "tc-on"])
@pytest.mark.parametrize("adapters", ["none", "per-sequence", "context-wide"])
@pytest.mark.parametrize("ver,fmt", [("6v0-3m", "Q5_1"), ("7v0-834K", "FP32"), ("5v2-730K", "Q5_1"), ("4v0-660K", "Q5_1")])
def test_ragged(lib, ver, fmt, tc, adapters):
    path = model_path(ver, fmt)
    base = Ctx(lib, path, tc=False)
    B = 5
    plain, snap = Batch(lib, base, B, tc), Batch(lib, base, B, tc)
    ads, adapter_of = [], [None] * B
    if adapters != "none":
        ads = [make_adapter(lib, base, 7), make_adapter(lib, base, 8)]
        adapter_of = [None, ads[0], None, ads[1], None] if adapters == "per-sequence" else [ads[0]] * B
        for bb in (plain, snap):
            if adapters == "per-sequence":
                assert lib.library.rwkv_b200_batch_set_adapter(bb.b, 1, ads[0]) and lib.library.rwkv_b200_batch_set_adapter(bb.b, 3, ads[1])
            else:
                assert lib.library.rwkv_b200_set_adapter(bb.b, ads[0])
    history = {s: [] for s in range(B)}
    exact = True
    for k, counts in enumerate(RAGGED_CALLS):
        seqs = [tokens_for(n, base.V, 10 * k + s) for s, n in enumerate(counts)]
        toks = [t for q in seqs for t in q]
        before_idle = snap.states()[2]
        plain.ragged(toks, counts)
        entries = ragged_checkpoints(counts)
        cps = lib.rwkv_b200_batch_eval_ragged_checkpoints(snap.ctx, toks, counts, entries, True)
        assert_bits(snap.states(), plain.states(), f"states after call {k}")
        assert_bits(snap.logits(), plain.logits(), f"logits after call {k}")
        assert_bits(snap.states()[2], before_idle, "the idle sequence")
        for s in range(B):
            history[s] += seqs[s]
        exact = exact and (not tc or sum(counts) < 16)
        if exact:      # every pass so far was bit-identical to serial evaluation: compare every checkpoint with it
            for i, (s, p) in enumerate(entries):
                prefix = history[s][:len(history[s]) - counts[s] + p + 1]
                want = serial_states(lib, path, prefix, [len(prefix) - 1], base, adapter_of[s])[len(prefix) - 1]
                assert_bits(cps[i], want, f"call {k} sequence {s} position {p}")
        for i, (s, p) in enumerate(entries):
            if p == counts[s] - 1:
                assert_bits(cps[i], snap.states()[s], f"the last checkpoint of sequence {s}")
    for bb in (plain, snap):
        lib.library.rwkv_free(bb.b)
    for a in ads:
        lib.rwkv_b200_adapter_free(a)
    base.close()


def test_destinations_give_the_same_bytes(lib):
    import torch
    path = model_path("6v0-3m", "Q5_1")
    c = Ctx(lib, path)
    toks = tokens_for(300, c.V, 4)
    pos = [5, 100, 255, 299]
    host, _ = c.checkpoints(toks, pos)
    outs = {"pinned": [torch.empty(c.n, dtype=torch.float32).pin_memory() for _ in pos],
            "device": [torch.empty(c.n, dtype=torch.float32, device="cuda:0") for _ in pos],
            "mixed": [torch.empty(c.n, dtype=torch.float32, device="cuda:0"), np.empty(c.n, np.float32),
                      torch.empty(c.n, dtype=torch.float32).pin_memory(), np.empty(c.n, np.float32)],
            # device and host memory at a 4-byte offset: wkv6_kernel stores float4s, so these go through the staging
            "unaligned": [torch.empty(c.n + 1, dtype=torch.float32, device="cuda:0")[1:], np.empty(c.n + 1, np.float32)[1:],
                          torch.empty(c.n + 3, dtype=torch.float32, device="cuda:0")[3:], torch.empty(c.n + 2, dtype=torch.float32, device="cuda:0")[2:]]}
    for kind, out in outs.items():
        c.load()
        c.checkpoints(toks, pos, out=out)
        torch.cuda.synchronize()
        for i in range(len(pos)):
            got = out[i].cpu().numpy() if hasattr(out[i], "cpu") else out[i]
            assert_bits(got, host[i], f"{kind} destination {i}")
    c.close()


SHAPE_FILES = ["rwkv4-169m", "rwkv4-14b", "rwkv5-0b4", "rwkv6-7b", "rwkv7-0b1", "rwkv7-0b4-S128"]


@pytest.fixture(scope="module")
def shape_files(tmp_path_factory):
    import synthetic_model as sm
    import test_gpu_model_shapes as ms
    d = tmp_path_factory.mktemp("cp-shapes")
    files = {}
    for name in SHAPE_FILES:
        s = ms.BY_NAME[name.replace("-S128", "")]
        p = ms.preset(s, L=1, V=1024)
        if name.endswith("S128"):
            p["S"] = 128
        files[name] = str(d / f"{name}.bin")
        sm.write_direct(files[name], p, "Q5_1", seed=3)
    return files


@pytest.mark.parametrize("name", SHAPE_FILES)
def test_model_shapes_serial_bits(lib, shape_files, name):
    """One-layer files at published shapes: wkv6 S = 64 with the 7B head count, wkv7 S = 64 and 128, the LayerNorm kernels of 4 and 8
    channels per thread (n_embed 4096 and 5120). Batch contexts take n_embed up to 4096, so the 14B shape has no ragged part."""
    path = shape_files[name]
    c = Ctx(lib, path, tc=False)
    toks = tokens_for(40, c.V, 6)
    pos = [0, 1, 7, 8, 9, 19, 20, 39]
    want = serial_states(lib, path, toks, pos)
    cps, _ = c.checkpoints(toks, pos)
    for i, p in enumerate(pos):
        assert_bits(cps[i], want[p], f"{name} position {p}")
    if lib.rwkv_get_n_embed(c.c) > 4096:
        c.close()
        return
    b = Batch(lib, c, 2, False)
    cps = lib.rwkv_b200_batch_eval_ragged_checkpoints(b.ctx, toks[:20] + toks[:3], [20, 3], [(0, 8), (0, 19), (1, 1)], True)
    for i, p in enumerate([8, 19, 1]):
        assert_bits(cps[i], want[p], f"{name} ragged checkpoint {i}")
    lib.library.rwkv_free(b.b)
    c.close()


def test_graph_replay_after_a_checkpoint_call(lib):
    path = model_path("6v0-3m", "Q5_1")
    a, b = Ctx(lib, path), Ctx(lib, path)
    toks = tokens_for(60, a.V, 8)
    for c in (a, b):
        for t in toks[:3]:
            c.plain([t])       # the second use of a slot captures its graph
    a.plain(toks[3:50])
    b.checkpoints(toks[3:50], [4, 20, 46])
    g0 = lib.library.rwkv_b200_graph_launch_count()
    la = [a.plain([t]) for t in toks[50:54]]
    g1 = lib.library.rwkv_b200_graph_launch_count()
    lb = [b.plain([t]) for t in toks[50:54]]
    g2 = lib.library.rwkv_b200_graph_launch_count()
    assert g2 - g1 == g1 - g0 > 0
    for x, y in zip(la, lb):
        assert_bits(y, x, "decode logits")
    assert_bits(b.state(), a.state(), "state")
    # a single-token call with its checkpoint at its end replays the graph too
    g3 = lib.library.rwkv_b200_graph_launch_count()
    cps, lg = b.checkpoints([toks[54]], [0])
    assert lib.library.rwkv_b200_graph_launch_count() == g3 + 1
    assert_bits(lg, a.plain([toks[54]]), "single-token logits")
    assert_bits(cps[0], a.state(), "single-token checkpoint")
    a.close(), b.close()


def test_refusals_change_nothing(lib):
    path = model_path("6v0-3m", "Q5_1")
    c = Ctx(lib, path)
    toks = tokens_for(40, c.V, 9)
    c.plain(toks[:5])
    st0 = c.state()
    lg0 = np.empty(c.V, np.float32)
    n = c.n
    bufs = np.zeros((4, n), np.float32)
    arr = u32(toks)
    import rwkv_cpp_b200.shared_library as sl

    def call(entries, n_tokens=40, null_cp=False):
        a = (sl.Checkpoint * max(1, len(entries)))()
        for i, (s, p, ptr) in enumerate(entries):
            a[i] = sl.Checkpoint(s, p, ctypes.cast(ptr, P_F))
        ok = lib.library.rwkv_b200_eval_checkpoints(c.c.ptr, arr.ctypes.data_as(P_U), n_tokens, True, None, None if null_cp else a, len(entries))
        return ok, lib.rwkv_get_last_error(c.c)

    b0, b1, b2 = (bufs[i].ctypes.data for i in range(3))
    cases = [([(0, 1, b0)], True, "NULL cp"), ([(0, 1, 0)], False, "NULL state_out"), ([(0, 3, b0), (0, 2, b1)], False, "order"),
             ([(0, 3, b0), (0, 3, b1)], False, "repeat"), ([(0, 40, b0)], False, "position"), ([(1, 3, b0)], False, "sequence"),
             ([(0, 1, b0), (0, 2, b0 + 4 * (n - 1))], False, "overlap")]
    for entries, null_cp, what in cases:
        ok, err = call(entries, null_cp=null_cp)
        assert not ok and err == ERR_ARGS, (what, err)
        assert_bits(c.state(), st0, what)
    # the wrong kind of context
    batch = lib.library.rwkv_b200_batch_create(c.c.ptr, 2)
    a = (sl.Checkpoint * 1)(sl.Checkpoint(0, 1, ctypes.cast(b0, P_F)))
    assert not lib.library.rwkv_b200_eval_checkpoints(batch, arr.ctypes.data_as(P_U), 4, True, None, a, 1)
    assert lib.library.rwkv_get_last_error(batch) == ERR_CTX_UNSUPPORTED
    counts = u32([2, 2])
    assert not lib.library.rwkv_b200_batch_eval_ragged_checkpoints(c.c.ptr, arr.ctypes.data_as(P_U), counts.ctypes.data_as(P_U), True, a, 1)
    assert lib.rwkv_get_last_error(c.c) == ERR_CTX_UNSUPPORTED
    a2 = (sl.Checkpoint * 1)(sl.Checkpoint(1, 2, ctypes.cast(b0, P_F)))
    assert not lib.library.rwkv_b200_batch_eval_ragged_checkpoints(batch, arr.ctypes.data_as(P_U), counts.ctypes.data_as(P_U), True, a2, 1)
    assert lib.library.rwkv_get_last_error(batch) == ERR_ARGS
    lib.library.rwkv_free(batch)
    # the logits of the last pass are still there and valid: a one-token eval from the stored state gives the same as a twin
    assert_bits(c.state(), st0, "after refusals")
    twin = Ctx(lib, path)
    twin.plain(toks[:5])
    assert_bits(c.plain(toks[5:6]), twin.plain(toks[5:6]), "logits after refusals")
    twin.close()
    import torch
    if torch.cuda.device_count() < 2:
        c.close()
        pytest.skip("a device pointer of another device needs a second GPU")
    other = torch.empty(n, dtype=torch.float32, device="cuda:1")
    ok, err = call([(0, 3, other.data_ptr())])
    assert not ok and err == ERR_ARGS
    c.close()


def test_refused_inside_a_streaming_callback(lib):
    path = model_path("6v0-3m", "Q5_1")
    c = Ctx(lib, path)
    c.plain([1, 2, 3])
    import rwkv_cpp_b200.shared_library as sl
    seen = []
    buf = np.zeros(c.n, np.float32)

    def on_token(user, seq, index, token):
        a = (sl.Checkpoint * 1)(sl.Checkpoint(0, 0, ctypes.cast(buf.ctypes.data, P_F)))
        t = u32([token])
        seen.append((lib.library.rwkv_b200_eval_checkpoints(c.c.ptr, t.ctypes.data_as(P_U), 1, False, None, a, 1),
                     lib.library.rwkv_get_last_error(c.c.ptr)))
        return 1
    cb = sl.RWKV_TOKEN_FN(on_token)
    out = np.zeros(4, np.uint32)
    n_gen = ctypes.c_size_t(0)
    u = np.full(4, 0.5)
    lib.library.rwkv_b200_generate_stream(c.c.ptr, 4, 1.0, 1.0, 0.0, 0.0, False, u.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), None, 0,
                                          cb, None, out.ctypes.data_as(P_U), ctypes.byref(n_gen))
    assert seen and all(not ok and err == ERR_CTX_UNSUPPORTED for ok, err in seen), seen
    c.close()
