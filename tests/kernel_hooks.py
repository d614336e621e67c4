"""ctypes bindings of the kernel test hooks (rwkv_b200_test_* in include/rwkv_b200.h). Activations go in and come out as numpy
[dim, T] arrays; every output comes back with the guard region the hook returns, so a test can tell a value the kernel never wrote
(still NaN from the 0xFF fill) and a write past the end (a guard byte that is no longer 0xFF) from a wrong value."""
import ctypes

import numpy as np

from kernel_ref import staged_bytes

GUARD = 64            # RWKV_B200_GUARD: floats after the end of every output
GUARD_BYTES = 4 * GUARD
VP = ctypes.c_void_p
F6, P5, I5 = VP * 6, VP * 5, ctypes.c_int * 5


class LnMixArgs(ctypes.Structure):
    _fields_ = [("x", VP), ("ln_w", VP), ("ln_b", VP), ("state_in", VP), ("state_out", VP), ("C", ctypes.c_int), ("T", ctypes.c_int),
                ("formula", ctypes.c_int), ("n_out", ctypes.c_int), ("coef", F6), ("out", F6), ("out_xx", VP), ("out_sx", VP),
                ("n_seq", ctypes.c_int), ("seq_stride", ctypes.c_longlong)]


class V6LerpArgs(ctypes.Structure):
    _fields_ = [("w2", VP), ("z", VP), ("xx", VP), ("sx", VP), ("maa", P5), ("out", P5), ("C", ctypes.c_int), ("T", ctypes.c_int),
                ("mix", ctypes.c_int), ("q_out", P5), ("q_type", I5)]


class Wkv4Args(ctypes.Structure):
    _fields_ = [("k", VP), ("v", VP), ("r", VP), ("time_first", VP), ("time_decay", VP), ("aa_in", VP), ("bb_in", VP), ("pp_in", VP),
                ("aa_out", VP), ("bb_out", VP), ("pp_out", VP), ("y", VP), ("C", ctypes.c_int), ("T", ctypes.c_int), ("q_out", VP),
                ("q_type", ctypes.c_int), ("n_seq", ctypes.c_int), ("seq_stride", ctypes.c_longlong)]


class Wkv6Args(ctypes.Structure):
    _fields_ = [("r", VP), ("k", VP), ("v", VP), ("td", VP), ("tf", VP), ("td_per_token", ctypes.c_int), ("per_head_scalars", ctypes.c_int),
                ("state_in", VP), ("state_out", VP), ("lnx_w", VP), ("lnx_b", VP), ("g", VP), ("y", VP), ("eps", ctypes.c_float),
                ("H", ctypes.c_int), ("S", ctypes.c_int), ("T", ctypes.c_int), ("q_out", VP), ("q_type", ctypes.c_int),
                ("n_seq", ctypes.c_int), ("seq_stride", ctypes.c_longlong)]


class Wkv7Args(ctypes.Structure):
    _fields_ = [("r", VP), ("w", VP), ("k", VP), ("v", VP), ("a", VP), ("g", VP), ("vgate", VP), ("v_first", VP), ("v_out", VP),
                ("k_k", VP), ("k_a", VP), ("r_k", VP), ("lnx_w", VP), ("lnx_b", VP), ("state_in", VP), ("state_out", VP), ("y", VP),
                ("H", ctypes.c_int), ("S", ctypes.c_int), ("T", ctypes.c_int), ("q_out", VP), ("q_type", ctypes.c_int),
                ("n_seq", ctypes.c_int), ("seq_stride", ctypes.c_longlong)]


class HookError(RuntimeError):
    def __init__(self, flags):
        super().__init__("kernel hook failed, error flags 0x%x" % flags)
        self.flags = flags


class Out:
    """A host output buffer of n elements plus the guard region (GUARD_BYTES bytes)."""

    def __init__(self, n, dtype=np.float32):
        self.n = n
        self.buf = np.zeros(n + GUARD_BYTES // np.dtype(dtype).itemsize, dtype)

    @property
    def ptr(self):
        return self.buf.ctypes.data

    @property
    def value(self):
        return self.buf[:self.n]

    def cols(self, C):
        """The value as a [C, T] array."""
        return self.value.reshape(-1, C).T

    def guard_intact(self):
        return bool((self.buf[self.n:].view(np.uint8) == 0xFF).all())


class Inputs:
    """Keeps the contiguous float32 copies of the inputs alive for the duration of a call."""

    def __init__(self):
        self.keep = []

    def __call__(self, a, columns=False):
        if a is None:
            return None
        a = np.ascontiguousarray(a.T if columns else a, np.float32)    # [C, T] -> column t contiguous
        self.keep.append(a)
        return a.ctypes.data


def _call(lib, fn, args):
    if not fn(ctypes.byref(args)):
        raise HookError(lib.rwkv_get_last_error(None))


def embed_ln0(lib, emb, tokens, w, b):
    """emb: [n_vocab, C] float32 or float16 table. Returns Out of C*T floats."""
    n_vocab, C = emb.shape
    emb = np.ascontiguousarray(emb)
    tok = np.ascontiguousarray(tokens, np.int32)
    w, b = np.ascontiguousarray(w, np.float32), np.ascontiguousarray(b, np.float32)
    x = Out(C * tok.size)
    ok = lib.library.rwkv_b200_test_embed_ln0(VP(emb.ctypes.data), ctypes.c_int(0 if emb.dtype == np.float32 else 1), ctypes.c_size_t(emb.strides[0]),
                                              ctypes.c_int(n_vocab), VP(tok.ctypes.data), ctypes.c_int(tok.size), ctypes.c_int(C), VP(w.ctypes.data),
                                              VP(b.ctypes.data), VP(x.ptr))
    if not ok:
        raise HookError(lib.rwkv_get_last_error(None))
    return x


def layer_norm_columns(lib, x, w, b):
    """x: [C, T]; w, b: [C] (None passes NULL). Returns Out of C*T floats: LN(x[:, t]; w, b) of every column."""
    C, T = x.shape
    i = Inputs()
    y = Out(C * T)
    ok = lib.library.rwkv_b200_test_layer_norm_columns(VP(i(x, True)), VP(i(w)), VP(i(b)), ctypes.c_int(C), ctypes.c_int(T), VP(y.ptr))
    if not ok:
        raise HookError(lib.rwkv_get_last_error(None))
    return y


def ln_mix(lib, x, w, b, state_in, coefs, formula, n_seq=0, seq_stride=0, xx=True, sx=True):
    """x: [C, T] (or [C, n_seq] with n_seq > 0, state_in then holding n_seq states seq_stride floats apart).
    Returns dict of Out: out0.., xx, sx, state."""
    C, cols = x.shape
    i = Inputs()
    a = LnMixArgs(x=i(x, True), ln_w=i(w), ln_b=i(b), state_in=i(state_in), C=C, T=1 if n_seq else cols, formula=formula, n_out=len(coefs),
                  n_seq=n_seq, seq_stride=seq_stride)
    o = {"state": Out(state_in.size)}
    a.state_out = o["state"].ptr
    for j, m in enumerate(coefs):
        o["out%d" % j] = Out(C * cols)
        a.coef[j], a.out[j] = i(m), o["out%d" % j].ptr
    if xx:
        o["xx"] = Out(C * cols)
        a.out_xx = o["xx"].ptr
    if sx:
        o["sx"] = Out(C * cols)
        a.out_sx = o["sx"].ptr
    _call(lib, lib.library.rwkv_b200_test_ln_mix, a)
    return o


def v6_lerp(lib, w2, z, xx, sx, maa, q_types=None):
    """w2: [5, C, mix]; z: [5*mix, T]; maa: [5, C]. Returns dict of Out: out0..out4 and q0..q4 when q_types is given."""
    _, C, mix = w2.shape
    T = z.shape[1]
    i = Inputs()
    a = V6LerpArgs(w2=i(w2), z=i(z, True), xx=i(xx, True), sx=i(sx, True), C=C, T=T, mix=mix)
    o = {}
    for j in range(5):
        o["out%d" % j] = Out(C * T)
        a.maa[j], a.out[j] = i(maa[j]), o["out%d" % j].ptr
        if q_types is not None:
            o["q%d" % j] = Out(staged_bytes(q_types[j], C), np.uint8)
            a.q_out[j], a.q_type[j] = o["q%d" % j].ptr, q_types[j]
    _call(lib, lib.library.rwkv_b200_test_v6_lerp, a)
    return o


def _staged(o, a, q_type, K):
    if q_type is not None:
        o["q"] = Out(staged_bytes(q_type, K), np.uint8)
        a.q_out, a.q_type = o["q"].ptr, q_type


def wkv4(lib, k, v, r, tf, td, aa, bb, pp, n_seq=0, seq_stride=0, q_type=None):
    C, cols = k.shape
    i = Inputs()
    a = Wkv4Args(k=i(k, True), v=i(v, True), r=i(r, True), time_first=i(tf), time_decay=i(td), aa_in=i(aa), bb_in=i(bb), pp_in=i(pp), C=C,
                 T=1 if n_seq else cols, n_seq=n_seq, seq_stride=seq_stride)
    o = {"aa": Out(aa.size), "bb": Out(bb.size), "pp": Out(pp.size), "y": Out(C * cols)}
    a.aa_out, a.bb_out, a.pp_out, a.y = o["aa"].ptr, o["bb"].ptr, o["pp"].ptr, o["y"].ptr
    _staged(o, a, q_type, C)
    _call(lib, lib.library.rwkv_b200_test_wkv4, a)
    return o


def wkv6(lib, r, k, v, td, tf, state, lnx_w, lnx_b, g, eps, H, S, td_per_token, per_head, n_seq=0, seq_stride=0, q_type=None):
    C, cols = r.shape
    i = Inputs()
    a = Wkv6Args(r=i(r, True), k=i(k, True), v=i(v, True), td=i(td, td_per_token), tf=i(tf), td_per_token=int(td_per_token),
                 per_head_scalars=int(per_head), state_in=i(state), lnx_w=i(lnx_w), lnx_b=i(lnx_b), g=i(g, True), eps=eps, H=H, S=S,
                 T=1 if n_seq else cols, n_seq=n_seq, seq_stride=seq_stride)
    o = {"state": Out(state.size), "y": Out(C * cols)}
    a.state_out, a.y = o["state"].ptr, o["y"].ptr
    _staged(o, a, q_type, C)
    _call(lib, lib.library.rwkv_b200_test_wkv6, a)
    return o


def wkv7(lib, r, w, k, v, aa, g, vgate, v_first, k_k, k_a, r_k, lnx_w, lnx_b, state, H, S, v_out=True, n_seq=0, seq_stride=0, q_type=None):
    C, cols = r.shape
    i = Inputs()
    a = Wkv7Args(r=i(r, True), w=i(w, True), k=i(k, True), v=i(v, True), a=i(aa, True), g=i(g, True), vgate=i(vgate, True),
                 v_first=i(v_first, True), k_k=i(k_k), k_a=i(k_a), r_k=i(r_k), lnx_w=i(lnx_w), lnx_b=i(lnx_b), state_in=i(state),
                 H=H, S=S, T=1 if n_seq else cols, n_seq=n_seq, seq_stride=seq_stride)
    o = {"state": Out(state.size), "y": Out(C * cols)}
    a.state_out, a.y = o["state"].ptr, o["y"].ptr
    if v_out:
        o["v"] = Out(C * cols)
        a.v_out = o["v"].ptr
    _staged(o, a, q_type, C)
    _call(lib, lib.library.rwkv_b200_test_wkv7, a)
    return o


class GemvProblem(ctypes.Structure):
    _fields_ = [("type", ctypes.c_int), ("K", ctypes.c_int), ("M", ctypes.c_int), ("weights", VP), ("tiled", ctypes.c_int), ("input", ctypes.c_int),
                ("epi", ctypes.c_int), ("pro", ctypes.c_int), ("res", VP), ("gate", VP), ("bias", VP), ("ln_w", VP), ("ln_b", VP), ("xq", VP),
                ("y_aliases_res", ctypes.c_int), ("y", VP)]


class GemvLaunch(ctypes.Structure):
    _fields_ = [(f, ctypes.c_int) for f in ("family", "nc", "only", "has_ln", "npad", "cluster")]


class GemvBatchArgs(ctypes.Structure):
    _fields_ = [("T", ctypes.c_int), ("n", ctypes.c_int), ("path", ctypes.c_int), ("x", VP * 8), ("p", GemvProblem * 8),
                ("launches", ctypes.POINTER(GemvLaunch)), ("max_launches", ctypes.c_int), ("n_launches", ctypes.POINTER(ctypes.c_int))]


GEMV_PATHS = {"engine": 0, "engine_batch_ctx": 1, "streaming": 2, "generic": 3, "tensor_cores": 4}
LAUNCH_FAMILIES = ("streaming", "generic", "tensor_cores", "convert", "expand", "kquant", "kquant_expand")


def _gemv_batch_args(T, problems, xs, path, i):
    a = GemvBatchArgs(T=T, n=len(problems), path=GEMV_PATHS[path])
    for j, x in enumerate(xs):
        a.x[j] = i(x, True)
    outs = []
    for j, p in enumerate(problems):
        raw = np.ascontiguousarray(p["raw"])
        i.keep.append(raw)
        q = a.p[j]
        q.type, q.K, q.M, q.weights = p["type"], p["K"], p["M"], raw.ctypes.data
        q.tiled, q.input, q.epi, q.pro = int(p.get("tiled", 0)), p.get("input", 0), p.get("epi", 0), p.get("pro", 0)
        q.res, q.gate = i(p.get("res"), True), i(p.get("gate"), True)
        q.bias, q.ln_w, q.ln_b = i(p.get("bias")), i(p.get("ln_w")), i(p.get("ln_b"))
        if p.get("xq") is not None:
            xq = np.ascontiguousarray(p["xq"], np.uint8)
            i.keep.append(xq)
            q.xq = xq.ctypes.data
        q.y_aliases_res = int(p.get("alias", 0))
        outs.append(Out(p["M"] * T))
        q.y = outs[-1].ptr
    rec = (GemvLaunch * 32)()
    n_rec = ctypes.c_int(0)
    a.launches, a.max_launches, a.n_launches = rec, 32, ctypes.pointer(n_rec)
    i.keep += [rec, n_rec]
    return a, outs, lambda: [(LAUNCH_FAMILIES[r.family], r.nc, r.only, r.has_ln, r.npad, r.cluster) for r in rec[:n_rec.value]]


def gemv_batch(lib, T, problems, xs, path="engine"):
    """rwkv_b200_test_gemv_batch. problems: dicts with type, K, M, raw (file-layout bytes), input (index into xs) and optionally
    tiled, epi, pro, res / gate ([M, T]), bias ([M]), ln_w / ln_b ([K]), xq (staged bytes), alias (y aliases res). xs: [K, T] arrays.
    Returns (one Out of M*T floats per problem, the launches as (family, nc, only, has_ln, npad, cluster) tuples)."""
    i = Inputs()
    a, outs, launches = _gemv_batch_args(T, problems, xs, path, i)
    _call(lib, lib.library.rwkv_b200_test_gemv_batch, a)
    return outs, launches()


MAX_DELTAS = 31           # deltas / adapters of one rwkv_b200_test_lora_gemv_batch call (LORA_MAX_ADAPTERS)


class LoraDelta(ctypes.Structure):
    _fields_ = [("K", ctypes.c_int), ("M", ctypes.c_int), ("rank", ctypes.c_int), ("scale", ctypes.c_float), ("a", VP), ("b", VP)]


class LoraGemvBatchArgs(ctypes.Structure):
    _fields_ = [("base", GemvBatchArgs), ("n_embed", ctypes.c_int), ("n_ffn", ctypes.c_int), ("n_deltas", ctypes.c_int),
                ("n_adapters", ctypes.c_int), ("d", LoraDelta * MAX_DELTAS), ("delta_of", (ctypes.c_int * MAX_DELTAS) * 8),
                ("col_adapter", ctypes.c_int * 256), ("n_groups", ctypes.c_int), ("u_used", ctypes.c_longlong), ("z_used", ctypes.c_longlong),
                ("u_floats", ctypes.c_longlong), ("z_floats", ctypes.c_longlong), ("scratch_guards_intact", ctypes.c_int)]


def lora_args(T, problems, xs, path, C, F, deltas, delta_of, col_adapter, i):
    """The argument struct of rwkv_b200_test_lora_gemv_batch (see lora_gemv_batch), and the outputs and launch record of its base."""
    base, outs, launches = _gemv_batch_args(T, problems, xs, path, i)
    a = LoraGemvBatchArgs(base=base, n_embed=C, n_ffn=F, n_deltas=len(deltas), n_adapters=max(1, max(len(r) for r in delta_of)))
    for j, (A, B, scale) in enumerate(deltas):
        a.d[j] = LoraDelta(A.shape[1], B.shape[0], A.shape[0], scale, i(A), i(B))
    for p in range(8):
        for k in range(MAX_DELTAS):
            a.delta_of[p][k] = delta_of[p][k] if p < len(delta_of) and k < len(delta_of[p]) else -1
    for t in range(256):
        a.col_adapter[t] = col_adapter[t] if t < len(col_adapter) else -1
    return a, outs, launches


def lora_gemv_batch(lib, T, problems, xs, path, C, F, deltas, delta_of, col_adapter):
    """rwkv_b200_test_lora_gemv_batch: gemv_batch's batch with low-rank deltas, on the scratch of a model of n_embed C and n_ffn F.
    deltas: [(A [rank, K], B [M, rank], scale)]; delta_of[i][k]: the delta adapter k carries on problem i, or -1; col_adapter[t]: column
    t's adapter, or -1. Returns (outs, launches, dict of n_groups, u_used, z_used, u_floats, z_floats, guards)."""
    i = Inputs()
    a, outs, launches = lora_args(T, problems, xs, path, C, F, deltas, delta_of, col_adapter, i)
    _call(lib, lib.library.rwkv_b200_test_lora_gemv_batch, a)
    info = dict(n_groups=a.n_groups, u_used=a.u_used, z_used=a.z_used, u_floats=a.u_floats, z_floats=a.z_floats,
                guards=bool(a.scratch_guards_intact))
    return outs, launches(), info
