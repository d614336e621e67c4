"""Adapted GEMV batches (low-rank deltas, csrc/kernels/lora.h) at the layer shapes of the published RWKV checkpoints, against float64.

rwkv_b200_test_lora_gemv_batch runs a batch as engine.cu's run_batch runs an adapted one: the LoraBatch built by the engine's own
build_lora_batch (column groups per adapter, nonlinear problems retargeted to EPI_NONE into the z scratch, residual ones adding the delta
in place), the shrink, the base batch on its route (streaming, generic, K-quant or tensor cores) and the expand, on scratch sized as a
context of that model sizes it, with a NaN guard behind u and z.
A. Every batch of test_gpu_model_shapes.engine_batches that holds a delta target, at every shape on every route of that module's
   ROUTES, with the formats of formats(s) and two layouts rotated over the routes: one adapter on every column (the context-wide case),
   and three adapters of different ranks and target sets with unadapted columns among them: the sampled rows of every column against float64 of epi(W.x + scale B16.A16.x) (nonlinear) and
   res + (gate *) (W.x + scale B16.A16.x) (residual), at that module's bars widened by lora_ref.lora_magnitude; no NaN of the fill
   anywhere, guards intact, the restated group count and u / z use; on the GEMV routes each column's bits equal that column run alone.
B. The limits of one launch: 128 groups, the most u and z an engine batch uses, and a 129th group refused before any launch.
C. Adapted one-layer model files at the ONE_LAYER shapes of test_gpu_model_shapes.py (and one Q4_K file), vocabulary 1024, through the
   engine: serial == sequence == chunks, tensor-core chunks within the end-to-end bars, zero B == no adapter, the v6 fold, mixed batches
   of 5 and of 64 sequences under 31 adapters; FP32 files at the smallest shape of each architecture against the merged file.
D. Every table entry ran.
tests/test_lora_model_shapes_host.py checks the table, the refusals and that these checks catch planted bugs, without a GPU."""
import collections

import numpy as np
import pytest

import kernel_hooks as kh
import kernel_ref as kr
import lora_ref as lr
import test_gpu_gemv as tg
import test_gpu_model_shapes as ms
from test_gpu_lora import HOOK_K
from test_gpu_model_shapes import sms  # noqa: F401  (the fixture)

pytestmark = pytest.mark.gpu
F32, F64 = np.float32, np.float64
RANKS = [8, 16, 32, 64, 128, 256]
RESIDUAL = (kr.EPI_ADD, kr.EPI_MUL_ADD)


def rank_for(s):
    """The rank of a shape's adapters, rotated over the shapes as formats() rotates the formats."""
    return RANKS[ms.SHAPES.index(s) % len(RANKS)]


def adapted_batches(s):
    """{batch: spec} of the engine's batches at shape s that hold a delta target (lora_ref.DELTA_TARGETS)."""
    return {b: spec for b, spec in ms.engine_batches(s).items() if any(t in lr.DELTA_TARGETS for t, *_ in spec)}


def delta(rng, rank, M, K, scale):
    """(A [rank, K], B [M, rank], scale): A.x of about |x|, B.u a fifth of that."""
    return ((rng.standard_normal((rank, K)) * K ** -0.5).astype(F32), (rng.standard_normal((M, rank)) * 0.2 * rank ** -0.5).astype(F32), scale)


def layout(kind, spec, T, r, rng):
    """(deltas, delta_of, col_adapter) of an adapter layout over the problems of spec. "wide": one adapter of rank r on every delta
    target and every column. "mixed": X (rank r, every target), Y (rank max(8, r / 4), the first target only) and Z (rank min(256, 2 r),
    the targets after the first, or the first when there is one), columns cycling X, Y, none, Z."""
    targets = [j for j, (t, *_) in enumerate(spec) if t in lr.DELTA_TARGETS]
    if kind == "wide":
        ads = [(r, targets, 1.0)]
        cols = [0] * T
    else:
        ads = [(r, targets, 1.5), (max(8, r // 4), targets[:1], 2.0), (min(256, 2 * r), targets[1:] or targets[:1], 0.5)]
        cols = [(0, 1, -1, 2)[t % 4] for t in range(T)]
    deltas, delta_of = [], [[-1] * len(ads) for _ in spec]
    for k, (rank, on, scale) in enumerate(ads):
        for j in on:
            _, M, K, _, _ = spec[j]
            delta_of[j][k] = len(deltas)
            deltas.append(delta(rng, rank, M, K, scale))
    return deltas, delta_of, cols


def restated_use(spec, T, deltas, delta_of, cols):
    """(groups, u floats, z floats) build_lora_batch takes for the layout: per problem with a column under a delta, a group per adapter
    with a delta there and columns, one of rank 0 for the rest of a nonlinear problem's columns; u its largest rank x T, z M x T for a
    nonlinear one."""
    groups = u = z = 0
    for j, (_, M, K, _, epi) in enumerate(spec):
        on = {k for k in set(cols) if k >= 0 and delta_of[j][k] >= 0}
        if not on:
            continue
        rest = any(k < 0 or delta_of[j][k] < 0 for k in cols)
        groups += len(on) + (rest and epi not in RESIDUAL)
        u += max(deltas[delta_of[j][k]][0].shape[0] for k in on) * T
        z += 0 if epi in RESIDUAL else M * T
    return groups, u, z


# ---- the float64 restatement -------------------------------------------------------------------------------------------------

def by_adapter(delta_of_j, cols):
    """{delta index: [its columns]} of a problem: the columns of each adapter with a delta on it."""
    out = {}
    for t, k in enumerate(cols):
        if k >= 0 and delta_of_j[k] >= 0:
            out.setdefault(delta_of_j[k], []).append(t)
    return out


def lora_term(deltas, delta_of_j, cols, rows, x, dt, bug=None):
    """scale B16[rows] . (A16 . x[:, t]) of every column t under its adapter's delta on this problem (zero without one), in dt."""
    d = np.zeros((len(rows), x.shape[1]), dt)
    if bug == "neighbour_adapter":
        cols = cols[1:] + cols[:1]
    for j, ts in by_adapter(delta_of_j, cols).items():
        A, B, scale = deltas[j]
        b16 = B[rows].astype(dt) if bug == "b_fp32" else lr.f16(B[rows]).astype(dt)
        d[:, ts] = dt(scale) * (b16 @ (lr.f16(A).astype(dt) @ x[:, ts].astype(dt)))
    return d


def adapted_reference(p, sub, rows, xs, dt, tc, deltas, delta_of_j, cols, bug=None, prev_base=None):
    """The restatement of adapted problem p over `rows` (sub: ms.row_subset(p, rows)): (output, base W.x, delta) in dt. bug plants one
    defect (tests/test_lora_model_shapes_host.py); prev_base is the previous problem's W.x, which "z_offset" reads instead of this one's."""
    base = ms.reference(dict(sub, epi=kr.EPI_NONE, res=None, gate=None, bias=None), xs, dt, tc)
    d = lora_term(deltas, delta_of_j, cols, rows, xs[p["input"]], dt, bug)
    epi = p["epi"]
    if bug == "z_offset" and prev_base is not None and epi not in RESIDUAL:
        base = prev_base
    if epi in RESIDUAL:
        res = sub["res"].astype(dt)
        gate = sub["gate"].astype(dt) if epi == kr.EPI_MUL_ADD else dt(1)
        out = res + gate * (base + d) if bug != "ungated" else res + gate * base + d
    elif bug == "delta_after_epilogue":
        out = kr.epilogue(base, epi, dt) + d
    else:
        out = kr.epilogue(base + d, epi, dt)
    return out, base, d


def bar_with_lora(r64, r32, factor, mag):
    """ms.check's bar (kr.bar: factor x the float32 restatement's distance, at least 1e-6 of the largest magnitude) per column, widened
    by HOOK_K fp32 spacings of the magnitudes the delta's arithmetic rounds (lora_ref.lora_magnitude), as test_gpu_lora.py's bars are."""
    return kr.bar(r64, r32, factor) + HOOK_K * np.finfo(F32).eps * np.asarray(mag, F64).max(axis=0)


def check_adapted(family, name, got, r64, r32, factor, mag):
    assert not np.isnan(got).any(), (family, name, "NaN left in the output")
    ratio = float((np.abs(np.asarray(got, F64) - r64).max(axis=0) / bar_with_lora(r64, r32, factor, mag)).max())
    WORST[family] = max(WORST[family], ratio)
    assert ratio <= 1, (family, name, ratio, float(np.abs(got - r64).max()))


def magnitude(p, sub, rows, xs, base64, deltas, delta_of_j, cols):
    """lora_ref.lora_magnitude of every column under its adapter; 0 (no widening) for a column without a delta."""
    x = xs[p["input"]]
    epi = p["epi"]
    z = base64 if epi not in RESIDUAL else sub["res"].astype(F64) + (sub["gate"] if epi == kr.EPI_MUL_ADD else 1) * base64
    mag = np.zeros_like(z)
    for j, ts in by_adapter(delta_of_j, cols).items():
        A, B, scale = deltas[j]
        g = sub["gate"][:, ts] if epi == kr.EPI_MUL_ADD else None
        mag[:, ts] = lr.lora_magnitude(A, B[rows], x[:, ts], z[:, ts], g, scale, epi)[1]
    return mag


WORST = collections.defaultdict(float)
RAN = set()


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    for family in sorted(WORST):
        print("\n%-13s worst error / widened bar = %.3f" % (family, WORST[family]), end="")
    print()


def run_adapted(lib, sms, s, name, T, probs, xs, path, spec, lay, check_bits=True):
    """Runs one adapted batch through the hook and checks everything part A asks. Returns the outputs."""
    deltas, delta_of, cols = lay
    outs, launches, info = kh.lora_gemv_batch(lib, T, probs, xs, path, s.C, s.F, deltas, delta_of, cols)
    assert info["guards"], (name, "write past the end of the u / z scratch")
    assert (info["n_groups"], info["u_used"], info["z_used"]) == restated_use(spec, T, deltas, delta_of, cols), (name, info)
    assert info["u_used"] <= info["u_floats"] and info["z_used"] <= info["z_floats"], (name, info)
    assert ms.observed(launches) == ms.expected_launches(T, probs, path, sms), (name, launches)
    fams = {l[0] for l in launches}
    for j, (p, o) in enumerate(zip(probs, outs)):
        assert o.guard_intact(), (name, j, "write past the end of an output")
        assert not np.isnan(o.cols(p["M"])).any(), (name, j, "NaN left in the output")
        tc = ms.takes_tc(p, T, path)
        fam = "tensor_cores" if tc else "kquant" if p["fmt"] in ms.KQ_BYTES else "generic" if "generic" in fams else "streaming"
        rows = ms.sample_rows(p, T, path, probs, sms, tg.rng_for("lora-rows", name, j))
        sub = ms.row_subset(p, rows)
        dj = delta_of[j]
        r64, base64, _ = adapted_reference(p, sub, rows, xs, F64, tc, deltas, dj, cols)
        r32, _, _ = adapted_reference(p, sub, rows, xs, F32, tc, deltas, dj, cols)
        mag = magnitude(p, sub, rows, xs, base64, deltas, dj, cols)
        check_adapted(fam, (name, p["fmt"], p["M"], p["K"], p["epi"]), o.cols(p["M"])[rows], r64, r32, ms.tc_factor(p) if tc else 4, mag)
    if check_bits and not any(ms.takes_tc(p, T, path) for p in probs):
        # a column alone (T = 1, the GEMV) with the same adapter: the same bits, the property "batch row == single context" rests on.
        # The mixed layout cycles X, Y, none, Z: columns 0 .. 3 hold one column of each.
        for t in sorted({0, T - 1} | (set(range(min(T, 4))) if len(set(cols)) > 1 else set())):
            one = [dict(p, res=p["res"][:, t:t + 1].copy() if p.get("res") is not None else None,
                        gate=p["gate"][:, t:t + 1].copy() if p.get("gate") is not None else None) for p in probs]
            one = [{k: v for k, v in q.items() if v is not None} for q in one]
            alone, _, _ = kh.lora_gemv_batch(lib, 1, one, [x[:, t:t + 1].copy() for x in xs], "engine", s.C, s.F, deltas, delta_of, [cols[t]])
            for j, p in enumerate(probs):
                assert alone[j].value.tobytes() == outs[j].cols(p["M"])[:, t].tobytes(), (name, "column", t, "problem", j)
    return outs, info


# ---- A. every adapted batch at every published shape ----------------------------------------------------------------------------

LAYOUTS = ("wide", "mixed")
# Every route of test_gpu_model_shapes.ROUTES at every shape, the formats of formats(s) and the two layouts rotated over the routes, so
# that every shape meets each of its formats and both layouts; a layout on all of GEMV_CASES would take most of an hour.
LORA_CASES = [(s.name, ms.formats(s)[i % len(ms.formats(s))], path, T, LAYOUTS[i % 2]) for s in ms.SHAPES for i, (path, T) in enumerate(ms.ROUTES)]


@pytest.mark.parametrize("shape,fmt,path,T,kind", LORA_CASES)
def test_adapted_batches_at_model_shape(lib, sms, shape, fmt, path, T, kind):
    s = ms.BY_NAME[shape]
    r = rank_for(s)
    for batch, spec in adapted_batches(s).items():
        rng = tg.rng_for("lora-shape-batch", shape, fmt, batch, path, T, kind)
        probs, xs = ms.build(s, fmt, batch, T, rng)
        lay = layout(kind, spec, T, r, rng)
        run_adapted(lib, sms, s, (shape, fmt, batch, path, T, kind), T, probs, xs, path, spec, lay)
        for j, (_, _, _, _, epi) in enumerate(spec):
            if any(k >= 0 for k in lay[1][j]):
                RAN.add((shape, fmt, path, T, epi, kind))


# ---- B. the limits of one launch ------------------------------------------------------------------------------------------------

def full_groups(spec, T, rng):
    """31 adapters of mixed ranks on each of the r / k / v / g problems of a v5.2 / v6 batch, columns cycling none, adapter 0 .. 30:
    4 x (31 + 1) = 128 groups. The four problems have one shape, so they draw from one set of 31 deltas, but adapter k carries delta
    (k + 7 q) % 31 on the q-th of them: a group given its delta from another problem's row (or another adapter's) gets other values."""
    _, M, K, _, _ = spec[0]
    deltas = [delta(rng, RANKS[d % len(RANKS)], M, K, 0.5 + d / 31) for d in range(kh.MAX_DELTAS)]
    targets = [j for j, (t, *_) in enumerate(spec) if t in lr.DELTA_TARGETS]
    delta_of = [[(k + 7 * targets.index(j)) % kh.MAX_DELTAS for k in range(kh.MAX_DELTAS)] if j in targets else [-1] * kh.MAX_DELTAS
                for j in range(len(spec))]
    cols = [t % 32 - 1 for t in range(T)]
    return deltas, delta_of, cols


@pytest.mark.parametrize("T", [64, 256])
def test_128_groups_in_one_launch(lib, sms, T):
    """The v6-7B r / k / v / g batch on the tensor cores with 4 x 32 groups, the most a LoraBatch holds: every column against float64,
    and its bits equal the same column of the batch with every column on its adapter (the context-wide case at the same width)."""
    s = ms.BY_NAME["rwkv6-7b"]
    spec = adapted_batches(s)["att"]
    rng = tg.rng_for("lora-128", T)
    probs, xs = ms.build(s, "Q5_1", "att", T, rng)
    lay = full_groups(spec, T, rng)
    outs, info = run_adapted(lib, sms, s, ("128 groups", T), T, probs, xs, "engine", spec, lay)
    assert info["n_groups"] == 128, info
    deltas, delta_of, cols = lay
    for k in range(-1, kh.MAX_DELTAS):
        wide, _, _ = kh.lora_gemv_batch(lib, T, probs, xs, "engine", s.C, s.F, deltas, delta_of, [k] * T)
        mine = [t for t in range(T) if cols[t] == k]
        for j, p in enumerate(probs):
            assert wide[j].cols(p["M"])[:, mine].tobytes() == outs[j].cols(p["M"])[:, mine].tobytes(), ("adapter", k, "problem", j)
    RAN.add(("128 groups", T))


def test_scratch_at_its_largest_use(lib, sms):
    """rank 256 on the four r / k / v / g problems at T = 256 (4 x 256 x 256 floats of u); the ffn key / receptance batch at T = 256,
    where F + C sets the z allocation and fills it (RWKV-4 14B: 5 C; RWKV-6 7B: F + C = 18432); the v5.2 r / k / v / g batch at
    T = 256, which takes exactly 4 C x 256 of z, less than F + C = 4.5 C allocates. Every use equals its restatement, the guards hold."""
    T = 256
    cases = [("rwkv6-7b", "att", "rank256"), ("rwkv4-14b", "ffn_kr", "wide"), ("rwkv6-7b", "ffn_kr", "wide"), ("rwkv5-7b", "att", "wide")]
    for shape, batch, kind in cases:
        s = ms.BY_NAME[shape]
        spec = adapted_batches(s)[batch]
        rng = tg.rng_for("lora-scratch", shape, batch)
        fmt = "FP16" if shape == "rwkv4-14b" else "Q5_1"
        probs, xs = ms.build(s, fmt, batch, T, rng)
        lay = layout("wide", spec, T, 256 if kind == "rank256" else 16, rng)
        _, info = run_adapted(lib, sms, s, ("scratch", shape, batch), T, probs, xs, "engine", spec, lay)
        assert info["u_floats"] == 8 * 256 * T and info["z_floats"] == max(4 * s.C, s.F + s.C) * T, info
        if kind == "rank256":
            assert info["u_used"] == 4 * 256 * T, info
        elif batch == "ffn_kr":
            assert info["z_used"] == (s.F + s.C) * T == info["z_floats"], info
        else:
            assert info["z_used"] == 4 * s.C * T < info["z_floats"], info
        RAN.add(("scratch", shape, batch))


def test_a_129th_group_is_refused_before_any_launch(lib):
    """The 128 groups of the v6-7B r / k / v / g batch plus att.output (a residual problem: its columns without a delta take no group)
    under adapter 0: 129 groups, one more than the engine can build (at most 4 adapted problems x 32 groups), refused with run_batch's
    error before anything is launched or written back."""
    import ctypes
    s = ms.BY_NAME["rwkv6-7b"]
    spec = adapted_batches(s)["att"][:4] + ms.engine_batches(s)["att_output"]
    T = 64
    rng = tg.rng_for("lora-129", T)
    types = ms.file_types(s, "Q5_1")
    probs = [ms.problem(types[name], M, K, T, rng, input=i, epi=epi) for name, M, K, i, epi in spec]
    xs = tg.inputs([s.C] * 4, T, rng)
    deltas, delta_of, cols = full_groups(spec, T, rng)
    delta_of[4] = [0] + [-1] * (kh.MAX_DELTAS - 1)
    assert restated_use(spec, T, deltas, delta_of, cols)[0] == 129
    i = kh.Inputs()
    a, outs, launches = kh.lora_args(T, probs, xs, "engine", s.C, s.F, deltas, delta_of, cols, i)
    before = lib.library.rwkv_b200_kernel_launch_count()
    assert not lib.library.rwkv_b200_test_lora_gemv_batch(ctypes.byref(a))
    assert lib.rwkv_get_last_error(None) == (6 << 8) | 9          # RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED
    assert lib.library.rwkv_b200_kernel_launch_count() == before and launches() == []
    assert all((o.buf == 0).all() for o in outs)
    RAN.add(("129 groups",))


# ---- C. adapted one-layer files at published shapes ----------------------------------------------------------------------------

# test_gpu_model_shapes.ONE_LAYER (Q5_1, and RWKV-4 14B in FP16) and one K-quant file, at a vocabulary of 1024: the engine's whole
# adapted path (delta_in, the sequence slots of a batch context, chunking, graphs) at the real C and F.
ONE_LAYER = ms.ONE_LAYER + [("rwkv6-1b6", "Q4_K")]
SMALLEST = [min((s for s in ms.SHAPES if s.arch[0] == a), key=lambda s: s.C).name for a in (4, 5, 6, 7)]
V_SMALL = 1024


def one_layer_file(tmp_path, s, fmt):
    import synthetic_model as sm
    path = str(tmp_path / ("%s-%s.bin" % (s.name, fmt)))
    sm.write_direct(path, ms.preset(s, V=V_SMALL), fmt, seed=11)
    return path


def adapter_entries(mf, rank, seed, keep=lambda name: True, zero_b=False):
    """lora_ref.make_entries' deltas (every delta target of the file read once into mf, or those `keep` admits), seeded."""
    rng = np.random.default_rng(seed)
    out = []
    for name, t in mf.tensors.items():
        if lr.is_delta_target(name) and keep(name):
            M, K = lr.matrix_shape(t)
            a = (rng.standard_normal((rank, K)) * K ** -0.5).astype(F32)
            b = np.zeros((M, rank), F32) if zero_b else (rng.standard_normal((M, rank)) * 0.05).astype(F32)
            out.append((name, rank, a, b, None))
    return out


@pytest.mark.parametrize("shape,fmt", ONE_LAYER)
def test_adapted_one_layer_file(lib, tmp_path, shape, fmt):
    """A context-wide rank-16 adapter on every delta target: serial == eval_sequence == chunks of 7 and 31 bit for bit, a 128-token
    chunk (tensor cores) within the end-to-end bars of serial, a zero-B adapter gives the unadapted bits, and a v6 layer still runs
    v6_prologue exactly where fold_expected says. Batch contexts (n_embed <= 4096): a mixed batch of 5 equals each sequence alone with
    its adapter, and a batch of 64 with 31 distinct adapters and unadapted sequences equals, row by row, the batch with that row's
    adapter attached to the whole context (tensor cores)."""
    from test_gpu_lora import Ctx, batch_run, prompt, same
    from test_gpu_lora_batch import MixedBatch, single_serial
    from test_gpu_v6_fused import traced_names
    s = ms.BY_NAME[shape]
    path = one_layer_file(tmp_path, s, fmt)
    mf = lr.read_model_file(path)
    c = Ctx(lib, path)
    ads = []
    try:
        toks = [(7919 * i + 11) % V_SMALL for i in range(128)]
        base = c.serial(toks[:40])
        # the unadapted file's own distance of a 128-token chunk (tensor cores) from serial
        base_serial, base_chunk = c.serial(toks), c.chunks(toks, 128)
        base_err = [float(np.abs(a - b).max()) for a, b in zip(base_chunk, base_serial)]
        ad = c.adapter(adapter_entries(mf, 16, 1), 1.0)
        zero = c.adapter(adapter_entries(mf, 16, 2, zero_b=True), 1.0)
        ads += [ad, zero]
        c.attach(ad)
        serial = ms.evaluate_serial(lib, c.c, toks, c.n_state, c.n_logits)
        assert all(np.isfinite(a).all() for a in serial[-1])
        want40 = (serial[39][1], serial[39][0])
        assert not same(want40, base), "the adapter has no effect"
        assert same(c.sequence(toks[:31]), (serial[30][1], serial[30][0])), "eval_sequence"
        for chunk in (7, 31):
            assert same(c.chunks(toks[:40], chunk), want40), chunk
        lg, st = c.chunks(toks, 128)
        err, serr = float(np.abs(lg - serial[-1][1]).max()), float(np.abs(st - serial[-1][0]).max())
        print("\n%s %s adapted: 128-token chunk - serial: logits %.2e, state %.2e (unadapted %.2e, %.2e)" % (shape, fmt, err, serr, *base_err),
              end="")
        if fmt in ms.E2E_TOL:
            tol = ms.E2E_TOL[fmt]
            assert err <= tol and serr <= 20 * tol, (err, serr)
        else:
            # No end-to-end bar is set for K-quant files: their GEMV quantises the activations to Q8_K (256-element blocks) where the
            # tensor cores take fp16, so their chunks land farther from serial than Q5_1's. The file's own unadapted distance sets the
            # scale; the adapter may not more than double it.
            assert err <= 2 * base_err[0] and serr <= 2 * base_err[1], (err, serr, base_err)
        if s.arch[0] == 6:
            names = traced_names(lib, c.c, toks[0])
            assert names.count("v6_prologue") == int(ms.fold_expected(s, fmt)), names
        c.attach(zero)
        assert same(c.serial(toks[:40]), base) and same(c.chunks(toks[:40], 31), base), "zero B"
        c.attach(None)
        if s.C > 4096:      # batch contexts take n_embed <= 4096
            RAN.add((shape, "one_layer", fmt))
            return
        # a mixed batch of 5 (GEMV): each row is that sequence alone with its adapter
        other = c.adapter(adapter_entries(mf, 64, 3, keep=lambda n: ".ffn." in n or "att.output" in n), 0.5)
        ads.append(other)
        assign = [ad, None, other, ad, zero]
        prompts = [prompt(3, V_SMALL, b) for b in range(5)]
        bt = MixedBatch(lib, c, assign)
        try:
            for step in range(3):
                assert bt.eval([q[step] for q in prompts])
            for b, (got, a) in enumerate(zip(bt.rows(), assign)):
                assert same(got, single_serial(c, a, prompts[b])), ("batch of 5", b)
        finally:
            bt.free()
        # 64 sequences, 31 distinct adapters of mixed ranks and targets, every 32nd sequence unadapted (tensor cores)
        many = [c.adapter(adapter_entries(mf, RANKS[k % len(RANKS)], 10 + k, keep=lambda n, k=k: k % 3 or ".att." in n), 1.0) for k in range(31)]
        ads += many
        assign = [many[b % 32 - 1] if b % 32 else None for b in range(64)]
        prompts = [prompt(2, V_SMALL, 20 + b) for b in range(64)]
        bt = MixedBatch(lib, c, assign)
        try:
            for step in range(2):
                assert bt.eval([q[step] for q in prompts])
            rows = bt.rows()
        finally:
            bt.free()
        for a in many + [None]:
            want = batch_run(lib, c, a, prompts, 2)
            for b in range(64):
                if assign[b] is a:
                    assert same(rows[b], want[b]), ("batch of 64", b)
    finally:
        c.attach(None)
        for a in ads:
            lib.rwkv_b200_adapter_free(a)
        c.free()
    RAN.add((shape, "one_layer", fmt))


@pytest.mark.parametrize("shape", SMALLEST)
def test_adapted_fp32_file_matches_the_merged_file(lib, tmp_path, shape):
    """The smallest shape of each architecture in FP32 with a rank-16 adapter against lora_ref.merged_file (the deltas merged in
    float64) over every kind of pass, at the bars of test_gpu_lora.test_adapted_fp32_matches_the_merged_file."""
    from test_gpu_lora import Ctx, all_passes, within
    s = ms.BY_NAME[shape]
    path = one_layer_file(tmp_path, s, "FP32")
    entries = adapter_entries(lr.read_model_file(path), 16, 11)
    scale = 0.5
    merged = str(tmp_path / "merged.bin")
    lr.merged_file(path, merged, entries, scale)
    a, m = Ctx(lib, path), Ctx(lib, merged)
    try:
        toks = [(7919 * i + 11) % V_SMALL for i in range(70)]
        base = all_passes(lib, a, None, toks)
        want = all_passes(lib, m, None, toks)
        ad = a.adapter(entries, scale)
        a.attach(ad)
        got = all_passes(lib, a, ad, toks)
        a.attach(None)
        lib.rwkv_b200_adapter_free(ad)
        for kind in want:
            for i, part in enumerate(want[kind]):
                within(got[kind][i], part, base[kind][i], 0.01, 1e-5, f"{shape} {kind}[{i}]")
    finally:
        a.free()
        m.free()
    RAN.add((shape, "merged"))


# ---- D. every table entry ran -----------------------------------------------------------------------------------------------------

def table():
    """Every (shape, format, route, epilogue, layout) part A must reach, and the cases of parts B and C."""
    want = set()
    for shape, fmt, path, T, kind in LORA_CASES:
        for spec in adapted_batches(ms.BY_NAME[shape]).values():
            want |= {(shape, fmt, path, T, epi, kind) for t, _, _, _, epi in spec if t in lr.DELTA_TARGETS}
    want |= {("128 groups", 64), ("128 groups", 256), ("129 groups",)}
    want |= {(n, "one_layer", f) for n, f in ONE_LAYER} | {(n, "merged") for n in SMALLEST}
    want |= {("scratch", n, b) for n, b in (("rwkv6-7b", "att"), ("rwkv4-14b", "ffn_kr"), ("rwkv6-7b", "ffn_kr"), ("rwkv5-7b", "att"))}
    return want


def test_every_adapted_shape_and_route_ran(request):
    """Runs last: every entry of table() ran. A run of part of the file (-k, a node id) skips it."""
    n_items = len(LORA_CASES) + 2 + 1 + 1 + len(ONE_LAYER) + len(SMALLEST)
    if sum(i.fspath == request.node.fspath for i in request.session.items) < n_items:
        pytest.skip("only part of the file was selected")
    want = table()
    print("\n%d table entries, %d ran" % (len(want), len(want & RAN)))
    assert want <= RAN, sorted(want - RAN, key=str)[:20]
