"""Every kernel launch of the eval path at the layer shapes of the published RWKV checkpoints, against float64.

The per-kernel suites (test_gpu_gemv.py, test_gpu_kernels.py, test_gpu_v6_fused.py) reach every instantiation, but at few layer shapes,
and what goes wrong when a shape changes is computed from the shape: the streaming GEMV's WK / lane groups / NC / stage bytes / CTA
shares, the fallback to the generic kernel, the tensor-core cluster size and npad, the K-quant wide budget, the v6 fold predicate. Here
SHAPES lists the published RWKV-4 / 5.2 / 6 / 7 layer shapes; each matrix gets the type the quantiser writes for it (file_types), and
the batches are built as engine.cu builds them (engine_batches), on every route of the eval path: a single context's SIMT launches
(T = 1 / 3 / 31) and tensor-core launches (T = 32 / 128 / 256), a batch context's (B = 5 / 15 SIMT, B = 16 / 64 / 256 tensor cores),
the head with its LayerNorm prologue at the real vocabulary (single tokens, scoring passes of up to 256 columns, batch contexts of up
to 256 sequences), and the tensor-core head of scoring passes (LayerNorm of columns, the GEMM, the score kernel). Each launch record is
checked against a host restatement of the plan (routing, NC, generic fallback, cluster size, npad). The float64 reference restates only some rows -- all rows of the first and last
128-row tile, both edge rows of every tensor-core tile and of the first tile of every streaming CTA, and a seeded sample -- and every
column, and no output may keep the NaN of the 0xFF fill in any row. The state kernels run at the same shapes (part A). One-layer model
files at the smallest and largest shape of each architecture and at RWKV-4 14B check the engine's own invariants there: serial ==
sequence == chunks, batch == alone, tensor-core passes within the end-to-end bars, where the v6 LoRA fold runs, and scoring at the
real vocabulary: GEMV-head passes and ragged passes below 16 columns bit for bit, tensor-core ones within the end-to-end bars (part B).
tests/test_model_shapes_host.py checks the table and the bars without a GPU."""
import collections
import ctypes
import functools
import types

import numpy as np
import pytest

import ggml_file as gf
import kernel_hooks as kh
import kernel_ref as kr
import kquant_ref as kq
import test_gpu_gemv as tg
from test_gpu_kernels import (F32, F64, ln_mix_inputs, lerp_inputs, ref_wkv4, ref_wkv6, ref_wkv7, run_wkv4, run_wkv6, run_wkv7, wkv4_inputs,
                              wkv6_inputs, wkv7_inputs)
from test_gpu_score import (NO, P_F, P_U, P_U8, SENTINEL, bits, check_rows, lp64, ragged_case, score_logits, text_targets, u32,
                            traced_names as score_trace)

pytestmark = pytest.mark.gpu

# ---- the published layer shapes ---------------------------------------------------------------------------------------------

Shape = collections.namedtuple("Shape", "name arch C F V S mix decay lora")


def lora_width(C, factor, power):
    """RWKV-LM's v7 LoRA widths: round(factor * C^power / 32) * 32, at least 32."""
    return max(32, round(factor * C ** power / 32) * 32)


def v7_lora(C):
    return dict(w=lora_width(C, 1.8, 0.5), a=lora_width(C, 1.8, 0.5), v=lora_width(C, 1.3, 0.5), g=lora_width(C, 0.6, 0.8))


def _v4(name, C):
    return Shape(name, (4, 0), C, 4 * C, 50277, 0, 0, 0, None)


def _v5(name, C):
    return Shape(name, (5, 2), C, int(3.5 * C) // 32 * 32, 65536, 64, 0, 0, None)


def _v6(name, C):
    return Shape(name, (6, 0), C, int(3.5 * C) // 32 * 32, 65536, 64, 64 if C >= 4096 else 32, 128 if C >= 4096 else 64, None)


def _v7(name, C):
    return Shape(name, (7, 0), C, 4 * C, 65536, 64, 0, 0, v7_lora(C))


SHAPES = ([_v4(n, C) for n, C in (("rwkv4-169m", 768), ("rwkv4-430m", 1024), ("rwkv4-1b5", 2048), ("rwkv4-3b", 2560), ("rwkv4-7b", 4096),
                                   ("rwkv4-14b", 5120))]
          + [_v5(n, C) for n, C in (("rwkv5-0b4", 1024), ("rwkv5-1b5", 2048), ("rwkv5-3b", 2560), ("rwkv5-7b", 4096))]
          + [_v6(n, C) for n, C in (("rwkv6-1b6", 2048), ("rwkv6-3b", 2560), ("rwkv6-7b", 4096))]      # the 14B has the 7B layer shape
          + [_v7(n, C) for n, C in (("rwkv7-0b1", 768), ("rwkv7-0b4", 1024), ("rwkv7-1b5", 2048), ("rwkv7-2b9", 2560))])
BY_NAME = {s.name: s for s in SHAPES}
LARGEST = {a: max((s for s in SHAPES if s.arch[0] == a), key=lambda s: s.C).name for a in (4, 5, 6, 7)}

CORE_FORMATS = ["Q5_1", "FP16"]
ROTATION = ["Q4_0", "Q4_1", "Q5_0", "Q8_0", "FP32", "Q4_K", "Q5_K"]
KQ_FALLBACK = {"Q4_K": "Q5_0", "Q5_K": "Q5_1"}
TYPE = dict(gf.TYPE_IDS, Q4_K=13, Q5_K=14)


def formats(s):
    """Q5_1 and FP16 everywhere; the largest C of each architecture also runs every format of the rotation, the other shapes one each."""
    if s.name == LARGEST[s.arch[0]]:
        return CORE_FORMATS + ROTATION
    i = [x for x in SHAPES if x.name not in LARGEST.values()].index(s)
    return CORE_FORMATS + [ROTATION[i % len(ROTATION)]]


def file_types(s, fmt):
    """{tensor name in a layer (or emb / head): format} as rwkv_quantize_model_file writes a quantised file from an FP16 master
    (quantizer.cpp: 2-D tensors except emb, head and the v7 LoRA / r_k ones; K-quant rows that are not whole super-blocks fall back to
    Q5_0 / Q5_1), or as an FP16 / FP32 file holds them (v6 LoRA matrices stay FP32 in an FP16 file)."""
    C, F = s.C, s.F
    dense = fmt in ("FP16", "FP32")
    wide = "FP32" if fmt == "FP32" else "FP16"
    q = lambda K: KQ_FALLBACK[fmt] if fmt in KQ_FALLBACK and K % 256 else fmt
    t = {"emb.weight": wide, "head.weight": wide, "ffn.key.weight": q(C), "ffn.value.weight": q(F)}
    att = {4: ("key", "value", "receptance", "output"), 5: ("key", "value", "receptance", "output", "gate"),
           6: ("receptance", "key", "value", "output", "gate"), 7: ("receptance", "key", "value", "output")}[s.arch[0]]
    t.update({"att.%s.weight" % n: q(C) for n in att})
    if s.arch[0] != 7:
        t["ffn.receptance.weight"] = q(C)
    if s.arch[0] == 6:
        lora = lambda K: "FP32" if dense else q(K)
        t.update({"att.time_maa_w1": lora(C), "att.time_decay_w1": lora(C), "att.time_decay_w2": lora(s.decay)})
    if s.arch[0] == 7:
        t.update({"att.%s%d" % (n, i): wide for n in "wavg" for i in (1, 2)})
    return t


def preset(s, L=1, V=None):
    """A tools/synthetic_model.py preset of L layers at shape s (its real vocabulary unless V is given)."""
    p = dict(arch=s.arch, C=s.C, F=s.F, L=L, V=V or s.V, out_scale=0.1, lora_fan_in=True)
    if s.S:
        p["S"] = s.S
    if s.arch[0] == 6:
        p.update(mix=s.mix, decay=s.decay)
    if s.arch[0] == 7:
        p.update(lora_w=s.lora["w"], lora_a=s.lora["a"], lora_v=s.lora["v"], lora_g=s.lora["g"])
    return p


# ---- the batches of engine.cu at a shape ------------------------------------------------------------------------------------


def engine_batches(s):
    """{batch: [(tensor, M, K, input, epilogue)]} of one layer, as engine.cu's att_v4 / att_v5 / att_v6 (the unfolded multi-token
    launches) / att_v7 (a layer after the first), ffn and att_output build them."""
    C, F, a = s.C, s.F, s.arch[0]
    mat = lambda n: "att.%s.weight" % n
    B = {}
    if a == 4:
        B["att"] = [(mat("receptance"), C, C, 0, kr.EPI_SIGMOID), (mat("key"), C, C, 1, 0), (mat("value"), C, C, 2, 0)]
    elif a == 5:
        B["att"] = [(mat("receptance"), C, C, 0, 0), (mat("key"), C, C, 1, 0), (mat("value"), C, C, 2, 0), (mat("gate"), C, C, 3, kr.EPI_SILU)]
    elif a == 6:
        B["maa_w1"] = [("att.time_maa_w1", 5 * s.mix, C, 0, kr.EPI_TANH)]
        B["att"] = [(mat("receptance"), C, C, 0, 0), (mat("key"), C, C, 1, 0), (mat("value"), C, C, 2, 0), (mat("gate"), C, C, 3, kr.EPI_SILU),
                    ("att.time_decay_w1", s.decay, C, 4, kr.EPI_TANH)]
        B["decay_w2"] = [("att.time_decay_w2", C, s.decay, 0, kr.EPI_BIAS_EXPNEGEXP)]
    else:
        L = s.lora
        B["lora_first"] = [(mat("receptance"), C, C, 0, 0), (mat("key"), C, C, 2, 0), (mat("value"), C, C, 3, 0), ("att.w1", L["w"], C, 1, kr.EPI_TANH),
                           ("att.a1", L["a"], C, 4, 0), ("att.g1", L["g"], C, 5, kr.EPI_SIGMOID), ("att.v1", L["v"], C, 3, 0)]
        B["lora_second"] = [("att.w2", C, L["w"], 0, kr.EPI_BIAS_W7), ("att.a2", C, L["a"], 1, kr.EPI_BIAS_SIGMOID), ("att.g2", C, L["g"], 2, 0),
                            ("att.v2", C, L["v"], 3, kr.EPI_BIAS_SIGMOID)]
    B["ffn_kr"] = [("ffn.key.weight", F, C, 0, kr.EPI_RELU_SQR)] + ([("ffn.receptance.weight", C, C, 1, kr.EPI_SIGMOID)] if a != 7 else [])
    B["ffn_value"] = [("ffn.value.weight", C, F, 0, kr.EPI_ADD if a == 7 else kr.EPI_MUL_ADD)]     # in place: y is the residual
    B["att_output"] = [(mat("output"), C, C, 0, kr.EPI_ADD)]
    return B


@functools.lru_cache(maxsize=8)          # a few of the largest matrices (400 MB at 14B in FP32) at a time
def weights(fmt, M, K):
    """(type, file-layout bytes): tg.random_raw's weights, F16 / F32 ones drawn in float32, K-quant ones random super-blocks."""
    rng = tg.rng_for("shape-raw", fmt, M, K)
    if fmt in KQ_FALLBACK:
        return TYPE[fmt], kq.random_blocks(TYPE[fmt], M, K, rng)
    if fmt in ("FP16", "FP32"):
        w = rng.standard_normal((M, K), dtype=F32) * F32(1 / np.sqrt(K))
        return TYPE[fmt], w.astype(np.float16 if fmt == "FP16" else F32).view(np.uint8).reshape(-1)
    return tg.random_raw.__wrapped__(fmt, M, K)


def head_weights(V, C, tiles=None):
    """float32 head weights of about 1 / sqrt(C), [rows of `tiles`, C]: every 128-row tile drawn from its own seed, so that a test can
    restate some tiles of a 65536-row head without drawing the rest (all tiles when None)."""
    tiles = range(-(-V // 128)) if tiles is None else tiles
    w = np.empty((sum(min(128, V - 128 * t) for t in tiles), C), F32)
    r = 0
    for t in tiles:
        n = min(128, V - 128 * t)
        w[r:r + n] = tg.rng_for("shape-head", V, C, t).standard_normal((n, C), dtype=F32)
        r += n
    w *= F32(1 / np.sqrt(C))
    return w


def head_raw(fmt, w):
    return TYPE[fmt], w.astype(np.float16 if fmt == "FP16" else F32).view(np.uint8).reshape(-1)


@pytest.fixture(scope="module")
def head():
    """head(fmt, V, C) -> (type, bytes) of a shape's head. The FP16 bytes of every head drawn stay for the module (11 heads, 3 GB); of
    the FP32 bytes only the last head's do (shapes of one vocabulary and width share a head)."""
    f16, f32 = {}, {}

    def get(fmt, V, C):
        if (V, C) not in (f32 if fmt == "FP32" else f16):
            w = head_weights(V, C)
            f16[(V, C)] = head_raw("FP16", w)
            if fmt == "FP32":
                f32.clear()
                f32[(V, C)] = head_raw("FP32", w)
        return (f32 if fmt == "FP32" else f16)[(V, C)]
    yield get
    f16.clear()
    f32.clear()


def problem(fmt, M, K, T, rng, input=0, epi=0, tiled=None, raw=None):
    """tg.problem with the weights above (or `raw` = (type, bytes)); the tile-major copy exists where gemm_tc_eligible (engine.cu keeps
    one for every layer matrix), which for K-quant rows means whole super-blocks."""
    if tiled is None:
        tiled = fmt != "FP32" and K % (256 if fmt in KQ_FALLBACK else 64) == 0
    return tg.problem(fmt, M, K, T, rng, input=input, epi=epi, tiled=tiled, weights=raw or weights(fmt, M, K))


def build(s, fmt, batch, T, rng):
    types = file_types(s, fmt)
    spec = engine_batches(s)[batch]
    probs = [problem(types[name], M, K, T, rng, input=i, epi=epi) for name, M, K, i, epi in spec]
    Ks = {i: K for name, M, K, i, epi in spec}
    xs = tg.inputs([Ks[i] for i in range(len(Ks))], T, rng)
    return probs, xs


# ---- host restatement of the launch plan ------------------------------------------------------------------------------------

CONSUMER_WARPS, NSTAGES, NOMINAL_STAGE, CTA_SMEM, MAX_TILE_ROWS, MAX_BLOCKS_PER_LANE = 8, 3, 28 * 1024, 110 * 1024, 64, 4
KQ_BYTES = {"Q4_K": 144, "Q5_K": 176}


def pitch(fmt, K):
    """matrix_pitch: row bytes (an even number of blocks for the *_0 formats), 16-byte aligned."""
    if fmt in KQ_BYTES:
        b = K // 256 * KQ_BYTES[fmt]
    else:
        elems, nbytes = gf.BLOCK[TYPE[fmt]]
        n = K // elems
        b = ((n + 1) // 2 * 2 if fmt in ("Q4_0", "Q5_0", "Q8_0") else n) * nbytes
    return (b + 15) // 16 * 16


def act_bytes(fmt, K):
    if fmt in KQ_BYTES:
        return (K // 256 * (256 + 4 + 32) + 15) // 16 * 16
    return kr.staged_bytes(TYPE[fmt], K)


def plan_wk(fmt, K):
    """WK of the streaming GEMV (gemv_tma.cu plan_wk), or None where the row does not fit it."""
    quant = fmt not in ("FP16", "FP32")
    for wk in (1, 2, 4, 8):
        if CONSUMER_WARPS // wk * pitch(fmt, K) > NOMINAL_STAGE or (quant and K // 32 > MAX_BLOCKS_PER_LANE * 32 * wk):
            continue
        return wk
    return None


def stage_for(nc, max_col, budget=CTA_SMEM):
    return (budget - nc * max_col - 2 * MAX_TILE_ROWS * CONSUMER_WARPS * nc * 4) // NSTAGES // 1024 * 1024


def streaming_plan(T, probs):
    """(NC, stage bytes) of gemv_tma_launch, or None where the batch takes the generic kernel."""
    if any(plan_wk(p["fmt"], p["K"]) is None for p in probs):
        return None
    mc = max(act_bytes(p["fmt"], p["K"]) for p in probs)
    nc = 4 if T >= 4 and stage_for(4, mc) >= NOMINAL_STAGE else 2 if T >= 2 and stage_for(2, mc) >= NOMINAL_STAGE else 1
    return (nc, stage_for(nc, mc)) if stage_for(nc, mc) >= NOMINAL_STAGE else None


def kquant_wk(p):
    """WK of the K-quant GEMV (gemv_kquant.cu plan_kq)."""
    for w in (1, 2, 4, 8):
        if CONSUMER_WARPS // w * pitch(p["fmt"], p["K"]) <= NOMINAL_STAGE:
            return w
    return 8


def kquant_plan(T, probs):
    """(NC, stage bytes, CTAs per SM) of gemv_kq_launch."""
    mc = max(act_bytes(p["fmt"], p["K"]) for p in probs)
    need = max(CONSUMER_WARPS // kquant_wk(p) * pitch(p["fmt"], p["K"]) for p in probs)
    wide = stage_for(1, mc) < need
    budget = 2 * CTA_SMEM if wide else CTA_SMEM
    floor = max(need, NOMINAL_STAGE)
    nc = 4 if T >= 4 and stage_for(4, mc, budget) >= floor else 2 if T >= 2 and stage_for(2, mc, budget) >= floor else 1
    return nc, stage_for(nc, mc, budget), 1 if wide else 2


def tile_shares(probs, total_ctas, stage, wk_of):
    """assign_tiles_and_ctas: (tile rows, CTAs) of every problem."""
    total = sum(p["M"] * pitch(p["fmt"], p["K"]) for p in probs)
    out = []
    for p in probs:
        wr = CONSUMER_WARPS // wk_of(p)
        rows = stage // pitch(p["fmt"], p["K"])
        rows = min(rows - rows % wr, MAX_TILE_ROWS)
        cap = -(-p["M"] // rows)
        share = total_ctas * p["M"] * pitch(p["fmt"], p["K"]) / total
        base = min(max(int(share), 1), cap)
        out.append([rows, base, share - base, cap])
    assigned = sum(o[1] for o in out)
    while assigned < total_ctas:
        cand = [i for i, o in enumerate(out) if o[1] < o[3]]
        if not cand:
            break
        best = max(cand, key=lambda i: (out[i][2], -i))
        out[best][1] += 1
        out[best][2] -= 1.0
        assigned += 1
    return [(o[0], o[1]) for o in out]


def tc_plan(T, probs, sms):
    """(npad, cluster, [splits]) of gemm_tc_launch."""
    tiles = [-(-p["M"] // 128) for p in probs]
    total = sum(tiles)
    want = sms // total if total * 4 < sms * 3 else 1
    cluster = 1
    while cluster * 2 <= want and cluster < 8:
        cluster *= 2
    splits = []
    for p in probs:
        n = p["K"] // 64
        per = -(-n // cluster)
        splits.append(cluster if cluster > 1 and n >= 4 * cluster and (cluster - 1) * per < n else 1)
    return (T + 15) // 16 * 16, cluster if max(splits) > 1 else 1, splits


takes_tc = tg.takes_tc                        # the routing of gemv_route


def expected_launches(T, probs, path, sms):
    """The launch record the routing (gemv_route / gemv_launch) must leave, without the weight expansions, as a sorted list."""
    tc = [p for p in probs if takes_tc(p, T, path)]
    rest = [p for p in probs if not takes_tc(p, T, path)]
    out = []
    if tc:
        npad, cluster, _ = tc_plan(T, tc, sms)
        kinds = {(p["input"], 0 if p["fmt"] == "FP16" else 2 if p["fmt"] in KQ_BYTES else 1) for p in tc}
        n16, nk = sum(1 for _, k in kinds if k < 2), sum(1 for _, k in kinds if k == 2)
        out += [("convert", n16, 0, 0, npad, 0)] * bool(n16) + [("convert", nk, 16, 0, npad, 0)] * bool(nk)
        out.append(("tensor_cores", 0, 0, 0, npad, cluster))
    for f in KQ_BYTES:
        part = [p for p in rest if p["fmt"] == f]
        if part:
            out.append(("kquant", kquant_plan(T, part)[0], TYPE[f], 0, 0, 0))
    legacy = [p for p in rest if p["fmt"] not in KQ_BYTES]
    if legacy:
        plan = streaming_plan(T, legacy)
        if plan is None:
            out.append(("generic",))
        else:
            only = legacy[0]["type"] if plan[0] == 1 and len({p["type"] for p in legacy}) == 1 else -1
            out.append(("streaming", plan[0], only, 1 if only < 0 else int(any(p.get("pro") for p in legacy)), 0, 0))
    return sorted(out)


def observed(launches):
    return sorted((l[:1] if l[0] == "generic" else l) for l in launches if l[0] not in ("expand", "kquant_expand"))


def sample_rows(p, T, path, probs, sms, rng):
    """Rows the float64 reference restates: the first and last 128-row tile, both edge rows of every tensor-core tile and of the first
    tile of every streaming CTA, and 64 seeded rows."""
    M = p["M"]
    rows = set(range(min(128, M))) | set(range((M - 1) // 128 * 128, M))
    if takes_tc(p, T, path):
        rows |= {r for t in range(0, M, 128) for r in (t, min(M, t + 128) - 1)}
    else:
        rest = [q for q in probs if not takes_tc(q, T, path) and (q["fmt"] in KQ_BYTES) == (p["fmt"] in KQ_BYTES)]
        plan = kquant_plan(T, rest) if p["fmt"] in KQ_BYTES else streaming_plan(T, rest)
        if plan is not None:
            per_sm = plan[2] if p["fmt"] in KQ_BYTES else 2
            wk_of = kquant_wk if p["fmt"] in KQ_BYTES else (lambda q: plan_wk(q["fmt"], q["K"]))
            h, n_cta = tile_shares(rest, per_sm * sms, plan[1], wk_of)[[id(q) for q in rest].index(id(p))]
            rows |= {r for t in range(min(n_cta, -(-M // h))) for r in (t * h, min(M, (t + 1) * h) - 1)}
    rows |= set(rng.choice(M, min(M, 64), replace=False).tolist())
    return np.array(sorted(rows))


# ---- the float64 restatement of some rows -----------------------------------------------------------------------------------

def row_subset(p, rows):
    """p restricted to `rows`: the weights of those rows in the file layout and their residual / gate / bias."""
    if p["fmt"] in KQ_BYTES:
        rb = p["K"] // 256 * KQ_BYTES[p["fmt"]]
    else:
        elems, nbytes = gf.BLOCK[p["type"]]
        rb = p["K"] // elems * nbytes
    q = dict(p, M=len(rows), raw=np.ascontiguousarray(np.asarray(p["raw"]).reshape(p["M"], rb)[rows]).reshape(-1))
    for key in ("res", "gate"):
        if p.get(key) is not None:
            q[key] = p[key][rows]
    if p.get("bias") is not None:
        q["bias"] = p["bias"][rows]
    return q


def kq_gemv(p, x, dt, bug=None):
    """ggml_vec_dot_q{4,5}_K_q8_K per column, the super-blocks combined in dt (kquant_ref.gemv64 for dt = float64)."""
    tid, M, K = p["type"], p["M"], p["K"]
    d, dmin, sc, mn, q = kq.unpack(tid, p["raw"], M, K)
    nsb = K // 256 - (bug == "drop_last_block")
    y = np.empty((M, x.shape[1]), dt)
    for t in range(x.shape[1]):
        yd, qs, bs = kq.quantize_q8k(x[:, t])
        dots = np.einsum("msjl,sjl->msj", q[:, :nsb], qs[:nsb].reshape(-1, 8, 32))
        isum = (dots * sc[:, :nsb]).sum(axis=2).astype(dt)
        msum = (mn[:, :nsb] * (bs[:nsb, 0::2] + bs[:nsb, 1::2])[None]).sum(axis=2).astype(dt)
        ydt = yd[:nsb].astype(dt)[None]
        y[:, t] = (ydt * d[:, :nsb].astype(dt) * isum - ydt * dmin[:, :nsb].astype(dt) * msum).sum(axis=1, dtype=dt)
    return y


def reference(p, xs, dt, tc, bug=None, ksplit=1):
    """The float64 (dt) restatement of problem p (possibly a row subset)."""
    x = xs[p["input"]]
    kw = dict(res=p.get("res"), gate=p.get("gate"), bias=p.get("bias"), bug=bug)
    if p["fmt"] in KQ_BYTES:
        v = kq.gemm_tc(p["type"], p["raw"], p["M"], p["K"], x, dt) if tc else kq_gemv(p, x, dt, bug)
        return kr.epilogue(v, p["epi"], dt, **kw)
    if tc:
        return kr.gemm_tc(p["type"], p["raw"], p["M"], x, dt, epi=p["epi"], ksplit=ksplit, **kw)
    ln = (p["ln_w"], p["ln_b"]) if p.get("pro") else None
    if bug == "drop_last_block":         # the last block (32 weights) of every row never added
        K = p["K"] - 32
        elems, nbytes = gf.BLOCK[p["type"]]
        raw = np.asarray(p["raw"]).reshape(p["M"], p["K"] // elems * nbytes)[:, :K // elems * nbytes].reshape(-1)
        return kr.gemv(p["type"], np.ascontiguousarray(raw), p["M"], np.ascontiguousarray(x[:K]), dt, epi=p["epi"], **dict(kw, bug=None))
    return kr.gemv(p["type"], p["raw"], p["M"], x, dt, ln=ln, epi=p["epi"], **kw)


# ---- checks -----------------------------------------------------------------------------------------------------------------

# The tensor-core bar of test_gpu_gemv.py (tg.TC_BAR_FACTOR: 64 times the float32 distance) was set on launches of at most 4096 x 14336
# and T = 64, where wgmma's truncated fp32 accumulation landed up to 43x as far from float64 as numpy's float32 matmul over all rows.
# The channel-mixing matrices of the 7B and 14B shapes (M * K >= 14336 * 4096) land farther: on an H100 80GB HBM3 at 700 W, up to 81x
# (RWKV-4 14B's ffn.key, 20480 x 5120 with relu^2, T = 128 / 256) and 74x (its ffn.value, K = 20480, T = 32). Part of that is the row
# sample: the float32 distance of a column is taken over the sampled rows only, which lowers the bar. Those matrices are held to twice
# the bar, every other tensor-core launch to the bar of test_gpu_gemv.py; every planning defect of tests/test_model_shapes_host.py still
# lands above the doubled bar. TC_NEEDED reports the factor each tensor-core shape needed.
WIDE_TC = 14336 * 4096


def tc_factor(p):
    return 2 * tg.TC_BAR_FACTOR if p["M"] * p["K"] >= WIDE_TC else tg.TC_BAR_FACTOR


WORST = collections.defaultdict(float)
NEEDED = collections.defaultdict(float)
TC_NEEDED = collections.defaultdict(float)    # (M, K) -> error / float32 distance of its tensor-core launches
HEADS_ON_TC = set()                           # (V, C) of the heads run on the tensor cores
RAN = set()                                   # (shape, route) pairs that ran
KEYS = collections.defaultdict(set)           # shape -> launch keys reached


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    for family in sorted(WORST):
        print("\n%-13s worst error / bar = %.3f (error / fp32 distance %.2f)" % (family, WORST[family], NEEDED[family]), end="")
    for (M, K), f in sorted(TC_NEEDED.items(), key=lambda kv: -kv[1])[:12]:
        print("\ntensor cores %5d x %5d: error / fp32 distance %.2f (bar factor %d)" % (M, K, f, tc_factor(dict(M=M, K=K))), end="")
    for V, C in sorted(HEADS_ON_TC):
        print("\ntensor-core head %5d x %4d: error / fp32 distance %.2f (bar factor %d)" % (V, C, TC_NEEDED[(V, C)], tc_factor(dict(M=V, K=C))),
              end="")
    print()


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def launch_key(l):
    fam, nc, only, has_ln, npad, cluster = l
    return {"streaming": (fam, nc, only, has_ln), "generic": (fam, nc), "tensor_cores": (fam, npad, "cluster", cluster),
            "kquant": (fam, nc, only)}.get(fam, (fam,))


def check(family, name, got, r64, r32, factor, shape=None):
    assert not np.isnan(got).any(), (family, name, "NaN left in the output")
    ratio = kr.error_over_bar(got, r64, r32, factor)
    WORST[family] = max(WORST[family], ratio)
    err, d32 = np.abs(got - r64).max(axis=0), np.abs(r32 - r64).max(axis=0)
    needed = float((err / np.maximum(d32, 1e-30))[err > kr.bar(r64, r32, 0)].max(initial=0))
    NEEDED[family] = max(NEEDED[family], needed)
    if family.startswith("tensor_cores"):
        TC_NEEDED[shape] = max(TC_NEEDED[shape], needed)
    assert ratio <= 1, (family, name, ratio, np.abs(got - r64).max())


def run_and_check(lib, shape, name, T, probs, xs, path, sms, tc_family="tensor_cores"):
    """Runs the batch, checks it and returns its outputs and launch record; tensor-core outputs count towards tc_family."""
    outs, launches = kh.gemv_batch(lib, T, probs, xs, path)
    for o in outs:
        assert o.guard_intact(), (name, "write past the end of an output")
    assert observed(launches) == expected_launches(T, probs, path, sms), (name, launches)
    KEYS[shape].update(launch_key(l) for l in launches if l[0] not in ("expand", "kquant_expand", "convert"))
    fams = {l[0] for l in launches}
    for j, (p, o) in enumerate(zip(probs, outs)):
        tc = takes_tc(p, T, path)
        fam = tc_family if tc else "kquant" if p["fmt"] in KQ_BYTES else "generic" if "generic" in fams else "streaming"
        # every row was written (no NaN of the 0xFF fill anywhere), before the float64 comparison of the sampled rows
        assert not np.isnan(o.cols(p["M"])).any(), (name, p["fmt"], p["M"], p["K"], "NaN left in the output")
        rows = sample_rows(p, T, path, probs, sms, tg.rng_for("rows", name, j))
        sub = row_subset(p, rows)
        got = o.cols(p["M"])[rows]
        check(fam, (name, p["fmt"], p["M"], p["K"], p["epi"]), got, reference(sub, xs, F64, tc), reference(sub, xs, F32, tc),
              tc_factor(p) if tc else 4, (p["M"], p["K"]))
    return outs, launches


# ---- A. the matrix kernels at every shape ------------------------------------------------------------------------------------

ROUTES = [("engine", 1), ("engine", 3), ("engine", 31), ("engine", 32), ("engine", 128), ("engine", 256),
          ("engine_batch_ctx", 5), ("engine_batch_ctx", 15), ("engine_batch_ctx", 16), ("engine_batch_ctx", 64), ("engine_batch_ctx", 256)]
ROTATION_ROUTES = [("engine", 1), ("engine", 31), ("engine", 128), ("engine_batch_ctx", 15), ("engine_batch_ctx", 64)]
GEMV_CASES = [(s.name, f, path, T) for s in SHAPES for f in formats(s) for path, T in (ROUTES if f in CORE_FORMATS else ROTATION_ROUTES)]


@pytest.mark.parametrize("shape,fmt,path,T", GEMV_CASES)
def test_engine_batches_at_model_shape(lib, sms, shape, fmt, path, T):
    s = BY_NAME[shape]
    for batch in engine_batches(s):
        rng = tg.rng_for("shape-batch", shape, fmt, batch, path, T)
        probs, xs = build(s, fmt, batch, T, rng)
        run_and_check(lib, shape, (shape, fmt, batch, path, T), T, probs, xs, path, sms)
    RAN.add((shape, "gemv", fmt, path, T))


# The GEMV with its LayerNorm prologue: a single token; the GEMV-head scoring passes of a single context (up to 31 tokens with tensor
# cores on, up to 256 with them off); batch contexts of 4 .. 256 sequences, whose head the tensor cores never take (they refuse the
# prologue).
HEAD_ROUTES = [("engine", 1), ("engine", 31), ("engine", 256), ("engine_batch_ctx", 4), ("engine_batch_ctx", 20), ("engine_batch_ctx", 64),
               ("engine_batch_ctx", 256)]


@pytest.mark.parametrize("shape", [s.name for s in SHAPES])
@pytest.mark.parametrize("fmt", ["FP16", "FP32"])
def test_head_at_model_shape(lib, sms, head, shape, fmt):
    """LN(x; ln_out) . W at the shape's real vocabulary (engine.cu's head and the GEMV head of score_head) on every route of
    HEAD_ROUTES. Beyond 64 columns ln_b keeps the fp16 operands of every column four times the kernel's own LayerNorm error away from
    a tie instead of a hundredth of an fp16 spacing, which no ln_b achieves for 256 columns at once."""
    s = BY_NAME[shape]
    for path, T in HEAD_ROUTES:
        rng = tg.rng_for("shape-head", shape, fmt, path, T)
        xs = tg.inputs([s.C], T, rng, scale=1.5)
        p = problem(fmt, s.V, s.C, T, rng, tiled=False, raw=head(fmt, s.V, s.C))
        tg.with_layernorm(p, xs[0], rng, kernel_error=T > 64)
        run_and_check(lib, shape, (shape, "head", fmt, path, T), T, [p], xs, path, sms)
        RAN.add((shape, "head", fmt, path, T))


# Columns of the tensor-core head: a batch context's smallest passes (16, 17) and a single context's (32 and up), ragged ones included.
SCORE_HEAD_T = [16, 17, 32, 33, 100, 256]


def score_head_targets(V, T, rng):
    """Targets of a [T, V] pass: every column's argmax is scored separately (score_head_case); these mix positions without a target,
    rows of the last row tile (101 rows at V = 50277) and any row."""
    last = (V - 1) // 128 * 128
    return [NO if t % 3 == 0 else int(rng.integers(last, V)) if t % 3 == 1 else int(rng.integers(0, V)) for t in range(T)]


@pytest.mark.parametrize("shape", [s.name for s in SHAPES])
def test_score_head_at_model_shape(lib, sms, head, shape):
    """score_head on the tensor cores at the shape's real vocabulary: layer_norm_columns (through its hook), then the FP16 head from
    its tile-major copy (gemm_tc_repack, as ensure_head_tiled builds it) on the tensor cores, then the score kernel on the [T, V]
    logits. The GEMM is checked as every tensor-core launch of this file is (launch record, no NaN anywhere, the sampled rows -- all
    of the first and last tile and both edges of every tile -- against float64), and the score kernel against float64 log_softmax of
    the logits the GEMM returned, so a GEMM error cannot hide one of the score kernel."""
    s = BY_NAME[shape]
    HEADS_ON_TC.add((s.V, s.C))
    for T in SCORE_HEAD_T:
        rng = tg.rng_for("shape-score-head", shape, T)
        x = tg.inputs([s.C], T, rng, scale=1.5)[0]
        w, b = (1 + 0.2 * rng.standard_normal(s.C)).astype(F32), (0.2 * rng.standard_normal(s.C)).astype(F32)
        ln = kh.layer_norm_columns(lib, x, w, b)
        assert ln.guard_intact() and not np.isnan(ln.value).any(), (shape, T)
        p = problem("FP16", s.V, s.C, T, rng, tiled=True, raw=head("FP16", s.V, s.C))
        (out,), launches = run_and_check(lib, shape, (shape, "score_head", T), T, [p], [ln.cols(s.C).copy()], "tensor_cores", sms,
                                         tc_family="tensor_cores_head")
        assert launches[0] == ("expand", 0, TYPE["FP16"], 0, 0, 0), launches       # the tile-major upload
        logits = out.value.reshape(T, s.V)
        for targets in ([int(a) for a in logits.argmax(axis=1)], score_head_targets(s.V, T, rng)):
            lp, g = score_logits(lib, logits, targets)
            check_rows(lp, g, logits, targets)
        RAN.add((shape, "score_head", T))


# ---- A.4 the state kernels at the same shapes --------------------------------------------------------------------------------

def state_check(name, got, r64, r32):
    r64, r32 = np.asarray(r64, F64), np.asarray(r32, F64)
    check(name, name, np.asarray(got, F64).reshape(r64.shape), r64, r32, 4)


def att_ln_form(s):
    """(formula, n_out) of the time-mixing ln_mix launch (engine.cu att_ln)."""
    return {4: (0, 3), 5: (0, 4), 6: (1, 1), 7: (1, 6)}[s.arch[0]]


@pytest.mark.parametrize("shape", [s.name for s in SHAPES])
def test_ln_mix_at_model_shape(lib, shape):
    s = BY_NAME[shape]
    formula, n_out = att_ln_form(s)
    for T in (1, 31, 256):
        x, w, b, state, coefs = ln_mix_inputs(s.C, T, n_out, tg.rng_for("shape-ln", shape, T))
        o = kh.ln_mix(lib, x, w, b, state, coefs, formula)
        assert all(v.guard_intact() for v in o.values())
        r64, r32 = kr.ln_mix(x, w, b, state, coefs, formula, F64), kr.ln_mix(x, w, b, state, coefs, formula, F32)
        for j in range(n_out):
            state_check("ln_mix", o["out%d" % j].cols(s.C), r64[0][j], r32[0][j])
        state_check("ln_mix", o["state"].value, r64[3], r32[3])
    n = 16
    x, w, b, _, coefs = ln_mix_inputs(s.C, n, n_out, tg.rng_for("shape-ln-b", shape))
    stride = s.C + 32
    states = tg.rng_for("shape-ln-bs", shape).standard_normal((n - 1) * stride + s.C).astype(F32)
    o = kh.ln_mix(lib, x, w, b, states, coefs, formula, n_seq=n, seq_stride=stride)
    assert all(v.guard_intact() for v in o.values())
    for q in range(n):
        carry = states[q * stride:q * stride + s.C]
        r64, r32 = (kr.ln_mix(x[:, q:q + 1], w, b, carry, coefs, formula, dt) for dt in (F64, F32))
        for j in range(n_out):
            state_check("ln_mix_batch", o["out%d" % j].cols(s.C)[:, q:q + 1], r64[0][j], r32[0][j])
        state_check("ln_mix_batch", o["state"].value[q * stride:q * stride + s.C], r64[3], r32[3])
    RAN.add((shape, "ln_mix"))


@pytest.mark.parametrize("shape", [s.name for s in SHAPES])
def test_wkv_at_model_shape(lib, shape):
    """wkv4 at every v4 C; wkv6 (v5.2 per-channel decay, v6 per-token decay) and wkv7 at H = C / 64; T = 1 / 32 / 256 and a batch of 16."""
    s = BY_NAME[shape]
    a = s.arch[0]
    for T in (1, 32, 256, "batch"):
        cols = 16 if T == "batch" else T
        rng = tg.rng_for("shape-wkv", shape, T)
        if a == 4:
            d = wkv4_inputs(s.C, cols, rng, False)
            if T == "batch":
                stride = s.C + 8
                st = {k: np.tile(np.concatenate([d[k], np.zeros(8, F32)]), 16)[:15 * stride + s.C] for k in ("aa", "bb", "pp")}
                o = run_wkv4(lib, dict(d, **st), n_seq=16, seq_stride=stride)
                y64, y32 = np.empty((s.C, 16)), np.empty((s.C, 16))
                for q in range(16):
                    one = dict(d, k=d["k"][:, q:q + 1], v=d["v"][:, q:q + 1], r=d["r"][:, q:q + 1])
                    y64[:, q:q + 1], y32[:, q:q + 1] = ref_wkv4(one, F64)[0], ref_wkv4(one, F32)[0]
                state_check("wkv4", o["y"].cols(s.C), y64, y32)
            else:
                o = run_wkv4(lib, d)
                r64, r32 = ref_wkv4(d, F64), ref_wkv4(d, F32)
                state_check("wkv4", o["y"].cols(s.C), r64[0], r32[0])
                for i, k in enumerate(("aa", "bb", "pp")):
                    state_check("wkv4", o[k].value, r64[1 + i], r32[1 + i])
        elif a in (5, 6):
            mode = "v5.2" if a == 5 else "v6"
            d = wkv6_inputs(mode, s.C // 64, 64, cols, rng)
            if T == "batch":
                SS = s.C * 64
                o = run_wkv6(lib, dict(d, state=np.tile(d["state"], 16)), mode, n_seq=16, seq_stride=SS)
                for q in range(16):
                    one = {k: (v[:, q:q + 1] if k in ("r", "k", "v", "g") or (k == "td" and mode == "v6") else v) for k, v in d.items()}
                    r64, r32 = ref_wkv6(one, F64), ref_wkv6(one, F32)
                    state_check("wkv6", o["y"].cols(s.C)[:, q:q + 1], r64[0], r32[0])
                    state_check("wkv6", o["state"].value[q * SS:(q + 1) * SS], r64[1], r32[1])
            else:
                o = run_wkv6(lib, d, mode)
                r64, r32 = ref_wkv6(d, F64), ref_wkv6(d, F32)
                state_check("wkv6", o["y"].cols(s.C), r64[0], r32[0])
                state_check("wkv6", o["state"].value, r64[1], r32[1])
        else:
            d = wkv7_inputs(s.C // 64, 64, cols, rng, True)
            if T == "batch":
                SS = s.C * 64
                o = run_wkv7(lib, dict(d, state=np.tile(d["state"], 16)), n_seq=16, seq_stride=SS)
                for q in range(16):
                    one = {k: (v[:, q:q + 1] if k in ("r", "w", "k", "v", "aa", "g", "vgate", "v_first") else v) for k, v in d.items()}
                    r64, r32 = ref_wkv7(one, F64), ref_wkv7(one, F32)
                    state_check("wkv7", o["y"].cols(s.C)[:, q:q + 1], r64[0], r32[0])
                    state_check("wkv7", o["state"].value[q * SS:(q + 1) * SS], r64[2], r32[2])
            else:
                o = run_wkv7(lib, d)
                r64, r32 = ref_wkv7(d, F64), ref_wkv7(d, F32)
                state_check("wkv7", o["y"].cols(s.C), r64[0], r32[0])
                state_check("wkv7", o["state"].value, r64[2], r32[2])
        assert all(v.guard_intact() for v in o.values())
    RAN.add((shape, "wkv"))


V6 = [s.name for s in SHAPES if s.arch[0] == 6]
FOLD_FORMATS = ["FP32", "FP16", "Q4_0", "Q4_1", "Q5_0", "Q5_1", "Q8_0", "Q4_K", "Q5_K"]


@pytest.mark.parametrize("shape", V6)
def test_v6_lerp_at_model_shape(lib, shape):
    s = BY_NAME[shape]
    for T in (1, 8, 32):
        w2, z, xx, sx, maa = lerp_inputs(s.C, T, s.mix, tg.rng_for("shape-lerp", shape, T))
        o = kh.v6_lerp(lib, w2, z, xx, sx, maa)
        assert all(v.guard_intact() for v in o.values())
        r64, r32 = kr.v6_lerp(w2, z, xx, sx, maa, F64), kr.v6_lerp(w2, z, xx, sx, maa, F32)
        for j in range(5):
            state_check("v6_lerp", o["out%d" % j].cols(s.C), r64[j], r32[j])
    RAN.add((shape, "v6_lerp"))


def fold_expected(s, fmt):
    """Where rwkv_b200_v6_lora_fold_supported admits a v6 layer of this file: both LoRA matrices legacy / F16 / F32 rows that one warp
    of the streaming plan owns (WK = 1), n_embed <= 4096 and a decay rank of 32 .. 128."""
    t = file_types(s, fmt)
    w1, w2 = t["att.time_maa_w1"], t["att.time_decay_w2"]
    legacy = lambda f: f not in KQ_BYTES
    return (legacy(w1) and legacy(w2) and s.C <= 4096 and 32 <= s.decay <= 128 and plan_wk(w1, s.C) == 1 and plan_wk(w2, s.decay) == 1)


@pytest.mark.parametrize("shape", V6)
@pytest.mark.parametrize("fmt", FOLD_FORMATS)
def test_v6_fold_at_model_shape(lib, shape, fmt):
    """v6_prologue and wkv6_decay against the unfused pair, bit for bit, wherever the fold predicate admits the file's shape."""
    from test_v6_fold_host import V6PrologueArgs, Wkv6DecayArgs
    s = BY_NAME[shape]
    t = file_types(s, fmt)
    w1t, w2t = TYPE[t["att.time_maa_w1"]], TYPE[t["att.time_decay_w2"]]
    ok = bool(lib.library.rwkv_b200_v6_lora_fold_supported(s.C, 64, w1t, s.mix, w2t, s.decay))
    assert ok == fold_expected(s, fmt), (shape, fmt, ok)
    RAN.add((shape, "v6_fold", fmt))
    if not ok:
        return
    C, M1, rng = s.C, 5 * s.mix, tg.rng_for("shape-fold", shape, fmt)
    vec = lambda *shape_, scale=1.0: (rng.standard_normal(shape_) * scale).astype(F32)
    x, lw, lb, st, coef = vec(C, 1, scale=3.0), 1 + vec(C, scale=0.1), vec(C, scale=0.1), vec(C), rng.uniform(0, 1, C).astype(F32)
    _, raw = tg.random_raw(t["att.time_maa_w1"], M1, C)
    ref = kh.ln_mix(lib, x, lw, lb, st, [coef], 1)
    (y_ref,), _ = kh.gemv_batch(lib, 1, [dict(type=w1t, K=C, M=M1, raw=raw, epi=3)], [ref["out0"].cols(C)])
    i = kh.Inputs()
    o = {k: kh.Out(n) for k, n in (("state", C), ("xx", C), ("sx", C), ("y1", M1))}
    i.keep.append(raw)
    a = V6PrologueArgs(x=i(x[:, 0]), ln_w=i(lw), ln_b=i(lb), state_in=i(st), coef=i(coef), state_out=o["state"].ptr, out_xx=o["xx"].ptr,
                       out_sx=o["sx"].ptr, w1=raw.ctypes.data, w1_type=w1t, M1=M1, y1=o["y1"].ptr, C=C)
    kh._call(lib, lib.library.rwkv_b200_test_v6_prologue, a)
    for k, r in (("state", ref["state"]), ("xx", ref["xx"]), ("sx", ref["sx"]), ("y1", y_ref)):
        assert o[k].guard_intact() and o[k].value.tobytes() == r.value.tobytes(), (k, np.abs(o[k].value - r.value).max())
    H = C // 64
    r, k, v, g = vec(C, 1), vec(C, 1), vec(C, 1), vec(C, 1)
    tf, lw, lb, st = vec(C, scale=0.3), 1 + vec(C, scale=0.1), vec(C, scale=0.1), vec(C * 64)
    lora1, td_bias = np.tanh(vec(s.decay, 1)), vec(C, scale=0.5) - 1.0
    _, raw2 = tg.random_raw(t["att.time_decay_w2"], C, s.decay)
    (w,), _ = kh.gemv_batch(lib, 1, [dict(type=w2t, K=s.decay, M=C, raw=raw2, epi=7, bias=td_bias)], [lora1])
    ref = kh.wkv6(lib, r, k, v, w.cols(C), tf, st, lw, lb, g, 64e-5, H, 64, True, False)
    o = {"state": kh.Out(st.size), "y": kh.Out(C)}
    i.keep.append(raw2)
    a = Wkv6DecayArgs(r=i(r[:, 0]), k=i(k[:, 0]), v=i(v[:, 0]), tf=i(tf), state_in=i(st), state_out=o["state"].ptr, lnx_w=i(lw), lnx_b=i(lb),
                      g=i(g[:, 0]), y=o["y"].ptr, eps=64e-5, H=H, w2=raw2.ctypes.data, w2_type=w2t, K2=s.decay, lora1=i(lora1[:, 0]),
                      td_bias=i(td_bias))
    kh._call(lib, lib.library.rwkv_b200_test_wkv6_decay, a)
    for key in ("state", "y"):
        assert o[key].guard_intact() and o[key].value.tobytes() == ref[key].value.tobytes(), (key, np.abs(o[key].value - ref[key].value).max())


# ---- B. engine invariants on one-layer files of real shapes ------------------------------------------------------------------

# the smallest and largest shape of each architecture in Q5_1; RWKV-4 14B in FP16, whose 40 KB ffn.value rows take the generic kernel
ONE_LAYER = [("rwkv4-169m", "Q5_1"), ("rwkv4-14b", "FP16"), ("rwkv5-0b4", "Q5_1"), ("rwkv5-7b", "Q5_1"), ("rwkv6-1b6", "Q5_1"),
             ("rwkv6-7b", "Q5_1"), ("rwkv7-0b1", "Q5_1"), ("rwkv7-2b9", "Q5_1")]
E2E_TOL = {"FP16": 5e-3, "Q5_1": 5e-2}      # test_gpu_full_shape.py's logit bars; states within 20 times that


def evaluate_serial(lib, ctx, toks, n_state, n_logits):
    """[(state, logits) after each token] of rwkv_eval token by token."""
    P = ctypes.POINTER(ctypes.c_float)
    state, logits, out = np.zeros(n_state, F32), np.zeros(n_logits, F32), []
    for i, t in enumerate(toks):
        assert lib.library.rwkv_eval(ctx.ptr, t, None if i == 0 else state.ctypes.data_as(P), state.ctypes.data_as(P), logits.ctypes.data_as(P))
        out.append((state.copy(), logits.copy()))
    return out


@pytest.mark.parametrize("shape,fmt", ONE_LAYER)
def test_one_layer_file_invariants(lib, tmp_path, shape, fmt):
    """One layer at the real C / F / V through the engine: serial == eval_sequence == chunks of 7 and 31 bit for bit; a batch of 5
    == each sequence alone bit for bit; a 128-token chunk and a batch of 16 (tensor cores) within the end-to-end bars of serial; the
    single-token pass of a v6 layer runs v6_prologue exactly where the fold predicate admits the file. Batch contexts take n_embed <=
    4096, so at the 14B shape the batch checks become a check that batch_create refuses it."""
    import synthetic_model as sm
    from test_gpu_batch import alone, check_batch
    from test_gpu_v6_fused import traced_names
    P = ctypes.POINTER(ctypes.c_float)
    s = BY_NAME[shape]
    path = str(tmp_path / ("%s-%s.bin" % (shape, fmt)))
    sm.write_direct(path, preset(s), fmt, seed=11)
    tol = E2E_TOL[fmt]
    ctx = lib.rwkv_init_from_file(path, 1, 0)
    try:
        n_state, n_logits = lib.rwkv_get_state_buffer_element_count(ctx), lib.rwkv_get_logits_buffer_element_count(ctx)
        assert n_logits == s.V
        toks = [(7919 * i + 11) % s.V for i in range(128)]
        serial = evaluate_serial(lib, ctx, toks, n_state, n_logits)
        assert all(np.isfinite(a).all() for a in serial[-1]) and serial[-1][1].std() > 0
        arr = (ctypes.c_uint32 * len(toks))(*toks)
        st, lg = np.zeros(n_state, F32), np.zeros(n_logits, F32)
        # below 32 tokens a pass stays off the tensor cores: bit for bit
        assert lib.library.rwkv_eval_sequence(ctx.ptr, arr, 31, None, st.ctypes.data_as(P), lg.ctypes.data_as(P))
        assert st.tobytes() == serial[30][0].tobytes() and lg.tobytes() == serial[30][1].tobytes(), "eval_sequence"
        for chunk in (7, 31):
            assert lib.library.rwkv_eval_sequence_in_chunks(ctx.ptr, arr, 40, chunk, None, st.ctypes.data_as(P), lg.ctypes.data_as(P))
            assert st.tobytes() == serial[39][0].tobytes() and lg.tobytes() == serial[39][1].tobytes(), chunk
        # one 128-token chunk: the tensor-core prefill
        assert lib.library.rwkv_eval_sequence_in_chunks(ctx.ptr, arr, 128, 128, None, st.ctypes.data_as(P), lg.ctypes.data_as(P))
        err, serr = float(np.abs(lg - serial[-1][1]).max()), float(np.abs(st - serial[-1][0]).max())
        print("\n%s %s: 128-token chunk - serial: logits %.2e, state %.2e" % (shape, fmt, err, serr), end="")
        assert err <= tol and serr <= 20 * tol, (err, serr)
        if s.arch[0] == 6:
            names = traced_names(lib, ctx, toks[0])
            assert names.count("v6_prologue") == int(fold_expected(s, fmt)), names
        score_at_real_vocabulary(lib, ctx, toks, serial, tol)
        if s.C > 4096:      # batch contexts take n_embed <= 4096 (rwkv_b200_batch_create): the 14B shape is refused
            assert not lib.library.rwkv_b200_batch_create(ctx.ptr, 16)
            assert lib.rwkv_get_last_error(None) & ((6 << 8) | 9) == (6 << 8) | 9      # RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED
            RAN.add((shape, "one_layer", fmt))
            return
        # a batch context of 16 sequences, 3 tokens each: its passes take the tensor cores
        n_seq, steps = 16, 3
        prompts = [[(131 * b + 977 * i + 5) % s.V for i in range(steps)] for b in range(n_seq)]
        want = [alone(lib, ctx, q, n_state, n_logits) for q in prompts]
        batch = ctypes.c_void_p(lib.library.rwkv_b200_batch_create(ctx.ptr, n_seq))
        assert batch.value, "batch_create failed"
        try:
            for step in range(steps):
                assert lib.library.rwkv_b200_batch_eval(batch, (ctypes.c_uint32 * n_seq)(*[q[step] for q in prompts]), True)
            for b in range(n_seq):
                assert lib.library.rwkv_b200_batch_get_logits(batch, b, lg.ctypes.data_as(P))
                assert lib.library.rwkv_b200_batch_get_state(batch, b, st.ctypes.data_as(P))
                err, serr = float(np.abs(lg - want[b][0][-1]).max()), float(np.abs(st - want[b][1]).max())
                assert err <= tol and serr <= 20 * tol, (b, err, serr)
        finally:
            lib.library.rwkv_free(batch)
    finally:
        lib.rwkv_free(ctx)
    check_batch(lib, path, n_seq=5, n_steps=5)            # a batch of 5 == each sequence alone, bit for bit
    # ragged scoring passes: below 16 columns the GEMV head, bit for bit each sequence alone; from 16 on the tensor-core head
    ragged_case(lib, path, [3, 0, 5, 1, 0, 6], tensor_cores=True, exact=True)
    ragged_case(lib, path, [20, 0, 13, 1], tensor_cores=True, exact=False, bar=2 * tol)
    RAN.add((shape, "one_layer", fmt))


def score_at_real_vocabulary(lib, ctx, toks, serial, tol):
    """rwkv_b200_score over the 128 tokens from a fresh state, tensor cores on. In calls below 32 tokens (the GEMV head): the bits
    rwkv_b200_score_logits gives on the serial logits, and the last serial logits left resident. In one call (the tensor-core head,
    trace ending layer_norm_columns, convert_f16, gemm_tc, score): within twice the end-to-end logits bar of float64 log_softmax over
    the serial logits (the error of log p is at most that of z_t plus that of the logsumexp), and the state eval_resident leaves."""
    L = lib.library
    V = len(serial[0][1])
    ref = np.stack([lg for _, lg in serial])
    targets = text_targets(toks, V)
    has = np.array([t != NO for t in targets])

    def score(lo, hi):
        lp, g = np.full(hi - lo, SENTINEL, F32), np.full(hi - lo, 7, np.uint8)
        assert L.rwkv_b200_score(ctx.ptr, u32(toks[lo:hi]).ctypes.data_as(P_U), u32(targets[lo:hi]).ctypes.data_as(P_U), hi - lo,
                                 lp.ctypes.data_as(P_F), g.ctypes.data_as(P_U8)), L.rwkv_get_last_error(ctx.ptr)
        return lp, g

    def state():
        st = np.zeros(len(serial[0][0]), F32)
        assert L.rwkv_b200_state_store(ctx.ptr, st.ctypes.data_as(P_F))
        return st
    L.rwkv_b200_set_tensor_cores(ctx.ptr, True)
    want_lp, want_g = score_logits(lib, ref, targets)
    assert L.rwkv_b200_state_load(ctx.ptr, None)
    parts, off = [], 0
    for n in (31, 1, 20, 18, 31, 27):
        parts.append(score(off, off + n))
        off += n
    assert off == len(toks)
    assert bits(np.concatenate([a for a, _ in parts])) == bits(want_lp) and bits(np.concatenate([g for _, g in parts])) == bits(want_g)
    lg = np.zeros(V, F32)
    assert L.rwkv_b200_stage_logits(ctx.ptr, lg.ctypes.data_as(P_F), None)
    assert bits(lg) == bits(serial[-1][1]), "resident logits"
    # the tensor-core head
    assert L.rwkv_b200_state_load(ctx.ptr, None)
    assert L.rwkv_b200_eval_resident(ctx.ptr, u32(toks).ctypes.data_as(P_U), len(toks), True, None)
    want_state = state()
    assert L.rwkv_b200_state_load(ctx.ptr, None) and L.rwkv_b200_trace_enable(ctx.ptr)
    lp, g = score(0, len(toks))
    names = score_trace(types.SimpleNamespace(L=L, ptr=ctx.ptr))
    L.rwkv_b200_trace_disable(ctx.ptr)
    assert names[-4:] == ["layer_norm_columns", "convert_f16", "gemm_tc", "score"], names[-6:]
    err = np.abs(lp[has].astype(F64) - lp64(ref, np.where(has, targets, 0))[has])
    print(" score on the tensor cores - float64 over serial: %.2e" % err.max(), end="")
    assert np.isfinite(lp[has]).all() and err.max() <= 2 * tol, err.max()
    assert (lp[~has] == SENTINEL).all() and (g[~has] == 7).all()
    assert bits(state()) == bits(want_state), "state after scoring on the tensor cores"


# ---- A.6 every (shape, route) of the table ran ---------------------------------------------------------------------------------

def test_every_shape_and_route_ran(request):
    """Runs last: every (shape, format, route) of GEMV_CASES, every head route (the GEMV ones and the tensor-core one of scoring), every
    state kernel of every shape and every one-layer file ran. Prints the launch keys each shape reached. A run of part of the file (-k, a node id) skips it."""
    n_items = len(GEMV_CASES) + 5 * len(SHAPES) + len(V6) * (1 + len(FOLD_FORMATS)) + len(ONE_LAYER) + 1
    if sum(i.fspath == request.node.fspath for i in request.session.items) < n_items:
        pytest.skip("only part of the file was selected")
    want = {(sh, "gemv", f, p, T) for sh, f, p, T in GEMV_CASES}
    want |= {(s.name, "head", f, p, T) for s in SHAPES for f in ("FP16", "FP32") for p, T in HEAD_ROUTES}
    want |= {(s.name, "score_head", T) for s in SHAPES for T in SCORE_HEAD_T}
    want |= {(s.name, k) for s in SHAPES for k in ("ln_mix", "wkv")} | {(n, "v6_lerp") for n in V6}
    want |= {(n, "v6_fold", f) for n in V6 for f in FOLD_FORMATS} | {(n, "one_layer", f) for n, f in ONE_LAYER}
    for s in SHAPES:
        print("\n%-11s %s" % (s.name, " ".join(str(k) for k in sorted(KEYS[s.name], key=str))), end="")
    print()
    assert want <= RAN, sorted(want - RAN)[:20]

