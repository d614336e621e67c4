"""The shape table of tests/test_gpu_model_shapes.py without a GPU: it reproduces the presets of tools/synthetic_model.py and the
types the quantiser writes, the fold predicate agrees with it at every v6 shape, and at every shape's bar each plausible planning
defect, injected into the float64 restatement, lands above the bar."""
import struct

import numpy as np
import pytest

import ggml_file as gf
import kernel_ref as kr
import synthetic_model as sm
import test_gpu_gemv as tg
import test_gpu_model_shapes as ms

F32, F64 = np.float32, np.float64


def test_table_reproduces_the_baseline_presets():
    for preset, name in (("rwkv4-169m", "rwkv4-169m"), ("rwkv5-1b5", "rwkv5-1b5"), ("rwkv6-7b", "rwkv6-7b"), ("rwkv7-2b9", "rwkv7-2b9")):
        p, s = sm.PRESETS[preset], ms.BY_NAME[name]
        assert (p["arch"], p["C"], p["F"], p["V"], p.get("S", 0)) == (s.arch, s.C, s.F, s.V, s.S), preset
        assert (p.get("mix", 0), p.get("decay", 0)) == (s.mix, s.decay), preset
        if s.lora:
            assert (p["lora_w"], p["lora_a"], p["lora_v"], p["lora_g"]) == (s.lora["w"], s.lora["a"], s.lora["v"], s.lora["g"]), preset
    assert ms.v7_lora(2560) == dict(w=96, a=96, v=64, g=320)
    assert len(ms.SHAPES) == 17 and all(s.F % 32 == 0 and s.C % 64 == 0 for s in ms.SHAPES)


def test_every_format_reaches_every_architecture_at_its_largest_shape():
    for a in (4, 5, 6, 7):
        big = ms.BY_NAME[ms.LARGEST[a]]
        assert set(ms.formats(big)) == set(ms.CORE_FORMATS + ms.ROTATION), a
    assert {f for s in ms.SHAPES for f in ms.formats(s)} == set(ms.CORE_FORMATS + ms.ROTATION)


def read_types(path):
    """{tensor name: type name} of a model file, K-quant records included."""
    names = {v: k for k, v in ms.TYPE.items()}
    buf = open(path, "rb").read()
    off, out = 24, {}
    while off < len(buf):
        n_dims, name_len, dtype = struct.unpack_from("<3I", buf, off)
        ne = struct.unpack_from("<%dI" % n_dims, buf, off + 12)
        off += 12 + 4 * n_dims
        name = buf[off:off + name_len].decode()
        off += name_len
        n = int(np.prod(ne))
        off += n // 256 * ms.KQ_BYTES[names[dtype]] if names[dtype] in ms.KQ_BYTES else gf.tensor_nbytes(dtype, ne)
        out[name] = names[dtype]
    return out


@pytest.mark.parametrize("name", ["rwkv4-169m", "rwkv5-0b4", "rwkv6-1b6", "rwkv7-0b1"])
@pytest.mark.parametrize("fmt", ["Q5_1", "Q4_K"])
def test_file_types_match_the_quantiser(lib, tmp_path, name, fmt):
    """A one-layer, small-vocabulary FP16 master at the real C / F, through rwkv_quantize_model_file: every 2-D tensor has the type
    file_types gives it."""
    s = ms.BY_NAME[name]
    preset = ms.preset(s, V=256)
    master, out = str(tmp_path / "master.bin"), str(tmp_path / "q.bin")
    sm.write_master(master, preset, "FP16", seed=1)
    lib.rwkv_quantize_model_file(master, out, fmt)
    got = read_types(out)
    want = ms.file_types(s, fmt)
    for tensor, t in got.items():
        key = tensor if tensor in want else tensor.split(".", 2)[-1]
        if key in want:
            assert t == want[key], (tensor, t, want[key])
    layer = {k.split(".", 2)[-1] for k in got if k.startswith("blocks.0.")}
    first = {"att.v1", "att.v2"} if s.arch[0] == 7 else set()      # v7's first layer has no value LoRA
    assert set(want) - {"emb.weight", "head.weight"} - first <= layer, sorted(set(want) - layer)


@pytest.mark.parametrize("shape", ms.V6)
@pytest.mark.parametrize("fmt", ms.FOLD_FORMATS)
def test_fold_predicate_at_every_v6_shape(lib, shape, fmt):
    s = ms.BY_NAME[shape]
    t = ms.file_types(s, fmt)
    got = lib.library.rwkv_b200_v6_lora_fold_supported(s.C, 64, ms.TYPE[t["att.time_maa_w1"]], s.mix, ms.TYPE[t["att.time_decay_w2"]], s.decay)
    assert bool(got) == ms.fold_expected(s, fmt), (shape, fmt, got)


# ---- planning defects at every shape's bar ------------------------------------------------------------------------------------

SMS = 132


def moved(p, xs, bugged, tc, rows):
    sub = ms.row_subset(p, rows)
    r64, r32 = ms.reference(sub, xs, F64, tc), ms.reference(sub, xs, F32, tc)
    return kr.error_over_bar(bugged, r64, r32, ms.tc_factor(p) if tc else 4)


def ffn_key(s, fmt, T):
    rng = tg.rng_for("bars-host", s.name, fmt, T)
    probs, xs = ms.build(s, fmt, "ffn_kr", T, rng)
    return probs[0], xs


@pytest.mark.parametrize("shape", [s.name for s in ms.SHAPES])
def test_neighbouring_row_tile_is_caught(shape):
    """Tensor cores, T = 32: row tile 1 of ffn.key written with tile 2's output."""
    s = ms.BY_NAME[shape]
    p, xs = ffn_key(s, "Q5_1", 32)
    rows = np.arange(128, 256)
    good = ms.reference(ms.row_subset(p, np.arange(256, 384)), xs, F64, True)
    assert moved(p, xs, good, True, rows) > 1


@pytest.mark.parametrize("shape", [s.name for s in ms.SHAPES])
def test_column_of_an_nc4_group_shifted_is_caught(shape):
    """SIMT, T = 31 (NC = 4 where it fits): column 1 of the first group written with column 2's output."""
    s = ms.BY_NAME[shape]
    p, xs = ffn_key(s, "Q5_1", 31)
    rows = np.arange(0, 128)
    r = ms.reference(ms.row_subset(p, rows), xs, F64, False)
    r[:, 1] = r[:, 2]
    assert moved(p, xs, r, False, rows) > 1


@pytest.mark.parametrize("shape", [s.name for s in ms.SHAPES])
def test_dropped_k_split_partial_is_caught(shape):
    """ffn.value alone at T = 32 (K = F) is cut over a cluster at every C: its last K-split dropped."""
    s = ms.BY_NAME[shape]
    rng = tg.rng_for("bars-ksplit", shape)
    probs, xs = ms.build(s, "Q5_1", "ffn_value", 32, rng)
    npad, cluster, splits = ms.tc_plan(32, probs, SMS)
    assert cluster > 1 and splits == [cluster], (shape, cluster)
    rows = np.arange(0, 128)
    sub = ms.row_subset(probs[0], rows)
    bugged = ms.reference(sub, xs, F64, True, bug="drop_last_ksplit", ksplit=cluster)
    assert moved(probs[0], xs, bugged, True, rows) > 1


def lora_problems(s):
    """(problem, inputs) of the LoRA rows a layer has: v7's second halves (F16), v6's decay_w2 (Q5_1) and maa_w1 (Q4_K super-blocks)."""
    if s.arch[0] == 7:
        probs, xs = ms.build(s, "Q5_1", "lora_second", 1, tg.rng_for("bars-lora", s.name))
        return [(p, xs) for p in probs]
    if s.arch[0] == 6:
        out = []
        for fmt, batch in (("Q5_1", "decay_w2"), ("Q4_K", "maa_w1")):
            probs, xs = ms.build(s, fmt, batch, 1, tg.rng_for("bars-lora", s.name, fmt))
            out.append((probs[0], xs))
        return out
    return []


@pytest.mark.parametrize("shape", [s.name for s in ms.SHAPES if s.arch[0] in (6, 7)])
def test_dropped_last_block_of_a_lora_row_is_caught(shape):
    s = ms.BY_NAME[shape]
    for p, xs in lora_problems(s):
        rows = np.arange(min(p["M"], 256))
        sub = ms.row_subset(p, rows)
        bugged = ms.reference(sub, xs, F64, False, bug="drop_last_block")
        assert moved(p, xs, bugged, False, rows) > 1, (p["fmt"], p["M"], p["K"])


def test_host_plan_matches_the_documented_routes():
    """The host restatement of the plan on shapes the kernels' comments name: 28 KB F16 rows (K = 14336) and 40 KB ones (K = 20480)
    take the generic kernel, a 14B ffn.value in Q5_K runs one CTA per SM, 40 tiles cluster by 2."""
    s = ms.BY_NAME["rwkv4-14b"]
    f16 = lambda K: dict(fmt="FP16", K=K, M=64, type=1)
    assert ms.streaming_plan(1, [f16(14336)]) is None and ms.streaming_plan(1, [f16(20480)]) is None
    assert ms.streaming_plan(1, [f16(4096)])[0] == 1
    assert ms.kquant_plan(1, [dict(fmt="Q5_K", K=s.F, M=s.C)])[2] == 1
    assert ms.tc_plan(32, [dict(M=5120, K=20480)], SMS)[1] == 2
    assert ms.tc_plan(32, [dict(M=768, K=3072)], SMS)[1] == 8
    assert ms.tc_plan(32, [dict(M=768, K=768)], SMS)[1] == 1          # 12 K-steps: too few for four per split of a cluster of 2+


# ---- the tensor-core head of scoring passes at every head shape ----------------------------------------------------------------

HEAD_SHAPES = sorted({(s.V, s.C) for s in ms.SHAPES})


def head_case(V, C, T, tiles):
    """Some row tiles of the head test_score_head_at_model_shape uploads, and an input of the same make: LayerNorm of columns of
    scale 1.5 with random w / b, here in float32 on the host."""
    rng = tg.rng_for("bars-head", V, C, T)
    x = tg.inputs([C], T, rng, scale=1.5)[0]
    w, b = (1 + 0.2 * rng.standard_normal(C)).astype(F32), (0.2 * rng.standard_normal(C)).astype(F32)
    _, raw = ms.head_raw("FP16", ms.head_weights(V, C, tiles))
    p = dict(type=ms.TYPE["FP16"], K=C, M=raw.size // (2 * C), raw=raw, input=0, epi=0, fmt="FP16", tiled=True)
    return p, [kr.layer_norm(x, w, b, F32).astype(F32)]


@pytest.mark.parametrize("V,C", HEAD_SHAPES)
@pytest.mark.parametrize("defect", ["neighbouring_row_tile", "shifted_npad_column", "drop_last_tile", "no_colscale"])
def test_head_defects_are_caught(V, C, defect):
    """At the head's own bar (tc_factor of V x C): row tile 1 written with tile 2's output (T = 32); column 1 of a 17-column pass (npad
    32) written with column 2's; the partial last row tile never written (101 rows at V = 50277); a column beyond the fp16 range
    without its power-of-two scale."""
    last = (V - 1) // 128
    T = {"shifted_npad_column": 17, "drop_last_tile": 33}.get(defect, 32)
    p, xs = head_case(V, C, T, [last] if defect == "drop_last_tile" else [1] if defect == "neighbouring_row_tile" else [0])
    if defect == "no_colscale":
        xs[0][:, 3] *= F32(3.0e5)
    r64, r32 = ms.reference(p, xs, F64, True), ms.reference(p, xs, F32, True)
    if defect == "neighbouring_row_tile":
        bugged = ms.reference(head_case(V, C, T, [2])[0], xs, F64, True)
    elif defect == "shifted_npad_column":
        bugged = r64.copy()
        bugged[:, 1] = bugged[:, 2]
    else:
        bugged = ms.reference(p, xs, F64, True, bug=defect)
    assert kr.error_over_bar(bugged, r64, r32, ms.tc_factor(dict(M=V, K=C))) > 1, (V, C, defect)
