"""Host side of the LoRA adapter tests (tests/test_gpu_lora.py, tests/test_lora_host.py): seeded adapters for a model file, the
float64 merge of an adapter into a model file, and the float64 restatement of the shrink / expand launches (csrc/kernels/lora.cu)."""
import numpy as np

import ggml_file
from ggml_file import ModelFile, Tensor, write_model_file

F32, F16 = 0, 1
# the layer matrices that take a low-rank delta (include/rwkv_b200.h: rwkv_b200_adapter_create)
DELTA_TARGETS = ("att.key.weight", "att.value.weight", "att.receptance.weight", "att.gate.weight", "att.output.weight",
                 "ffn.key.weight", "ffn.value.weight", "ffn.receptance.weight")
# epilogue ids of the test hook (csrc/kernels/gemv.h: GemvEpilogue)
EPI_NONE, EPI_SIGMOID, EPI_SILU, EPI_RELU_SQR, EPI_ADD, EPI_MUL_ADD = 0, 1, 2, 4, 5, 6


KQUANT_BLOCK = {13: (256, 144), 14: (256, 176)}     # Q4_K, Q5_K: weights and bytes per super-block


def read_model_file(path):
    """ggml_file.read_model_file, also for files with Q4_K / Q5_K tensors."""
    buf = np.fromfile(path, dtype=np.uint8)
    _, version, n_vocab, n_embed, n_layer, data_type = np.frombuffer(buf[:24].tobytes(), "<u4")
    off, tensors = 24, {}
    while off < len(buf):
        dim_count, key_len, dtype = np.frombuffer(buf[off:off + 12].tobytes(), "<u4")
        off += 12
        ne = tuple(int(v) for v in np.frombuffer(buf[off:off + 4 * dim_count].tobytes(), "<u4"))
        off += 4 * int(dim_count)
        name = bytes(buf[off:off + key_len]).decode("utf-8")
        off += int(key_len)
        blck, size = KQUANT_BLOCK.get(int(dtype)) or ggml_file.BLOCK[int(dtype)]
        nbytes = size * int(np.prod(ne)) // blck
        tensors[name] = Tensor(name, int(dtype), ne, buf[off:off + nbytes])
        off += nbytes
    return ModelFile(int(version), int(n_vocab), int(n_embed), int(n_layer), int(data_type), tensors)


def is_delta_target(name):
    return name.startswith("blocks.") and name.split(".", 2)[2] in DELTA_TARGETS


def matrix_shape(t):
    """(M, K) of a file tensor: K = ne0, M = ne1 * ne2."""
    return t.ne3[1] * t.ne3[2], t.ne3[0]


def f16(x):
    return np.asarray(x, np.float32).astype(np.float16).astype(np.float64)


def tensor_f32(t):
    """The values of an FP32 / FP16 file tensor as float32, in file order."""
    if t.dtype == F32:
        return np.frombuffer(t.raw.tobytes(), np.float32).copy()
    assert t.dtype == F16
    return np.frombuffer(t.raw.tobytes(), np.float16).astype(np.float32)


# matrices inside a layer that take no delta but may be replaced: the v6 / v7 LoRA weights RWKV-PEFT trains with the time_* parameters
REPLACED_MATRICES = ("att.time_maa_w1", "att.time_decay_w1", "att.time_decay_w2", "att.w1")


def is_replaced_matrix(name):
    return name.split(".", 2)[-1] in REPLACED_MATRICES


def make_entries(path, rank, seed, zero_b=False, vectors=False, b_scale=0.05, matrices=False, deltas=True):
    """Adapter entries (name, rank, A, B, values) for every delta target of the model file at `path`, A and B seeded; with
    vectors, also replacements of the LayerNorm and time_* / mixing vectors (the base values moved by a seeded offset); with
    matrices, also seeded replacements of the REPLACED_MATRICES the file has. deltas=False leaves the delta targets out."""
    rng = np.random.default_rng(seed)
    mf = read_model_file(path)
    out = []
    for name, t in mf.tensors.items():
        if matrices and is_replaced_matrix(name):
            M, K = matrix_shape(t)
            out.append((name, 0, None, None, (rng.standard_normal(M * K) * 0.5 * K ** -0.5).astype(np.float32)))
        elif is_delta_target(name):
            if not deltas:
                continue
            M, K = matrix_shape(t)
            a = (rng.standard_normal((rank, K)) * K ** -0.5).astype(np.float32)
            b = np.zeros((M, rank), np.float32) if zero_b else (rng.standard_normal((M, rank)) * b_scale).astype(np.float32)
            out.append((name, rank, a, b, None))
        elif vectors and t.dtype in (F32, F16) and len([d for d in t.ne if d > 1]) <= 1 and name not in ("emb.weight", "head.weight") and \
                any(s in name for s in ("ln", "time_mix", "time_maa_k", "time_first", "x_k", "k_k")):
            base = tensor_f32(t)
            out.append((name, 0, None, None, (base + rng.standard_normal(base.size) * 0.02).astype(np.float32)))
    return out


def merged_file(src, dst, entries, scale):
    """src (an FP32 file) with every entry applied in float64: W + scale * B16 . A16 for a delta (A and B rounded to fp16 as the
    library stores them), the values for a replacement; written as FP32."""
    mf = read_model_file(src)
    assert mf.data_type == F32 or all(t.dtype == F32 for t in mf.tensors.values())
    by_name = {e[0]: e for e in entries}
    tensors = []
    for name, t in mf.tensors.items():
        raw = t.raw
        if name in by_name:
            _, rank, a, b, values = by_name[name]
            if rank:
                M, K = matrix_shape(t)
                w = tensor_f32(t).astype(np.float64).reshape(M, K) + scale * (f16(b) @ f16(a))
                raw = w.astype(np.float32)
            else:
                raw = np.asarray(values, np.float32)
        tensors.append((name, t.dtype, t.ne, raw))
    write_model_file(dst, mf.n_vocab, mf.n_embed, mf.n_layer, mf.data_type, tensors, mf.version)


def epilogue64(epi, v, res=None, gate=None):
    if epi == EPI_SIGMOID:
        return 1.0 / (1.0 + np.exp(-v))
    if epi == EPI_SILU:
        return v / (1.0 + np.exp(-v))
    if epi == EPI_RELU_SQR:
        return np.maximum(v, 0.0) ** 2
    if epi == EPI_ADD:
        return res + v
    if epi == EPI_MUL_ADD:
        return res + gate * v
    return v


def lora_magnitude(a, b, x, z, gate, scale, epi):
    """Per output element, the sum of the magnitudes its fp32 arithmetic rounds: |A16| . |x| for u, and for y the magnitudes that
    reach the epilogue's argument, times the epilogue's slope there (relu^2: 2 |v| + 1; the others at most 1.1) plus |y|. A
    summation order's error is a small multiple of eps32 times this, whatever the order."""
    mu = np.abs(f16(a)) @ np.abs(x.astype(np.float64))
    md = abs(scale) * (np.abs(f16(b)) @ mu)
    if epi == EPI_MUL_ADD:
        md = np.abs(gate.astype(np.float64)) * md
    pre_mag = np.abs(z.astype(np.float64)) + md
    _, y = lora_ref(a, b, x, z, gate, scale, epi)
    if epi == EPI_RELU_SQR:
        pre = z.astype(np.float64) + scale * (f16(b) @ (f16(a) @ x.astype(np.float64)))
        return mu, pre_mag * (2 * np.abs(pre) + 1) + np.abs(y)
    return mu, 1.1 * pre_mag + np.abs(y)


def lora_ref(a, b, x, z, gate, scale, epi, dtype=np.float64):
    """The hook's result: u = A16 . x, then y = epi(z + scale * B16 . u) for the nonlinear epilogues, and z + scale * B16 . u /
    z + gate * (scale * B16 . u) for add / gated add (z being the base's output there). Column-major [dim, T] arrays in the
    restatement's dtype."""
    a16, b16 = f16(a).astype(dtype), f16(b).astype(dtype)
    x, z = x.astype(dtype), z.astype(dtype)
    u = a16 @ x
    d = dtype(scale) * (b16 @ u)
    if epi == EPI_ADD:
        y = z + d
    elif epi == EPI_MUL_ADD:
        y = z + gate.astype(dtype) * d
    else:
        y = epilogue64(epi, z + d)
    return u, y
