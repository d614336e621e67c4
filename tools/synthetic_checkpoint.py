"""Seeded synthetic RWKV checkpoints in PYTORCH layout (what BlinkDL's .pth files hold, before conversion): inputs for the
converter parity tests (tests/test_converter.py, tests/golden/make_converter_golden.py)."""
import torch

SHAPES = {
    "v4": dict(arch=(4, 0), C=64, F=256, L=2, V=50, H=0, S=0),
    "v5.1": dict(arch=(5, 1), C=64, F=224, L=2, V=50, H=8, S=8),
    "v5.2": dict(arch=(5, 2), C=64, F=224, L=2, V=50, H=8, S=8),
    "v6": dict(arch=(6, 0), C=128, F=448, L=2, V=50, H=2, S=64, mix=32, decay=64),
    "v7": dict(arch=(7, 0), C=128, F=512, L=3, V=50, H=2, S=64, lora_w=32, lora_a=32, lora_v=32, lora_g=64),
}


def make_state_dict(kind: str, seed: int = 0):
    p = SHAPES[kind]
    g = torch.Generator().manual_seed(seed)
    C, F, L, V, H, S = p["C"], p["F"], p["L"], p["V"], p["H"], p["S"]
    major, minor = p["arch"]

    def n(*shape, scale=1.0):
        return torch.randn(*shape, generator=g) * scale

    def u(*shape, lo=0.0, hi=1.0):
        return torch.rand(*shape, generator=g) * (hi - lo) + lo

    sd = {"emb.weight": n(V, C, scale=0.1)}
    for i in range(L):
        b = f"blocks.{i}."
        if i == 0:
            sd[b + "ln0.weight"] = 1 + n(C, scale=0.1); sd[b + "ln0.bias"] = n(C, scale=0.1)
        for ln in ("ln1", "ln2"):
            sd[b + ln + ".weight"] = 1 + n(C, scale=0.1); sd[b + ln + ".bias"] = n(C, scale=0.1)
        a = b + "att."
        if major == 4:
            sd[a + "time_decay"] = u(C, lo=-5, hi=1); sd[a + "time_first"] = n(C, scale=0.3)
            for m in "kvr":
                sd[a + "time_mix_" + m] = u(1, 1, C)
        elif major == 5:
            if minor == 1:
                sd[a + "time_decay"] = u(H, lo=-6, hi=-1); sd[a + "time_first"] = n(H, scale=0.3)
            else:
                sd[a + "time_decay"] = u(H, S, lo=-6, hi=-1); sd[a + "time_faaaa"] = n(H, S, scale=0.1)
            for m in ("kvr" if minor == 1 else "kvrg"):
                sd[a + "time_mix_" + m] = u(1, 1, C)
        elif major == 6:
            for m in "xwkvrg":
                sd[a + "time_maa_" + m] = u(1, 1, C)
            sd[a + "time_maa_w1"] = n(C, 5 * p["mix"], scale=0.01); sd[a + "time_maa_w2"] = n(5, p["mix"], C, scale=0.01)
            sd[a + "time_decay"] = u(1, 1, C, lo=-6, hi=-1)
            sd[a + "time_decay_w1"] = n(C, p["decay"], scale=0.01); sd[a + "time_decay_w2"] = n(p["decay"], C, scale=0.01)
            sd[a + "time_faaaa"] = n(H, S, scale=0.1)
        else:
            for m in "rwkvag":
                sd[a + "x_" + m] = u(1, 1, C)
            sd[a + "w0"] = n(1, 1, C, scale=0.1); sd[a + "w1"] = n(C, p["lora_w"], scale=0.05); sd[a + "w2"] = n(p["lora_w"], C, scale=0.05)
            sd[a + "a0"] = n(1, 1, C, scale=0.1); sd[a + "a1"] = n(C, p["lora_a"], scale=0.05); sd[a + "a2"] = n(p["lora_a"], C, scale=0.05)
            if i > 0:
                sd[a + "v0"] = n(1, 1, C, scale=0.1); sd[a + "v1"] = n(C, p["lora_v"], scale=0.05); sd[a + "v2"] = n(p["lora_v"], C, scale=0.05)
            sd[a + "g1"] = n(C, p["lora_g"], scale=0.05); sd[a + "g2"] = n(p["lora_g"], C, scale=0.05)
            sd[a + "k_k"] = u(1, 1, C); sd[a + "k_a"] = u(1, 1, C); sd[a + "r_k"] = n(H, S, scale=0.1)
        mats = ["receptance", "key", "value", "output"] + (["gate"] if (major, minor) in ((5, 2), (6, 0)) else [])
        for m in mats:
            sd[a + m + ".weight"] = n(C, C, scale=C ** -0.5)
        if major >= 5:
            sd[a + "ln_x.weight"] = 1 + n(C, scale=0.1); sd[a + "ln_x.bias"] = n(C, scale=0.1)
        f = b + "ffn."
        if major == 7:
            sd[f + "x_k"] = u(1, 1, C)
        elif major == 6:
            sd[f + "time_maa_k"] = u(1, 1, C); sd[f + "time_maa_r"] = u(1, 1, C)
        else:
            sd[f + "time_mix_k"] = u(1, 1, C); sd[f + "time_mix_r"] = u(1, 1, C)
        sd[f + "key.weight"] = n(F, C, scale=C ** -0.5); sd[f + "value.weight"] = n(C, F, scale=F ** -0.5)
        if major != 7:
            sd[f + "receptance.weight"] = n(C, C, scale=C ** -0.5)
    sd["ln_out.weight"] = 1 + n(C, scale=0.1); sd["ln_out.bias"] = n(C, scale=0.1)
    sd["head.weight"] = n(V, C, scale=C ** -0.5)
    return sd


def make_lora_state_dict(kind: str, rank: int = 8, seed: int = 1):
    """A seeded RWKV-PEFT-style LoRA checkpoint for make_state_dict(kind): `lora_A` [rank, in] / `lora_B` [out, rank] pairs on the
    att and ffn layer matrices (`.lora_A.weight` naming on the ffn ones, as PEFT writes it), and trained copies of every layer's
    ln1 / ln2, time_* (v4 .. v6: the v6 time_maa_w1 / time_decay_w1 / time_decay_w2 matrices included) or x_* / k_k and the att.w1
    matrix (v7) parameters, moved by a small offset."""
    base = make_state_dict(kind, seed=0)
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, t in base.items():
        if not name.startswith("blocks."):
            continue
        short = name.split(".", 2)[2]
        if short in ("att.key.weight", "att.value.weight", "att.receptance.weight", "att.gate.weight", "att.output.weight",
                     "ffn.key.weight", "ffn.value.weight", "ffn.receptance.weight"):
            stem = name[: -len(".weight")]
            suffix = ".weight" if short.startswith("ffn.") else ""
            sd[stem + ".lora_A" + suffix] = torch.randn(rank, t.shape[1], generator=g) * t.shape[1] ** -0.5
            sd[stem + ".lora_B" + suffix] = torch.randn(t.shape[0], rank, generator=g) * 0.05
        elif short.startswith(("ln1.", "ln2.", "att.time_", "ffn.time_", "att.x_", "ffn.x_", "att.k_k")) or short == "att.w1":
            small = short in ("att.time_maa_w1", "att.time_maa_w2", "att.time_decay_w1", "att.time_decay_w2", "att.w1")   # LoRA weights ~0.01
            sd[name] = t + torch.randn(t.shape, generator=g) * (0.002 if small else 0.02)
    return sd
