"""LoRA fine-tunes (RWKV-LM-LoRA / RWKV-PEFT .pth checkpoints) as adapters of a loaded model, applied on the GPU beside the base
weights (include/rwkv_b200.h: rwkv_b200_adapter_create), whatever the type of the model file, quantized ones included.

    adapter = lora.Adapter(model, "my-lora.pth", lora_alpha=32)
    model.set_adapter(adapter)      # model.set_adapter(None) detaches

A checkpoint holds, per adapted layer matrix `blocks.N.att.key.weight`, the pair `blocks.N.att.key.lora_A` [rank, in] and
`blocks.N.att.key.lora_B` [out, rank] (`.lora_A.weight` / `.lora_B.weight` are accepted too), and, usually, trained parameters
such as `time_*` and `ln*`, which replace the model's. The replacements go through the converter's rewrites
(convert_pytorch_to_ggml.transform_tensor), so they reach the library in the file's element order. Every delta gets the scale
lora_alpha / rank * scale, so all deltas of a checkpoint must share one rank. A key that cannot be placed is an error.

An adapter made of deltas alone can also be attached to single sequences of a batch context, so that one pass over the base weights
serves several fine-tunes (rwkv_b200_batch_set_adapter). An adapter with replacements cannot: a replaced vector or matrix is read by
kernels that take one pointer for every column of a pass. Checkpoints trained with RWKV-LM-LoRA's `time` / `ln` parts carry such
replacements; attach those to a whole context with set_adapter.
"""
from typing import Dict, List, Optional, Tuple

import numpy as np

from . import convert_pytorch_to_ggml as _conv

V7_SHIFT = ("r", "w", "k", "v", "a", "g")     # the order of att.x_rwkvag in the file


def _np(t) -> np.ndarray:
    return np.ascontiguousarray(t.detach().float().cpu().numpy(), dtype=np.float32)


def _lora_part(key: str) -> Tuple[Optional[str], Optional[str]]:
    """("blocks.N.att.key.weight", "lora_A") for "blocks.N.att.key.lora_A[.weight]"; (None, None) for any other key."""
    for part in ("lora_A", "lora_B"):
        for suffix in ("." + part + ".weight", "." + part):
            if key.endswith(suffix):
                return key[: -len(suffix)] + ".weight", part
    return None, None


def checkpoint_entries(state_dict: Dict, arch: Tuple[int, int], lora_alpha: float, scale: float = 1.0) -> Tuple[List[tuple], float]:
    """The adapter entries (name, rank, A, B, values) of a checkpoint's state dict for a model of architecture arch = (major, minor),
    and the scale of its deltas."""
    pairs: Dict[str, Dict[str, object]] = {}
    plain: Dict[str, object] = {}
    for key, t in state_dict.items():
        name, part = _lora_part(key)
        if name:
            pairs.setdefault(name, {})[part] = t
        else:
            plain[key] = t
    entries: List[tuple] = []
    ranks = set()
    for name, ab in pairs.items():
        if set(ab) != {"lora_A", "lora_B"}:
            raise ValueError(f"{name}: lora_A and lora_B must both be present")
        a, b = _np(ab["lora_A"]), _np(ab["lora_B"])
        if a.ndim != 2 or b.ndim != 2 or b.shape[1] != a.shape[0]:
            raise ValueError(f"{name}: lora_A {tuple(a.shape)} and lora_B {tuple(b.shape)} do not make a low-rank pair")
        ranks.add(a.shape[0])
        entries.append((name, int(a.shape[0]), a, b, None))
    if len(ranks) > 1:
        raise ValueError(f"the deltas have different ranks {sorted(ranks)}; one scale serves every delta of an adapter")
    if arch[0] == 7:      # att.x_r .. x_g of a layer travel as one att.x_rwkvag
        shifts: Dict[int, Dict[str, object]] = {}
        for key in [k for k in plain if ".att.x_" in k]:
            shifts.setdefault(int(key.split(".")[1]), {})[key.rsplit("x_", 1)[1]] = plain.pop(key)
        for layer, parts in sorted(shifts.items()):
            if set(parts) != set(V7_SHIFT):
                raise ValueError(f"blocks.{layer}: att.x_{{r,w,k,v,a,g}} must all be present to replace att.x_rwkvag, got {sorted(parts)}")
            import torch
            plain[f"blocks.{layer}.att.x_rwkvag"] = torch.cat([parts[m].reshape(-1) for m in V7_SHIFT])
    for name, t in plain.items():
        # n_head only reshapes (v6 time_decay), which leaves the element order as it is
        values = _np(_conv.transform_tensor(name, t, arch, 1, False)).reshape(-1)
        entries.append((name, 0, None, None, values))
    rank = ranks.pop() if ranks else 1
    return entries, float(lora_alpha) / rank * float(scale)


class Adapter:
    """A checkpoint (path or state dict) uploaded as an adapter of `model`'s weights. It serves every context of that model; free it
    (or let it be collected) once no model has it attached."""

    def __init__(self, model, checkpoint, lora_alpha: float, scale: float = 1.0) -> None:
        if isinstance(checkpoint, str):
            import torch
            checkpoint = torch.load(checkpoint, map_location="cpu")
        self._library = model._library
        entries, self.scale = checkpoint_entries(checkpoint, model.arch, lora_alpha, scale)
        self.names = [e[0] for e in entries]
        self.handle: Optional[int] = self._library.rwkv_b200_adapter_create(model._ctx, entries, self.scale)

    def free(self) -> None:
        if self.handle:
            self._library.rwkv_b200_adapter_free(self.handle)
            self.handle = None

    def __del__(self) -> None:
        try:
            self.free()
        except Exception:
            pass
