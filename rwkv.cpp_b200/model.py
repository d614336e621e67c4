"""RWKVModel -- the reference's model wrapper (python/rwkv_cpp/rwkv_cpp_model.py:21-364) over the H100
library: same constructor arguments, eval / eval_sequence / eval_sequence_in_chunks / free, numpy in
and out (PyTorch CPU tensors are accepted too, as in the reference)."""
import multiprocessing
import os
from typing import List, Optional, Tuple

import numpy as np

from . import shared_library as _sl


def _is_torch(x) -> bool:
    return x is not None and type(x).__module__.startswith("torch")


class RWKVModel:
    def __init__(self, shared_library: "_sl.RWKVSharedLibrary", model_path: str,
                 thread_count: int = max(1, multiprocessing.cpu_count() // 2), gpu_layer_count: int = 0, **kwargs) -> None:
        if "gpu_layers_count" in kwargs:
            gpu_layer_count = kwargs["gpu_layers_count"]
        if not os.path.isfile(model_path):
            raise ValueError(f"{model_path} is not a file")
        if not thread_count > 0:
            raise ValueError("Thread count must be > 0")
        if not gpu_layer_count >= 0:
            raise ValueError("GPU layer count must be >= 0")
        self._library = shared_library
        self._path = model_path
        self._adapter = None
        self._ctx = shared_library.rwkv_init_from_file(model_path, thread_count, gpu_layer_count)
        self._state_buffer_element_count = shared_library.rwkv_get_state_buffer_element_count(self._ctx)
        self._logits_buffer_element_count = shared_library.rwkv_get_logits_buffer_element_count(self._ctx)
        self._valid = True

    # -- properties (rwkv_cpp_model.py:72-83) ---------------------------------------------------
    @property
    def n_vocab(self) -> int:
        return self._library.rwkv_get_n_vocab(self._ctx)

    @property
    def n_embed(self) -> int:
        return self._library.rwkv_get_n_embed(self._ctx)

    @property
    def n_layer(self) -> int:
        return self._library.rwkv_get_n_layer(self._ctx)

    @property
    def state_len(self) -> int:
        return self._state_buffer_element_count

    def gpu_offload_layers(self, layer_count: int) -> bool:
        """Kept for source compatibility (rwkv_cpp_model.py:85-100 was removed upstream): all layers are always on the GPU."""
        return False

    # -- helpers ---------------------------------------------------------------------------------
    def _validate(self, buf, name: str, size: int) -> None:
        """rwkv_cpp_model.py:330-351: float32, contiguous, exact shape. Unlike the reference (which rejects non-CPU tensors,
        :334) CUDA tensors are accepted: the library copies with cudaMemcpyDefault, so a state or logits tensor that already
        lives on the GPU never crosses PCIe."""
        if _is_torch(buf):
            if buf.device.type not in ("cpu", "cuda"):
                raise ValueError(f"{name} is neither on CPU nor on a CUDA device")
            import torch
            if buf.dtype != torch.float32:
                raise ValueError(f"{name} is not of type float32")
            if not buf.is_contiguous():
                raise ValueError(f"{name} is not contiguous")
            if tuple(buf.shape) != (size,):
                raise ValueError(f"{name} has invalid shape {tuple(buf.shape)}, expected ({size})")
        else:
            if buf.dtype != np.float32:
                raise ValueError(f"{name} is not of type float32")
            if not buf.data.contiguous:
                raise ValueError(f"{name} is not contiguous")
            if buf.shape != (size,):
                raise ValueError(f"{name} has invalid shape {buf.shape}, expected ({size})")

    @staticmethod
    def _ptr(buf) -> int:
        if buf is None:
            return 0
        return buf.data_ptr() if _is_torch(buf) else buf.ctypes.data

    def _prepare(self, state_in, state_out, logits_out, use_numpy: bool):
        if not self._valid:
            raise ValueError("Model was freed")
        use_numpy = use_numpy or not any(_is_torch(b) for b in (state_in, state_out, logits_out))
        if any(_is_torch(b) and b.device.type == "cuda" for b in (state_in, state_out, logits_out)):
            import torch
            torch.cuda.current_stream().synchronize()     # the library works on its own stream: the caller's writes must have landed
        if state_in is not None:
            self._validate(state_in, "state_in", self._state_buffer_element_count)
        if state_out is not None:
            self._validate(state_out, "state_out", self._state_buffer_element_count)
        else:
            state_out = self._zeros(self._state_buffer_element_count, use_numpy, state_in)     # outputs follow the input's device
        if logits_out is not None:
            self._validate(logits_out, "logits_out", self._logits_buffer_element_count)
        else:
            logits_out = self._zeros(self._logits_buffer_element_count, use_numpy, state_in)
        return state_out, logits_out

    @staticmethod
    def _zeros(n: int, use_numpy: bool, like=None):
        if use_numpy:
            return np.zeros(n, dtype=np.float32)
        import torch
        return torch.zeros(n, dtype=torch.float32, device=like.device if like is not None and _is_torch(like) else "cpu")

    # -- evaluation (rwkv_cpp_model.py:85-298) -------------------------------------------------
    def eval(self, token: int, state_in, state_out=None, logits_out=None, use_numpy: bool = False) -> Tuple:
        state_out, logits_out = self._prepare(state_in, state_out, logits_out, use_numpy)
        self._library.rwkv_eval(self._ctx, token, self._ptr(state_in), self._ptr(state_out), self._ptr(logits_out))
        return logits_out, state_out

    def eval_sequence(self, tokens: List[int], state_in, state_out=None, logits_out=None, use_numpy: bool = False) -> Tuple:
        state_out, logits_out = self._prepare(state_in, state_out, logits_out, use_numpy)
        self._library.rwkv_eval_sequence(self._ctx, tokens, self._ptr(state_in), self._ptr(state_out), self._ptr(logits_out))
        return logits_out, state_out

    def eval_sequence_in_chunks(self, tokens: List[int], state_in, state_out=None, logits_out=None, chunk_size: int = 16,
                                use_numpy: bool = False) -> Tuple:
        state_out, logits_out = self._prepare(state_in, state_out, logits_out, use_numpy)
        self._library.rwkv_eval_sequence_in_chunks(self._ctx, tokens, chunk_size, self._ptr(state_in), self._ptr(state_out), self._ptr(logits_out))
        return logits_out, state_out

    @property
    def arch(self) -> Tuple[int, int]:
        """(major, minor) RWKV version of the model file."""
        info = self._library.rwkv_b200_inspect_file(self._path)
        return int(info.arch_major), int(info.arch_minor)

    def set_adapter(self, adapter) -> None:
        """Runs every later evaluation with `adapter` (a lora.Adapter made for this model) applied; None detaches. The state is
        untouched. See rwkv_b200_set_adapter in include/rwkv_b200.h."""
        self._library.rwkv_b200_set_adapter(self._ctx, adapter.handle if adapter is not None else None)
        self._adapter = adapter

    def free(self) -> None:
        if not self._valid:
            raise ValueError("Already freed")
        self._valid = False
        self._library.rwkv_free(self._ctx)
        self._adapter = None

    def __del__(self) -> None:
        if getattr(self, "_valid", False):
            self.free()
