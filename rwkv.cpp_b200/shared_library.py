"""ctypes binding of librwkv.so -- same class and method names as the reference binding
(python/rwkv_cpp/rwkv_cpp_shared_library.py:26-426) so code written against it ports by changing one
import. Every method raises ValueError when the C call reports failure, like the reference's asserts.

There is no CPU fallback anywhere in this package: if the CUDA library is missing, loading raises.
"""
import ctypes
import os
from typing import Optional

import numpy as np

P_FLOAT = ctypes.POINTER(ctypes.c_float)
P_U32 = ctypes.POINTER(ctypes.c_uint32)
# rwkv_b200_token_fn (include/rwkv_b200.h): int (*)(void * user, size_t sequence, size_t index, uint32_t token)
RWKV_TOKEN_FN = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_uint32)

SCORE_NO_TARGET = 0xFFFFFFFF   # RWKV_B200_SCORE_NO_TARGET (include/rwkv_b200.h)
QUANTIZED_FORMAT_NAMES = ("Q4_0", "Q4_1", "Q4_K", "Q5_0", "Q5_1", "Q5_K", "Q8_0")   # the reference binding's list, in its order

_HERE = os.path.dirname(os.path.abspath(__file__))


def library_path() -> str:
    return os.path.join(_HERE, "librwkv.so")


class FileInfo(ctypes.Structure):   # include/rwkv_b200.h: struct rwkv_b200_file_info
    _fields_ = [(n, ctypes.c_uint32) for n in ("version", "n_vocab", "n_embed", "n_layer", "data_type",
                                               "arch_major", "arch_minor", "head_count", "head_size")] + \
               [(n, ctypes.c_uint64) for n in ("n_tensors", "file_size", "state_len", "bytes_per_token")]


class ProfileResult(ctypes.Structure):   # include/rwkv_b200.h: struct rwkv_b200_profile
    _fields_ = [(n, ctypes.c_double) for n in ("gemv_ms", "gemv_bytes", "pass_ms", "top_ms", "top_bytes")] + \
               [(n, ctypes.c_uint32) for n in ("gemv_launches", "total_launches")]


class Logprobs(ctypes.Structure):   # include/rwkv_b200.h: struct rwkv_b200_logprobs
    _fields_ = [("top_n", ctypes.c_size_t), ("logprobs", ctypes.POINTER(ctypes.c_float)), ("top_ids", ctypes.POINTER(ctypes.c_uint32)),
                ("top_logprobs", ctypes.POINTER(ctypes.c_float)), ("sample_probs", ctypes.POINTER(ctypes.c_float))]


class Sampler(ctypes.Structure):   # include/rwkv_b200.h: struct rwkv_b200_sampler
    _fields_ = [("temperature", ctypes.c_float), ("top_p", ctypes.c_float), ("top_k", ctypes.c_uint32), ("min_p", ctypes.c_float),
                ("presence_penalty", ctypes.c_float), ("frequency_penalty", ctypes.c_float), ("n_bias", ctypes.c_size_t),
                ("bias_ids", ctypes.POINTER(ctypes.c_uint32)), ("bias_values", ctypes.POINTER(ctypes.c_float))]


class AdapterTensor(ctypes.Structure):   # include/rwkv_b200.h: struct rwkv_b200_adapter_tensor
    _fields_ = [("name", ctypes.c_char_p), ("rank", ctypes.c_uint32), ("a", ctypes.POINTER(ctypes.c_float)),
                ("b", ctypes.POINTER(ctypes.c_float)), ("values", ctypes.POINTER(ctypes.c_float))]


class RWKVContext:
    def __init__(self, ptr: ctypes.c_void_p) -> None:
        self.ptr = ptr


class RWKVSharedLibrary:
    """Thin wrapper: one method per exported C function (include/rwkv.h, include/rwkv_b200.h)."""

    def __init__(self, shared_library_path: str) -> None:
        if not os.path.isfile(shared_library_path):
            raise FileNotFoundError(
                f"{shared_library_path} not found: build it with `python rwkv.cpp_b200/build.py` (nvcc, sm_90a). "
                "This package has no CPU fallback.")
        self.path = shared_library_path
        lib = self.library = ctypes.cdll.LoadLibrary(shared_library_path)
        vp = ctypes.c_void_p
        lib.rwkv_init_from_file.argtypes = [ctypes.c_char_p, ctypes.c_uint32, ctypes.c_uint32]
        lib.rwkv_init_from_file.restype = vp
        lib.rwkv_clone_context.argtypes = [vp, ctypes.c_uint32]
        lib.rwkv_clone_context.restype = vp
        lib.rwkv_eval.argtypes = [vp, ctypes.c_int32, P_FLOAT, P_FLOAT, P_FLOAT]
        lib.rwkv_eval.restype = ctypes.c_bool
        lib.rwkv_eval_sequence.argtypes = [vp, P_U32, ctypes.c_size_t, P_FLOAT, P_FLOAT, P_FLOAT]
        lib.rwkv_eval_sequence.restype = ctypes.c_bool
        lib.rwkv_eval_sequence_in_chunks.argtypes = [vp, P_U32, ctypes.c_size_t, ctypes.c_size_t, P_FLOAT, P_FLOAT, P_FLOAT]
        lib.rwkv_eval_sequence_in_chunks.restype = ctypes.c_bool
        for name in ("rwkv_get_n_vocab", "rwkv_get_n_embed", "rwkv_get_n_layer", "rwkv_get_state_len", "rwkv_get_logits_len"):
            getattr(lib, name).argtypes = [vp]
            getattr(lib, name).restype = ctypes.c_size_t
        for name in ("rwkv_get_state_buffer_element_count", "rwkv_get_logits_buffer_element_count"):
            getattr(lib, name).argtypes = [vp]
            getattr(lib, name).restype = ctypes.c_uint32
        lib.rwkv_init_state.argtypes = [vp, P_FLOAT]
        lib.rwkv_init_state.restype = None
        lib.rwkv_free.argtypes = [vp]
        lib.rwkv_free.restype = None
        lib.rwkv_quantize_model_file.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_char_p]
        lib.rwkv_quantize_model_file.restype = ctypes.c_bool
        lib.rwkv_get_system_info_string.argtypes = []
        lib.rwkv_get_system_info_string.restype = ctypes.c_char_p
        lib.rwkv_set_print_errors.argtypes = [vp, ctypes.c_bool]
        lib.rwkv_set_print_errors.restype = None
        lib.rwkv_get_print_errors.argtypes = [vp]
        lib.rwkv_get_print_errors.restype = ctypes.c_bool
        lib.rwkv_get_last_error.argtypes = [vp]
        lib.rwkv_get_last_error.restype = ctypes.c_int
        # additive API
        lib.rwkv_b200_inspect_file.argtypes = [ctypes.c_char_p, ctypes.POINTER(FileInfo)]
        lib.rwkv_b200_inspect_file.restype = ctypes.c_bool
        lib.rwkv_b200_v6_lora_fold_supported.argtypes = [ctypes.c_int] * 6
        lib.rwkv_b200_v6_lora_fold_supported.restype = ctypes.c_bool
        lib.rwkv_b200_init_from_file_ex.argtypes = [ctypes.c_char_p, ctypes.c_int, ctypes.c_int, ctypes.c_int]
        lib.rwkv_b200_init_from_file_ex.restype = vp
        lib.rwkv_b200_state_load.argtypes = [vp, P_FLOAT]
        lib.rwkv_b200_state_load.restype = ctypes.c_bool
        lib.rwkv_b200_state_store.argtypes = [vp, P_FLOAT]
        lib.rwkv_b200_state_store.restype = ctypes.c_bool
        lib.rwkv_b200_synchronize.argtypes = [vp]
        lib.rwkv_b200_synchronize.restype = ctypes.c_bool
        lib.rwkv_b200_eval_resident.argtypes = [vp, P_U32, ctypes.c_size_t, ctypes.c_bool, P_FLOAT]
        lib.rwkv_b200_eval_resident.restype = ctypes.c_bool
        lib.rwkv_b200_stage_hidden_len.argtypes = [vp, ctypes.c_size_t]
        lib.rwkv_b200_stage_hidden_len.restype = ctypes.c_size_t
        lib.rwkv_b200_stage_eval.argtypes = [vp, P_U32, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_bool, ctypes.c_void_p]
        lib.rwkv_b200_stage_eval.restype = ctypes.c_bool
        lib.rwkv_b200_stage_logits.argtypes = [vp, P_FLOAT, ctypes.c_void_p]
        lib.rwkv_b200_stage_logits.restype = ctypes.c_bool
        lib.rwkv_b200_last_device_ms.argtypes = [vp]
        lib.rwkv_b200_last_device_ms.restype = ctypes.c_float
        lib.rwkv_b200_kernel_launch_count.argtypes = []
        lib.rwkv_b200_kernel_launch_count.restype = ctypes.c_uint64
        lib.rwkv_b200_graph_launch_count.argtypes = []
        lib.rwkv_b200_graph_launch_count.restype = ctypes.c_uint64
        lib.rwkv_b200_bytes_per_token.argtypes = [vp, ctypes.c_bool]
        lib.rwkv_b200_bytes_per_token.restype = ctypes.c_uint64
        lib.rwkv_b200_time_resident.argtypes = [vp, P_U32, ctypes.c_size_t, ctypes.c_int, ctypes.c_int, ctypes.c_bool]
        lib.rwkv_b200_time_resident.restype = ctypes.c_float
        lib.rwkv_b200_profile_pass.argtypes = [vp, P_U32, ctypes.c_size_t, ctypes.c_bool, ctypes.POINTER(ProfileResult)]
        lib.rwkv_b200_profile_pass.restype = ctypes.c_bool
        lib.rwkv_b200_trace_enable.argtypes = [vp]
        lib.rwkv_b200_trace_enable.restype = ctypes.c_bool
        lib.rwkv_b200_trace_read.argtypes = [vp, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_double), ctypes.c_void_p, ctypes.c_int]
        lib.rwkv_b200_trace_read.restype = ctypes.c_int
        lib.rwkv_b200_init_pipeline.argtypes = [ctypes.c_char_p, ctypes.POINTER(ctypes.c_int), ctypes.c_size_t]
        lib.rwkv_b200_init_pipeline.restype = vp
        lib.rwkv_b200_pipeline_stages.argtypes = [vp]
        lib.rwkv_b200_pipeline_stages.restype = ctypes.c_size_t
        lib.rwkv_b200_stream.argtypes = [vp]
        lib.rwkv_b200_stream.restype = ctypes.c_void_p
        lib.rwkv_b200_pipe_handle_size.argtypes = []
        lib.rwkv_b200_pipe_handle_size.restype = ctypes.c_size_t
        lib.rwkv_b200_pipe_export.argtypes = [vp, ctypes.c_void_p]
        lib.rwkv_b200_pipe_export.restype = ctypes.c_bool
        lib.rwkv_b200_pipe_connect.argtypes = [vp, ctypes.c_void_p, ctypes.c_void_p]
        lib.rwkv_b200_pipe_connect.restype = ctypes.c_bool
        lib.rwkv_b200_pipe_connect_local.argtypes = [vp, vp, vp]
        lib.rwkv_b200_pipe_connect_local.restype = ctypes.c_bool
        lib.rwkv_b200_pipe_eval.argtypes = [vp, P_U32, ctypes.c_size_t, ctypes.c_bool, ctypes.c_void_p]
        lib.rwkv_b200_pipe_eval.restype = ctypes.c_bool
        lib.rwkv_b200_trace_disable.argtypes = [vp]
        lib.rwkv_b200_trace_disable.restype = None
        lib.rwkv_b200_gemv_bytes_per_token.argtypes = [vp, ctypes.c_bool]
        lib.rwkv_b200_gemv_bytes_per_token.restype = ctypes.c_uint64
        lib.rwkv_b200_set_graphs.argtypes = [vp, ctypes.c_bool]
        lib.rwkv_b200_set_graphs.restype = None
        lib.rwkv_b200_set_tensor_cores.argtypes = [vp, ctypes.c_bool]
        lib.rwkv_b200_set_tensor_cores.restype = None
        lib.rwkv_b200_set_overlap.argtypes = [vp, ctypes.c_bool]
        lib.rwkv_b200_set_overlap.restype = None
        lib.rwkv_b200_set_bounce_min_bytes.argtypes = [ctypes.c_size_t]
        lib.rwkv_b200_set_bounce_min_bytes.restype = None
        lib.rwkv_b200_overlap_groups.argtypes = [vp]
        lib.rwkv_b200_overlap_groups.restype = ctypes.c_int
        lib.rwkv_b200_batch_create.argtypes = [vp, ctypes.c_size_t]
        lib.rwkv_b200_batch_create.restype = vp
        lib.rwkv_b200_batch_set_state.argtypes = [vp, ctypes.c_size_t, P_FLOAT]
        lib.rwkv_b200_batch_set_state.restype = ctypes.c_bool
        lib.rwkv_b200_batch_get_state.argtypes = [vp, ctypes.c_size_t, P_FLOAT]
        lib.rwkv_b200_batch_get_state.restype = ctypes.c_bool
        lib.rwkv_b200_batch_eval.argtypes = [vp, P_U32, ctypes.c_bool]
        lib.rwkv_b200_batch_eval.restype = ctypes.c_bool
        lib.rwkv_b200_batch_eval_ragged.argtypes = [vp, P_U32, P_U32, ctypes.c_bool]
        lib.rwkv_b200_batch_eval_ragged.restype = ctypes.c_bool
        lib.rwkv_b200_batch_get_logits.argtypes = [vp, ctypes.c_size_t, P_FLOAT]
        lib.rwkv_b200_batch_get_logits.restype = ctypes.c_bool
        lib.rwkv_b200_batch_size.argtypes = [vp]
        lib.rwkv_b200_batch_size.restype = ctypes.c_size_t
        lib.rwkv_b200_sample.argtypes = [vp, ctypes.c_float, ctypes.c_float, ctypes.c_double, P_U32, P_FLOAT, ctypes.c_size_t, P_U32]
        lib.rwkv_b200_sample.restype = ctypes.c_bool
        lib.rwkv_b200_sample_logits.argtypes = [P_FLOAT, ctypes.c_size_t, ctypes.c_float, ctypes.c_float, ctypes.c_double, P_U32, P_FLOAT, ctypes.c_size_t, P_U32, P_FLOAT]
        lib.rwkv_b200_sample_logits.restype = ctypes.c_bool
        lib.rwkv_b200_eval_sample.argtypes = [vp, ctypes.c_uint32, ctypes.c_float, ctypes.c_float, ctypes.c_double, P_U32]
        lib.rwkv_b200_eval_sample.restype = ctypes.c_bool
        P_DOUBLE = ctypes.POINTER(ctypes.c_double)
        lib.rwkv_b200_batch_sample.argtypes = [vp, P_FLOAT, P_FLOAT, P_DOUBLE, P_U32, P_U32, P_FLOAT, P_U32]
        lib.rwkv_b200_batch_sample.restype = ctypes.c_bool
        lib.rwkv_b200_batch_eval_sample.argtypes = [vp, P_U32, P_FLOAT, P_FLOAT, P_DOUBLE, P_U32]
        lib.rwkv_b200_batch_eval_sample.restype = ctypes.c_bool
        lib.rwkv_b200_sample_logits_batch.argtypes = [P_FLOAT, ctypes.c_size_t, ctypes.c_size_t, P_FLOAT, P_FLOAT, P_DOUBLE, P_U32, P_U32, P_FLOAT,
                                                      P_U32, P_FLOAT]
        lib.rwkv_b200_sample_logits_batch.restype = ctypes.c_bool
        lib.rwkv_b200_generate.argtypes = [vp, ctypes.c_size_t, ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_bool, P_DOUBLE,
                                           P_U32, ctypes.c_size_t, P_U32, ctypes.POINTER(ctypes.c_size_t)]
        lib.rwkv_b200_generate.restype = ctypes.c_bool
        P_U8 = ctypes.POINTER(ctypes.c_uint8)
        lib.rwkv_b200_batch_generate.argtypes = [vp, P_U32, P_FLOAT, P_FLOAT, P_FLOAT, P_FLOAT, P_U8, P_DOUBLE, P_U32, ctypes.c_size_t, P_U32, P_U32]
        lib.rwkv_b200_batch_generate.restype = ctypes.c_bool
        lib.rwkv_b200_generate_stream.argtypes = [vp, ctypes.c_size_t, ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_bool,
                                                  P_DOUBLE, P_U32, ctypes.c_size_t, RWKV_TOKEN_FN, ctypes.c_void_p, P_U32, ctypes.POINTER(ctypes.c_size_t)]
        lib.rwkv_b200_generate_stream.restype = ctypes.c_bool
        lib.rwkv_b200_batch_generate_stream.argtypes = [vp, P_U32, P_FLOAT, P_FLOAT, P_FLOAT, P_FLOAT, P_U8, P_DOUBLE, P_U32, ctypes.c_size_t,
                                                        RWKV_TOKEN_FN, ctypes.c_void_p, P_U32, P_U32]
        lib.rwkv_b200_batch_generate_stream.restype = ctypes.c_bool
        lib.rwkv_b200_test_generate_step.argtypes = [ctypes.c_void_p]
        lib.rwkv_b200_test_generate_step.restype = ctypes.c_bool
        P_U16 = ctypes.POINTER(ctypes.c_uint16)
        lib.rwkv_b200_automaton_create.argtypes = [vp, P_U16, ctypes.c_size_t]
        lib.rwkv_b200_automaton_create.restype = vp
        lib.rwkv_b200_automaton_free.argtypes = [vp]
        lib.rwkv_b200_automaton_free.restype = None
        lib.rwkv_b200_generate_constrained.argtypes = [vp, vp, P_U32, ctypes.c_size_t, ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_float,
                                                       ctypes.c_bool, P_DOUBLE, P_U32, ctypes.c_size_t, RWKV_TOKEN_FN, ctypes.c_void_p, P_U32,
                                                       ctypes.POINTER(ctypes.c_size_t)]
        lib.rwkv_b200_generate_constrained.restype = ctypes.c_bool
        lib.rwkv_b200_batch_generate_constrained.argtypes = [vp, ctypes.POINTER(vp), P_U32, P_U32, P_FLOAT, P_FLOAT, P_FLOAT, P_FLOAT, P_U8, P_DOUBLE,
                                                             P_U32, ctypes.c_size_t, RWKV_TOKEN_FN, ctypes.c_void_p, P_U32, P_U32]
        lib.rwkv_b200_batch_generate_constrained.restype = ctypes.c_bool
        lib.rwkv_b200_test_generate_step_constrained.argtypes = [ctypes.c_void_p, P_U16, ctypes.c_size_t, P_U32]
        lib.rwkv_b200_adapter_create.argtypes = [vp, ctypes.POINTER(AdapterTensor), ctypes.c_size_t, ctypes.c_float]
        lib.rwkv_b200_adapter_create.restype = vp
        lib.rwkv_b200_adapter_free.argtypes = [vp]
        lib.rwkv_b200_adapter_free.restype = ctypes.c_bool
        lib.rwkv_b200_set_adapter.argtypes = [vp, vp]
        lib.rwkv_b200_set_adapter.restype = ctypes.c_bool
        lib.rwkv_b200_test_lora.argtypes = [ctypes.c_int] * 4 + [ctypes.c_float, ctypes.c_int] + [P_FLOAT] * 7
        lib.rwkv_b200_test_lora.restype = ctypes.c_bool
        lib.rwkv_b200_test_encode_rows.argtypes = [ctypes.c_int, P_FLOAT, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_void_p]
        lib.rwkv_b200_test_encode_rows.restype = ctypes.c_bool
        lib.rwkv_b200_test_generate_step_constrained.restype = ctypes.c_bool
        P_LOGPROBS = ctypes.POINTER(Logprobs)
        lib.rwkv_b200_generate_logprobs.argtypes = [vp, vp, P_U32, ctypes.c_size_t, ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_float,
                                                    ctypes.c_bool, P_DOUBLE, P_U32, ctypes.c_size_t, RWKV_TOKEN_FN, ctypes.c_void_p, P_U32,
                                                    ctypes.POINTER(ctypes.c_size_t), P_LOGPROBS]
        lib.rwkv_b200_generate_logprobs.restype = ctypes.c_bool
        lib.rwkv_b200_batch_generate_logprobs.argtypes = [vp, ctypes.POINTER(vp), P_U32, P_U32, P_FLOAT, P_FLOAT, P_FLOAT, P_FLOAT, P_U8, P_DOUBLE,
                                                          P_U32, ctypes.c_size_t, RWKV_TOKEN_FN, ctypes.c_void_p, P_U32, P_U32, P_LOGPROBS]
        lib.rwkv_b200_batch_generate_logprobs.restype = ctypes.c_bool
        lib.rwkv_b200_test_generate_step_logprobs.argtypes = [ctypes.c_void_p, P_U16, ctypes.c_size_t, P_U32, P_LOGPROBS]
        lib.rwkv_b200_test_generate_step_logprobs.restype = ctypes.c_bool
        P_SAMPLER = ctypes.POINTER(Sampler)
        lib.rwkv_b200_generate_sampled.argtypes = [vp, P_SAMPLER, vp, P_U32, ctypes.c_size_t, ctypes.c_bool, P_DOUBLE, P_U32, ctypes.c_size_t,
                                                   RWKV_TOKEN_FN, ctypes.c_void_p, P_U32, ctypes.POINTER(ctypes.c_size_t), P_LOGPROBS]
        lib.rwkv_b200_generate_sampled.restype = ctypes.c_bool
        lib.rwkv_b200_batch_generate_sampled.argtypes = [vp, P_SAMPLER, ctypes.POINTER(vp), P_U32, P_U32, P_U8, P_DOUBLE, P_U32, ctypes.c_size_t,
                                                         RWKV_TOKEN_FN, ctypes.c_void_p, P_U32, P_U32, P_LOGPROBS]
        lib.rwkv_b200_batch_generate_sampled.restype = ctypes.c_bool
        lib.rwkv_b200_test_generate_step_sampled.argtypes = [ctypes.c_void_p, P_SAMPLER, P_U16, ctypes.c_size_t, P_U32, P_LOGPROBS]
        lib.rwkv_b200_test_generate_step_sampled.restype = ctypes.c_bool
        lib.rwkv_b200_test_generate_step_streaming.argtypes = [ctypes.c_void_p, ctypes.c_int, P_SAMPLER, P_U16, ctypes.c_size_t, P_U32, P_LOGPROBS,
                                                               P_U32, P_U32, P_U32, P_U32, P_U32]
        lib.rwkv_b200_test_generate_step_streaming.restype = ctypes.c_bool
        lib.rwkv_b200_score.argtypes = [vp, P_U32, P_U32, ctypes.c_size_t, P_FLOAT, P_U8]
        lib.rwkv_b200_score.restype = ctypes.c_bool
        lib.rwkv_b200_batch_score_ragged.argtypes = [vp, P_U32, P_U32, P_U32, P_FLOAT, P_U8]
        lib.rwkv_b200_batch_score_ragged.restype = ctypes.c_bool
        lib.rwkv_b200_score_logits.argtypes = [P_FLOAT, ctypes.c_size_t, ctypes.c_size_t, P_U32, P_FLOAT, P_U8]
        lib.rwkv_b200_score_logits.restype = ctypes.c_bool
        lib.rwkv_b200_matvec.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, P_FLOAT, P_FLOAT, ctypes.c_int]
        lib.rwkv_b200_matvec.restype = ctypes.c_bool

    # --- rwkv.h -------------------------------------------------------------------------------
    def rwkv_init_from_file(self, model_file_path: str, thread_count: int, gpu_layer_count: int = 0) -> RWKVContext:
        ptr = self.library.rwkv_init_from_file(model_file_path.encode("utf-8"), ctypes.c_uint32(thread_count), ctypes.c_uint32(gpu_layer_count))
        if not ptr:
            raise ValueError(f"rwkv_init_from_file failed (error flags 0x{self.rwkv_get_last_error(None):x}), check stderr")
        return RWKVContext(ptr)

    def rwkv_clone_context(self, ctx: RWKVContext, thread_count: int) -> RWKVContext:
        ptr = self.library.rwkv_clone_context(ctx.ptr, ctypes.c_uint32(thread_count))
        if not ptr:
            raise ValueError("rwkv_clone_context failed, check stderr")
        return RWKVContext(ptr)

    def rwkv_eval(self, ctx: RWKVContext, token: int, state_in_address: Optional[int], state_out_address: int, logits_out_address: int) -> None:
        if not self.library.rwkv_eval(ctx.ptr, ctypes.c_int32(token), ctypes.cast(state_in_address or 0, P_FLOAT),
                                      ctypes.cast(state_out_address or 0, P_FLOAT), ctypes.cast(logits_out_address or 0, P_FLOAT)):
            raise ValueError("rwkv_eval failed, check stderr")

    def rwkv_eval_sequence(self, ctx: RWKVContext, tokens, state_in_address: Optional[int], state_out_address: int, logits_out_address: int) -> None:
        arr = (ctypes.c_uint32 * len(tokens))(*tokens)
        if not self.library.rwkv_eval_sequence(ctx.ptr, arr, ctypes.c_size_t(len(tokens)), ctypes.cast(state_in_address or 0, P_FLOAT),
                                               ctypes.cast(state_out_address or 0, P_FLOAT), ctypes.cast(logits_out_address or 0, P_FLOAT)):
            raise ValueError("rwkv_eval_sequence failed, check stderr")

    def rwkv_eval_sequence_in_chunks(self, ctx: RWKVContext, tokens, chunk_size: int, state_in_address: Optional[int],
                                     state_out_address: int, logits_out_address: int) -> None:
        arr = (ctypes.c_uint32 * len(tokens))(*tokens)
        if not self.library.rwkv_eval_sequence_in_chunks(ctx.ptr, arr, ctypes.c_size_t(len(tokens)), ctypes.c_size_t(chunk_size),
                                                         ctypes.cast(state_in_address or 0, P_FLOAT), ctypes.cast(state_out_address or 0, P_FLOAT),
                                                         ctypes.cast(logits_out_address or 0, P_FLOAT)):
            raise ValueError("rwkv_eval_sequence_in_chunks failed, check stderr")

    def rwkv_get_n_vocab(self, ctx: RWKVContext) -> int:
        return self.library.rwkv_get_n_vocab(ctx.ptr)

    def rwkv_get_n_embed(self, ctx: RWKVContext) -> int:
        return self.library.rwkv_get_n_embed(ctx.ptr)

    def rwkv_get_n_layer(self, ctx: RWKVContext) -> int:
        return self.library.rwkv_get_n_layer(ctx.ptr)

    def rwkv_get_state_buffer_element_count(self, ctx: RWKVContext) -> int:
        return self.library.rwkv_get_state_buffer_element_count(ctx.ptr)

    def rwkv_get_logits_buffer_element_count(self, ctx: RWKVContext) -> int:
        return self.library.rwkv_get_logits_buffer_element_count(ctx.ptr)

    def rwkv_get_state_len(self, ctx: RWKVContext) -> int:
        return self.library.rwkv_get_state_len(ctx.ptr)

    def rwkv_get_logits_len(self, ctx: RWKVContext) -> int:
        return self.library.rwkv_get_logits_len(ctx.ptr)

    def rwkv_init_state(self, ctx: RWKVContext, state_address: int) -> None:
        self.library.rwkv_init_state(ctx.ptr, ctypes.cast(state_address, P_FLOAT))

    def rwkv_free(self, ctx: RWKVContext) -> None:
        self.library.rwkv_free(ctx.ptr)
        ctx.ptr = ctypes.c_void_p(0)

    def rwkv_quantize_model_file(self, model_file_path_in: str, model_file_path_out: str, format_name: str) -> None:
        if format_name not in QUANTIZED_FORMAT_NAMES:
            raise ValueError(f"Unknown format name {format_name}, use one of {QUANTIZED_FORMAT_NAMES}")
        if not self.library.rwkv_quantize_model_file(model_file_path_in.encode("utf-8"), model_file_path_out.encode("utf-8"), format_name.encode("utf-8")):
            raise ValueError("rwkv_quantize_model_file failed, check stderr")

    def rwkv_get_system_info_string(self) -> str:
        return self.library.rwkv_get_system_info_string().decode("utf-8")

    def rwkv_set_print_errors(self, ctx: Optional[RWKVContext], print_errors: bool) -> None:
        self.library.rwkv_set_print_errors(ctx.ptr if ctx else None, ctypes.c_bool(print_errors))

    def rwkv_get_print_errors(self, ctx: Optional[RWKVContext]) -> bool:
        return self.library.rwkv_get_print_errors(ctx.ptr if ctx else None)

    def rwkv_get_last_error(self, ctx: Optional[RWKVContext]) -> int:
        return self.library.rwkv_get_last_error(ctx.ptr if ctx else None)

    # --- rwkv_b200.h --------------------------------------------------------------------------
    def rwkv_b200_inspect_file(self, model_file_path: str) -> FileInfo:
        info = FileInfo()
        if not self.library.rwkv_b200_inspect_file(model_file_path.encode("utf-8"), ctypes.byref(info)):
            raise ValueError(f"rwkv_b200_inspect_file failed (error flags 0x{self.rwkv_get_last_error(None):x})")
        return info

    def rwkv_b200_adapter_create(self, ctx: RWKVContext, tensors, scale: float) -> int:
        """tensors: (name, rank, a, b, values) tuples, the arrays float32 C-contiguous numpy arrays (or None), as
        struct rwkv_b200_adapter_tensor describes them. Returns the adapter handle."""
        P = ctypes.POINTER(ctypes.c_float)
        arr = (AdapterTensor * max(1, len(tensors)))()
        keep = []
        for i, (name, rank, a, b, values) in enumerate(tensors):
            ptrs = []
            for x in (a, b, values):
                if x is None:
                    ptrs.append(None)
                else:
                    x = np.ascontiguousarray(x, dtype=np.float32)
                    keep.append(x)
                    ptrs.append(x.ctypes.data_as(P))
            arr[i] = AdapterTensor(name.encode("utf-8"), rank, *ptrs)
        ptr = self.library.rwkv_b200_adapter_create(ctx.ptr, arr, len(tensors), ctypes.c_float(scale))
        if not ptr:
            raise ValueError(f"rwkv_b200_adapter_create failed (error flags 0x{self.rwkv_get_last_error(None):x}), check stderr")
        return ptr

    def rwkv_b200_adapter_free(self, adapter: int) -> None:
        if not self.library.rwkv_b200_adapter_free(adapter):
            raise ValueError("rwkv_b200_adapter_free failed: the adapter is still attached to a context")

    def rwkv_b200_set_adapter(self, ctx: RWKVContext, adapter: Optional[int]) -> None:
        if not self.library.rwkv_b200_set_adapter(ctx.ptr, adapter):
            raise ValueError(f"rwkv_b200_set_adapter failed (error flags 0x{self.rwkv_get_last_error(ctx):x})")

    def rwkv_b200_init_from_file_ex(self, model_file_path: str, device: int, layer_begin: int = 0, layer_end: int = -1) -> RWKVContext:
        ptr = self.library.rwkv_b200_init_from_file_ex(model_file_path.encode("utf-8"), device, layer_begin, layer_end)
        if not ptr:
            raise ValueError(f"rwkv_b200_init_from_file_ex failed (error flags 0x{self.rwkv_get_last_error(None):x}), check stderr")
        return RWKVContext(ptr)


def load_rwkv_shared_library() -> RWKVSharedLibrary:
    """Loads librwkv.so from the package directory (reference: load_rwkv_shared_library,
    rwkv_cpp_shared_library.py:383-426, which searches several build directories)."""
    return RWKVSharedLibrary(library_path())
