"""ctypes binding of libesmb200.so (the C ABI declared in include/esmb200.h).

This is the reference-side binding a maintainer would add (INTEGRATION.md shows the same stub): plain pointers and
sizes, no torch types cross the boundary.  PyTorch is used by the callers only to own device memory and streams.

There is deliberately no fallback: if the shared library is missing or a call fails, an exception is raised.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_float, c_int32, c_int64, c_size_t, c_uint8, c_uint64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("ESMB200_LIB_PATH") or os.path.join(_HERE, "libesmb200.so")  # override: developer builds

# every symbol include/esmb200.h declares (tests/test_abi.py checks the .so exports exactly these)
EXPORTS = (
    "esmb200_abi_version",
    "esmb200_last_error",
    "esmb200_layer_create",
    "esmb200_layer_destroy",
    "esmb200_workspace_bytes",
    "esmb200_layer_forward",
    "esmb200_stack_forward",
    "esmb200_embed_tokens",
    "esmb200_esm1b_embed",
    "esmb200_layernorm",
    "esmb200_mean_pool",
    "esmb200_log_softmax_rows",
    "esmb200_gemm_f16",
    "esmb200_gemm_qkv_f16",
    "esmb200_gemm_qkv_heads",
    "esmb200_attention_scratch_bytes",
    "esmb200_attention",
    "esmb200_attention128",
    "esmb200_tied_row_attention_scratch_bytes",
    "esmb200_tied_row_attention",
    "esmb200_column_attention",
    "esmb200_axial_workspace_bytes",
    "esmb200_axial_stack_forward",
    "esmb200_msa_embed",
    "esmb200_contact_accumulate",
    "esmb200_contact_finalize",
    "esmb200_layernorm_f16",
    "esmb200_convert_f16",
    "esmb200_launch_count",
    "esmb200_profile_enable",
    "esmb200_profile_read",
    "esmb200_set_option",
    "esmb200_layernorm_split",
    "esmb200_convert_split",
    "esmb200_gemm_split",
    "esmb200_attention_split",
    "esmb200_axial_workspace_bytes_split",
    "esmb200_gemm_qkv_split",
    "esmb200_tied_row_attention_split_scratch_bytes",
    "esmb200_tied_row_attention_split",
    "esmb200_column_attention_split",
    "esmb200_layer_packed_bytes",
    "esmb200_layer_offload",
    "esmb200_stack_forward_streamed",
    "esmb200_layernorm_fp8",
    "esmb200_quantize_fp8",
    "esmb200_gemm_fp8",
    "esmb200_stack_contacts_bytes",
    "esmb200_stack_contacts",
    "esmb200_window_merge",
    "esmb200_jacobian_scratch_bytes",
    "esmb200_jacobian_contacts",
    "esmb200_sample_order",
    "esmb200_sample_rows",
    "esmb200_msa_select_scratch_bytes",
    "esmb200_msa_greedy_select",
    "esmb200_knn_scratch_bytes",
    "esmb200_knn_search",
    "esmb200_knn_search_accumulate",
    "esmb200_knn_decode",
    "esmb200_knn_range",
    "esmb200_knn_range_finish_scratch_bytes",
    "esmb200_knn_range_finish",
    "esmb200_ivf_scratch_bytes",
    "esmb200_ivf_search",
    "esmb200_kmeans_means",
    "esmb200_align_scratch_bytes",
    "esmb200_align_similarity",
    "esmb200_align",
)

ABI_VERSION = 4
SELECT_MAX, SELECT_MIN = 0, 1  # ESMB200_SELECT_MAX / ESMB200_SELECT_MIN
ALIGN_LOCAL, ALIGN_GLOBAL = 0, 1  # ESMB200_ALIGN_LOCAL / ESMB200_ALIGN_GLOBAL
EPI_QKV_ROPE, EPI_BIAS_RESIDUAL, EPI_BIAS_GELU, EPI_BIAS_F32, EPI_BIAS_GELU_F32, EPI_GELU_FP8 = range(6)


class LayerWeights(ctypes.Structure):
    """struct esmb200_layer_weights"""

    _fields_ = [
        ("embed_dim", c_int32),
        ("num_heads", c_int32),
        ("ffn_dim", c_int32),
        ("ln_eps", c_float),
        ("ln1_weight", c_void_p),
        ("ln1_bias", c_void_p),
        ("q_weight", c_void_p),
        ("q_bias", c_void_p),
        ("k_weight", c_void_p),
        ("k_bias", c_void_p),
        ("v_weight", c_void_p),
        ("v_bias", c_void_p),
        ("out_weight", c_void_p),
        ("out_bias", c_void_p),
        ("ln2_weight", c_void_p),
        ("ln2_bias", c_void_p),
        ("fc1_weight", c_void_p),
        ("fc1_bias", c_void_p),
        ("fc2_weight", c_void_p),
        ("fc2_bias", c_void_p),
        ("head_dim", c_int32),
        ("precision", c_int32),
    ]


class ContactJob(ctypes.Structure):
    """struct esmb200_contact_job"""

    _fields_ = [("weights", c_void_p), ("keep", c_void_p), ("acc", c_void_p), ("row_part", c_void_p),
                ("col_part", c_void_p), ("lo", c_int32), ("hi", c_int32)]


class Esmb200Error(RuntimeError):
    pass


_lib = None


def _declare(lib):
    lib.esmb200_abi_version.restype = c_int32
    lib.esmb200_abi_version.argtypes = []
    lib.esmb200_last_error.restype = c_char_p
    lib.esmb200_last_error.argtypes = []
    lib.esmb200_layer_create.restype = c_int32
    lib.esmb200_layer_create.argtypes = [POINTER(LayerWeights), c_void_p, POINTER(c_void_p)]
    lib.esmb200_layer_destroy.restype = c_int32
    lib.esmb200_layer_destroy.argtypes = [c_void_p]
    lib.esmb200_workspace_bytes.restype = c_size_t
    lib.esmb200_workspace_bytes.argtypes = [c_int32, c_int32, c_int32, c_int32, c_int32, c_int32]
    lib.esmb200_layer_forward.restype = c_int32
    lib.esmb200_layer_forward.argtypes = [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_void_p,
                                          c_void_p, c_void_p, c_size_t, c_void_p]
    lib.esmb200_stack_forward.restype = c_int32
    lib.esmb200_stack_forward.argtypes = [POINTER(c_void_p), c_int32, c_void_p, c_void_p, c_int32, c_int32, c_void_p,
                                          c_void_p, POINTER(c_void_p), POINTER(c_void_p), c_int64, c_int32,
                                          POINTER(ContactJob), c_void_p, c_size_t, c_void_p]
    lib.esmb200_layer_packed_bytes.restype = c_size_t
    lib.esmb200_layer_packed_bytes.argtypes = [c_int32, c_int32, c_int32, c_int32]
    lib.esmb200_layer_offload.restype = c_int32
    lib.esmb200_layer_offload.argtypes = [c_void_p, c_void_p, c_size_t, c_void_p]
    lib.esmb200_stack_forward_streamed.restype = c_int32
    lib.esmb200_stack_forward_streamed.argtypes = [POINTER(c_void_p), c_int32, c_void_p, c_void_p, c_int32, c_int32,
                                                   c_void_p, c_void_p, POINTER(c_void_p), POINTER(c_void_p), c_int64,
                                                   c_int32, POINTER(ContactJob), c_void_p, c_size_t, c_void_p,
                                                   c_size_t, c_void_p, c_void_p]
    lib.esmb200_stack_contacts_bytes.restype = c_int32
    lib.esmb200_stack_contacts_bytes.argtypes = [c_int32, c_int32, c_int32, c_int32, c_int32, c_int32,
                                                 POINTER(c_size_t), POINTER(c_size_t), POINTER(c_size_t)]
    lib.esmb200_stack_contacts.restype = c_int32
    lib.esmb200_stack_contacts.argtypes = [POINTER(c_void_p), c_int32, c_void_p, c_void_p, c_int32, c_int32, c_void_p,
                                           c_void_p, POINTER(c_void_p), POINTER(ContactJob), c_void_p, c_size_t,
                                           c_void_p, c_size_t, c_void_p, c_size_t, c_void_p, c_void_p]
    lib.esmb200_embed_tokens.restype = c_int32
    lib.esmb200_embed_tokens.argtypes = [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_int32,
                                         c_int32, c_void_p]
    lib.esmb200_esm1b_embed.restype = c_int32
    lib.esmb200_esm1b_embed.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_int32, c_int32,
                                        c_int32, c_void_p, c_int32, c_int32, c_int32, c_void_p]
    lib.esmb200_layernorm.restype = c_int32
    lib.esmb200_layernorm.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_float, c_void_p]
    lib.esmb200_mean_pool.restype = c_int32
    lib.esmb200_mean_pool.argtypes = [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_void_p]
    lib.esmb200_log_softmax_rows.restype = c_int32
    lib.esmb200_log_softmax_rows.argtypes = [c_void_p, c_int64, c_int32, c_int32, c_void_p, c_void_p, c_void_p]
    lib.esmb200_window_merge.restype = c_int32
    lib.esmb200_window_merge.argtypes = [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_void_p,
                                         c_int64, c_void_p]
    lib.esmb200_jacobian_scratch_bytes.restype = c_size_t
    lib.esmb200_jacobian_scratch_bytes.argtypes = [c_int32]
    lib.esmb200_jacobian_contacts.restype = c_int32
    lib.esmb200_jacobian_contacts.argtypes = [c_void_p, c_int32, c_void_p, c_size_t, c_void_p, c_void_p]
    lib.esmb200_sample_order.restype = c_int32
    lib.esmb200_sample_order.argtypes = [c_void_p, c_int32, c_int32, c_int64, c_int64, c_uint64, c_void_p, c_void_p]
    lib.esmb200_sample_rows.restype = c_int32
    lib.esmb200_sample_rows.argtypes = [c_void_p, c_int64, c_int32, c_void_p, c_int32, c_float, c_uint64, c_int64,
                                        c_int64, c_int32, c_void_p, c_void_p, c_int64, c_int32, c_int32, c_void_p,
                                        c_void_p, c_int64, c_void_p]
    lib.esmb200_msa_select_scratch_bytes.restype = c_size_t
    lib.esmb200_msa_select_scratch_bytes.argtypes = [c_int32, c_int32, c_int32]
    lib.esmb200_msa_greedy_select.restype = c_int32
    lib.esmb200_msa_greedy_select.argtypes = [c_void_p, c_int64, c_int32, c_int32, c_int32, c_int32, c_void_p,
                                              c_void_p, c_size_t, c_void_p]
    lib.esmb200_knn_scratch_bytes.restype = c_int32
    lib.esmb200_knn_scratch_bytes.argtypes = [c_int32, c_int32, c_int32, POINTER(c_size_t)]
    lib.esmb200_knn_search.restype = c_int32
    lib.esmb200_knn_search.argtypes = [c_void_p, c_int64, c_int32, c_void_p, c_int64, c_int64, c_int32, c_void_p,
                                       c_float, c_int64, c_int32, c_int32, c_void_p, c_size_t, c_void_p, c_void_p,
                                       c_void_p]
    lib.esmb200_knn_search_accumulate.restype = c_int32
    lib.esmb200_knn_search_accumulate.argtypes = [c_void_p, c_int64, c_int32, c_void_p, c_int64, c_int64, c_int64,
                                                  c_int32, c_void_p, c_float, c_int64, c_int32, c_int32, c_void_p,
                                                  c_size_t, c_void_p, c_void_p]
    lib.esmb200_knn_decode.restype = c_int32
    lib.esmb200_knn_decode.argtypes = [c_void_p, c_int32, c_int32, c_void_p, c_void_p, c_void_p]
    lib.esmb200_knn_range.restype = c_int32
    lib.esmb200_knn_range.argtypes = [c_void_p, c_int64, c_int32, c_void_p, c_int64, c_int64, c_int64, c_int32,
                                      c_void_p, c_float, c_int64, c_void_p, c_int32, c_void_p, c_void_p, c_int64,
                                      c_void_p, c_void_p, c_void_p]
    lib.esmb200_knn_range_finish_scratch_bytes.restype = c_int32
    lib.esmb200_knn_range_finish_scratch_bytes.argtypes = [c_int32, POINTER(c_size_t)]
    lib.esmb200_knn_range_finish.restype = c_int32
    lib.esmb200_knn_range_finish.argtypes = [c_void_p, c_void_p, c_int64, c_void_p, c_int32, c_int64, c_void_p,
                                             c_size_t, c_void_p, c_void_p, c_void_p, c_void_p]
    lib.esmb200_ivf_scratch_bytes.restype = c_int32
    lib.esmb200_ivf_scratch_bytes.argtypes = [c_int32, c_int32, c_int32, c_int64, c_int32, c_int32, POINTER(c_size_t)]
    lib.esmb200_ivf_search.restype = c_int32
    lib.esmb200_ivf_search.argtypes = [c_void_p, c_int64, c_int32, c_void_p, c_int64, c_int64, c_void_p, c_void_p,
                                       c_int32, c_int32, c_void_p, c_float, c_void_p, c_int32, c_void_p, c_int32,
                                       c_void_p, c_size_t, c_void_p, c_void_p, c_void_p]
    lib.esmb200_kmeans_means.restype = c_int32
    lib.esmb200_kmeans_means.argtypes = [c_void_p, c_int64, c_int64, c_int32, c_void_p, c_int32, c_void_p, c_void_p,
                                         c_void_p, c_void_p]
    lib.esmb200_align_scratch_bytes.restype = c_size_t
    lib.esmb200_align_scratch_bytes.argtypes = [c_int32, c_int64, c_int64, c_int64]
    lib.esmb200_align_similarity.restype = c_int32
    lib.esmb200_align_similarity.argtypes = [c_void_p, c_void_p, c_int32, c_void_p, c_void_p, c_void_p, c_int32, c_int64,
                                             c_int64, c_int64, c_int32, c_void_p, c_void_p, c_size_t, c_void_p]
    lib.esmb200_align.restype = c_int32
    lib.esmb200_align.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int64, c_int64, c_int64, c_int32,
                                  c_float, c_float, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]
    lib.esmb200_layernorm_f16.restype = c_int32
    lib.esmb200_layernorm_f16.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_float, c_void_p]
    lib.esmb200_gemm_f16.restype = c_int32
    lib.esmb200_gemm_f16.argtypes = [c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32,
                                     c_void_p, c_void_p, c_int32, c_int32, c_void_p]
    lib.esmb200_gemm_qkv_f16.restype = c_int32
    lib.esmb200_gemm_qkv_f16.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_float, c_void_p,
                                         c_void_p, c_int32, c_void_p]
    lib.esmb200_gemm_qkv_heads.restype = c_int32
    lib.esmb200_gemm_qkv_heads.argtypes = [c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int32,
                                           c_int32, c_int32, c_float, c_void_p, c_void_p, c_int32, c_void_p]
    lib.esmb200_attention_scratch_bytes.restype = c_size_t
    lib.esmb200_attention_scratch_bytes.argtypes = [c_int32, c_int32]
    lib.esmb200_attention.restype = c_int32
    lib.esmb200_attention.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_void_p,
                                      c_void_p]
    lib.esmb200_tied_row_attention_scratch_bytes.restype = c_size_t
    lib.esmb200_tied_row_attention_scratch_bytes.argtypes = [c_int32, c_int32, c_int32]
    lib.esmb200_tied_row_attention.restype = c_int32
    lib.esmb200_tied_row_attention.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32,
                                               c_int32, c_void_p, c_size_t, c_void_p]
    lib.esmb200_column_attention.restype = c_int32
    lib.esmb200_column_attention.argtypes = [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_void_p,
                                             c_void_p]
    lib.esmb200_axial_workspace_bytes.restype = c_size_t
    lib.esmb200_axial_workspace_bytes.argtypes = [c_int32, c_int32, c_int32, c_int32, c_int32]
    lib.esmb200_axial_stack_forward.restype = c_int32
    lib.esmb200_axial_stack_forward.argtypes = [POINTER(c_void_p), POINTER(c_void_p), c_int32, c_void_p, c_void_p,
                                                c_void_p, c_int32, c_int32, c_int32, POINTER(c_void_p),
                                                POINTER(c_void_p), c_void_p, c_size_t, c_void_p]
    lib.esmb200_msa_embed.restype = c_int32
    lib.esmb200_msa_embed.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_void_p, c_void_p, c_float,
                                      c_void_p, c_int32, c_int32, c_int32, c_int32, c_int32, c_void_p]
    lib.esmb200_contact_accumulate.restype = c_int32
    lib.esmb200_contact_accumulate.argtypes = [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                               c_int32, c_int32, c_int32, c_int32, c_int32, c_void_p]
    lib.esmb200_contact_finalize.restype = c_int32
    lib.esmb200_contact_finalize.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32,
                                             c_void_p]
    lib.esmb200_launch_count.restype = ctypes.c_longlong
    lib.esmb200_launch_count.argtypes = []
    lib.esmb200_profile_enable.restype = c_int32
    lib.esmb200_profile_enable.argtypes = [c_int32]
    lib.esmb200_profile_read.restype = c_int32
    lib.esmb200_profile_read.argtypes = [POINTER(c_int32), POINTER(c_float), c_int32]
    lib.esmb200_layernorm_split.restype = c_int32
    lib.esmb200_layernorm_split.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_float, c_void_p]
    lib.esmb200_convert_split.restype = c_int32
    lib.esmb200_convert_split.argtypes = [c_void_p, c_void_p, c_int64, c_int32, c_void_p]
    lib.esmb200_gemm_split.restype = c_int32
    lib.esmb200_gemm_split.argtypes = [c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32,
                                       c_void_p, c_void_p, c_int32, c_int32, c_void_p]
    lib.esmb200_attention128.restype = c_int32
    lib.esmb200_attention128.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_void_p,
                                         c_void_p]
    lib.esmb200_attention_split.restype = c_int32
    lib.esmb200_attention_split.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_void_p,
                                            c_void_p]
    lib.esmb200_axial_workspace_bytes_split.restype = c_size_t
    lib.esmb200_axial_workspace_bytes_split.argtypes = [c_int32, c_int32, c_int32, c_int32, c_int32]
    lib.esmb200_gemm_qkv_split.restype = c_int32
    lib.esmb200_gemm_qkv_split.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_float, c_void_p]
    lib.esmb200_tied_row_attention_split_scratch_bytes.restype = c_size_t
    lib.esmb200_tied_row_attention_split_scratch_bytes.argtypes = [c_int32, c_int32, c_int32]
    lib.esmb200_tied_row_attention_split.restype = c_int32
    lib.esmb200_tied_row_attention_split.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32,
                                                     c_int32, c_void_p, c_size_t, c_void_p]
    lib.esmb200_column_attention_split.restype = c_int32
    lib.esmb200_column_attention_split.argtypes = [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32,
                                                   c_void_p, c_void_p]
    lib.esmb200_set_option.restype = c_int32
    lib.esmb200_set_option.argtypes = [c_char_p, c_int32]
    lib.esmb200_layernorm_fp8.restype = c_int32
    lib.esmb200_layernorm_fp8.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_float,
                                          c_void_p]
    lib.esmb200_quantize_fp8.restype = c_int32
    lib.esmb200_quantize_fp8.argtypes = [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_void_p]
    lib.esmb200_gemm_fp8.restype = c_int32
    lib.esmb200_gemm_fp8.argtypes = [c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                     c_int32, c_int32, c_int32, c_void_p, c_void_p, c_int32, c_int32, c_void_p]
    lib.esmb200_convert_f16.restype = c_int32
    lib.esmb200_convert_f16.argtypes = [c_void_p, c_void_p, c_size_t, c_void_p]


def load():
    """Load libesmb200.so (built in-tree by `__graft_entry__.build()` / `python -m esm_b200.build`)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise Esmb200Error(
                f"{LIB_PATH} not found: build it with `python -m esm_b200.build` (nvcc, sm_90a). "
                "esm_b200 has no CPU or PyTorch fallback for the transformer-layer path."
            )
        lib = ctypes.CDLL(LIB_PATH)
        _declare(lib)
        if lib.esmb200_abi_version() != ABI_VERSION:
            raise Esmb200Error("libesmb200.so ABI version mismatch")
        _lib = lib
    return _lib


def check(rc: int) -> None:
    """Turn a negative return code into a RuntimeError carrying esmb200_last_error()."""
    if rc != 0:
        msg = load().esmb200_last_error()
        raise Esmb200Error((msg.decode() if msg else "unknown error") + f" (esmb200 rc={rc})")
