"""ctypes binding of libb200awq.so (include/b200awq.h).  No fallback: if the CUDA library is missing
or a call fails, this raises - the product path never routes through the CPU oracle."""
from __future__ import annotations

import ctypes
import os

_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib", "libb200awq.so")

OK = 0
ABI_VERSION = 1

_c_void_p, _c_int, _c_i64, _c_size_t, _c_float = (
    ctypes.c_void_p,
    ctypes.c_int,
    ctypes.c_int64,
    ctypes.c_size_t,
    ctypes.c_float,
)



class Op(ctypes.Structure):
    """b200awq_op_t (include/b200awq.h): one recorded operator call of a decode program."""

    _fields_ = [
        ("kind", ctypes.c_int32), ("M", ctypes.c_int32), ("K", ctypes.c_int32), ("N", ctypes.c_int32),
        ("group_size", ctypes.c_int32), ("eps", ctypes.c_float), ("ldx", ctypes.c_int64),
        ("x", ctypes.c_void_p), ("qweight", ctypes.c_void_p), ("scales", ctypes.c_void_p),
        ("qzeros", ctypes.c_void_p), ("bias", ctypes.c_void_p), ("weight", ctypes.c_void_p), ("y", ctypes.c_void_p),
    ]


class Moe(ctypes.Structure):
    """b200awq_moe_t (include/b200awq.h): the descriptor a SPARSE_MOE op's `weight` points at."""

    _fields_ = [
        ("E", ctypes.c_int32), ("top_k", ctypes.c_int32), ("renormalize", ctypes.c_int32),
        ("group_size", ctypes.c_int32), ("H", ctypes.c_int32), ("I", ctypes.c_int32), ("block_size", ctypes.c_int32),
        ("sorted_len", ctypes.c_int32), ("gate_weight", ctypes.c_void_p),
        ("w1_qweight", ctypes.c_void_p), ("w1_scales", ctypes.c_void_p), ("w1_qzeros", ctypes.c_void_p),
        ("w2_qweight", ctypes.c_void_p), ("w2_scales", ctypes.c_void_p), ("w2_qzeros", ctypes.c_void_p),
        ("logits", ctypes.c_void_p), ("topk_weights", ctypes.c_void_p), ("topk_ids", ctypes.c_void_p),
        ("token_expert_indices", ctypes.c_void_p), ("sorted_ids", ctypes.c_void_p), ("expert_ids", ctypes.c_void_p),
        ("num_tokens_post_pad", ctypes.c_void_p), ("gate_up", ctypes.c_void_p), ("act", ctypes.c_void_p),
        ("down", ctypes.c_void_p),
    ]


class DeepseekMoe(ctypes.Structure):
    """b200awq_deepseek_moe_t (include/b200awq.h): the descriptor a DEEPSEEK_MOE op's `weight` points at."""

    _fields_ = [
        ("moe", Moe), ("scoring", ctypes.c_int32), ("n_group", ctypes.c_int32), ("topk_group", ctypes.c_int32),
        ("norm_topk_prob", ctypes.c_int32), ("routed_scaling_factor", ctypes.c_float), ("I_s", ctypes.c_int32),
        ("bias", ctypes.c_void_p), ("ws1_qweight", ctypes.c_void_p), ("ws1_scales", ctypes.c_void_p),
        ("ws1_qzeros", ctypes.c_void_p), ("ws2_qweight", ctypes.c_void_p), ("ws2_scales", ctypes.c_void_p),
        ("ws2_qzeros", ctypes.c_void_p), ("shared_out", ctypes.c_void_p),
    ]


class Rope(ctypes.Structure):
    """b200awq_rope_t (include/b200awq.h): the descriptor of b200awq_rope_kv and of a ROPE_KV op's `weight`."""

    _fields_ = [
        ("n_heads", ctypes.c_int32), ("n_kv_heads", ctypes.c_int32), ("head_dim", ctypes.c_int32),
        ("cache_len", ctypes.c_int32), ("freqs_len", ctypes.c_int32), ("rotary_dim", ctypes.c_int32),
        ("cache_batch_stride", ctypes.c_int64), ("pos", ctypes.c_void_p), ("freqs", ctypes.c_void_p),
        ("q_out", ctypes.c_void_p), ("k_cache", ctypes.c_void_p), ("v_cache", ctypes.c_void_p),
    ]


class QkNormRope(ctypes.Structure):
    """b200awq_qk_norm_rope_t (include/b200awq.h): the descriptor of b200awq_qk_norm_rope_kv and of a QK_NORM_ROPE_KV
    op's `weight`."""

    _fields_ = [
        ("rope", Rope), ("q_norm_weight", ctypes.c_void_p), ("k_norm_weight", ctypes.c_void_p), ("eps", ctypes.c_float),
        ("pad_", ctypes.c_int32),
    ]


class RopeOffset(ctypes.Structure):
    """b200awq_rope_offset_t (include/b200awq.h): the descriptor of b200awq_rope_kv_offset and of a ROPE_KV_OFFSET op's
    `weight` (null norm weights: no q / k norm)."""

    _fields_ = [("qk", QkNormRope), ("rot_offset", ctypes.c_void_p)]


class Mla(ctypes.Structure):
    """b200awq_mla_t (include/b200awq.h): the descriptor of b200awq_mla_rope / _kv / _k_rope / _q_rope and of an
    MLA_ROPE / MLA_KV / MLA_K_ROPE / MLA_Q_ROPE op's `weight`."""

    _fields_ = [
        ("n_heads", ctypes.c_int32), ("nope_dim", ctypes.c_int32), ("rope_dim", ctypes.c_int32),
        ("v_dim", ctypes.c_int32), ("kv_lora_rank", ctypes.c_int32), ("style", ctypes.c_int32),
        ("cache_len", ctypes.c_int32), ("freqs_len", ctypes.c_int32), ("k_batch_stride", ctypes.c_int64),
        ("v_batch_stride", ctypes.c_int64), ("v_head_stride", ctypes.c_int32), ("pad_", ctypes.c_int32),
        ("pos", ctypes.c_void_p), ("freqs", ctypes.c_void_p), ("q_out", ctypes.c_void_p), ("k_cache", ctypes.c_void_p),
        ("v_cache", ctypes.c_void_p),
    ]


OP_RMSNORM, OP_LINEAR_GEMM, OP_SILU_AND_MUL, OP_SPARSE_MOE, OP_ADD, OP_ROPE_KV = 1, 2, 3, 4, 5, 6
OP_QK_NORM_ROPE_KV, OP_QWEN3_MOE, OP_DEEPSEEK_MOE, OP_MLA_ROPE, OP_MLA_KV = 7, 8, 9, 10, 11
OP_MLA_K_ROPE, OP_MLA_Q_ROPE = 12, 13
OP_LAYER_NORM, OP_GELU, OP_GELU_TANH = 14, 15, 16
OP_ROPE_KV_SEQ, OP_QK_NORM_ROPE_KV_SEQ, OP_ROPE_KV_OFFSET = 17, 18, 19
OP_SCALED_ADD = 20
EUNSUPPORTED = 2

# name -> (restype, argtypes); mirrors include/b200awq.h one to one
SIGNATURES = {
    "b200awq_abi_version": (_c_int, []),
    "b200awq_error_string": (ctypes.c_char_p, [_c_int]),
    "b200awq_last_cuda_error": (ctypes.c_char_p, []),
    "b200awq_workspace_bytes": (_c_size_t, [_c_int, _c_int, _c_int]),
    "b200awq_dequantize_gemm": (_c_int, [_c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_int, _c_int, _c_int, _c_void_p]),
    "b200awq_gemm_forward": (
        _c_int,
        [_c_void_p, _c_i64, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_int, _c_int, _c_int, _c_int,
         _c_void_p, _c_size_t, _c_void_p],
    ),
    "b200awq_gemv_forward": (
        _c_int,
        [_c_void_p, _c_i64, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_int, _c_int, _c_int, _c_int,
         _c_void_p, _c_size_t, _c_void_p],
    ),
    "b200awq_fast_forward": (
        _c_int,
        [_c_void_p, _c_i64, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_int, _c_int, _c_int, _c_int,
         _c_void_p, _c_size_t, _c_void_p],
    ),
    "b200awq_rmsnorm": (_c_int, [_c_void_p, _c_void_p, _c_void_p, _c_int, _c_int, _c_float, _c_void_p]),
    "b200awq_silu_and_mul": (_c_int, [_c_void_p, _c_void_p, _c_int, _c_int, _c_void_p]),
    "b200awq_layer_norm": (_c_int, [_c_void_p, _c_i64, _c_void_p, _c_void_p, _c_void_p, _c_int, _c_int, _c_float,
                                    _c_void_p]),
    "b200awq_gelu": (_c_int, [_c_void_p, _c_void_p, _c_int, _c_int, _c_int, _c_void_p]),
    "b200awq_rope_kv": (_c_int, [_c_void_p, _c_i64, ctypes.POINTER(Rope), _c_int, _c_void_p]),
    "b200awq_qk_norm_rope_kv": (_c_int, [_c_void_p, _c_i64, ctypes.POINTER(QkNormRope), _c_int, _c_void_p]),
    "b200awq_rope_kv_seq": (_c_int, [_c_void_p, _c_i64, ctypes.POINTER(Rope), _c_int, _c_int, _c_void_p]),
    "b200awq_qk_norm_rope_kv_seq": (_c_int, [_c_void_p, _c_i64, ctypes.POINTER(QkNormRope), _c_int, _c_int,
                                             _c_void_p]),
    "b200awq_rope_kv_offset": (_c_int, [_c_void_p, _c_i64, ctypes.POINTER(RopeOffset), _c_int, _c_int, _c_void_p]),
    "b200awq_mla_rope": (_c_int, [_c_void_p, _c_i64, ctypes.POINTER(Mla), _c_int, _c_void_p]),
    "b200awq_mla_kv": (_c_int, [_c_void_p, _c_i64, ctypes.POINTER(Mla), _c_int, _c_void_p]),
    "b200awq_mla_k_rope": (_c_int, [_c_void_p, _c_i64, _c_i64, ctypes.POINTER(Mla), _c_int, _c_void_p]),
    "b200awq_mla_q_rope": (_c_int, [_c_void_p, _c_i64, ctypes.POINTER(Mla), _c_int, _c_void_p]),
    "b200awq_set_knob": (_c_int, [_c_int, _c_int]),
    "b200awq_get_knob": (_c_int, [_c_int]),
    "b200awq_debug_read": (_c_int, [_c_void_p, _c_size_t]),
    "b200awq_tcq_plan": (_c_int, [_c_int, _c_int, _c_int, _c_int, _c_int, _c_int, _c_void_p, _c_void_p]),
    "b200awq_topk_softmax": (_c_int, [_c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_int, _c_int, _c_int, _c_void_p]),
    "b200awq_moe_align_block_size": (_c_int, [_c_void_p, _c_int, _c_int, _c_int, _c_void_p, _c_void_p, _c_void_p,
                                              _c_void_p]),
    "b200awq_grouped_gemm_forward": (
        _c_int,
        [_c_void_p, _c_int, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p,
         _c_int, _c_int, _c_int, _c_int, _c_int, _c_int, _c_int, _c_int, _c_int, _c_void_p, _c_size_t, _c_void_p],
    ),
    "b200awq_moe_tc_plan": (_c_int, [_c_void_p, _c_int, _c_int, _c_int, _c_int, _c_int, _c_int, _c_void_p, _c_int,
                                     _c_void_p]),
    "b200awq_comm_create": (_c_int, [_c_int, _c_int, _c_int, ctypes.POINTER(_c_void_p)]),
    "b200awq_comm_ipc_handle": (_c_int, [_c_void_p, _c_void_p]),
    "b200awq_comm_open": (_c_int, [_c_void_p, _c_void_p]),
    "b200awq_comm_all_reduce": (_c_int, [_c_void_p, _c_void_p, _c_int, _c_void_p]),
    "b200awq_comm_error": (_c_int, [_c_void_p]),
    "b200awq_comm_destroy": (_c_int, [_c_void_p]),
    "b200awq_program_create": (_c_int, [ctypes.POINTER(Op), _c_int, ctypes.POINTER(_c_void_p)]),
    "b200awq_program_create_batched": (_c_int, [ctypes.POINTER(Op), _c_int, _c_int, ctypes.POINTER(_c_void_p)]),
    "b200awq_program_tokens": (_c_int, [_c_void_p]),
    "b200awq_program_plan": (_c_int, [ctypes.POINTER(Op), _c_int, _c_int, _c_int, _c_int, _c_void_p]),
    "b200awq_moe_plan": (_c_int, [_c_int, _c_int, _c_int, _c_int, _c_int, _c_int, _c_void_p]),
    "b200awq_qwen3_moe_plan": (_c_int, [_c_int, _c_int, _c_int, _c_int, _c_int, _c_int, _c_void_p]),
    "b200awq_deepseek_moe_plan": (_c_int, [_c_int, _c_int, _c_int, _c_int, _c_int, _c_int, _c_int, _c_void_p]),
    "b200awq_program_num_ops": (_c_int, [_c_void_p]),
    "b200awq_program_kind": (_c_int, [_c_void_p]),
    "b200awq_stream_bytes": (_c_size_t, [_c_int, _c_int, _c_int]),
    "b200awq_stream_pack": (_c_int, [_c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_int, _c_int, _c_int, _c_int, _c_void_p]),
    "b200awq_stream_pack_rotary": (_c_int, [_c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_int, _c_int, _c_int, _c_int,
                                            _c_void_p]),
    "b200awq_stream_pack_partial_rotary": (_c_int, [_c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_int, _c_int, _c_int,
                                                    _c_int, _c_int, _c_void_p]),
    "b200awq_program_run": (_c_int, [_c_void_p, _c_void_p, _c_size_t, _c_void_p]),
    "b200awq_program_destroy": (_c_int, [_c_void_p]),
}


class B200AwqError(RuntimeError):
    """Raised for every non-zero return code of the C ABI (the reference's kernels raise
    RuntimeError through TORCH_CHECK; same class hierarchy here)."""


def _load():
    if not os.path.exists(_LIB_PATH):
        raise ImportError(
            f"{_LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). There is no CPU fallback."
        )
    lib = ctypes.CDLL(_LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the library does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    v = lib.b200awq_abi_version()
    if v != ABI_VERSION:
        raise ImportError(f"libb200awq ABI {v} != expected {ABI_VERSION}")
    return lib


lib = _load()


def check(code: int, what: str) -> None:
    if code != OK:
        msg = lib.b200awq_error_string(code).decode()
        cu = lib.b200awq_last_cuda_error().decode()
        raise B200AwqError(f"{what}: {msg}" + (f" [{cu}]" if code == 4 and cu else ""))


def lib_path() -> str:
    return _LIB_PATH
