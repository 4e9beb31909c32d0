"""ctypes binding of libb2m.so (include/b2m.h).  There is NO CPU fallback: if the CUDA
library is missing this module raises at import of the symbols, and b2m_ctx_create fails
without a GPU."""
from __future__ import annotations

import ctypes as C
import os

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(PKG_DIR, "libb2m.so")

# status codes (include/b2m.h)
B2M_OK, B2M_EINVAL, B2M_ECUDA, B2M_ENOMEM, B2M_ESTATE, B2M_EUNSUPPORTED, B2M_EIO = 0, -1, -2, -3, -4, -5, -6
STORE_NO_ODIRECT = 1
DTYPE_BF16, DTYPE_F32, DTYPE_F16, DTYPE_FP8 = 0, 1, 2, 3
EXPERT_SWITCH, EXPERT_SWITCH_GATED, EXPERT_NLLB, EXPERT_FSGPT, EXPERT_MIXTRAL, EXPERT_DEEPSEEK = 0, 1, 2, 3, 4, 5
ROUTER_MIXTRAL, ROUTER_DEEPSEEK_GREEDY, ROUTER_DEEPSEEK_GROUP, ROUTER_SWITCH_TOP1, ROUTER_DEEPSEEK_V3 = 0, 1, 2, 3, 4
ROUTER_QWEN_MOE = 5
ROUTER_LLAMA4 = 6
NUMERICS_REFERENCE, NUMERICS_FP32 = 0, 1
CACHE_REFERENCE, CACHE_SLOTS, CACHE_ACTIVATION_AWARE = 0, 1, 2
WEIGHTS_MODEL_DTYPE, WEIGHTS_FP8_E4M3_B128 = 0, 1
WEIGHTS_INT4_G128, WEIGHTS_INT4_G128_F16 = 4, 6
WEIGHTS_FP8_E4M3_ROW = 7
WS = dict(topk_idx=0, topk_w=1, row_of=2, perm_token=3, counts=4, offsets=5, xp=6, hmid=7, y=8, scores=9, logits=10,
          shared_gate=11, y_shared=12)


class Config(C.Structure):
    _fields_ = [
        ("struct_size", C.c_int32), ("device", C.c_int32), ("num_layers", C.c_int32), ("num_experts", C.c_int32),
        ("hidden", C.c_int32), ("inter", C.c_int32), ("top_k", C.c_int32), ("dtype", C.c_int32),
        ("expert_type", C.c_int32), ("router", C.c_int32), ("numerics", C.c_int32), ("max_tokens", C.c_int32),
        ("num_slots", C.c_int32), ("shared_inter", C.c_int32), ("n_group", C.c_int32), ("topk_group", C.c_int32),
        ("norm_topk_prob", C.c_int32), ("expert_capacity", C.c_int32), ("routed_scaling_factor", C.c_float),
        ("gate_dtype", C.c_int32), ("device_memory_ratio", C.c_double), ("max_inflight_prefetch", C.c_int32),
        ("h2d_chunk_bytes", C.c_int32), ("gemm_impl", C.c_int32), ("cache_policy", C.c_int32),
        ("lookahead_prefetch", C.c_int32), ("freq_alpha", C.c_float),
    ]


class Stats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in (
        "dispatches", "hits", "misses", "prefetch_issued", "prefetch_useful", "evictions", "h2d_bytes",
        "host_syncs", "kernel_launches", "resident", "slots", "slot_bytes")]

    def as_dict(self):
        return {n: int(getattr(self, n)) for n, _ in self._fields_}


# every symbol include/b2m.h declares: (name, restype, argtypes)
_VP, _I, _SZ = C.c_void_p, C.c_int, C.c_size_t
SYMBOLS = [
    ("b2m_last_error", C.c_char_p, [_VP]),
    ("b2m_version", _I, []),
    ("b2m_ctx_create", _I, [C.POINTER(Config), C.POINTER(_VP)]),
    ("b2m_ctx_create_ex", _I, [C.POINTER(Config), _I, C.POINTER(_VP)]),
    ("b2m_ctx_destroy", _I, [_VP]),
    ("b2m_register_expert", _I, [_VP, _I, _I, _VP, _SZ]),
    ("b2m_register_shared", _I, [_VP, _I, _VP, _SZ]),
    ("b2m_set_gate", _I, [_VP, _I, _VP]),
    ("b2m_set_gate_bias", _I, [_VP, _I, _VP]),
    ("b2m_set_input_perm", _I, [_VP, _I, _VP]),
    ("b2m_set_shared_gate", _I, [_VP, _I, _VP]),
    ("b2m_host_pin", _I, [_VP, _VP, _SZ]),
    ("b2m_host_unpin", _I, [_VP, _VP]),
    ("b2m_make_resident", _I, [_VP, _I, _I, _I, _VP]),
    ("b2m_expert_dev_ptr", _I, [_VP, _I, _I, C.POINTER(_VP)]),
    ("b2m_shared_dev_ptr", _I, [_VP, _I, C.POINTER(_VP)]),
    ("b2m_moe_forward", _I, [_VP, _I, _VP, _VP, _I, _I, _I, _I, _VP, _VP]),
    ("b2m_route", _I, [_VP, _I, _VP, _VP, _I, _I, _I, _I, _VP]),
    ("b2m_route_from_mask", _I, [_VP, _I, _VP, _VP, _I, _VP]),
    ("b2m_run_experts", _I, [_VP, _I, _I, _VP]),
    ("b2m_run_experts_ex", _I, [_VP, _I, _I, _I, _VP]),
    ("b2m_combine", _I, [_VP, _I, _VP, _I, _VP, _VP]),
    ("b2m_expert_outputs", _I, [_VP, _I, _VP, C.POINTER(C.c_int), _VP]),
    ("b2m_check_errors", _I, [_VP, _VP]),
    ("b2m_ws_ptr", _I, [_VP, _I, C.POINTER(_VP)]),
    ("b2m_replace_cache_candidates", _I, [_VP, _I, C.POINTER(C.c_int32)]),
    ("b2m_enqueue_prefetch", _I, [_VP, _I, _I]),
    ("b2m_prefetch_hint", _I, [_VP, _I, C.POINTER(C.c_int32), C.POINTER(C.c_float)]),
    ("b2m_prefetch_pump", _I, [_VP]),
    ("b2m_prefetch_drain", _I, [_VP]),
    ("b2m_clear_expert_cache_counts", _I, [_VP]),
    ("b2m_is_resident", _I, [_VP, _I, _I]),
    ("b2m_stats_get", _I, [_VP, C.POINTER(Stats)]),
    ("b2m_last_counts", _I, [_VP, C.POINTER(C.c_int32)]),
    ("b2m_last_lookahead", _I, [_VP, C.POINTER(C.c_int32)]),
    ("b2m_ep_pack", _I, [_VP, _I, _I, _I, _I, _VP, _VP, _VP]),
    ("b2m_ep_regroup", _I, [_VP, _I, _I, _I, _I, _VP, _VP, _VP]),
    ("b2m_ep_ungroup", _I, [_VP, _I, _I, _I, _VP, _VP]),
    ("b2m_ep_unpack", _I, [_VP, _I, _I, _I, _I, _VP, _VP]),
    ("b2m_ep_p2p_init", _I, [_VP, _I, _I, _I, _VP]),
    ("b2m_ep_p2p_open", _I, [_VP, _I, _VP]),
    ("b2m_ep_p2p_dispatch", _I, [_VP, _I, _VP]),
    ("b2m_ep_p2p_regroup", _I, [_VP, _I, _VP]),
    ("b2m_ep_p2p_return", _I, [_VP, _VP]),
    ("b2m_ep_p2p_collect", _I, [_VP, _I, _VP]),
    ("b2m_ep_p2p_route", _I, [_VP, _I, _VP, _VP, _I, _I, _I, _VP]),
    ("b2m_ep_p2p_combine", _I, [_VP, _I, _VP, _I, _VP, _VP]),
    ("b2m_ep_p2p_layer", _I, [_VP, _I, _VP, _VP, _I, _I, _I, _VP, _VP]),
    ("b2m_timeline_read", _I, [_VP, C.POINTER(C.c_uint64), _I]),
    ("b2m_trace_init", _I, [_VP, _I, _I, _I]),
    ("b2m_trace_load", _I, [_VP, _I, _VP]),
    ("b2m_trace_reset_seq", _I, [_VP, _I, _VP]),
    ("b2m_trace_update_predict", _I, [_VP, _I, _I, _I, _I, _VP]),
    ("b2m_trace_finish_seq", _I, [_VP, _I, _VP]),
    ("b2m_trace_read", _I, [_VP, _I, _I, _VP]),
    # disk tier (host code: usable without a GPU)
    ("b2m_store_open", _I, [C.c_char_p, _I, _I, _I, C.POINTER(_VP)]),
    ("b2m_store_close", _I, [_VP]),
    ("b2m_store_last_error", C.c_char_p, [_VP]),
    ("b2m_store_count", _I, [_VP]),
    ("b2m_store_tensor", _I, [_VP, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_int64), C.POINTER(C.c_uint64)]),
    ("b2m_store_blob_bytes", _I, [_VP, C.POINTER(C.c_uint32), _I, C.POINTER(C.c_uint64)]),
    ("b2m_store_read_async", _I, [_VP, C.POINTER(C.c_uint32), _I, _VP, C.c_uint64, _I, C.POINTER(C.c_uint64)]),
    ("b2m_store_read_range_async", _I, [_VP, C.POINTER(C.c_uint32), _I, C.c_uint64, C.c_uint64, _VP, _I, C.POINTER(C.c_uint64)]),
    ("b2m_store_poll", _I, [_VP, C.c_uint64]),
    ("b2m_store_wait", _I, [_VP, C.c_uint64]),
    ("b2m_store_stats", _I, [_VP, C.POINTER(C.c_uint64)]),
    ("b2m_register_expert_on_store", _I, [_VP, _I, _I, _VP, C.POINTER(C.c_uint32), _I]),
]

_lib = None


class B2MError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"libb2m error {code}: {msg}")
        self.code = code


def load():
    """dlopen libb2m.so and bind every declared symbol.  Raises if the library is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is not built. Run `python -m moe_infinity_b200.build` (nvcc, sm_90a). "
            "This package has no CPU or PyTorch fallback for the MoE dispatch path.")
    lib = C.CDLL(LIB_PATH)
    for name, res, args in SYMBOLS:
        fn = getattr(lib, name)   # AttributeError if the .so lacks a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(ctx, code):
    if code != 0:
        msg = load().b2m_last_error(ctx)
        raise B2MError(code, msg.decode() if msg else "")
    return code
