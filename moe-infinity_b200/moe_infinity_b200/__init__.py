"""moe_infinity_b200 -- H100-native (sm_90a) MoE expert dispatch/offload hot path.

Drop-in for the one hot path of EfficientMoE/MoE-Infinity (router top-k -> permute -> grouped expert GEMM ->
combine, plus HBM expert cache and prefetch).  Everything numerical runs in libb2m.so (hand-written CUDA);
this package is the Python host side mirroring the reference's plugin surface.  No CPU fallback exists.
"""
from . import _lib  # noqa: F401
from ._lib import (DTYPE_BF16, DTYPE_F16, DTYPE_F32, EXPERT_DEEPSEEK, EXPERT_MIXTRAL, EXPERT_SWITCH,  # noqa: F401
                   EXPERT_SWITCH_GATED, NUMERICS_FP32, NUMERICS_REFERENCE, ROUTER_DEEPSEEK_GREEDY,
                   ROUTER_DEEPSEEK_GROUP, ROUTER_MIXTRAL, ROUTER_SWITCH_TOP1, B2MError)

__all__ = ["MoEEngine", "DecodeSession", "B2MError"]


def __getattr__(name):
    if name == "MoEEngine":
        from .engine import MoEEngine
        return MoEEngine
    if name == "DecodeSession":
        from .engine import DecodeSession
        return DecodeSession
    raise AttributeError(name)
