"""HuggingFace plug-in helpers: run a `transformers` Mixtral or DeepSeek-V3 model with its MoE blocks executed by the CUDA
engine (`patch_mixtral`, `patch_deepseek_v3`).

The reference achieves this by monkey-patching HF classes at load time (moe_infinity/runtime/model_offload.py:285-321:
`MixtralSparseMoeBlock -> SyncMixtralSparseMoeBlock`).  The installed transformers (5.x) stores the experts of a layer as
fused 3-D parameters (`MixtralExperts.gate_up_proj [E, 2I, H]`, `down_proj [E, H, I]`) and its block returns the hidden
states only, so this helper swaps `layer.mlp` for an adapter with that signature; the adapter keeps the router GEMM in
PyTorch (same logits as HF) and hands everything after it to `MoEEngine.forward`.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib as L
from . import fp8 as F8
from . import int4 as I4
from .engine import MoEEngine


def _load(engine: MoEEngine, layer: int, expert: int, ws, resident: bool):
    """Hand one expert's bf16 matrices to `engine`, quantised first when the engine stores fp8 (`fp8.quantize_block128`) or
    int4 (`int4.quantize_g128`) experts."""
    kw = {}
    if engine.fp8:
        ws, scales = zip(*[F8.quantize_block128(w) for w in ws])
        kw = dict(scales=scales)
    elif engine.int4:
        ws, scales, zeros = zip(*[I4.quantize_g128(w) for w in ws])
        kw = dict(scales=scales, zeros=zeros)
    if resident:
        engine.load_expert(layer, expert, ws, **kw)
    else:
        engine.register_expert(layer, expert, ws, **kw)


class B200MixtralMoeAdapter(nn.Module):
    """Drop-in for transformers>=5 `MixtralSparseMoeBlock`: forward(hidden[B,S,H]) -> hidden[B,S,H]."""

    def __init__(self, engine: MoEEngine, layer_id: int, gate_weight: torch.Tensor):
        super().__init__()
        self.engine = engine
        self.layer_id = layer_id
        self.gate_weight = nn.Parameter(gate_weight.detach().clone(), requires_grad=False)

    def forward(self, hidden_states: torch.Tensor) -> torch.Tensor:
        shape = hidden_states.shape
        x = hidden_states.reshape(-1, shape[-1])
        router_logits = F.linear(x, self.gate_weight)      # same GEMM HF's MixtralTopKRouter runs
        out = self.engine.forward(self.layer_id, x, router_logits=router_logits)
        return out.reshape(shape)


def patch_mixtral(model, max_tokens: int = 4096, num_slots: int = 0, device_memory_ratio: float = 0.0,
                  resident: bool = True, engine: Optional[MoEEngine] = None) -> MoEEngine:
    """Move every expert of `model` (a transformers MixtralForCausalLM / MixtralModel on a CUDA device) into a
    MoEEngine and replace the MoE blocks.  `resident=False` registers experts as pinned host blobs (offload mode,
    budget from num_slots / device_memory_ratio) instead of loading all of them into HBM.  `engine` may be given (built with
    the model's shapes), e.g. one with expert_dtype=torch.uint4: the experts are then quantised with `int4.quantize_g128`."""
    cfg = model.config
    layers = model.model.layers if hasattr(model, "model") else model.layers
    dev = next(model.parameters()).device
    dtype = next(model.parameters()).dtype
    L, E, H, I, k = len(layers), cfg.num_local_experts, cfg.hidden_size, cfg.intermediate_size, cfg.num_experts_per_tok
    if engine is None:
        engine = MoEEngine(num_layers=L, num_experts=E, hidden=H, inter=I, top_k=k, dtype=dtype, max_tokens=max_tokens,
                           num_slots=(L * E if resident and not num_slots else num_slots),
                           device_memory_ratio=device_memory_ratio, device=dev.index or 0)
    for l, layer in enumerate(layers):
        moe = layer.mlp
        gu, dn = moe.experts.gate_up_proj.data, moe.experts.down_proj.data     # [E,2I,H], [E,H,I]
        for e in range(E):
            w1, w3, w2 = gu[e, :I], gu[e, I:], dn[e]                            # reference order: w1 | w2 | w3
            _load(engine, l, e, [w1, w2, w3], resident)
        layer.mlp = B200MixtralMoeAdapter(engine, l, moe.gate.weight.data)
    return engine


class B200DeepseekV3MoeAdapter(nn.Module):
    """Drop-in for transformers>=5 `DeepseekV3MoE`: forward(hidden[B,S,H]) -> hidden[B,S,H].  The router (fp32 gate GEMM,
    sigmoid, correction bias, group selection, weights), the routed experts, the shared expert and the combine all run in
    the engine (fused gate, router_in_kind 0)."""

    def __init__(self, engine: MoEEngine, layer_id: int):
        super().__init__()
        self.engine = engine
        self.layer_id = layer_id

    def forward(self, hidden_states: torch.Tensor) -> torch.Tensor:
        shape = hidden_states.shape
        out = self.engine.forward(self.layer_id, hidden_states.reshape(-1, shape[-1]))
        return out.reshape(shape)


def patch_deepseek_v3(model, max_tokens: int = 4096, num_slots: int = 0, device_memory_ratio: float = 0.0,
                      resident: bool = True, engine: Optional[MoEEngine] = None) -> MoEEngine:
    """Move the routed experts, shared experts, router weights and correction biases of `model` (a transformers
    DeepseekV3ForCausalLM / DeepseekV3Model on a CUDA device) into a MoEEngine (ROUTER_DEEPSEEK_V3) and replace its MoE
    blocks (layers >= config.first_k_dense_replace; the dense layers before them stay as they are).  `engine` may be
    given (built with router=ROUTER_DEEPSEEK_V3 and the model's shapes), e.g. one with expert_dtype=torch.float8_e4m3fn or
    torch.uint4: the experts are then quantised with `fp8.quantize_block128` or `int4.quantize_g128`.  `resident=False` registers experts as pinned host
    blobs (offload mode, budget from num_slots / device_memory_ratio)."""
    cfg = model.config
    if cfg.num_experts_per_tok == 1 and cfg.norm_topk_prob:
        # transformers normalises a single weight to 1 here; the reference gate (and this engine) only normalise for k > 1
        raise ValueError("num_experts_per_tok == 1 with norm_topk_prob: transformers and the reference gate disagree")
    layers = model.model.layers if hasattr(model, "model") else model.layers
    dev = next(model.parameters()).device
    dtype = next(model.parameters()).dtype
    L_, E, H, I, k = len(layers), cfg.n_routed_experts, cfg.hidden_size, cfg.moe_intermediate_size, cfg.num_experts_per_tok
    moe_layers = [l for l in range(L_) if l >= cfg.first_k_dense_replace]
    if engine is None:
        engine = MoEEngine(num_layers=L_, num_experts=E, hidden=H, inter=I, top_k=k, dtype=dtype, expert_type=L.EXPERT_DEEPSEEK,
                           router=L.ROUTER_DEEPSEEK_V3, max_tokens=max_tokens, num_slots=(L_ * E if resident and not num_slots else num_slots),
                           device_memory_ratio=device_memory_ratio, shared_inter=I * cfg.n_shared_experts, n_group=cfg.n_group,
                           topk_group=cfg.topk_group, norm_topk_prob=cfg.norm_topk_prob,
                           routed_scaling_factor=cfg.routed_scaling_factor, gate_dtype=torch.float32, device=dev.index or 0)
    elif engine.router != L.ROUTER_DEEPSEEK_V3:
        raise ValueError("patch_deepseek_v3 needs an engine built with router=ROUTER_DEEPSEEK_V3")
    for l in moe_layers:
        moe = layers[l].mlp
        gu, dn = moe.experts.gate_up_proj.data, moe.experts.down_proj.data     # [E,2I,H], [E,H,I]
        for e in range(E):
            _load(engine, l, e, [gu[e, :I], gu[e, I:], dn[e]], resident)     # DeepSeek order: gate | up | down
        sh = moe.shared_experts
        engine.register_shared(l, [sh.gate_proj.weight.data, sh.up_proj.weight.data, sh.down_proj.weight.data])
        engine.set_gate(l, moe.gate.weight.data)
        engine.set_gate_bias(l, moe.gate.e_score_correction_bias.data)
        layers[l].mlp = B200DeepseekV3MoeAdapter(engine, l)
    return engine
