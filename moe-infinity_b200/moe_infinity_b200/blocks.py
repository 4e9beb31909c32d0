"""Drop-in MoE blocks: same class names, constructor arguments, injected attributes and forward signatures as
the reference's moe_infinity/models/{mixtral,deepseek,switch_transformers}.py, so a user of
`moe_infinity.MoE(...)` finds the same plugin surface.

forward() keeps the router GEMM in PyTorch exactly where the reference has it (mixtral.py:46 `self.gate`;
MoEGate's fp32 F.linear), so the logits the routing sees are the ones the reference would see, and hands
everything after it -- softmax/top-k, permute, expert FFNs, combine -- to ONE asynchronous call into the CUDA
engine through the attribute the reference already injects (`self.expert_executor`, model_offload.py:572-604).
If the injected executor only offers the reference's `dispatch_local`, the reference's own Python combine loop
is used with it (compat path); no arithmetic of the path is ever done by PyTorch on the host.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F


def _is_fast(executor) -> bool:
    return hasattr(executor, "moe_forward")


class SyncMixtralSparseMoeBlock(nn.Module):
    """moe_infinity/models/mixtral.py:18-118."""
    archer_config = None
    layer_id: int = None

    def __init__(self, config):
        super().__init__()
        self.hidden_dim = config.hidden_size
        self.ffn_dim = config.intermediate_size
        self.num_experts = config.num_local_experts
        self.top_k = config.num_experts_per_tok
        self.gate = nn.Linear(self.hidden_dim, self.num_experts, bias=False)   # mixtral.py:30
        self.expert_executor = None
        self.expert_prefetcher = None
        self.expert_predictor = None
        self.expert_tensor_ids: Dict[int, int] = None
        self.seq_id_list = None

    def forward(self, hidden_states: torch.Tensor):
        batch_size, sequence_length, hidden_dim = hidden_states.shape
        x = hidden_states.view(-1, hidden_dim)
        router_logits = self.gate(x)                                            # mixtral.py:46
        if _is_fast(self.expert_executor):
            final = self.expert_executor.moe_forward(self.layer_id, x, router_logits=router_logits)
            if self.expert_predictor is not None and self.seq_id_list is not None:
                self._predict_and_prefetch(batch_size, sequence_length)
            return final.reshape(batch_size, sequence_length, hidden_dim), router_logits
        # ---- compat path: reference algorithm verbatim in structure, expert math in the executor (mixtral.py:48-101)
        routing_weights = F.softmax(router_logits, dim=1, dtype=torch.float)
        routing_weights, selected_experts = torch.topk(routing_weights, self.top_k, dim=-1)
        routing_weights /= routing_weights.sum(dim=-1, keepdim=True)
        routing_weights = routing_weights.to(x.dtype)
        router_mask = F.one_hot(selected_experts, num_classes=self.num_experts)
        routing_weights_mask = (routing_weights[:, :, None] * router_mask).permute(0, 2, 1)
        router_mask = router_mask.permute(0, 2, 1)
        rm = router_mask[:, :, 0].bool()
        for j in range(1, self.top_k):
            rm = torch.logical_or(rm, router_mask[:, :, j])
        routing_weights_mask = torch.sum(routing_weights_mask, dim=-1)
        final = torch.zeros((batch_size * sequence_length, hidden_dim), dtype=x.dtype, device=x.device)
        results = self.expert_executor.dispatch_local(x, rm, self.layer_id)
        for output, _, idx, _ in results:
            token_indices = rm[:, idx].bool()
            final[token_indices, :] += output.to(final.device) * routing_weights_mask[token_indices, idx][:, None]
        return final.reshape(batch_size, sequence_length, hidden_dim), router_logits

    def _predict_and_prefetch(self, batch_size, sequence_length):
        """The calls the reference has commented out on this block (mixtral.py:71-85): per sequence,
        predict(seq_id, expert_index[i], layer) -> prefetch_experts(layer, matrix)."""
        eng = self.expert_executor.expert_dispatcher.engine if hasattr(self.expert_executor.expert_dispatcher, "engine") \
            else self.expert_executor.expert_dispatcher
        idx = eng.ws("topk_idx", batch_size * sequence_length).reshape(batch_size, sequence_length, self.top_k).cpu().numpy()
        for i in range(batch_size):
            m = self.expert_predictor.predict(self.seq_id_list[i], idx[i], self.layer_id)
            self.expert_prefetcher.prefetch_experts(self.layer_id, m)


def _engine_of(executor):
    d = executor.expert_dispatcher
    return d.engine if hasattr(d, "engine") else d


class DeepseekMoEBlock(nn.Module):
    """moe_infinity/models/deepseek.py:8-137 (DeepSeek-V2 gate: modeling_deepseek.py:436-512; DeepSeek-V3 gate when
    config.model_type == "deepseek_v3" or config.topk_method == "noaux_tc": modeling_deepseek_v3/modeling_deepseek.py:436-527,
    routed by an engine built with ROUTER_DEEPSEEK_V3)."""
    layer_id: int = None

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.num_experts_per_tok = config.num_experts_per_tok
        self.v3 = getattr(config, "model_type", None) == "deepseek_v3" or getattr(config, "topk_method", None) == "noaux_tc"
        self.gate_weight = nn.Parameter(torch.empty((config.n_routed_experts, config.hidden_size)))
        nn.init.kaiming_uniform_(self.gate_weight, a=5 ** 0.5)
        if self.v3:   # MoEGate.e_score_correction_bias (modeling_deepseek_v3/modeling_deepseek.py:455-458)
            self.e_score_correction_bias = nn.Parameter(torch.zeros(config.n_routed_experts, dtype=torch.float32))
        self._bias_handed = None
        self.expert_executor = None
        self.expert_prefetcher = None
        self.expert_predictor = None

    def _hand_bias(self):
        """Give the engine this layer's correction bias, once per (engine, tensor, version): a captured graph keeps reading
        the tensor the engine holds."""
        eng = _engine_of(self.expert_executor)
        b = self.e_score_correction_bias
        key = (id(eng), b.data_ptr(), b._version)
        if self._bias_handed != key:
            eng.set_gate_bias(self.layer_id, b)
            self._bias_handed = key

    def forward(self, hidden_states):
        orig_shape = hidden_states.shape
        x = hidden_states.view(-1, orig_shape[-1])
        logits = F.linear(x.type(torch.float32), self.gate_weight.type(torch.float32), None)   # modeling_deepseek.py:467-471
        if not _is_fast(self.expert_executor):
            raise RuntimeError("DeepseekMoEBlock needs the CUDA executor (expert_executor.moe_forward)")
        if self.v3:
            scores = logits.sigmoid()                                  # modeling_deepseek_v3/modeling_deepseek.py:475-476
            self._hand_bias()                                          # bias, groups, top-k, weights: in the engine
        else:
            scores = logits.softmax(dim=-1, dtype=torch.float32)                               # :473
        out = self.expert_executor.moe_forward(self.layer_id, x, scores=scores)   # top-k, experts, combine, shared experts
        return out.view(orig_shape)


class SyncSwitchTransformersSparseMLP(nn.Module):
    """moe_infinity/models/switch_transformers.py:41-113 (router: HF 4.x SwitchTransformersTop1Router)."""
    layer_id: int = None

    def __init__(self, config):
        super().__init__()
        self.num_experts = config.num_experts
        self.classifier = nn.Linear(config.d_model, config.num_experts, bias=getattr(config, "router_bias", False))
        self.expert_executor = None
        self.expert_prefetcher = None
        self.expert_predictor = None

    def forward(self, hidden_states):
        if not _is_fast(self.expert_executor):
            raise RuntimeError("SyncSwitchTransformersSparseMLP needs the CUDA executor")
        B, S, D = hidden_states.shape
        bias = self.classifier.bias                       # config.router_bias (HF 4.x Top1Router: self.classifier(hidden_states))
        router_logits = F.linear(hidden_states.to(torch.float32), self.classifier.weight.to(torch.float32),
                                 None if bias is None else bias.to(torch.float32))
        out = self.expert_executor.moe_forward(self.layer_id, hidden_states.reshape(-1, D), router_logits=router_logits,
                                               seq_len=S)
        eng = self.expert_executor.expert_dispatcher.engine if hasattr(self.expert_executor.expert_dispatcher, "engine") \
            else self.expert_executor.expert_dispatcher
        expert_index = eng.ws("topk_idx", B * S).reshape(B, S).clamp_min(0).long()   # dropped tokens: argmax of zeros = 0
        return out.view(B, S, D), (router_logits, expert_index)
