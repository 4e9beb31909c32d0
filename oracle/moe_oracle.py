"""CPU oracle for the MoE dispatch hot path  --  TEST INFRASTRUCTURE ONLY.

This module restates, operator for operator, what the reference computes on the path
router-softmax/top-k -> mask build -> per-expert gather -> expert FFN -> weighted
combine.  It exists so that tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference leg can CHECK (or time) the CUDA path; the product
package never imports it and fails loudly when its CUDA extension is missing.

Where the arithmetic lives: the reference performs all math through libtorch/ATen
(third-party, pinned only as `torch>=2.1.1` in /root/reference/requirements.txt:18).
The same library is importable here, so this restatement calls the *same operators*
in the same order and dtypes as the reference call sites cited below.

Parity status: the reference ships no golden vectors, KATs or fixtures for this path (SURVEY.md §4, §8c), so the
pin is made from outputs of the reference itself run in the dev container:
  (a) expert FFN (D1-D3): the reference's OWN core/parallel/expert_module.cpp is compiled as-is into
      oracle/_ref/ref_expert_module.so (oracle/ref_build/Makefile); tests/test_oracle_expert_ref.py demands bit equality
      of `expert_ffn` with it for all six expert types x three dtypes, live and through tests/golden/expert_ffn_ref.pt;
  (b) routing / mask build / combine (A1-A6, G1-G2): the literal reference block files (mixtral.py, deepseek.py, MoEGate,
      switch_transformers.py) are executed on CPU through tests/shims/ref_loader.py -- from /root/reference, or from their
      byte-compiled staging oracle/_ref/pyref where that tree does not exist; tests/test_oracle_golden.py demands bit equality
      with this module and tests/golden/*.pt hold their outputs (tests/golden/make_golden.py).  The Switch block runs on a
      4.x-order router shim (HF 5.5's router returns another tuple), which restates the transformers 4.x forward;
  (c) cache policy: oracle/policy_oracle.py is pinned on a trace recorded from the reference's real engine
      (tests/golden/policy_ref_trace.json, tools/ref_engine_harness.py --mode policy).

Determinism choices (the reference itself is nondeterministic, SURVEY §9 Q1):
  * experts are combined in ascending expert id (reference: thread completion order,
    core/parallel/expert_dispatcher.cpp:419-450);
  * top-k ties break towards the lowest expert index (torch.topk leaves it unspecified);
    `tied_tokens()` reports tokens whose k-th and (k+1)-th scores are equal so a test can
    assert exact indices everywhere else and set-equality there.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

# expert-type ints: /root/reference/core/parallel/expert_module.h:13-18
SWITCH_DENSE_ACT_DENSE = 0
SWITCH_DENSE_GATED_ACT_DENSE = 1
NLLB_MOE_DENSE_ACT_DENSE = 2
FSGPT_MOE_DENSE_ACT_DENSE = 3
MIXTRAL_MOE_DENSE_ACT_DENSE = 4
DEEPSEEK_MOE_DENSE_ACT_DENSE = 5
# dtype ints: expert_module.h:20-23
DTYPE_BF16, DTYPE_F32, DTYPE_F16, DTYPE_FP8 = 0, 1, 2, 3
DTYPE_TO_TORCH = {DTYPE_BF16: torch.bfloat16, DTYPE_F32: torch.float32, DTYPE_F16: torch.float16}


# --------------------------------------------------------------------------------------
# top-k with a defined tie-break
# --------------------------------------------------------------------------------------
def topk_lowest_index(scores: torch.Tensor, k: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """torch.topk(scores, k, dim=-1) (values sorted descending) with ties broken towards
    the lowest index.  Used wherever the reference calls torch.topk
    (moe_infinity/models/mixtral.py:49-51, modeling_deepseek.py:481-483)."""
    order = torch.sort(scores, dim=-1, descending=True, stable=True).indices[..., :k]
    return torch.gather(scores, -1, order), order


def tied_tokens(scores: torch.Tensor, k: int) -> torch.Tensor:
    """bool[T]: tokens whose top-k membership is ambiguous (k-th == (k+1)-th score)."""
    if scores.shape[-1] <= k:
        return torch.zeros(scores.shape[0], dtype=torch.bool)
    s = torch.sort(scores, dim=-1, descending=True, stable=True).values
    return s[:, k - 1] == s[:, k]


# --------------------------------------------------------------------------------------
# A2/A3: Mixtral routing  (moe_infinity/models/mixtral.py:44-65)
# --------------------------------------------------------------------------------------
@dataclass
class Routing:
    topk_idx: torch.Tensor            # int64 [T,k]  (descending score for Mixtral; any order for DeepSeek)
    topk_weight: torch.Tensor         # [T,k]  dtype of the combine multiplier (bf16 Mixtral, fp32 DeepSeek)
    router_mask: torch.Tensor         # [T,E]  bool (Mixtral) / int64 0-1 (DeepSeek)
    routing_weights_mask: torch.Tensor  # [T,E]
    scores: torch.Tensor              # fp32 [T,E] softmax probabilities


def mixtral_route(router_logits: torch.Tensor, top_k: int, out_dtype: torch.dtype) -> Routing:
    """mixtral.py:48-65.  router_logits [T,E] in the gate's dtype; out_dtype = hidden dtype."""
    E = router_logits.shape[-1]
    scores = F.softmax(router_logits, dim=1, dtype=torch.float)            # :48
    routing_weights, selected_experts = topk_lowest_index(scores, top_k)    # :49-51
    routing_weights = routing_weights / routing_weights.sum(dim=-1, keepdim=True)  # :52
    routing_weights = routing_weights.to(out_dtype)                         # :54
    router_mask = F.one_hot(selected_experts, num_classes=E)                # :56  int64 [T,k,E]
    routing_weights_mask = (routing_weights[:, :, None] * router_mask).permute(0, 2, 1)  # :57-59
    router_mask = router_mask.permute(0, 2, 1)                              # :60
    rm = router_mask[:, :, 0].bool()
    for j in range(1, top_k):                                               # :62-64 ("assume top-2")
        rm = torch.logical_or(rm, router_mask[:, :, j])
    routing_weights_mask = torch.sum(routing_weights_mask, dim=-1)          # :65
    return Routing(selected_experts, routing_weights, rm, routing_weights_mask, scores)


# --------------------------------------------------------------------------------------
# A4/A5: DeepSeek-V2 gate  (modeling_deepseek/modeling_deepseek.py:463-512, models/deepseek.py:76-91)
# --------------------------------------------------------------------------------------
def deepseek_gate_scores(hidden: torch.Tensor, gate_weight: torch.Tensor) -> torch.Tensor:
    """modeling_deepseek.py:467-474: fp32 linear + fp32 softmax."""
    logits = F.linear(hidden.type(torch.float32), gate_weight.type(torch.float32), None)
    return logits.softmax(dim=-1, dtype=torch.float32)


def deepseek_route(scores: torch.Tensor, top_k: int, *, topk_method: str = "greedy",
                   n_group: int = 1, topk_group: int = 1, norm_topk_prob: bool = False,
                   routed_scaling_factor: float = 1.0) -> Routing:
    T, E = scores.shape
    if topk_method == "greedy":                                             # :480-483
        topk_weight, topk_idx = topk_lowest_index(scores, top_k)
    elif topk_method == "group_limited_greedy":                             # :484-505
        group_scores = scores.view(T, n_group, -1).max(dim=-1).values
        group_idx = topk_lowest_index(group_scores, topk_group)[1]
        group_mask = torch.zeros_like(group_scores)
        group_mask.scatter_(1, group_idx, 1)
        score_mask = group_mask.unsqueeze(-1).expand(T, n_group, E // n_group).reshape(T, -1)
        tmp_scores = scores.masked_fill(~score_mask.bool(), 0.0)
        topk_weight, topk_idx = topk_lowest_index(tmp_scores, top_k)
    else:
        raise NotImplementedError(topk_method)
    if top_k > 1 and norm_topk_prob:                                        # :508-510
        topk_weight = topk_weight / (topk_weight.sum(dim=-1, keepdim=True) + 1e-20)
    else:
        topk_weight = topk_weight * routed_scaling_factor                   # :512
    # models/deepseek.py:77-91
    router_mask = F.one_hot(topk_idx, num_classes=E)
    routing_weights_mask = (topk_weight[:, :, None] * router_mask).permute(0, 2, 1)
    routing_weights_mask = torch.sum(routing_weights_mask, dim=-1)
    router_mask = router_mask.permute(0, 2, 1).contiguous()
    for i in range(top_k):
        router_mask[:, :, 0] = torch.logical_or(router_mask[:, :, 0], router_mask[:, :, i])
    router_mask = router_mask[:, :, 0]
    return Routing(topk_idx, topk_weight, router_mask, routing_weights_mask, scores)


# --------------------------------------------------------------------------------------
# A6: Switch top-1 router with capacity  (HF transformers 4.x SwitchTransformersTop1Router,
# third-party, pinned `transformers>=4.37.1` in requirements.txt:19; called at
# moe_infinity/models/switch_transformers.py:76)
# --------------------------------------------------------------------------------------
def switch_route(hidden: torch.Tensor, classifier_weight: torch.Tensor, expert_capacity: int,
                 router_dtype: torch.dtype = torch.float32):
    """hidden [B,S,D].  Returns (router_mask int64 [B,S,E], router_probs [B,S,1], router_logits)."""
    input_dtype = hidden.dtype
    h = hidden.to(router_dtype)
    router_logits = F.linear(h, classifier_weight.to(router_dtype))
    router_probs = F.softmax(router_logits, dim=-1, dtype=router_dtype).to(input_dtype)
    expert_index = torch.argmax(router_probs, dim=-1)
    expert_index = F.one_hot(expert_index, num_classes=classifier_weight.shape[0])
    token_priority = torch.cumsum(expert_index, dim=-2)
    expert_capacity_mask = token_priority <= expert_capacity
    expert_index = expert_index * expert_capacity_mask
    router_probs = torch.max(router_probs, dim=-1).values.unsqueeze(-1)
    return expert_index, router_probs, router_logits


# --------------------------------------------------------------------------------------
# D1-D3: expert FFNs  (core/parallel/expert_module.cpp)
# --------------------------------------------------------------------------------------
def expert_ffn(x: torch.Tensor, weights: Sequence[torch.Tensor], expert_type: int) -> torch.Tensor:
    """weights in the reference's `tensor_ids` order (named_parameters order of the HF module)."""
    if expert_type in (MIXTRAL_MOE_DENSE_ACT_DENSE,):
        w1, w2, w3 = weights                                    # expert_module.cpp:139-145
        return torch.matmul(F.silu(torch.matmul(x, w1.transpose(0, 1))) *
                            torch.matmul(x, w3.transpose(0, 1)), w2.transpose(0, 1))  # :171-175
    if expert_type == DEEPSEEK_MOE_DENSE_ACT_DENSE:
        gate, up, down = weights                                # :185-191
        return torch.matmul(F.silu(torch.matmul(x, gate.transpose(0, 1))) *
                            torch.matmul(x, up.transpose(0, 1)), down.transpose(0, 1))  # :200-203
    if expert_type == SWITCH_DENSE_ACT_DENSE:
        wi, wo = weights                                        # :17-23
        return torch.matmul(torch.relu(torch.matmul(x, wi.transpose(0, 1).to(x.dtype))),
                            wo.transpose(0, 1).to(x.dtype))     # :31-35
    if expert_type == SWITCH_DENSE_GATED_ACT_DENSE:
        wi_0, wi_1, wo = weights                                # :45-52
        g = F.gelu(torch.matmul(x, wi_0.transpose(0, 1)))
        return torch.matmul(torch.mul(g, torch.matmul(x, wi_1.transpose(0, 1))), wo.transpose(0, 1))  # :54-59
    if expert_type in (NLLB_MOE_DENSE_ACT_DENSE, FSGPT_MOE_DENSE_ACT_DENSE):
        fc1, fc1_bias, fc2, fc2_bias = weights                  # :70-77, :104-111
        if expert_type == FSGPT_MOE_DENSE_ACT_DENSE and x.dtype != fc1.dtype:
            x = x.to(fc1.dtype)                                 # :122-123 (only the FSGPT module casts)
        return torch.matmul(torch.relu(torch.matmul(x, fc1.transpose(0, 1)) + fc1_bias),
                            fc2.transpose(0, 1)) + fc2_bias     # :88-92, :124-128
    raise ValueError(f"unknown expert type {expert_type}")


# --------------------------------------------------------------------------------------
# B1-F1: dispatch_local stand-in  (distributed/expert_executor.py:32-58 +
# core/parallel/expert_dispatcher.cpp:274-285 gather, :397-434 output)
# --------------------------------------------------------------------------------------
def dispatch_local(hidden: torch.Tensor, router_mask: torch.Tensor,
                   experts: Sequence[Sequence[torch.Tensor]], expert_type: int,
                   layer_id: int = 0) -> List[Tuple[torch.Tensor, int, int, int]]:
    """Returns [(out[n_e,H], layer, expert, hit)] for experts with >=1 token, ascending expert id.
    Rows of each result are in ascending token order (boolean-mask gather order)."""
    E = router_mask.shape[-1]
    mask2d = router_mask.reshape(-1, E)
    x2d = hidden.reshape(-1, hidden.shape[-1])
    expert_count = torch.sum(mask2d, dim=0)                      # expert_executor.py:34-39
    results = []
    for e in range(E):
        if int(expert_count[e]) <= 0:                            # :41-44
            continue
        token_indices = mask2d[:, e].to(torch.bool)              # expert_dispatcher.cpp:274-275
        xin = x2d[token_indices]                                 # :283-285
        out = expert_ffn(xin, experts[e], expert_type)           # :341-372
        results.append((out.to(hidden.dtype), layer_id, e, 1))   # :403-405, :420-422
    return results


# --------------------------------------------------------------------------------------
# G1/G2: blocks
# --------------------------------------------------------------------------------------
def mixtral_block(hidden: torch.Tensor, gate_weight: Optional[torch.Tensor],
                  experts: Sequence[Sequence[torch.Tensor]], top_k: int,
                  router_logits: Optional[torch.Tensor] = None):
    """SyncMixtralSparseMoeBlock.forward, mixtral.py:40-118.  hidden [B,S,H].
    Returns (final[B,S,H], router_logits[T,E], Routing)."""
    B, S, H = hidden.shape
    x = hidden.view(-1, H)
    if router_logits is None:
        router_logits = F.linear(x, gate_weight)                 # :46
    r = mixtral_route(router_logits, top_k, x.dtype)
    final = torch.zeros((B * S, H), dtype=x.dtype)               # :87-91
    results = dispatch_local(x, r.router_mask, experts, MIXTRAL_MOE_DENSE_ACT_DENSE)  # :93-95
    for output, _, idx, _ in results:                            # :96-101
        token_indices = r.router_mask[:, idx].bool()
        final[token_indices, :] += output * r.routing_weights_mask[token_indices, idx][:, None]
    return final.reshape(B, S, H), router_logits, r


def deepseek_block(hidden: torch.Tensor, gate_weight: torch.Tensor,
                   experts: Sequence[Sequence[torch.Tensor]], top_k: int,
                   shared: Optional[Sequence[torch.Tensor]] = None, *, scores: Optional[torch.Tensor] = None,
                   topk_method: str = "greedy", n_group: int = 1, topk_group: int = 1,
                   norm_topk_prob: bool = False, routed_scaling_factor: float = 1.0):
    """DeepseekMoEBlock.forward, models/deepseek.py:51-137."""
    B, S, H = hidden.shape
    x = hidden.view(-1, H)
    if scores is None:
        scores = deepseek_gate_scores(x, gate_weight)
    r = deepseek_route(scores, top_k, topk_method=topk_method, n_group=n_group, topk_group=topk_group,
                       norm_topk_prob=norm_topk_prob, routed_scaling_factor=routed_scaling_factor)
    final = torch.zeros((B * S, H), dtype=x.dtype)               # :115-119
    results = dispatch_local(x, r.router_mask, experts, DEEPSEEK_MOE_DENSE_ACT_DENSE)
    for output, _, idx, _ in results:                            # :123-128
        token_indices = r.router_mask[:, idx].bool()
        final[token_indices, :] += output * r.routing_weights_mask[token_indices, idx][:, None]
    final = final.view(B, S, H)
    if shared is not None:                                       # :133-136
        final = final + expert_ffn(hidden, shared, DEEPSEEK_MOE_DENSE_ACT_DENSE)
    return final, r


def switch_block(hidden: torch.Tensor, classifier_weight: torch.Tensor,
                 experts: Sequence[Sequence[torch.Tensor]], expert_capacity: int):
    """SyncSwitchTransformersSparseMLP.forward, switch_transformers.py:74-113. hidden [B,S,D]."""
    router_mask, router_probs, router_logits = switch_route(hidden, classifier_weight, expert_capacity)
    expert_index = torch.argmax(router_mask, dim=-1)             # :77
    next_states = hidden.clone()                                 # :81
    results = dispatch_local(hidden, router_mask, experts, SWITCH_DENSE_ACT_DENSE)
    for output, _, idx, _ in results:                            # :99-101
        token_indices = router_mask[:, :, idx].bool()
        next_states[token_indices] = output
    return router_probs * next_states, (router_logits, expert_index), router_mask  # :109-113


# --------------------------------------------------------------------------------------
# fp32 twin: same routing decisions, FFN + combine in fp32 (the error yardstick)
# --------------------------------------------------------------------------------------
def combine_fp32(hidden: torch.Tensor, experts: Sequence[Sequence[torch.Tensor]],
                 topk_idx: torch.Tensor, topk_weight: torch.Tensor, expert_type: int,
                 shared: Optional[Sequence[torch.Tensor]] = None) -> torch.Tensor:
    """y[t] = sum_j w[t,j] * FFN_{idx[t,j]}(x[t]) in fp32 with the (already rounded) routing weights."""
    x = hidden.reshape(-1, hidden.shape[-1]).float()
    E = len(experts)
    out = torch.zeros_like(x)
    for e in range(E):
        sel = (topk_idx == e)
        tok = sel.any(dim=-1)
        if not bool(tok.any()):
            continue
        w = (topk_weight.float() * sel).sum(dim=-1)[tok]
        y = expert_ffn(x[tok], [t.float() for t in experts[e]], expert_type)
        out[tok] += y * w[:, None]
    if shared is not None:
        out += expert_ffn(x, [t.float() for t in shared], expert_type)
    return out.reshape(hidden.shape)


# --------------------------------------------------------------------------------------
# synthetic model pieces (SURVEY §8d "Synthetic inputs")
# --------------------------------------------------------------------------------------
def make_experts(E: int, H: int, I: int, dtype: torch.dtype, seed: int, expert_type: int = MIXTRAL_MOE_DENSE_ACT_DENSE,
                 std: float = 0.02) -> List[List[torch.Tensor]]:
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(E):
        if expert_type in (MIXTRAL_MOE_DENSE_ACT_DENSE,):
            shapes = [(I, H), (H, I), (I, H)]          # w1, w2, w3
        elif expert_type == DEEPSEEK_MOE_DENSE_ACT_DENSE:
            shapes = [(I, H), (I, H), (H, I)]          # gate, up, down
        elif expert_type == SWITCH_DENSE_ACT_DENSE:
            shapes = [(I, H), (H, I)]                  # wi, wo
        elif expert_type in (NLLB_MOE_DENSE_ACT_DENSE, FSGPT_MOE_DENSE_ACT_DENSE):
            shapes = [(I, H), (I,), (H, I), (H,)]      # fc1, fc1_bias, fc2, fc2_bias (named_parameters order)
        else:
            raise ValueError(expert_type)
        out.append([(torch.randn(s, generator=g) * std).to(dtype) for s in shapes])
    return out
