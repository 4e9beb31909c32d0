"""CPU oracle of the DeepSeek-V3 gate and block  --  TEST INFRASTRUCTURE ONLY.

Restates MoEGate with topk_method "noaux_tc" and scoring_func "sigmoid" (models/modeling_deepseek_v3/modeling_deepseek.py:
466-527) and the DeepseekMoEBlock built around it (models/deepseek.py:23-27, 51-137) with the operators and dtypes of those
call sites, on top of oracle/moe_oracle.py's building blocks (lowest-index top-k, dispatch_local stand-in, expert FFN).
Pinned on the literal reference block through tests/golden/deepseek_v3_*.pt (tests/golden/make_golden_deepseek_v3.py).
The product package never imports it.
"""
from __future__ import annotations

from typing import Optional, Sequence

import torch
import torch.nn.functional as F

from oracle import moe_oracle as O


def _masks(topk_idx: torch.Tensor, topk_weight: torch.Tensor, E: int, top_k: int):
    """models/deepseek.py:77-91: one-hot mask merged over the k choices + per-expert combining weights."""
    router_mask = F.one_hot(topk_idx, num_classes=E)
    routing_weights_mask = (topk_weight[:, :, None] * router_mask).permute(0, 2, 1)
    routing_weights_mask = torch.sum(routing_weights_mask, dim=-1)
    router_mask = router_mask.permute(0, 2, 1).contiguous()
    for i in range(top_k):
        router_mask[:, :, 0] = torch.logical_or(router_mask[:, :, 0], router_mask[:, :, i])
    return router_mask[:, :, 0], routing_weights_mask


def _kept_choices(choice: torch.Tensor, n_group: int, topk_group: int):
    """Steps 3-4: group score = top1 + top2 of the group's choices, the topk_group best groups kept, the other choices
    set to 0.0 (masked_fill, not -inf).  Returns (group scores, masked choices)."""
    T, E = choice.shape
    group_scores = O.topk_lowest_index(choice.view(T, n_group, -1), 2)[0].sum(dim=-1)            # :488-492
    group_idx = O.topk_lowest_index(group_scores, topk_group)[1]                                 # :493-495
    group_mask = torch.zeros_like(group_scores)
    group_mask.scatter_(1, group_idx, 1)
    score_mask = group_mask.unsqueeze(-1).expand(T, n_group, E // n_group).reshape(T, -1)
    return group_scores, choice.masked_fill(~score_mask.bool(), 0.0)                             # :507-509


def deepseek_v3_route(logits_or_scores: torch.Tensor, bias: torch.Tensor, k: int, n_group: int, topk_group: int,
                      norm_topk_prob: bool, routed_scaling_factor: float, *, are_scores: bool = False) -> O.Routing:
    """The six steps of the V3 gate with ties broken towards the lowest index.  `logits_or_scores` [T,E]: fp32 router
    logits (sigmoid applied here, :475-476) or, with are_scores=True, the sigmoid scores themselves.  Experts come out in
    descending choice order; the normalising sum runs in that order (the reference sums in torch.topk(sorted=False)
    order)."""
    T, E = logits_or_scores.shape
    scores = logits_or_scores.float() if are_scores else logits_or_scores.float().sigmoid()       # 1
    choice = scores + bias.float().unsqueeze(0)                                                  # 2  (:485-487)
    _, tmp = _kept_choices(choice, n_group, topk_group)                                          # 3, 4
    topk_idx = O.topk_lowest_index(tmp, k)[1]                                                    # 5  (:510-513)
    topk_weight = scores.gather(1, topk_idx)
    if k > 1 and norm_topk_prob:                                                                 # 6  (:520-526)
        denom = topk_weight[:, 0].clone()
        for j in range(1, k):                                                                    # selection order
            denom = denom + topk_weight[:, j]
        topk_weight = topk_weight / (denom.unsqueeze(-1) + 1e-20)
    topk_weight = topk_weight * routed_scaling_factor
    router_mask, routing_weights_mask = _masks(topk_idx, topk_weight, E, k)
    return O.Routing(topk_idx, topk_weight, router_mask, routing_weights_mask, scores)


def deepseek_v3_choice_ties(scores: torch.Tensor, bias: torch.Tensor, k: int, n_group: int, topk_group: int,
                            rel: float = 0.0) -> torch.Tensor:
    """bool[T]: tokens whose V3 selection is ambiguous -- the topk_group-th and next group scores, or the k-th and next
    masked choices, are equal (rel = 0) or closer than rel times their magnitude."""
    T, E = scores.shape
    gs, tmp = _kept_choices(scores.float() + bias.float().unsqueeze(0), n_group, topk_group)
    near = torch.zeros(T, dtype=torch.bool)
    if n_group > topk_group:
        s = gs.sort(dim=-1, descending=True).values
        near |= (s[:, topk_group - 1] - s[:, topk_group]).abs() <= rel * s[:, topk_group - 1].abs()
    if E > k:
        s = tmp.sort(dim=-1, descending=True).values
        near |= (s[:, k - 1] - s[:, k]).abs() <= rel * s[:, k - 1].abs()
    return near


def deepseek_v3_block(hidden: torch.Tensor, gate_weight: torch.Tensor, bias: torch.Tensor,
                      experts: Sequence[Sequence[torch.Tensor]], top_k: int,
                      shared: Optional[Sequence[torch.Tensor]] = None, *, scores: Optional[torch.Tensor] = None,
                      n_group: int = 1, topk_group: int = 1, norm_topk_prob: bool = True,
                      routed_scaling_factor: float = 1.0):
    """DeepseekMoEBlock.forward (models/deepseek.py:51-137) with the V3 gate; `scores` = sigmoid scores if given."""
    B, S, H = hidden.shape
    x = hidden.view(-1, H)
    if scores is None:
        scores = F.linear(x.type(torch.float32), gate_weight.type(torch.float32), None).sigmoid()
    r = deepseek_v3_route(scores, bias, top_k, n_group, topk_group, norm_topk_prob, routed_scaling_factor,
                          are_scores=True)
    final = torch.zeros((B * S, H), dtype=x.dtype)                                               # :115-119
    results = O.dispatch_local(x, r.router_mask, experts, O.DEEPSEEK_MOE_DENSE_ACT_DENSE)
    for output, _, idx, _ in results:                                                           # :123-128
        token_indices = r.router_mask[:, idx].bool()
        final[token_indices, :] += output * r.routing_weights_mask[token_indices, idx][:, None]
    final = final.view(B, S, H)
    if shared is not None:                                                                      # :133-136
        final = final + O.expert_ffn(hidden, shared, O.DEEPSEEK_MOE_DENSE_ACT_DENSE)
    return final, r
