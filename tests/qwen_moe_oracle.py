"""CPU/GPU oracle of the Qwen2-MoE / Qwen3-MoE sparse block  --  TEST INFRASTRUCTURE ONLY.

Restates transformers 5.5's Qwen2MoeTopKRouter / Qwen3MoeTopKRouter (identical), Qwen2MoeExperts.forward and
Qwen2MoeSparseMoeBlock.forward (modeling_qwen2_moe.py; the Qwen3 block is the same without the shared expert) per token, with
the dtypes of those call sites:

  router   logits = F.linear(x, W_gate) in the model dtype; p = softmax(logits, fp32); top-k with ties to the lowest index;
           norm_topk_prob: w /= (sum of the k weights in selection order), for every k, no epsilon; w stays fp32
  combine  acc = 0 (model dtype); for each chosen expert in ascending id (index_add_ order):
               acc = round(acc + round(round(y) * w))
  shared   (Qwen2) g = round(sigmoid(round(x . w_sg)));  out = round(acc + round(g * round(s)))

The functions run on whatever device their inputs are on, so the GPU tests replay the chain on the engine's own tensors.
Pinned on the literal transformers blocks by tests/golden/make_golden_qwen_moe.py.  The product package never imports it.
"""
from __future__ import annotations

from typing import Optional, Sequence

import torch
import torch.nn.functional as F


def topk_lowest_index(v: torch.Tensor, k: int):
    """(values, indices) of the k largest entries per row; equal values go to the lowest index."""
    idx = torch.sort(-v, dim=-1, stable=True).indices[..., :k]     # stable: equal values keep ascending index order
    return v.gather(-1, idx), idx


def qwen_route(logits: torch.Tensor, k: int, norm_topk_prob: bool):
    """Router steps 2-5 from model-dtype (or any-dtype) logits [T,E] -> (topk_idx int64 [T,k], topk_w fp32 [T,k]).
    Experts come out in selection (descending probability) order; the normalising sum runs in that order."""
    return qwen_route_from_probs(torch.softmax(logits.float(), dim=-1), k, norm_topk_prob)


def qwen_route_from_probs(p: torch.Tensor, k: int, norm_topk_prob: bool):
    """Router steps 3-5 from fp32 probabilities [T,E] (e.g. the engine's own B2M_WS_SCORES)."""
    w, idx = topk_lowest_index(p, k)
    if norm_topk_prob:
        denom = w[:, 0].clone()
        for j in range(1, k):
            denom = denom + w[:, j]
        w = w / denom.unsqueeze(-1)
    return idx, w


def qwen_logits(x: torch.Tensor, gate_w: torch.Tensor) -> torch.Tensor:
    """Router step 1: F.linear in the model dtype (what HF and the hf.py adapter compute)."""
    return F.linear(x, gate_w)


def shared_gate_values(x: torch.Tensor, sg_w: torch.Tensor) -> torch.Tensor:
    """[T] sigmoid(shared_expert_gate(x)) in the model dtype."""
    return torch.sigmoid(F.linear(x, sg_w.reshape(1, -1))).reshape(-1)


def qwen_combine(y: torch.Tensor, topk_idx: torch.Tensor, topk_w: torch.Tensor, dtype: torch.dtype,
                 shared_out: Optional[torch.Tensor] = None, gate: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The combine chain.  y [T,k,H]: the expert output of (token, choice) j, fp32 or already in the model dtype (rounded
    here either way); topk_idx / topk_w [T,k]; shared_out [T,H] (fp32 or model dtype) and gate [T] (model dtype) for a
    Qwen2 layer.  Choices with idx < 0 are skipped.  Returns [T,H] in `dtype`."""
    T, k, H = y.shape
    order = torch.argsort(torch.where(topk_idx < 0, torch.iinfo(torch.int64).max, topk_idx.long()), dim=1, stable=True)
    acc = torch.zeros(T, H, dtype=dtype, device=y.device)
    for j in range(k):
        sel = order[:, j]
        rows = torch.arange(T, device=y.device)
        yj = y[rows, sel].to(dtype)
        wj = topk_w[rows, sel].float()
        ok = (topk_idx[rows, sel] >= 0).unsqueeze(-1)
        prod = (yj * wj.unsqueeze(-1)).to(dtype)             # bf16 * fp32 -> fp32, then .to(model dtype)
        acc = torch.where(ok, acc + prod, acc)                # index_add_: model-dtype add, rounded
    if shared_out is not None:
        sh = gate.to(dtype).unsqueeze(-1) * shared_out.to(dtype)
        acc = acc + sh
    return acc


def expert_outputs(x: torch.Tensor, topk_idx: torch.Tensor, gate_up: torch.Tensor, down: torch.Tensor) -> torch.Tensor:
    """y [T,k,H] in the model dtype, computed as Qwen2MoeExperts.forward computes each expert's rows: the expert's tokens in
    torch.where(expert_mask[e]) order (choice position first), gate/up from one F.linear, silu(gate) * up, F.linear down."""
    T, k = topk_idx.shape
    H = x.shape[-1]
    y = torch.zeros(T, k, H, dtype=x.dtype, device=x.device)
    E = gate_up.shape[0]
    mask = F.one_hot(topk_idx.long(), num_classes=E).permute(2, 1, 0)     # [E, k, T]
    for e in range(E):
        pos, tok = torch.where(mask[e])
        if tok.numel() == 0:
            continue
        g, u = F.linear(x[tok], gate_up[e]).chunk(2, dim=-1)
        y[tok, pos] = F.linear(F.silu(g) * u, down[e])
    return y


def shared_expert(x: torch.Tensor, gate_w: torch.Tensor, up_w: torch.Tensor, down_w: torch.Tensor) -> torch.Tensor:
    """Qwen2MoeMLP: down(silu(gate(x)) * up(x)) in the model dtype."""
    return F.linear(F.silu(F.linear(x, gate_w)) * F.linear(x, up_w), down_w)


def qwen_block(x: torch.Tensor, gate_w: torch.Tensor, gate_up: torch.Tensor, down: torch.Tensor, k: int,
               norm_topk_prob: bool, shared: Optional[Sequence[torch.Tensor]] = None,
               shared_gate_w: Optional[torch.Tensor] = None):
    """The whole block on x [T,H] -> (out [T,H], logits, topk_idx, topk_w)."""
    logits = qwen_logits(x, gate_w)
    idx, w = qwen_route(logits, k, norm_topk_prob)
    y = expert_outputs(x, idx, gate_up, down)
    s = g = None
    if shared is not None:
        s = shared_expert(x, *shared)
        g = shared_gate_values(x, shared_gate_w)
    return qwen_combine(y, idx, w, x.dtype, s, g), logits, idx, w


def topk_ties(logits: torch.Tensor, k: int) -> torch.Tensor:
    """bool[T]: tokens whose k-th and (k+1)-th probabilities are equal (the choice depends on the tie rule)."""
    p = torch.softmax(logits.float(), dim=-1)
    if p.shape[-1] <= k:
        return torch.zeros(p.shape[0], dtype=torch.bool, device=p.device)
    s = p.sort(dim=-1, descending=True).values
    return s[:, k - 1] == s[:, k]
