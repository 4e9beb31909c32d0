"""CPU/GPU oracle of the Llama 4 MoE block  --  TEST INFRASTRUCTURE ONLY.

Restates transformers 5.5's Llama4Router, Llama4TextExperts.forward and Llama4TextMoe.forward (modeling_llama4.py) per
token, with the dtypes of those call sites:

  router   logits = F.linear(x, W_router) in the model dtype; top-k BY THE LOGITS, ties to the lowest index;
           w = round(sigmoid(fp32(logit))) for each chosen expert (the others get sigmoid(-inf) = 0)
  inputs   the row of (t, e) is round(x[t] * w): the routing weight scales the expert's input, not its output
  experts  SwiGLU with every op rounded to the model dtype; y = the down projection
  combine  r = round(sum of round(y_e) over the chosen experts, in fp32, ascending id)   (routed_out...sum(dim=0))
           out = round(r + round(s)), s the shared expert (shared_expert(x).add_(r))
           NUMERICS_FP32: out = round(sum of y_e + s)

HF runs every expert on every token (the rows of unselected experts are x * 0 and add exact zeros), which the sparse form
here computes.  The functions run on whatever device their inputs are on, so the GPU tests replay the chain on the engine's
own tensors.  Pinned on the literal transformers block by tests/golden/make_golden_llama4.py.  The product package never
imports it.
"""
from __future__ import annotations

from typing import Optional, Sequence

import torch
import torch.nn.functional as F


def topk_lowest_index(v: torch.Tensor, k: int):
    """(values, indices) of the k largest entries per row; equal values go to the lowest index."""
    idx = torch.sort(-v.float(), dim=-1, stable=True).indices[..., :k]
    return v.gather(-1, idx), idx


def llama4_logits(x: torch.Tensor, router_w: torch.Tensor) -> torch.Tensor:
    """Router step 1: F.linear in the model dtype (what Llama4Router and the hf.py adapter compute)."""
    return F.linear(x, router_w)


def llama4_route(logits: torch.Tensor, k: int):
    """Router steps 2-3 from model-dtype logits [T,E] -> (topk_idx int64 [T,k] in descending-logit order, topk_w fp32
    [T,k]: the model-dtype rounding of the fp32 sigmoid of each chosen logit)."""
    v, idx = topk_lowest_index(logits, k)
    return idx, torch.sigmoid(v.float()).to(logits.dtype).float()


def scaled_inputs(x: torch.Tensor, topk_w: torch.Tensor) -> torch.Tensor:
    """[T,k,H]: round(x[t] * w[t,j]) in the model dtype (the product of two 16-bit values is exact in fp32)."""
    return (x.float().unsqueeze(1) * topk_w.float().unsqueeze(-1)).to(x.dtype)


def expert_outputs(x: torch.Tensor, topk_idx: torch.Tensor, topk_w: torch.Tensor, gate_up: torch.Tensor,
                   down: torch.Tensor) -> torch.Tensor:
    """y [T,k,H] in the model dtype, computed as Llama4TextExperts computes it: one torch.bmm per projection over the
    dense [E, T, H] input (row (e, t) = x[t] * score[t, e], zero for unselected experts), gate_up [E,H,2I], down [E,I,H]."""
    T, k = topk_idx.shape
    E = gate_up.shape[0]
    scores = torch.zeros(T, E, dtype=x.dtype, device=x.device)
    scores.scatter_(1, topk_idx.long(), topk_w.to(x.dtype))
    routed_in = x.repeat(E, 1) * scores.transpose(0, 1).reshape(-1, 1)
    h = routed_in.view(E, T, -1)
    g, u = torch.bmm(h, gate_up).chunk(2, dim=-1)
    y = torch.bmm(u * F.silu(g), down)                                          # [E, T, H]
    return y[topk_idx.long(), torch.arange(T, device=x.device).unsqueeze(1)]     # [T, k, H]


def shared_expert(x: torch.Tensor, gate_w: torch.Tensor, up_w: torch.Tensor, down_w: torch.Tensor) -> torch.Tensor:
    """Llama4TextMLP: down(silu(gate(x)) * up(x)) in the model dtype."""
    return F.linear(F.silu(F.linear(x, gate_w)) * F.linear(x, up_w), down_w)


def llama4_combine(y: torch.Tensor, topk_idx: torch.Tensor, dtype: torch.dtype, shared_out: torch.Tensor,
                   fp32: bool = False) -> torch.Tensor:
    """The combine chain.  y [T,k,H]: the expert output of (token, choice) j, fp32 or already in the model dtype;
    topk_idx [T,k] (choices with idx < 0 are skipped); shared_out [T,H] fp32 or model dtype.  Returns [T,H] in `dtype`."""
    T, k, H = y.shape
    order = torch.argsort(torch.where(topk_idx < 0, torch.iinfo(torch.int64).max, topk_idx.long()), dim=1, stable=True)
    rows = torch.arange(T, device=y.device)
    acc = torch.zeros(T, H, dtype=torch.float32, device=y.device)
    for j in range(k):
        sel = order[:, j]
        yj = y[rows, sel].float() if fp32 else y[rows, sel].to(dtype).float()
        ok = (topk_idx[rows, sel] >= 0).unsqueeze(-1)
        acc = torch.where(ok, acc + yj, acc)                                   # fp32 adds, ascending expert id
    if fp32:
        return (acc + shared_out.float()).to(dtype)
    return (acc.to(dtype).float() + shared_out.to(dtype).float()).to(dtype)   # r rounded once; + round(s), rounded


def llama4_block(x: torch.Tensor, router_w: torch.Tensor, gate_up: torch.Tensor, down: torch.Tensor, k: int,
                 shared: Sequence[torch.Tensor]):
    """The whole block on x [T,H] -> (out [T,H], logits, topk_idx, topk_w).  gate_up [E,H,2I] and down [E,I,H] in HF's
    Llama4TextExperts layout."""
    logits = llama4_logits(x, router_w)
    idx, w = llama4_route(logits, k)
    y = expert_outputs(x, idx, w, gate_up, down)
    return llama4_combine(y, idx, x.dtype, shared_expert(x, *shared)), logits, idx, w


def kth_ties(logits: torch.Tensor, k: int) -> torch.Tensor:
    """bool[T]: tokens whose k-th and (k+1)-th largest logits are equal (the choice depends on the tie rule)."""
    if logits.shape[-1] <= k:
        return torch.zeros(logits.shape[0], dtype=torch.bool, device=logits.device)
    s = logits.float().sort(dim=-1, descending=True).values
    return s[:, k - 1] == s[:, k]


def sigmoid_near_boundary(logits: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """bool, logits' shape: the fp32 sigmoid lies within one fp32 ulp of a `dtype` rounding boundary, so a sigmoid one ulp
    off (another exp implementation) could round to a different weight."""
    p = torch.sigmoid(logits.float())
    r = p.to(dtype)
    up = torch.nextafter(p, torch.full_like(p, float("inf"))).to(dtype)
    dn = torch.nextafter(p, torch.full_like(p, -float("inf"))).to(dtype)
    return (up != r) | (dn != r)
