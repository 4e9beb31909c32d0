"""Test-side act-order GPTQ (desc_act=True, group size 128) checkpoints: random column orders and the g_idx GPTQ writes for
them, written from GPTQ's own definition of act-order groups and independent of moe_infinity_b200.int4.

GPTQ with desc_act quantises the columns of a layer in an order P (it sorts them by the Hessian's diagonal) and starts a new
group every 128 columns of that order, so g_idx[P[j]] = j // 128.  The checkpoint keeps the codes in natural column order;
scales and qzeros are indexed by group, and its own dequantisation is (q - z[:, g_idx]) * s[:, g_idx] in fp16."""
from __future__ import annotations

from typing import Dict, Tuple

import torch

import int4_checkpoint_packers as P


def random_g_idx(n_in: int, gen: torch.Generator) -> Tuple[torch.Tensor, torch.Tensor]:
    """-> (order P int64 [n_in], g_idx int32 [n_in]) with g_idx[P[j]] = j // 128."""
    order = torch.randperm(n_in, generator=gen)
    g_idx = torch.empty(n_in, dtype=torch.int32)
    g_idx[order] = (torch.arange(n_in) // 128).to(torch.int32)
    return order, g_idx


def fp16_dequant_g_idx(q: torch.Tensor, s: torch.Tensor, z: torch.Tensor, g_idx: torch.Tensor) -> torch.Tensor:
    """GPTQ's fp16 dequantisation of codes q [out, in] (natural order) with group-indexed s, z [out, in / 128]."""
    gi = g_idx.long()
    return (q.to(torch.int64) - z.to(torch.int64)[:, gi]).to(torch.float16) * s[:, gi]


def gptq_act_order_pack(q: torch.Tensor, s: torch.Tensor, z: torch.Tensor, g_idx: torch.Tensor, v1: bool = True):
    """-> (qweight, qzeros, scales, g_idx) as an act-order GPTQ checkpoint stores them (layouts of P.gptq_pack)."""
    qweight, qzeros, scales, _ = P.gptq_pack(q, s, z, v1=v1)
    return qweight, qzeros, scales, g_idx


def put_linear(tensors: Dict[str, torch.Tensor], truth: Dict[str, torch.Tensor], pre: str, out: int, n_in: int,
               gen: torch.Generator, g_idx: torch.Tensor, v1: bool = True, s_std: float = 0.002):
    """Write one act-order GPTQ linear layer under `pre` and record its fp16 dequantisation in natural order."""
    q, s, z = P.random_qsz(out, n_in, gen, z_lo=1 if v1 else 0, s_std=s_std)
    qw, qz, sc, gi = gptq_act_order_pack(q, s, z, g_idx, v1=v1)
    tensors.update({f"{pre}.qweight": qw, f"{pre}.qzeros": qz, f"{pre}.scales": sc, f"{pre}.g_idx": gi.clone()})
    truth[pre] = fp16_dequant_g_idx(q, s, z, g_idx)
