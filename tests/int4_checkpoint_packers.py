"""Test-side packers for published 4-bit checkpoints, written from the layouts AWQ ("gemm" version) and GPTQ store, and the
fp16 dequantisation those libraries run.  They are independent of moe_infinity_b200.int4 so that the library's unpackers
(`from_awq`, `from_gptq`) are checked against a second statement of each layout.

All take codes q [out, in] (0..15, one per element, int64), fp16 scales s [out, in / 128] and zero points z [out, in / 128]."""
from __future__ import annotations

import os
from typing import Dict, List

import torch

AWQ_ORDER = [0, 2, 4, 6, 1, 3, 5, 7]   # nibble i of an AWQ word holds output row 8 j + AWQ_ORDER[i]


def _words(nib: torch.Tensor) -> torch.Tensor:
    """[..., 8] nibbles (nibble i at bits 4i..4i+3) -> int32 [...] words (two's complement)."""
    w = torch.zeros(nib.shape[:-1], dtype=torch.int64)
    for i in range(8):
        w |= (nib[..., i].to(torch.int64) & 15) << (4 * i)
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)


def awq_pack(q: torch.Tensor, s: torch.Tensor, z: torch.Tensor):
    """-> (qweight int32 [in, out / 8], qzeros int32 [in / 128, out / 8], scales fp16 [in / 128, out])."""
    out, n_in = q.shape
    qt = q.t().reshape(n_in, out // 8, 8)            # [c, j, p]: row 8 j + p
    zt = z.t().reshape(-1, out // 8, 8)
    qweight = _words(qt[..., AWQ_ORDER])             # nibble i <- row 8 j + AWQ_ORDER[i]
    qzeros = _words(zt[..., AWQ_ORDER])
    return qweight, qzeros, s.t().contiguous()


def gptq_pack(q: torch.Tensor, s: torch.Tensor, z: torch.Tensor, v1: bool = True):
    """-> (qweight int32 [in / 8, out], qzeros int32 [in / 128, out / 8], scales fp16 [in / 128, out], g_idx int32 [in]).
    v1 ("gptq") stores z - 1 (z must be >= 1), v2 stores z."""
    out, n_in = q.shape
    qweight = _words(q.t().reshape(n_in // 8, 8, out).permute(0, 2, 1))   # nibble i of [j, r] <- column 8 j + i
    zs = z.t().to(torch.int64) - (1 if v1 else 0)
    qzeros = _words(zs.reshape(-1, out // 8, 8))                            # nibble i of [g, j] <- row 8 j + i
    g_idx = (torch.arange(n_in) // 128).to(torch.int32)
    return qweight, qzeros, s.t().contiguous(), g_idx


def fp16_dequant(q: torch.Tensor, s: torch.Tensor, z: torch.Tensor) -> torch.Tensor:
    """What AWQ's and GPTQ's dequantisation computes: (q - z) in integers, then one fp16 multiply by the scale."""
    ze = z.to(torch.int64).repeat_interleave(128, 1)
    se = s.repeat_interleave(128, 1)
    return (q.to(torch.int64) - ze).to(torch.float16) * se


def random_qsz(out: int, n_in: int, gen: torch.Generator, z_lo: int = 0, s_std: float = 0.002):
    q = torch.randint(0, 16, (out, n_in), generator=gen)
    z = torch.randint(z_lo, 16, (out, n_in // 128), generator=gen)
    s = (torch.randn(out, n_in // 128, generator=gen) * s_std).to(torch.float16)
    return q, s, z


def write_shards(tmp_dir: str, tensors: Dict[str, torch.Tensor], nshards: int = 2) -> List[str]:
    """Save `tensors` into `nshards` safetensors files, keys dealt round-robin."""
    from safetensors.torch import save_file
    keys = sorted(tensors)
    paths = []
    for i in range(nshards):
        part = {k: tensors[k].contiguous() for k in keys[i::nshards]}
        path = os.path.join(tmp_dir, f"model-{i + 1:05d}-of-{nshards:05d}.safetensors")
        save_file(part, path)
        paths.append(path)
    return paths
