"""4-bit integer expert weights with a bf16 scale and a 4-bit zero point per 128 inputs (W4A16 group quantisation).

`MoEEngine(..., expert_dtype=torch.uint4)` runs such experts; the numbers it computes are defined by `dequantize_g128`: the
bf16 engine on W = bf16(s[r][c // 128] * (q[r][c] - z[r][c // 128])), the exact product rounded once (include/b2m.h,
B2M_WEIGHTS_INT4_G128).  `quantize_g128` turns a bf16 / fp32 checkpoint into that format; `pack_groups` builds the
tile-major group grid an expert blob stores after its code matrices."""
from __future__ import annotations

from typing import Tuple

import torch

GROUP = 128
TILE_ROWS = 128   # rows of one GEMM tile: the group grid keeps a tile's 128 words of one group together


def _groups(rows: int, cols: int) -> int:
    if rows % TILE_ROWS or cols % GROUP:
        raise ValueError(f"a [{rows}, {cols}] matrix does not divide into {TILE_ROWS}-row tiles and {GROUP}-input groups")
    return cols // GROUP


def quantize_g128(w: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """w [out, in] (any float dtype) -> (q uint8 [out, in / 2], s bfloat16 [out, in / 128], z uint8 [out, in / 128]).

    Asymmetric min/max round-to-nearest per group of 128 inputs of a row: s = bf16((max - min) / 15), rounded to bf16
    BEFORE the codes are computed; z = clamp(round(-min / s), 0, 15); code = clamp(round(w / s) + z, 0, 15).  A group
    whose scale rounds to zero (every all-equal group among them) gets s = bf16(max), z = 0 and every code 1, so it holds
    bf16(max) exactly -- or s = 1, z = 0, codes 0 when bf16(max) is zero (an all-zero group).
    q packs two codes per byte: column c in the low nibble of byte c // 2 when c is even, in the high nibble when odd."""
    if w.dim() != 2:
        raise ValueError("quantize_g128 takes a 2-D [out, in] matrix")
    rows, cols = w.shape
    g = _groups(rows, cols)
    b = w.detach().float().reshape(rows, g, GROUP)
    mn, mx = b.amin(dim=2), b.amax(dim=2)
    s = ((mx - mn) / 15).to(torch.bfloat16).float()
    degenerate = s == 0
    mxb = mx.to(torch.bfloat16).float()
    s = torch.where(degenerate, torch.where(mxb == 0, torch.ones_like(s), mxb), s)
    z = torch.where(degenerate, torch.zeros_like(s), (-mn / s).round().clamp(0, 15))
    codes = ((b / s[..., None]).round() + z[..., None]).clamp(0, 15)
    fill = torch.where(mxb == 0, torch.zeros_like(s), torch.ones_like(s))
    codes = torch.where(degenerate[..., None], fill[..., None].expand_as(codes), codes)
    codes = codes.to(torch.uint8).reshape(rows, cols)
    q = codes[:, 0::2] | (codes[:, 1::2] << 4)
    return q.contiguous(), s.to(torch.bfloat16).contiguous(), z.to(torch.uint8).contiguous()


def unpack_codes(q: torch.Tensor) -> torch.Tensor:
    """[out, in / 2] packed bytes -> [out, in] codes 0..15 (uint8)."""
    return torch.stack([q & 15, q >> 4], dim=-1).reshape(q.shape[0], 2 * q.shape[1])


def _check(q: torch.Tensor, s: torch.Tensor, z: torch.Tensor) -> Tuple[int, int, int]:
    if q.dtype != torch.uint8 or q.dim() != 2:
        raise ValueError(f"q must be a 2-D uint8 [out, in / 2] tensor, got {q.dtype} {tuple(q.shape)}")
    rows, cols = q.shape[0], 2 * q.shape[1]
    g = _groups(rows, cols)
    if s.dtype != torch.bfloat16 or tuple(s.shape) != (rows, g):
        raise ValueError(f"expected a bfloat16 {(rows, g)} scale grid, got {s.dtype} {tuple(s.shape)}")
    if z.dtype != torch.uint8 or tuple(z.shape) != (rows, g):
        raise ValueError(f"expected a uint8 {(rows, g)} zero-point grid, got {z.dtype} {tuple(z.shape)}")
    return rows, cols, g


def dequantize_g128(q: torch.Tensor, s: torch.Tensor, z: torch.Tensor, dtype: torch.dtype = torch.bfloat16) -> torch.Tensor:
    """The weights an int4 engine computes with: (s_expanded.float() * (q.float() - z_expanded.float())).to(dtype) -- an
    exact fp32 product, one rounding.  Zero points above 15 are taken modulo 16, as the GEMMs read only 4 bits."""
    _check(q, s, z)
    codes = unpack_codes(q).float()
    se = s.float().repeat_interleave(GROUP, 1)
    ze = (z & 15).float().repeat_interleave(GROUP, 1)
    return (se * (codes - ze)).to(dtype)


def pack_groups(s: torch.Tensor, z: torch.Tensor) -> torch.Tensor:
    """[out, in / 128] scales and zero points -> the matrix's group grid as it sits in an expert blob: one little-endian
    uint32 (bf16 bits of s | z << 16) per (row, group), tile-major -- the word of (r, g) at index
    ((r // 128) * (in / 128) + g) * 128 + r % 128.  Returned as a flat uint8 tensor."""
    rows, g = s.shape
    if rows % TILE_ROWS or tuple(z.shape) != (rows, g) or s.dtype != torch.bfloat16 or z.dtype != torch.uint8:
        raise ValueError("pack_groups takes bfloat16 scales and uint8 zero points of the same [out, in / 128] shape")
    words = (s.view(torch.int16).to(torch.int32) & 0xffff) | ((z.to(torch.int32) & 15) << 16)
    words = words.reshape(rows // TILE_ROWS, TILE_ROWS, g).permute(0, 2, 1).contiguous()
    return words.view(torch.uint8).reshape(-1)


def expert_blob_bytes(hidden: int, inter: int) -> int:
    """Bytes of one int4 expert slot: three code matrices, then their three group grids (csrc/int4_weights.cuh
    expert_blob_bytes)."""
    _groups(inter, hidden)
    return 3 * hidden * inter // 2 + 3 * (hidden * inter // GROUP) * 4
