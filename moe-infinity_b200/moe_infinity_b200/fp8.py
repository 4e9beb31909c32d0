"""FP8 E4M3 expert weights with one fp32 scale per 128x128 block (the format of DeepSeek-V3 / Qwen3-MoE FP8 checkpoints) or
one fp32 scale per output channel (Llama 4 Maverick FP8 and other fbgemm FP8 checkpoints; per-tensor scales repeated).

`MoEEngine(..., expert_dtype=torch.float8_e4m3fn)` runs block-scaled experts; the numbers it computes are defined by
`dequantize_block128`: the bf16 engine on W = bf16(fp32(w_q) * s[r // 128][c // 128]) (include/b2m.h,
B2M_WEIGHTS_FP8_E4M3_B128).  `MoEEngine(..., expert_dtype=torch.float8_e4m3fn, fp8_scales="row")` runs row-scaled
experts, defined by `dequantize_row`: W = bf16(fp32(w_q) * s[r]) (B2M_WEIGHTS_FP8_E4M3_ROW).  `quantize_block128` and
`quantize_row` turn a bf16 / fp32 checkpoint into those formats."""
from __future__ import annotations

from typing import Tuple

import torch

BLOCK = 128
E4M3_MAX = 448.0


def _blocks(rows: int, cols: int) -> Tuple[int, int]:
    if rows % BLOCK or cols % BLOCK:
        raise ValueError(f"a [{rows}, {cols}] matrix does not divide into {BLOCK}x{BLOCK} blocks")
    return rows // BLOCK, cols // BLOCK


def quantize_block128(w: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """w [out, in] (any float dtype) -> (w_q float8_e4m3fn [out, in], s float32 [out / 128, in / 128]).

    s = amax(|block|) / 448 (an all-zero block gets s = 1); w / s is clamped to +-448 before the cast to e4m3."""
    if w.dim() != 2:
        raise ValueError("quantize_block128 takes a 2-D [out, in] matrix")
    br, bc = _blocks(*w.shape)
    b = w.detach().float().reshape(br, BLOCK, bc, BLOCK)
    amax = b.abs().amax(dim=(1, 3))
    s = torch.where(amax == 0, torch.ones_like(amax), amax / E4M3_MAX)
    q = (b / s[:, None, :, None]).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    return q.reshape(w.shape), s.contiguous()


def expand_scales(s: torch.Tensor) -> torch.Tensor:
    """[out / 128, in / 128] block scales -> one scale per element [out, in]."""
    return s.float().repeat_interleave(BLOCK, 0).repeat_interleave(BLOCK, 1)


def dequantize_block128(w_q: torch.Tensor, s: torch.Tensor, dtype: torch.dtype = torch.bfloat16) -> torch.Tensor:
    """The weights an fp8 engine computes with: (fp32(w_q) * s_expanded).to(dtype) -- one fp32 multiply, one rounding."""
    if w_q.dtype != torch.float8_e4m3fn:
        raise ValueError(f"w_q must be float8_e4m3fn, got {w_q.dtype}")
    br, bc = _blocks(*w_q.shape)
    if tuple(s.shape) != (br, bc):
        raise ValueError(f"scale grid {tuple(s.shape)} does not match a {tuple(w_q.shape)} matrix (want {(br, bc)})")
    return (w_q.float() * expand_scales(s.to(w_q.device))).to(dtype)


def quantize_row(w: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """w [out, in] (any float dtype) -> (w_q float8_e4m3fn [out, in], s float32 [out]).

    s = amax(|row|) / 448 (an all-zero row gets s = 1); w / s is clamped to +-448 before the cast to e4m3."""
    if w.dim() != 2:
        raise ValueError("quantize_row takes a 2-D [out, in] matrix")
    wf = w.detach().float()
    amax = wf.abs().amax(dim=1)
    s = torch.where(amax == 0, torch.ones_like(amax), amax / E4M3_MAX)
    q = (wf / s[:, None]).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    return q, s.contiguous()


def dequantize_row(w_q: torch.Tensor, s: torch.Tensor, dtype: torch.dtype = torch.bfloat16) -> torch.Tensor:
    """The weights a row-scaled fp8 engine computes with: (fp32(w_q) * s[:, None]).to(dtype) -- one fp32 multiply, one
    rounding.  s is float32 [out] or [out, 1]."""
    if w_q.dtype != torch.float8_e4m3fn or w_q.dim() != 2:
        raise ValueError(f"w_q must be a 2-D float8_e4m3fn matrix, got {w_q.dtype} {tuple(w_q.shape)}")
    if s.dtype != torch.float32 or tuple(s.shape) not in ((w_q.shape[0],), (w_q.shape[0], 1)):
        raise ValueError(f"row scales must be float32 [{w_q.shape[0]}] or [{w_q.shape[0]}, 1], got {s.dtype} {tuple(s.shape)}")
    return (w_q.float() * s.to(w_q.device).reshape(-1, 1)).to(dtype)


def expert_blob_bytes(hidden: int, inter: int, scales: str = "block128") -> int:
    """Bytes of one fp8 expert slot: three e4m3 matrices, then their three fp32 scale grids ("block128") or scale vectors
    of inter, inter and hidden rows ("row"), padded to 16 B (csrc/fp8_weights.cuh expert_blob_bytes /
    row_expert_blob_bytes)."""
    if scales == "row":
        return (3 * hidden * inter + 4 * (2 * inter + hidden) + 15) // 16 * 16
    if scales != "block128":
        raise ValueError(f"fp8 scales {scales!r}: 'block128' or 'row'")
    br, bc = _blocks(inter, hidden)
    return (3 * hidden * inter + 3 * br * bc * 4 + 15) // 16 * 16
