"""4-bit integer expert weights with a 16-bit scale and a 4-bit zero point per 128 inputs (W4A16 group quantisation).

`MoEEngine(..., expert_dtype=torch.uint4)` runs such experts; the scales are of the engine's dtype T (bfloat16:
B2M_WEIGHTS_INT4_G128; float16: B2M_WEIGHTS_INT4_G128_F16, the AWQ / GPTQ format).  The numbers it computes are defined by
`dequantize_g128`: the T engine on W = T(s[r][c // 128] * (q[r][c] - z[r][c // 128])), the exact product rounded once
(include/b2m.h).  `quantize_g128` turns a bf16 / fp32 checkpoint into that format; `from_awq` and `from_gptq` unpack the
tensors of published AWQ / GPTQ checkpoints into it without changing a weight, and `from_gptq_act_order` unpacks an
act-order GPTQ layer into it with its input columns permuted (`dequantize_g_idx` is GPTQ's own dequantisation of such a
layer); `pack_groups` builds the tile-major group grid an expert blob stores after its code matrices."""
from __future__ import annotations

from typing import Optional, Tuple

import torch

GROUP = 128
TILE_ROWS = 128   # rows of one GEMM tile: the group grid keeps a tile's 128 words of one group together
SCALE_DTYPES = (torch.bfloat16, torch.float16)


def _groups(rows: int, cols: int) -> int:
    if rows % TILE_ROWS or cols % GROUP:
        raise ValueError(f"a [{rows}, {cols}] matrix does not divide into {TILE_ROWS}-row tiles and {GROUP}-input groups")
    return cols // GROUP


def quantize_g128(w: torch.Tensor, scale_dtype: torch.dtype = torch.bfloat16) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """w [out, in] (any float dtype) -> (q uint8 [out, in / 2], s scale_dtype [out, in / 128], z uint8 [out, in / 128]).

    Asymmetric min/max round-to-nearest per group of 128 inputs of a row: s = S((max - min) / 15) with S = scale_dtype
    (bfloat16, or float16 for an f16 engine), rounded to S BEFORE the codes are computed; z = clamp(round(-min / s), 0, 15);
    code = clamp(round(w / s) + z, 0, 15).  A group whose scale rounds to zero (every all-equal group among them) gets
    s = S(max), z = 0 and every code 1, so it holds S(max) exactly -- or s = 1, z = 0, codes 0 when S(max) is zero (an
    all-zero group).  A float16 scale that overflows is refused.
    q packs two codes per byte: column c in the low nibble of byte c // 2 when c is even, in the high nibble when odd."""
    if w.dim() != 2:
        raise ValueError("quantize_g128 takes a 2-D [out, in] matrix")
    if scale_dtype not in SCALE_DTYPES:
        raise ValueError(f"scale_dtype must be torch.bfloat16 or torch.float16, got {scale_dtype}")
    rows, cols = w.shape
    g = _groups(rows, cols)
    b = w.detach().float().reshape(rows, g, GROUP)
    mn, mx = b.amin(dim=2), b.amax(dim=2)
    s = ((mx - mn) / 15).to(scale_dtype).float()
    if scale_dtype == torch.float16 and not bool(torch.isfinite(s).all()):
        raise ValueError("a group's range does not fit a float16 scale (max - min > 15 * 65504)")
    degenerate = s == 0
    mxb = mx.to(scale_dtype).float()
    s = torch.where(degenerate, torch.where(mxb == 0, torch.ones_like(s), mxb), s)
    z = torch.where(degenerate, torch.zeros_like(s), (-mn / s).round().clamp(0, 15))
    codes = ((b / s[..., None]).round() + z[..., None]).clamp(0, 15)
    fill = torch.where(mxb == 0, torch.zeros_like(s), torch.ones_like(s))
    codes = torch.where(degenerate[..., None], fill[..., None].expand_as(codes), codes)
    codes = codes.to(torch.uint8).reshape(rows, cols)
    q = codes[:, 0::2] | (codes[:, 1::2] << 4)
    return q.contiguous(), s.to(scale_dtype).contiguous(), z.to(torch.uint8).contiguous()


def unpack_codes(q: torch.Tensor) -> torch.Tensor:
    """[out, in / 2] packed bytes -> [out, in] codes 0..15 (uint8)."""
    return torch.stack([q & 15, q >> 4], dim=-1).reshape(q.shape[0], 2 * q.shape[1])


def _check(q: torch.Tensor, s: torch.Tensor, z: torch.Tensor) -> Tuple[int, int, int]:
    if q.dtype != torch.uint8 or q.dim() != 2:
        raise ValueError(f"q must be a 2-D uint8 [out, in / 2] tensor, got {q.dtype} {tuple(q.shape)}")
    rows, cols = q.shape[0], 2 * q.shape[1]
    g = _groups(rows, cols)
    if s.dtype not in SCALE_DTYPES or tuple(s.shape) != (rows, g):
        raise ValueError(f"expected a bfloat16 or float16 {(rows, g)} scale grid, got {s.dtype} {tuple(s.shape)}")
    if z.dtype != torch.uint8 or tuple(z.shape) != (rows, g):
        raise ValueError(f"expected a uint8 {(rows, g)} zero-point grid, got {z.dtype} {tuple(z.shape)}")
    return rows, cols, g


def dequantize_g128(q: torch.Tensor, s: torch.Tensor, z: torch.Tensor, dtype: torch.dtype = torch.bfloat16) -> torch.Tensor:
    """The weights an int4 engine computes with: (s_expanded.float() * (q.float() - z_expanded.float())).to(dtype) -- an
    exact fp32 product, one rounding (dtype = the engine's dtype, which is also the type of s; float16 products beyond
    65504 become +-Inf).  Zero points above 15 are taken modulo 16, as the GEMMs read only 4 bits."""
    _check(q, s, z)
    codes = unpack_codes(q).float()
    se = s.float().repeat_interleave(GROUP, 1)
    ze = (z & 15).float().repeat_interleave(GROUP, 1)
    return (se * (codes - ze)).to(dtype)


def pack_groups(s: torch.Tensor, z: torch.Tensor) -> torch.Tensor:
    """[out, in / 128] scales and zero points -> the matrix's group grid as it sits in an expert blob: one little-endian
    uint32 (bf16 or fp16 bits of s | z << 16) per (row, group), tile-major -- the word of (r, g) at index
    ((r // 128) * (in / 128) + g) * 128 + r % 128.  Returned as a flat uint8 tensor."""
    rows, g = s.shape
    if rows % TILE_ROWS or tuple(z.shape) != (rows, g) or s.dtype not in SCALE_DTYPES or z.dtype != torch.uint8:
        raise ValueError("pack_groups takes bfloat16 or float16 scales and uint8 zero points of the same [out, in / 128] shape")
    words = (s.view(torch.int16).to(torch.int32) & 0xffff) | ((z.to(torch.int32) & 15) << 16)
    words = words.reshape(rows // TILE_ROWS, TILE_ROWS, g).permute(0, 2, 1).contiguous()
    return words.view(torch.uint8).reshape(-1)


def expert_blob_bytes(hidden: int, inter: int) -> int:
    """Bytes of one int4 expert slot: three code matrices, then their three group grids (csrc/int4_weights.cuh
    expert_blob_bytes)."""
    _groups(inter, hidden)
    return 3 * hidden * inter // 2 + 3 * (hidden * inter // GROUP) * 4


# ---------------------------------------------------------------- published 4-bit checkpoints (AWQ, GPTQ)
_AWQ_ORDER = (0, 2, 4, 6, 1, 3, 5, 7)   # nibble i of an AWQ word holds output row 8 j + _AWQ_ORDER[i]


def _nibbles(w: torch.Tensor) -> torch.Tensor:
    """int32 [..., n] -> its eight nibbles, least significant first: int64 [..., n, 8] in 0..15."""
    return (w.to(torch.int64)[..., None] >> (4 * torch.arange(8, device=w.device))) & 15


def _pack_codes(codes: torch.Tensor) -> torch.Tensor:
    """[out, in] codes 0..15 -> [out, in / 2] bytes (column c in the low nibble of byte c // 2 when c is even)."""
    codes = codes.to(torch.uint8)
    return (codes[:, 0::2] | (codes[:, 1::2] << 4)).contiguous()


def _checkpoint_groups(what: str, n_in: int, scales: torch.Tensor, n_out: int) -> int:
    if scales.dtype != torch.float16 or scales.dim() != 2 or scales.shape[1] != n_out:
        raise ValueError(f"{what} scales must be float16 [in / group, {n_out}], got {scales.dtype} {tuple(scales.shape)}")
    if scales.shape[0] * GROUP != n_in:
        raise ValueError(f"{what}: only group size {GROUP} is supported ({n_in} inputs, {scales.shape[0]} groups)")
    return scales.shape[0]


def _check_int32(name: str, t: torch.Tensor, shape: Tuple[int, int]):
    if t.dtype != torch.int32 or tuple(t.shape) != shape:
        raise ValueError(f"{name} must be int32 {shape}, got {t.dtype} {tuple(t.shape)}")


def from_awq(qweight: torch.Tensor, qzeros: torch.Tensor, scales: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """One AWQ ("gemm" version, zero_point=True, group size 128) linear layer -> (q, s, z) of this library: q uint8
    [out, in / 2], s float16 [out, in / 128], z uint8 [out, in / 128].  No weight changes: `dequantize_g128(q, s, z,
    torch.float16)` is AWQ's own (q - z) * s in fp16.

    qweight int32 [in, out / 8]: nibble i of qweight[c, j] is the code of output row 8 j + (0, 2, 4, 6, 1, 3, 5, 7)[i];
    qzeros int32 [in / 128, out / 8] in the same nibble order holds z; scales float16 [in / 128, out]."""
    if qweight.dim() != 2:
        raise ValueError(f"AWQ qweight must be int32 [in, out / 8], got {qweight.dtype} {tuple(qweight.shape)}")
    n_in, n_out = qweight.shape[0], 8 * qweight.shape[1]
    _check_int32("AWQ qweight", qweight, (n_in, n_out // 8))
    g = _checkpoint_groups("AWQ", n_in, scales, n_out)
    _check_int32("AWQ qzeros", qzeros, (g, n_out // 8))
    _groups(n_out, n_in)
    inv = [_AWQ_ORDER.index(p) for p in range(8)]                  # row 8 j + p sits in nibble inv[p]
    codes = _nibbles(qweight)[..., inv].reshape(n_in, n_out).t()
    z = _nibbles(qzeros)[..., inv].reshape(g, n_out).t()
    return _pack_codes(codes), scales.t().contiguous(), z.to(torch.uint8).contiguous()


def from_gptq(qweight: torch.Tensor, qzeros: torch.Tensor, scales: torch.Tensor, g_idx: Optional[torch.Tensor] = None,
              checkpoint_format: str = "gptq") -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """One GPTQ (4 bits, group size 128, no act-order) linear layer -> (q, s, z) of this library (as `from_awq`).  No weight
    changes: `dequantize_g128(q, s, z, torch.float16)` is GPTQ's own (q - z) * s in fp16.

    qweight int32 [in / 8, out]: nibble i of qweight[j, r] is input column 8 j + i; qzeros int32 [in / 128, out / 8]: nibble i
    of qzeros[g, j] belongs to row 8 j + i; scales float16 [in / 128, out].  checkpoint_format "gptq" (v1) stores z - 1, so a
    stored 15 (z = 16) cannot be represented and is refused; "gptq_v2" stores z.  g_idx, if given, must be c // 128
    (act-order checkpoints are refused)."""
    n_in = 8 * qweight.shape[0] if qweight.dim() == 2 else 0
    codes, s, z = _gptq_unpack(qweight, qzeros, scales, checkpoint_format)
    if g_idx is not None:
        want = torch.arange(n_in, device=g_idx.device) // GROUP
        if tuple(g_idx.shape) != (n_in,) or not torch.equal(g_idx.to(torch.int64), want):
            raise ValueError("GPTQ g_idx is not c // 128: act-order (desc_act) checkpoints are not supported")
    return _pack_codes(codes), s, z


def _gptq_unpack(qweight: torch.Tensor, qzeros: torch.Tensor, scales: torch.Tensor,
                 checkpoint_format: str) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """GPTQ tensors -> (codes int64 [out, in] in the checkpoint's column order, s float16 [out, groups], z uint8 [out, groups])."""
    if checkpoint_format not in ("gptq", "gptq_v2"):
        raise ValueError(f"GPTQ checkpoint_format must be 'gptq' or 'gptq_v2', got {checkpoint_format!r}")
    if qweight.dim() != 2:
        raise ValueError(f"GPTQ qweight must be int32 [in / 8, out], got {qweight.dtype} {tuple(qweight.shape)}")
    n_in, n_out = 8 * qweight.shape[0], qweight.shape[1]
    _check_int32("GPTQ qweight", qweight, (n_in // 8, n_out))
    g = _checkpoint_groups("GPTQ", n_in, scales, n_out)
    _check_int32("GPTQ qzeros", qzeros, (g, n_out // 8))
    _groups(n_out, n_in)
    codes = _nibbles(qweight).permute(0, 2, 1).reshape(n_in, n_out).t()
    z = _nibbles(qzeros).reshape(g, n_out).t()
    if checkpoint_format == "gptq":
        if bool((z == 15).any()):
            raise ValueError("GPTQ qzeros holds 15, i.e. a zero point of 16 in the v1 format (stored z - 1), "
                             "which 4 bits cannot represent")
        z = z + 1
    return codes, scales.t().contiguous(), z.to(torch.uint8).contiguous()


def act_order_perm(g_idx: torch.Tensor, n_in: int) -> torch.Tensor:
    """An act-order GPTQ layer's g_idx [in] -> P = stable argsort(g_idx) (int64 [in]), the column order in which every
    group is 128 consecutive columns: g_idx[P[j]] = j // 128.  Refused unless every group 0 .. in / 128 - 1 has exactly
    128 columns (GPTQ with desc_act and group size 128 quantises 128 consecutive columns of its order per group)."""
    if g_idx.dim() != 1 or g_idx.numel() != n_in or g_idx.dtype not in (torch.int32, torch.int64):
        raise ValueError(f"GPTQ g_idx must be an int32 [{n_in}] vector, got {g_idx.dtype} {tuple(g_idx.shape)}")
    gi = g_idx.to(torch.int64)
    ng = n_in // GROUP
    if bool((gi < 0).any()) or bool((gi >= ng).any()) or not bool((torch.bincount(gi, minlength=ng) == GROUP).all()):
        raise ValueError(f"GPTQ g_idx does not put exactly {GROUP} columns in each of the {ng} groups")
    return torch.sort(gi, stable=True).indices


def from_gptq_act_order(qweight: torch.Tensor, qzeros: torch.Tensor, scales: torch.Tensor, g_idx: torch.Tensor,
                        checkpoint_format: str = "gptq") -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """One act-order GPTQ (desc_act=True, 4 bits, group size 128) linear layer W [out, in] -> (q, s, z, perm): (q, s, z)
    of this library hold W[:, perm], whose groups are contiguous, and perm = `act_order_perm(g_idx)`.  No weight changes:
    `dequantize_g128(q, s, z, torch.float16)[:, perm.argsort()]` is GPTQ's own dequantisation (`dequantize_g_idx`).
    Since W x = W[:, perm] x[perm], an engine runs the layer on inputs gathered through perm (`MoEEngine.set_input_perm`).
    Tensors as `from_gptq`; any g_idx with 128 columns per group is taken, c // 128 included (then perm is the identity)."""
    codes, s, z = _gptq_unpack(qweight, qzeros, scales, checkpoint_format)
    perm = act_order_perm(g_idx, codes.shape[1])
    return _pack_codes(codes[:, perm]), s, z, perm


def dequantize_g_idx(q: torch.Tensor, s: torch.Tensor, z: torch.Tensor, g_idx: torch.Tensor,
                     dtype: torch.dtype = torch.float16) -> torch.Tensor:
    """GPTQ's own dequantisation of a layer in its checkpoint's column order: W[r][c] = dtype(s[r][g_idx[c]] * (q[r][c] -
    z[r][g_idx[c]])), the exact product rounded once.  q uint8 [out, in / 2] (`unpack_codes` layout, natural columns), s
    and z [out, in / 128] indexed by group; g_idx [in]."""
    _, cols, ng = _check(q, s, z)
    gi = g_idx.to(device=q.device, dtype=torch.int64)
    if tuple(gi.shape) != (cols,) or bool((gi < 0).any()) or bool((gi >= ng).any()):
        raise ValueError(f"g_idx must be [{cols}] group indices below {ng}")
    codes = unpack_codes(q).float()
    return (s.float()[:, gi] * (codes - (z & 15).float()[:, gi])).to(dtype)
