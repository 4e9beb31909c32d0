// weight_pack.cuh -- lossless 12-bit packed copy of a K-major bf16 weight matrix, one record per 128-row x 64-k tile.
//
// A bf16 weight spends 8 bits on its exponent, but inside one tile of a weight matrix the exponents span a narrow range.
// A tile is coded against a 15-exponent window [base, base + 14] anchored at its largest exponent: every value keeps its
// sign and 7 mantissa bits and gets a 4-bit exponent code (0 = +-0, c = 1..15: exponent base + c - 1).  Nonzero values
// below the window (subnormals included) are stored as code 0 and listed as patches that hold their original bits.  A tile
// with more than MAX_PATCH such values, an Inf/NaN, or a window above exponent 142 (|w| >= 2^15: the decode multiplier
// would not be a finite bf16) cannot be coded: the encoder marks it raw and its matrix is read from the bf16 copy.
//
// Record = 128-B header + 12 288-B body (0.758 of the tile's 16 384 bf16 bytes):
//   header word 0: base | npatch << 8 | raw << 16; words 4..19: patch i = pos | bf16 bits << 16; the rest is zero.
//   body: the tile as the wgmma m64k16 A fragments of the two consumer warpgroups hold it.  "Lane" L = 0..255 is consumer
//   thread L (warpgroup L >> 7 owns rows 64 * (L >> 7) ..); it owns 32 values (lane_coord) = 16 bf16x2 register pairs,
//   stored as 12 words W[0..11]: word i sits at body byte ((i >> 2) * 256 + L) * 16 + (i & 3) * 4, so one warp's 16-byte
//   shared loads of a chunk are contiguous (no bank conflicts).  pos of a patch = L * 32 + value index.
// A value's 12 bits in "pre" form are its bf16 bits with the exponent field replaced by the code (bits 11..14 zero).
// Pairs 0..11 are carried by W[0..11] in pre form; the 8 free bits (11..14, 27..30) of W[3r], W[3r+1], W[3r+2] hold
// pair 12 + r.  Decoding is a mask (or four shift/mask steps) per pair and one exact bf16x2 multiply by 2^(base - 1):
// code c >= 1 is a normal bf16 with exponent c, the product has exponent base - 1 + c; +-0 stays +-0.
//
// This header is the only place that knows the layout: grouped_gemm.cu (pack kernel, GEMM consumers) and
// tests/host/weight_pack_check.cpp (host round trip) call the functions below.
#pragma once
#include <stdint.h>
#include <stddef.h>

#if defined(__CUDACC__)
#define WP_HD __host__ __device__ __forceinline__
#else
#define WP_HD inline
#endif

namespace b2m {
namespace wp {

constexpr int ROWS = 128, COLS = 64;          // tile of a K-major matrix: 128 rows x 64 k
constexpr int LANES = 256, VALS = 32;         // consumer threads per tile, values per thread
constexpr int HDR_BYTES = 128, BODY_BYTES = 12288, REC_BYTES = HDR_BYTES + BODY_BYTES;
constexpr int MAX_PATCH = 16;
constexpr int MAX_BASE = 128;                 // 2^(base - 1) must be a finite bf16

// tile-local (row, col) of value v (0..31) of lane L: the m64k16 A fragment of k16 step j = v >> 3, register r = (v >> 1) & 3
WP_HD void lane_coord(int L, int v, int* row, int* col) {
  const int t = L & 127, g = (t & 31) >> 2, tig = t & 3;
  const int q = v >> 1, j = q >> 2, r = q & 3;
  *row = (L >> 7) * 64 + (t >> 5) * 16 + g + ((r & 1) ? 8 : 0);
  *col = j * 16 + ((r & 2) ? 8 : 0) + tig * 2 + (v & 1);
}
WP_HD int bf16_exp(uint16_t u) { return (u >> 7) & 0xff; }
// window base from the tile's largest exponent; > MAX_BASE: not codable
WP_HD int window_base(int max_exp) { return max_exp - 14 > 1 ? max_exp - 14 : 1; }
// pre form of u in the window of `base`; false: u is nonzero and below the window (a patch, stored as +0)
WP_HD bool to_pre(uint16_t u, int base, uint16_t* pre) {
  const int e = bf16_exp(u);
  if (e == 0 && (u & 0x7f) == 0) { *pre = u; return true; }   // +-0
  if (e < base) { *pre = 0; return false; }
  *pre = (uint16_t)((u & 0x807f) | ((e - base + 1) << 7));
  return true;
}
WP_HD uint32_t pair_at(const uint16_t (&pre)[VALS], int q) { return (uint32_t)pre[2 * q] | ((uint32_t)pre[2 * q + 1] << 16); }

WP_HD void pack_lane(const uint16_t (&pre)[VALS], uint32_t (&w)[12]) {
#pragma unroll
  for (int q = 0; q < 12; ++q) w[q] = pair_at(pre, q);
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const uint32_t pw = pair_at(pre, 12 + r);
    w[3 * r] |= (pw & 0x07800780u) << 4;
    w[3 * r + 1] |= (pw & 0x00780078u) << 8;
    w[3 * r + 2] |= ((pw & 0x00070007u) << 11) | ((pw & 0x80008000u) >> 1);
  }
}
// the 16 pairs of a lane in pre form
WP_HD void unpack_lane(const uint32_t (&w)[12], uint32_t (&pw)[16]) {
#pragma unroll
  for (int q = 0; q < 12; ++q) pw[q] = w[q] & 0x87ff87ffu;
#pragma unroll
  for (int r = 0; r < 4; ++r)
    pw[12 + r] = ((w[3 * r] >> 4) & 0x07800780u) | ((w[3 * r + 1] >> 8) & 0x00780078u) | ((w[3 * r + 2] >> 11) & 0x00070007u) |
                 ((w[3 * r + 2] << 1) & 0x80008000u);
}
WP_HD uint32_t body_word_offset(int L, int i) { return (uint32_t)HDR_BYTES + (uint32_t)(((i >> 2) * LANES + L) * 16 + (i & 3) * 4); }
WP_HD uint32_t header_word0(int base, int npatch, bool raw) { return (uint32_t)base | ((uint32_t)npatch << 8) | (raw ? 1u << 16 : 0u); }
// bf16x2 multiplier 2^(base - 1) in both halves
WP_HD uint32_t scale_pair(int base) { const uint32_t s = (uint32_t)(base + 126) << 7; return s | (s << 16); }

#if defined(__CUDACC__)
// pre-form pair -> bf16 pair: exact (a power-of-two scale of a normal value or of +-0, the result is a normal bf16)
__device__ __forceinline__ uint32_t scale_dev(uint32_t pw, uint32_t mul) {
  uint32_t d;
  asm("mul.rn.bf16x2 %0, %1, %2;" : "=r"(d) : "r"(pw), "r"(mul));
  return d;
}
// lane L's A fragments of one k-block from a record in shared memory: a[4j..4j+3] = registers of k16 step j
__device__ __forceinline__ void decode_lane(const uint8_t* rec, int L, uint32_t (&a)[16]) {
  const uint32_t* hdr = reinterpret_cast<const uint32_t*>(rec);
  const uint4* body = reinterpret_cast<const uint4*>(rec + HDR_BYTES);
  const uint32_t h0 = hdr[0];
  const uint4 c0 = body[L], c1 = body[LANES + L], c2 = body[2 * LANES + L];
  const uint32_t w[12] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w, c2.x, c2.y, c2.z, c2.w};
  uint32_t pw[16];
  unpack_lane(w, pw);
  const uint32_t mul = scale_pair((int)(h0 & 0xff));
#pragma unroll
  for (int q = 0; q < 16; ++q) a[q] = scale_dev(pw[q], mul);
  // patches (about one per tile): a patched value decodes to +0, then takes its original bits.  The register is picked with an
  // opaque compare/select per register, so the array stays in registers (no indexed local-memory access).
  const int np = (int)((h0 >> 8) & 0xff);
  for (int i = 0; i < np; ++i) {
    const uint32_t pt = hdr[4 + i];
    if ((int)((pt & 0xffff) >> 5) != L) continue;
    const uint32_t qv = (pt >> 1) & 15, half = (pt & 1) ? 0xffff0000u : 0x0000ffffu, bits = (pt >> 16) * 0x10001u;
#pragma unroll
    for (int q = 0; q < 16; ++q) {
      uint32_t m;
      asm("{\n.reg .pred p;\nsetp.eq.u32 p, %1, %2;\nselp.b32 %0, %3, 0, p;\n}" : "=r"(m) : "r"((uint32_t)q), "r"(qv), "r"(half));
      a[q] = (a[q] & ~m) | (bits & m);
    }
  }
  // the warpgroup reconverges before the registers feed a wgmma: the last definition of a[] is this point, not the divergent
  // patch branch (ptxas would otherwise serialise every wgmma of the kernel)
  __syncwarp();
#pragma unroll
  for (int q = 0; q < 16; ++q) asm volatile("" : "+r"(a[q]));
}
#endif
// host mirror of scale_dev (pre form has exponent field = code; code 0 only with a zero mantissa)
inline uint16_t scale_host(uint16_t pre, int base) {
  const int c = bf16_exp(pre);
  return c == 0 ? pre : (uint16_t)((pre & 0x807f) | ((c + base - 1) << 7));
}

// ---- host encoder / decoder of one tile (the device pack kernel runs the same steps with one lane per thread)
// src: the tile's top-left value in a K-major matrix with row stride ld (elements).  Returns false (record marked raw,
// body zero) when the tile cannot be coded.
inline bool encode_tile(const uint16_t* src, size_t ld, uint8_t* rec) {
  for (int i = 0; i < REC_BYTES; ++i) rec[i] = 0;
  int max_e = 0;
  bool special = false;
  for (int r = 0; r < ROWS; ++r)
    for (int c = 0; c < COLS; ++c) {
      const int e = bf16_exp(src[(size_t)r * ld + c]);
      special |= e == 255;
      max_e = e > max_e ? e : max_e;
    }
  const int base = window_base(max_e);
  uint32_t* hdr = reinterpret_cast<uint32_t*>(rec);
  int np = 0;
  bool ok = !special && base <= MAX_BASE;
  for (int L = 0; L < LANES && ok; ++L) {
    uint16_t pre[VALS];
    for (int v = 0; v < VALS; ++v) {
      int row, col;
      lane_coord(L, v, &row, &col);
      const uint16_t u = src[(size_t)row * ld + col];
      if (!to_pre(u, base, &pre[v])) {
        if (np == MAX_PATCH) { ok = false; break; }
        hdr[4 + np++] = (uint32_t)(L * VALS + v) | ((uint32_t)u << 16);
      }
    }
    if (!ok) break;
    uint32_t w[12];
    pack_lane(pre, w);
    for (int i = 0; i < 12; ++i) *reinterpret_cast<uint32_t*>(rec + body_word_offset(L, i)) = w[i];
  }
  if (!ok) {
    for (int i = 0; i < REC_BYTES; ++i) rec[i] = 0;
    hdr[0] = header_word0(0, 0, true);
    return false;
  }
  hdr[0] = header_word0(base, np, false);
  return true;
}
// decode a coded record into the tile at dst (row stride ld); false for a raw record
inline bool decode_tile(const uint8_t* rec, uint16_t* dst, size_t ld) {
  const uint32_t* hdr = reinterpret_cast<const uint32_t*>(rec);
  if ((hdr[0] >> 16) & 1) return false;
  const int base = hdr[0] & 0xff, np = (hdr[0] >> 8) & 0xff;
  for (int L = 0; L < LANES; ++L) {
    uint32_t w[12], pw[16];
    for (int i = 0; i < 12; ++i) w[i] = *reinterpret_cast<const uint32_t*>(rec + body_word_offset(L, i));
    unpack_lane(w, pw);
    for (int v = 0; v < VALS; ++v) {
      int row, col;
      lane_coord(L, v, &row, &col);
      uint16_t u = scale_host((uint16_t)(pw[v >> 1] >> (16 * (v & 1))), base);
      for (int p = 0; p < np; ++p)
        if ((int)(hdr[4 + p] & 0xffff) == L * VALS + v) u = (uint16_t)(hdr[4 + p] >> 16);
      dst[(size_t)row * ld + col] = u;
    }
  }
  return true;
}

}  // namespace wp
}  // namespace b2m
