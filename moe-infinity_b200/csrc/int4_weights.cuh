// int4_weights.cuh -- routed experts stored as 4-bit integers with a bf16 scale and a 4-bit zero point per 128 inputs
// (B2M_WEIGHTS_INT4_G128; W4A16: 4-bit weights, bf16 activations).
//
// Semantics (include/b2m.h): every routed matrix (nn.Linear [out, in], row-major) is stored as codes q[r][c] in 0..15, a
// bf16 scale s[r][c / 128] and a zero point z[r][c / 128] in 0..15, and the experts compute exactly what the bf16 engine
// computes on
//   W[r][c] = bf16(s[r][c / 128] * (q[r][c] - z[r][c / 128]))
// -- the product is exact in fp32 (s has 8 significant bits, |q - z| <= 15, and bf16 shares fp32's exponent range), so W is
// that product rounded ONCE to nearest-even, subnormals included (torch:
// `(s_expanded.float() * (q.float() - z_expanded.float())).to(torch.bfloat16)`).  The GEMM consumers build exactly these W as
// their register A fragments and feed the unchanged bf16 register-A wgmma, so an int4 context is bit-identical to a bf16
// context loaded with the dequantised weights.
//
// Expert blob in a slot (no padding: H and I are multiples of 128):
//   1. the three code matrices in the model's tensor order (Mixtral w1 | w2 | w3, DeepSeek gate | up | down), each
//      [rows][cols / 2] bytes; byte c / 2 holds column c in its low nibble when c is even, in its high nibble when c is odd;
//   2. the three group grids in the same order: one uint32 per (row, 128-column group) = bf16 bits of s (bits 0..15) |
//      z << 16 (bits 16..19; the other bits are ignored), TILE-MAJOR: the word of (r, g) sits at index
//      ((r / 128) * (cols / 128) + g) * 128 + r % 128, so the 128 rows of one GEMM tile's group are 512 contiguous bytes.
//
// GEMM A tile: 128 rows x 64 k = 32-byte rows, 4 KiB, loaded by TMA (uint8 elements, box {32 B, 128 rows}) with SWIZZLE_32B:
// byte (row, b) sits at row * 32 + ((b >> 4) ^ ((row >> 2) & 1)) * 16 + (b & 15).  A consumer thread reads each of its two
// rows with two 16-byte shared loads; the eight rows a warp reads then cover all 32 banks once (rows 4..7 of the eight take
// the other 16-B half of the 128-B bank window), so the loads are free of bank conflicts.
//
// Decode of one bf16x2 fragment register (two neighbouring k of one row, one code byte): lop3 places each nibble under the
// bf16 exponent of 128 (0x4300 | q is exactly 128 + q), sub.rn.bf16x2 subtracts 128 + z (exact: both are integers below
// 256), mul.rn.bf16x2 multiplies by {s, s} -- the one rounding of the definition.
//
// This header is the only place that knows the format: api.cu (slot layout), grouped_gemm.cu (GEMM consumers) and
// tests/host/int4_weights_check.cpp (host decode against torch's rounding) use the functions below.
#pragma once
#include <stdint.h>
#include <stddef.h>
#include <string.h>

#include "fp8_weights.cuh"   // f8::float_to_bf16_rn

#if defined(__CUDACC__)
#define I4_HD __host__ __device__ __forceinline__
#else
#define I4_HD inline
#endif

namespace b2m {
namespace i4 {

constexpr int GROUP = 128;                        // inputs per scale / zero point
constexpr int ROWS = 128, COLS = 64;              // GEMM A tile: 128 rows x 64 k (two codes per byte)
constexpr int ROW_BYTES = COLS / 2;               // 32 = the SWIZZLE_32B span
constexpr int TILE_BYTES = ROWS * ROW_BYTES;      // 4 KiB

// ---- slot layout (matrix m = 0, 1, 2 in the blob's order; every matrix of an expert holds H * I codes)
I4_HD size_t code_bytes(int H, int I) { return (size_t)H * (size_t)I / 2; }
I4_HD size_t grid_bytes(int H, int I) { return (size_t)H * (size_t)I / GROUP * 4; }
I4_HD size_t expert_blob_bytes(int H, int I) { return 3 * code_bytes(H, I) + 3 * grid_bytes(H, I); }
I4_HD size_t code_offset(int H, int I, int m) { return (size_t)m * code_bytes(H, I); }
I4_HD size_t grid_offset(int H, int I, int m) { return 3 * code_bytes(H, I) + (size_t)m * grid_bytes(H, I); }
// word index of (row r, group g) inside the tile-major group grid of a matrix with `cols` columns
I4_HD size_t grid_index(int r, int g, int cols) {
  return ((size_t)(r / ROWS) * (size_t)(cols / GROUP) + (size_t)g) * ROWS + (size_t)(r % ROWS);
}

// ---- per-element decode (host and device; the device GEMM path below does the same arithmetic two values at a time)
I4_HD float bf16_to_float(uint16_t b) {
  const uint32_t u = (uint32_t)b << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}
// the dequantised bf16 bits of code q (0..15) under zero point z (0..15) and scale bits s
I4_HD uint16_t dequant(uint32_t q, uint32_t z, uint16_t s) {
  return f8::float_to_bf16_rn(bf16_to_float(s) * (float)((int)(q & 15) - (int)(z & 15)));
}
// byte offset of (row, code byte b) inside a SWIZZLE_32B A tile
I4_HD uint32_t tile_offset(int row, int b) {
  return (uint32_t)(row * ROW_BYTES + (((b >> 4) ^ ((row >> 2) & 1)) << 4) + (b & 15));
}

#if defined(__CUDACC__)
// two code bytes -> the bf16x2 registers of their k pairs, dequantised: t holds byte b0 in bits 0..7 and b1 in bits 16..23;
// ra = {W(b0 low nibble), W(b0 high nibble)}, rb = the same of b1.  zz = {128 + z, 128 + z}, ss = {s, s}.
__device__ __forceinline__ void dequant_pairs(uint32_t t, uint32_t zz, uint32_t ss, uint32_t& ra, uint32_t& rb) {
  const uint32_t lo = (t & 0x000f000fu) | 0x43004300u;           // one lop3 each: {128 + low nibbles}, {128 + high nibbles}
  const uint32_t hi = ((t >> 4) & 0x000f000fu) | 0x43004300u;
  asm("prmt.b32 %0, %1, %2, 0x5410;" : "=r"(ra) : "r"(lo), "r"(hi));
  asm("prmt.b32 %0, %1, %2, 0x7632;" : "=r"(rb) : "r"(lo), "r"(hi));
  asm("sub.rn.bf16x2 %0, %0, %1;" : "+r"(ra) : "r"(zz));                           // q - z, exact
  asm("sub.rn.bf16x2 %0, %0, %1;" : "+r"(rb) : "r"(zz));
  asm("mul.rn.bf16x2 %0, %0, %1;" : "+r"(ra) : "r"(ss));                           // * s, one rounding
  asm("mul.rn.bf16x2 %0, %0, %1;" : "+r"(rb) : "r"(ss));
}
// {128 + z, 128 + z} and {s, s} of a group word
__device__ __forceinline__ uint32_t group_zz(uint32_t w) { return 0x43004300u | (((w >> 16) & 15u) * 0x10001u); }
__device__ __forceinline__ uint32_t group_ss(uint32_t w) { return __byte_perm(w, 0, 0x1010); }

// lane L's A fragments of one k-block (m64k16 layout of weight_pack.cuh's lane_coord: a[4j + r] = register r of k16 step j,
// r & 1 -> row + 8, r & 2 -> k + 8) from a SWIZZLE_32B int4 tile in shared memory.  g0 / g1 are the group words of the
// lane's rows r0 and r0 + 8.  Register (j, r) holds k = 16 j + 8 (r >> 1) + 2 tig + {0, 1}: code byte 8 j + 4 (r >> 1) + tig
// of its row, i.e. byte tig of word 2 j + (r >> 1).
__device__ __forceinline__ void decode_lane(const uint8_t* tile, int L, uint32_t g0, uint32_t g1, uint32_t (&a)[16]) {
  const int t = L & 127, g = (t & 31) >> 2, tig = t & 3;
  const int r0 = (L >> 7) * 64 + (t >> 5) * 16 + g;                 // rows r0, r0 + 8 share (row >> 2) & 1
  const uint32_t sw = (uint32_t)((r0 >> 2) & 1);
  const uint32_t sel = (uint32_t)(tig | (tig << 4) | ((4 + tig) << 8) | ((4 + tig) << 12));   // byte tig of two words
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const uint32_t zz = group_zz(h ? g1 : g0), ss = group_ss(h ? g1 : g0);
    const uint8_t* row = tile + (r0 + 8 * h) * ROW_BYTES;
#pragma unroll
    for (int c = 0; c < 2; ++c) {                                   // 16-B chunk c = code bytes 16 c .. 16 c + 15 = k16 steps 2c, 2c + 1
      const uint4 v = *reinterpret_cast<const uint4*>(row + (((uint32_t)c ^ sw) << 4));
      const int j = 2 * c;
      dequant_pairs(__byte_perm(v.x, v.y, sel), zz, ss, a[4 * j + h], a[4 * j + 2 + h]);
      dequant_pairs(__byte_perm(v.z, v.w, sel), zz, ss, a[4 * (j + 1) + h], a[4 * (j + 1) + 2 + h]);
    }
  }
}
#endif

}  // namespace i4
}  // namespace b2m
