// int4_weights.cuh -- routed experts stored as 4-bit integers with a 16-bit scale and a 4-bit zero point per 128 inputs
// (W4A16): B2M_WEIGHTS_INT4_G128 (bf16 scales, bf16 activations) and B2M_WEIGHTS_INT4_G128_F16 (fp16 scales, f16
// activations: the layout AWQ and GPTQ checkpoints use).
//
// Semantics (include/b2m.h): every routed matrix (nn.Linear [out, in], row-major) is stored as codes q[r][c] in 0..15, a
// scale s[r][c / 128] of the context's 16-bit type T (bf16 or f16) and a zero point z[r][c / 128] in 0..15, and the experts
// compute exactly what the T engine computes on
//   W[r][c] = T(s[r][c / 128] * (q[r][c] - z[r][c / 128]))
// -- the product is exact in fp32 (s has 8 (bf16) or 11 (f16) significant bits, |q - z| <= 15, and both types lie inside
// fp32's exponent range), so W is that product rounded ONCE to nearest-even, subnormals included, overflow (f16) to +-Inf
// (torch: `(s_expanded.float() * (q.float() - z_expanded.float())).to(T)`).  The GEMM consumers build exactly these W as
// their register A fragments and feed the unchanged T register-A wgmma, so an int4 context is bit-identical to a T context
// loaded with the dequantised weights.
//
// Expert blob in a slot (no padding: H and I are multiples of 128; the same bytes for both scale types):
//   1. the three code matrices in the model's tensor order (Mixtral w1 | w2 | w3, DeepSeek gate | up | down), each
//      [rows][cols / 2] bytes; byte c / 2 holds column c in its low nibble when c is even, in its high nibble when c is odd;
//   2. the three group grids in the same order: one uint32 per (row, 128-column group) = the T bits of s (bits 0..15) |
//      z << 16 (bits 16..19; the other bits are ignored), TILE-MAJOR: the word of (r, g) sits at index
//      ((r / 128) * (cols / 128) + g) * 128 + r % 128, so the 128 rows of one GEMM tile's group are 512 contiguous bytes.
//
// GEMM A tile: 128 rows x 64 k = 32-byte rows, 4 KiB, loaded by TMA (uint8 elements, box {32 B, 128 rows}) with SWIZZLE_32B:
// byte (row, b) sits at row * 32 + ((b >> 4) ^ ((row >> 2) & 1)) * 16 + (b & 15).  A consumer thread reads each of its two
// rows with two 16-byte shared loads; the eight rows a warp reads then cover all 32 banks once (rows 4..7 of the eight take
// the other 16-B half of the 128-B bank window), so the loads are free of bank conflicts.
//
// Decode of one T x2 fragment register (two neighbouring k of one row, one code byte): lop3 places each nibble under the
// exponent of 128 (bf16: 0x4300 | q is exactly 128 + q) or of 1024 (f16: 0x6400 | q is exactly 1024 + q), sub.rn.{bf16x2,
// f16x2} subtracts {128 + z} / {1024 + z} (exact: both are integers T represents), mul.rn by {s, s} -- the one rounding of
// the definition.
//
// This header is the only place that knows the format: api.cu (slot layout), grouped_gemm.cu (GEMM consumers) and
// tests/host/int4_weights_check.cpp (host decode against torch's rounding) use the functions below.
#pragma once
#include <stdint.h>
#include <stddef.h>
#include <string.h>

#include "fp8_weights.cuh"   // f8::float_to_bf16_rn

#if defined(__CUDACC__)
#include <cuda_bf16.h>
#include <cuda_fp16.h>
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
I4_HD float f16_to_float(uint16_t h) {
  const uint32_t sign = (uint32_t)(h & 0x8000u) << 16, e = (h >> 10) & 31u, m = h & 0x3ffu;
  uint32_t u;
  if (e == 0) {                                                     // +-0 and subnormals: m * 2^-24, exact in fp32
    const float f = (float)m * 5.9604644775390625e-8f;
    memcpy(&u, &f, 4);
    u |= sign;
  } else {
    u = sign | (e == 31 ? 0x7f800000u : (e + 112) << 23) | (m << 13);
  }
  float f;
  memcpy(&f, &u, 4);
  return f;
}
// fp32 -> f16 bits, round to nearest-even; subnormal results kept, overflow to +-Inf
I4_HD uint16_t float_to_f16_rn(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  const uint16_t sign = (uint16_t)((u >> 16) & 0x8000u);
  const uint32_t a = u & 0x7fffffffu;
  if (a > 0x7f800000u) return (uint16_t)(sign | 0x7e00u | ((a >> 13) & 0x3ffu));   // NaN (quiet)
  if (a >= 0x477ff000u) return (uint16_t)(sign | 0x7c00u);                        // >= 65520 (half-way past 65504): Inf
  if (a >= 0x38800000u)                                                             // >= 2^-14: a normal f16
    return (uint16_t)(sign | (((a + 0xfffu + ((a >> 13) & 1u)) >> 13) - (112u << 10)));
  // below 2^-14: n units of 2^-24 (n = 1024, a carry into the exponent field, is the smallest normal)
  const int e = (int)(a >> 23);
  const int shift = 126 - e;                                        // a = m * 2^(e - 150) = m * 2^-24 / 2^shift
  if (e == 0 || shift > 24) return sign;                            // below 2^-25: rounds to +-0
  const uint32_t m = (a & 0x7fffffu) | 0x800000u;
  uint32_t n = m >> shift;
  const uint32_t rem = m & ((1u << shift) - 1u), half = 1u << (shift - 1);
  if (rem > half || (rem == half && (n & 1u))) ++n;
  return (uint16_t)(sign | n);
}
// the dequantised f16 bits of code q (0..15) under zero point z (0..15) and f16 scale bits s
I4_HD uint16_t dequant_f16(uint32_t q, uint32_t z, uint16_t s) {
  return float_to_f16_rn(f16_to_float(s) * (float)((int)(q & 15) - (int)(z & 15)));
}
// byte offset of (row, code byte b) inside a SWIZZLE_32B A tile
I4_HD uint32_t tile_offset(int row, int b) {
  return (uint32_t)(row * ROW_BYTES + (((b >> 4) ^ ((row >> 2) & 1)) << 4) + (b & 15));
}

#if defined(__CUDACC__)
// the x2 instructions of the 16-bit type T (__nv_bfloat16 or __half: the activations' type, Half16<DT>::T) and the bits of
// {B + 0, B + 0} whose low mantissa bits a code fills in: B = 128 (bf16 0x4300) or 1024 (f16 0x6400), where the unit is 1
template <typename T> struct X2;
template <> struct X2<__nv_bfloat16> {
  static constexpr uint32_t CODE_BASE = 0x43004300u;
  __device__ __forceinline__ static void sub(uint32_t& d, uint32_t b) { asm("sub.rn.bf16x2 %0, %0, %1;" : "+r"(d) : "r"(b)); }
  __device__ __forceinline__ static void mul(uint32_t& d, uint32_t b) { asm("mul.rn.bf16x2 %0, %0, %1;" : "+r"(d) : "r"(b)); }
};
template <> struct X2<__half> {
  static constexpr uint32_t CODE_BASE = 0x64006400u;
  __device__ __forceinline__ static void sub(uint32_t& d, uint32_t b) { asm("sub.rn.f16x2 %0, %0, %1;" : "+r"(d) : "r"(b)); }
  __device__ __forceinline__ static void mul(uint32_t& d, uint32_t b) { asm("mul.rn.f16x2 %0, %0, %1;" : "+r"(d) : "r"(b)); }
};

// two code bytes -> the T x2 registers of their k pairs, dequantised: t holds byte b0 in bits 0..7 and b1 in bits 16..23;
// ra = {W(b0 low nibble), W(b0 high nibble)}, rb = the same of b1.  zz = {B + z, B + z}, ss = {s, s}.
template <typename T>
__device__ __forceinline__ void dequant_pairs(uint32_t t, uint32_t zz, uint32_t ss, uint32_t& ra, uint32_t& rb) {
  const uint32_t lo = (t & 0x000f000fu) | X2<T>::CODE_BASE;     // one lop3 each: {B + low nibbles}, {B + high nibbles}
  const uint32_t hi = ((t >> 4) & 0x000f000fu) | X2<T>::CODE_BASE;
  asm("prmt.b32 %0, %1, %2, 0x5410;" : "=r"(ra) : "r"(lo), "r"(hi));
  asm("prmt.b32 %0, %1, %2, 0x7632;" : "=r"(rb) : "r"(lo), "r"(hi));
  X2<T>::sub(ra, zz);                                              // q - z, exact
  X2<T>::sub(rb, zz);
  X2<T>::mul(ra, ss);                                              // * s, one rounding
  X2<T>::mul(rb, ss);
}
// {B + z, B + z} and {s, s} of a group word
template <typename T>
__device__ __forceinline__ uint32_t group_zz(uint32_t w) { return X2<T>::CODE_BASE | (((w >> 16) & 15u) * 0x10001u); }
__device__ __forceinline__ uint32_t group_ss(uint32_t w) { return __byte_perm(w, 0, 0x1010); }

// lane L's A fragments of one k-block (m64k16 layout of weight_pack.cuh's lane_coord: a[4j + r] = register r of k16 step j,
// r & 1 -> row + 8, r & 2 -> k + 8) from a SWIZZLE_32B int4 tile in shared memory.  g0 / g1 are the group words of the
// lane's rows r0 and r0 + 8.  Register (j, r) holds k = 16 j + 8 (r >> 1) + 2 tig + {0, 1}: code byte 8 j + 4 (r >> 1) + tig
// of its row, i.e. byte tig of word 2 j + (r >> 1).
template <typename T>
__device__ __forceinline__ void decode_lane(const uint8_t* tile, int L, uint32_t g0, uint32_t g1, uint32_t (&a)[16]) {
  const int t = L & 127, g = (t & 31) >> 2, tig = t & 3;
  const int r0 = (L >> 7) * 64 + (t >> 5) * 16 + g;                 // rows r0, r0 + 8 share (row >> 2) & 1
  const uint32_t sw = (uint32_t)((r0 >> 2) & 1);
  const uint32_t sel = (uint32_t)(tig | (tig << 4) | ((4 + tig) << 8) | ((4 + tig) << 12));   // byte tig of two words
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const uint32_t zz = group_zz<T>(h ? g1 : g0), ss = group_ss(h ? g1 : g0);
    const uint8_t* row = tile + (r0 + 8 * h) * ROW_BYTES;
#pragma unroll
    for (int c = 0; c < 2; ++c) {                                   // 16-B chunk c = code bytes 16 c .. 16 c + 15 = k16 steps 2c, 2c + 1
      const uint4 v = *reinterpret_cast<const uint4*>(row + (((uint32_t)c ^ sw) << 4));
      const int j = 2 * c;
      dequant_pairs<T>(__byte_perm(v.x, v.y, sel), zz, ss, a[4 * j + h], a[4 * j + 2 + h]);
      dequant_pairs<T>(__byte_perm(v.z, v.w, sel), zz, ss, a[4 * (j + 1) + h], a[4 * (j + 1) + 2 + h]);
    }
  }
}
#endif

}  // namespace i4
}  // namespace b2m
