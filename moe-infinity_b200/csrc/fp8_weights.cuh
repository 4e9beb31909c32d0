// fp8_weights.cuh -- routed experts stored as FP8 E4M3 with one fp32 scale per 128 x 128 block (B2M_WEIGHTS_FP8_E4M3_B128)
// or one fp32 scale per output channel, i.e. per matrix row (B2M_WEIGHTS_FP8_E4M3_ROW).
//
// Semantics (include/b2m.h): the experts compute exactly what the bf16 engine computes on
//   W[r][c] = bf16(fp32(w_q[r][c]) * s[r / 128][c / 128])
// -- the e4m3 value is exact in fp32, the product is ONE fp32 multiply rounded to nearest-even, then ONE rounding to bf16
// (torch: `(w_q.float() * s_expanded).to(torch.bfloat16)`).  The GEMM consumers dequantise their A fragments in registers
// with exactly these two roundings and feed the unchanged bf16 register-A wgmma, so an fp8 context is bit-identical to a bf16
// context loaded with the dequantised weights.  (Scaling in the epilogue would round differently, and the scale changes every
// 128 k inside one accumulation.)
//
// Expert blob in a slot: the three e4m3 matrices in the model's tensor order (Mixtral w1 | w2 | w3, DeepSeek gate | up |
// down), then their three fp32 scale grids [rows / 128][cols / 128] in the same order, zero-padded to a multiple of 16 B so
// that TMA global strides stay multiples of 16 B.
// Row format: the same, with s[r][c] = s[r] and scale vectors s[rows] in place of the grids (lengths I, H, I for Mixtral;
// I, I, H for gate | up | down).  A consumer thread's A fragments cover two rows of the tile (ra and ra + 8), so it loads
// their two scales once per tile and decodes every k-block with them (decode_lane's two-scale form).
//
// GEMM A tile: 128 rows x 64 k = 64-byte rows, 8 KiB, loaded by TMA (uint8 elements) with SWIZZLE_64B: byte (row, col) sits
// at row * 64 + ((col >> 4) ^ ((row >> 1) & 3)) * 16 + (col & 15).  A consumer thread reads the two bytes of each register
// half with one 32-bit shared load per (row, 8-k group): the 8 rows of a warp's load fall into 8 different 16-B columns of
// the 128-B bank window (g & 1 picks the half, (g >> 1) the swizzled chunk) and the two lanes sharing a word read the same
// address, so the loads are free of bank conflicts.
//
// This header is the only place that knows the format: api.cu (slot layout), grouped_gemm.cu (GEMM consumers) and
// tests/host/fp8_weights_check.cpp (host decode against torch's rounding) use the functions below.
#pragma once
#include <stdint.h>
#include <stddef.h>
#include <string.h>

#if defined(__CUDACC__)
#define F8_HD __host__ __device__ __forceinline__
#else
#define F8_HD inline
#endif

namespace b2m {
namespace f8 {

constexpr int BLOCK = 128;                        // scale block: 128 rows x 128 k
constexpr int ROWS = 128, COLS = 64;              // GEMM A tile: 128 rows x 64 k (one byte each)
constexpr int TILE_BYTES = ROWS * COLS;           // 8 KiB
constexpr int ROW_BYTES = COLS;                   // = the SWIZZLE_64B span

// ---- slot layout
F8_HD size_t scale_grid_bytes(int rows, int cols) { return (size_t)(rows / BLOCK) * (size_t)(cols / BLOCK) * 4; }
// an expert of three [H x I] / [I x H] matrices: 3 e4m3 matrices + 3 scale grids, rounded up to 16 B
F8_HD size_t expert_blob_bytes(int H, int I) {
  const size_t b = 3 * (size_t)H * (size_t)I + 3 * scale_grid_bytes(H, I);
  return (b + 15) & ~(size_t)15;
}
// byte offset of the scale grid of the matrix at byte offset `mat_off` of the blob
F8_HD size_t scale_grid_offset(int H, int I, size_t mat_off) {
  const size_t m = (size_t)H * (size_t)I;
  return 3 * m + (mat_off / m) * scale_grid_bytes(H, I);
}
// row format: one fp32 scale per row of a rows x cols matrix
F8_HD size_t row_scale_bytes(int rows, int cols) { return (size_t)rows * 4; }
// an expert of two [I x H] matrices and one [H x I]: 3 e4m3 matrices + scale vectors of I, I and H rows, rounded up to 16 B
F8_HD size_t row_expert_blob_bytes(int H, int I) {
  const size_t b = 3 * (size_t)H * (size_t)I + 2 * row_scale_bytes(I, H) + row_scale_bytes(H, I);
  return (b + 15) & ~(size_t)15;
}

// ---- per-element decode (host and device; the device GEMM path below does the same arithmetic two values at a time)
// e4m3fn code -> its exact fp32 value (exponent bias 7, no infinities, S.1111.111 = NaN)
F8_HD float e4m3_to_float(uint8_t c) {
  const uint32_t s = (uint32_t)(c & 0x80) << 24, e = (c >> 3) & 15, m = c & 7;
  uint32_t u;
  if ((c & 0x7f) == 0x7f) u = 0x7fc00000u;                          // NaN
  else if (e) u = s | ((e + 120) << 23) | (m << 20);                // normal: 2^(e-7) * 1.m
  else if (m) {                                                     // subnormal: m * 2^-9, normal in fp32
    const int lz = m >= 4 ? 0 : m >= 2 ? 1 : 2;                     // leading bit of m at position 2 - lz
    u = s | ((uint32_t)(120 - lz) << 23) | (((m << (lz + 1)) & 7) << 20);
  } else u = s;                                                     // +-0
  float f;
  memcpy(&f, &u, 4);
  return f;
}
// fp32 -> bf16, round to nearest even (subnormals kept, overflow to +-Inf); NaN -> quiet NaN
F8_HD uint16_t float_to_bf16_rn(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40);
  return (uint16_t)((u + 0x7fffu + ((u >> 16) & 1)) >> 16);
}
// the dequantised bf16 bits of code c under scale s
F8_HD uint16_t dequant(uint8_t c, float s) { return float_to_bf16_rn(e4m3_to_float(c) * s); }
// row format: the dequantised bf16 bits of a row-major rows x cols e4m3 matrix q under its row scales s[rows]
inline void dequant_rows(const uint8_t* q, const float* s, int rows, int cols, uint16_t* w) {
  for (int r = 0; r < rows; ++r)
    for (int c = 0; c < cols; ++c) w[(size_t)r * cols + c] = dequant(q[(size_t)r * cols + c], s[r]);
}

// byte offset of (row, col) inside a SWIZZLE_64B A tile
F8_HD uint32_t tile_offset(int row, int col) {
  return (uint32_t)(row * ROW_BYTES + (((col >> 4) ^ ((row >> 1) & 3)) << 4) + (col & 15));
}

#if defined(__CUDACC__)
// two e4m3 codes (low byte = lower column) -> bf16x2 = {bf16(fp32(c0) * s), bf16(fp32(c1) * s)}
__device__ __forceinline__ uint32_t dequant2(uint16_t codes, float s) {
  uint32_t h2, d;
  float lo, hi;
  asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h2) : "h"(codes));                                   // exact
  asm("{\n.reg .b16 l, h;\nmov.b32 {l, h}, %2;\ncvt.f32.f16 %0, l;\ncvt.f32.f16 %1, h;\n}" : "=f"(lo), "=f"(hi) : "r"(h2));
  lo = __fmul_rn(lo, s);
  hi = __fmul_rn(hi, s);
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));
  return d;
}
// lane L's A fragments of one k-block (m64k16 layout of weight_pack.cuh's lane_coord: a[4j + r] = register r of k16 step j,
// r & 1 -> row + 8, r & 2 -> k + 8) from a SWIZZLE_64B e4m3 tile in shared memory, dequantised with scale s0 in row r0 and
// s1 in row r0 + 8 (row format: the two rows' scales; block format: s0 == s1, the block's scale)
__device__ __forceinline__ void decode_lane(const uint8_t* tile, int L, float s0, float s1, uint32_t (&a)[16]) {
  const int t = L & 127, g = (t & 31) >> 2, tig = t & 3;
  const int r0 = (L >> 7) * 64 + (t >> 5) * 16 + g;                 // rows r0, r0 + 8 share (row >> 1) & 3
  const uint32_t sw = (uint32_t)((r0 >> 1) & 3);
  const uint8_t* row0 = tile + r0 * ROW_BYTES + (tig >> 1) * 4;     // the word holding columns 2 tig, 2 tig + 1 of a group
  const uint32_t sel = (tig & 1) ? 0x7632u : 0x5410u;               // that half of two words
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint32_t chunk = (((uint32_t)j ^ sw) << 4);               // 16-k step j = one 16-B chunk of the row
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint8_t* p = row0 + h * 8 * ROW_BYTES + chunk;
      const uint32_t w_lo = *reinterpret_cast<const uint32_t*>(p);       // k 16j + 0..7
      const uint32_t w_hi = *reinterpret_cast<const uint32_t*>(p + 8);   // k 16j + 8..15
      uint32_t q;
      asm("prmt.b32 %0, %1, %2, %3;" : "=r"(q) : "r"(w_lo), "r"(w_hi), "r"(sel));
      const float s = h ? s1 : s0;
      a[4 * j + h] = dequant2((uint16_t)(q & 0xffff), s);
      a[4 * j + 2 + h] = dequant2((uint16_t)(q >> 16), s);
    }
  }
}
__device__ __forceinline__ void decode_lane(const uint8_t* tile, int L, float s, uint32_t (&a)[16]) { decode_lane(tile, L, s, s, a); }
#endif

}  // namespace f8
}  // namespace b2m
