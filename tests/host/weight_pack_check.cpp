// Host round trip of the 12-bit packed weight format (moe-infinity_b200/csrc/weight_pack.cuh): encode, then decode, must
// reproduce every bf16 bit of a tile, and tiles the format cannot code must come out raw.  Driven by tests/test_weight_pack.py.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

#include "weight_pack.cuh"

using namespace b2m;

static uint16_t to_bf16(float f) {   // round to nearest even, as torch does
  uint32_t u;
  std::memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return 0x7fc0;
  u += 0x7fff + ((u >> 16) & 1);
  return (uint16_t)(u >> 16);
}

static int fails = 0, coded = 0, raw = 0;

// expect_coded: 1 = must code, 0 = must be raw, -1 = either
static void check(const char* what, const std::vector<uint16_t>& m, size_t ld, int expect_coded) {
  std::vector<uint8_t> rec(wp::REC_BYTES);
  const bool ok = wp::encode_tile(m.data(), ld, rec.data());
  ok ? ++coded : ++raw;
  if (expect_coded >= 0 && ok != (expect_coded == 1)) {
    std::printf("FAIL %s: expected %s\n", what, expect_coded ? "a coded tile" : "a raw tile");
    ++fails;
    return;
  }
  const uint32_t h0 = *reinterpret_cast<const uint32_t*>(rec.data());
  if (((h0 >> 16) & 1) != (ok ? 0u : 1u)) { std::printf("FAIL %s: raw flag\n", what); ++fails; return; }
  if (!ok) return;
  std::vector<uint16_t> out(wp::ROWS * ld, 0xdead);
  if (!wp::decode_tile(rec.data(), out.data(), ld)) { std::printf("FAIL %s: decode refused\n", what); ++fails; return; }
  for (int r = 0; r < wp::ROWS; ++r)
    for (int c = 0; c < wp::COLS; ++c)
      if (out[r * ld + c] != m[r * ld + c]) {
        std::printf("FAIL %s: (%d,%d) %04x -> %04x\n", what, r, c, m[r * ld + c], out[r * ld + c]);
        ++fails;
        return;
      }
}

int main() {
  std::mt19937 rng(1234);
  const size_t ld = 96;   // row stride wider than the tile: the encoder reads a tile out of a larger matrix
  std::vector<uint16_t> m(wp::ROWS * ld);
  auto fill_normal = [&](float sigma) {
    std::normal_distribution<float> nd(0.f, sigma);
    for (auto& v : m) v = to_bf16(nd(rng));
  };
  auto fill_window = [&]() {   // normal values with exponents 110..120: nothing below the window
    for (auto& v : m) v = (uint16_t)(((rng() & 1) << 15) | ((110 + rng() % 11) << 7) | (rng() & 0x7f));
  };
  // random N(0, sigma) tiles
  for (float sigma : {0.02f, 1e-3f, 0.3f, 5.0f, 1e-30f, 1000.f})
    for (int rep = 0; rep < 20; ++rep) {
      fill_normal(sigma);
      check("normal", m, ld, -1);
    }
  // every lane position patched once in turn: the patch list addresses each value of the fragment order
  for (int pos = 0; pos < wp::LANES * wp::VALS; pos += 97) {
    fill_window();
    int row, col;
    wp::lane_coord(pos / wp::VALS, pos % wp::VALS, &row, &col);
    m[row * ld + col] = 0x0001;   // smallest subnormal: below every window
    check("one patch", m, ld, 1);
  }
  // +-0 and subnormals
  fill_window();
  for (size_t i = 0; i < m.size(); i += 3) m[i] = (i & 1) ? 0x8000 : 0x0000;
  check("signed zeros", m, ld, 1);
  std::vector<uint16_t> z(m.size(), 0);
  check("all zero", z, ld, 1);
  for (size_t i = 0; i < z.size(); ++i) z[i] = (i % 5 == 0) ? 0x8000 : 0;
  check("all +-0", z, ld, 1);
  for (int n : {1, 7, 16, 17, 40}) {
    fill_window();
    for (int i = 0; i < n; ++i) m[(i * 37 % wp::ROWS) * ld + (i * 11 % wp::COLS)] = (uint16_t)(0x0001 + i + ((i & 1) << 15));
    check(n <= 16 ? "subnormal patches" : "too many subnormals", m, ld, n <= 16 ? 1 : 0);
  }
  // exactly 16 and 17 values below the window of normal values
  for (int n : {16, 17}) {
    fill_normal(0.02f);
    for (int c = 0; c < wp::COLS; ++c) m[c] = to_bf16(0.5f);          // window top: exponent 126 -> base 112
    for (int i = 0; i < n; ++i) m[(1 + i) * ld + 3] = to_bf16(-1e-6f * (1 + i));   // exponents < 112
    for (int r = 1 + n; r < wp::ROWS; ++r)
      for (int c = 0; c < wp::COLS; ++c)
        if (wp::bf16_exp(m[r * ld + c]) < 112) m[r * ld + c] = to_bf16(0.01f);
    for (int r = 1; r < 1 + n; ++r)
      for (int c = 0; c < wp::COLS; ++c)
        if (c != 3 && wp::bf16_exp(m[r * ld + c]) < 112) m[r * ld + c] = to_bf16(0.01f);
    check(n == 16 ? "16 patches" : "17 patches", m, ld, n == 16 ? 1 : 0);
  }
  // Inf / NaN: raw
  for (uint16_t special : {(uint16_t)0x7f80, (uint16_t)0xff80, (uint16_t)0x7fc0, (uint16_t)0xffff}) {
    fill_normal(0.02f);
    m[17 * ld + 5] = special;
    check("inf/nan", m, ld, 0);
  }
  // windows across the whole exponent range, with values at both ends of each window
  for (int top = 0; top <= 254; ++top) {
    for (size_t i = 0; i < m.size(); ++i) {
      const int e = top - (int)(rng() % 15);
      const uint16_t mant = (uint16_t)(rng() & 0x7f);
      m[i] = (uint16_t)(((rng() & 1) << 15) | ((e > 0 ? e : 0) << 7) | (e > 0 ? mant : 0));
    }
    m[3] = (uint16_t)(top << 7);
    check("exponent range", m, ld, wp::window_base(top) <= wp::MAX_BASE ? 1 : 0);
  }
  // random bit patterns: raw or exact, never wrong
  for (int rep = 0; rep < 50; ++rep) {
    for (auto& v : m) v = (uint16_t)rng();
    check("random bits", m, ld, -1);
  }
  if (fails) return 1;
  std::printf("OK coded=%d raw=%d\n", coded, raw);
  return 0;
}
