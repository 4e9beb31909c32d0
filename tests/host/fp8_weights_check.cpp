// Host side of the fp8 weight format (moe-infinity_b200/csrc/fp8_weights.cuh): prints the header's dequantisation of every
// e4m3 code under each scale given on the command line (fp32 bit patterns in hex), one line per scale:
//   <scale bits> <bf16 bits of code 0> ... <bf16 bits of code 255>
// tests/test_fp8_weights.py compares the table with torch's (w_q.float() * s).to(torch.bfloat16), and checks the slot layout
// helpers and the swizzled tile offsets printed after it.
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "fp8_weights.cuh"

int main(int argc, char** argv) {
  using namespace b2m::f8;
  for (int i = 1; i < argc; ++i) {
    const uint32_t bits = (uint32_t)strtoul(argv[i], nullptr, 16);
    float s;
    memcpy(&s, &bits, 4);
    printf("%08x", bits);
    for (int c = 0; c < 256; ++c) printf(" %04x", dequant((uint8_t)c, s));
    printf("\n");
  }
  // layout: blob sizes of the Mixtral and DeepSeek-V2-Lite experts, scale-grid offsets, and the swizzled tile is a permutation
  printf("blob %zu %zu\n", expert_blob_bytes(4096, 14336), expert_blob_bytes(2048, 1408));
  printf("grid %zu %zu %zu\n", scale_grid_offset(2048, 1408, 0), scale_grid_offset(2048, 1408, (size_t)2048 * 1408),
         scale_grid_offset(2048, 1408, (size_t)2 * 2048 * 1408));
  static int seen[TILE_BYTES];
  int ok = 1;
  for (int r = 0; r < ROWS; ++r)
    for (int c = 0; c < COLS; ++c) {
      const uint32_t o = tile_offset(r, c);
      if (o >= (uint32_t)TILE_BYTES || seen[o]++) ok = 0;
      if (o / ROW_BYTES != (uint32_t)r) ok = 0;                  // SWIZZLE_64B permutes 16-B chunks inside a row
    }
  printf("tile %s\n", ok ? "ok" : "bad");
  return 0;
}
