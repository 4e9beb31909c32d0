// Host side of the int4 weight format (moe-infinity_b200/csrc/int4_weights.cuh): prints the header's dequantisation of every
// (code q, zero point z) pair under each scale given on the command line (bf16 bit patterns in hex), one line per scale:
//   <scale bits> <bf16 bits of (q=0,z=0)> <(q=0,z=1)> ... <(q=15,z=15)>        (pair index q * 16 + z)
// tests/test_int4_weights.py compares the table with torch's (s.float() * (q.float() - z.float())).to(torch.bfloat16), and
// checks the slot layout helpers, the group-grid index and the swizzled tile offsets printed after it.
#include <cstdio>
#include <cstdlib>

#include "int4_weights.cuh"

int main(int argc, char** argv) {
  using namespace b2m::i4;
  for (int i = 1; i < argc; ++i) {
    const uint16_t bits = (uint16_t)strtoul(argv[i], nullptr, 16);
    printf("%04x", bits);
    for (int q = 0; q < 16; ++q)
      for (int z = 0; z < 16; ++z) printf(" %04x", dequant((uint32_t)q, (uint32_t)z, bits));
    printf("\n");
  }
  // layout: blob sizes of the Mixtral-8x7B, DeepSeek-V2-Lite and Mixtral-8x22B experts, then the part offsets of one expert
  printf("blob %zu %zu %zu\n", expert_blob_bytes(4096, 14336), expert_blob_bytes(2048, 1408), expert_blob_bytes(6144, 16384));
  printf("parts");
  for (int m = 0; m < 3; ++m) printf(" %zu %zu", code_offset(2048, 1408, m), grid_offset(2048, 1408, m));
  printf("\n");
  // a few group-grid indices of a [384 x 512] matrix (rows, groups of 128 columns): (r, g) -> word index
  printf("grid");
  const int rg[][2] = {{0, 0}, {1, 0}, {127, 0}, {0, 1}, {127, 3}, {128, 0}, {200, 2}, {383, 3}};
  for (const auto& p : rg) printf(" %zu", grid_index(p[0], p[1], 512));
  printf("\n");
  // the swizzled tile is a permutation that keeps every row in its own 32 bytes
  static int seen[TILE_BYTES];
  int ok = 1;
  for (int r = 0; r < ROWS; ++r)
    for (int b = 0; b < ROW_BYTES; ++b) {
      const uint32_t o = tile_offset(r, b);
      if (o >= (uint32_t)TILE_BYTES || seen[o]++) ok = 0;
      if (o / ROW_BYTES != (uint32_t)r) ok = 0;
    }
  printf("tile %s\n", ok ? "ok" : "bad");
  return 0;
}
