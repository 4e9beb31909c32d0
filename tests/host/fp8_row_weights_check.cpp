// Host side of the row-scaled fp8 weight format (moe-infinity_b200/csrc/fp8_weights.cuh, B2M_WEIGHTS_FP8_E4M3_ROW): decodes
// one e4m3 matrix with a row per scale given on the command line (fp32 bit patterns in hex), every row holding the 256
// codes in order, through the header's per-row decode, and prints one line per row:
//   <scale bits> <bf16 bits of code 0> ... <bf16 bits of code 255>
// tests/test_fp8_row_weights.py compares the table with torch's (q.float() * s[:, None]).to(torch.bfloat16), and checks the
// blob sizes printed after it.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "fp8_weights.cuh"

int main(int argc, char** argv) {
  using namespace b2m::f8;
  const int rows = argc - 1, cols = 256;
  std::vector<uint8_t> q((size_t)rows * cols);
  std::vector<float> s(rows);
  std::vector<uint16_t> w((size_t)rows * cols);
  std::vector<uint32_t> bits(rows);
  for (int r = 0; r < rows; ++r) {
    bits[r] = (uint32_t)strtoul(argv[r + 1], nullptr, 16);
    memcpy(&s[r], &bits[r], 4);
    for (int c = 0; c < cols; ++c) q[(size_t)r * cols + c] = (uint8_t)c;
  }
  dequant_rows(q.data(), s.data(), rows, cols, w.data());
  for (int r = 0; r < rows; ++r) {
    printf("%08x", bits[r]);
    for (int c = 0; c < cols; ++c) printf(" %04x", w[(size_t)r * cols + c]);
    printf("\n");
  }
  // blob sizes of a Mixtral-8x7B, a Llama 4 Maverick and a DeepSeek-V2-Lite expert, and one scale vector
  printf("blob %zu %zu %zu\n", row_expert_blob_bytes(4096, 14336), row_expert_blob_bytes(5120, 8192),
         row_expert_blob_bytes(2048, 1408));
  printf("vector %zu\n", row_scale_bytes(14336, 4096));
  return 0;
}
