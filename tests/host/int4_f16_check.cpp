// Host side of the int4 weight format with fp16 scales (B2M_WEIGHTS_INT4_G128_F16, moe-infinity_b200/csrc/int4_weights.cuh):
// prints the header's f16 dequantisation of every (code q, zero point z) pair under each scale given on the command line
// (fp16 bit patterns in hex), one line per scale:
//   <scale bits> <f16 bits of (q=0,z=0)> <(q=0,z=1)> ... <(q=15,z=15)>        (pair index q * 16 + z)
// tests/test_int4_f16_weights.py compares the table with torch's (s.float() * (q.float() - z.float())).to(torch.float16).
#include <cstdio>
#include <cstdlib>

#include "int4_weights.cuh"

int main(int argc, char** argv) {
  using namespace b2m::i4;
  for (int i = 1; i < argc; ++i) {
    const uint16_t bits = (uint16_t)strtoul(argv[i], nullptr, 16);
    printf("%04x", bits);
    for (int q = 0; q < 16; ++q)
      for (int z = 0; z < 16; ++z) printf(" %04x", dequant_f16((uint32_t)q, (uint32_t)z, bits));
    printf("\n");
  }
  return 0;
}
