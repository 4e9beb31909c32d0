// Host-side exhaustive check of the persistent grouped GEMM's tile scheduling (csrc/tile_walker.cuh), compiled with g++ by
// tests/test_tile_walker.py.  For seeded random routing tables it replays every CTA's walk exactly as the kernel does
// (grouped_gemm.cu: tile_start table, tile0/tile_stride, stream-K ranges) and demands that every (expert, weight-row
// tile, token tile, k-block) unit of every activated, resident expert is processed exactly once -- for the fixed
// split-K factor, the stream-K partition and the 2-CTA cluster (multicast) variant.
#include <cstdio>
#include <cstdlib>
#include <map>
#include <random>
#include <tuple>
#include <vector>

#include "tile_walker.cuh"

using namespace b2m;

struct Case {
  int E, NT, MC, ksplit, stream, kblocks, m_tiles, m_step, grid;
  std::vector<int> offs, slots;
};

static int check(const Case& c, unsigned long long id) {
  const int E = c.E;
  std::vector<int> tile_start(E + 1);
  int acc = 0;
  for (int e = 0; e < E; ++e) {   // grouped_gemm.cu, thread 0 after the routing tables are staged in shared memory
    tile_start[e] = acc;
    const int n_e = c.offs[e + 1] - c.offs[e];
    if (n_e > 0 && c.slots[e] >= 0) acc += c.m_tiles * (((n_e + c.NT - 1) / c.NT + c.MC - 1) / c.MC) * (c.stream ? 1 : c.ksplit);
  }
  tile_start[E] = acc;
  std::map<std::tuple<int, int, int, int>, int> seen;   // (e, m0, n, kb) -> times processed
  long long ghost = 0;
  for (int b = 0; b < c.grid; ++b) {
    const int crank = c.MC > 1 ? b % c.MC : 0;
    TileWalker w{tile_start.data(), c.offs.data(), c.slots.data(), E, c.NT, c.stream ? 1 : c.ksplit, c.kblocks, 0, c.m_step,
                 c.MC, crank, 0, 0, 0};
    if (c.MC == 1 && c.stream) {
      const long long units = (long long)tile_start[E] * c.kblocks;
      w.stream = 1;
      w.u_cur = (int)(units * b / c.grid);
      w.u_end = (int)(units * (b + 1) / c.grid);
    }
    const int tile0 = b / c.MC, stride = c.grid / c.MC;
    TileInfo t;
    long long guard = 0;
    for (int tile = tile0; w.get(tile, t); tile += stride) {
      if (++guard > 10000000) { std::printf("case %llu: walk does not terminate\n", id); return 1; }
      if (t.slot != c.slots[t.e] || t.slot < 0) { std::printf("case %llu: wrong slot\n", id); return 1; }
      if (t.kb_begin >= t.kb_end || t.kb_begin < 0 || t.kb_end > c.kblocks) { std::printf("case %llu: empty/out-of-range k range [%d,%d)\n", id, t.kb_begin, t.kb_end); return 1; }
      if (t.m0 % c.m_step || t.m0 / c.m_step >= c.m_tiles) { std::printf("case %llu: bad m0\n", id); return 1; }
      if (t.ncols == 0) { if (c.MC == 1) { std::printf("case %llu: ghost tile without clusters\n", id); return 1; } ++ghost; continue; }
      const int rel = t.row0 - c.offs[t.e];
      if (rel < 0 || rel % c.NT || t.row0 + t.ncols > c.offs[t.e + 1] || t.ncols > c.NT) { std::printf("case %llu: bad token tile\n", id); return 1; }
      if (t.row0 + t.ncols < c.offs[t.e + 1] && t.ncols != c.NT) { std::printf("case %llu: short inner token tile\n", id); return 1; }
      for (int kb = t.kb_begin; kb < t.kb_end; ++kb) ++seen[{t.e, t.m0, rel / c.NT, kb}];
    }
  }
  long long expect = 0;
  for (int e = 0; e < E; ++e) {
    const int n_e = c.offs[e + 1] - c.offs[e];
    if (n_e <= 0 || c.slots[e] < 0) continue;
    const int n_tiles = (n_e + c.NT - 1) / c.NT;
    for (int m = 0; m < c.m_tiles; ++m)
      for (int n = 0; n < n_tiles; ++n)
        for (int kb = 0; kb < c.kblocks; ++kb) {
          ++expect;
          auto it = seen.find({e, m * c.m_step, n, kb});
          if (it == seen.end() || it->second != 1) {
            std::printf("case %llu: unit (e=%d m=%d n=%d kb=%d) processed %d times (E=%d NT=%d MC=%d ksplit=%d stream=%d kblocks=%d grid=%d)\n",
                        id, e, m, n, kb, it == seen.end() ? 0 : it->second, E, c.NT, c.MC, c.ksplit, c.stream, c.kblocks, c.grid);
            return 1;
          }
        }
  }
  if ((long long)seen.size() != expect) { std::printf("case %llu: %zu units processed, %lld expected\n", id, seen.size(), expect); return 1; }
  return 0;
}

int main(int argc, char** argv) {
  const int ncases = argc > 1 ? std::atoi(argv[1]) : 2000;
  std::mt19937_64 rng(12345);
  auto U = [&](int lo, int hi) { return (int)(lo + rng() % (unsigned long long)(hi - lo + 1)); };
  long long units = 0;
  for (int i = 0; i < ncases; ++i) {
    Case c;
    static const int nts[] = {16, 32, 64, 128, 256};
    c.E = U(1, 24);
    c.NT = nts[U(0, 4)];
    c.MC = (c.NT == 128 && U(0, 3) == 0) ? 2 : 1;
    c.kblocks = U(1, 40);
    c.m_step = U(0, 1) ? 256 : 128;                      // dual_m pairs two 128-row tiles
    c.m_tiles = U(1, 6);
    c.grid = U(0, 4) == 0 ? 132 : U(1, 40);
    if (c.MC == 2) c.grid = 2 * U(1, 20);
    // split-K factor as pick_ksplit (api.cu) produces it: every split non-empty
    c.ksplit = U(1, 8);
    while (c.ksplit > 1) {
      const int per = (c.kblocks + c.ksplit - 1) / c.ksplit;
      if ((c.ksplit - 1) * per < c.kblocks) break;
      --c.ksplit;
    }
    c.stream = (c.MC == 1 && c.ksplit > 1) ? U(0, 1) : 0;  // api.cu: stream_k only with ksplit > 1 and no cluster
    c.offs.assign(c.E + 1, 0);
    c.slots.assign(c.E, 0);
    for (int e = 0; e < c.E; ++e) {
      const int kind = U(0, 5);
      const int n = kind == 0 ? 0 : (kind < 4 ? U(1, 40) : U(1, 700));
      c.offs[e + 1] = c.offs[e] + n;
      c.slots[e] = U(0, 9) == 0 ? -1 : U(0, 300);         // -1: not resident in this wave -> skipped
    }
    if (check(c, i)) return 1;
    units += c.offs[c.E];
  }
  std::printf("OK %d cases, %lld routed rows\n", ncases, units);
  return 0;
}
