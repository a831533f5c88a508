// Host enumeration of the persistent GEMM's tile schedule (gemm_sched.cuh), compiled from the same source as the
// kernels.  For every pair count C = 1..66 and the tile counts of L = 2..8 levels, num_n in {1..5, 8, 16} N tiles and
// num_m = 1..40 row blocks it walks each pair's list as gemm_kernel does (pairs = min(tiles, C), as launch_gemm_impl
// launches) and checks:
//   K2 (MODE 1): every tile dealt exactly once; the half-cost tiles are exactly the top level's (decode_tile gives them
//                K = 4d); the per-pair cost (full tile = 2, half = 1) differs by at most 2 between pairs;
//   K1 (MODE 0): every tile dealt exactly once, from group z0 = 0 and z0 = 1 (the later steps), each pair's count
//                within one of the others'.
// Prints one line "configs <n> failures <f> worst_k2_spread <s> worst_k1_spread <s>" and the first failures.
#include "gemm_sched.cuh"

#include <stdio.h>

#include <vector>

using glom::GemmParams;

static int failures = 0;

static void fail(const char* what, int C, int L, int nn, int nm) {
  if (++failures <= 10) printf("FAIL %s C=%d L=%d num_n=%d num_m=%d\n", what, C, L, nn, nm);
}

int main() {
  const int num_ns[] = {1, 2, 3, 4, 5, 8, 16};
  long configs = 0;
  int worst2 = 0, worst1 = 0;
  std::vector<int> seen;
  for (int C = 1; C <= 66; ++C)
    for (int L = 2; L <= 8; ++L)
      for (int nn : num_ns)
        for (int nm = 1; nm <= 40; ++nm) {
          ++configs;
          const int d = 256;
          // ---- K2: all L levels, the top level's num_m * num_n tiles last and half cost
          GemmParams p{};
          p.d = d; p.L = L; p.num_m = nm; p.num_n = nn; p.z0 = 0;
          p.num_tiles = L * nm * nn; p.n_half = nm * nn;
          int pairs = p.num_tiles < C ? p.num_tiles : C;
          seen.assign(p.num_tiles, 0);
          int lo = 1 << 30, hi = 0;
          for (int c = 0; c < pairs; ++c) {
            int cost = 0;
            for (int it = 0, tile; (tile = glom::sched_tile<1>(p, c, pairs, it)) >= 0; ++it) {
              if (tile >= p.num_tiles) { fail("k2 tile out of range", C, L, nn, nm); break; }
              ++seen[tile];
              const glom::TileInfo t = glom::decode_tile<1>(p, tile);
              const bool half = tile >= p.num_tiles - p.n_half;
              if (half != (t.z == L - 1) || t.num_kb != (half ? 4 : 8) * d / glom::BK)
                fail("k2 half-cost tile is not the top level's", C, L, nn, nm);
              cost += half ? 1 : 2;
            }
            lo = cost < lo ? cost : lo;
            hi = cost > hi ? cost : hi;
          }
          for (int v : seen) if (v != 1) { fail("k2 tile not dealt exactly once", C, L, nn, nm); break; }
          if (hi - lo > 2) fail("k2 cost spread > 2", C, L, nn, nm);
          worst2 = hi - lo > worst2 ? hi - lo : worst2;
          // ---- K1: groups z0 .. 2L-2
          for (int z0 = 0; z0 <= 1; ++z0) {
            GemmParams q{};
            q.d = d; q.L = L; q.num_m = nm; q.num_n = 4 * nn; q.z0 = z0;
            q.num_tiles = (2 * L - 1 - z0) * nm * q.num_n;
            pairs = q.num_tiles < C ? q.num_tiles : C;
            seen.assign(q.num_tiles, 0);
            lo = 1 << 30; hi = 0;
            for (int c = 0; c < pairs; ++c) {
              int cnt = 0;
              for (int it = 0, tile; (tile = glom::sched_tile<0>(q, c, pairs, it)) >= 0; ++it) {
                if (tile >= q.num_tiles) { fail("k1 tile out of range", C, L, nn, nm); break; }
                ++seen[tile];
                const glom::TileInfo t = glom::decode_tile<0>(q, tile);
                if (t.z < z0 || t.z >= 2 * L - 1) fail("k1 group out of range", C, L, nn, nm);
                ++cnt;
              }
              lo = cnt < lo ? cnt : lo;
              hi = cnt > hi ? cnt : hi;
            }
            for (int v : seen) if (v != 1) { fail("k1 tile not dealt exactly once", C, L, nn, nm); break; }
            if (hi - lo > 1) fail("k1 count spread > 1", C, L, nn, nm);
            worst1 = hi - lo > worst1 ? hi - lo : worst1;
          }
        }
  printf("configs %ld failures %d worst_k2_spread %d worst_k1_spread %d\n", configs, failures, worst2, worst1);
  return failures ? 1 : 0;
}
