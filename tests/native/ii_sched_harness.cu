// Host enumeration of the reduced schedules of a forward from init_levels (gemm_sched.cuh: decode_tile<MODE, true>,
// sched_tile, set_reduced, attn_item and the ii_* dependency rules), set up as step_bf16 sets up K1, K3 and K2 at the
// steps t < L it reduces.  For every pair count C = 1..66 (K3: CTA count 1..132) and the shapes below it checks that every
// required K1 / K2 tile and K3 item is dealt exactly once and nothing else is: groups / levels / K3 levels that differ
// between images over every row block (image), the others over the representative row blocks (image 0) only.
// Prints "configs <n> failures <f>", then the executed totals of configs[1] (d 512, L 6, n 256, B 32, iters 12):
// "c1 k1_tiles <x> <parent> k2_cost <x> <parent> k3_items <x> <parent>".
#include "gemm_sched.cuh"

#include <stdio.h>

#include <vector>

using glom::GemmParams;

static int failures = 0;

static void fail(const char* what, int C, int L, int n, int B, int t) {
  if (++failures <= 10) printf("FAIL %s C=%d L=%d n=%d B=%d t=%d\n", what, C, L, n, B, t);
}

// K1 (MODE 0) or K2 (MODE 1) of step t, as step_bf16 sets it up; reduced = false: the parent's launch
template <int MODE>
static GemmParams gemm_params(int d, int L, int n, int B, int t, bool reduced) {
  GemmParams p{};
  const int rows = B * n, G = 2 * L - 1;
  p.d = d; p.L = L; p.n = n; p.num_m = (rows + 255) / 256;
  if (MODE == 0) {
    p.z0 = (t > 0 && G > 1) ? 1 : 0;
    p.num_n = 4 * d / 256; p.num_tiles = (G - p.z0) * p.num_m * p.num_n;
    if (reduced) glom::set_reduced(p, G, glom::rep_row_blocks(n), [&](int z) { return glom::ii_k1_full(z, t); });
  } else {
    p.num_n = d / 256; p.num_tiles = L * p.num_m * p.num_n; p.n_half = p.num_m * p.num_n;
    if (reduced) {
      glom::set_reduced(p, L, glom::rep_row_blocks(n), [&](int l) { return glom::ii_k2_full(l, t); });
      p.n_half = (L - 1 <= t ? p.num_m : p.num_m_rep) * p.num_n;
    }
  }
  return p;
}

// every pair's list; -> executed tiles (K1) or cost units (K2: full 2, top level 1)
template <int MODE>
static long check_gemm(const GemmParams& p, int C, int G_or_L, int t, int L, int n, int B) {
  const int pairs = p.num_tiles < C ? p.num_tiles : C;
  std::vector<int> seen((size_t)G_or_L * p.num_m * p.num_n, 0);
  long work = 0;
  for (int c = 0; c < pairs; ++c)
    for (int it = 0, tile; (tile = glom::sched_tile<MODE>(p, c, pairs, it)) >= 0; ++it) {
      if (tile >= p.num_tiles) { fail("tile out of range", C, L, n, B, t); return work; }
      const glom::TileInfo ti = glom::decode_tile<MODE, true>(p, tile);
      if (ti.z < p.z0 || ti.z >= G_or_L || ti.m_blk >= p.num_m || ti.n_blk >= p.num_n) { fail("bad tile", C, L, n, B, t); return work; }
      ++seen[((size_t)ti.z * p.num_m + ti.m_blk) * p.num_n + ti.n_blk];
      const bool half = MODE == 1 && tile >= p.num_tiles - p.n_half;
      if (MODE == 1 && (half != (ti.z == L - 1) || ti.num_kb != (half ? 4 : 8) * p.d / glom::BK))
        fail("k2 half-cost tile is not the top level's", C, L, n, B, t);
      work += MODE == 1 ? (half ? 1 : 2) : 1;
    }
  const int nrep = glom::rep_row_blocks(n);
  for (int z = 0; z < G_or_L; ++z)
    for (int m = 0; m < p.num_m; ++m) {
      const bool full = MODE == 0 ? glom::ii_k1_full(z, t) : glom::ii_k2_full(z, t);
      const int want = (z >= p.z0 && (full || m < nrep)) ? 1 : 0;
      for (int nb = 0; nb < p.num_n; ++nb)
        if (seen[((size_t)z * p.num_m + m) * p.num_n + nb] != want) { fail(MODE ? "k2 coverage" : "k1 coverage", C, L, n, B, t); return work; }
    }
  return work;
}

// K3 items of step t as launch_attention enumerates them (reduced: l_full = ii_k3_full_levels(t)) over `ctas` CTAs
static long check_attn(int L, int n, int B, int t, int ctas, bool reduced) {
  const int ntiles = (n + 127) / 128, l_full = reduced ? glom::ii_k3_full_levels(t) : L;
  const int num_items = ntiles * (l_full * B + L - l_full);
  const int full_items = num_items - ntiles * (L - l_full), per_img = ntiles * l_full;
  std::vector<int> seen((size_t)B * L * ntiles, 0);
  for (int c = 0; c < ctas && c < num_items; ++c)
    for (int it = c; it < num_items; it += ctas) {
      int b, l;
      glom::attn_item(it, full_items, per_img, ntiles, l_full, b, l);
      if (b < 0 || b >= B || l < 0 || l >= L) { fail("k3 bad item", ctas, L, n, B, t); return num_items; }
      ++seen[((size_t)b * L + l) * ntiles + it % ntiles];
    }
  for (int b = 0; b < B; ++b)
    for (int l = 0; l < L; ++l)
      for (int q = 0; q < ntiles; ++q)
        if (seen[((size_t)b * L + l) * ntiles + q] != ((l < l_full || b == 0) ? 1 : 0)) { fail("k3 coverage", ctas, L, n, B, t); return num_items; }
  return num_items;
}

int main() {
  const int ns[] = {1, 36, 64, 128, 144, 256, 576, 784};
  const int Bs[] = {2, 3, 8, 32};
  const int ds[] = {256, 512};
  long configs = 0;
  for (int L = 2; L <= 8; ++L)
    for (int n : ns)
      for (int B : Bs)
        for (int d : ds) {
          if (glom::rep_row_blocks(n) >= (B * n + 255) / 256) continue;     // not eligible: the forward runs in full
          for (int t = 0; t < L; ++t) {
            const GemmParams k1 = gemm_params<0>(d, L, n, B, t, true), k2 = gemm_params<1>(d, L, n, B, t, true);
            for (int C = 1; C <= 66; ++C) {
              ++configs;
              check_gemm<0>(k1, C, 2 * L - 1, t, L, n, B);
              check_gemm<1>(k2, C, L, t, L, n, B);
              check_attn(L, n, B, t, 2 * C, true);
              check_attn(L, n, B, t, 2 * C - 1, true);
            }
          }
        }
  printf("configs %ld failures %d\n", configs, failures);
  // configs[1], 12 steps on 66 pairs / 132 SMs: executed against the parent's full launches
  long k1 = 0, k1p = 0, k2 = 0, k2p = 0, k3 = 0, k3p = 0;
  for (int t = 0; t < 12; ++t) {
    const bool red = t < 6;
    k1 += check_gemm<0>(gemm_params<0>(512, 6, 256, 32, t, red), 66, 11, red ? t : 99, 6, 256, 32);
    k1p += gemm_params<0>(512, 6, 256, 32, t, false).num_tiles;
    k2 += check_gemm<1>(gemm_params<1>(512, 6, 256, 32, t, red), 66, 6, red ? t : 99, 6, 256, 32);
    k2p += 2 * (5 * 32 * 2) + 32 * 2;
    k3 += check_attn(6, 256, 32, red ? t : 99, 132, red);
    k3p += 2 * 6 * 32;
  }
  printf("c1 k1_tiles %ld %ld k2_cost %ld %ld k3_items %ld %ld\n", k1, k1p, k2, k2p, k3, k3p);
  return failures ? 1 : 0;
}
