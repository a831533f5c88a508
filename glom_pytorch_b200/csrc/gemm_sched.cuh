// The persistent grouped GEMM's launch parameters and its static tile schedule (K1, K2, the tokeniser).
// decode_tile / sched_tile are __host__ __device__ so that a host program can enumerate the schedule for any pair
// count (tests/native/sched_tile_harness.cu): a GPU run only exercises the pair count of the card it runs on.
#pragma once
#include "tc_common.cuh"

namespace glom {

struct GemmParams {
  int rows, d, L, n, G;
  int num_m, num_n, num_tiles;       // num_m counts 256-row pair tiles
  int m128;                          // 128-row blocks of the (padded) hidden buffer H
  int z0;                            // first MLP group (K1) / level (K2) of this launch, see level batching below
  int n_half;                        // K2: number of half-cost (top-level) tiles in this launch
  const float* bias;
  // K2
  const float* s32_in;
  int s_bcast;                       // s32_in = init_levels broadcast (see K2Chunk)
  const __nv_bfloat16* c_in;
  const float* pos;
  float* s32_out;
  __nv_bfloat16* sb_out;
  __nv_bfloat16* sp_out;
  float* nsq_out;
  int nparts;
  // tokeniser (MODE 2)
  float* tok_out;
  int tok_kb;      // K blocks of 64 of the zero-padded patch dimension
  // SETTLE instantiations (Glom.settle), flags written by the convergence kernel of the previous step
  const int* frozen;        // [B] 1: the image has stopped
  const int* block_frozen;  // [num_m] 1: every row of the 256-row block belongs to a stopped image
  float* dsq_out;           // K2: squared-change partials |S_{t+1} - S_t|^2, laid out like nsq_out
  // K1 of the settle queue (NULL otherwise): [num_m] 1 = the 256-row block holds a slot admitted at this step.  The
  // launch covers group 0 (z0 = 0) at every step, and only the blocks marked here run its tiles
  const int* block_fresh;
  // Image-independent work of a forward from init_levels (DESIGN.md, "Image-independent levels"); num_m_rep = 0: off.
  // The groups (K1) / levels (K2) of full_mask run all num_m row blocks, those of rep_mask only the first num_m_rep: the
  // representative rows, whose values every image shares.  full_mask's num_full_tiles tiles come first, each mask's
  // groups in increasing order.
  int num_m_rep, num_full_tiles;
  unsigned long long full_mask, rep_mask;
  // K2: levels l >= remap_l read S_t and C from row r mod n, and levels l >= remap_l - 1 read their top-down H from
  // 128-row block k mod h_period (the representative block holding the same patches)
  int remap_l, h_period;
};

struct TileInfo {
  int z;        // K1: group g ; K2: level l
  int m_blk, n_blk;
  int num_kb;   // K blocks of 64
};

// index of the k-th set bit of m (m has more than k set bits)
__host__ __device__ __forceinline__ int nth_set_bit(unsigned long long m, int k) {
  int z = 0;
  for (;; ++z)
    if ((m >> z) & 1ull) { if (k == 0) return z; --k; }
}

// REDUCED: the instantiation that honours num_m_rep (the default K1 and K2 builds)
template <int MODE, bool REDUCED = false>
__host__ __device__ __forceinline__ TileInfo decode_tile(const GemmParams& p, int tile) {
  TileInfo t;
  if (REDUCED && p.num_m_rep > 0) {
    const bool full = tile < p.num_full_tiles;
    const int nm = full ? p.num_m : p.num_m_rep;
    const int r = full ? tile / p.num_n : (tile - p.num_full_tiles) / p.num_n;
    t.n_blk = tile % p.num_n;              // num_full_tiles is a multiple of num_n
    t.m_blk = r % nm;
    t.z = nth_set_bit(full ? p.full_mask : p.rep_mask, r / nm);
  } else {
    t.n_blk = tile % p.num_n;
    const int r = tile / p.num_n;
    t.m_blk = r % p.num_m;
    t.z = p.z0 + r / p.num_m;
  }
  if (MODE == 0) t.num_kb = p.d / BK;
  else if (MODE == 1) t.num_kb = ((t.z == p.L - 1) ? 4 * p.d : 8 * p.d) / BK;   // top level: no top-down half (:137)
  else t.num_kb = p.tok_kb;
  return t;
}

// Static tile schedule of pair `c` (of `C`): the it-th tile it processes, or -1 when done.
//   K1 / tokeniser: uniform tiles, plain round-robin.
//   K2: the top level's tiles cost half (K = 4d instead of 8d, :137).  Full-cost tiles are dealt round-robin
//   first; the half-cost ones then go to the pairs that received one full tile fewer (up to two each, which
//   levels them with the others) and only after that round-robin over everybody.  Closed form, so every warp
//   role of both CTAs walks the same list without communication.
template <int MODE>
__host__ __device__ __forceinline__ int sched_tile(const GemmParams& p, int c, int C, int it) {
  if (MODE != 1) { const int t = c + it * C; return t < p.num_tiles ? t : -1; }
  const int S = p.n_half;                     // half-cost tiles (top level, last in the launch), ids [B, B + S)
  const int B = p.num_tiles - S;              // full-cost tiles, ids [0, B)
  const int heavy = B % C;                    // pairs [0, heavy) hold one more full tile than the rest
  const int nb = (B - c + C - 1) / C;         // full tiles of this pair (B - c may be <= 0)
  const int nbig = nb > 0 ? nb : 0;
  if (it < nbig) return c + it * C;
  int k = it - nbig;                          // k-th half-cost tile of this pair
  const int light = C - heavy;
  const int first = (2 * light < S) ? 2 * light : S;     // half tiles dealt to the light pairs first
  if (c >= heavy) {
    if (k < 2) { const int j = k * light + (c - heavy); if (j < first) return B + j; }
    k -= 2;
    if (k < 0) return -1;
  }
  const int j = first + k * C + c;            // the rest: round-robin over all pairs
  return j < S ? B + j : -1;
}

// ---- Image-independent work at step t of a forward from init_levels (DESIGN.md, "Image-independent levels").  S_t[k]
// differs between images only for k <= t - 1, so the work below runs for every row block only where its input does.
// K1 group z: bottom-up l (z = 2l) reads S_t[l-1] (group 0: the tokens), top-down l (z = 2l + 1) reads S_t[l+1]
__host__ __device__ __forceinline__ bool ii_k1_full(int z, int t) { return (z & 1) ? z <= 2 * t - 3 : z <= 2 * t; }
// K2 level l writes S_{t+1}[l]
__host__ __device__ __forceinline__ bool ii_k2_full(int l, int t) { return l <= t; }
// K3 level l reads S_t[l]: levels [0, ii_k3_full_levels) run for every image, the others for image 0 only
__host__ __device__ __forceinline__ int ii_k3_full_levels(int t) { return t; }

// The groups / levels z in [p.z0, z_end) with full(z) run every row block, the others the num_m_rep representative ones.
// Sets the masks and the tile counts (p.num_m, p.num_n and p.z0 set)
template <typename Full>
__host__ __forceinline__ void set_reduced(GemmParams& p, int z_end, int num_m_rep, Full full) {
  p.num_m_rep = num_m_rep;
  p.full_mask = p.rep_mask = 0;
  for (int z = p.z0; z < z_end; ++z) (full(z) ? p.full_mask : p.rep_mask) |= 1ull << z;
  p.num_full_tiles = __builtin_popcountll(p.full_mask) * p.num_m * p.num_n;
  p.num_tiles = p.num_full_tiles + __builtin_popcountll(p.rep_mask) * num_m_rep * p.num_n;
}

// K3 (attn_kernel) item -> (image b, level l): the full_items = B * per_img items of levels [0, l_full) of every image,
// image-major (per_img = ntiles * l_full), then levels [l_full, L) of image 0
__host__ __device__ __forceinline__ void attn_item(int it, int full_items, int per_img, int ntiles, int l_full, int& b, int& l) {
  if (it >= full_items) { b = 0; l = l_full + (it - full_items) / ntiles; }
  else { b = it / per_img; l = (it % per_img) / ntiles; }
}

}  // namespace glom
