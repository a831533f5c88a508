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
};

struct TileInfo {
  int z;        // K1: group g ; K2: level l
  int m_blk, n_blk;
  int num_kb;   // K blocks of 64
};

template <int MODE>
__host__ __device__ __forceinline__ TileInfo decode_tile(const GemmParams& p, int tile) {
  TileInfo t;
  t.n_blk = tile % p.num_n;
  const int r = tile / p.num_n;
  t.m_blk = r % p.num_m;
  t.z = p.z0 + r / p.num_m;
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

}  // namespace glom
