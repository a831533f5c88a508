// Merged persistent MLP kernel of the GLOM column update for sm_90a (dim % 256 == 0).
//
//   mlp_kernel: one launch per Jacobi step runs BOTH grouped GEMMs of GroupedFeedForward for all levels
//     K1 tiles  H_g   = gelu_erf(A_g . W1_g^T + b1_g)                         (glom_pytorch.py:29-30, calls :134/:136)
//     K2 tiles  S'_l  = (S_l + C_l + [H_bu,l | H_td,l] . [W2bu_l | W2td_l]^T + b2_l) / c_l   (:31, :137, :141-142)
//   as 256 x 256 tiles of a cluster of two CTAs (each CTA computes 128 of the rows with the TMA + wgmma machinery of
//   gemm_kernel in tc_kernels.cu) drawn from ONE ordered work list by a dynamic scheduler, with per-(level, row block)
//   dependency counters in global memory:
//
//   * Work lists: two ordered lists, both level-major (top level last: its GEMM2 tiles cost half, which keeps the
//     tail short) and then by 256-row block: the K1 list (per row block: both MLP groups x 4d/256 column tiles) and the
//     K2 list (per row block: d/256 column tiles).  A K2 tile depends on the K1 tiles of its (level, row block).
//   * Scheduler (adaptive cluster roles): the leader CTA's TMA producer lane draws the next tile while it issues the last
//     loads of the current one.  It looks at the heads of both lists: `lag` = row blocks between the K1 head and the K2
//     head.  If the lag has reached a threshold and the K2 head's dependencies are complete, it takes the K2 head
//     (compare-and-swap on the K2 counter), else the next K1 tile (atomicAdd); once the K1 list is exhausted everybody
//     takes K2 tiles in order (their dependencies are claimed, running, and never wait themselves: no deadlock).  The
//     threshold is lower for a cluster whose previous tile was a K2 tile, so clusters keep their role for long stretches
//     while the NUMBER of clusters on each kind adapts to the two kinds' actual rates.  H is consumed a few row blocks
//     after it was written, while still in L2: the HBM round trip of H in the two-kernel path becomes L2 traffic plus
//     the eventual write-back.
//     The drawn tile is published through an 8-slot shared-memory ring to the consumer / publisher roles of BOTH
//     CTAs of the pair and to the peer's TMA lane (local store + mbarrier for its own CTA, st.async + complete_tx for
//     the peer).
//   * Dependencies: the 8 consumer warps of a CTA arrive on a shared-memory mbarrier once their stores of a tile are
//     issued; one publisher lane per CTA turns that into ONE gpu-scope release (red.release.gpu.add on
//     ready[level][row block]) per CTA and K1 tile, off the consumer warps' critical path (cumulativity: stores ->
//     warp barrier -> mbarrier arrive / wait -> release).  The TMA producers of a K2 tile wait (ld.acquire.gpu) for all
//     2 x (K1 tiles of the row block) arrivals and cross into the async proxy (fence.proxy.async.global) before their
//     first load of H.
#include "tc_common.cuh"

#include <stdlib.h>
#include <string.h>

namespace glom {

constexpr int MLP_BN = 256;
constexpr int MLP_STAGES = 3;
constexpr int MLP_CONSUMER_WARPS = 8;             // two warpgroups of 64 rows each: wgmma main loop + epilogue
constexpr int MLP_CTRL_WARPS = 2;                 // TMA (+ scheduler in the leader), publisher
constexpr int MLP_THREADS = 32 * (MLP_CONSUMER_WARPS + MLP_CTRL_WARPS);
constexpr int MLP_SLOTS = 8;                      // scheduler ring
constexpr uint32_t MLP_STAGE_BYTES = A_STAGE_BYTES + MLP_BN * BK * 2;     // 48 KB: A (128 x 64) + B (256 x 64)
constexpr uint32_t MLP_PATCH_BYTES = 4096;        // per-warp transpose patch (K2: 32 x 32 fp32; K1: 2 KB)
constexpr size_t MLP_SMEM_BYTES = 1024 + (size_t)MLP_STAGES * MLP_STAGE_BYTES + 4 * (size_t)STG_BYTES +
                                  (size_t)MLP_CONSUMER_WARPS * MLP_PATCH_BYTES + 4 * 32 * 4 + 512;
constexpr int MLP_SEMPTY_COUNT = (MLP_CONSUMER_WARPS + 1) + (MLP_CONSUMER_WARPS + 2);   // leader: consumers + publisher; peer: consumers + TMA + publisher
constexpr int MLP_MAX_LEVELS = 16;

__device__ unsigned long long g_mlp_clk[2];     // in-kernel clock sample (cycles, ns), see clock_sample_begin

struct MlpParams {
  int rows, d, L, n;
  int num_m;                 // 256-row pair tiles
  int nN1, nN2;              // column tiles of GEMM1 (4d / 256) and GEMM2 (d / 256)
  int m128;                  // 128-row blocks of the (padded) hidden buffer H
  int n1_tiles, n2_tiles;    // lengths of the K1 / K2 lists
  int lvl1_base[MLP_MAX_LEVELS + 1];    // first K1-list index of level l (the top level has one group, the others two)
  int lag_hi, lag_lo;        // row blocks the K1 head must lead the K2 head by before a cluster takes the K2 head:
                             // lag_hi after a K1 tile, lag_lo after a K2 tile (sticky roles)
  const float* b1;           // (G * 4d)
  const float* b2;           // (L * d)   b2bu + b2td
  __nv_bfloat16* h;
  const float* s32_in;  int s_bcast;  const __nv_bfloat16* c_in;  const float* pos;
  float* s32_out;  __nv_bfloat16* sb_out;  __nv_bfloat16* sp_out;  float* nsq_out;
  int nparts;
  int* counter;              // [2] heads of the K1 and K2 lists of this launch (zeroed by the caller)
  int* ready;                // [L * num_m] K1 arrivals per (level, row block) (zeroed by the caller)
  unsigned long long* dbg;   // DBG instantiation only: 16 cycle counters per CTA (GLOM_B200_MLP_DBG=1)
  int h_load_policy;         // L2 hint of the GEMM2 tiles' H loads: 0 = evict-first on the last column tile only, 1 = on all, 2 = none
  int h_store_policy;        // H stores: 0 = evict-last, 1 = default write-back policy
};

struct MlpTile {
  int kind;                  // 0 = K1 (GEMM1 + GELU -> H), 1 = K2 (GEMM2 + combine -> state t+1)
  int z;                     // K1: MLP group (2l = bottom-up l, 2l + 1 = top-down l); K2: level l
  int l, m_blk, n_blk, num_kb;
};

// i-th tile of the K1 list / j-th tile of the K2 list
__host__ __device__ __forceinline__ MlpTile mlp_decode1(const MlpParams& p, int i) {
  int l = 0;
  while (l + 1 < p.L && i >= p.lvl1_base[l + 1]) ++l;
  const int idx = i - p.lvl1_base[l];
  const int c1 = ((l == p.L - 1) ? 1 : 2) * p.nN1;      // the top level has no top-down group (:137)
  const int m = idx / c1, r = idx - m * c1;
  const int gi = r / p.nN1;
  MlpTile t;
  t.kind = 0; t.l = l; t.m_blk = m; t.z = 2 * l + gi; t.n_blk = r - gi * p.nN1; t.num_kb = p.d / BK;
  return t;
}
__host__ __device__ __forceinline__ MlpTile mlp_decode2(const MlpParams& p, int j) {
  const int per = p.num_m * p.nN2;
  const int l = j / per, r = j - l * per;
  MlpTile t;
  t.kind = 1; t.l = l; t.z = l; t.m_blk = r / p.nN2; t.n_blk = r - t.m_blk * p.nN2;
  t.num_kb = ((l == p.L - 1) ? 4 * p.d : 8 * p.d) / BK;
  return t;
}

// Ring entries are PACKED tile descriptors (decoded once, by the claiming lane: the list position -> tile mapping
// needs integer divisions, ~100 instructions that every warp of the pair would otherwise repeat for every tile):
//   bit 0 kind | bits 1-4 level | bit 5 group within the level (K1) | bits 6-11 n_blk | bits 12-30 m_blk ; -1 = end
__host__ __device__ __forceinline__ int mlp_pack(const MlpTile& t) {
  return t.kind | (t.l << 1) | ((t.kind == 0 ? (t.z & 1) : 0) << 5) | (t.n_blk << 6) | (t.m_blk << 12);
}
__device__ __forceinline__ MlpTile mlp_unpack(const MlpParams& p, int w) {
  MlpTile t;
  t.kind = w & 1;
  t.l = (w >> 1) & 15;
  t.n_blk = (w >> 6) & 63;
  t.m_blk = (w >> 12) & 0x7FFFF;
  t.z = t.kind ? t.l : 2 * t.l + ((w >> 5) & 1);
  t.num_kb = t.kind ? ((t.l == p.L - 1) ? 4 * p.d : 8 * p.d) / BK : p.d / BK;
  return t;
}

// next tile descriptor of the cluster's sequence (slot seq % MLP_SLOTS of the ring); -1 = no more work
__device__ __forceinline__ int mlp_fetch(uint64_t* sfull, const volatile int* stile, uint32_t sempty_leader, uint32_t seq) {
  const uint32_t slot = seq % MLP_SLOTS, ph = (seq / MLP_SLOTS) & 1u;
  // plain (cta-scope) wait in both CTAs: the leader's slot is written by a thread of the same CTA, the peer's by
  // st.async, whose data is visible to whoever observes the barrier's transaction count complete (like TMA data)
  mbar_wait(&sfull[slot], ph);
  const int tile = stile[slot];
  // the release of the slot must not overtake the read above: make the arrive depend on the value
  if (tile >= -1) mbar_arrive_cluster(sempty_leader + 8u * slot);
  return tile;
}
// the same for a converged warp (control warps, see elect_one): every lane waits and reads, the elected lane releases
__device__ __forceinline__ int mlp_fetch_warp(uint64_t* sfull, const volatile int* stile, uint32_t sempty_leader, uint32_t seq,
                                              uint32_t elected) {
  const uint32_t slot = seq % MLP_SLOTS, ph = (seq / MLP_SLOTS) & 1u;
  mbar_wait(&sfull[slot], ph);
  const int tile = stile[slot];
  __syncwarp();                                    // every lane has read the slot before it is handed back
  if (elected && tile >= -1) mbar_arrive_cluster(sempty_leader + 8u * slot);
  return tile;
}

// cycles spent inside `stmt` added to `acc` (DBG builds only)
#define MLP_TIMED(acc, stmt)                               \
  do {                                                     \
    if (DBG) { const long long t_ = clock64(); stmt; acc += (unsigned long long)(clock64() - t_); } \
    else { stmt; }                                         \
  } while (0)

template <bool DBG>
__global__ void __launch_bounds__(MLP_THREADS, 1)
mlp_kernel(const __grid_constant__ CUtensorMap map_x,    // tokens Xb (rows, d)
           const __grid_constant__ CUtensorMap map_sb,   // state shadow Sb (rows, L*d)
           const __grid_constant__ CUtensorMap map_sp,   // Sb[:,1:]+pos shadow Sp (rows, (L-1)*d)
           const __grid_constant__ CUtensorMap map_w1,   // W1p (G*4d, d)
           const __grid_constant__ CUtensorMap map_h,    // H as 16 KB blocks
           const __grid_constant__ CUtensorMap map_w2,   // W2p (L*d, 8d)
           const MlpParams p) {
  constexpr int STAGES = MLP_STAGES;
  constexpr int BN = MLP_BN;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  float* stg_all = reinterpret_cast<float*>(smem + (size_t)STAGES * MLP_STAGE_BYTES);
  uint8_t* patches = reinterpret_cast<uint8_t*>(stg_all) + 4 * STG_BYTES;
  float* xch = reinterpret_cast<float*>(patches + (size_t)MLP_CONSUMER_WARPS * MLP_PATCH_BYTES);   // [4 pairs][32]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(xch + 4 * 32);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* sfull_bar = empty_bar + STAGES;           // [MLP_SLOTS] own: tile index of the slot published
  uint64_t* sempty_bar = sfull_bar + MLP_SLOTS;       // [MLP_SLOTS] leader's: every consumer of both CTAs has read it
  uint64_t* pub_bar = sempty_bar + MLP_SLOTS;         // [2] own: the consumer warps issued their stores of the tile
  int* stile = reinterpret_cast<int*>(pub_bar + 2);   // [MLP_SLOTS]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  constexpr int W_TMA = MLP_CONSUMER_WARPS, W_SCHED = MLP_CONSUMER_WARPS + 1;
  const uint32_t cta_rank = cluster_ctarank();
  const bool leader = cta_rank == 0;

  if (warp == W_TMA && lane == 0) {
    tma_prefetch_desc(&map_x); tma_prefetch_desc(&map_sb); tma_prefetch_desc(&map_sp);
    tma_prefetch_desc(&map_w1); tma_prefetch_desc(&map_h); tma_prefetch_desc(&map_w2);
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], MLP_CONSUMER_WARPS); }
    for (int i = 0; i < 2; ++i) mbar_init(&pub_bar[i], MLP_CONSUMER_WARPS);
    for (int i = 0; i < MLP_SLOTS; ++i) { mbar_init(&sfull_bar[i], 1); mbar_init(&sempty_bar[i], MLP_SEMPTY_COUNT); }
    fence_barrier_init();
  }
  __syncthreads();
  cluster_sync_all();          // peer barriers initialised before any cross-CTA traffic
  pdl_launch_dependents();
  pdl_wait();                  // global memory (counters included) is touched only after the previous kernel finished
  const bool clk_thread = blockIdx.x == 0 && warp == W_SCHED && lane == 0;
  ClockSample clk_s{};
  if (clk_thread) clk_s = clock_sample_begin();

  const uint32_t sempty_leader = mapa_shared(smem_u32(&sempty_bar[0]), 0);
  const long long k_t0 = DBG ? clock64() : 0;
  unsigned long long dw0 = 0, dw1 = 0, dw2 = 0, dw3 = 0, dw4 = 0;     // per-role wait / work counters (DBG)
  unsigned long long* dbg = DBG ? p.dbg + (size_t)blockIdx.x * 16 : nullptr;

  if (warp == W_SCHED) {
    // ------------------------------------------------------------------ publisher (both CTAs, one lane)
    // once all consumer warps of this CTA have issued their stores of a K1 tile: one gpu-scope release of the
    // (level, row block) counter for the whole CTA
    if (lane == 0) {
      int as = 0; uint32_t aphase = 0;
      for (uint32_t seq = 0;; ++seq) {
        const int tile = mlp_fetch(sfull_bar, stile, sempty_leader, seq);
        if (tile < 0) break;
        const MlpTile t = mlp_unpack(p, tile);
        MLP_TIMED(dw0, mbar_wait(&pub_bar[as], aphase));
        if (t.kind == 0) MLP_TIMED(dw1, red_release_gpu_add(p.ready + t.l * p.num_m + t.m_blk, 1));
        if (++as == 2) { as = 0; aphase ^= 1; }
      }
      if (DBG) { dbg[0] = dw0; dbg[1] = dw1; }
    }
  } else if (warp == W_TMA) {
    // ------------------------------------------------------------------ TMA producer (both CTAs)
    // warp-converged (see elect_one): all lanes walk the tile sequence and poll the ring barriers, the elected lane
    // claims tiles, waits for dependencies and issues the loads
    const uint32_t elected = elect_one();
    const int elected_lane = __ffs(__ballot_sync(0xffffffffu, elected != 0)) - 1;
    int stage = 0; uint32_t phase = 0;
    const uint64_t pol_first = l2_policy_evict_first();
    const uint32_t smem0 = smem_u32(smem);
    const int kbg_n = 4 * p.d / BK;
    const int blk_skip = (p.m128 - 1) * kbg_n;
    // leader: draws the tile index and publishes it to the ring (both CTAs); peer: reads the ring like everyone else
    uint32_t pub_seq = 0;
    int last_kind = 0;
    // The draw is a chain of dependent L2 round trips (list heads -> dependency counter -> compare-and-swap / add, ~1.5 k
    // cycles).  Done in one piece between two loads it would stall the load stream feeding the consumers; it is therefore
    // split into four phases issued two k-blocks apart, so each phase's result has arrived when the next one needs it
    // and the TMA issue stream never waits on it.
    int c_i1 = 0, c_j = 0, c_ready = 0, c_res = 0, c_mode = 0;      // c_mode: 0 = K1 add pending, 1 = K2 cas pending
    auto claim_a = [&]() {                          // list heads (approximate: others move them)
      c_i1 = *reinterpret_cast<volatile int*>(p.counter);
      c_j = *reinterpret_cast<volatile int*>(p.counter + 1);
    };
    auto claim_b = [&]() {                          // lag reached? -> look at the K2 head's dependency counter
      c_mode = 0;
      if (c_i1 < p.n1_tiles && c_j < p.n2_tiles) {
        const MlpTile h1 = mlp_decode1(p, c_i1), h2 = mlp_decode2(p, c_j);
        const int lag = (h1.l - h2.l) * p.num_m + (h1.m_blk - h2.m_blk);
        if (lag >= (last_kind ? p.lag_lo : p.lag_hi)) {
          c_mode = 1;
          c_ready = ld_acquire_gpu(p.ready + h2.l * p.num_m + h2.m_blk);
        }
      }
    };
    auto claim_c = [&]() {                          // take the K2 head (its producers have retired) or the next K1 tile
      if (c_mode == 1) {
        const int l2 = c_j / (p.num_m * p.nN2);
        if (c_ready >= ((l2 == p.L - 1) ? 1 : 2) * p.nN1 * 2) { c_res = atomicCAS(p.counter + 1, c_j, c_j + 1); return; }
        c_mode = 0;
      }
      c_res = atomicAdd(p.counter, 1);
    };
    auto claim_d = [&]() -> int {                   // resolve and publish to the ring of both CTAs
      int tile;
      if (c_mode == 1 && c_res == c_j) tile = mlp_pack(mlp_decode2(p, c_j));
      else {
        const int i = c_mode == 1 ? atomicAdd(p.counter, 1) : c_res;       // lost the race for the K2 head: a K1 tile
        if (i < p.n1_tiles) tile = mlp_pack(mlp_decode1(p, i));
        else {                                      // K1 list exhausted: K2 tiles in order (the TMA lane waits for their producers)
          const int j = atomicAdd(p.counter + 1, 1);
          tile = j < p.n2_tiles ? mlp_pack(mlp_decode2(p, j)) : -1;
        }
      }
      if (DBG && tile >= 0) { if (tile & 1) { ++dw4; if (!last_kind) dw4 += 1ull << 32; } }
      last_kind = tile >= 0 ? (tile & 1) : 0;
      const uint32_t slot = pub_seq % MLP_SLOTS, ph = (pub_seq / MLP_SLOTS) & 1u;
      mbar_wait(&sempty_bar[slot], ph ^ 1u);                  // all readers of the slot's previous use are done
      *reinterpret_cast<volatile int*>(&stile[slot]) = tile;
      mbar_arrive(&sfull_bar[slot]);                                        // own CTA (release.cta)
      const uint32_t rbar = mapa_shared(smem_u32(&sfull_bar[slot]), 1);
      mbar_arrive_expect_tx_cluster(rbar, 4);                               // peer CTA: value + completion in one
      st_async_b32(mapa_shared(smem_u32(&stile[slot]), 1), (uint32_t)tile, rbar);
      ++pub_seq;
      return tile;
    };
    auto claim = [&]() -> int { claim_a(); claim_b(); claim_c(); return claim_d(); };     // first tile: nothing to overlap with
    int next_tile = -2;
    if (leader) {
      if (elected) MLP_TIMED(dw0, next_tile = claim());
      next_tile = __shfl_sync(0xffffffffu, next_tile, elected_lane);
    }
    for (uint32_t seq = 0;; ++seq) {
      int tile;
      if (leader) tile = next_tile;
      else MLP_TIMED(dw0, tile = mlp_fetch_warp(sfull_bar, stile, sempty_leader, seq, elected));
      if (tile < 0) break;
      next_tile = -2;
      const MlpTile t = mlp_unpack(p, tile);
      const CUtensorMap* amap;
      int a_col = 0, b_row;
      const CUtensorMap* bmap;
      if (t.kind == 0) {
        const int l = t.l;
        if (t.z == 0) { amap = &map_x; a_col = 0; }                          // bottom-up level 0 reads the tokens (:132)
        else if (t.z & 1) { amap = &map_sp; a_col = l * p.d; }               // top-down l reads S[l+1]+pos (:136)
        else { amap = &map_sb; a_col = (l - 1) * p.d; }                      // bottom-up l reads S[l-1]   (:134)
        bmap = &map_w1;
        b_row = t.z * 4 * p.d + t.n_blk * BN;
      } else {
        amap = &map_h; bmap = &map_w2;
        b_row = t.z * p.d + t.n_blk * BN;
        if (elected) {
          // all K1 tiles of this (level, row block) have published their part of H
          const int need = ((t.l == p.L - 1) ? 1 : 2) * p.nN1 * 2;              // one arrival per CTA and K1 tile
          const int* ctr = p.ready + t.l * p.num_m + t.m_blk;
          if (ld_acquire_gpu(ctr) < need) {
            const long long t0 = clock64();
            if (DBG) ++dw3;
            while (ld_acquire_gpu(ctr) < need) {
              __nanosleep(64);
              if (clock64() - t0 > GLOM_WAIT_TIMEOUT_CYCLES) asm volatile("trap;");
            }
            if (DBG) dw1 += (unsigned long long)(clock64() - t0);
          }
          fence_proxy_async_global();          // generic-proxy stores of H (other SMs) -> this thread's TMA loads
        }
        __syncwarp();
      }
      const int a_row = t.m_blk * 256 + (int)cta_rank * BM;
      // K2: block (group g, 128-row block, 64-wide k block); [H_bu,l | H_td,l] are groups 2l and 2l+1
      const int blk0 = (2 * t.z * p.m128 + (a_row >> 7)) * kbg_n;
      // the row block's H is read by all nN2 column tiles: only the last one may mark it evict-first
      const bool h_first = p.h_load_policy == 1 || (p.h_load_policy == 0 && t.n_blk == p.nN2 - 1);
      // claim phases at k-blocks ca, ca + 1, ca + 2, ca + 3 (late look-ahead: a claimed tile starts loading
      // ~1-2 us later; claiming further ahead lets a cluster busy with a long tile sit on tiles others wait for)
      // (the draw is published 4 k-blocks before the tile's last load: the peer CTA's TMA lane learns about the next
      // tile through the ring and must not start it late)
      const int cs = 1;
      const int ca = t.num_kb >= 7 ? t.num_kb - 7 : 0;
      for (int kb = 0; kb < t.num_kb; ++kb) {
        if (leader) {
          if (elected) {
            if (kb == ca) MLP_TIMED(dw0, claim_a());
            else if (kb == ca + cs) MLP_TIMED(dw0, claim_b());
            else if (kb == ca + 2 * cs) MLP_TIMED(dw0, claim_c());
            else if (kb == ca + 2 * cs + 1) MLP_TIMED(dw0, next_tile = claim_d());
          }
          __syncwarp();
        }
        MLP_TIMED(dw2, mbar_wait(&empty_bar[stage], phase ^ 1));
        if (elected) {
          const uint32_t sa = smem0 + (uint32_t)stage * MLP_STAGE_BYTES;
          uint64_t* bar = &full_bar[stage];
          mbar_arrive_expect_tx(bar, MLP_STAGE_BYTES);
          if (t.kind == 1) {
            const int blk = blk0 + kb + (kb >= kbg_n ? blk_skip : 0);
            // last use of these lines by this column tile: evict-first keeps them from displacing weights / state
            if (h_first) tma_load_2d_hint(sa, amap, bar, 0, blk * BM, pol_first);
            else tma_load_2d(sa, amap, bar, 0, blk * BM);
          } else {
            tma_load_2d(sa, amap, bar, a_col + kb * BK, a_row);
          }
          // the B tile as two boxes of 128 rows
          tma_load_2d(sa + A_STAGE_BYTES, bmap, bar, kb * BK, b_row);
          tma_load_2d(sa + A_STAGE_BYTES + (BN / 2) * BK * 2, bmap, bar, kb * BK, b_row + BN / 2);
        }
        __syncwarp();
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      if (leader) next_tile = __shfl_sync(0xffffffffu, next_tile, elected_lane);
    }
    if (DBG && elected) { dbg[2] = dw0; dbg[3] = dw1; dbg[4] = dw2; dbg[15] = dw3; if (leader) dbg[12] = dw4; }
  } else if (warp < MLP_CONSUMER_WARPS) {
    // ------------------------------------------------------------------ consumers: wgmma main loop + epilogue (8 warps)
    const int wg = warp >> 2, wi = warp & 3;
    const int pair = warp >> 1, x = warp & 1;  // warp pair = 32-row band `pair` of the CTA's 128 rows; x = its 32-column half
    float* stg = stg_all + pair * (STG_BYTES / 4);
    uint8_t* patch = patches + (size_t)warp * MLP_PATCH_BYTES;
    float* xch_p = xch + pair * 32;
    const uint32_t smem0 = smem_u32(smem);
    // H should stay in L2 until this launch's GEMM2 tiles have read it
    const uint64_t pol_h = p.h_store_policy == 0 ? l2_policy_evict_last() : l2_policy_evict_normal();
    int stage = 0; uint32_t phase = 0;
    int as = 0; uint32_t aphase = 0;
    float acc[BN / 2];
    for (uint32_t seq = 0;; ++seq) {
      int tile = 0;
      if (lane == 0) MLP_TIMED(dw0, tile = mlp_fetch(sfull_bar, stile, sempty_leader, seq));
      tile = __shfl_sync(0xffffffffu, tile, 0);
      if (tile < 0) break;
      const MlpTile t = mlp_unpack(p, tile);
      const int row0 = t.m_blk * 256 + (int)cta_rank * BM + pair * 32;   // first row of this warp pair's 32-row band
      const int rows_left = p.rows - row0;                                // >= 32: whole band valid (warp-uniform)
      if (t.kind == 1 && lane < rows_left) {
        // The combine reads this band's fp32 state and C lines: pull them into L2 before the main loop, so the epilogue's
        // dependent global loads hit L2
        const size_t o = ((size_t)(row0 + lane) * p.L + t.z) * p.d + t.n_blk * BN + x * (BN / 2);
#pragma unroll
        for (int c = 0; c < BN / 2; c += 32) {
          if (!p.s_bcast) prefetch_l2(p.s32_in + o + c);
          if ((c & 63) == 0) prefetch_l2(p.c_in + o + c);
        }
      }
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      int prev = -1;                    // slot of the k-block whose MMAs may still be running
      for (int kb = 0; kb < t.num_kb; ++kb) {
        MLP_TIMED(dw1, mbar_wait(&full_bar[stage], phase));
        const uint32_t sa = smem0 + (uint32_t)stage * MLP_STAGE_BYTES;
        wgmma_fence_regs(acc);
        wgmma_fence();
        wgmma_kblock<BN, 0>(acc, sa + (uint32_t)wg * (A_STAGE_BYTES / 2), sa + A_STAGE_BYTES);
        wgmma_commit();
        wgmma_wait<1>();                  // the previous k-block's MMAs are complete: release its slot
        wgmma_fence_regs(acc);
        if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty_bar[prev]); }
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[prev]);
      const long long e_t0 = DBG ? clock64() : 0;
#pragma unroll 1
      for (int s = 0; s < BN / 64; ++s) {
        stage_write(acc, stg, s, wi, lane);
        named_bar_sync(1 + pair, 64);
        uint32_t v[32];
        stage_read(stg, x, lane, v);
        const int cc = 64 * s + 32 * x;                               // column of this chunk inside the tile
        if (t.kind == 0) {
          // H block (group, 128-row block, k block = this 64-column step): 16 KB contiguous, row pitch 64
          const int hblk = (t.z * p.m128 + (t.m_blk * 2 + (int)cta_rank)) * (4 * p.d / BK) + t.n_blk * (BN / BK) + s;
          __nv_bfloat16* hrow = p.h + ((size_t)hblk * BM + pair * 32) * BK + 32 * x;
          const float* bias = p.b1 + (size_t)t.z * 4 * p.d + t.n_blk * BN + cc;
          if (rows_left >= 32) k1_chunk<true, 1>(v, bias, patch, hrow, (size_t)BK, lane, 32, pol_h);
          else k1_chunk<false, 1>(v, bias, patch, hrow, (size_t)BK, lane, rows_left, pol_h);
        } else {
          K2Chunk kc;
          kc.l = t.z; kc.L = p.L; kc.d = p.d; kc.n = p.n; kc.row0 = row0; kc.prow0 = row0 % p.n; kc.s_bcast = p.s_bcast;
          kc.s32_in = p.s32_in; kc.c_in = p.c_in; kc.pos = p.pos;
          kc.s32_out = p.s32_out; kc.sb_out = p.sb_out; kc.sp_out = p.sp_out;
          const int col = t.n_blk * BN + cc;
          const float4 b4 = __ldg(reinterpret_cast<const float4*>(p.b2 + (size_t)t.z * p.d + col + (lane & 7) * 4));
          float rowsq[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) rowsq[i] = 0.f;
          if (rows_left >= 32) k2_chunk<true>(v, b4, patch, kc, col, lane, 32, rowsq);
          else k2_chunk<false>(v, b4, patch, kc, col, lane, rows_left, rowsq);
          // one squared-norm partial per 64 columns: the two warps of the pair hold its 32-column halves, summed in chunk
          // order (0 + first) + second as in prep_state_kernel
          if (x == 1 && (lane & 7) == 0) {
#pragma unroll
            for (int i = 0; i < 8; ++i) xch_p[i * 4 + (lane >> 3)] = rowsq[i];
          }
          named_bar_sync(1 + pair, 64);
          if (x == 0 && (lane & 7) == 0) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const int r = i * 4 + (lane >> 3);
              const float q = rowsq[i] + xch_p[i * 4 + (lane >> 3)];
              if (r < rows_left) p.nsq_out[((size_t)(row0 + r) * p.L + t.z) * p.nparts + t.n_blk * 4 + s] = q;
            }
          }
        }
        named_bar_sync(1 + pair, 64);                                   // staging tile free for the next step
      }
      // this warp's stores of the tile are issued: tell the CTA's publisher lane (it releases them at gpu scope for
      // K1 tiles; the lanes' stores are ordered before lane 0's arrive by the warp barrier)
      __syncwarp();
      if (lane == 0) mbar_arrive(&pub_bar[as]);
      if (++as == 2) { as = 0; aphase ^= 1; }
      if (DBG) { if (t.kind == 0) dw2 += (unsigned long long)(clock64() - e_t0); else dw3 += (unsigned long long)(clock64() - e_t0); }
    }
    if (DBG && warp == 0 && lane == 0) {
      dbg[8] = dw0; dbg[9] = dw1; dbg[10] = dw2; dbg[11] = dw3;
      dbg[13] = (unsigned long long)(clock64() - k_t0);
    }
  }

  __syncthreads();
  if (clk_thread) clock_sample_end(clk_s, g_mlp_clk);
  cluster_sync_all();          // no CTA exits while its pair can still touch its shared memory
}

cudaError_t mlp_kernel_clocks(unsigned long long* out /* [2] */, bool reset) {
  cudaError_t e = cudaMemcpyFromSymbol(out, g_mlp_clk, sizeof(unsigned long long) * 2);
  if (e == cudaSuccess && reset) {
    static const unsigned long long zeros[2] = {};
    e = cudaMemcpyToSymbol(g_mlp_clk, zeros, sizeof(zeros));
  }
  return e;
}

// =====================================================================================
// Host side
// =====================================================================================
bool mlp_fused_supported(const Geometry& g) {     // limits of the packed tile descriptor: 16 levels, 64 column tiles, 2^19 row blocks
  return g.d % 256 == 0 && g.d <= 4096 && g.L <= MLP_MAX_LEVELS && g.L >= 2 && (g.rows + 255) / 256 < (1 << 19);
}

size_t mlp_sched_ints(const Geometry& g) {                       // per launch: two list heads + ready[L * num_m], padded
  const size_t n = 2 + (size_t)g.L * ((g.rows + 255) / 256);
  return (n + 31) / 32 * 32;
}

// work-list geometry of one launch (everything mlp_decode1 / mlp_decode2 and the claim policy need)
static void mlp_list_params(const Geometry& g, int num_sms, MlpParams* pp) {
  MlpParams& p = *pp;
  const int d = g.d, L = g.L, rows = g.rows;
  p.rows = rows; p.d = d; p.L = L; p.n = g.n;
  p.num_m = (rows + 255) / 256;
  p.nN1 = 4 * d / MLP_BN; p.nN2 = d / MLP_BN;
  p.m128 = (rows + BM - 1) / BM;
  int base = 0;
  for (int l = 0; l < L; ++l) {
    p.lvl1_base[l] = base;
    base += p.num_m * ((l == L - 1) ? 1 : 2) * p.nN1;
  }
  p.lvl1_base[L] = base;
  p.n1_tiles = base;
  p.n2_tiles = L * p.num_m * p.nN2;
  // lag thresholds: with every cluster on K1 tiles, num_sms / 2 tiles = that many / (2 nN1) row blocks are in flight; a K2
  // head that far behind the K1 head has normally retired all its producers
  const int max_clusters = num_sms / 2;
  const int inflight = (max_clusters + 2 * p.nN1 - 1) / (2 * p.nN1);
  static int lag_override = -2, lag_lo_override = -2;
  if (lag_override == -2) { const char* e = getenv("GLOM_B200_MLP_LAG"); lag_override = e ? atoi(e) : -1; }
  if (lag_lo_override == -2) { const char* e = getenv("GLOM_B200_MLP_LAG_LO"); lag_lo_override = e ? atoi(e) : -1; }
  p.lag_hi = lag_override >= 0 ? lag_override : inflight + 3;
  p.lag_lo = lag_lo_override >= 0 ? lag_lo_override : (p.lag_hi + 1) / 2;
  if (p.lag_hi < 1) p.lag_hi = 1;
  if (p.lag_lo < 1) p.lag_lo = 1;
  if (p.lag_lo > p.lag_hi) p.lag_lo = p.lag_hi;
}

// diagnostics / host tests: the two ordered work lists, K1 list first, as (kind, z, m_blk, n_blk) quadruples;
// *delay = the lag threshold (row blocks) at which a cluster coming from a K1 tile takes the K2 head
int mlp_schedule_dump(const Geometry& g, int num_sms, int* out, int capacity, int* num_tiles, int* delay) {
  if (!mlp_fused_supported(g)) return -1;
  MlpParams p{};
  mlp_list_params(g, num_sms, &p);
  const int total = p.n1_tiles + p.n2_tiles;
  if (num_tiles) *num_tiles = total;
  if (delay) *delay = p.lag_hi;
  for (int i = 0; i < total && i < capacity; ++i) {
    const MlpTile t = i < p.n1_tiles ? mlp_decode1(p, i) : mlp_decode2(p, i - p.n1_tiles);
    out[4 * i] = t.kind; out[4 * i + 1] = t.z; out[4 * i + 2] = t.m_blk; out[4 * i + 3] = t.n_blk;
  }
  return 0;
}

int step_bf16_mlp_fused(const Geometry& g, const Bf16Buffers& b, int* sched, EncodeTiledFn enc, int num_sms,
                        cudaStream_t st, int* launches, char* err, size_t errlen, Profiler* prof) {
  const int d = g.d, L = g.L, rows = g.rows;
  const int m128 = (rows + BM - 1) / BM;
  CUtensorMap mh, mx, msb, msp, mw1, mw2;
  if (!map2d(enc, &mh, b.h, (uint64_t)g.G * m128 * (4 * d / BK) * BM, BK, BM, err, errlen, "H")) return -3;
  if (!map2d(enc, &mx, b.xb, rows, d, BM, err, errlen, "Xb")) return -3;
  if (!map2d(enc, &msb, b.sb_in, rows, (uint64_t)L * d, BM, err, errlen, "Sb")) return -3;
  if (!map2d(enc, &msp, b.sp_in, rows, (uint64_t)(L - 1) * d, BM, err, errlen, "Sp")) return -3;
  if (!map2d(enc, &mw1, b.w1, (uint64_t)g.G * 4 * d, d, 128, err, errlen, "W1p")) return -3;
  if (!map2d(enc, &mw2, b.w2, (uint64_t)L * d, (uint64_t)8 * d, 128, err, errlen, "W2p")) return -3;
  MlpParams p{};
  mlp_list_params(g, num_sms, &p);
  const int max_clusters = num_sms / 2;
  p.b1 = b.b1; p.b2 = b.b2; p.h = b.h;
  p.s32_in = b.s32_in; p.s_bcast = b.s32_in_bcast; p.c_in = b.c; p.pos = b.pos;
  p.s32_out = b.s32_out; p.sb_out = b.sb_out; p.sp_out = b.sp_out; p.nsq_out = b.nsq_out; p.nparts = g.nparts;
  p.counter = sched; p.ready = sched + 2;
  static int hpol = -1;
  if (hpol < 0) { const char* e = getenv("GLOM_B200_MLP_HPOL"); hpol = e ? atoi(e) : 0; }      // diagnostics: 10 * store + load
  p.h_load_policy = hpol % 10; p.h_store_policy = hpol / 10;

  // GLOM_B200_MLP_DBG=1 (diagnostics): the instrumented instantiation, synchronised and summarised on stderr for the
  // first launches of the process.  Never set in production: it allocates a small device buffer and blocks the stream.
  static int dbg_mode = -1;
  static unsigned long long* dbg_buf = nullptr;
  static int dbg_left = 4;
  if (dbg_mode < 0) { const char* e = getenv("GLOM_B200_MLP_DBG"); dbg_mode = (e && e[0] == '1') ? 1 : 0; }
  const bool dbg = dbg_mode == 1 && dbg_left > 0;
  if (dbg && !dbg_buf && cudaMalloc(&dbg_buf, (size_t)num_sms * 16 * sizeof(unsigned long long)) != cudaSuccess) return -3;
  if (dbg) { cudaMemsetAsync(dbg_buf, 0, (size_t)num_sms * 16 * sizeof(unsigned long long), st); p.dbg = dbg_buf; }
  static SmemOptIn optin, optin_dbg;
  if (cudaError_t e = dbg ? optin_dbg.ensure(mlp_kernel<true>, MLP_SMEM_BYTES) : optin.ensure(mlp_kernel<false>, MLP_SMEM_BYTES)) {
    snprintf(err, errlen, "cudaFuncSetAttribute(mlp_kernel): %s", cudaGetErrorString(e));
    return -3;
  }
  const int total_tiles = p.n1_tiles + p.n2_tiles;
  const int clusters = total_tiles < max_clusters ? total_tiles : max_clusters;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(2 * clusters);
  cfg.blockDim = dim3(MLP_THREADS);
  cfg.dynamicSmemBytes = MLP_SMEM_BYTES;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 2; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = 2;
  cudaError_t e;
  {
    ProfScope scope(prof, PROF_MLP, st);
    e = dbg ? cudaLaunchKernelEx(&cfg, mlp_kernel<true>, mx, msb, msp, mw1, mh, mw2, p)
            : cudaLaunchKernelEx(&cfg, mlp_kernel<false>, mx, msb, msp, mw1, mh, mw2, p);
  }
  if (launches) ++*launches;
  if (e != cudaSuccess) { snprintf(err, errlen, "mlp_kernel launch: %s", cudaGetErrorString(e)); return -3; }
  if (dbg) {
    --dbg_left;
    static const char* names[16] = {"pub: wait epilogue stores", "pub: release", "tma: claim / fetch tile", "tma: dependency wait",
                                    "tma: wait smem slot", "-", "-", "-",
                                    "consumer w0: fetch tile", "consumer w0: wait operands", "consumer w0: K1 tiles epilogue", "consumer w0: K2 tiles epilogue",
                                    "tma: K2 tiles (+ 2^32 per K1->K2 switch)", "consumer w0: kernel total", "-", "tma: dependency waits (count)"};
    std::vector<unsigned long long> h((size_t)num_sms * 16);
    if (cudaStreamSynchronize(st) == cudaSuccess &&
        cudaMemcpy(h.data(), dbg_buf, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost) == cudaSuccess) {
      fprintf(stderr, "[mlp_kernel dbg] %d + %d tiles, lag thresholds %d / %d row blocks, %d clusters; cycles per CTA: mean (max)\n", p.n1_tiles, p.n2_tiles, p.lag_hi, p.lag_lo, clusters);
      for (int k = 0; k < 16; ++k) {
        double sum = 0, mx_ = 0; int cnt = 0;
        for (int c = 0; c < 2 * clusters; ++c) {
          const double v = (double)h[(size_t)c * 16 + k];
          if (k == 12 && (c & 1)) continue;     // leader-only role
          sum += v; if (v > mx_) mx_ = v; ++cnt;
        }
        if (k == 12) {      // packed: K2 tiles in the low word, K1 -> K2 role switches in the high word
          double k2 = 0, sw = 0, k2max = 0;
          for (int c = 0; c < 2 * clusters; c += 2) {
            const unsigned long long v = h[(size_t)c * 16 + k];
            k2 += (double)(v & 0xffffffffull); sw += (double)(v >> 32);
            if ((double)(v & 0xffffffffull) > k2max) k2max = (double)(v & 0xffffffffull);
          }
          fprintf(stderr, "[mlp_kernel dbg]   K2 tiles per cluster %.2f (max %.0f), K1->K2 role switches per cluster %.2f\n",
                  k2 / clusters, k2max, sw / clusters);
          continue;
        }
        fprintf(stderr, "[mlp_kernel dbg]   %-32s %12.0f (%12.0f)\n", names[k], cnt ? sum / cnt : 0.0, mx_);
      }
    }
  }
  return 0;
}

}  // namespace glom
