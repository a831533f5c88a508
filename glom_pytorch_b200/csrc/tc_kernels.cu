// Tensor-core (wgmma / TMA / mbarrier) kernels of the GLOM column update for sm_90a.
//
//   gemm_kernel<0>  K1: H = gelu_erf(A_g . W1_g^T + b1_g)         all 2L-1 MLP groups, one launch
//                       (GroupedFeedForward first Conv1d + GELU, glom_pytorch.py:29-30, calls :134/:136)
//   gemm_kernel<1>  K2: S' = (S + C + [H_bu,l | H_td,l] . [W2bu_l | W2td_l]^T + b2) / c_l
//                       (second Conv1d :31 of both nets, F.pad zero top level :137, combine :141-142)
//   attn_kernel     K3: C = softmax_j(<S_i, S_j/|S_j|> d^-1/2, diag := -5e-4, radius mask) . S
//                       (ConsensusAttention.forward :56-73)
//
// All three are warp-specialised: one TMA producer warp feeds a ring of 128B-swizzled shared-memory stages, two consumer
// warpgroups run wgmma with the accumulators in registers and then the epilogue / softmax.
#include "gemm_sched.cuh"
#include "tc_common.cuh"

#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <type_traits>

namespace glom {

// =====================================================================================
// K1 / K2: persistent grouped GEMM, fused epilogues
//   The schedule deals 256 x BN output tiles to pairs of CTAs, launched as two-CTA clusters; CTA 2c + r of pair c owns
//   rows [128 r, 128 r + 128) of each tile of pair c.  Both CTAs need the same B (weight) k-blocks in the same order, so
//   each loads one BN/2-row half and multicasts it to both.  Warpgroup 0 is the producer: its first warp fills a ring of
//   (A 128 x 64, B BN x 64) stages, and the warpgroup gives up registers (setmaxnreg) to the two consumer warpgroups,
//   which each run wgmma m64 x BN x 16 on 64 of the rows with the accumulator in registers.
//   After the tile's K loop, K1 applies bias + GELU on the accumulator fragment itself and stores H through per-warpgroup
//   swizzled output tiles with TMA.  K2 and the tokeniser hand the accumulator, 64 columns at a time, through
//   per-warp-pair staging tiles into row-per-thread 32 x 32 chunks, and each chunk through a private transpose patch so
//   that every global load / store instruction covers whole cache lines (the reference's 4-way combine / residual
//   write, glom_pytorch.py:141-142).
// =====================================================================================
constexpr int GEMM_CONSUMER_WARPS = 8;
constexpr int GEMM_THREADS = 128 + 32 * GEMM_CONSUMER_WARPS;
// 40 x 128 + 232 x 256 = 64,512 of the SM's 65,536 registers: the 64 x 256 fp32 accumulator (128 registers) and the
// epilogue fit the consumers without spilling
constexpr uint32_t GEMM_PRODUCER_REGS = 40;
constexpr uint32_t GEMM_CONSUMER_REGS = 232;

// in-kernel clock samples (see clock_sample_begin): [kind][cycles, ns], kinds = ProfKind
// + wait-cycle counters of block 0: [2] first consumer warp waiting for operands, [4] TMA lane waiting for a free ring
// slot, [6] first consumer warp busy in the epilogue ([3] and [5] stay 0: the accumulator lives in the consumers' registers)
__device__ unsigned long long g_kernel_clk[PROF_KINDS][8];


template <int MODE, int BN>
struct GemmCfg {
  // squared-norm partials per tile row (K2; Geometry::part_w columns each)
  static constexpr int PARTS = (BN == 256) ? 4 : 2;
  static constexpr int PART_COLS = BN / PARTS;                      // 64 / 64 / 32
  static constexpr int THREADS = GEMM_THREADS;
  static constexpr uint32_t B_STAGE_BYTES = BN * BK * 2;
  static constexpr uint32_t STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static_assert(MODE >= 0 && MODE <= 2, "0 = GEMM1+GELU, 1 = GEMM2+combine, 2 = tokeniser");
  // ring + epilogue buffers within 227 KB
  static constexpr int STAGES = (BN == 256) ? 3 : (BN == 128) ? 4 : 5;
  // K1 (MODE 0): a 64-row x BN-column bf16 output tile per consumer warpgroup, BN / 64 TMA boxes of 64 x 64, written
  // from the accumulator fragment and stored to H by TMA.  K2 / tokeniser: per-pair staging tiles, per-warp 32 x 32 f32
  // transpose patches and the squared-norm exchange of the warp pairs.
  static constexpr uint32_t OUT_BOX_BYTES = 64 * BK * 2;
  static constexpr uint32_t PATCH_BYTES = 4096;
  static constexpr size_t EPI_BYTES = (MODE == 0) ? 2 * (BN / 64) * (size_t)OUT_BOX_BYTES
                                                  : 4 * (size_t)STG_BYTES + (size_t)GEMM_CONSUMER_WARPS * PATCH_BYTES + 4 * 32 * 4;
  static constexpr size_t SMEM_BYTES = 1024 /*align slack*/ + (size_t)STAGES * STAGE_BYTES + EPI_BYTES + 256 /*barriers*/;
  static_assert(SMEM_BYTES <= 232448, "over the 227 KB of shared memory a block may opt in to");
};

// ---- tokeniser epilogue chunk (image_to_tokens Linear bias, glom_pytorch.py:96): f32 out, whole 128-byte lines.
__device__ __forceinline__ void tok_chunk(const uint32_t (&v)[32], const float4 b4, uint8_t* patch, float* dst,
                                          size_t pitch, int lane, int rows_left) {
#pragma unroll
  for (int c = 0; c < 8; ++c)
    *reinterpret_cast<uint4*>(patch + lane * 128 + ((c ^ (lane & 7)) << 4)) =
        make_uint4(v[4 * c], v[4 * c + 1], v[4 * c + 2], v[4 * c + 3]);
  __syncwarp();
  const int c = lane & 7, rsub = lane >> 3;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int r = i * 4 + rsub;
    const float4 a = *reinterpret_cast<const float4*>(patch + r * 128 + ((c ^ (r & 7)) << 4));
    if (r < rows_left)
      *reinterpret_cast<float4*>(dst + (size_t)r * pitch + c * 4) = make_float4(a.x + b4.x, a.y + b4.y, a.z + b4.z, a.w + b4.w);
  }
  __syncwarp();
}

// SETTLE (K1 / K2 of Glom.settle): tiles of 256-row blocks whose images have all stopped are skipped by every warp role
// of both CTAs (the same flag, written by an earlier launch and read after pdl_wait, keeps the multicast and empty-barrier
// protocol in step); K2 stores nothing for rows of stopped images and also writes the squared-change partials.
// K1 of the settle queue also skips the group-0 tiles of blocks that admitted no image at this step: their group-0
// hidden activations (tokens only) are still in H from the step that admitted the block's images.
template <int MODE>
__device__ __forceinline__ bool settle_skip(const GemmParams& p, const TileInfo& t) {
  if (p.block_frozen[t.m_blk]) return true;
  return MODE == 0 && t.z == 0 && p.block_fresh != nullptr && !p.block_fresh[t.m_blk];
}

template <int MODE, int BN, bool CNT, bool SETTLE = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap map_a0,   // K1: tokens Xb (rows, d)        K2: H (rows, G*4d)
            const __grid_constant__ CUtensorMap map_a1,   // K1: state shadow Sb (rows, L*d)
            const __grid_constant__ CUtensorMap map_a2,   // K1: Sb[:,1:]+pos shadow Sp (rows, (L-1)*d)
            const __grid_constant__ CUtensorMap map_b,    // K1: W1p (G*4d, d)              K2: W2p (L*d, 8d)   box BN/2 rows
            const __grid_constant__ CUtensorMap map_out,  // K1: H, box 64 x 64 (the TMA stores)   K2 / tokeniser: unused
            const GemmParams p) {
  using Cfg = GemmCfg<MODE, BN>;
  constexpr int STAGES = Cfg::STAGES;
  constexpr bool RED = MODE != 2 && !SETTLE;     // honours GemmParams::num_m_rep (image-independent work)
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment (128-byte swizzle atoms) by pointer arithmetic on the __shared__ array (keeps the shared address
  // space visible to the compiler: LDS/STS instead of generic LD/ST for every staging / patch access)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* epi = smem + (size_t)STAGES * Cfg::STAGE_BYTES;      // K1: output tiles; K2 / tokeniser: staging, patches, exchange
  float* stg_all = reinterpret_cast<float*>(epi);
  uint8_t* patches = epi + 4 * STG_BYTES;
  float* xch = reinterpret_cast<float*>(patches + (size_t)GEMM_CONSUMER_WARPS * Cfg::PATCH_BYTES);   // [4 pairs][32]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(epi + Cfg::EPI_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;

  // warpgroup 0 = producer (its warp 0 issues the TMA loads), warpgroups 1 and 2 = consumers
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  constexpr int W_TMA = 0;
  constexpr int W_CONSUMER0 = 4;
  const int cta_rank = (int)(blockIdx.x & 1);
  const int cluster_id = blockIdx.x >> 1;
  const int num_clusters = gridDim.x >> 1;

  if (warp == W_TMA && lane == 0) {
    tma_prefetch_desc(&map_a0);
    tma_prefetch_desc(&map_b);
    if (MODE == 0) { tma_prefetch_desc(&map_a1); tma_prefetch_desc(&map_a2); tma_prefetch_desc(&map_out); }
    // a slot is free once the consumers of BOTH CTAs are done with it: the peer's producer writes half of its B tile
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 2 * GEMM_CONSUMER_WARPS); }
    fence_barrier_init();
  }
  cluster_sync_all();          // both CTAs' barriers initialised before any multicast load or remote arrive
  pdl_launch_dependents();     // the next kernel may start its own set-up on SMs we vacate
  pdl_wait();                  // ... and we touch global memory only after the previous kernel has finished
  const bool clk_thread = blockIdx.x == 0 && warp == W_TMA && lane == 0;
  // the sample's start waits in shared memory: held in a register it would be live across the consumers' code
  ClockSample* clk_s = reinterpret_cast<ClockSample*>(empty_bar + STAGES);
  if (clk_thread) *clk_s = clock_sample_begin();
  const bool cnt_cta = CNT && blockIdx.x == 0;          // wait-cycle counters (diagnostic instantiation): block 0 only
  unsigned long long* const cnt = g_kernel_clk[MODE == 0 ? PROF_GEMM1 : MODE == 1 ? PROF_GEMM2 : PROF_TOKENIZE];
  unsigned long long w0 = 0, w1 = 0;
#define GLOM_CNT_WAIT(acc, stmt) do { if (cnt_cta) { const long long t_ = clock64(); stmt; acc += (unsigned long long)(clock64() - t_); } else { stmt; } } while (0)

  if (warp < W_CONSUMER0) {
    setmaxnreg_dec<GEMM_PRODUCER_REGS>();
    if (warp == W_TMA) {
      // ------------------------------------------------------------------ TMA producer
      // warp-converged: all lanes walk the schedule and poll the barriers, the elected lane issues (see elect_one)
      const uint32_t elected = elect_one();
      int stage = 0; uint32_t phase = 0;
      const uint32_t smem0 = smem_u32(smem);
      const uint64_t pol_first = l2_policy_evict_first();
      const int kbg_n = 4 * p.d / BK;
      const int blk_skip = (p.m128 - 1) * kbg_n;
      for (int it = 0, tile; (tile = sched_tile<MODE>(p, cluster_id, num_clusters, it)) >= 0; ++it) {
        const TileInfo t = decode_tile<MODE, RED>(p, tile);
        if constexpr (SETTLE) { if (settle_skip<MODE>(p, t)) continue; }
        const CUtensorMap* amap;
        int a_col, b_row;
        if (MODE == 0) {
          const int l = t.z >> 1;
          if (t.z == 0) { amap = &map_a0; a_col = 0; }                        // bottom-up level 0 reads the tokens (:132)
          else if (t.z & 1) { amap = &map_a2; a_col = l * p.d; }              // top-down l reads S[l+1]+pos (:136)
          else { amap = &map_a1; a_col = (l - 1) * p.d; }                     // bottom-up l reads S[l-1]   (:134)
          b_row = t.z * 4 * p.d + t.n_blk * BN;
        } else if (MODE == 1) {
          amap = &map_a0; a_col = 0;             // H is stored as contiguous 16 KB (128 x 64) blocks, see below
          b_row = t.z * p.d + t.n_blk * BN;
        } else {
          amap = &map_a0; a_col = 0;               // patches (rows, Kp) x Wtok (d, Kp)
          b_row = t.n_blk * BN;
        }
        const int a_row = t.m_blk * 256 + cta_rank * BM;
        // K2: block (group g, 128-row block, 64-wide k block); [H_bu,l | H_td,l] are groups 2l and 2l+1, so k block kb
        // of the concatenation is block blk0 + kb of group 2l and, from kb = kbg_n on, of the group behind it
        const int blk0 = (2 * t.z * p.m128 + (a_row >> 7)) * kbg_n;
        int td_skip = blk_skip;
        if constexpr (RED && MODE == 1) {
          // the top-down group's H was computed for the representative blocks only: read block k mod h_period instead
          if (p.num_m_rep > 0 && t.z + 1 >= p.remap_l) td_skip -= ((a_row >> 7) - (a_row >> 7) % p.h_period) * kbg_n;
        }
        for (int kb = 0; kb < t.num_kb; ++kb) {
          GLOM_CNT_WAIT(w0, mbar_wait(&empty_bar[stage], phase ^ 1));
          if (elected) {
            const uint32_t sa = smem0 + (uint32_t)stage * Cfg::STAGE_BYTES;
            uint64_t* bar = &full_bar[stage];
            mbar_arrive_expect_tx(bar, Cfg::STAGE_BYTES);
            if (MODE == 1) {
              const int blk = blk0 + kb + (kb >= kbg_n ? td_skip : 0);
              // H streams through once per pair of column tiles: evict-first keeps it from displacing weights / state
              tma_load_2d_hint(sa, amap, bar, 0, blk * BM, pol_first);
            } else {
              tma_load_2d(sa, amap, bar, a_col + kb * BK, a_row);
            }
            // the B tile is the same in both CTAs of the pair: each loads one box of BN/2 rows and multicasts it to both
            const uint32_t b_half = (uint32_t)cta_rank * (BN / 2);
            tma_load_2d_multicast(sa + A_STAGE_BYTES + b_half * BK * 2, &map_b, bar, kb * BK, b_row + (int)b_half, 0x3);
          }
          __syncwarp();
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
      if (cnt_cta && elected) atomicAdd(&cnt[4], w0);
    }
  } else {
    // ------------------------------------------------------------------ consumers: wgmma main loop + epilogue
    setmaxnreg_inc<GEMM_CONSUMER_REGS>();
    const int cw = warp - W_CONSUMER0;       // consumer warp 0-7
    const int wg = cw >> 2, wi = cw & 3;
    const int pair = cw >> 1, x = cw & 1;    // warp pair = 32-row band `pair` of the CTA's 128 rows; x = its 32-column half
    float* stg = stg_all + pair * (STG_BYTES / 4);
    uint8_t* patch = patches + (size_t)cw * Cfg::PATCH_BYTES;
    float* xch_p = xch + pair * 32;
    const uint32_t smem0 = smem_u32(smem);
    const uint64_t pol_stream = l2_policy_evict_first();
    // K1: the thread that issues the warpgroup's TMA stores (bulk groups are tracked per thread) and the lane's part of the
    // stmatrix addresses: lanes 8i .. 8i + 7 address the rows of matrix i = (column group j & 1, row half h)
    const bool st_issuer = (threadIdx.x & 127) == 0;
    const uint32_t out_wg = smem_u32(epi) + (uint32_t)wg * (BN / 64) * Cfg::OUT_BOX_BYTES;
    const uint32_t st_row = (uint32_t)(16 * wi + 8 * ((lane >> 3) & 1) + (lane & 7)) * 128;
    const int st_jx = lane >> 4, st_sw = lane & 7;     // tile row r of this lane: r & 7 == st_sw
    const uint32_t empty_peer = mapa_shared(smem_u32(empty_bar), (uint32_t)cta_rank ^ 1u);
    auto release = [&](int slot) {     // this warp is done reading `slot`: free it for both CTAs' producers
      __syncwarp();
      if (lane == 0) { mbar_arrive(&empty_bar[slot]); mbar_arrive_cluster(empty_peer + 8u * (uint32_t)slot); }
    };
    int stage = 0; uint32_t phase = 0;
    float acc[BN / 2];
    for (int it = 0, tile; (tile = sched_tile<MODE>(p, cluster_id, num_clusters, it)) >= 0; ++it) {
      const TileInfo t = decode_tile<MODE, RED>(p, tile);
      if constexpr (SETTLE) { if (settle_skip<MODE>(p, t)) continue; }
      const int row0 = t.m_blk * 256 + cta_rank * BM + pair * 32;     // first row of this warp pair's 32-row band
      const int rows_left = p.rows - row0;                              // >= 32: whole band valid (warp-uniform)
      uint32_t live = ~0u;                                              // SETTLE, K2: bit r = row row0 + r is stored
      if constexpr (SETTLE && MODE == 1)
        live = __ballot_sync(0xffffffffu, row0 + lane < p.rows && !p.frozen[(row0 + lane) / p.n]);
      // RED, K2: this level's S_t and C hold the representative rows only; row r reads row r mod n (k2_chunk)
      bool remap = false;
      if constexpr (RED && MODE == 1) remap = p.num_m_rep > 0 && t.z >= p.remap_l;
      if (MODE == 1 && lane < rows_left) {
        // The combine reads this band's fp32 state and C lines: pull them into L2 before the main loop, so the epilogue's
        // dependent global loads hit L2 instead of paying the HBM latency
        const int src_row = remap ? (row0 + lane) % p.n : row0 + lane;
        const size_t o = ((size_t)src_row * p.L + t.z) * p.d + t.n_blk * BN + x * (BN / 2);
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
        GLOM_CNT_WAIT(w0, mbar_wait(&full_bar[stage], phase));
        const uint32_t sa = smem0 + (uint32_t)stage * Cfg::STAGE_BYTES;
        wgmma_fence_regs(acc);
        wgmma_fence();
        wgmma_kblock<BN, 0>(acc, sa + (uint32_t)wg * (A_STAGE_BYTES / 2), sa + A_STAGE_BYTES);
        wgmma_commit();
        wgmma_wait<1>();                  // the previous k-block's MMAs are complete: release its slot
        wgmma_fence_regs(acc);
        if (prev >= 0) release(prev);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      release(prev);
      const long long busy_t0 = cnt_cta ? clock64() : 0;
      if constexpr (MODE == 0) {
        // K1 epilogue on the accumulator fragment: bias + GELU per column pair, bf16x2 words into the warpgroup's output
        // tile by stmatrix, then one TMA store per 64-column box s into H block (group, 128-row block, k block s of the
        // tile): 16 KB contiguous, row pitch 64.  Each box is 64 x 64 in the 128-byte swizzle (16-byte chunk c of row r at
        // c ^ (r & 7)).  The stores drain during the next tile's main loop, so one tile per warpgroup suffices.
        // Whole 64-row boxes are stored, so in the last, padded 128-row block the rows past p.rows receive gelu(b1) (their
        // A rows are zero-filled by the TMA loads).  Only GEMM2 rows >= p.rows read them, and k2_chunk discards those
        // results and zeroes their squared-norm contribution.  A box that starts at or past p.rows is not stored: it may
        // lie in a 128-row block H does not have.
        const int wrow0 = t.m_blk * 256 + cta_rank * BM + 64 * wg;     // first row of this warpgroup's 64
        if (wrow0 < p.rows) {                                           // warpgroup-uniform
          const int hblk0 = (t.z * p.m128 + (t.m_blk * 2 + cta_rank)) * (4 * p.d / BK) + t.n_blk * (BN / BK);
          const float* bias = p.bias + (size_t)t.z * 4 * p.d + t.n_blk * BN + 2 * (lane & 3);
          // all of the tile's GELU work first, with no barrier in between: pk[16 s + 2 j + h] holds columns
          // 64 s + 8 j + 2 (lane & 3) + {0, 1} of row half h
          uint32_t pk[BN / 4];
#pragma unroll
          for (int s = 0; s < BN / 64; ++s) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const float2 b = __ldg(reinterpret_cast<const float2*>(bias + 64 * s + 8 * j));
#pragma unroll
              for (int h = 0; h < 2; ++h)
                pk[16 * s + 2 * j + h] = gelu_pair_bf16(acc[4 * (8 * s + j) + 2 * h], acc[4 * (8 * s + j) + 2 * h + 1], b.x, b.y);
            }
          }
          if (st_issuer) bulk_wait_group_read<0>();       // the previous tile's stores have read the output tile
          named_bar_sync(1 + wg, 128);
#pragma unroll
          for (int s = 0; s < BN / 64; ++s)
#pragma unroll
            for (int q = 0; q < 4; ++q)                   // column groups 2q, 2q + 1 of box s
              stmatrix_x4(out_wg + (uint32_t)s * Cfg::OUT_BOX_BYTES + st_row + ((uint32_t)((2 * q + st_jx) ^ st_sw) << 4),
                          pk[16 * s + 4 * q], pk[16 * s + 4 * q + 1], pk[16 * s + 4 * q + 2], pk[16 * s + 4 * q + 3]);
          fence_proxy_async_smem();                       // the tile -> visible to the TMA stores
          named_bar_sync(1 + wg, 128);
          if (st_issuer) {
#pragma unroll
            for (int s = 0; s < BN / 64; ++s)
              tma_store_2d_hint(&map_out, out_wg + (uint32_t)s * Cfg::OUT_BOX_BYTES, 0, (hblk0 + s) * BM + 64 * wg, pol_stream);
            bulk_commit_group();
          }
        }
      } else {
#pragma unroll 1
        for (int s = 0; s < BN / 64; ++s) {
          stage_write(acc, stg, s, wi, lane);
          named_bar_sync(1 + pair, 64);
          uint32_t v[32];
          stage_read(stg, x, lane, v);
          const int cc = 64 * s + 32 * x;                               // column of this chunk inside the tile
          if (MODE == 2) {
            float* trow = p.tok_out + (size_t)row0 * p.d + t.n_blk * BN + cc;
            const float4 b4 = __ldg(reinterpret_cast<const float4*>(p.bias + t.n_blk * BN + cc + (lane & 7) * 4));
            tok_chunk(v, b4, patch, trow, (size_t)p.d, lane, rows_left);
          } else {
            K2Chunk kc;
            kc.l = t.z; kc.L = p.L; kc.d = p.d; kc.n = p.n; kc.row0 = row0; kc.prow0 = row0 % p.n; kc.s_bcast = p.s_bcast;
            kc.remap = remap;
            kc.s32_in = p.s32_in; kc.c_in = p.c_in; kc.pos = p.pos;
            kc.s32_out = p.s32_out; kc.sb_out = p.sb_out; kc.sp_out = p.sp_out;
            const int col = t.n_blk * BN + cc;
            const float4 b4 = __ldg(reinterpret_cast<const float4*>(p.bias + (size_t)t.z * p.d + col + (lane & 7) * 4));
            float rowsq[8], rowdsq[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) rowsq[i] = rowdsq[i] = 0.f;
            const bool want_dsq = SETTLE && p.dsq_out != nullptr;         // settle: yes; forward_steps: no
            if (rows_left >= 32) k2_chunk<true, SETTLE>(v, b4, patch, kc, col, lane, 32, rowsq, live, rowdsq, want_dsq);
            else k2_chunk<false, SETTLE>(v, b4, patch, kc, col, lane, rows_left, rowsq, live, rowdsq, want_dsq);
            // one squared-norm partial per PART_COLS columns: with 64-column parts the two warps of the pair hold the two
            // 32-column halves, summed in chunk order (0 + first) + second as in prep_state_kernel.  SETTLE: the
            // squared changes take the same exchange through the second warp's transpose patch, which k2_chunk no
            // longer reads and which the pair barrier at the end of the step frees again
            int part = cc / Cfg::PART_COLS;
            bool writer = true;
            if (Cfg::PART_COLS == 64) {
              float* dxch = reinterpret_cast<float*>(patches + (size_t)(cw | 1) * Cfg::PATCH_BYTES);
              if (x == 1 && (lane & 7) == 0) {
#pragma unroll
                for (int i = 0; i < 8; ++i) xch_p[i * 4 + (lane >> 3)] = rowsq[i];
                if (want_dsq) {
#pragma unroll
                  for (int i = 0; i < 8; ++i) dxch[i * 4 + (lane >> 3)] = rowdsq[i];
                }
              }
              named_bar_sync(1 + pair, 64);
              if (x == 0) {
#pragma unroll
                for (int i = 0; i < 8; ++i) rowsq[i] += xch_p[i * 4 + (lane >> 3)];
                if (want_dsq) {
#pragma unroll
                  for (int i = 0; i < 8; ++i) rowdsq[i] += dxch[i * 4 + (lane >> 3)];
                }
              }
              writer = x == 0;
            }
            if (writer && (lane & 7) == 0) {
              const size_t po = ((size_t)row0 * p.L + t.z) * p.nparts + t.n_blk * Cfg::PARTS + part;
              float* nsq = p.nsq_out + po;
              const int ldn = p.L * p.nparts;   // row offsets r * ldn (r < 32) in 32 bits: half the registers once hoisted
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                const int r = i * 4 + (lane >> 3);
                if (r < rows_left && (!SETTLE || ((live >> r) & 1u))) {
                  nsq[(unsigned)(r * ldn)] = rowsq[i];
                  if (want_dsq) p.dsq_out[po + (unsigned)(r * ldn)] = rowdsq[i];
                }
              }
            }
          }
          named_bar_sync(1 + pair, 64);                                   // staging tile free for the next step
        }
      }
      if (cnt_cta) w1 += (unsigned long long)(clock64() - busy_t0);
    }
    if (cnt_cta && cw == 0 && lane == 0) { atomicAdd(&cnt[2], w0); atomicAdd(&cnt[6], w1); }
    if (MODE == 0 && st_issuer) bulk_wait_group<0>();   // the output tiles stay allocated until the last stores are done
  }
#undef GLOM_CNT_WAIT

  cluster_sync_all();          // no CTA exits while its peer can still multicast into it or arrive on its barriers
  if (clk_thread) clock_sample_end(*clk_s, g_kernel_clk[MODE == 0 ? PROF_GEMM1 : MODE == 1 ? PROF_GEMM2 : PROF_TOKENIZE]);
}

// =====================================================================================
// K3: consensus attention.  Persistent CTAs; a work item is (128-query tile, level l, image b).
//   Warpgroup 0 is the producer and gives up registers (setmaxnreg) to the two consumer warpgroups.  Its warp 0 streams
//   the operands through a ring of shared-memory slots with TMA; its warps 1-3 compute the next item's per-key scales
//   into one of two scale buffers (mbarrier hand-off), so the consumers never wait on the squared-norm loads.
//   phase 1: S = Q K^T per key block of KEYS keys over d: each slot holds a (Q, K) 64-column chunk; the two consumer
//            warpgroups run wgmma m64 x KEYS x 16 on 64 query rows each with S in registers and turn it in place into
//            unnormalised bf16 probabilities P in shared memory (wgmma A-operand layout, 128-byte swizzle).
//            KEYS = 256 when all keys fit one block (n <= 256): S is a single pass over d and Q is loaded once per item.
//   phase 2: O = P V in 256-wide slices of d (V read MN-major straight from the state shadow, 64 keys per ring slot),
//            O in registers, scaled by 1/rowsum and written as bf16 C: the four lanes of a row exchange their words so
//            that each stores 16 contiguous bytes (a row's quad covers 64 contiguous bytes).
// Softmax stabiliser: every key is unit-normalised, so |logit_ij| <= |S_i| d^-1/2 (Cauchy-Schwarz); that bound
// replaces the row maximum (softmax is shift-invariant) and S needs one pass.  The diagonal is never masked (its logit
// is -5e-4 or, with attend_self, ~ the bound itself), so the row sum cannot underflow while the bound stays below
// 2^BOUND_MAX; warps with a row beyond that take the exact-maximum path.
// =====================================================================================
constexpr int ATTN_CONSUMER_WARPS = 8;
constexpr int ATTN_THREADS = 128 + 32 * ATTN_CONSUMER_WARPS;
// 56 x 128 + 224 x 256 = 64,512 of the SM's 65,536 registers: the 64 x 256 fp32 S or O fragment (128 registers) and the
// softmax / output work fit the consumers, and the scale warps' loads fit the producers, without spilling
constexpr uint32_t ATTN_PRODUCER_REGS = 56;
constexpr uint32_t ATTN_CONSUMER_REGS = 224;
constexpr int ATTN_SCALE_WARPS = 3;               // producer warps 1-3: per-key scales of the next item
constexpr float ATTN_BOUND_MAX = 96.f;            // log2 units
constexpr int ATTN_SINGLE_PASS_MAX = 576;         // columns whose probabilities (128 queries x all keys) fit in shared memory
constexpr int ATTN_PASS_KEYS = 512;               // keys per pass beyond that

template <int KEYS>
struct AttnCfg {
  static_assert(KEYS == 128 || KEYS == 256, "S block = one wgmma N");
  static constexpr int MAX_KB = (KEYS == 256) ? 1 : 5;                  // key blocks per pass (<= 576 keys)
  // ring slot: Q chunk (128 x 64) + K chunk (KEYS x 64), or 64 keys x 256 columns of V (4 boxes of 64 x 64)
  static constexpr uint32_t SLOT_BYTES = A_STAGE_BYTES + (uint32_t)KEYS * BK * 2;
  static_assert(SLOT_BYTES >= 4 * 8192, "a slot holds a V chunk");
};

struct AttnParams {
  int n, L, d;
  int attend_self, mask_side, mask_d2_max;
  int n_pad16, n_pad64, nkb, nchunk;   // key padding, key blocks of KEYS, 64-key chunks
  int num_stages;
  int ntiles, num_items;               // 128-query tiles per (l, b); ntiles * L * B
  int nparts;
  const float* nsq;                    // (rows, L, nparts) squared-norm partials of the state
  __nv_bfloat16* c_out;                // (rows, L, d)
  float scale;                         // d^-1/2 (:60)
  // Key passes (n > 576 columns: the probabilities of a 128-query tile against ALL keys no longer fit in shared memory).
  // One launch handles the keys [key0, key0 + nk) (the n_pad* / nkb / nchunk fields above describe THIS range); the
  // unnormalised output and the per-row (stabiliser, row sum) are carried in fp32 scratch from pass to pass and the last
  // pass normalises and writes C.  A single pass (key0 = 0, nk = n, first = last = 1) is the plain kernel.
  int key0, nk, pass_first, pass_last;
  float* o_acc;                        // (rows, L, d) fp32
  float* ml_acc;                       // (rows, L, 2) fp32: stabiliser (log2 units), row sum
  const int* frozen;                   // SETTLE: [B] 1 = the image has stopped, its items are skipped
  // Levels [0, l_full) are items of every image, image-major; levels [l_full, L) follow for image 0 only: their state is
  // the same in every image (a forward from init_levels, DESIGN.md "Image-independent levels").  L: every item.  The
  // SETTLE instantiations ignore it (l_full = L)
  int l_full;
};

// shared-memory bytes of a pass: P (nchunk x [128 x 64] bf16), the ring, two scale buffers (rs, bnd) + key coordinates,
// barriers and the clock sample
constexpr size_t attn_fixed_smem(int nchunk, int n_pad16) {
  return 1024 /*align slack*/ + (size_t)nchunk * A_STAGE_BYTES + (size_t)n_pad16 * (2 * 2 * 4 + 4) + 256;
}
static_assert(attn_fixed_smem(4, 256) + 3 * AttnCfg<256>::SLOT_BYTES <= 232448, "n = 256: three 48 KB slots");
static_assert(attn_fixed_smem(9, 576) + 2 * AttnCfg<128>::SLOT_BYTES <= 232448, "n = 576: two 32 KB slots");

// sum of a row's squared-norm partials, in order
__device__ __forceinline__ float attn_row_norm(const float* ns, int nparts) {
  float ss = 0.f;
  if ((nparts & 3) == 0 && nparts <= 16) {      // one round trip: all partials in flight, then summed in order
    float4 q[4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
      q[i] = 4 * i < nparts ? __ldg(reinterpret_cast<const float4*>(ns) + i) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int i = 0; i < 4; ++i) ss = (((ss + q[i].x) + q[i].y) + q[i].z) + q[i].w;
  } else {
    for (int i = 0; i < nparts; ++i) ss += ns[i];
  }
  return sqrtf(ss);
}

// SETTLE (Glom.settle): the items of stopped images are skipped by all three roles (TMA warp, scale warps, consumers),
// which read the same flag after pdl_wait; the scale-buffer sequence number k counts processed items only.
template <int KEYS, bool CNT, bool SETTLE = false>
__global__ void __launch_bounds__(ATTN_THREADS, 1)
attn_kernel(const __grid_constant__ CUtensorMap map_q,    // (L*d, n, B) box (64, 128, 1)
            const __grid_constant__ CUtensorMap map_k,    // box (64, KEYS, 1)
            const __grid_constant__ CUtensorMap map_v,    // box (64, 64, 1)
            const AttnParams p) {
  using Cfg = AttnCfg<KEYS>;
  constexpr uint32_t SLOT = Cfg::SLOT_BYTES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* p_smem = smem;                                                  // nchunk x [128 x 64] bf16, SW128
  uint8_t* stages = p_smem + (size_t)p.nchunk * A_STAGE_BYTES;
  // scale buffer b: rs = sc + 2 b n_pad16 [n_pad16] per-key scales, bnd = rs + n_pad16 [n_pad16] per-row logit bounds
  float* sc = reinterpret_cast<float*>(stages + (size_t)p.num_stages * SLOT);
  uint32_t* key_hw = reinterpret_cast<uint32_t*>(sc + 4 * p.n_pad16);      // [n_pad16] (grid row << 16) | grid column
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(key_hw + p.n_pad16);
  uint64_t* empty_bar = full_bar + p.num_stages;
  uint64_t* sc_full = empty_bar + p.num_stages;                           // [2] scale buffer filled (3 scale warps)
  uint64_t* sc_empty = sc_full + 2;                                       // [2] scale buffer released (8 consumer warps)
  ClockSample* clk_s = reinterpret_cast<ClockSample*>(sc_empty + 2);

  // warpgroup 0 = producer (warp 0: TMA, warps 1-3: scales), warpgroups 1 and 2 = consumers
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  constexpr int W_TMA = 0;
  constexpr int W_CONSUMER0 = 4;
  const int nsub = (p.d + 255) / 256;                  // O slices per item
  const int per_img = p.ntiles * (SETTLE ? p.L : p.l_full);
  const int full_items = p.num_items - p.ntiles * (p.L - p.l_full);
  // item -> (image, level): image 0's image-independent levels after the items of every image
  auto item_bl = [&](int it, int& b, int& l) {
    if (SETTLE) { b = it / per_img; l = (it % per_img) / p.ntiles; }
    else attn_item(it, full_items, per_img, p.ntiles, p.l_full, b, l);
  };
  const int nkb = (KEYS == 256) ? 1 : p.nkb;           // compile-time single key block on the 256-key path
  constexpr float LOG2E = 1.4426950408889634f;

  if (warp == W_TMA && lane == 0) {
    tma_prefetch_desc(&map_q); tma_prefetch_desc(&map_k); tma_prefetch_desc(&map_v);
    for (int i = 0; i < p.num_stages; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], ATTN_CONSUMER_WARPS); }
    for (int i = 0; i < 2; ++i) { mbar_init(&sc_full[i], ATTN_SCALE_WARPS); mbar_init(&sc_empty[i], ATTN_CONSUMER_WARPS); }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();
  const bool clk_thread = blockIdx.x == 0 && warp == W_TMA && lane == 0;
  // the sample's start waits in shared memory: held in a register it would be live across the consumers' code
  if (clk_thread) *clk_s = clock_sample_begin();
  // diagnostic instantiation (GLOM_B200_WAIT_COUNTERS=1): block 0's wait / busy cycles per role, in g_kernel_clk[PROF_ATTN]:
  // [4] TMA lane waiting for a free slot, [5] consumer warp 0 waiting for operands (ring slots and scale buffers),
  // [6] its softmax work, [7] its output work
  const bool cnt_cta = CNT && blockIdx.x == 0;
  unsigned long long* const cnt = g_kernel_clk[PROF_ATTN];
  unsigned long long w0 = 0, w1 = 0, w2 = 0;
#define GLOM_CNT_WAIT(acc, stmt) do { if (cnt_cta) { const long long t_ = clock64(); stmt; acc += (unsigned long long)(clock64() - t_); } else { stmt; } } while (0)

  if (warp < W_CONSUMER0) {
    setmaxnreg_dec<ATTN_PRODUCER_REGS>();
    if (warp == W_TMA) {
      // ---------------------------------------------------------------- TMA producer, warp-converged
      const uint32_t elected = elect_one();
      int stage = 0; uint32_t phase = 0;
      const uint32_t stages0 = smem_u32(stages);
      for (int it = blockIdx.x; it < p.num_items; it += gridDim.x) {
        int b, l;
        item_bl(it, b, l);
        if constexpr (SETTLE) { if (p.frozen[b]) continue; }
        const int q0 = (it % p.ntiles) * BM;
        for (int kb = 0; kb < nkb; ++kb) {
          for (int dc = 0; dc < p.d / BK; ++dc) {
            GLOM_CNT_WAIT(w0, mbar_wait(&empty_bar[stage], phase ^ 1));
            if (elected) {
              const uint32_t s = stages0 + (uint32_t)stage * SLOT;
              mbar_arrive_expect_tx(&full_bar[stage], SLOT);
              tma_load_3d(s, &map_q, &full_bar[stage], l * p.d + dc * BK, q0, b);
              tma_load_3d(s + A_STAGE_BYTES, &map_k, &full_bar[stage], l * p.d + dc * BK, p.key0 + kb * KEYS, b);
            }
            __syncwarp();
            if (++stage == p.num_stages) { stage = 0; phase ^= 1; }
          }
        }
        for (int sp = 0; sp < nsub; ++sp) {
          for (int kc = 0; kc < p.nchunk; ++kc) {
            GLOM_CNT_WAIT(w0, mbar_wait(&empty_bar[stage], phase ^ 1));
            if (elected) {
              const uint32_t s = stages0 + (uint32_t)stage * SLOT;
              mbar_arrive_expect_tx(&full_bar[stage], 4u * 8192u);
              for (int i = 0; i < 4; ++i) {
                const int dcol = sp * 256 + i * 64;
                tma_load_3d(s + i * 8192, &map_v, &full_bar[stage], dcol < p.d ? l * p.d + dcol : p.L * p.d,
                            p.key0 + kc * 64, b);                              // past d: out of bounds -> zeros
              }
            }
            __syncwarp();
            if (++stage == p.num_stages) { stage = 0; phase ^= 1; }
          }
        }
      }
      if (cnt_cta && elected) atomicAdd(&cnt[4], w0);
    } else {
      // ---------------------------------------------------------------- scale warps: per-key scales, one item ahead
      const int t = threadIdx.x - 32;
      // key coordinates for the careful path, written once: padding keys sit 20000 rows away, so one distance test masks
      // them as well (:67-69; without a radius every real key is at (0, 0), the query at (0, 0) and the threshold 1).
      // The consumers read them only after their first scale-buffer wait, which orders them after these writes.
      const bool use_mask = p.mask_side > 0;
      for (int j = t; j < p.n_pad16; j += 32 * ATTN_SCALE_WARPS)
        key_hw[j] = j >= p.nk ? (20000u << 16)
                              : use_mask ? ((uint32_t)((p.key0 + j) / p.mask_side) << 16) | (uint32_t)((p.key0 + j) % p.mask_side) : 0u;
      int k = 0;
      for (int it = blockIdx.x; it < p.num_items; it += gridDim.x) {
        int b, l;
        item_bl(it, b, l);
        if constexpr (SETTLE) { if (p.frozen[b]) continue; }
        const size_t img_row0 = (size_t)b * p.n;
        const int buf = k & 1;
        mbar_wait(&sc_empty[buf], ((k >> 1) & 1) ^ 1);
        float* rs = sc + 2 * buf * p.n_pad16;
        float* bnd = rs + p.n_pad16;
        // per-key scale  log2(e) d^-1/2 / max(|S_j|, 1e-12)  (F.normalize eps, :58; logits are kept in log2 units)
        // and per-row bound  log2(e) d^-1/2 |S_j|  on the magnitude of row j's logits
        for (int j = t; j < p.n_pad16; j += 32 * ATTN_SCALE_WARPS) {
          float v = 0.f, bd = 0.f;
          if (j < p.nk) {
            const float nrm = attn_row_norm(p.nsq + ((img_row0 + p.key0 + j) * p.L + l) * p.nparts, p.nparts);
            v = p.scale * LOG2E / fmaxf(nrm, 1e-12f);
            bd = p.scale * LOG2E * nrm;
          }
          rs[j] = v;
          bnd[j] = bd;
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&sc_full[buf]);
        ++k;
      }
    }
  } else {
    // ---------------------------------------------------------------- consumers: 2 warpgroups x 64 query rows
    setmaxnreg_inc<ATTN_CONSUMER_REGS>();
    // thread rows (fragment layout of wgmma, see ptx.cuh): tile rows r_h = 64 wg + 16 wi + lane / 4 + 8 h, h = 0, 1;
    // fragment element i holds column 8 (i / 4) + 2 (lane % 4) + (i % 2) of row r_{(i / 2) % 2}
    const int cw = warp - W_CONSUMER0;
    const int wg = cw >> 2, wi = cw & 3;
    const int rbase = 64 * wg + 16 * wi + (lane >> 2);
    const int cq = 2 * (lane & 3);
    const float NEG_INF = __int_as_float(0xff800000);
    const bool use_mask = p.mask_side > 0;
    const uint32_t stages0 = smem_u32(stages);
    const uint32_t p0 = smem_u32(p_smem);
    int stage = 0; uint32_t phase = 0;

    const int d2_max = use_mask ? p.mask_d2_max : 1;
    // K-padding keys of the last 64-key chunk, this warpgroup's rows: P = 0, never written again (visible to the
    // warpgroup's wgmma reads through the fence + barrier before its first P V)
    const int npadk = (p.n_pad64 - p.n_pad16) >> 3;
    for (int idx = threadIdx.x & 127; idx < 64 * npadk; idx += 128) {
      const int t = 64 * wg + (idx & 63), key = p.n_pad16 + 8 * (idx >> 6);
      *reinterpret_cast<uint4*>(p_smem + (size_t)(key >> 6) * A_STAGE_BYTES + (size_t)t * 128 + ((((key & 63) >> 3) ^ (t & 7)) << 4)) =
          make_uint4(0, 0, 0, 0);
    }
    fence_proxy_async_smem();
    // bf16 pair (key, key + 1) of tile row r in P
    auto p_word = [&](int r, int key) -> uint32_t* {
      return reinterpret_cast<uint32_t*>(p_smem + (size_t)(key >> 6) * A_STAGE_BYTES + (size_t)r * 128 +
                                         ((((key & 63) >> 3) ^ (r & 7)) << 4) + (key & 7) * 2);
    };

    int k = 0;
    for (int it = blockIdx.x; it < p.num_items; it += gridDim.x) {
      int b, l;
      item_bl(it, b, l);
      if constexpr (SETTLE) { if (p.frozen[b]) continue; }
      const int q0 = (it % p.ntiles) * BM;
      const size_t img_row0 = (size_t)b * p.n;
      const long long cnt_t0 = cnt_cta ? clock64() : 0;
      const unsigned long long cnt_w0 = w0;
      const int buf = k & 1;
      GLOM_CNT_WAIT(w0, mbar_wait(&sc_full[buf], (k >> 1) & 1));     // this item's scales
      const float* rs = sc + 2 * buf * p.n_pad16;
      const float* bnd = rs + p.n_pad16;

      const bool multi = !(p.pass_first && p.pass_last);
      int qi[2];
      float row_bound[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        qi[h] = q0 + rbase + 8 * h;
        row_bound[h] = 0.f;
        if (qi[h] < p.n) {
          if (!multi) row_bound[h] = bnd[qi[h]];
          else row_bound[h] = p.scale * LOG2E * attn_row_norm(p.nsq + ((img_row0 + qi[h]) * p.L + l) * p.nparts, p.nparts);
        }
      }
      const bool exact_max = __any_sync(0xffffffffu, !(row_bound[0] <= ATTN_BOUND_MAX) || !(row_bound[1] <= ATTN_BOUND_MAX));
      float m_run[2], l_run[2] = {0.f, 0.f}, m_used[Cfg::MAX_KB][2];
#pragma unroll
      for (int h = 0; h < 2; ++h) m_run[h] = exact_max ? NEG_INF : row_bound[h];
      const int qh[2] = {use_mask ? qi[0] / p.mask_side : 0, use_mask ? qi[1] / p.mask_side : 0};
      const int qw[2] = {use_mask ? qi[0] % p.mask_side : 0, use_mask ? qi[1] % p.mask_side : 0};
      const int wrow0 = q0 + 64 * wg + 16 * wi;                 // first query of this warp's 16 rows

#pragma unroll 1
      for (int kb = 0; kb < nkb; ++kb) {
        float s[KEYS / 2];
#pragma unroll
        for (int i = 0; i < KEYS / 2; ++i) s[i] = 0.f;
        int prev = -1;                    // slot of the k-block whose MMAs may still be running
        for (int dc = 0; dc < p.d / BK; ++dc) {
          GLOM_CNT_WAIT(w0, mbar_wait(&full_bar[stage], phase));
          const uint32_t sa = stages0 + (uint32_t)stage * SLOT;
          wgmma_fence_regs(s);
          wgmma_fence();
          wgmma_kblock<KEYS, 0>(s, sa + (uint32_t)wg * (A_STAGE_BYTES / 2), sa + A_STAGE_BYTES);
          wgmma_commit();
          wgmma_wait<1>();                  // the previous k-block's MMAs are complete: release its slot
          wgmma_fence_regs(s);
          if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty_bar[prev]); }
          prev = stage;
          if (++stage == p.num_stages) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        wgmma_fence_regs(s);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
        const int kbase = kb * KEYS;                            // pass-local index of the block's first key
        const int w = min(KEYS, p.n_pad16 - kbase);
        // logits (log2 units).  Blocks of real keys without a radius mask (every block of configs[1]) take one multiply
        // and one diagonal select per key, in straight-line code: per-element branches between the variants would
        // leave the two consumer warps of each scheduler waiting on branch and dependency latency.  The others take
        // the select chain of the reference's masking.
        const int gk0 = p.key0 + kbase;
        const bool plain_keys = !use_mask && kbase + KEYS <= p.nk;      // implies w == KEYS
        if (plain_keys) {
          // key 8 jj + e of this lane's columns is row h's diagonal iff 8 jj + e == dq[h]; -1 never matches
          const bool diag = !p.attend_self && wrow0 + 16 > gk0 && wrow0 < gk0 + KEYS;
          const int dq[2] = {diag ? qi[0] - gk0 - cq : -1, diag ? qi[1] - gk0 - cq : -1};
#pragma unroll
          for (int jj = 0; jj < KEYS / 8; ++jj) {
            const float2 r2 = *reinterpret_cast<const float2*>(rs + kbase + 8 * jj + cq);
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const float sv = s[4 * jj + 2 * h + e] * (e ? r2.y : r2.x);                   // (:60)
                s[4 * jj + 2 * h + e] = (8 * jj + e == dq[h]) ? -5e-4f * LOG2E : sv;         // (:62-65)
              }
          }
        } else {
#pragma unroll
          for (int jj = 0; jj < KEYS / 8; ++jj) {
            const int col = 8 * jj + cq;
            if (col < w) {
              const int j = kbase + col;
              const float2 r2 = *reinterpret_cast<const float2*>(rs + j);
#pragma unroll
              for (int h = 0; h < 2; ++h) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  float sv = s[4 * jj + 2 * h + e] * (e ? r2.y : r2.x);                       // (:60)
                  sv = (!p.attend_self && p.key0 + j + e == qi[h]) ? -5e-4f * LOG2E : sv;     // (:62-65)
                  const uint32_t hw = key_hw[j + e];
                  const int dh = qh[h] - (int)(hw >> 16), dw = qw[h] - (int)(hw & 0xFFFFu);
                  sv = (dh * dh + dw * dw > d2_max) ? NEG_INF : sv;                           // (:67-69) and key padding
                  s[4 * jj + 2 * h + e] = sv;
                }
              }
            } else {
#pragma unroll
              for (int e = 0; e < 4; ++e) s[4 * jj + e] = NEG_INF;
            }
          }
        }
        float m_safe[2] = {m_run[0], m_run[1]};
        if (exact_max) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float bm = NEG_INF;
#pragma unroll
            for (int i = 0; i < KEYS / 2; ++i) if (((i >> 1) & 1) == h) bm = fmaxf(bm, s[i]);
            bm = fmaxf(bm, __shfl_xor_sync(0xffffffffu, bm, 1));
            bm = fmaxf(bm, __shfl_xor_sync(0xffffffffu, bm, 2));
            const float m_new = fmaxf(m_run[h], bm);
            m_safe[h] = (m_new == NEG_INF) ? 0.f : m_new;
            l_run[h] *= (m_run[h] == NEG_INF) ? 0.f : ex2_approx(m_run[h] - m_safe[h]);
            m_run[h] = m_new;
          }
        }
        // unnormalised probabilities 2^(logit - m) -> bf16 P and their running sum (a whole block: no column test)
        auto probs = [&](auto full) {
#pragma unroll
          for (int jj = 0; jj < KEYS / 8; ++jj) {
            const int col = 8 * jj + cq;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const float e0 = ex2_approx(s[4 * jj + 2 * h] - m_safe[h]), e1 = ex2_approx(s[4 * jj + 2 * h + 1] - m_safe[h]);
              l_run[h] += e0 + e1;
              if (decltype(full)::value || col < w) *p_word(rbase + 8 * h, kbase + col) = pack_bf16x2(e0, e1);
            }
          }
        };
        if (w == KEYS) probs(std::true_type{});
        else probs(std::false_type{});
#pragma unroll
        for (int i = 0; i < Cfg::MAX_KB; ++i)             // static indices: m_used stays in registers
          if (i == kb) { m_used[i][0] = m_safe[0]; m_used[i][1] = m_safe[1]; }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&sc_empty[buf]);             // done with this item's scales
      if (exact_max) {
        // bring every block's probabilities onto the final stabiliser
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float m_fin = (m_run[h] == NEG_INF) ? 0.f : m_run[h];
#pragma unroll
          for (int kb = 0; kb < Cfg::MAX_KB; ++kb) {
            if (kb >= nkb || m_used[kb][h] == m_fin) continue;
            const float f = ex2_approx(m_used[kb][h] - m_fin);
            const int w = min(KEYS, p.n_pad16 - kb * KEYS);
            for (int col = cq; col < w; col += 8) {
              uint32_t* ptr = p_word(rbase + 8 * h, kb * KEYS + col);
              const uint32_t wv = *ptr;
              *ptr = pack_bf16x2(__uint_as_float(wv << 16) * f, __uint_as_float(wv & 0xFFFF0000u) * f);
            }
          }
        }
      }
      float l_pass[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        l_pass[h] = l_run[h] + __shfl_xor_sync(0xffffffffu, l_run[h], 1);
        l_pass[h] += __shfl_xor_sync(0xffffffffu, l_pass[h], 2);
      }
      fence_proxy_async_smem();                // this warpgroup's P rows -> visible to its wgmma reads
      named_bar_sync(2 + wg, 128);
      const long long cnt_t1 = cnt_cta ? clock64() : 0;
      const unsigned long long cnt_w1 = w0;
      if (cnt_cta) w1 += (unsigned long long)(cnt_t1 - cnt_t0) - (cnt_w1 - cnt_w0);       // softmax work (waits excluded)

      // key passes: this row's carried (stabiliser, row sum)
      size_t acc_row[2];
      float inv_l[2], f_old[2] = {0.f, 0.f}, f_new[2] = {1.f, 1.f};
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        acc_row[h] = (img_row0 + (size_t)qi[h]) * p.L + l;
        inv_l[h] = 1.0f / l_pass[h];
        if (multi) {
          float m_acc = NEG_INF, l_acc = 0.f;
          if (!p.pass_first && qi[h] < p.n) {
            const float2 ml = *reinterpret_cast<const float2*>(p.ml_acc + acc_row[h] * 2);
            m_acc = ml.x; l_acc = ml.y;
          }
          // partial results of different key ranges are on different stabilisers only for rows on the exact-maximum path
          float m_pass = exact_max ? m_run[h] : row_bound[h];
          if (l_pass[h] == 0.f) m_pass = NEG_INF;                       // no unmasked key in this range
          const float m_new = fmaxf(m_acc, m_pass);
          f_old[h] = (m_acc == NEG_INF) ? 0.f : ex2_approx(m_acc - m_new);
          f_new[h] = (m_pass == NEG_INF) ? 0.f : ex2_approx(m_pass - m_new);
          const float l_new = l_acc * f_old[h] + l_pass[h] * f_new[h];
          inv_l[h] = p.pass_last ? 1.0f / l_new : 1.0f;
          __syncwarp();                                                 // every lane of the row has read the carried pair
          if (!p.pass_last && (lane & 3) == 0 && qi[h] < p.n)
            *reinterpret_cast<float2*>(p.ml_acc + acc_row[h] * 2) = make_float2(m_new, l_new);
        }
      }

      // output: O slice (64 rows x 256 columns per warpgroup), scaled by 1/rowsum, bf16
#pragma unroll 1
      for (int sp = 0; sp < nsub; ++sp) {
        float o[128];
#pragma unroll
        for (int i = 0; i < 128; ++i) o[i] = 0.f;
        int prev = -1;                    // slot of the k-block whose MMAs may still be running
        for (int kc = 0; kc < p.nchunk; ++kc) {
          GLOM_CNT_WAIT(w0, mbar_wait(&full_bar[stage], phase));
          const uint32_t sa = stages0 + (uint32_t)stage * SLOT;
          wgmma_fence_regs(o);
          wgmma_fence();
          wgmma_kblock<256, 1>(o, p0 + (uint32_t)kc * A_STAGE_BYTES + (uint32_t)wg * (A_STAGE_BYTES / 2), sa);
          wgmma_commit();
          wgmma_wait<1>();                  // the previous k-block's MMAs are complete: release its slot
          wgmma_fence_regs(o);
          if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty_bar[prev]); }
          prev = stage;
          if (++stage == p.num_stages) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        wgmma_fence_regs(o);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
        if (multi) {
#pragma unroll
          for (int i = 0; i < 128; i += 2) {
            const int h = (i >> 1) & 1;
            const int col = sp * 256 + 8 * (i >> 2) + cq;               // columns past d hold zeros
            if (col >= p.d || qi[h] >= p.n) continue;
            float v0 = o[i], v1 = o[i + 1];
            float2* accp = reinterpret_cast<float2*>(p.o_acc + acc_row[h] * p.d + col);
            float2 prev = make_float2(0.f, 0.f);
            if (!p.pass_first) prev = *accp;
            v0 = v0 * f_new[h] + prev.x * f_old[h];
            v1 = v1 * f_new[h] + prev.y * f_old[h];
            if (!p.pass_last) { *accp = make_float2(v0, v1); continue; }
            *reinterpret_cast<uint32_t*>(p.c_out + acc_row[h] * p.d + col) = pack_bf16x2(v0 * inv_l[h], v1 * inv_l[h]);
          }
        } else {
          // Lane q of a row's quad holds word t of every group of 4 column octets (columns 32 g + 8 t + 2 q, + 1).  A 4 x 4
          // transpose across the quad (two xor-shuffle rounds) gives lane q all 4 words of octet q: 16 contiguous bytes.
          const int q = lane & 3;
          const bool b1 = q & 1, b2 = q & 2;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            __nv_bfloat16* crow = p.c_out + acc_row[h] * p.d + sp * 256 + 8 * q;
            const bool row_ok = qi[h] < p.n;
#pragma unroll
            for (int g = 0; g < 8; ++g) {
              uint32_t a[4];
#pragma unroll
              for (int t = 0; t < 4; ++t)
                a[t] = pack_bf16x2(o[4 * (4 * g + t) + 2 * h] * inv_l[h], o[4 * (4 * g + t) + 2 * h + 1] * inv_l[h]);
#pragma unroll
              for (int pr = 0; pr < 2; ++pr) {          // swap the words whose lane and word bit 0 differ
                const uint32_t r = __shfl_xor_sync(0xffffffffu, b1 ? a[2 * pr] : a[2 * pr + 1], 1);
                if (b1) a[2 * pr] = r; else a[2 * pr + 1] = r;
              }
#pragma unroll
              for (int pr = 0; pr < 2; ++pr) {          // ... then those whose bit 1 differs
                const uint32_t r = __shfl_xor_sync(0xffffffffu, b2 ? a[pr] : a[2 + pr], 2);
                if (b2) a[pr] = r; else a[2 + pr] = r;
              }
              if (row_ok && sp * 256 + 32 * g < p.d)   // d is a multiple of 64: a 32-column group is all in or all out
                *reinterpret_cast<uint4*>(crow + 32 * g) = make_uint4(a[0], a[1], a[2], a[3]);
            }
          }
        }
      }
      if (cnt_cta) w2 += (unsigned long long)(clock64() - cnt_t1) - (w0 - cnt_w1);          // output work
      ++k;
    }
    if (cnt_cta && cw == 0 && lane == 0) { atomicAdd(&cnt[5], w0); atomicAdd(&cnt[6], w1); atomicAdd(&cnt[7], w2); }
  }
#undef GLOM_CNT_WAIT

  __syncthreads();
  if (clk_thread) clock_sample_end(*clk_s, g_kernel_clk[PROF_ATTN]);
}

// cycles / ns accumulated by the kernels of this translation unit since the last call (and reset)
cudaError_t tc_kernel_clocks(unsigned long long* out /* [PROF_KINDS][8] */, bool reset) {
  cudaError_t e = cudaMemcpyFromSymbol(out, g_kernel_clk, sizeof(unsigned long long) * PROF_KINDS * 8);
  if (e == cudaSuccess && reset) {
    static const unsigned long long zeros[PROF_KINDS * 8] = {};
    e = cudaMemcpyToSymbol(g_kernel_clk, zeros, sizeof(zeros));
  }
  return e;
}

// =====================================================================================
// Host side: tensor maps + launches for one Jacobi step
// =====================================================================================
template <int MODE, int BN, bool CNT, bool SETTLE = false>
static cudaError_t launch_gemm_impl(const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& a2, const CUtensorMap& bm,
                                    const CUtensorMap& out, const GemmParams& p, int num_sms, cudaStream_t st);

// GLOM_B200_WAIT_COUNTERS=1 (diagnostics): the kernel instantiations whose block 0 accumulates its roles' wait cycles
static bool count_waits() {
  static const bool on = [] { const char* ev = getenv("GLOM_B200_WAIT_COUNTERS"); return ev && ev[0] == '1'; }();
  return on;
}

template <int MODE, int BN>
static cudaError_t launch_gemm(const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& a2, const CUtensorMap& bm,
                               const CUtensorMap& out, const GemmParams& p, int num_sms, cudaStream_t st) {
  // Glom.settle: the instantiation that skips stopped images (no wait-counting variant)
  if constexpr (MODE != 2) {
    if (p.block_frozen) return launch_gemm_impl<MODE, BN, false, true>(a0, a1, a2, bm, out, p, num_sms, st);
  }
  if (count_waits()) return launch_gemm_impl<MODE, BN, true>(a0, a1, a2, bm, out, p, num_sms, st);
  return launch_gemm_impl<MODE, BN, false>(a0, a1, a2, bm, out, p, num_sms, st);
}

template <int MODE, int BN, bool CNT, bool SETTLE>
static cudaError_t launch_gemm_impl(const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& a2, const CUtensorMap& bm,
                                    const CUtensorMap& out, const GemmParams& p, int num_sms, cudaStream_t st) {
  using Cfg = GemmCfg<MODE, BN>;
  static SmemOptIn optin;
  if (cudaError_t e = optin.ensure(gemm_kernel<MODE, BN, CNT, SETTLE>, Cfg::SMEM_BYTES)) return e;
  cudaLaunchConfig_t cfg{};
  cfg.blockDim = dim3(Cfg::THREADS);
  cfg.dynamicSmemBytes = Cfg::SMEM_BYTES;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;      // PDL: see pdl_wait() in the kernel
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  attr[1].id = cudaLaunchAttributeClusterDimension;                     // the pair shares its B tiles (multicast)
  attr[1].val.clusterDim.x = 2; attr[1].val.clusterDim.y = 1; attr[1].val.clusterDim.z = 1;
  // Both CTAs of a cluster need an SM of the same GPC, so fewer than num_sms / 2 pairs may be co-resident; a grid beyond
  // that would run its last clusters as a second wave.  The co-resident count is a property of the device (queried once
  // per device for its full SM count); num_sms, which the SM-count target may lower, bounds it on every call.
  static std::atomic<int> co_resident[64];
  int dev = 0;
  if (cudaError_t e = cudaGetDevice(&dev)) return e;
  if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
  int occ = co_resident[dev].load(std::memory_order_relaxed);
  if (occ == 0) {
    int dev_sms = 0;
    if (cudaError_t e = cudaDeviceGetAttribute(&dev_sms, cudaDevAttrMultiProcessorCount, dev)) return e;
    cfg.gridDim = dim3(2 * (dev_sms / 2));
    cfg.attrs = &attr[1]; cfg.numAttrs = 1;
    if (cudaError_t e = cudaOccupancyMaxActiveClusters(&occ, gemm_kernel<MODE, BN, CNT, SETTLE>, &cfg)) return e;
    if (occ < 1) return cudaErrorInvalidConfiguration;
    co_resident[dev].store(occ, std::memory_order_relaxed);
  }
  const int max_pairs = occ < num_sms / 2 ? occ : num_sms / 2;
  cfg.attrs = attr; cfg.numAttrs = 2;
  const int pairs = p.num_tiles < max_pairs ? p.num_tiles : max_pairs;
  cfg.gridDim = dim3(2 * pairs);
  return cudaLaunchKernelEx(&cfg, gemm_kernel<MODE, BN, CNT, SETTLE>, a0, a1, a2, bm, out, p);
}

template <int KEYS, bool CNT, bool SETTLE = false>
static cudaError_t launch_attn_impl(const CUtensorMap& mq, const CUtensorMap& mk, const CUtensorMap& mv, const AttnParams& ap,
                                    size_t smem, int ctas, cudaStream_t st) {
  static SmemOptIn optin;
  if (cudaError_t e = optin.ensure(attn_kernel<KEYS, CNT, SETTLE>, smem)) return e;
  cudaLaunchConfig_t acfg{};
  acfg.gridDim = dim3(ctas); acfg.blockDim = dim3(ATTN_THREADS); acfg.dynamicSmemBytes = smem; acfg.stream = st;
  cudaLaunchAttribute aattr[1];
  aattr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;      // PDL: see pdl_wait() in the kernel
  aattr[0].val.programmaticStreamSerializationAllowed = 1;
  acfg.attrs = aattr; acfg.numAttrs = 1;
  return cudaLaunchKernelEx(&acfg, attn_kernel<KEYS, CNT, SETTLE>, mq, mk, mv, ap);
}

// K3: consensus attention -> C.  Levels [l_full, L) run for image 0 only (see AttnParams::l_full)
static int launch_attention(const Geometry& g, const Bf16Buffers& b, int l_full, Launch& ln) {
  const int d = g.d, L = g.L, n = g.n;
  // Up to 576 columns the probabilities of a 128-query tile against all keys fit in shared memory: one launch.  Beyond,
  // the keys are processed in passes of ATTN_PASS_KEYS (one launch each, see AttnParams): no shape falls to CUDA cores.
  const int npass = (n <= ATTN_SINGLE_PASS_MAX) ? 1 : (n + ATTN_PASS_KEYS - 1) / ATTN_PASS_KEYS;
  if (npass > 1 && !b.attn_acc)
    return ln.fail(GLOM_B200_ERR_CUDA, "consensus for n = %d columns needs the key-pass scratch buffer (workspace too old?)", n);
  // All keys of a single pass of more than 128 and at most 256 (padded) keys form one 256-key S block; every other
  // pass uses 128-key blocks
  const int keys = (npass == 1 && (n + 15) / 16 * 16 > 128 && (n + 15) / 16 * 16 <= 256) ? 256 : 128;
  CUtensorMap mq, mk, mv;
  const uint64_t dims[3] = {(uint64_t)L * d, (uint64_t)n, (uint64_t)g.B};
  const uint64_t strides[2] = {(uint64_t)L * d * 2, (uint64_t)n * L * d * 2};
  const uint32_t boxq[3] = {(uint32_t)BK, (uint32_t)BM, 1}, boxk[3] = {(uint32_t)BK, (uint32_t)keys, 1};
  const uint32_t boxv[3] = {(uint32_t)BK, 64, 1};
  GLOM_TRY(encode_map(ln, &mq, b.sb_in, 3, dims, strides, boxq, "attn.q"));
  GLOM_TRY(encode_map(ln, &mk, b.sb_in, 3, dims, strides, boxk, "attn.k"));
  GLOM_TRY(encode_map(ln, &mv, b.sb_in, 3, dims, strides, boxv, "attn.v"));
  const bool cnt = count_waits();
  cudaStream_t st = ln.st;
  for (int pass = 0; pass < npass; ++pass) {
    AttnParams ap{};
    ap.n = n; ap.L = L; ap.d = d;
    ap.attend_self = g.attend_self; ap.mask_side = g.mask_side; ap.mask_d2_max = g.mask_d2_max;
    ap.key0 = npass == 1 ? 0 : pass * ATTN_PASS_KEYS;
    ap.nk = npass == 1 ? n : (n - ap.key0 < ATTN_PASS_KEYS ? n - ap.key0 : ATTN_PASS_KEYS);
    ap.pass_first = pass == 0; ap.pass_last = pass == npass - 1;
    ap.o_acc = b.attn_acc;
    ap.ml_acc = b.attn_acc ? b.attn_acc + (size_t)g.rows * L * d : nullptr;
    ap.n_pad16 = (ap.nk + 15) / 16 * 16;
    ap.n_pad64 = (ap.nk + 63) / 64 * 64;
    ap.nkb = (ap.n_pad16 + keys - 1) / keys;
    ap.nchunk = ap.n_pad64 / 64;
    ap.nparts = g.nparts;
    ap.nsq = b.nsq_in;
    ap.c_out = b.c;
    ap.scale = 1.0f / sqrtf((float)d);
    ap.ntiles = (n + BM - 1) / BM;
    ap.l_full = l_full;
    ap.num_items = ap.ntiles * (l_full * g.B + L - l_full);
    ap.frozen = b.frozen;
    // 256 keys: 3 slots of 48 KB next to 64 KB of P (n = 256: 219,392 B); 128 keys: 2 slots of 32 KB at 576 keys
    const uint32_t slot = keys == 256 ? AttnCfg<256>::SLOT_BYTES : AttnCfg<128>::SLOT_BYTES;
    const size_t fixed = attn_fixed_smem(ap.nchunk, ap.n_pad16);
    const size_t max_smem = 232448;                       // the 227 KB of shared memory a block may opt in to
    int stages = 4;
    while (stages > 0 && fixed + (size_t)stages * slot > max_smem) --stages;
    // the consumers release a slot only after the next one's MMAs are issued: the ring needs two slots
    if (stages < 2 || ap.nkb > (keys == 256 ? AttnCfg<256>::MAX_KB : AttnCfg<128>::MAX_KB))
      return ln.fail(GLOM_B200_ERR_CUDA, "consensus pass of %d keys does not fit shared memory", ap.nk);
    ap.num_stages = stages;
    const size_t smem = fixed + (size_t)stages * slot;
    const int ctas = ap.num_items < ln.num_sms ? ap.num_items : ln.num_sms;
    ProfScope scope(ln.prof, PROF_ATTN, st);
    cudaError_t e;
    if (b.frozen) e = keys == 256 ? launch_attn_impl<256, false, true>(mq, mk, mv, ap, smem, ctas, st)
                                  : launch_attn_impl<128, false, true>(mq, mk, mv, ap, smem, ctas, st);
    else if (keys == 256) e = cnt ? launch_attn_impl<256, true>(mq, mk, mv, ap, smem, ctas, st)
                                          : launch_attn_impl<256, false>(mq, mk, mv, ap, smem, ctas, st);
    else e = cnt ? launch_attn_impl<128, true>(mq, mk, mv, ap, smem, ctas, st)
                         : launch_attn_impl<128, false>(mq, mk, mv, ap, smem, ctas, st);
    GLOM_TRY(ln.launched(e, "attn_kernel launch"));
  }
  return 0;
}

int step_bf16(const Geometry& g, const Bf16Buffers& b, int step_index, Launch& ln) {
  const int d = g.d, L = g.L, n = g.n, rows = g.rows, num_sms = ln.num_sms;
  cudaStream_t st = ln.st;
  // One launch each of K1 (all groups), K3, K2 (all levels).
  // H: (group, 128-row block, 64-column k block) blocks of 128 x 64, read by K2 a block at a time (mh) and written by
  // K1 a warpgroup's 64 rows at a time (mh_out)
  CUtensorMap mh, mh_out;
  const int m128 = (rows + BM - 1) / BM;
  const uint64_t h_rows = (uint64_t)g.G * m128 * (4 * d / BK) * BM;
  GLOM_TRY(map2d(ln, &mh, b.h, h_rows, BK, BM, "H"));
  GLOM_TRY(map2d(ln, &mh_out, b.h, h_rows, BK, 64, "H out"));
  CUtensorMap mx, msb, msp, mw1, mw2;
  GLOM_TRY(map2d(ln, &mx, b.xb, rows, d, BM, "Xb"));
  GLOM_TRY(map2d(ln, &msb, b.sb_in, rows, (uint64_t)L * d, BM, "Sb"));
  GLOM_TRY(map2d(ln, &msp, b.sp_in, rows, (uint64_t)(L - 1) * d, BM, "Sp"));
  GLOM_TRY(map2d(ln, &mw1, b.w1, (uint64_t)g.G * 4 * d, d, 128, "W1p"));
  GLOM_TRY(map2d(ln, &mw2, b.w2, (uint64_t)L * d, (uint64_t)8 * d, (uint32_t)g.bn2 / 2, "W2p"));
  // ---------------- K1: grouped GEMM1 + bias + GELU -> H   (all 2L-1 groups)
  {
    GemmParams p{};
    p.rows = rows; p.d = d; p.L = L; p.n = n; p.G = g.G;
    // group 0 (bottom-up net of level 0) reads the tokens, which are the same in every step of a call (:132-134): its block
    // of H is written by the call's first step and stays valid; the later steps run the other 2L - 2 groups only.
    // The groups are walked upward from z0, and every H box is stored evict-first: H streams through L2 and must not
    // displace the weights and state shadows that the GEMMs and the consensus kernel re-read
    // The settle queue (b.block_fresh) admits images at any step: group 0 is in every launch, and its tiles run only for
    // the row blocks that admitted an image at this step.
    p.z0 = (step_index > 0 && g.G > 1 && !b.block_fresh) ? 1 : 0;
    p.num_m = (rows + 255) / 256; p.num_n = 4 * d / 256; p.num_tiles = (g.G - p.z0) * p.num_m * p.num_n;
    p.bias = b.b1; p.m128 = m128;
    p.frozen = b.frozen; p.block_frozen = b.block_frozen; p.block_fresh = b.block_fresh;
    // a forward from init_levels: the groups whose input is the same in every image run the representative rows only
    if (b.ii_reduce) set_reduced(p, g.G, rep_row_blocks(n), [&](int z) { return ii_k1_full(z, step_index); });
    ProfScope scope(ln.prof, PROF_GEMM1, st);
    GLOM_TRY(ln.launched(launch_gemm<0, 256>(mx, msb, msp, mw1, mh_out, p, num_sms, st), "gemm1 launch"));
  }
  // ---------------- K3 between K1 and K2 (C is then written shortly before K2's epilogue reads it)
  GLOM_TRY(launch_attention(g, b, b.ii_reduce ? ii_k3_full_levels(step_index) : L, ln));
  // ---------------- K2: grouped GEMM2 + combine -> state t+1 (+ shadows, norms)   (all levels)
  {
    GemmParams p{};
    p.rows = rows; p.d = d; p.L = L; p.n = n; p.G = g.G;
    p.num_m = (rows + 255) / 256; p.num_n = d / g.bn2; p.z0 = 0; p.num_tiles = L * p.num_m * p.num_n;
    p.n_half = p.num_m * p.num_n;
    p.m128 = m128;
    p.bias = b.b2; p.s32_in = b.s32_in; p.s_bcast = b.s32_in_bcast; p.c_in = b.c; p.pos = b.pos;
    p.s32_out = b.s32_out; p.sb_out = b.sb_out; p.sp_out = b.sp_out; p.nsq_out = b.nsq_out; p.nparts = g.nparts;
    p.frozen = b.frozen; p.block_frozen = b.block_frozen; p.dsq_out = b.dsq_out;
    if (b.ii_reduce) {     // S_{t+1}[l] differs between images only for l <= t; the top level stays last (half cost)
      set_reduced(p, L, rep_row_blocks(n), [&](int l) { return ii_k2_full(l, step_index); });
      p.n_half = (L - 1 <= step_index ? p.num_m : p.num_m_rep) * p.num_n;
      p.remap_l = step_index; p.h_period = rep_h_blocks(n);
    }
    cudaError_t e;
    ProfScope scope(ln.prof, PROF_GEMM2, st);
    if (g.bn2 == 256) e = launch_gemm<1, 256>(mh, mh, mh, mw2, mh, p, num_sms, st);
    else if (g.bn2 == 128) e = launch_gemm<1, 128>(mh, mh, mh, mw2, mh, p, num_sms, st);
    else e = launch_gemm<1, 64>(mh, mh, mh, mw2, mh, p, num_sms, st);
    GLOM_TRY(ln.launched(e, "gemm2 launch"));
  }
  return 0;
}


// ---------------- tensor-core tokeniser: tokens = patches(bf16) . Wtok(bf16)^T + bias   (glom_pytorch.py:94-97)
int tokenize_tc(const __nv_bfloat16* patches, const __nv_bfloat16* wtok, const float* bias, float* tokens, int rows,
                int d, int kp, Launch& ln) {
  const int num_sms = ln.num_sms;
  cudaStream_t st = ln.st;
  const int bn = (d % 256 == 0) ? 256 : (d % 128 == 0) ? 128 : 64;
  CUtensorMap ma, mb;
  GLOM_TRY(map2d(ln, &ma, patches, rows, kp, BM, "patches"));
  GLOM_TRY(map2d(ln, &mb, wtok, d, kp, (uint32_t)bn / 2, "Wtok"));
  GemmParams p{};
  p.rows = rows; p.d = d; p.L = 1; p.n = 1; p.G = 1;
  p.num_m = (rows + 255) / 256; p.num_n = d / bn; p.num_tiles = p.num_m * p.num_n;
  p.bias = bias; p.tok_out = tokens; p.tok_kb = kp / BK;
  cudaError_t e;
  if (bn == 256) e = launch_gemm<2, 256>(ma, ma, ma, mb, ma, p, num_sms, st);
  else if (bn == 128) e = launch_gemm<2, 128>(ma, ma, ma, mb, ma, p, num_sms, st);
  else e = launch_gemm<2, 64>(ma, ma, ma, mb, ma, p, num_sms, st);
  return ln.launched(e, "tokeniser gemm launch");
}

}  // namespace glom
