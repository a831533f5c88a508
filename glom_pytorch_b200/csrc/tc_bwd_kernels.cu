// Tensor-core backward of the two grouped MLPs.
//
// Per reverse step and MLP group g (bottom-up l / top-down l), with x the group's input rows, dY = dL/dS_{t+1}[:, l]/c_l:
//   P  : pre  = x W1^T + b1 ;  h = gelu(pre), gp = gelu'(pre)  (NT GEMM, K = d) -> bf16, 16 KB blocks like the forward's H
//   H  : dh   = dY W2 ;  dpre = dh * gp                        (NT GEMM, K = d, B = W2^T)   -> dpre blocks
//   X  : dx   = dpre W1                          (NT GEMM, K = 4d, B = W1^T)  -> fp32 (R, G, d)
//   W  : dW2 += dY^T h ;  dW1 += dpre^T x        (TN GEMMs, K = rows; both operands read MN-major by TMA)
// All four use the forward's pipeline structure (tc_kernels.cu): 256 x 256 tiles dealt to pairs of CTAs that compute 128
// rows each, a TMA producer warp feeding 128B-swizzled smem stages, two wgmma consumer warpgroups with register
// accumulators that run the epilogue, bounded mbarrier waits.  The attention backward, reductions and the scatter of dx stay on CUDA cores (bwd_kernels.cu).
// The deterministic backward (MlpBwdTc::deterministic) runs the DET instantiations of DH and DX, whose epilogues store
// what the default ones add with red.add atomics (see BwdParams::dx_td / b1_part and DESIGN.md).
#include "tc_common.cuh"

#include <stdio.h>

namespace glom {

namespace {

constexpr int BN = 256;
constexpr uint32_t A_BYTES = BM * BK * 2;          // 16 KB: this CTA's A tile (128 rows or 128 M-columns x 64 k)
constexpr uint32_t B_BYTES = BN * BK * 2;          // 32 KB: the B tile
constexpr uint32_t STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int STAGES = 3;
constexpr int CONSUMER_WARPS = 8;
constexpr int THREADS = 32 * (CONSUMER_WARPS + 1);
constexpr uint32_t PATCH_BYTES = 4096;
constexpr size_t SMEM_BYTES = 1024 + (size_t)STAGES * STAGE_BYTES + 4 * (size_t)STG_BYTES + (size_t)CONSUMER_WARPS * PATCH_BYTES +
                              BN * 4 + 256;

// one k-block for warpgroup `wg`; TA / TB: operand MN-major (64-wide boxes 8 KB apart) instead of K-major
template <int TA, int TB>
__device__ __forceinline__ void kblock(float (&acc)[BN / 2], uint32_t a_smem, uint32_t b_smem) {
  const uint64_t ad = TA ? wgmma_desc_sw128(a_smem, 8192, 1024) : wgmma_desc_sw128(a_smem, 16, 1024);
  const uint64_t bd = TB ? wgmma_desc_sw128(b_smem, 8192, 1024) : wgmma_desc_sw128(b_smem, 16, 1024);
#pragma unroll
  for (int k = 0; k < BK / 16; ++k) wgmma_bf16<BN, TA, TB>(acc, ad + (TA ? (2048 >> 4) : 2) * k, bd + (TB ? (2048 >> 4) : 2) * k);
}

enum { BW_PRE = 0, BW_DH = 1, BW_DX = 2, BW_DW = 3, BW_BATCH = 4 };

struct BwdParams {
  int rows, d, L, n, G;
  int m128;            // 128-row blocks of the blocked (R_pad, G*4d) buffers
  int num_tiles;
  const float* b1p;    // (G*4d) first-layer biases in group order
  // blocked bf16 buffers [G][m128][4d/64][128][64]
  __nv_bfloat16* pre;
  __nv_bfloat16* h;
  __nv_bfloat16* dpre;
  float *ds, *d_tokens, *d_pos;   // BW_DX reduces dx of group g into dL/dS_t level l-1 (bottom-up l; tokens for l = 0) or
                                  // l+1 (top-down l, which also feeds dL/dpos, :136)
  // weight gradients in the reference layout (accumulated into)
  float *d_bu_w1, *d_bu_w2, *d_td_w1, *d_td_w2;
  float *d_bu_b1, *d_td_b1;       // first-layer bias gradients (L*4d), ((L-1)*4d): column sums of dpre, reduced by BW_DH
  // BW_BATCH: C[z] (M = n rows, N cols) (+)= A[z] . B[z]^T-like, z = (image, level); operands come from 3-D tensor
  // maps over state-like (R, L*d) tensors (inner offset l*d, batch = image) or attention-like (Z, n, n) ones
  int bN, bK;                // N and K extents
  int a_mn, b_mn;            // 1: operand is MN-major (k runs over rows of the source), 0: K-major
  int a_state, b_state;      // 1: state-like source, 0: attention-like
  int out_kind;              // 0: store (Z, n, n) fp32; 1: accumulate into state-like fp32; 2: store state-like fp32
  float* out;
  // optional second product accumulated into the same tile (K-concatenation): k blocks >= k_split read the second
  // operand pair (maps a1 / b1) with its own layout flags; 0 = single product
  int k_split;
  int a_mn2, b_mn2, a_state2, b_state2;
  // per-image step counts (NULL: none): at reverse step t the rows of images with steps[b] <= t have dY = 0, so BW_PRE /
  // BW_DH / BW_DX skip a CTA's 128-row block and BW_DW a 64-row k-block when all its rows are such rows; BW_BATCH skips
  // the problems of such images
  const int32_t* steps;
  int t;
  // deterministic instantiations (DET): BW_DX stores the top-down groups' dx tiles into dx_td (R, L-1, d) instead of
  // reducing them into ds / d_pos, and BW_DH stores each warp's 32-row column sum of dpre into b1_part
  // [G][nbands = ceil(R / 32)][4d] instead of reducing it into d_*_b1; CUDA-core kernels of bwd_kernels.cu then reduce
  // both in a fixed order
  float* dx_td;
  float* b1_part;
  int nbands;
};

// rows [r0, r0 + nr) below p.rows all belong to images frozen at this step (an empty range counts as frozen).  Every warp
// role evaluates it for the same block, so producer and consumers skip the same tiles / k-blocks.  Warp-collective: the
// lanes test one image each.
__device__ __forceinline__ bool rows_frozen(const BwdParams& p, int r0, int nr, int lane) {
  const int r1 = min(r0 + nr, p.rows);
  bool live = false;
  if (r0 < r1)
    for (int b = r0 / p.n + lane; b <= (r1 - 1) / p.n; b += 32) live |= __ldg(p.steps + b) > p.t;
  return !__any_sync(0xffffffffu, live);
}

// BW_BATCH: problem z = image * L + level belongs to an image frozen at this step.  It depends on z alone, so the two
// CTAs of a pair (which split one problem's rows) and every warp role skip the same tiles.
__device__ __forceinline__ bool problem_frozen(const BwdParams& p, int z) { return __ldg(p.steps + z / p.L) <= p.t; }

struct Tile {
  int g, m_blk, n_blk, num_kb;
  int kind;            // BW_DW only: 0 = dW2_g (M = d rows o, N = 4d), 1 = dW1_g (M = 4d rows j, N = d)
};

template <int MODE>
__device__ __forceinline__ Tile decode(const BwdParams& p, int tile) {
  Tile t{};
  if (MODE == BW_PRE || MODE == BW_DH) {            // output (R, 4d) per group
    const int nn = 4 * p.d / BN, nm = (p.rows + 255) / 256;
    t.n_blk = tile % nn; t.m_blk = (tile / nn) % nm; t.g = tile / (nn * nm); t.num_kb = p.d / BK;
  } else if (MODE == BW_DX) {                        // output (R, d) per group
    const int nn = p.d / BN, nm = (p.rows + 255) / 256;
    t.n_blk = tile % nn; t.m_blk = (tile / nn) % nm; t.g = tile / (nn * nm); t.num_kb = 4 * p.d / BK;
  } else if (MODE == BW_BATCH) {
    const int nm = (p.n + 255) / 256, nn = (p.bN + BN - 1) / BN;
    t.n_blk = tile % nn; t.m_blk = (tile / nn) % nm; t.g = tile / (nn * nm);      // g = problem z
    t.num_kb = p.k_split ? 2 * p.k_split : (p.bK + BK - 1) / BK;
  } else {                                           // weight gradients: 2 * (d/256) * (4d/256) tiles per group
    const int per_kind = (p.d / 256) * (4 * p.d / BN);
    t.g = tile / (2 * per_kind);
    const int r = tile % (2 * per_kind);
    t.kind = r / per_kind;
    const int q = r % per_kind;
    const int nn = t.kind == 0 ? 4 * p.d / BN : p.d / BN;
    t.n_blk = q % nn; t.m_blk = q / nn;
    t.num_kb = (p.rows + BK - 1) / BK;
  }
  return t;
}

// Phi(x) and phi(x) of the standard normal: gelu(x) = x Phi(x), gelu'(x) = Phi(x) + x phi(x)   (exact-erf form, :30)
// Over every float32 x: |gelu error| <= 3.8e-7 and |gelu' error| <= 4.5e-6 (both inside [-6, 6]); past |x| = 6 at most
// 6e-9 and 3.7e-8 (tests/test_backward_oracle.py, test_backward_gelu_fit_within_documented_bound)
__device__ __forceinline__ void normal_cdf_pdf(float x, float& cdf, float& pdf) {
  const float a = fabsf(x), t = fminf(a, 6.0f);
  float q = 3.290448512416333e-05f;
  q = fmaf(q, t, -0.0007621519616805017f);
  q = fmaf(q, t, 0.008038812316954136f);
  q = fmaf(q, t, -0.05331535264849663f);
  q = fmaf(q, t, -0.45887142419815063f);
  q = fmaf(q, t, -1.1511567831039429f);
  q = fmaf(q, t, -0.9999995827674866f);
  // Phi(-|x|); zero past 6, where it is below 1e-9: cdf becomes 0 or 1 and pdf 0, so that gelu' = cdf + x pdf does not
  // grow with |x| as the fit's x * phi(6) would
  const float tail = a > 6.0f ? 0.0f : ex2_approx(q);
  cdf = x >= 0.f ? 1.0f - tail : tail;
  // phi(t) = Phi(-t) * hazard(t): the hazard function is smooth, a degree-6 fit on [0, 6] is good to 2.4e-5 relative,
  // and the epilogue (XU-bound: ex2 + bf16 packing) saves its second ex2 per element
  float hz = 7.497369551856536e-06f;
  hz = fmaf(hz, t, -0.00023059015802573413f);
  hz = fmaf(hz, t, 0.003048981074243784f);
  hz = fmaf(hz, t, -0.023022783920168877f);
  hz = fmaf(hz, t, 0.11135400831699371f);
  hz = fmaf(hz, t, 0.6360868811607361f);
  hz = fmaf(hz, t, 0.7979033589363098f);
  pdf = tail * hz;
}

template <int MODE, bool DET = false>
__global__ void __launch_bounds__(THREADS, 1)
bwd_gemm_kernel(const __grid_constant__ CUtensorMap map_a0,   // PRE: Xb           DH: gsb (R, L*d)   DX: dpre blocks   DW: gsb
                const __grid_constant__ CUtensorMap map_a1,   // PRE: Sb                                              DW: dpre blocks
                const __grid_constant__ CUtensorMap map_a2,   // PRE: Sp                                              DW: h blocks
                const __grid_constant__ CUtensorMap map_b,    // PRE: W1p (G*4d,d)  DH: W2T (G*4d,d)   DX: W1T (G*d,4d)  DW: Xb
                const __grid_constant__ CUtensorMap map_b1,   //                                                      DW: Sb
                const __grid_constant__ CUtensorMap map_b2,   //                                                      DW: Sp
                const BwdParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  float* stg_all = reinterpret_cast<float*>(smem + (size_t)STAGES * STAGE_BYTES);
  uint8_t* patches = reinterpret_cast<uint8_t*>(stg_all) + 4 * STG_BYTES;
  float* bias_s = reinterpret_cast<float*>(patches + (size_t)CONSUMER_WARPS * PATCH_BYTES);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(bias_s + BN);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int W_TMA = CONSUMER_WARPS;
  const int cta_rank = (int)(blockIdx.x & 1);           // the pair's two CTAs own rows [128 r, 128 r + 128) of each tile
  const int cluster_id = blockIdx.x >> 1, num_clusters = gridDim.x >> 1;
  const int kbg_n = 4 * p.d / BK;                     // 64-column blocks per group in the blocked buffers

  if (warp == W_TMA && lane == 0) {
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], CONSUMER_WARPS); }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();

  if (warp == W_TMA) {
    // warp-converged control loop: every lane polls, the elected lane issues (see elect_one in ptx.cuh)
    const uint32_t elected = elect_one();
    {
      int stage = 0; uint32_t phase = 0;
      for (int tile = cluster_id; tile < p.num_tiles; tile += num_clusters) {
        const Tile t = decode<MODE>(p, tile);
        const int l = t.g >> 1;
        if ((MODE == BW_PRE || MODE == BW_DH || MODE == BW_DX) && p.steps &&
            rows_frozen(p, t.m_blk * 256 + cta_rank * BM, BM, lane))
          continue;
        if (MODE == BW_BATCH && p.steps && problem_frozen(p, t.g)) continue;
        if (MODE == BW_DW && p.steps && rows_frozen(p, 0, p.rows, lane)) continue;     // every image frozen: no k-block runs
        for (int kb = 0; kb < t.num_kb; ++kb) {
          if (MODE == BW_DW && p.steps && rows_frozen(p, kb * BK, BK, lane)) continue;
          mbar_wait(&empty_bar[stage], phase ^ 1);
          if (elected) {
          const uint32_t sa = smem_u32(smem + (size_t)stage * STAGE_BYTES);
          const uint32_t sb = sa + A_BYTES;
          uint64_t* bar = &full_bar[stage];
          mbar_arrive_expect_tx(bar, STAGE_BYTES);
          if (MODE == BW_PRE || MODE == BW_DH) {
            const int a_row = t.m_blk * 256 + (int)cta_rank * BM;
            const int b_row = t.g * 4 * p.d + t.n_blk * BN;
            if (MODE == BW_PRE) {
              const CUtensorMap* amap = (t.g == 0) ? &map_a0 : ((t.g & 1) ? &map_a2 : &map_a1);
              const int a_col = (t.g == 0) ? 0 : ((t.g & 1) ? l * p.d : (l - 1) * p.d);
              tma_load_2d(sa, amap, bar, a_col + kb * BK, a_row);
            } else {
              tma_load_2d(sa, &map_a0, bar, l * p.d + kb * BK, a_row);          // dY = gs[:, l, :]
            }
            for (int i = 0; i < 2; ++i) tma_load_2d(sb + i * 16384, &map_b, bar, kb * BK, b_row + i * (BN / 2));
          } else if (MODE == BW_DX) {
            const int m128 = t.m_blk * 2 + (int)cta_rank;
            tma_load_2d(sa, &map_a0, bar, 0, ((t.g * p.m128 + m128) * kbg_n + kb) * BM);    // dpre block (16 KB)
            for (int i = 0; i < 2; ++i) tma_load_2d(sb + i * 16384, &map_b, bar, kb * BK, t.g * p.d + t.n_blk * BN + i * (BN / 2));
          } else if (MODE == BW_BATCH) {
            const int z = t.g, bb = z / p.L, lv = z % p.L;
            const bool seg2 = p.k_split && kb >= p.k_split;          // second product of a K-concatenated pair
            const int kk = seg2 ? kb - p.k_split : kb;
            const CUtensorMap* am = seg2 ? &map_a1 : &map_a0;
            const CUtensorMap* bm = seg2 ? &map_b1 : &map_b;
            const int a_st = seg2 ? p.a_state2 : p.a_state, b_st = seg2 ? p.b_state2 : p.b_state;
            const int a_mn = seg2 ? p.a_mn2 : p.a_mn, b_mn = seg2 ? p.b_mn2 : p.b_mn;
            const int a_off = a_st ? lv * p.d : 0, a_bt = a_st ? bb : z;
            const int b_off = b_st ? lv * p.d : 0, b_bt = b_st ? bb : z;
            const int mrow = t.m_blk * 256 + cta_rank * BM, ncol = t.n_blk * BN;
            if (!a_mn) tma_load_3d(sa, am, bar, a_off + kk * BK, mrow, a_bt);
            else for (int i = 0; i < 2; ++i) tma_load_3d(sa + i * 8192, am, bar, a_off + mrow + i * 64, kk * BK, a_bt);
            if (!b_mn) for (int i = 0; i < 2; ++i) tma_load_3d(sb + i * 16384, bm, bar, b_off + kk * BK, ncol + i * BM, b_bt);
            else for (int i = 0; i < 4; ++i) tma_load_3d(sb + i * 8192, bm, bar, b_off + ncol + i * 64, kk * BK, b_bt);
          } else {
            // TN: k runs over rows.  A tile = 64 k-rows x this CTA's 128 M-columns (two [64 x 64] boxes), B tile = 64 k-rows
            // x 256 N-columns (four boxes); MN-major operands: 128-byte rows of 64 consecutive columns.
            const int r0 = kb * BK;
            const int blk_row = (t.g * p.m128 + (r0 >> 7)) * kbg_n;          // first block of this 128-row band
            const int half = (r0 >> 6) & 1;
            const int mcol = t.m_blk * 256 + cta_rank * BM;                  // first M column of this CTA
            const int ncol = t.n_blk * BN;                                    // first N column of the tile
            for (int i = 0; i < 4; ++i) {
              if (t.kind == 0) {   // dW2_g = dY^T h:  A = gs[:, l, o] (row-major), B = h blocks of group g
                if (i < 2) tma_load_2d(sa + i * 8192, &map_a0, bar, l * p.d + mcol + i * 64, r0);
                tma_load_2d(sb + i * 8192, &map_a2, bar, 0, (blk_row + (ncol >> 6) + i) * BM + half * 64);
              } else {             // dW1_g = dpre^T x:  A = dpre blocks of group g, B = x of group g (row-major)
                if (i < 2) tma_load_2d(sa + i * 8192, &map_a1, bar, 0, (blk_row + (mcol >> 6) + i) * BM + half * 64);
                const CUtensorMap* bmap = (t.g == 0) ? &map_b : ((t.g & 1) ? &map_b2 : &map_b1);
                const int b_col = (t.g == 0) ? 0 : ((t.g & 1) ? l * p.d : (l - 1) * p.d);
                tma_load_2d(sb + i * 8192, bmap, bar, b_col + ncol + i * 64, r0);
              }
            }
          }
          }
          __syncwarp();
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else if (warp < W_TMA) {
    const int wg = warp >> 2, wi = warp & 3;
    const int quad = warp >> 1, x = warp & 1;     // warp pair = 32-row band `quad` of the CTA's 128 rows; x = 32-column half
    float* stg = stg_all + quad * (STG_BYTES / 4);
    uint8_t* patch = patches + (size_t)warp * PATCH_BYTES;
    const int c = lane & 7, rsub = lane >> 3;
    const int a_mn1 = (MODE == BW_DW) ? 1 : (MODE == BW_BATCH ? p.a_mn : 0);
    const int b_mn1 = (MODE == BW_DW) ? 1 : (MODE == BW_BATCH ? p.b_mn : 0);
    int stage = 0; uint32_t phase = 0;
    float frag[BN / 2];
    for (int tile = cluster_id; tile < p.num_tiles; tile += num_clusters) {
      const Tile t = decode<MODE>(p, tile);
      if ((MODE == BW_PRE || MODE == BW_DH || MODE == BW_DX) && p.steps &&
          rows_frozen(p, t.m_blk * 256 + cta_rank * BM, BM, lane))
        continue;
      if (MODE == BW_BATCH && p.steps && problem_frozen(p, t.g)) continue;
      if (MODE == BW_DW && p.steps && rows_frozen(p, 0, p.rows, lane)) continue;
      if (MODE == BW_PRE) {
        named_bar_sync(5, CONSUMER_WARPS * 32);
        for (int i = threadIdx.x; i < BN; i += CONSUMER_WARPS * 32) bias_s[i] = __ldg(p.b1p + (size_t)t.g * 4 * p.d + t.n_blk * BN + i);
        named_bar_sync(5, CONSUMER_WARPS * 32);
      }
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) frag[i] = 0.f;
      int prev = -1;                    // slot of the k-block whose MMAs may still be running
      for (int kb = 0; kb < t.num_kb; ++kb) {
        if (MODE == BW_DW && p.steps && rows_frozen(p, kb * BK, BK, lane)) continue;
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + (size_t)stage * STAGE_BYTES) + (uint32_t)wg * 8192u;   // this warpgroup's 64 rows
        const uint32_t sb = smem_u32(smem + (size_t)stage * STAGE_BYTES) + A_BYTES;
        const bool seg2 = MODE == BW_BATCH && p.k_split && kb >= p.k_split;
        const int sel = seg2 ? 2 * p.a_mn2 + p.b_mn2 : 2 * a_mn1 + b_mn1;
        wgmma_fence_regs(frag);
        wgmma_fence();
        if (sel == 0) kblock<0, 0>(frag, sa, sb);
        else if (sel == 1) kblock<0, 1>(frag, sa, sb);
        else if (sel == 2) kblock<1, 0>(frag, sa, sb);
        else kblock<1, 1>(frag, sa, sb);
        wgmma_commit();
        wgmma_wait<1>();                  // the previous k-block's MMAs are complete: release its slot
        wgmma_fence_regs(frag);
        if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty_bar[prev]); }
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      if (MODE == BW_DW && prev < 0) continue;     // every k-block was skipped: the tile adds nothing
      wgmma_wait<0>();
      wgmma_fence_regs(frag);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[prev]);
      const int row0 = t.m_blk * 256 + cta_rank * BM + quad * 32;      // output row band of this warp pair
#pragma unroll 1
      for (int part = 0; part < BN / 64; ++part) {
        const int c0 = 32 * x;
        // blocked address of this lane's 4 values of row r: block (g, row / 128, col / 64), row % 128, col % 64
        auto blocked_off = [&](int r) -> size_t {
          const int row = row0 + r, col = t.n_blk * BN + part * 64 + c0 + c * 4;
          return ((size_t)((t.g * p.m128 + (row >> 7)) * kbg_n + (col >> 6)) * BM + (row & 127)) * BK + (col & 63);
        };
        // BW_DH: gelu'(pre) of this chunk, in flight while the accumulator is staged
        uint2 gp_cur[8];
        if (MODE == BW_DH) {
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int r = i * 4 + rsub;
            gp_cur[i] = row0 + r < p.rows ? __ldg(reinterpret_cast<const uint2*>(p.pre + blocked_off(r))) : make_uint2(0u, 0u);
          }
        }
        stage_write(frag, stg, part, wi, lane);
        named_bar_sync(1 + quad, 64);
        uint32_t v[32];
        stage_read(stg, x, lane, v);
        // accumulator chunk -> patch (f32 rows of 128 B, chunk j of row r at j ^ (r & 7)) -> 4 columns x 8 rows per lane
#pragma unroll
        for (int j = 0; j < 8; ++j)
          *reinterpret_cast<uint4*>(patch + lane * 128 + ((j ^ (lane & 7)) << 4)) =
              make_uint4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
        __syncwarp();
        const int col = t.n_blk * BN + part * 64 + c0 + c * 4;     // output column of this lane's 4 values
        float colsum[4] = {0.f, 0.f, 0.f, 0.f};                           // BW_DH: first-layer bias gradient partials
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int r = i * 4 + rsub;
          const float4 acc = *reinterpret_cast<const float4*>(patch + r * 128 + ((c ^ (r & 7)) << 4));
          const int row = row0 + r;
          if (MODE == BW_PRE || MODE == BW_DH) {
            if (row < p.rows) {
              const size_t off = blocked_off(r);
              if (MODE == BW_PRE) {
                // pre-activation -> h = gelu(pre) and gp = gelu'(pre), both bf16 (the `pre` buffer holds gp)
                const float4 b4 = *reinterpret_cast<const float4*>(bias_s + part * 64 + c0 + c * 4);
                const float xv[4] = {acc.x + b4.x, acc.y + b4.y, acc.z + b4.z, acc.w + b4.w};
                float hv[4], gp[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                  float cdf, pdf;
                  normal_cdf_pdf(xv[e], cdf, pdf);
                  hv[e] = xv[e] * cdf;
                  gp[e] = fmaf(xv[e], pdf, cdf);
                }
                *reinterpret_cast<uint2*>(p.h + off) = make_uint2(pack_bf16x2(hv[0], hv[1]), pack_bf16x2(hv[2], hv[3]));
                *reinterpret_cast<uint2*>(p.pre + off) = make_uint2(pack_bf16x2(gp[0], gp[1]), pack_bf16x2(gp[2], gp[3]));
              } else {
                const uint2 pw = gp_cur[i];                                           // gelu'(pre)
                const float q0 = acc.x * __uint_as_float(pw.x << 16), q1 = acc.y * __uint_as_float(pw.x & 0xFFFF0000u);
                const float q2 = acc.z * __uint_as_float(pw.y << 16), q3 = acc.w * __uint_as_float(pw.y & 0xFFFF0000u);
                colsum[0] += q0; colsum[1] += q1; colsum[2] += q2; colsum[3] += q3;
                *reinterpret_cast<uint2*>(p.dpre + off) = make_uint2(pack_bf16x2(q0, q1), pack_bf16x2(q2, q3));
              }
            }
          } else if (MODE == BW_DX) {
            if constexpr (DET) {
              // every element below has one writer in this launch: group 0 owns d_tokens, bottom-up group 2l owns level
              // l-1 of ds (top-down groups no longer add there), top-down group 2l+1 owns slice l of dx_td
              const int lg = t.g >> 1;
              if (row < p.rows && (t.g & 1)) {
                *reinterpret_cast<float4*>(p.dx_td + ((size_t)row * (p.L - 1) + lg) * p.d + col) = acc;
              } else if (row < p.rows) {
                float* dst = t.g == 0 ? p.d_tokens + (size_t)row * p.d + col : p.ds + ((size_t)row * p.L + lg - 1) * p.d + col;
                float4 o = *reinterpret_cast<const float4*>(dst);
                o.x += acc.x; o.y += acc.y; o.z += acc.z; o.w += acc.w;
                *reinterpret_cast<float4*>(dst) = o;
              }
            } else if (row < p.rows) {
              // several groups (and, for pos, all images) add into the same element: reduce in L2, no dx round trip
              const int lg = t.g >> 1;
              if (t.g == 0) {
                red_add_f32x4(p.d_tokens + (size_t)row * p.d + col, acc);
              } else if (t.g & 1) {
                red_add_f32x4(p.ds + ((size_t)row * p.L + lg + 1) * p.d + col, acc);
                red_add_f32x4(p.d_pos + (size_t)(row % p.n) * p.d + col, acc);
              } else {
                red_add_f32x4(p.ds + ((size_t)row * p.L + lg - 1) * p.d + col, acc);
              }
            }
          } else if (MODE == BW_BATCH) {
            const int z = t.g;
            if (row < p.n && col < p.bN) {
              if (p.out_kind == 0) {
                float* dst = p.out + ((size_t)z * p.n + row) * p.bN + col;
                if ((p.bN & 3) == 0) *reinterpret_cast<float4*>(dst) = acc;
                else {
                  const float a4[4] = {acc.x, acc.y, acc.z, acc.w};
                  for (int e = 0; e < 4 && col + e < p.bN; ++e) dst[e] = a4[e];
                }
              } else {
                float* dst = p.out + (((size_t)(z / p.L) * p.n + row) * p.L + (z % p.L)) * p.d + col;
                float4 o = acc;
                if (p.out_kind == 1) { const float4 old = *reinterpret_cast<const float4*>(dst); o.x += old.x; o.y += old.y; o.z += old.z; o.w += old.w; }
                *reinterpret_cast<float4*>(dst) = o;
              }
            }
          } else {
            // weight gradient tile: output row = M index (o or j), accumulate into the reference-layout tensor
            const int lw = t.g >> 1;
            float* dst;
            if (t.kind == 0) dst = ((t.g & 1) ? p.d_td_w2 : p.d_bu_w2) + ((size_t)lw * p.d + row) * 4 * p.d + col;   // (L*d, 4d)
            else dst = ((t.g & 1) ? p.d_td_w1 : p.d_bu_w1) + ((size_t)lw * 4 * p.d + row) * p.d + col;              // (L*4d, d)
            float4 old = *reinterpret_cast<const float4*>(dst);
            old.x += acc.x; old.y += acc.y; old.z += acc.z; old.w += acc.w;
            *reinterpret_cast<float4*>(dst) = old;
          }
        }
        if (MODE == BW_DH) {
          // db1[g, col] += sum over this warp's 32 rows of dpre: the four row sub-lanes of a column group, then L2
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            colsum[e] += __shfl_xor_sync(0xffffffffu, colsum[e], 8);
            colsum[e] += __shfl_xor_sync(0xffffffffu, colsum[e], 16);
          }
          if constexpr (DET) {
            // deterministic: the band's partial goes to its own slot, reduced over bands in order by bias_partials_kernel
            if (rsub == 0 && row0 < p.rows)
              *reinterpret_cast<float4*>(p.b1_part + ((size_t)t.g * p.nbands + row0 / 32) * 4 * p.d + col) =
                  make_float4(colsum[0], colsum[1], colsum[2], colsum[3]);
          } else if (rsub == 0) {
            red_add_f32x4(((t.g & 1) ? p.d_td_b1 : p.d_bu_b1) + (size_t)(t.g >> 1) * 4 * p.d + col,
                          make_float4(colsum[0], colsum[1], colsum[2], colsum[3]));
          }
        }
        __syncwarp();
        named_bar_sync(1 + quad, 64);                                   // staging tile free for the next step
      }
    }
  }

  __syncthreads();
}

// -> 0 or GLOM_B200_ERR_CUDA
int map2d_box(Launch& ln, CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows, const char* what) {
  cuuint64_t gd[2] = {cols, rows};
  cuuint64_t gs[1] = {cols * 2};
  cuuint32_t bx[2] = {(cuuint32_t)BK, box_rows};
  cuuint32_t es[2] = {1, 1};
  const CUresult r = ln.enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gd, gs, bx, es,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return ln.fail(GLOM_B200_ERR_CUDA, "cuTensorMapEncodeTiled(%s) failed with CUresult %d", what, (int)r);
  return 0;
}

template <int MODE, bool DET = false>
cudaError_t launch(const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& a2, const CUtensorMap& b0,
                   const CUtensorMap& b1, const CUtensorMap& b2, const BwdParams& p, int num_sms, cudaStream_t st) {
  static SmemOptIn optin;
  if (cudaError_t e = optin.ensure(bwd_gemm_kernel<MODE, DET>, SMEM_BYTES)) return e;
  const int max_pairs = num_sms / 2;
  const int pairs = p.num_tiles < max_pairs ? p.num_tiles : max_pairs;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(2 * pairs);
  cfg.blockDim = dim3(THREADS);
  cfg.dynamicSmemBytes = SMEM_BYTES;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, bwd_gemm_kernel<MODE, DET>, a0, a1, a2, b0, b1, b2, p);
}

int map3d_box(Launch& ln, CUtensorMap* m, const void* base, uint64_t inner, uint64_t rows, uint64_t batches,
              uint64_t row_stride_elems, uint64_t batch_stride_elems, uint32_t box_rows, const char* what) {
  cuuint64_t gd[3] = {inner, rows, batches};
  cuuint64_t gs[2] = {row_stride_elems * 2, batch_stride_elems * 2};
  cuuint32_t bx[3] = {(cuuint32_t)BK, box_rows, 1};
  cuuint32_t es[3] = {1, 1, 1};
  const CUresult r = ln.enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), gd, gs, bx, es,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return ln.fail(GLOM_B200_ERR_CUDA, "cuTensorMapEncodeTiled(%s) failed with CUresult %d", what, (int)r);
  return 0;
}

}  // namespace

// Batched C[z] (n x N) (+)= A[z] B[z] on tensor cores for the attention backward (z = image * L + level).
//   state-like operands: bf16 (B*n, L*d) tensors; attention-like: bf16 (Z, n, n).  a.mn / b.mn: see BwdParams.
//   a2.src != nullptr: a second product A2[z] B2[z] of the same shape is accumulated into the same tile (its k blocks
//   follow the first product's), so both land in `out` with one read-modify-write.
int attn_bwd_gemm_tc(const Geometry& g, AttnBwdOperand a, AttnBwdOperand b, int N, int K, int out_kind, float* out,
                     const int32_t* steps, int t, Launch& ln, AttnBwdOperand a2, AttnBwdOperand b2) {
  const int n = g.n, L = g.L, d = g.d, Z = g.B * L;
  CUtensorMap ma, mb, ma2, mb2;
  auto mk = [&](CUtensorMap* m, const AttnBwdOperand& o, const char* what) {
    const uint32_t box_rows = o.mn ? 64u : (uint32_t)BM;
    if (o.state) return map3d_box(ln, m, o.src, (uint64_t)L * d, n, g.B, (uint64_t)L * d, (uint64_t)n * L * d, box_rows, what);
    return map3d_box(ln, m, o.src, n, n, Z, n, (uint64_t)n * n, box_rows, what);
  };
  GLOM_TRY(mk(&ma, a, "attn-bwd A"));
  GLOM_TRY(mk(&mb, b, "attn-bwd B"));
  ma2 = ma; mb2 = mb;
  if (a2.src) {
    GLOM_TRY(mk(&ma2, a2, "attn-bwd A2"));
    GLOM_TRY(mk(&mb2, b2, "attn-bwd B2"));
  }
  BwdParams p{};
  p.rows = g.rows; p.d = d; p.L = L; p.n = n; p.G = g.G;
  p.bN = N; p.bK = K; p.a_mn = a.mn; p.b_mn = b.mn; p.a_state = a.state; p.b_state = b.state; p.out_kind = out_kind; p.out = out;
  p.steps = steps; p.t = t;
  if (a2.src) { p.k_split = (K + BK - 1) / BK; p.a_mn2 = a2.mn; p.b_mn2 = b2.mn; p.a_state2 = a2.state; p.b_state2 = b2.state; }
  p.num_tiles = Z * ((n + 255) / 256) * ((N + BN - 1) / BN);
  return ln.launched(launch<BW_BATCH>(ma, ma2, ma, mb, mb2, mb, p, ln.num_sms, ln.st), "attention-backward gemm launch");
}

// One reverse step of the MLPs on tensor cores.  Inputs are bf16 shadows prepared by the caller:
//   xb (R, d), sb (R, L*d), sp (R, (L-1)*d) of S_t ; gsb (R, L*d) = bf16(dL/dS_{t+1} / c)
//   w1p (G*4d, d), w2t (G*4d, d), w1t (G*d, 4d) bf16 packs of the current weights.
int mlp_backward_tc(const Geometry& g, const MlpBwdTc& a, Launch& ln) {
  const int d = g.d, L = g.L, rows = g.rows, G = g.G, num_sms = ln.num_sms;
  cudaStream_t st = ln.st;
  if (d % 256) return ln.fail(GLOM_B200_ERR_INVALID, "tensor-core backward needs dim %% 256 == 0 (got %d)", d);
  const int m128 = (rows + 127) / 128;
  const uint64_t blocked_rows = (uint64_t)G * m128 * (4 * d / BK) * BM;
  CUtensorMap mxb, msb, msp, mgs, mw1p, mw2t, mw1t, mdpre128, mdpre64, mh64, mxb64, msb64, msp64, mgs64;
  int bad = 0;                  // every map is attempted; the message is the last failure's
  bad |= map2d_box(ln, &mxb, a.xb, rows, d, BM, "Xb");
  bad |= map2d_box(ln, &msb, a.sb, rows, (uint64_t)L * d, BM, "Sb");
  bad |= map2d_box(ln, &msp, a.sp, rows, (uint64_t)(L - 1) * d, BM, "Sp");
  bad |= map2d_box(ln, &mgs, a.gsb, rows, (uint64_t)L * d, BM, "gsb");
  bad |= map2d_box(ln, &mw1p, a.w1p, (uint64_t)G * 4 * d, d, BN / 2, "W1p");
  bad |= map2d_box(ln, &mw2t, a.w2t, (uint64_t)G * 4 * d, d, BN / 2, "W2T");
  bad |= map2d_box(ln, &mw1t, a.w1t, (uint64_t)G * d, (uint64_t)4 * d, BN / 2, "W1T");
  bad |= map2d_box(ln, &mdpre128, a.dpre, blocked_rows, BK, BM, "dpre");
  bad |= map2d_box(ln, &mdpre64, a.dpre, blocked_rows, BK, 64, "dpre64");
  bad |= map2d_box(ln, &mh64, a.h, blocked_rows, BK, 64, "h64");
  bad |= map2d_box(ln, &mxb64, a.xb, rows, d, 64, "Xb64");
  bad |= map2d_box(ln, &msb64, a.sb, rows, (uint64_t)L * d, 64, "Sb64");
  bad |= map2d_box(ln, &msp64, a.sp, rows, (uint64_t)(L - 1) * d, 64, "Sp64");
  bad |= map2d_box(ln, &mgs64, a.gsb, rows, (uint64_t)L * d, 64, "gsb64");
  if (bad) return bad;
  BwdParams p{};
  p.rows = rows; p.d = d; p.L = L; p.n = g.n; p.G = G; p.m128 = m128;
  p.b1p = a.b1p; p.pre = a.pre; p.h = a.h; p.dpre = a.dpre; p.ds = a.ds; p.d_tokens = a.d_tokens; p.d_pos = a.d_pos;
  p.d_bu_w1 = a.d_bu_w1; p.d_bu_w2 = a.d_bu_w2; p.d_td_w1 = a.d_td_w1; p.d_td_w2 = a.d_td_w2;
  p.d_bu_b1 = a.d_bu_b1; p.d_td_b1 = a.d_td_b1;
  p.steps = a.steps; p.t = a.t;
  p.dx_td = a.dx_td; p.b1_part = a.b1_part; p.nbands = (rows + 31) / 32;
  const int nm = (rows + 255) / 256;
  cudaError_t e;
  p.num_tiles = G * nm * (4 * d / BN);
  if (!a.skip_pre) {
    GLOM_TRY(ln.launched(launch<BW_PRE>(mxb, msb, msp, mw1p, mw1p, mw1p, p, num_sms, st), "bwd pre launch"));
  }
  e = a.deterministic ? launch<BW_DH, true>(mgs, mgs, mgs, mw2t, mw2t, mw2t, p, num_sms, st)
                      : launch<BW_DH>(mgs, mgs, mgs, mw2t, mw2t, mw2t, p, num_sms, st);
  GLOM_TRY(ln.launched(e, "bwd dh launch"));
  p.num_tiles = G * nm * (d / BN);
  e = a.deterministic ? launch<BW_DX, true>(mdpre128, mdpre128, mdpre128, mw1t, mw1t, mw1t, p, num_sms, st)
                      : launch<BW_DX>(mdpre128, mdpre128, mdpre128, mw1t, mw1t, mw1t, p, num_sms, st);
  GLOM_TRY(ln.launched(e, "bwd dx launch"));
  if (a.skip_dw) return 0;
  p.num_tiles = G * 2 * (d / 256) * (4 * d / BN);
  return ln.launched(launch<BW_DW>(mgs64, mdpre64, mh64, mxb64, msb64, msp64, p, num_sms, st), "bwd dw launch");
}

}  // namespace glom
