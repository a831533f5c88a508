// Pieces shared by the tensor-core kernels: tile constants, the accumulator hand-off, the K2 epilogue chunk body and the
// tensor-map helpers.
#pragma once
#include "engine.h"
#include "ptx.cuh"

#include <stdio.h>

namespace glom {

constexpr int BM = 128;            // rows of the state per CTA tile (two warpgroups of wgmma M = 64)
constexpr int BK = 64;             // bf16 elements per 128-byte swizzle row
constexpr uint32_t A_STAGE_BYTES = BM * BK * 2;   // 16 KB

// ---- hand-off of a warpgroup's wgmma accumulator to the row-per-thread epilogue chunks
// Warps 2h and 2h + 1 of a warpgroup hold rows [32 h, 32 h + 32) of its 64 accumulator rows, 16 each.  For the 64-column
// step s of the tile they write those 32 rows x 64 columns into the pair's staging tile (fp32, row pitch STG_PITCH
// floats: 16-byte row reads of 8 consecutive rows hit distinct banks); after a pair barrier warp 2h + x reads row `lane`,
// columns [32 x, 32 x + 32): the 32 x 32 chunk the epilogue functions below take, one row per thread.
constexpr int STG_PITCH = 68;
constexpr uint32_t STG_BYTES = 32 * STG_PITCH * 4;    // per warp pair
template <int S, int R>
__device__ __forceinline__ void stage_write_step(const float (&acc)[R], float* stg, int warp_in_wg, int lane) {
  const int r = 16 * (warp_in_wg & 1) + (lane >> 2), c = 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
#pragma unroll
    for (int h = 0; h < 2; ++h)
      *reinterpret_cast<float2*>(stg + (r + 8 * h) * STG_PITCH + 8 * j + c) =
          make_float2(acc[4 * (8 * S + j) + 2 * h], acc[4 * (8 * S + j) + 2 * h + 1]);
  }
}
// runtime step index, accumulator indices stay compile-time (registers, no local-memory copy)
template <int R>
__device__ __forceinline__ void stage_write(const float (&acc)[R], float* stg, int s, int warp_in_wg, int lane) {
  static_assert(R % 32 == 0 && R <= 128, "m64 x N fragment, N in {64, 128, 256}");
  if (s == 0) stage_write_step<0>(acc, stg, warp_in_wg, lane);
  if constexpr (R >= 64) { if (s == 1) stage_write_step<1>(acc, stg, warp_in_wg, lane); }
  if constexpr (R >= 128) {
    if (s == 2) stage_write_step<2>(acc, stg, warp_in_wg, lane);
    if (s == 3) stage_write_step<3>(acc, stg, warp_in_wg, lane);
  }
}
__device__ __forceinline__ void stage_read(const float* stg, int x, int lane, uint32_t (&v)[32]) {
  const float4* src = reinterpret_cast<const float4*>(stg + lane * STG_PITCH + 32 * x);
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const float4 f = src[q];
    v[4 * q] = __float_as_uint(f.x); v[4 * q + 1] = __float_as_uint(f.y);
    v[4 * q + 2] = __float_as_uint(f.z); v[4 * q + 3] = __float_as_uint(f.w);
  }
}

// One k-block (64 of K) of a 128-row tile for warpgroup `wg`: A rows [64 wg, 64 wg + 64) of the stage's K-major A tile,
// B = N rows (K-major, TB = 0) or 64 k-rows x N columns in 64-wide boxes 8 KB apart (MN-major, TB = 1).
template <int N, int TB>
__device__ __forceinline__ void wgmma_kblock(float (&acc)[N / 2], uint32_t a_smem, uint32_t b_smem) {
  const uint64_t ad = wgmma_desc_sw128(a_smem, 16, 1024);
  const uint64_t bd = TB ? wgmma_desc_sw128(b_smem, 8192, 1024) : wgmma_desc_sw128(b_smem, 16, 1024);
#pragma unroll
  for (int k = 0; k < BK / 16; ++k) wgmma_bf16<N, 0, TB>(acc, ad + 2 * k, bd + (TB ? (2048 >> 4) : 2) * k);
}

// Sum of squares of a 32-column chunk row, in the canonical order shared with prep_state_kernel:
// 8 lanes hold 4 consecutive columns each (sequential fmaf), then an xor tree over the 8 lanes.
__device__ __forceinline__ float row_chunk_sumsq(float a, float b, float c, float d) {
  float q = a * a;
  q = fmaf(b, b, q);
  q = fmaf(c, c, q);
  q = fmaf(d, d, q);
  q += __shfl_xor_sync(0xffffffffu, q, 1);
  q += __shfl_xor_sync(0xffffffffu, q, 2);
  q += __shfl_xor_sync(0xffffffffu, q, 4);
  return q;
}

// ---- K2 epilogue chunk: the 4-way combine (glom_pytorch.py:141-142) on a 32 x 32 accumulator chunk.
// The accumulators go through the warp's 4 KB patch (f32, 128-byte rows, chunk c of row r at c ^ (r & 7)) so
// that each lane then owns 4 consecutive columns of 8 rows and every global access covers whole 128-byte lines.
struct K2Chunk {
  int l, L, d, n, row0;
  int prow0;            // row0 % n: patch index of the band's first row (position table row), computed once per tile
  int s_bcast;          // 1: s32_in is init_levels (L, d), the same for every row (first step of a call without carried state)
  bool remap;           // 1: row r of s32_in and c_in is read from row r mod n (only the representative rows hold them)
  const float* s32_in; const __nv_bfloat16* c_in; const float* pos;
  float* s32_out; __nv_bfloat16* sb_out; __nv_bfloat16* sp_out;
};
// SETTLE (Glom.settle): row r of the band loads and stores nothing unless bit r of `live` is set (rows of images that
// have stopped keep their state), and rowdsq[i] accumulates the squared change |S_{t+1} - S_t|^2 of row i * 4 + rsub
// in the same order as rowsq (only when want_dsq: the per-image step counts of forward_steps need no change partials).
template <bool FULL, bool SETTLE = false>
__device__ __forceinline__ void k2_chunk(const uint32_t (&v)[32], const float4 b4, uint8_t* patch, const K2Chunk& k,
                                         int col, int lane, int rows_left, float (&rowsq)[8], uint32_t live = ~0u,
                                         float* rowdsq = nullptr, bool want_dsq = false) {
#pragma unroll
  for (int c = 0; c < 8; ++c)
    *reinterpret_cast<uint4*>(patch + lane * 128 + ((c ^ (lane & 7)) << 4)) =
        make_uint4(v[4 * c], v[4 * c + 1], v[4 * c + 2], v[4 * c + 3]);
  __syncwarp();
  const int c = lane & 7, rsub = lane >> 3;
  const bool top = (k.l == k.L - 1);                  // 3 contributions on the top level, 4 elsewhere (:128-129)
  const bool has_td = (k.l >= 1);
  // row offsets r * ld and r * ldp (r < 32) in 32 bits: the compiler hoists them out of the caller's column loop, and
  // as 64-bit values they would cost twice the registers
  const int ld = k.L * k.d, ldp = (k.L - 1) * k.d;
  const size_t base = ((size_t)k.row0 * k.L + k.l) * k.d + col + c * 4;
  const size_t pbase = ((size_t)k.row0 * (k.L - 1) + (k.l - 1)) * k.d + col + c * 4;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    // global loads of four rows first (independent, all in flight), then combine + store
    float4 sv[4], pp[4];
    uint2 cw[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int r = (h * 4 + j) * 4 + rsub;
      sv[j] = make_float4(0.f, 0.f, 0.f, 0.f); pp[j] = sv[j]; cw[j] = make_uint2(0u, 0u);
      if ((FULL || r < rows_left) && (!SETTLE || ((live >> r) & 1u))) {
        size_t so = base + (unsigned)(r * ld);
        if (!SETTLE && k.remap) {
          int sr = k.prow0 + r;                       // (row0 + r) % n
          if (k.n >= 32) { if (sr >= k.n) sr -= k.n; } else sr %= k.n;
          so = (size_t)k.l * k.d + col + c * 4 + (unsigned)(sr * ld);
        }
        sv[j] = k.s_bcast ? __ldg(reinterpret_cast<const float4*>(k.s32_in + (size_t)k.l * k.d + col + c * 4))
                          : __ldcs(reinterpret_cast<const float4*>(k.s32_in + so));
        cw[j] = __ldcs(reinterpret_cast<const uint2*>(k.c_in + so));
        if (has_td) {
          int pr = k.prow0 + r;                       // (row0 + r) % n without a division per row (r < 32)
          if (k.n >= 32) { if (pr >= k.n) pr -= k.n; } else pr %= k.n;
          pp[j] = __ldg(reinterpret_cast<const float4*>(k.pos + (size_t)pr * k.d + col + c * 4));
        }
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int i = h * 4 + j;
      const int r = i * 4 + rsub;
      const float4 acc = *reinterpret_cast<const float4*>(patch + r * 128 + ((c ^ (r & 7)) << 4));
      float o0 = (sv[j].x + (acc.x + b4.x)) + __uint_as_float(cw[j].x << 16);               // (:141)
      float o1 = (sv[j].y + (acc.y + b4.y)) + __uint_as_float(cw[j].x & 0xFFFF0000u);
      float o2 = (sv[j].z + (acc.z + b4.z)) + __uint_as_float(cw[j].y << 16);
      float o3 = (sv[j].w + (acc.w + b4.w)) + __uint_as_float(cw[j].y & 0xFFFF0000u);
      if (top) { o0 = o0 / 3.0f; o1 = o1 / 3.0f; o2 = o2 / 3.0f; o3 = o3 / 3.0f; }          // (:142) IEEE division
      else { o0 *= 0.25f; o1 *= 0.25f; o2 *= 0.25f; o3 *= 0.25f; }                          // x/4 == x*0.25 exactly
      const bool store = (FULL || r < rows_left) && (!SETTLE || ((live >> r) & 1u));
      if constexpr (SETTLE) if (want_dsq) {
        // rows that store nothing contribute no change (and, below, no norm)
        const float e0 = store ? o0 - sv[j].x : 0.f, e1 = store ? o1 - sv[j].y : 0.f;
        const float e2 = store ? o2 - sv[j].z : 0.f, e3 = store ? o3 - sv[j].w : 0.f;
        rowdsq[i] += row_chunk_sumsq(e0, e1, e2, e3);
      }
      if (store) {
        const size_t o = base + (unsigned)(r * ld);
        __stcs(reinterpret_cast<float4*>(k.s32_out + o), make_float4(o0, o1, o2, o3));
        *reinterpret_cast<uint2*>(k.sb_out + o) = make_uint2(pack_bf16x2(o0, o1), pack_bf16x2(o2, o3));
        if (has_td)
          *reinterpret_cast<uint2*>(k.sp_out + pbase + (unsigned)(r * ldp)) =
              make_uint2(pack_bf16x2(o0 + pp[j].x, o1 + pp[j].y), pack_bf16x2(o2 + pp[j].z, o3 + pp[j].w));
      } else {
        o0 = o1 = o2 = o3 = 0.f;
      }
      rowsq[i] += row_chunk_sumsq(o0, o1, o2, o3);
    }
  }
  __syncwarp();
}

// -> 0 or GLOM_B200_ERR_CUDA
static inline int encode_map(Launch& ln, CUtensorMap* m, const void* base, int rank, const uint64_t* dims,
                             const uint64_t* strides_bytes /* rank-1 */, const uint32_t* box, const char* what) {
  cuuint64_t gd[3]; cuuint64_t gs[2]; cuuint32_t bx[3]; cuuint32_t es[3] = {1, 1, 1};
  for (int i = 0; i < rank; ++i) { gd[i] = dims[i]; bx[i] = box[i]; }
  for (int i = 0; i < rank - 1; ++i) gs[i] = strides_bytes[i];
  const CUresult r = ln.enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), gd, gs, bx, es,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return ln.fail(GLOM_B200_ERR_CUDA, "cuTensorMapEncodeTiled(%s) failed with CUresult %d", what, (int)r);
  return 0;
}

static inline int map2d(Launch& ln, CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows,
                        const char* what) {
  const uint64_t dims[2] = {cols, rows};
  const uint64_t strides[1] = {cols * 2};
  const uint32_t box[2] = {(uint32_t)BK, box_rows};
  return encode_map(ln, m, base, 2, dims, strides, box, what);
}

}  // namespace glom
