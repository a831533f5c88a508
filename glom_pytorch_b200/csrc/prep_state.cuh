// The bf16 engine's state prologue for one (row, level), and the token cast, as device functions: prep_state_kernel
// (simt_kernels.cu) runs them over a whole batch, and the settle queue's slot fill (settle_kernels.cu) over the rows of
// the images it admits.  Both must produce the same bits, so both call these.
#pragma once
#include "ptx.cuh"

namespace glom {

// bf16 words of four fp32 values (the tokens' cast, cast_bf16_kernel)
__device__ __forceinline__ uint2 cast4_bf16(const float4 v) {
  uint2 pk;
  pk.x = pack_bf16x2(v.x, v.y);
  pk.y = pack_bf16x2(v.z, v.w);
  return pk;
}

// One warp, level l of one row: src (d) fp32 is the row's S_0 at level l, p (d) the row's position embedding.
// Writes the fp32 master copy (s32, nullable), the bf16 shadow sb (d), for l >= 1 the shadow of S + pos sp (d), and the
// nparts squared-norm partials nsq (nparts).
__device__ __forceinline__ void prep_state_row(int lane, int l, int d, int nparts, int part_w, const float* __restrict__ src,
                                               const float* __restrict__ p, float* __restrict__ s32,
                                               __nv_bfloat16* __restrict__ sb, __nv_bfloat16* __restrict__ sp,
                                               float* __restrict__ nsq) {
  for (int c = lane * 4; c < d; c += 128) {
    const float4 v = *reinterpret_cast<const float4*>(src + c);
    if (s32) *reinterpret_cast<float4*>(s32 + c) = v;
    *reinterpret_cast<uint2*>(sb + c) = cast4_bf16(v);
    if (l >= 1) {
      const float4 q = *reinterpret_cast<const float4*>(p + c);
      uint2 pq;
      pq.x = pack_bf16x2(v.x + q.x, v.y + q.y);
      pq.y = pack_bf16x2(v.z + q.z, v.w + q.w);
      *reinterpret_cast<uint2*>(sp + c) = pq;
    }
  }
  // squared-norm partials in exactly the order the GEMM2 epilogue accumulates them (row_chunk_sumsq in
  // tc_kernels.cu), so a carried-in state continues bit-identically (:123).
  // (per 32-column chunk: 8 four-column fmaf chains, pairwise tree; chunks added in order)
  for (int part = 0; part < nparts; ++part) {
    float ss = 0.f;
    for (int c0 = 0; c0 < part_w; c0 += 32) {
      const float4 v = *reinterpret_cast<const float4*>(src + part * part_w + c0 + (lane & 7) * 4);
      float q = v.x * v.x;
      q = fmaf(v.y, v.y, q);
      q = fmaf(v.z, v.z, q);
      q = fmaf(v.w, v.w, q);
      q += __shfl_xor_sync(0xffffffffu, q, 1);
      q += __shfl_xor_sync(0xffffffffu, q, 2);
      q += __shfl_xor_sync(0xffffffffu, q, 4);
      ss += q;
    }
    if (lane == 0) nsq[part] = ss;
  }
}

}  // namespace glom
