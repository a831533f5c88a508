// Island analytics on the column states.
//
// Input: `slabs` states of shape (n = side_h * side_w patches, L levels, d) fp32 -- e.g. the (T+1) * B slabs of
// Glom.forward(..., return_all=True).  Per slab and level, on the patch grid (patch i = h * side_w + w):
//   cos_right[h, w] = cosine similarity of the level vectors of patches (h, w) and (h, w + 1)   (0 in the last column)
//   cos_down [h, w] = ... of (h, w) and (h + 1, w)                                               (0 in the last row)
//   agreement[i]    = mean cosine similarity of patch i with its existing 4-neighbours
//   labels[i]       = island id: the smallest patch index of the 4-connected component of i in the graph whose edges
//                     are the neighbour pairs with cosine similarity >= threshold
//   num_islands     = number of components
// Bound: HBM (each state vector is read once from DRAM; its use as "right" / "down" neighbour hits L1 / L2);
// algorithmic bytes = slabs * n * L * d * 4 read + slabs * L * n * 16 written.  No tensor-core work: per pair only
// 3 dot products of length d are needed, never the n x n Gram matrix.
#include "engine.h"

namespace glom {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// grid (side_h, L, slabs), 256 threads: warp k of the block handles patches (h, k), (h, k + 8), ...
__global__ void __launch_bounds__(256)
island_edges_kernel(const float* __restrict__ states, int side_h, int side_w, int L, int d,
                    float* __restrict__ cos_right, float* __restrict__ cos_down) {
  const int h = blockIdx.x, l = blockIdx.y, slab = blockIdx.z;
  const int n = side_h * side_w;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t pitch = (size_t)L * d;                                  // floats between consecutive patches
  const float* base = states + ((size_t)slab * n * L + l) * d;
  const int d4 = d >> 2;
  for (int w = warp; w < side_w; w += 8) {
    const int i = h * side_w + w;
    const float4* a = reinterpret_cast<const float4*>(base + (size_t)i * pitch);
    const bool has_r = w + 1 < side_w, has_d = h + 1 < side_h;
    const float4* r = reinterpret_cast<const float4*>(base + (size_t)(i + 1) * pitch);
    const float4* dn = reinterpret_cast<const float4*>(base + (size_t)(i + side_w) * pitch);
    float aa = 0.f, ar = 0.f, rr = 0.f, ad = 0.f, dd = 0.f;
    for (int k = lane; k < d4; k += 32) {
      const float4 va = __ldg(a + k);
      aa += va.x * va.x + va.y * va.y + va.z * va.z + va.w * va.w;
      if (has_r) {
        const float4 vr = __ldg(r + k);
        ar += va.x * vr.x + va.y * vr.y + va.z * vr.z + va.w * vr.w;
        rr += vr.x * vr.x + vr.y * vr.y + vr.z * vr.z + vr.w * vr.w;
      }
      if (has_d) {
        const float4 vd = __ldg(dn + k);
        ad += va.x * vd.x + va.y * vd.y + va.z * vd.z + va.w * vd.w;
        dd += vd.x * vd.x + vd.y * vd.y + vd.z * vd.z + vd.w * vd.w;
      }
    }
    aa = warp_sum(aa); ar = warp_sum(ar); rr = warp_sum(rr); ad = warp_sum(ad); dd = warp_sum(dd);
    if (lane == 0) {
      const size_t o = ((size_t)slab * L + l) * n + i;
      cos_right[o] = has_r ? ar / fmaxf(sqrtf(aa) * sqrtf(rr), 1e-12f) : 0.f;
      cos_down[o] = has_d ? ad / fmaxf(sqrtf(aa) * sqrtf(dd), 1e-12f) : 0.f;
    }
  }
}

// one block per (level, slab): agreement from the edge maps, then min-label propagation over the thresholded edges
__global__ void __launch_bounds__(256)
island_label_kernel(const float* __restrict__ cos_right, const float* __restrict__ cos_down, int side_h, int side_w,
                    float threshold, float* __restrict__ agreement, int* __restrict__ labels,
                    int* __restrict__ num_islands) {
  extern __shared__ int sm[];
  const int n = side_h * side_w;
  int* lab = sm;                                           // [n]
  unsigned char* er = reinterpret_cast<unsigned char*>(lab + n);   // [n] edge to the right neighbour present
  unsigned char* ed = er + n;                                      // [n] edge to the lower neighbour present
  const size_t o = ((size_t)blockIdx.y * gridDim.x + blockIdx.x) * n;       // (slab, level) -> offset; gridDim.x = L
  const float* cr = cos_right + o;
  const float* cd = cos_down + o;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int h = i / side_w, w = i - h * side_w;
    float s = 0.f;
    int cnt = 0;
    if (w + 1 < side_w) { s += cr[i]; ++cnt; }
    if (w > 0) { s += cr[i - 1]; ++cnt; }
    if (h + 1 < side_h) { s += cd[i]; ++cnt; }
    if (h > 0) { s += cd[i - side_w]; ++cnt; }
    agreement[o + i] = cnt ? s / (float)cnt : 1.f;
    er[i] = (w + 1 < side_w) && cr[i] >= threshold;
    ed[i] = (h + 1 < side_h) && cd[i] >= threshold;
    lab[i] = i;
  }
  __syncthreads();
  // Jacobi min-label propagation: converges in at most (longest shortest path in a component) sweeps <= n
  for (int sweep = 0; sweep < n; ++sweep) {
    int changed = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const int h = i / side_w, w = i - h * side_w;
      int m = lab[i];
      if (er[i]) m = min(m, lab[i + 1]);
      if (w > 0 && er[i - 1]) m = min(m, lab[i - 1]);
      if (ed[i]) m = min(m, lab[i + side_w]);
      if (h > 0 && ed[i - side_w]) m = min(m, lab[i - side_w]);
      if (m < lab[i]) { atomicMin(&lab[i], m); changed = 1; }
    }
    if (!__syncthreads_or(changed)) break;
  }
  __shared__ int total;
  if (threadIdx.x == 0) total = 0;
  __syncthreads();
  int roots = 0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    labels[o + i] = lab[i];
    roots += lab[i] == i;                                  // a component's id is its smallest patch index
  }
  if (roots) atomicAdd(&total, roots);
  __syncthreads();
  if (threadIdx.x == 0) num_islands[(size_t)blockIdx.y * gridDim.x + blockIdx.x] = total;
}

int launch_islands(const float* states, int slabs, int side_h, int side_w, int L, int d, float threshold, float* cos_right,
                   float* cos_down, float* agreement, int* labels, int* num_islands, Launch& ln) {
  cudaStream_t st = ln.st;
  const int n = side_h * side_w;
  island_edges_kernel<<<dim3(side_h, L, slabs), 256, 0, st>>>(states, side_h, side_w, L, d, cos_right, cos_down);
  GLOM_TRY(ln.launched());
  const size_t smem = (size_t)n * 4 + 2 * (size_t)n;
  // 6n bytes plus the kernel's static shared memory exceed the default 48 KB per block from n = 8190 on (the API allows
  // n <= 8192): opt in above 46 KB
  static SmemOptIn optin;
  if (smem > 46 * 1024) GLOM_TRY(ln.check(optin.ensure(island_label_kernel, smem)));
  island_label_kernel<<<dim3(L, slabs), 256, smem, st>>>(cos_right, cos_down, side_h, side_w, threshold, agreement,
                                                          labels, num_islands);
  return ln.launched();
}

}  // namespace glom
