// Glom.settle on CUDA cores: the per-image stopping rule applied after every step, and the final gather of the images
// whose last state sits in the workspace's half of the ping-pong.  Also the per-image step counts of
// glom_b200_forward_steps: the flags of each step from the given counts, and the return_all fill of stopped images' slabs.
#include "engine.h"
#include "ptx.cuh"

#include <math.h>

namespace glom {

constexpr int SETTLE_THREADS = 256;

// Grid (L, B), after the GEMM2+combine launch of step `step` (which wrote S_step and the partials of every row of the
// images still running).  Block (l, b) of a running image reduces
//   q_bl = sqrt( sum_i |S_step[b,i,l] - S_{step-1}[b,i,l]|^2 / sum_i |S_step[b,i,l]|^2 )
// from the squared-change and squared-norm partials (rows, L, nparts) in a fixed order: thread t sums the rows
// t, t + 256, ... (each row's partials in order), then an xor tree per warp and the 8 warp sums in order.  0/0 counts
// as 0, x/0 (x > 0) as inf.  The block that finishes last applies the rule, max_l q_bl <= tol, i.e. q_bl <= tol for
// every level (a NaN never stops an image): steps[b] = step for every running image, frozen[b] = 1 for those that stop
// (so an image that never stops ends with steps[b] = max_iters), and recomputes the per-256-row-block flags.
__global__ void __launch_bounds__(SETTLE_THREADS)
settle_converge_kernel(int n, int L, int nparts, int B, int rows, int step, float tol, const float* __restrict__ dsq,
                       const float* __restrict__ nsq, int* frozen, int* block_frozen, unsigned int* done, float* level_q,
                       int32_t* steps) {
  pdl_launch_dependents();
  pdl_wait();                                       // the partials of this step are complete and visible
  const int l = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  __shared__ float red[2][SETTLE_THREADS / 32];
  __shared__ bool last;
  if (!frozen[b]) {                                 // block-uniform
    float num = 0.f, den = 0.f;
    for (int i = tid; i < n; i += SETTLE_THREADS) {
      const size_t o = (((size_t)b * n + i) * L + l) * nparts;
      float a = 0.f, c = 0.f;
      for (int q = 0; q < nparts; ++q) { a += dsq[o + q]; c += nsq[o + q]; }
      num += a; den += c;
    }
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
      num += __shfl_xor_sync(0xffffffffu, num, s);
      den += __shfl_xor_sync(0xffffffffu, den, s);
    }
    if (lane == 0) { red[0][warp] = num; red[1][warp] = den; }
    __syncthreads();
    if (tid == 0) {
      num = red[0][0]; den = red[1][0];
      for (int w = 1; w < SETTLE_THREADS / 32; ++w) { num += red[0][w]; den += red[1][w]; }
      level_q[(size_t)b * L + l] = (num == 0.f && den == 0.f) ? 0.f : sqrtf(num / den);
    }
  }
  // last block of the grid: every q of this step is written (fence before the count, fence after it)
  if (tid == 0) {
    __threadfence();
    last = atomicAdd(done, 1u) == gridDim.x * gridDim.y - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  for (int bb = tid; bb < B; bb += SETTLE_THREADS) {
    if (frozen[bb]) continue;
    bool stop = true;
    for (int ll = 0; ll < L; ++ll) stop = stop && __ldcg(level_q + (size_t)bb * L + ll) <= tol;
    steps[bb] = step;
    if (stop) frozen[bb] = 1;
  }
  __syncthreads();
  const int nblk = (rows + 255) / 256;
  for (int m = tid; m < nblk; m += SETTLE_THREADS) {
    const int b0 = m * 256 / n, b1 = (min(rows, m * 256 + 256) - 1) / n;
    int all = 1;
    for (int bb = b0; bb <= b1 && all; ++bb) all = frozen[bb];
    block_frozen[m] = all;
  }
  if (tid == 0) *done = 0u;                         // ready for the next step's launch
}

cudaError_t launch_settle_converge(const Geometry& g, int step, float tol, const float* dsq, const float* nsq, int* frozen,
                                   int* block_frozen, unsigned int* done, float* level_q, int32_t* steps, cudaStream_t st,
                                   int* launches) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(g.L, g.B);
  cfg.blockDim = dim3(SETTLE_THREADS);
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;      // PDL: see pdl_wait() in the kernel
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  if (launches) ++*launches;
  return cudaLaunchKernelEx(&cfg, settle_converge_kernel, g.n, g.L, g.nparts, g.B, g.rows, step, tol, dsq, nsq, frozen,
                            block_frozen, done, level_q, steps);
}

__device__ __forceinline__ int clamp_steps(int s, int max_steps) { return min(max(s, 0), max_steps); }

// Grid (chunks, B): image b stopped after steps[b] steps; its state S_steps[b] was written by that step into the buffer
// of the ping-pong that holds S_t for t of the same parity, and never again.  Copy it into state_out when that buffer
// is the workspace slab, i.e. when max_iters - steps[b] is odd.  An image with steps[b] == 0 (forward_steps only) when
// no step materialised S_0 (s0 != NULL) is copied from the carried state, or init_levels (L, d) broadcast over its columns.
__global__ void settle_gather_kernel(int max_iters, const int32_t* __restrict__ steps, size_t per_img4,
                                     const float4* __restrict__ src, float4* __restrict__ dst,
                                     const float4* __restrict__ s0, int s0_bcast, unsigned ld4) {
  const int b = blockIdx.y;
  const int s = clamp_steps(steps[b], max_iters);
  const size_t o = (size_t)b * per_img4;
  if (s == 0 && s0) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < per_img4; i += (size_t)gridDim.x * blockDim.x)
      dst[o + i] = s0_bcast ? s0[i % ld4] : s0[o + i];
    return;
  }
  if (((max_iters - s) & 1) == 0) return;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < per_img4; i += (size_t)gridDim.x * blockDim.x)
    dst[o + i] = src[o + i];
}

static unsigned copy_chunks(const Geometry& g, size_t per_img4) {
  const size_t want = (per_img4 + 255) / 256, cap = (size_t)(4 * sm_count() + g.B - 1) / g.B;
  return (unsigned)(want < cap ? want : cap);
}

cudaError_t launch_settle_gather(const Geometry& g, int max_iters, const int32_t* steps, const float* slab, float* state_out,
                                 const float* s0, int s0_bcast, cudaStream_t st, int* launches) {
  const size_t per_img4 = (size_t)g.n * g.L * g.d / 4;
  settle_gather_kernel<<<dim3(copy_chunks(g, per_img4), g.B), 256, 0, st>>>(
      max_iters, steps, per_img4, reinterpret_cast<const float4*>(slab), reinterpret_cast<float4*>(state_out),
      reinterpret_cast<const float4*>(s0), s0_bcast, (unsigned)(g.L * g.d / 4));
  if (launches) ++*launches;
  return cudaGetLastError();
}

// glom_b200_forward_steps, before step t: frozen[b] = steps[b] <= t (steps clamped to [0, max_steps]) and
// block_frozen[m] = 1 when every image with rows in the 256-row block m is frozen.  One thread per image and per block.
__global__ void __launch_bounds__(SETTLE_THREADS)
steps_schedule_kernel(int n, int B, int rows, int t, int max_steps, const int32_t* __restrict__ steps, int* frozen,
                      int* block_frozen) {
  pdl_launch_dependents();
  pdl_wait();                                       // the previous step's kernels have stopped reading the flags
  const int nblk = (rows + 255) / 256;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < B + nblk; i += gridDim.x * blockDim.x) {
    if (i < B) {
      frozen[i] = clamp_steps(steps[i], max_steps) <= t;
    } else {
      const int m = i - B;
      const int b0 = m * 256 / n, b1 = (min(rows, m * 256 + 256) - 1) / n;
      int all = 1;
      for (int bb = b0; bb <= b1 && all; ++bb) all = clamp_steps(steps[bb], max_steps) <= t;
      block_frozen[m] = all;
    }
  }
}

cudaError_t launch_steps_schedule(const Geometry& g, int t, int max_steps, const int32_t* steps, int* frozen, int* block_frozen,
                                  cudaStream_t st, int* launches) {
  const int items = g.B + (g.rows + 255) / 256;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((items + SETTLE_THREADS - 1) / SETTLE_THREADS);
  cfg.blockDim = dim3(SETTLE_THREADS);
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;      // PDL: see pdl_wait() in the kernel
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  if (launches) ++*launches;
  return cudaLaunchKernelEx(&cfg, steps_schedule_kernel, g.n, g.B, g.rows, t, max_steps, steps, frozen, block_frozen);
}

// Grid (chunks, B), return_all: the step kernels store nothing for the rows of a frozen image, so slabs
// steps[b]+1 .. max_steps of image b were never written.  Each of them receives a copy of slab steps[b].
__global__ void steps_fill_kernel(int max_steps, const int32_t* __restrict__ steps, size_t per_img4, size_t slab4,
                                  float4* __restrict__ states) {
  const int b = blockIdx.y;
  const int s = clamp_steps(steps[b], max_steps);
  if (s == max_steps) return;
  const size_t o = (size_t)b * per_img4;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < per_img4; i += (size_t)gridDim.x * blockDim.x) {
    const float4 v = states[(size_t)s * slab4 + o + i];
    for (int t = s + 1; t <= max_steps; ++t) states[(size_t)t * slab4 + o + i] = v;
  }
}

cudaError_t launch_steps_fill(const Geometry& g, int max_steps, const int32_t* steps, float* states, cudaStream_t st,
                              int* launches) {
  const size_t per_img4 = (size_t)g.n * g.L * g.d / 4;
  steps_fill_kernel<<<dim3(copy_chunks(g, per_img4), g.B), 256, 0, st>>>(max_steps, steps, per_img4, per_img4 * g.B,
                                                                         reinterpret_cast<float4*>(states));
  if (launches) ++*launches;
  return cudaGetLastError();
}

}  // namespace glom
