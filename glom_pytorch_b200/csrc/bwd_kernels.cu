// Backward of the GLOM column update -- the reverse loop, the fp32 CUDA-core kernels, and the dispatch to
// the tensor-core GEMMs of tc_bwd_kernels.cu for the bf16 engine.
//
// Differentiates glom_pytorch/glom_pytorch.py:131-145 step by step in reverse, recomputing the per-step
// intermediates (MLP pre-activations, attention probabilities) from the saved states S_0..S_T instead of
// storing them:
//   S_{t+1} = (S_t + BU(S_t, X) + TD(S_t + P) + C(S_t)) / c          (:141-142)
// All contractions go through one strided, batched fp32 GEMM (NN / NT / TN are just stride choices), the rest
// are small element-wise / row-reduction kernels.  With precision fp32 (or dim % 256 != 0) this file is the whole
// backward; with precision bf16 `backward_run` sends the MLP and consensus GEMMs to the tensor cores (`mlp_backward_tc`,
// `attn_bwd_gemm_tc`) and keeps the softmax / normalisation / bias reductions here.
#include "engine.h"
#include "ptx.cuh"

namespace glom {

// =====================================================================================
// C[z](m, n) = alpha * sum_k A[z](m, k) * B[z](k, n) + beta * C[z](m, n) (+ bias[n])
// element (i, j) of an operand of batch z = (z / zdiv, z % zdiv) lives at
//   base + (z / zdiv) * s_b0 + (z % zdiv) * s_b1 + i * s_row + j * s_col
// =====================================================================================
struct Mat {
  const float* p;
  long long s_row, s_col, s_b0, s_b1;
};
struct MatOut {
  float* p;
  long long s_row, s_col, s_b0, s_b1;
};
struct GemmF32 {
  int M, N, K, zdiv;
  Mat A;        // (m, k)
  Mat B;        // (k, n)
  MatOut C;     // (m, n)
  float alpha, beta;
  const float* bias;   // optional, per n
};

__global__ void __launch_bounds__(256) gemm_f32_kernel(GemmF32 q) {
  __shared__ float As[16][64 + 4];
  __shared__ float Bs[16][64 + 4];
  const int z = blockIdx.z, z0 = z / q.zdiv, z1 = z % q.zdiv;
  const float* A = q.A.p + z0 * q.A.s_b0 + z1 * q.A.s_b1;
  const float* B = q.B.p + z0 * q.B.s_b0 + z1 * q.B.s_b1;
  float* C = q.C.p + z0 * q.C.s_b0 + z1 * q.C.s_b1;
  const int m0 = blockIdx.x * 64, n0 = blockIdx.y * 64;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  // pick the load order that walks the operand's unit-stride dimension with consecutive threads
  const bool a_k_fast = (q.A.s_col == 1), b_k_fast = (q.B.s_row == 1);
  float acc[4][4] = {};
  for (int k0 = 0; k0 < q.K; k0 += 16) {
    for (int i = threadIdx.x; i < 64 * 16; i += 256) {
      int kk, rr;
      if (a_k_fast) { kk = i & 15; rr = i >> 4; } else { rr = i & 63; kk = i >> 6; }
      As[kk][rr] = (m0 + rr < q.M && k0 + kk < q.K) ? A[(long long)(m0 + rr) * q.A.s_row + (long long)(k0 + kk) * q.A.s_col] : 0.f;
      if (b_k_fast) { kk = i & 15; rr = i >> 4; } else { rr = i & 63; kk = i >> 6; }
      Bs[kk][rr] = (n0 + rr < q.N && k0 + kk < q.K) ? B[(long long)(k0 + kk) * q.B.s_row + (long long)(n0 + rr) * q.B.s_col] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Bs[kk][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = m0 + ty * 4 + i;
    if (r >= q.M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = n0 + tx * 4 + j;
      if (c >= q.N) continue;
      float* dst = C + (long long)r * q.C.s_row + (long long)c * q.C.s_col;
      float v = q.alpha * acc[i][j];
      if (q.bias) v += q.bias[c];
      if (q.beta != 0.f) v += q.beta * *dst;
      *dst = v;
    }
  }
}

static cudaError_t gemm_f32(const GemmF32& q, int batches, cudaStream_t st, int* launches) {
  dim3 grid((q.M + 63) / 64, (q.N + 63) / 64, batches);
  gemm_f32_kernel<<<grid, 256, 0, st>>>(q);
  if (launches) ++*launches;
  return cudaGetLastError();
}

// =====================================================================================
// element-wise / reduction helpers
// =====================================================================================
// g (R, L, d)  <-  (gin + extra) (R, L, d) / c_l   (:142);   ds (R, L, d) <- g (residual term of the sum, :141)
// `extra` (nullable) is the upstream gradient of this time step's own output when every step is returned (:147-148)
// steps (nullable): per-image step counts; an image with steps[b] <= t is the identity at step t, so its rows get
// g = 0 (every later contribution of theirs is an exact zero) and ds = gin + extra unscaled.  g_kept: g already holds
// those zeros (written at reverse step t + 1, where the image was frozen too), so they are not stored again
__global__ void scale_by_contrib_kernel(size_t total, int L, int d, const float* __restrict__ gin,
                                        const float* __restrict__ extra, float* __restrict__ g, float* __restrict__ ds,
                                        const int32_t* __restrict__ steps, int t, size_t img4, int g_kept) {
  const size_t total4 = total / 4;
  const unsigned d4 = (unsigned)d / 4;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (size_t)gridDim.x * blockDim.x) {
    const unsigned l = (unsigned)((i / d4) % (unsigned)L);
    float4 v = reinterpret_cast<const float4*>(gin)[i];
    if (extra) { const float4 e = reinterpret_cast<const float4*>(extra)[i]; v.x += e.x; v.y += e.y; v.z += e.z; v.w += e.w; }
    if (steps && __ldg(steps + i / img4) <= t) {
      if (!g_kept) reinterpret_cast<float4*>(g)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      reinterpret_cast<float4*>(ds)[i] = v;
      continue;
    }
    if (l == (unsigned)L - 1) { v.x /= 3.0f; v.y /= 3.0f; v.z /= 3.0f; v.w /= 3.0f; }
    else { v.x *= 0.25f; v.y *= 0.25f; v.z *= 0.25f; v.w *= 0.25f; }
    reinterpret_cast<float4*>(g)[i] = v;
    reinterpret_cast<float4*>(ds)[i] = v;
  }
}
// xp (R, d) = S[:, l, :] + pos[row % n]     (top-down input, :136)
__global__ void add_pos_kernel(int rows, int n, int L, int d, int l, const float* __restrict__ s,
                               const float* __restrict__ pos, float* __restrict__ xp) {
  const size_t total = (size_t)rows * d;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t r = i / d;
    const int c = (int)(i % d);
    xp[i] = s[(r * L + l) * d + c] + pos[(size_t)(r % n) * d + c];
  }
}
// h = gelu(pre) ; dpre = dh * gelu'(pre)   (exact erf form, :30), dpre overwrites dh
__global__ void gelu_bwd_kernel(size_t total, const float* __restrict__ pre, float* __restrict__ h,
                                float* __restrict__ dh) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const float x = pre[i];
    const float cdf = 0.5f * (1.0f + erff(x * 0.70710678118654752440f));
    const float pdf = 0.39894228040143267794f * expf(-0.5f * x * x);
    h[i] = x * cdf;
    dh[i] = dh[i] * (cdf + x * pdf);
  }
}
// out[c] += sum_r src[r * row_stride + c]          (bias gradients); grid (cols / 32, row chunks)
// out2 (nullable) receives the same sums for its first cols2 columns (the top-down second-layer biases see the
// same upstream gradient as the bottom-up ones on levels 0 .. L-2)
// steps (nullable): rows r of images frozen at reverse step t (steps[r / n] <= t) hold zeros and are not read; the sums
// are the same bits
__global__ void colsum_acc_kernel(int rows, int cols, long long row_stride, const float* __restrict__ src,
                                  float* __restrict__ out, float* __restrict__ out2 = nullptr, int cols2 = 0,
                                  const int32_t* __restrict__ steps = nullptr, int t = 0, int n = 1) {
  const int c = blockIdx.x * 32 + (threadIdx.x & 31);
  const int part = threadIdx.x >> 5;                 // 8 row slices per block
  const int r_begin = (int)(((long long)rows * blockIdx.y) / gridDim.y), r_end = (int)(((long long)rows * (blockIdx.y + 1)) / gridDim.y);
  __shared__ float red[8][33];
  float acc = 0.f;
  if (c < cols && !steps)
    for (int r = r_begin + part; r < r_end; r += 8) acc += src[(long long)r * row_stride + c];
  else if (c < cols)
    for (int r = r_begin + part; r < r_end; r += 8)
      if (__ldg(steps + r / n) > t) acc += src[(long long)r * row_stride + c];
  red[part][threadIdx.x & 31] = acc;
  __syncthreads();
  if (part == 0 && c < cols) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += red[i][threadIdx.x & 31];
    atomicAdd(out + c, s);
    if (out2 && c < cols2) atomicAdd(out2 + c, s);
  }
}
// dpos[nn, c] += sum_b dx[(b * n + nn), c]          (positional-embedding gradient, :136)
__global__ void pos_grad_kernel(int B, int n, int d, const float* __restrict__ dx, float* __restrict__ dpos) {
  const size_t total = (size_t)n * d;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    float acc = 0.f;
    for (int b = 0; b < B; ++b) acc += dx[(size_t)b * total + i];
    dpos[i] += acc;
  }
}
// dst[:, l, :] += src (R, d)
__global__ void add_into_level_kernel(int rows, int L, int d, int l, const float* __restrict__ src,
                                      float* __restrict__ dst) {
  const size_t total = (size_t)rows * d;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x)
    dst[((i / d) * L + l) * d + (i % d)] += src[i];
}
__global__ void add_kernel(size_t total, const float* __restrict__ src, float* __restrict__ dst) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x)
    dst[i] += src[i];
}
// The four warp-per-row kernels of the attention backward take `FrozenRows`: at reverse step t of the tensor-core
// backward with per-image step counts, the rows of images with steps[b] <= t are skipped.  Their rows are image-major in
// both row spaces, (row, level) and (image * L + level, query), so image = row / (n L).  A skipped row's outputs (khat,
// rnorm, khat_b, A, a_b, dA, dsim_b; ds is not touched) keep whatever they held, possibly never written: every reader of
// them skips the same rows.
struct FrozenRows {
  const int32_t* steps;      // NULL: no row is skipped
  int t, rows_per_image;
  __device__ __forceinline__ bool operator()(int row) const {
    return steps && __ldg(steps + row / rows_per_image) <= t;
  }
};

// khat = S / max(|S|, 1e-12) per (row, level) ; rnorm = 1 / max(|S|, 1e-12)      (F.normalize, :58)
__global__ void normalize_rows_kernel(int nrows, int d, const float* __restrict__ s, float* __restrict__ khat,
                                      float* __restrict__ rnorm, __nv_bfloat16* __restrict__ khat_b, FrozenRows frozen) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= nrows || frozen(row)) return;
  const float* p = s + (size_t)row * d;
  float ss = 0.f;
  for (int c = lane; c < d; c += 32) ss = fmaf(p[c], p[c], ss);
#pragma unroll
  for (int o = 16; o; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float r = 1.0f / fmaxf(sqrtf(ss), 1e-12f);
  for (int c = lane; c < d; c += 32) {
    const float v = p[c] * r;
    khat[(size_t)row * d + c] = v;
    if (khat_b) khat_b[(size_t)row * d + c] = __float2bfloat16_rn(v);
  }
  if (lane == 0) rnorm[row] = r;
}
// in-place masked softmax over the last dim of sim (Z, n, n)     (:62-71); one warp per row
__global__ void attn_softmax_kernel(int Z, int n, int attend_self, int mask_side, int mask_d2_max, float scale,
                                    float* __restrict__ sim, __nv_bfloat16* __restrict__ a_b, FrozenRows frozen) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= Z * n || frozen(row)) return;
  const int i = row % n;
  float* p = sim + (size_t)row * n;
  float m = -3.402823466e+38f;
  for (int j = lane; j < n; j += 32) {
    float v = p[j] * scale;
    if (!attend_self && j == i) v = -5e-4f;
    if (mask_side > 0) {
      const int dh = i / mask_side - j / mask_side, dw = i % mask_side - j % mask_side;
      if (dh * dh + dw * dw > mask_d2_max) v = -3.402823466e+38f;
    }
    p[j] = v;
    m = fmaxf(m, v);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  float sum = 0.f;
  for (int j = lane; j < n; j += 32) { const float e = expf(p[j] - m); p[j] = e; sum += e; }
#pragma unroll
  for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float inv = 1.0f / sum;
  for (int j = lane; j < n; j += 32) {
    const float a = p[j] * inv;
    p[j] = a;
    if (a_b) a_b[(size_t)row * n + j] = __float2bfloat16_rn(a);
  }
}
// dsim = A * (dA - sum_j A dA), zero where the logit was a constant (diagonal fill, radius mask); in place on dA
__global__ void attn_softmax_bwd_kernel(int Z, int n, int attend_self, int mask_side, int mask_d2_max,
                                        const float* __restrict__ A, float* __restrict__ dA, float scale,
                                        __nv_bfloat16* __restrict__ dsim_b, FrozenRows frozen) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= Z * n || frozen(row)) return;
  const int i = row % n;
  const float* a = A + (size_t)row * n;
  float* g = dA + (size_t)row * n;
  float dot = 0.f;
  for (int j = lane; j < n; j += 32) dot = fmaf(a[j], g[j], dot);
#pragma unroll
  for (int o = 16; o; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
  for (int j = lane; j < n; j += 32) {
    float v = a[j] * (g[j] - dot);
    if (!attend_self && j == i) v = 0.f;
    if (mask_side > 0) {
      const int dh = i / mask_side - j / mask_side, dw = i % mask_side - j % mask_side;
      if (dh * dh + dw * dw > mask_d2_max) v = 0.f;
    }
    g[j] = v;
    if (dsim_b) dsim_b[(size_t)row * n + j] = __float2bfloat16_rn(v * scale);
  }
}
// ds[row] += (dkhat - khat (khat . dkhat)) * rnorm        (backward of F.normalize); one warp per (row, level)
__global__ void normalize_bwd_kernel(int nrows, int d, const float* __restrict__ khat, const float* __restrict__ dkhat,
                                     const float* __restrict__ rnorm, float* __restrict__ ds, FrozenRows frozen) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= nrows || frozen(row)) return;
  const float* k = khat + (size_t)row * d;
  const float* g = dkhat + (size_t)row * d;
  float dot = 0.f;
  for (int c = lane; c < d; c += 32) dot = fmaf(k[c], g[c], dot);
#pragma unroll
  for (int o = 16; o; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
  const float r = rnorm[row];
  for (int c = lane; c < d; c += 32) ds[(size_t)row * d + c] += (g[c] - k[c] * dot) * r;
}
// dinit[l, c] = sum over rows of g[(row, l, c)]           (broadcast of init_levels, :124); grid (L*d/256, row chunks)
__global__ void init_grad_kernel(int rows, int L, int d, const float* __restrict__ g, float* __restrict__ dinit) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L * d) return;
  const int r_begin = (int)(((long long)rows * blockIdx.y) / gridDim.y), r_end = (int)(((long long)rows * (blockIdx.y + 1)) / gridDim.y);
  float acc = 0.f;
  for (int r = r_begin; r < r_end; ++r) acc += g[(size_t)r * L * d + i];
  atomicAdd(dinit + i, acc);
}

// ---- the deterministic backward's reductions (BackwardArgs::deterministic): no floating-point atomics, and every sum
// runs in an order fixed by the shapes alone -- never by the grid size, the SM count or the order blocks run in.
// colsum_acc_kernel and init_grad_kernel as one fixed-order column sum: out[c] += sum_r src[r * row_stride + c], out2 as
// in colsum_acc_kernel, the same frozen rows skipped.  One block owns 32 columns and every row: thread (x, y) sums rows
// y, y + 32, ... of its column in order, then row y = 0 adds the 32 slice sums in slice order.
__global__ void __launch_bounds__(1024) colsum_det_kernel(int rows, int cols, long long row_stride,
                                                          const float* __restrict__ src, float* __restrict__ out,
                                                          float* __restrict__ out2, int cols2,
                                                          const int32_t* __restrict__ steps, int t, int n) {
  const int c = blockIdx.x * 32 + threadIdx.x, y = threadIdx.y;
  __shared__ float red[32][33];
  float acc = 0.f;
  if (c < cols) {
#pragma unroll 4
    for (int r = y; r < rows; r += 32)
      if (!steps || __ldg(steps + r / n) > t) acc += src[(long long)r * row_stride + c];
  }
  red[y][threadIdx.x] = acc;
  __syncthreads();
  if (y == 0 && c < cols) {
    float s = red[0][threadIdx.x];
#pragma unroll
    for (int i = 1; i < 32; ++i) s += red[i][threadIdx.x];
    out[c] += s;
    if (out2 && c < cols2) out2[c] += s;
  }
}
static cudaError_t colsum(bool det, int rows, int cols, long long row_stride, const float* src, float* out, float* out2,
                          int cols2, const int32_t* steps, int t, int n, cudaStream_t st, int* launches) {
  if (det)
    colsum_det_kernel<<<(cols + 31) / 32, dim3(32, 32), 0, st>>>(rows, cols, row_stride, src, out, out2, cols2, steps, t, n);
  else
    colsum_acc_kernel<<<dim3((cols + 31) / 32, 16), 256, 0, st>>>(rows, cols, row_stride, src, out, out2, cols2, steps, t, n);
  if (launches) ++*launches;
  return cudaGetLastError();
}
// After BW_DX<DET>: ds[r, l + 1] += dx_td[r, l] for the top-down groups l = 0 .. L-2, and dpos[i] += the sum of
// dx_td[b n + i, l] over images b, and groups l within an image.  Block = 32 float4 columns x 8 image slices of one
// position i: slice y takes images y, y + 8, ... in order, then slice 0 adds the 8 slice sums in slice order.  Images
// frozen at reverse step t (steps[b] <= t) are skipped: BW_DX skipped their row blocks and wrote nothing for them
__global__ void __launch_bounds__(256) dx_td_reduce_kernel(int B, int n, int L, int d, const float* __restrict__ dx_td,
                                                           float* __restrict__ ds, float* __restrict__ dpos,
                                                           const int32_t* __restrict__ steps, int t) {
  const int d4 = d / 4, chunks = (d4 + 31) / 32;
  const int i = blockIdx.x / chunks, c4 = (blockIdx.x % chunks) * 32 + threadIdx.x, y = threadIdx.y;
  __shared__ float4 red[8][32];
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (c4 < d4) {
    for (int b = y; b < B; b += 8) {
      if (steps && __ldg(steps + b) <= t) continue;
      const size_t r = (size_t)b * n + i;
      const float4* src = reinterpret_cast<const float4*>(dx_td) + r * (L - 1) * d4 + c4;
      float4* dst = reinterpret_cast<float4*>(ds) + (r * L + 1) * d4 + c4;
#pragma unroll 4
      for (int l = 0; l < L - 1; ++l) {
        const float4 v = src[(size_t)l * d4];
        float4 o = dst[(size_t)l * d4];
        o.x += v.x; o.y += v.y; o.z += v.z; o.w += v.w;
        dst[(size_t)l * d4] = o;
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
      }
    }
  }
  red[y][threadIdx.x] = acc;
  __syncthreads();
  if (y == 0 && c4 < d4) {
    float4 s = red[0][threadIdx.x];
#pragma unroll
    for (int k = 1; k < 8; ++k) { const float4 v = red[k][threadIdx.x]; s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w; }
    float4* p = reinterpret_cast<float4*>(dpos) + (size_t)i * d4 + c4;
    float4 o = *p;
    o.x += s.x; o.y += s.y; o.z += s.z; o.w += s.w;
    *p = o;
  }
}
// After BW_DH<DET>: d_*_b1[g, j] += the sum over 32-row bands k of part[g][k][j].  Block = 32 float4 columns x 16 band
// slices: slice y takes bands y, y + 16, ... in order, then slice 0 adds the 16 slice sums in slice order.  A band whose
// rows all belong to images frozen at reverse step t is skipped: BW_DH wrote nothing there when it skipped the band's
// 128-row block, and exact zeros otherwise
__global__ void __launch_bounds__(512) bias_partials_kernel(int G, int nbands, int rows, int n, int d,
                                                            const float* __restrict__ part, float* __restrict__ d_bu_b1,
                                                            float* __restrict__ d_td_b1, const int32_t* __restrict__ steps,
                                                            int t) {
  const int q = blockIdx.x * 32 + threadIdx.x, y = threadIdx.y;     // q: float4 column of the (G, 4d) bias gradients
  __shared__ float4 red[16][32];
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (q < G * d) {
    const float4* src = reinterpret_cast<const float4*>(part) + (size_t)(q / d) * nbands * d + q % d;
    for (int k = y; k < nbands; k += 16) {
      if (steps) {
        const int r1 = min(32 * k + 32, rows);
        bool live = false;
        for (int b = 32 * k / n; b <= (r1 - 1) / n && !live; ++b) live = __ldg(steps + b) > t;
        if (!live) continue;
      }
      const float4 v = src[(size_t)k * d];
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
  }
  red[y][threadIdx.x] = acc;
  __syncthreads();
  if (y == 0 && q < G * d) {
    float4 s = red[0][threadIdx.x];
#pragma unroll
    for (int k = 1; k < 16; ++k) { const float4 v = red[k][threadIdx.x]; s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w; }
    const int g = q / d;
    float4* p = reinterpret_cast<float4*>(((g & 1) ? d_td_b1 : d_bu_b1) + (size_t)(g >> 1) * 4 * d) + q % d;
    float4 o = *p;
    o.x += s.x; o.y += s.y; o.z += s.z; o.w += s.w;
    *p = o;
  }
}

// =====================================================================================
// Tokeniser backward (image_to_tokens: Rearrange + Linear, glom_pytorch.py:94-97) -- fp32 on CUDA cores
//   d_weight (d, 3p^2) += dTok^T . patches,  d_bias (d) += column sums of dTok,
//   d_img (B, 3, H, W)  = fold(dTok . W)     (patches do not overlap: the fold is a permutation)
// =====================================================================================
// 'b c (h p1) (w p2) -> b (h w) (p1 p2 c)' (:95): patches[r][k] with r = (b, ph, pw), k = (p1 p + p2) 3 + c
__global__ void patchify_f32_kernel(const float* __restrict__ img, float* __restrict__ patches, int B, int H, int W, int p) {
  const int hp = H / p, wp = W / p, k3 = 3 * p * p;
  const size_t total = (size_t)B * hp * wp * k3;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t r = i / k3;
    const int k = (int)(i % k3);
    const int b = (int)(r / ((size_t)hp * wp)), pr = (int)(r % ((size_t)hp * wp)), ph = pr / wp, pw = pr % wp;
    const int c = k % 3, p12 = k / 3, p1 = p12 / p, p2 = p12 % p;
    patches[i] = img[(((size_t)b * 3 + c) * H + ph * p + p1) * W + pw * p + p2];
  }
}
// the inverse permutation: d_img[b][c][y][x] += dpatches[r][k]
__global__ void unpatchify_add_kernel(const float* __restrict__ dpatches, float* __restrict__ dimg, int B, int H, int W, int p) {
  const int hp = H / p, wp = W / p, k3 = 3 * p * p;
  const size_t total = (size_t)B * 3 * H * W;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % W), y = (int)((i / W) % H), c = (int)((i / ((size_t)W * H)) % 3), b = (int)(i / ((size_t)3 * W * H));
    const int ph = y / p, p1 = y % p, pw = x / p, p2 = x % p;
    const size_t r = ((size_t)b * hp + ph) * wp + pw;
    dimg[i] += dpatches[r * k3 + (p1 * p + p2) * 3 + c];
  }
}

size_t tokenize_backward_workspace_bytes(int B, int H, int W, int p, int need_dimg) {
  const size_t rk = (size_t)B * (H / p) * (W / p) * 3 * p * p * sizeof(float);
  return align_up(rk, 1024) * (need_dimg ? 2 : 1);
}

cudaError_t tokenize_backward(const float* img, const float* weight, const float* d_tokens, float* d_weight, float* d_bias,
                              float* d_img, int B, int H, int W, int p, int d, void* workspace, cudaStream_t st, int* launches,
                              int deterministic) {
  const int rows = B * (H / p) * (W / p), k3 = 3 * p * p;
  float* patches = static_cast<float*>(workspace);
  float* dpatches = reinterpret_cast<float*>(static_cast<char*>(workspace) + align_up((size_t)rows * k3 * sizeof(float), 1024));
  cudaError_t e = cudaSuccess;
  if (d_weight) {
    const size_t total = (size_t)rows * k3;
    const size_t want = (total + 255) / 256;
    patchify_f32_kernel<<<(int)(want < sm_count() * 32 ? want : sm_count() * 32), 256, 0, st>>>(img, patches, B, H, W, p);
    if (launches) ++*launches;
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    // d_weight (d, k3) += dTok^T (d x rows) . patches (rows x k3)
    GemmF32 q{};
    q.M = d; q.N = k3; q.K = rows; q.zdiv = 1;
    q.A = {d_tokens, 1, d, 0, 0};
    q.B = {patches, k3, 1, 0, 0};
    q.C = {d_weight, k3, 1, 0, 0};
    q.alpha = 1.f; q.beta = 1.f; q.bias = nullptr;
    if ((e = gemm_f32(q, 1, st, launches)) != cudaSuccess) return e;
  }
  if (d_bias && (e = colsum(deterministic != 0, rows, d, (long long)d, d_tokens, d_bias, nullptr, 0, nullptr, 0, 1, st,
                            launches)) != cudaSuccess)
    return e;
  if (d_img) {
    // dpatches (rows, k3) = dTok (rows x d) . W (d x k3)
    GemmF32 q{};
    q.M = rows; q.N = k3; q.K = d; q.zdiv = 1;
    q.A = {d_tokens, d, 1, 0, 0};
    q.B = {weight, k3, 1, 0, 0};
    q.C = {dpatches, k3, 1, 0, 0};
    q.alpha = 1.f; q.beta = 0.f; q.bias = nullptr;
    if ((e = gemm_f32(q, 1, st, launches)) != cudaSuccess) return e;
    const size_t total = (size_t)B * 3 * H * W;
    const size_t want = (total + 255) / 256;
    unpatchify_add_kernel<<<(int)(want < sm_count() * 32 ? want : sm_count() * 32), 256, 0, st>>>(dpatches, d_img, B, H, W, p);
    if (launches) ++*launches;
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
  }
  return cudaSuccess;
}

__global__ void cast_bf16_rows(size_t n4, const float* __restrict__ src, __nv_bfloat16* __restrict__ dst) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(src)[i];
    reinterpret_cast<uint2*>(dst)[i] = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
  }
}

static inline int nblk(size_t total, int block = 256) {
  const size_t want = (total + block - 1) / block;
  return (int)(want < (size_t)sm_count() * 32 ? (want ? want : 1) : (size_t)sm_count() * 32);
}
#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return e_; } while (0)
#define CKL() do { if (launches) ++*launches; cudaError_t e_ = cudaGetLastError(); if (e_ != cudaSuccess) return e_; } while (0)

BackwardLayout backward_layout(const Geometry& g, int precision) {
  BackwardLayout w{};
  const size_t state = (size_t)g.rows * g.L * g.d * 4, hid = (size_t)g.rows * 4 * g.d * 4;
  const size_t attn = (size_t)g.B * g.L * g.n * g.n * 4;
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off = align_up(off + bytes, 1024); return o; };
  w.g_off = take(state); w.gs_off = take(state); w.ds_off = take(state);
  w.khat_off = take(state); w.dkhat_off = take(state);
  w.rnorm_off = take((size_t)g.rows * g.L * 4);
  w.pre_off = take(hid); w.h_off = take(hid); w.dh_off = take(hid);
  w.xp_off = take((size_t)g.rows * g.d * 4); w.dx_off = take((size_t)g.rows * g.d * 4);
  w.attn_off = take(attn); w.dattn_off = take(attn);
  if (precision == 1 && g.d % 256 == 0) {     // tensor-core MLP backward
    const size_t m128 = (g.rows + 127) / 128;
    w.blocked_bytes = (size_t)g.G * m128 * 128 * 4 * g.d * 2;
    w.xb_off = take((size_t)g.rows * g.d * 2);
    w.sb_off = take((size_t)g.rows * g.L * g.d * 2);
    w.sp_off = take((size_t)g.rows * (g.L - 1) * g.d * 2);
    w.gsb_off = take((size_t)g.rows * g.L * g.d * 2);
    w.w1p_off = take((size_t)g.G * 4 * g.d * g.d * 2);
    w.w2t_off = take((size_t)g.G * 4 * g.d * g.d * 2);
    w.w1t_off = take((size_t)g.G * 4 * g.d * g.d * 2);
    w.b1p_off = take((size_t)g.G * 4 * g.d * 4);
    w.bpre_off = take(w.blocked_bytes); w.bh_off = take(w.blocked_bytes); w.bdpre_off = take(w.blocked_bytes);
    w.khatb_off = take((size_t)g.rows * g.L * g.d * 2);
    w.ab_off = take((size_t)g.B * g.L * g.n * g.n * 2);
    w.dsimb_off = take((size_t)g.B * g.L * g.n * g.n * 2);
    // deterministic backward: BW_DH's bias partials [G][ceil(R/32)][4d] fp32 go to the fp32 pre / h / dh buffers, which
    // this path leaves unused; only shapes with very few rows per group need a region of their own.  (Its top-down dx
    // buffer (R, L-1, d) fp32 is dkhat, dead once normalize_bwd_kernel has run.)
    const size_t part = (size_t)g.G * ((g.rows + 31) / 32) * 4 * g.d * 4;
    w.b1part_off = part <= w.xp_off - w.pre_off ? w.pre_off : take(part);
  }
  w.total = off;
  return w;
}

// One reverse step: given gin = dL/dS_{t+1}, produce ds = dL/dS_t (without the external grad of slab t) and
// accumulate parameter / token / pos gradients.
static cudaError_t backward_step(const Geometry& g, const BackwardArgs& a, const float* s_t, const float* gin,
                                 const float* gextra, float* ds, char* ws, const BackwardLayout& wl, bool mlp_on_tc,
                                 bool attn_on_tc, const int32_t* steps, int t, bool gs_kept, cudaStream_t st, int* launches) {
  const int R = g.rows, L = g.L, d = g.d, n = g.n, h4 = 4 * g.d;
  const long long ld = (long long)L * d;
  float* gs = reinterpret_cast<float*>(ws + wl.gs_off);       // (gin + gextra) / c
  float* pre = reinterpret_cast<float*>(ws + wl.pre_off);
  float* hb = reinterpret_cast<float*>(ws + wl.h_off);
  float* dh = reinterpret_cast<float*>(ws + wl.dh_off);
  float* xp = reinterpret_cast<float*>(ws + wl.xp_off);
  float* dx = reinterpret_cast<float*>(ws + wl.dx_off);
  const size_t state = (size_t)R * L * d;
  scale_by_contrib_kernel<<<nblk(state), 256, 0, st>>>(state, L, d, gin, gextra, gs, ds, steps, t, (size_t)n * ld / 4,
                                                       gs_kept ? 1 : 0);
  CKL();

  // ---- the two grouped MLPs (:23-36), one group at a time (fp32 path; the bf16 engine runs them on tensor cores)
  for (int net = 0; net < 2 && !mlp_on_tc; ++net) {
    const int groups = net == 0 ? L : L - 1;
    const float* w1 = net == 0 ? a.bu_w1 : a.td_w1;
    const float* b1 = net == 0 ? a.bu_b1 : a.td_b1;
    const float* w2 = net == 0 ? a.bu_w2 : a.td_w2;
    float* dw1 = net == 0 ? a.d_bu_w1 : a.d_td_w1;
    float* db1 = net == 0 ? a.d_bu_b1 : a.d_td_b1;
    float* dw2 = net == 0 ? a.d_bu_w2 : a.d_td_w2;
    float* db2 = net == 0 ? a.d_bu_b2 : a.d_td_b2;
    for (int l = 0; l < groups; ++l) {
      // input of the group: bottom-up l reads tokens (l == 0) or S[l-1]; top-down l reads S[l+1] + pos
      Mat X{};
      if (net == 0 && l == 0) X = Mat{a.tokens, d, 1, 0, 0};
      else if (net == 0) X = Mat{s_t + (size_t)(l - 1) * d, ld, 1, 0, 0};
      else {
        add_pos_kernel<<<nblk((size_t)R * d), 256, 0, st>>>(R, n, L, d, l + 1, s_t, a.pos, xp);
        CKL();
        X = Mat{xp, d, 1, 0, 0};
      }
      const float* W1 = w1 + (size_t)l * h4 * d;       // (4d, d)
      const float* W2 = w2 + (size_t)l * d * h4;       // (d, 4d)
      const Mat DY{gs + (size_t)l * d, ld, 1, 0, 0};   // (R, d) slice of the scaled upstream gradient
      GemmF32 q{};
      // pre = X W1^T + b1                                 (R x 4d)
      q = GemmF32{R, h4, d, 1, X, Mat{W1, 1, d, 0, 0}, MatOut{pre, h4, 1, 0, 0}, 1.f, 0.f, b1 + (size_t)l * h4};
      CK(gemm_f32(q, 1, st, launches));
      // dh = DY W2                                        (R x 4d)
      q = GemmF32{R, h4, d, 1, DY, Mat{W2, h4, 1, 0, 0}, MatOut{dh, h4, 1, 0, 0}, 1.f, 0.f, nullptr};
      CK(gemm_f32(q, 1, st, launches));
      gelu_bwd_kernel<<<nblk((size_t)R * h4), 256, 0, st>>>((size_t)R * h4, pre, hb, dh);   // dh := dpre
      CKL();
      // dW2 += DY^T h                                     (d x 4d)
      q = GemmF32{d, h4, R, 1, Mat{DY.p, 1, ld, 0, 0}, Mat{hb, h4, 1, 0, 0}, MatOut{dw2 + (size_t)l * d * h4, h4, 1, 0, 0}, 1.f, 1.f, nullptr};
      CK(gemm_f32(q, 1, st, launches));
      CK(colsum(a.deterministic != 0, R, d, ld, DY.p, db2 + (size_t)l * d, nullptr, 0, nullptr, 0, 1, st, launches));
      // dW1 += dpre^T X                                   (4d x d)
      q = GemmF32{h4, d, R, 1, Mat{dh, 1, h4, 0, 0}, Mat{X.p, X.s_row, 1, 0, 0}, MatOut{dw1 + (size_t)l * h4 * d, d, 1, 0, 0}, 1.f, 1.f, nullptr};
      CK(gemm_f32(q, 1, st, launches));
      CK(colsum(a.deterministic != 0, R, h4, h4, dh, db1 + (size_t)l * h4, nullptr, 0, nullptr, 0, 1, st, launches));
      // dX = dpre W1                                      (R x d)
      q = GemmF32{R, d, h4, 1, Mat{dh, h4, 1, 0, 0}, Mat{W1, d, 1, 0, 0}, MatOut{dx, d, 1, 0, 0}, 1.f, 0.f, nullptr};
      CK(gemm_f32(q, 1, st, launches));
      if (net == 0 && l == 0) {
        add_kernel<<<nblk((size_t)R * d), 256, 0, st>>>((size_t)R * d, dx, a.d_tokens);
        CKL();
      } else if (net == 0) {
        add_into_level_kernel<<<nblk((size_t)R * d), 256, 0, st>>>(R, L, d, l - 1, dx, ds);
        CKL();
      } else {
        add_into_level_kernel<<<nblk((size_t)R * d), 256, 0, st>>>(R, L, d, l + 1, dx, ds);
        CKL();
        pos_grad_kernel<<<nblk((size_t)n * d), 256, 0, st>>>(g.B, n, d, dx, a.d_pos);
        CKL();
      }
    }
  }

  // ---- consensus attention (:56-73), all (image, level) problems batched (fp32 path)
  if (!attn_on_tc) {
    float* khat = reinterpret_cast<float*>(ws + wl.khat_off);
    float* dkhat = reinterpret_cast<float*>(ws + wl.dkhat_off);
    float* rnorm = reinterpret_cast<float*>(ws + wl.rnorm_off);
    float* A = reinterpret_cast<float*>(ws + wl.attn_off);
    float* dA = reinterpret_cast<float*>(ws + wl.dattn_off);
    const int Z = g.B * L;
    const long long sb = (long long)n * ld, sl = d, nn = (long long)n * n;
    const float scale = 1.0f / sqrtf((float)d);
    const int wblocks = (R * L * 32 + 255) / 256;
    const FrozenRows all_rows{nullptr, 0, 1};           // masked by gs = 0 instead
    normalize_rows_kernel<<<wblocks, 256, 0, st>>>(R * L, d, s_t, khat, rnorm, nullptr, all_rows);
    CKL();
    GemmF32 q{};
    // sim = scale * Q Khat^T                              (n x n per (b, l))
    q = GemmF32{n, n, d, L, Mat{s_t, ld, 1, sb, sl}, Mat{khat, 1, ld, sb, sl}, MatOut{A, n, 1, nn * L, nn}, 1.f, 0.f, nullptr};
    CK(gemm_f32(q, Z, st, launches));
    attn_softmax_kernel<<<(Z * n * 32 + 255) / 256, 256, 0, st>>>(Z, n, g.attend_self, g.mask_side, g.mask_d2_max, scale, A, nullptr, all_rows);
    CKL();
    // dA = dC V^T
    q = GemmF32{n, n, d, L, Mat{gs, ld, 1, sb, sl}, Mat{s_t, 1, ld, sb, sl}, MatOut{dA, n, 1, nn * L, nn}, 1.f, 0.f, nullptr};
    CK(gemm_f32(q, Z, st, launches));
    // dV: ds += A^T dC
    q = GemmF32{n, d, n, L, Mat{A, 1, n, nn * L, nn}, Mat{gs, ld, 1, sb, sl}, MatOut{ds, ld, 1, sb, sl}, 1.f, 1.f, nullptr};
    CK(gemm_f32(q, Z, st, launches));
    attn_softmax_bwd_kernel<<<(Z * n * 32 + 255) / 256, 256, 0, st>>>(Z, n, g.attend_self, g.mask_side, g.mask_d2_max, A, dA, 1.f, nullptr, all_rows);
    CKL();
    // dQ: ds += scale * dsim Khat
    q = GemmF32{n, d, n, L, Mat{dA, n, 1, nn * L, nn}, Mat{khat, ld, 1, sb, sl}, MatOut{ds, ld, 1, sb, sl}, scale, 1.f, nullptr};
    CK(gemm_f32(q, Z, st, launches));
    // dKhat = scale * dsim^T Q
    q = GemmF32{n, d, n, L, Mat{dA, 1, n, nn * L, nn}, Mat{s_t, ld, 1, sb, sl}, MatOut{dkhat, ld, 1, sb, sl}, scale, 0.f, nullptr};
    CK(gemm_f32(q, Z, st, launches));
    normalize_bwd_kernel<<<wblocks, 256, 0, st>>>(R * L, d, khat, dkhat, rnorm, ds, all_rows);
    CKL();
  }
  return cudaSuccess;
}

// =====================================================================================
// helpers of the tensor-core MLP backward
// =====================================================================================
// bf16 packs of the current weights: W1p (G*4d, d), W2T (G*4d, d) = W2^T, W1T (G*d, 4d) = W1^T, b1p (G*4d); groups
// interleaved bu_0, td_0, bu_1, ...
__global__ void pack_bwd_weights_kernel(int d, int L, const float* __restrict__ bu_w1, const float* __restrict__ bu_b1,
                                        const float* __restrict__ bu_w2, const float* __restrict__ td_w1,
                                        const float* __restrict__ td_b1, const float* __restrict__ td_w2,
                                        __nv_bfloat16* __restrict__ w1p, __nv_bfloat16* __restrict__ w2t,
                                        __nv_bfloat16* __restrict__ w1t, float* __restrict__ b1p) {
  const int G = 2 * L - 1, h = 4 * d;
  const size_t nw = (size_t)G * h * d;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nw + (size_t)G * h; i += (size_t)gridDim.x * blockDim.x) {
    if (i < nw) {
      const int g = (int)(i / ((size_t)h * d)), l = g >> 1;
      const size_t q = i % ((size_t)h * d);
      const int j = (int)(q / d), c = (int)(q % d);                 // element (j, c) of W1_g (4d x d)
      const float* W1 = ((g & 1) ? td_w1 : bu_w1) + (size_t)l * h * d;
      const float* W2 = ((g & 1) ? td_w2 : bu_w2) + (size_t)l * d * h;
      const float v1 = W1[(size_t)j * d + c];
      w1p[i] = __float2bfloat16_rn(v1);                             // (g*4d + j, c)
      w1t[((size_t)g * d + c) * h + j] = __float2bfloat16_rn(v1);   // (g*d + c, j)
      w2t[i] = __float2bfloat16_rn(W2[(size_t)c * h + j]);          // (g*4d + j, o = c)  <- W2[o][j]
    } else {
      const size_t q = i - nw;
      const int g = (int)(q / h), l = g >> 1, j = (int)(q % h);
      b1p[q] = ((g & 1) ? td_b1 : bu_b1)[(size_t)l * h + j];
    }
  }
}
// bf16 shadows of a step: sb = bf16(S_t), sp = bf16(S_t[:, 1:] + pos), gsb = bf16(gs)
// kept (nullable): the rows of images with kept[b] <= t are not rewritten.  Such an image was frozen at step t + 1 too,
// so its gsb rows already hold the exact zeros the MLP GEMMs of partially frozen blocks need, and its sb / sp rows hold
// finite values those GEMMs only multiply by zero (with return_all states they are the same bits: S_t == S_{t+1})
__global__ void bwd_shadows_kernel(int rows, int n, int L, int d, const float* __restrict__ s, const float* __restrict__ gs,
                                   const float* __restrict__ pos, __nv_bfloat16* __restrict__ sb,
                                   __nv_bfloat16* __restrict__ sp, __nv_bfloat16* __restrict__ gsb,
                                   const int32_t* __restrict__ kept, int t) {
  const size_t total4 = (size_t)rows * L * d / 4;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (size_t)gridDim.x * blockDim.x) {
    const size_t e = i * 4;
    const int c = (int)(e % d), l = (int)((e / d) % L);
    const size_t r = e / ((size_t)L * d);
    if (kept && __ldg(kept + r / n) <= t) continue;
    const float4 v = *reinterpret_cast<const float4*>(s + e);
    const float4 gv = *reinterpret_cast<const float4*>(gs + e);
    *reinterpret_cast<uint2*>(sb + e) = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
    *reinterpret_cast<uint2*>(gsb + e) = make_uint2(pack_bf16x2(gv.x, gv.y), pack_bf16x2(gv.z, gv.w));
    if (l >= 1) {
      const float4 q = *reinterpret_cast<const float4*>(pos + (size_t)(r % n) * d + c);
      *reinterpret_cast<uint2*>(sp + (r * (L - 1) + (l - 1)) * d + c) =
          make_uint2(pack_bf16x2(v.x + q.x, v.y + q.y), pack_bf16x2(v.z + q.z, v.w + q.w));
    }
  }
}

int backward_run(const Geometry& g, const BackwardArgs& a, int precision, int iters, int grad_all, const int32_t* steps,
                 void* workspace, EncodeTiledFn enc, int num_sms, cudaStream_t st, int* launches, char* err, size_t errlen) {
#define CKI(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { snprintf(err, errlen, "backward: %s", cudaGetErrorString(e_)); return -3; } } while (0)
#define CKLI() do { if (launches) ++*launches; CKI(cudaGetLastError()); } while (0)
  const BackwardLayout wl = backward_layout(g, precision);
  const bool tc = precision == 1 && g.d % 256 == 0;
  const bool attn_tc = tc && g.n % 8 == 0;      // TMA row pitch of the (Z, n, n) bf16 buffers must be a multiple of 16 B
  char* ws = static_cast<char*>(workspace);
  const size_t state = (size_t)g.rows * g.L * g.d;
  // gradient w.r.t. the state walks backwards through two ping-pong slabs: step t reads (gin + gextra) and writes ds
  float* slab[2] = {reinterpret_cast<float*>(ws + wl.ds_off), reinterpret_cast<float*>(ws + wl.g_off)};
  float* gs = reinterpret_cast<float*>(ws + wl.gs_off);
  MlpBwdTc m{};
  if (tc) {
    __nv_bfloat16* xb = reinterpret_cast<__nv_bfloat16*>(ws + wl.xb_off);
    m.xb = xb;
    m.sb = reinterpret_cast<__nv_bfloat16*>(ws + wl.sb_off);
    m.sp = reinterpret_cast<__nv_bfloat16*>(ws + wl.sp_off);
    m.gsb = reinterpret_cast<__nv_bfloat16*>(ws + wl.gsb_off);
    m.w1p = reinterpret_cast<__nv_bfloat16*>(ws + wl.w1p_off);
    m.w2t = reinterpret_cast<__nv_bfloat16*>(ws + wl.w2t_off);
    m.w1t = reinterpret_cast<__nv_bfloat16*>(ws + wl.w1t_off);
    m.b1p = reinterpret_cast<float*>(ws + wl.b1p_off);
    m.pre = reinterpret_cast<__nv_bfloat16*>(ws + wl.bpre_off);
    m.h = reinterpret_cast<__nv_bfloat16*>(ws + wl.bh_off);
    m.dpre = reinterpret_cast<__nv_bfloat16*>(ws + wl.bdpre_off);
    m.d_tokens = a.d_tokens; m.d_pos = a.d_pos;
    m.d_bu_w1 = a.d_bu_w1; m.d_bu_w2 = a.d_bu_w2; m.d_td_w1 = a.d_td_w1; m.d_td_w2 = a.d_td_w2;
    m.d_bu_b1 = a.d_bu_b1; m.d_td_b1 = a.d_td_b1;
    m.deterministic = a.deterministic;
    m.dx_td = reinterpret_cast<float*>(ws + wl.dkhat_off);
    m.b1_part = reinterpret_cast<float*>(ws + wl.b1part_off);
    pack_bwd_weights_kernel<<<sm_count() * 8, 256, 0, st>>>(g.d, g.L, a.bu_w1, a.bu_b1, a.bu_w2, a.td_w1, a.td_b1, a.td_w2,
                                                     const_cast<__nv_bfloat16*>(m.w1p), const_cast<__nv_bfloat16*>(m.w2t),
                                                     const_cast<__nv_bfloat16*>(m.w1t), const_cast<float*>(m.b1p));
    CKLI();
    const size_t n4 = (size_t)g.rows * g.d / 4;
    cast_bf16_rows<<<nblk(n4), 256, 0, st>>>(n4, a.tokens, xb);
    CKLI();
    if (g.rows % 128) {     // rows of the last 128-row block beyond R are read as K entries of the dW GEMMs: keep them zero
      CKI(cudaMemsetAsync(m.h, 0, wl.blocked_bytes, st));
      CKI(cudaMemsetAsync(m.dpre, 0, wl.blocked_bytes, st));
    }
  }
  // pending upstream gradient of S_{t+1}: gin (+ gextra, the cotangent of that step's own output under return_all)
  const float* gin = grad_all ? a.grad_out + (size_t)iters * state : a.grad_out;
  const float* gextra = nullptr;
  for (int t = iters - 1, k = 0; t >= 0; --t, ++k) {
    const float* s_t = a.states + (size_t)t * state;
    float* ds = slab[k & 1];
    // an image frozen at step t (steps[b] <= t) below the first reverse step was frozen at step t + 1 as well: its rows
    // of gs and of the bf16 shadows still hold what step t + 1 wrote (zeros in gs / gsb), so they are not rewritten.  A
    // reverse step at which every image is frozen (t >= max(steps), the tail of a settle_all backward) then only passes
    // ds = gin + gextra through; its other launches find no work.
    const int32_t* kept = (steps && t < iters - 1) ? steps : nullptr;
    CKI(backward_step(g, a, s_t, gin, gextra, ds, ws, wl, tc, attn_tc, steps, t, kept != nullptr, st,
                      launches));   // scale (+ the fp32 MLP / attention backward)
    if (tc) {
      bwd_shadows_kernel<<<nblk(state / 4), 256, 0, st>>>(g.rows, g.n, g.L, g.d, s_t, gs, a.pos,
                                                          const_cast<__nv_bfloat16*>(m.sb), const_cast<__nv_bfloat16*>(m.sp),
                                                          const_cast<__nv_bfloat16*>(m.gsb), kept, t);
      CKLI();
      // ---- consensus attention backward: the five (n x n x d) GEMM families on tensor cores, softmax in fp32.  With
      // per-image step counts, the problems / rows of images frozen at step t are skipped in every launch (their
      // contribution to ds is an exact zero); the buffers they would have written are left stale and read by no one.
      if (attn_tc) {
        float* khat = reinterpret_cast<float*>(ws + wl.khat_off);
        float* dkhat = reinterpret_cast<float*>(ws + wl.dkhat_off);
        float* rnorm = reinterpret_cast<float*>(ws + wl.rnorm_off);
        float* A = reinterpret_cast<float*>(ws + wl.attn_off);
        float* dA = reinterpret_cast<float*>(ws + wl.dattn_off);
        __nv_bfloat16* khat_b = reinterpret_cast<__nv_bfloat16*>(ws + wl.khatb_off);
        __nv_bfloat16* a_b = reinterpret_cast<__nv_bfloat16*>(ws + wl.ab_off);
        __nv_bfloat16* dsim_b = reinterpret_cast<__nv_bfloat16*>(ws + wl.dsimb_off);
        const int Z = g.B * g.L, n = g.n, d = g.d;
        const float scale = 1.0f / sqrtf((float)d);
        const int wblocks = (g.rows * g.L * 32 + 255) / 256, rblocks = (Z * n * 32 + 255) / 256;
        const FrozenRows frozen{steps, t, n * g.L};
        normalize_rows_kernel<<<wblocks, 256, 0, st>>>(g.rows * g.L, d, s_t, khat, rnorm, khat_b, frozen);
        CKLI();
        // logits = Q Khat^T (scaled inside the softmax), dA = dC V^T
        if (int r = attn_bwd_gemm_tc(g, m.sb, 1, 0, khat_b, 1, 0, n, d, 0, A, steps, t, enc, num_sms, st, launches, err,
                                     errlen)) return r;
        attn_softmax_kernel<<<rblocks, 256, 0, st>>>(Z, n, g.attend_self, g.mask_side, g.mask_d2_max, scale, A, a_b, frozen);
        CKLI();
        if (int r = attn_bwd_gemm_tc(g, m.gsb, 1, 0, m.sb, 1, 0, n, d, 0, dA, steps, t, enc, num_sms, st, launches, err,
                                     errlen)) return r;
        attn_softmax_bwd_kernel<<<rblocks, 256, 0, st>>>(Z, n, g.attend_self, g.mask_side, g.mask_d2_max, A, dA, scale, dsim_b,
                                                         frozen);
        CKLI();
        // dV and dQ in one K-concatenated product: ds += [A^T | scale dsim] [dC ; Khat] ;  dKhat = (scale dsim)^T Q
        if (int r = attn_bwd_gemm_tc(g, a_b, 0, 1, m.gsb, 1, 1, d, n, 1, ds, steps, t, enc, num_sms, st, launches, err, errlen,
                                     dsim_b, 0, 0, khat_b, 1, 1)) return r;
        if (int r = attn_bwd_gemm_tc(g, dsim_b, 0, 1, m.sb, 1, 1, d, n, 2, dkhat, steps, t, enc, num_sms, st, launches, err,
                                     errlen)) return r;
        normalize_bwd_kernel<<<wblocks, 256, 0, st>>>(g.rows * g.L, d, khat, dkhat, rnorm, ds, frozen);
        CKLI();
      }
      m.ds = ds;
      m.steps = steps; m.t = t;
      if (int r = mlp_backward_tc(g, m, enc, num_sms, st, launches, err, errlen)) return r;
      if (a.deterministic) {     // what the default DH / DX epilogues reduce with atomics, in a fixed order
        bias_partials_kernel<<<(g.G * g.d + 31) / 32, dim3(32, 16), 0, st>>>(g.G, (g.rows + 31) / 32, g.rows, g.n, g.d,
                                                                             m.b1_part, a.d_bu_b1, a.d_td_b1, steps, t);
        CKLI();
        dx_td_reduce_kernel<<<g.n * ((g.d / 4 + 31) / 32), dim3(32, 8), 0, st>>>(g.B, g.n, g.L, g.d, m.dx_td, ds, a.d_pos,
                                                                                  steps, t);
        CKLI();
      }
      CKI(colsum(a.deterministic != 0, g.rows, g.L * g.d, (long long)g.L * g.d, gs, a.d_bu_b2, a.d_td_b2, (g.L - 1) * g.d,
                 steps, t, g.n, st, launches));
    }
    gin = ds;
    gextra = grad_all ? a.grad_out + (size_t)t * state : nullptr;
  }
  // gradient w.r.t. S_0 = gin + gextra
  for (const float* part : {gin, gextra}) {
    if (!part) continue;
    if (a.d_state0) {
      add_kernel<<<nblk(state), 256, 0, st>>>(state, part, a.d_state0);
      CKLI();
    }
    if (a.d_init && a.deterministic) {
      CKI(colsum(true, g.rows, g.L * g.d, (long long)g.L * g.d, part, a.d_init, nullptr, 0, nullptr, 0, 1, st, launches));
    } else if (a.d_init) {
      init_grad_kernel<<<dim3((g.L * g.d + 255) / 256, 64), 256, 0, st>>>(g.rows, g.L, g.d, part, a.d_init);
      CKLI();
    }
  }
  return 0;
#undef CKI
#undef CKLI
}

}  // namespace glom
