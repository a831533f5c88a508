// Glom.settle on CUDA cores: the per-image stopping rule applied after every step, and the final gather of the images
// whose last state sits in the workspace's half of the ping-pong.  Also the per-image step counts of
// glom_b200_forward_steps: the flags of each step from the given counts, and the return_all fill of stopped images' slabs.
// And the slot kernels of Glom.settle_queue and Glom.settle_video: queue initialisation, the slot schedule and the slot
// fill of every step.
#include "engine.h"
#include "prep_state.cuh"
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
// Settle queue (q.slot_img != NULL): b is a slot.  Each running slot's age goes up by one, the slot also stops when its
// age reaches q.max_iters, steps[q.slot_img[b]] = age, and a stopping slot is marked pending (its final state is
// handed over by the next fill) and leaves the unfinished count.
__global__ void __launch_bounds__(SETTLE_THREADS)
settle_converge_kernel(int n, int L, int nparts, int B, int rows, int step, float tol, const float* __restrict__ dsq,
                       const float* __restrict__ nsq, int* frozen, int* block_frozen, unsigned int* done, float* level_q,
                       int32_t* steps, QueueSlots q) {
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
    if (q.slot_img) {
      const int age = ++q.age[bb];
      stop = stop || age >= q.max_iters;
      steps[q.slot_img[bb]] = age;
      if (stop) { q.pending[bb] = 1; atomicSub(q.unfinished, 1); }
    } else {
      steps[bb] = step;
    }
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

// a block of SETTLE_THREADS threads per grid point, launched with programmatic stream serialisation
template <typename... Params, typename... Args>
static cudaError_t launch_pdl(void (*kernel)(Params...), dim3 grid, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = dim3(SETTLE_THREADS);
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;      // PDL: see pdl_wait() in the kernels
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, args...);
}

int launch_settle_converge(const Geometry& g, int step, float tol, const float* dsq, const float* nsq, int* frozen,
                           int* block_frozen, unsigned int* done, float* level_q, int32_t* steps, Launch& ln,
                           const QueueSlots* q) {
  return ln.launched(launch_pdl(settle_converge_kernel, dim3(g.L, g.B), ln.st, g.n, g.L, g.nparts, g.B, g.rows, step, tol, dsq,
                                nsq, frozen, block_frozen, done, level_q, steps, q ? *q : QueueSlots{}));
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

int launch_settle_gather(const Geometry& g, int max_iters, const int32_t* steps, const float* slab, float* state_out,
                         const float* s0, int s0_bcast, Launch& ln) {
  const size_t per_img4 = (size_t)g.n * g.L * g.d / 4;
  settle_gather_kernel<<<dim3(copy_chunks(g, per_img4), g.B), 256, 0, ln.st>>>(
      max_iters, steps, per_img4, reinterpret_cast<const float4*>(slab), reinterpret_cast<float4*>(state_out),
      reinterpret_cast<const float4*>(s0), s0_bcast, (unsigned)(g.L * g.d / 4));
  return ln.launched();
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

int launch_steps_schedule(const Geometry& g, int t, int max_steps, const int32_t* steps, int* frozen, int* block_frozen,
                          Launch& ln) {
  const int items = g.B + (g.rows + 255) / 256;
  return ln.launched(launch_pdl(steps_schedule_kernel, dim3((items + SETTLE_THREADS - 1) / SETTLE_THREADS), ln.st, g.n, g.B,
                                g.rows, t, max_steps, steps, frozen, block_frozen));
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

int launch_steps_fill(const Geometry& g, int max_steps, const int32_t* steps, float* states, Launch& ln) {
  const size_t per_img4 = (size_t)g.n * g.L * g.d / 4;
  steps_fill_kernel<<<dim3(copy_chunks(g, per_img4), g.B), 256, 0, ln.st>>>(max_steps, steps, per_img4, per_img4 * g.B,
                                                                            reinterpret_cast<float4*>(states));
  return ln.launched();
}

// Grid (chunks, B - 1): slab s of a return_all forward from init_levels holds levels l >= s for image 0 only (steps
// 0 .. L-2 ran them for the representative rows, see step_bf16); image b >= 1 receives image 0's rows of those levels.
__global__ void level_fill_kernel(int L, int d4, size_t per_img4, size_t slab4, float4* __restrict__ states) {
  const size_t o = (size_t)(blockIdx.y + 1) * per_img4;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < per_img4; i += (size_t)gridDim.x * blockDim.x) {
    const int l = (int)(i / d4 % L);
    for (int s = 1; s <= l; ++s) states[(size_t)s * slab4 + o + i] = states[(size_t)s * slab4 + i];
  }
}

int launch_level_fill(const Geometry& g, float* states, Launch& ln) {
  const size_t per_img4 = (size_t)g.n * g.L * g.d / 4;
  level_fill_kernel<<<dim3(copy_chunks(g, per_img4), g.B - 1), 256, 0, ln.st>>>(g.L, g.d / 4, per_img4, per_img4 * g.B,
                                                                               reinterpret_cast<float4*>(states));
  return ln.launched();
}

// ---- Glom.settle_queue: N images through B slots.  Slot s holds image slot_img[s]; its rows are rows s*n .. s*n+n-1
// of every step buffer, exactly as image s's rows in a settle call of batch B.  S_t of the slots lives in the private
// slab t & 1, the shadows and norm partials in buffer t & 1, as in settle.  A slot whose image stops after step t-1 hands
// that image's final state (slab t & 1) to state_out in the fill of step t, which then writes the next image's S_0 over
// it; K1 recomputes group 0 for the blocks that admitted an image (block_fresh), K3 and K2 skip frozen slots as in settle.
// Glom.settle_video runs the same kernels with q.frames = F > 1: the images are the frames i = stream * F + f, a slot
// whose frame f < F - 1 stops takes frame f + 1 of its own stream, and that frame's S_0 is the slot's own S_k (the
// settle_queue call is the case F = 1, where no slot continues).

// One block: every slot empty (frozen, no image), every image queued.
__global__ void __launch_bounds__(SETTLE_THREADS)
queue_init_kernel(int B, int nblk, QueueSlots q, int* frozen, int* block_frozen, unsigned int* done) {
  pdl_launch_dependents();
  pdl_wait();                                       // the previous call's kernels have stopped reading the workspace
  for (int s = threadIdx.x; s < B; s += SETTLE_THREADS) {
    q.slot_img[s] = -1; q.age[s] = 0; q.pending[s] = 0; q.gather_img[s] = -1; q.fresh[s] = 0;
    frozen[s] = 1;
  }
  for (int m = threadIdx.x; m < nblk; m += SETTLE_THREADS) { block_frozen[m] = 1; q.block_fresh[m] = 0; }
  if (threadIdx.x == 0) { *q.head = 0; *q.unfinished = q.images; *done = 0u; }
}

int launch_queue_init(const Geometry& g, const QueueSlots& q, int* frozen, int* block_frozen, unsigned int* done, Launch& ln) {
  ProfScope scope(ln.prof, PROF_PREP, ln.st);
  return ln.launched(launch_pdl(queue_init_kernel, dim3(1), ln.st, g.B, (g.rows + 255) / 256, q, frozen, block_frozen, done));
}

// One block, before a step.  The open slots (frozen: their image stopped, or empty) hand a pending image over to the fill
// (gather_img).  With `admit`, an open slot whose frame f < F - 1 stopped takes frame f + 1 of the same stream; the other
// open slots are ranked in slot order by a block-wide count, and number k takes frame 0 of queued stream head + k while
// there is one, so the assignment does not depend on timing.  Then the per-256-row-block flags: block_frozen = every slot
// of the block is frozen, block_fresh = one of them took a frame.
__global__ void __launch_bounds__(SETTLE_THREADS)
queue_schedule_kernel(int n, int B, int rows, int admit, QueueSlots q, int* frozen, int* block_frozen) {
  pdl_launch_dependents();
  pdl_wait();                                       // the previous step's convergence launch has set the flags
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int streams = q.images / q.frames;
  __shared__ int wsum[SETTLE_THREADS / 32];
  int head = *q.head;
  for (int base = 0; base < B; base += SETTLE_THREADS) {
    const int s = base + tid;
    const bool open = s < B && frozen[s];
    const int gi = open && q.pending[s] ? q.slot_img[s] : -1;
    const bool next = admit && gi >= 0 && gi % q.frames != q.frames - 1;
    const unsigned m = __ballot_sync(0xffffffffu, open && !next);
    if (lane == 0) wsum[warp] = __popc(m);
    __syncthreads();
    int before = 0, total = 0;
    for (int w = 0; w < SETTLE_THREADS / 32; ++w) { before += w < warp ? wsum[w] : 0; total += wsum[w]; }
    if (open) {
      q.gather_img[s] = gi;
      q.pending[s] = 0;
      const int stream = head + before + __popc(m & ((1u << lane) - 1u));
      const bool take = next || (admit && stream < streams);
      q.slot_img[s] = next ? gi + 1 : take ? stream * q.frames : -1;
      q.fresh[s] = take;
      if (take) { q.age[s] = 0; frozen[s] = 0; }
    } else if (s < B) {
      q.gather_img[s] = -1;
      q.fresh[s] = 0;
    }
    if (admit) head = min(head + total, streams);
    __syncthreads();                                // wsum is reused
  }
  if (tid == 0) *q.head = head;
  const int nblk = (rows + 255) / 256;
  for (int m = tid; m < nblk; m += SETTLE_THREADS) {
    const int b0 = m * 256 / n, b1 = (min(rows, m * 256 + 256) - 1) / n;
    int all = 1, any = 0;
    for (int bb = b0; bb <= b1; ++bb) { all = all && frozen[bb]; any = any || q.fresh[bb]; }
    block_frozen[m] = all;
    q.block_fresh[m] = any;
  }
}

int launch_queue_schedule(const Geometry& g, const QueueSlots& q, int admit, int* frozen, int* block_frozen, Launch& ln) {
  ProfScope scope(ln.prof, PROF_PREP, ln.st);
  return ln.launched(launch_pdl(queue_schedule_kernel, dim3(1), ln.st, g.n, g.B, g.rows, admit, q, frozen, block_frozen));
}

constexpr int FILL_ROWS = 8;                        // rows of one slot per block of the fill

// Grid (ceil(n / FILL_ROWS), B), after the schedule.  Block (c, s) covers rows c*FILL_ROWS.. of slot s: first the copy
// of the handed-over image's final state from the slab into state_out, then (admitted slot) the admitted image's S_0
// into the same slab rows with prep_state_row, one warp per (row, level), and its token rows cast to bf16.  Frame 0 of a
// stream starts from state_in[stream] or init_levels.  A later frame's S_0 is the previous frame's final state, already
// in the slab rows: prep_state_row recomputes the shadows and norm partials from it in place, as the prologue of a
// settle call given that state as `levels` does.
__global__ void __launch_bounds__(SETTLE_THREADS)
queue_fill_kernel(int n, int L, int d, int nparts, int part_w, QueueSlots q, const float* __restrict__ tokens,
                  const float* __restrict__ pos, const float* __restrict__ state_in, const float* __restrict__ init_levels,
                  float* __restrict__ state_out, float* slab, __nv_bfloat16* __restrict__ sb, __nv_bfloat16* __restrict__ sp,
                  float* __restrict__ nsq, __nv_bfloat16* __restrict__ xb) {
  pdl_launch_dependents();
  pdl_wait();                                       // the schedule is written, the previous step's K2 has stored S_t
  const int s = blockIdx.y, i0 = blockIdx.x * FILL_ROWS, ni = min(FILL_ROWS, n - i0);
  const int gi = q.gather_img[s], fresh = q.fresh[s];
  const size_t ld = (size_t)L * d, r0 = (size_t)s * n + i0;
  if (gi >= 0) {
    const float4* src = reinterpret_cast<const float4*>(slab + r0 * ld);
    float4* dst = reinterpret_cast<float4*>(state_out + ((size_t)gi * n + i0) * ld);
    for (size_t k = threadIdx.x; k < (size_t)ni * ld / 4; k += SETTLE_THREADS) dst[k] = src[k];
  }
  if (!fresh) return;                               // block-uniform
  __syncthreads();                                  // the handed-over state is read before S_0 replaces it
  const int img = q.slot_img[s], stream = img / q.frames, cont = img % q.frames != 0;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int w = warp; w < ni * L; w += SETTLE_THREADS / 32) {
    const int i = i0 + w / L, l = w % L;
    const size_t r = (size_t)s * n + i;
    float* row = slab + (r * L + l) * d;
    const float* src = cont ? row : state_in ? state_in + (((size_t)stream * n + i) * L + l) * d : init_levels + (size_t)l * d;
    prep_state_row(lane, l, d, nparts, part_w, src, pos + (size_t)i * d, cont ? nullptr : row, sb + (r * L + l) * d,
                   l >= 1 ? sp + (r * (L - 1) + (l - 1)) * d : nullptr, nsq + (r * L + l) * nparts);
  }
  const float4* tk = reinterpret_cast<const float4*>(tokens + ((size_t)img * n + i0) * d);
  uint2* xo = reinterpret_cast<uint2*>(xb + r0 * d);
  for (int k = threadIdx.x; k < ni * d / 4; k += SETTLE_THREADS) xo[k] = cast4_bf16(tk[k]);
}

int launch_queue_fill(const Geometry& g, const QueueSlots& q, const float* tokens, const float* pos, const float* state_in,
                      const float* init_levels, float* state_out, float* slab, __nv_bfloat16* sb, __nv_bfloat16* sp,
                      float* nsq, __nv_bfloat16* xb, Launch& ln) {
  ProfScope scope(ln.prof, PROF_PREP, ln.st);
  return ln.launched(launch_pdl(queue_fill_kernel, dim3((g.n + FILL_ROWS - 1) / FILL_ROWS, g.B), ln.st, g.n, g.L, g.d, g.nparts,
                                g.part_w, q, tokens, pos, state_in, init_levels, state_out, slab, sb, sp, nsq, xb));
}

}  // namespace glom
