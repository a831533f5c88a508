// C ABI of libglom_b200.so (see include/glom_b200.h).  Host logic only: argument checking,
// buffer layout, the per-step launch sequence.  No device allocation, no stream sync.
#include "../../include/glom_b200.h"
#include "../../include/glom_b200_track.h"
#include "../../include/glom_b200_tree.h"
#include "engine.h"

#include <mutex>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

namespace glom {

static thread_local char g_err[512] = "";
static thread_local Profiler g_prof;
// the launch context of this thread's last launching entry point; glom_b200_last_launch_count reports its count
static thread_local Launch g_launch{};

static int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

static bool misaligned(const void* p, size_t a) { return reinterpret_cast<uintptr_t>(p) % a != 0; }

PackedLayout packed_layout(int d, int L, int precision) {
  const size_t es = precision == GLOM_B200_BF16 ? 2 : 4;
  const size_t G = 2 * (size_t)L - 1;
  PackedLayout p;
  size_t off = 0;
  p.w1_off = off; off = align_up(off + G * 4 * d * d * es, 1024);
  p.w2_off = off; off = align_up(off + (size_t)L * d * 8 * d * es, 1024);
  p.b1_off = off; off = align_up(off + G * 4 * d * 4, 1024);
  p.b2_off = off; off = align_up(off + (size_t)L * d * 4, 1024);
  p.total = off;
  return p;
}

WorkspaceLayout workspace_layout(const Geometry& g, int precision, int iters, int return_all) {
  WorkspaceLayout w{};
  const size_t state_elems = (size_t)g.rows * g.L * g.d;
  size_t off = 0;
  w.s32_off = off;
  w.s32_bytes = (return_all || iters == 0) ? 0 : state_elems * 4;
  off = align_up(off + w.s32_bytes, 1024);
  if (precision == GLOM_B200_BF16) {
    for (int i = 0; i < 2; ++i) { w.sb_off[i] = off; off = align_up(off + state_elems * 2, 1024); }
    for (int i = 0; i < 2; ++i) { w.sp_off[i] = off; off = align_up(off + (size_t)g.rows * (g.L - 1) * g.d * 2, 1024); }
    w.xb_off = off; off = align_up(off + (size_t)g.rows * g.d * 2, 1024);
    w.h_bytes = (size_t)((g.rows + 127) / 128 * 128) * g.G * 4 * g.d * 2;   // 128-row blocks, padded
    w.c_bytes = state_elems * 2;
    w.nsq_bytes = (size_t)g.rows * g.L * g.nparts * 4;
  } else {
    w.h_bytes = (size_t)g.rows * g.G * 4 * g.d * 4;
    w.c_bytes = state_elems * 4;
    w.nsq_bytes = 0;
  }
  w.h_off = off; off = align_up(off + w.h_bytes, 1024);
  w.c_off = off; off = align_up(off + w.c_bytes, 1024);
  for (int i = 0; i < 2; ++i) { w.nsq_off[i] = off; off = align_up(off + w.nsq_bytes, 1024); }
  w.attn_acc_off = off;
  w.attn_acc_bytes = (precision == GLOM_B200_BF16 && g.n > 576) ? (state_elems + (size_t)g.rows * g.L * 2) * 4 : 0;
  off = align_up(off + w.attn_acc_bytes, 1024);
  w.total = off > 0 ? off : 1024;
  return w;
}

SettleLayout settle_layout(const Geometry& g, int max_iters, int return_all) {
  SettleLayout s{};
  s.fwd = workspace_layout(g, GLOM_B200_BF16, max_iters, return_all);
  size_t off = s.fwd.total;
  s.dsq_off = off; off = align_up(off + s.fwd.nsq_bytes, 1024);
  s.flags_off = off;                  // each flag buffer 16-byte aligned: glom_b200_settle_workspace_offset hands them out
  s.frozen_off = off; off = align_up(off + (size_t)g.B * 4, 16);
  s.block_frozen_off = off; off = align_up(off + (size_t)(g.rows + 255) / 256 * 4, 16);
  s.done_off = off; off = align_up(off + 4, 16);
  s.level_q_off = off; off += (size_t)g.B * g.L * 4;
  s.flags_bytes = off - s.flags_off;
  s.total = align_up(off, 1024);
  return s;
}

QueueLayout queue_layout(const Geometry& g, int max_iters) {
  QueueLayout q{};
  q.settle = settle_layout(g, max_iters, 0);
  size_t off = q.settle.total;
  q.slab_off[0] = q.settle.fwd.s32_off;
  q.slab_off[1] = off; off = align_up(off + q.settle.fwd.s32_bytes, 1024);
  const size_t slots = align_up((size_t)g.B * 4, 16), blocks = align_up((size_t)(g.rows + 255) / 256 * 4, 16);
  q.queue_off = off;
  q.slot_img_off = off; off += slots;
  q.age_off = off; off += slots;
  q.pending_off = off; off += slots;
  q.gather_off = off; off += slots;
  q.fresh_off = off; off += slots;
  q.block_fresh_off = off; off += blocks;
  q.head_off = off; off += 16;
  q.unfinished_off = off; off += 16;
  q.queue_bytes = off - q.queue_off;
  q.total = align_up(off, 1024);
  return q;
}

static int check_cfg(const glom_b200_cfg* cfg) {
  if (!cfg) return fail(GLOM_B200_ERR_INVALID, "cfg is NULL");
  if (cfg->struct_size != sizeof(glom_b200_cfg))
    return fail(GLOM_B200_ERR_INVALID, "cfg.struct_size %u != %zu (ABI mismatch)", cfg->struct_size, sizeof(glom_b200_cfg));
  if (cfg->levels < 2) return fail(GLOM_B200_ERR_INVALID, "levels must be >= 2 (got %d)", cfg->levels);
  if (cfg->dim < 4 || cfg->dim % 4) return fail(GLOM_B200_ERR_INVALID, "dim must be a positive multiple of 4 (got %d)", cfg->dim);
  if (cfg->n < 1) return fail(GLOM_B200_ERR_INVALID, "n must be >= 1 (got %d)", cfg->n);
  if (cfg->precision != GLOM_B200_FP32 && cfg->precision != GLOM_B200_BF16)
    return fail(GLOM_B200_ERR_INVALID, "unknown precision %d", cfg->precision);
  if (cfg->precision == GLOM_B200_BF16 && cfg->dim % 64)
    return fail(GLOM_B200_ERR_INVALID, "bf16 (tensor-core) precision needs dim %% 64 == 0 (got %d); use fp32 precision", cfg->dim);
  if (cfg->mask_side < 0 || (cfg->mask_side > 0 && cfg->n % cfg->mask_side))
    return fail(GLOM_B200_ERR_INVALID, "mask_side %d does not tile n = %d", cfg->mask_side, cfg->n);
  return 0;
}

static Geometry make_geometry(const glom_b200_cfg* cfg, int batch) {
  Geometry g{};
  g.d = cfg->dim; g.L = cfg->levels; g.n = cfg->n; g.B = batch;
  g.rows = batch * cfg->n;
  g.G = 2 * g.L - 1;
  g.hidden = 4 * g.d;
  g.attend_self = cfg->attend_self; g.mask_side = cfg->mask_side; g.mask_d2_max = cfg->mask_d2_max;
  g.bn2 = (g.d % 256 == 0) ? 256 : (g.d % 128 == 0) ? 128 : 64;
  g.part_w = (g.bn2 == 256) ? 64 : g.bn2 / 2;   // columns per GEMM2 epilogue warp group (GemmCfg<1, BN>::PART_COLS)
  g.nparts = g.d / g.part_w;
  return g;
}

struct DeviceInfo { bool ok; int sms; };
static std::mutex g_mu;
static DeviceInfo g_dev[64];
static bool g_dev_known[64];
static EncodeTiledFn g_encode = nullptr;

static int device_info(DeviceInfo* out) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return fail(GLOM_B200_ERR_CUDA, "cudaGetDevice: %s", cudaGetErrorString(e));
  if (dev < 0 || dev >= 64) return fail(GLOM_B200_ERR_CUDA, "device ordinal %d out of range", dev);
  std::lock_guard<std::mutex> lk(g_mu);
  if (!g_dev_known[dev]) {
    int major = 0, sms = 0;
    e = cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) return fail(GLOM_B200_ERR_CUDA, "cudaDeviceGetAttribute: %s", cudaGetErrorString(e));
    g_dev[dev].ok = (major == 9);
    g_dev[dev].sms = sms;
    g_dev_known[dev] = true;
  }
  if (!g_encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qr;
    e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qr);
    if (e != cudaSuccess || qr != cudaDriverEntryPointSuccess || !fn)
      return fail(GLOM_B200_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable (%s)", cudaGetErrorString(e));
    g_encode = reinterpret_cast<EncodeTiledFn>(fn);
  }
  *out = g_dev[dev];
  if (!out->ok) return fail(GLOM_B200_ERR_DEVICE, "device %d is not compute capability 9.x (sm_90a kernels only)", dev);
  out->sms = planned_sms(out->sms);
  return 0;
}

// The launch context of an entry point whose arguments and device have been checked: the thread's count starts at 0 and
// stands at what the call enqueued when it returns, failed or not.  sms: DeviceInfo::sms (0: the call plans no
// tensor-core grid and queried no device)
static Launch& begin_launch(int sms, void* stream) {
  g_launch = Launch{g_encode, sms, static_cast<cudaStream_t>(stream), &g_prof, 0, ""};
  return g_launch;
}

std::atomic<int> g_sm_count_target{0};

}  // namespace glom

using namespace glom;

extern "C" {

GLOM_B200_API int glom_b200_abi_version(void) { return GLOM_B200_ABI_VERSION; }

GLOM_B200_API const char* glom_b200_last_error(void) { return g_err; }

GLOM_B200_API int glom_b200_last_launch_count(void) { return g_launch.launches; }

GLOM_B200_API int glom_b200_set_sm_count_target(int sms) {
  if (sms < 0 || sms == 1)
    return fail(GLOM_B200_ERR_INVALID, "SM-count target must be 0 or >= 2 (got %d): a CTA pair needs two SMs", sms);
  return g_sm_count_target.exchange(sms);
}

GLOM_B200_API int glom_b200_packed_weight_bytes(const glom_b200_cfg* cfg, size_t* out_bytes) {
  if (int r = check_cfg(cfg)) return r;
  if (!out_bytes) return fail(GLOM_B200_ERR_INVALID, "out_bytes is NULL");
  *out_bytes = packed_layout(cfg->dim, cfg->levels, cfg->precision).total;
  return 0;
}

GLOM_B200_API int glom_b200_pack_weights(const glom_b200_cfg* cfg, const glom_b200_weights_ref* w, void* packed, size_t packed_bytes,
                           void* stream) {
  if (int r = check_cfg(cfg)) return r;
  if (!w || w->struct_size != sizeof(glom_b200_weights_ref)) return fail(GLOM_B200_ERR_INVALID, "weights struct missing or wrong size");
  if (!w->bu_w1 || !w->bu_b1 || !w->bu_w2 || !w->bu_b2 || !w->td_w1 || !w->td_b1 || !w->td_w2 || !w->td_b2)
    return fail(GLOM_B200_ERR_INVALID, "a weight pointer is NULL");
  const PackedLayout pl = packed_layout(cfg->dim, cfg->levels, cfg->precision);
  if (!packed || packed_bytes < pl.total) return fail(GLOM_B200_ERR_WORKSPACE, "packed buffer: need %zu bytes, got %zu", pl.total, packed_bytes);
  if (misaligned(packed, 1024)) return fail(GLOM_B200_ERR_INVALID, "packed buffer must be 1024-byte aligned");
  Launch& ln = begin_launch(0, stream);
  if (int r = launch_pack(cfg->dim, cfg->levels, cfg->precision, w->bu_w1, w->bu_b1, w->bu_w2, w->bu_b2, w->td_w1, w->td_b1,
                          w->td_w2, w->td_b2, packed, ln))
    return fail(r, "pack_weights launch: %s", ln.err);
  return 0;
}

GLOM_B200_API int glom_b200_workspace_bytes(const glom_b200_cfg* cfg, int batch, int iters, int return_all, size_t* out_bytes) {
  if (int r = check_cfg(cfg)) return r;
  if (batch < 1 || iters < 0 || !out_bytes) return fail(GLOM_B200_ERR_INVALID, "bad batch/iters/out_bytes");
  *out_bytes = workspace_layout(make_geometry(cfg, batch), cfg->precision, iters, return_all).total;
  return 0;
}

GLOM_B200_API int glom_b200_workspace_offset(const glom_b200_cfg* cfg, int batch, int iters, int return_all, int which,
                               size_t* out_offset, size_t* out_bytes) {
  if (int r = check_cfg(cfg)) return r;
  if (batch < 1 || iters < 0 || !out_offset || !out_bytes) return fail(GLOM_B200_ERR_INVALID, "bad arguments");
  const WorkspaceLayout w = workspace_layout(make_geometry(cfg, batch), cfg->precision, iters, return_all);
  switch (which) {
    case 0: *out_offset = w.h_off; *out_bytes = w.h_bytes; return 0;
    case 1: *out_offset = w.c_off; *out_bytes = w.c_bytes; return 0;
    case 2: *out_offset = w.nsq_off[0]; *out_bytes = w.nsq_bytes; return 0;
    default: return fail(GLOM_B200_ERR_INVALID, "unknown workspace buffer id %d", which);
  }
}

// ---- what the forward, settle and queue calls share ------------------------------------------------------------------

// The tensor arguments of a forward or queue call, checked in this order.  `pre`: "" or "<entry point>: ".  A forward
// passes its packed weights (they are required, and aligned like the workspace); the queue calls check theirs themselves
// (queue_run) or take none (queue_begin): has_packed = false.
static int check_tensors(const char* pre, bool has_packed, const void* packed_weights, const float* tokens, const float* pos,
                         const float* state_in, const float* init_levels, const float* state_out, const void* workspace) {
  if ((has_packed && !packed_weights) || !tokens || !pos || !state_out)
    return fail(GLOM_B200_ERR_INVALID, "%sa required pointer is NULL", pre);
  if (!state_in && !init_levels) return fail(GLOM_B200_ERR_INVALID, "%sneed state_in or init_levels", pre);
  if (state_in == state_out) return fail(GLOM_B200_ERR_INVALID, "%sstate_out must not alias state_in", pre);
  if (has_packed && (misaligned(packed_weights, 1024) || misaligned(workspace, 1024)))
    return fail(GLOM_B200_ERR_INVALID, "%spacked weights and workspace must be 1024-byte aligned", pre);
  if (!has_packed && misaligned(workspace, 1024)) return fail(GLOM_B200_ERR_INVALID, "%sworkspace must be 1024-byte aligned", pre);
  if (misaligned(tokens, 16) || misaligned(pos, 16) || misaligned(state_out, 16) || misaligned(state_in, 16) ||
      misaligned(init_levels, 16))
    return fail(GLOM_B200_ERR_INVALID, "%stensor pointers must be 16-byte aligned", pre);
  return 0;
}

// The bf16 engine's buffers inside a forward workspace and a packed-weight buffer: `step` with every field set that does
// not change from step to step, and the ping-pong halves that set_parity() points its in / out fields at.
struct StepBuffers {
  Bf16Buffers step;
  __nv_bfloat16 *sb[2], *sp[2], *xb;
  float* nsq[2];
};
static StepBuffers bind_step_buffers(const WorkspaceLayout& wl, const PackedLayout& pl, void* workspace,
                                     const void* packed_weights, const float* pos) {
  char* ws = static_cast<char*>(workspace);
  const char* pw = static_cast<const char*>(packed_weights);
  StepBuffers s{};
  for (int i = 0; i < 2; ++i) {
    s.sb[i] = reinterpret_cast<__nv_bfloat16*>(ws + wl.sb_off[i]);
    s.sp[i] = reinterpret_cast<__nv_bfloat16*>(ws + wl.sp_off[i]);
    s.nsq[i] = reinterpret_cast<float*>(ws + wl.nsq_off[i]);
  }
  s.xb = reinterpret_cast<__nv_bfloat16*>(ws + wl.xb_off);
  s.step.xb = s.xb;
  s.step.h = reinterpret_cast<__nv_bfloat16*>(ws + wl.h_off);
  s.step.c = reinterpret_cast<__nv_bfloat16*>(ws + wl.c_off);
  s.step.attn_acc = wl.attn_acc_bytes ? reinterpret_cast<float*>(ws + wl.attn_acc_off) : nullptr;
  s.step.pos = pos;
  s.step.w1 = reinterpret_cast<const __nv_bfloat16*>(pw + pl.w1_off);
  s.step.w2 = reinterpret_cast<const __nv_bfloat16*>(pw + pl.w2_off);
  s.step.b1 = reinterpret_cast<const float*>(pw + pl.b1_off);
  s.step.b2 = reinterpret_cast<const float*>(pw + pl.b2_off);
  return s;
}
// the step reads the shadows / norm partials of buffer p and writes those of the other one
static void set_parity(StepBuffers& s, int p) {
  s.step.sb_in = s.sb[p]; s.step.sb_out = s.sb[p ^ 1];
  s.step.sp_in = s.sp[p]; s.step.sp_out = s.sp[p ^ 1];
  s.step.nsq_in = s.nsq[p]; s.step.nsq_out = s.nsq[p ^ 1];
}

// the freeze flags and settle's change partials inside a settle workspace
struct SettleFlags { int *frozen, *block_frozen; float* dsq; unsigned int* done; float* level_q; };
static SettleFlags bind_settle_flags(const SettleLayout& sl, void* workspace) {
  char* ws = static_cast<char*>(workspace);
  return {reinterpret_cast<int*>(ws + sl.frozen_off), reinterpret_cast<int*>(ws + sl.block_frozen_off),
          reinterpret_cast<float*>(ws + sl.dsq_off), reinterpret_cast<unsigned int*>(ws + sl.done_off),
          reinterpret_cast<float*>(ws + sl.level_q_off)};
}

// glom_b200_settle / glom_b200_settle_all: a forward of max_iters steps (return_all = 0 / 1) that stops each image at the
// first step whose change criterion is <= tol
struct SettleRun { float tol; int32_t* steps; };

// One forward call: the operands of glom_b200_forward, and what selects the other forms
struct ForwardArgs {
  const glom_b200_cfg* cfg; const void* packed_weights; const float *tokens, *pos, *state_in, *init_levels; float* state_out;
  int batch, iters, return_all; void* workspace; size_t workspace_bytes; void* stream;
  int resume_parity = -1;              // glom_b200_forward_resume: the shadow buffer that holds state_in's shadows
  const SettleRun* settle = nullptr;   // glom_b200_settle / _settle_all
  const int32_t* steps = nullptr;      // glom_b200_forward_steps: per-image step counts (device memory)
};

static int forward_impl(const ForwardArgs& a) {
  const glom_b200_cfg* cfg = a.cfg;
  const float *state_in = a.state_in, *init_levels = a.init_levels;
  float* state_out = a.state_out;
  const int iters = a.iters, return_all = a.return_all;
  const SettleRun* settle = a.settle;
  const int32_t* steps = a.steps;
  if (int r = check_cfg(cfg)) return r;
  if (a.batch < 1 || iters < 0) return fail(GLOM_B200_ERR_INVALID, "batch must be >= 1 and iters >= 0");
  if (cfg->precision == GLOM_B200_FP32 && cfg->dim + cfg->n > kAttnF32MaxDimPlusN)
    return fail(GLOM_B200_ERR_INVALID,
                "fp32 consensus keeps %d (dim + n) floats per block in shared memory: dim + n must be <= %d (got %d)",
                kAttnF32Queries, kAttnF32MaxDimPlusN, cfg->dim + cfg->n);
  if (int r = check_tensors("", true, a.packed_weights, a.tokens, a.pos, state_in, init_levels, state_out, a.workspace)) return r;
  DeviceInfo di{};
  if (int r = device_info(&di)) return r;
  const Geometry g = make_geometry(cfg, a.batch);
  // settle and forward_steps freeze images: the SETTLE instantiations of the step kernels, driven by per-image flags
  const bool freeze = settle || steps;
  const SettleLayout sl = freeze ? settle_layout(g, iters, return_all) : SettleLayout{};
  const WorkspaceLayout wl = freeze ? sl.fwd : workspace_layout(g, cfg->precision, iters, return_all);
  const size_t ws_need = freeze ? sl.total : wl.total;
  if (!a.workspace || a.workspace_bytes < ws_need)
    return fail(GLOM_B200_ERR_WORKSPACE, "workspace: need %zu bytes, got %zu", ws_need, a.workspace_bytes);
  const PackedLayout pl = packed_layout(g.d, g.L, cfg->precision);
  char* ws = static_cast<char*>(a.workspace);
  Launch& ln = begin_launch(di.sms, a.stream);
  const size_t slab = (size_t)g.rows * g.L * g.d;

  // where the fp32 master of step t lives
  float* wslab = reinterpret_cast<float*>(ws + wl.s32_off);
  auto loc = [&](int t) -> float* {
    if (return_all) return state_out + (size_t)t * slab;
    return ((iters - t) % 2 == 0) ? state_out : wslab;
  };

  if (cfg->precision == GLOM_B200_BF16) {
    StepBuffers sbuf = bind_step_buffers(wl, pl, a.workspace, a.packed_weights, a.pos);
    Bf16Buffers& b = sbuf.step;
    // resumed call (glom_b200_forward_resume): the shadows / norm partials of state_in are the ones the previous call left
    // in buffer `p0`; the state prologue is skipped and step 0 reads the fp32 master straight from state_in
    const bool resume = a.resume_parity >= 0;
    const int p0 = resume ? a.resume_parity : 0;
    const bool s0_direct = resume || (!return_all && iters >= 1);
    int prep;
    if (resume) {
      prep = launch_prep(g, nullptr, nullptr, a.pos, a.tokens, nullptr, nullptr, nullptr, sbuf.xb, nullptr, ln);
      if (prep == 0 && return_all)         // slab 0 of the return_all form is S_0 (:126)
        prep = ln.launched(cudaMemcpyAsync(state_out, state_in, slab * sizeof(float), cudaMemcpyDeviceToDevice, ln.st));
    } else {
      // S_0 as an fp32 slab is only materialised when it is part of the result (return_all slab 0, iters == 0): otherwise
      // step 0 reads the carried state from the caller's tensor, or init_levels broadcast over the rows
      prep = launch_prep(g, state_in, init_levels, a.pos, a.tokens, s0_direct ? nullptr : loc(0), sbuf.sb[0], sbuf.sp[0], sbuf.xb,
                         sbuf.nsq[0], ln);
    }
    if (prep) return fail(prep, "prep launch: %s", ln.err);
    // settle: no image has stopped yet.  forward_steps: the schedule kernel writes every flag before each step
    const SettleFlags fl = freeze ? bind_settle_flags(sl, a.workspace) : SettleFlags{};
    b.frozen = fl.frozen; b.block_frozen = fl.block_frozen;
    b.dsq_out = settle ? fl.dsq : nullptr;     // NULL: K2 sums no squared change
    if (settle) {
      if (int r = ln.check(cudaMemsetAsync(ws + sl.flags_off, 0, sl.flags_bytes, ln.st)))
        return fail(r, "settle flags memset: %s", ln.err);
    }
    // Image-independent levels (DESIGN.md): every image starts from init_levels, and S_t[l] differs between images only
    // for l <= t - 1.  Steps t < L then run the work whose inputs are the same in every image for the representative rows
    // only.  From iters >= L + 1 on the last step, and so every buffer the call leaves behind, runs in full.  The
    // representative blocks must leave other blocks to skip, and K2 indexes an image's state in 32 bits.
    const bool ii = !state_in && !resume && !freeze && iters >= g.L + 1 && g.L <= 32 &&
                    rep_row_blocks(g.n) < (g.rows + 255) / 256 && (size_t)g.n * g.L * g.d < (1u << 31);
    for (int t = 0; t < iters; ++t) {
      if (steps) {         // images with steps[b] <= t are frozen from step t on (from the start when steps[b] == 0)
        if (int r = launch_steps_schedule(g, t, iters, steps, fl.frozen, fl.block_frozen, ln))
          return fail(r, "step schedule launch before step %d: %s", t, ln.err);
      }
      b.s32_in = (s0_direct && t == 0) ? (state_in ? state_in : init_levels) : loc(t); b.s32_out = loc(t + 1);
      b.s32_in_bcast = (s0_direct && t == 0 && !state_in) ? 1 : 0;
      set_parity(sbuf, (t + p0) & 1);
      b.ii_reduce = ii && t < g.L;
      if (int r = step_bf16(g, b, t, ln)) return fail(r, "step %d: %s", t, ln.err);
      if (settle) {
        if (int r = launch_settle_converge(g, t + 1, settle->tol, fl.dsq, b.nsq_out, fl.frozen, fl.block_frozen, fl.done,
                                           fl.level_q, settle->steps, ln))
          return fail(r, "settle convergence launch after step %d: %s", t, ln.err);
      }
    }
    // settle and forward_steps: return_all slab t of image b must be S_min(t, steps[b]).  Otherwise S_steps[b] is in
    // loc(steps[b]) and the ones in the workspace slab move to state_out; steps[b] == 0 (forward_steps only) takes S_0,
    // which step 0 read straight from state_in / init_levels
    const int32_t* image_steps = settle ? settle->steps : steps;
    if (ii && return_all) {
      if (int r = launch_level_fill(g, state_out, ln)) return fail(r, "return_all level fill launch: %s", ln.err);
    }
    if (image_steps && return_all) {
      if (int r = launch_steps_fill(g, iters, image_steps, state_out, ln)) return fail(r, "return_all fill launch: %s", ln.err);
    } else if (image_steps && iters > 0) {
      if (int r = launch_settle_gather(g, iters, image_steps, wslab, state_out, state_in ? state_in : init_levels,
                                       state_in ? 0 : 1, ln))
        return fail(r, "%s gather launch: %s", settle ? "settle" : "step", ln.err);
    }
  } else {
    const char* pw = static_cast<const char*>(a.packed_weights);
    if (int r = launch_broadcast_init(g, state_in, init_levels, loc(0), ln)) return fail(r, "init launch: %s", ln.err);
    for (int t = 0; t < iters; ++t) {
      F32Buffers b{};
      b.s_in = loc(t); b.s_out = loc(t + 1);
      b.x = a.tokens; b.pos = a.pos;
      b.h = reinterpret_cast<float*>(ws + wl.h_off);
      b.c = reinterpret_cast<float*>(ws + wl.c_off);
      b.w1 = reinterpret_cast<const float*>(pw + pl.w1_off);
      b.w2 = reinterpret_cast<const float*>(pw + pl.w2_off);
      b.b1 = reinterpret_cast<const float*>(pw + pl.b1_off);
      b.b2 = reinterpret_cast<const float*>(pw + pl.b2_off);
      if (int r = step_f32(g, b, ln)) return fail(r, "fp32 step %d launch: %s", t, ln.err);
    }
  }
  g_err[0] = 0;
  return 0;
}

// The freeze modes: settle / settle_all (bound max_iters >= 1) and forward_steps (bound max_steps >= 0) run the bf16
// engine's SETTLE step kernels.  Their workspace is the forward's plus the freeze flags (settle_layout).
struct FreezeMode { const char* name; const char* bound; int min_bound; };
static const FreezeMode kSettle{"settle", "max_iters", 1}, kForwardSteps{"forward_steps", "max_steps", 0};

static int check_freeze(const FreezeMode& m, const glom_b200_cfg* cfg, int batch, int bound) {
  if (int r = check_cfg(cfg)) return r;
  if (cfg->precision != GLOM_B200_BF16) return fail(GLOM_B200_ERR_INVALID, "%s: bf16 engine only (precision fp32 given)", m.name);
  if (batch < 1) return fail(GLOM_B200_ERR_INVALID, "%s: batch must be >= 1 (got %d)", m.name, batch);
  if (bound < m.min_bound) return fail(GLOM_B200_ERR_INVALID, "%s: %s must be >= %d (got %d)", m.name, m.bound, m.min_bound, bound);
  return 0;
}

static int freeze_workspace_bytes(const FreezeMode& m, const glom_b200_cfg* cfg, int batch, int bound, int return_all,
                                  size_t* out_bytes) {
  if (int r = check_freeze(m, cfg, batch, bound)) return r;
  if (!out_bytes) return fail(GLOM_B200_ERR_INVALID, "out_bytes is NULL");
  *out_bytes = settle_layout(make_geometry(cfg, batch), bound, return_all ? 1 : 0).total;
  return 0;
}

static int check_steps_ptr(const char* fn, const char* arg, const int32_t* steps) {
  if (!steps) return fail(GLOM_B200_ERR_INVALID, "%s: %s is NULL", fn, arg);
  if (misaligned(steps, 4)) return fail(GLOM_B200_ERR_INVALID, "%s: %s must be 4-byte aligned", fn, arg);
  return 0;
}

static int settle_impl(ForwardArgs a, float tol, int32_t* steps_out) {
  if (int r = check_freeze(kSettle, a.cfg, a.batch, a.iters)) return r;
  if (tol != tol) return fail(GLOM_B200_ERR_INVALID, "settle: tol is NaN");
  if (int r = check_steps_ptr("settle", "steps_out", steps_out)) return r;
  const SettleRun run{tol, steps_out};
  a.settle = &run;
  return forward_impl(a);
}

GLOM_B200_API int glom_b200_settle_workspace_bytes(const glom_b200_cfg* cfg, int batch, int max_iters, size_t* out_bytes) {
  return freeze_workspace_bytes(kSettle, cfg, batch, max_iters, 0, out_bytes);
}

GLOM_B200_API int glom_b200_settle_workspace_offset(const glom_b200_cfg* cfg, int batch, int max_iters, int return_all,
                                                    int which, size_t* out_offset, size_t* out_bytes) {
  if (int r = check_freeze(kSettle, cfg, batch, max_iters)) return r;
  if (!out_offset || !out_bytes) return fail(GLOM_B200_ERR_INVALID, "settle: out_offset / out_bytes is NULL");
  const Geometry g = make_geometry(cfg, batch);
  const SettleLayout s = settle_layout(g, max_iters, return_all ? 1 : 0);
  switch (which) {
    case 0: *out_offset = s.dsq_off; *out_bytes = s.fwd.nsq_bytes; return 0;
    case 1: *out_offset = s.level_q_off; *out_bytes = (size_t)g.B * g.L * 4; return 0;
    case 2: *out_offset = s.frozen_off; *out_bytes = (size_t)g.B * 4; return 0;
    case 3: *out_offset = s.block_frozen_off; *out_bytes = (size_t)(g.rows + 255) / 256 * 4; return 0;
    default: return fail(GLOM_B200_ERR_INVALID, "unknown settle buffer id %d", which);
  }
}

GLOM_B200_API int glom_b200_settle(const glom_b200_cfg* cfg, const void* packed_weights, const float* tokens, const float* pos,
                                   const float* state_in, const float* init_levels, float* state_out, int batch, int max_iters,
                                   float tol, int32_t* steps_out, void* workspace, size_t workspace_bytes, void* stream) {
  return settle_impl({cfg, packed_weights, tokens, pos, state_in, init_levels, state_out, batch, max_iters, 0, workspace,
                      workspace_bytes, stream}, tol, steps_out);
}

// glom_b200_settle_all: glom_b200_settle with every state kept (the return_all form of forward_steps)
GLOM_B200_API int glom_b200_settle_all_workspace_bytes(const glom_b200_cfg* cfg, int batch, int max_iters, size_t* out_bytes) {
  return freeze_workspace_bytes(kSettle, cfg, batch, max_iters, 1, out_bytes);
}

GLOM_B200_API int glom_b200_settle_all(const glom_b200_cfg* cfg, const void* packed_weights, const float* tokens,
                                       const float* pos, const float* state_in, const float* init_levels, float* states_out,
                                       int batch, int max_iters, float tol, int32_t* steps_out, void* workspace,
                                       size_t workspace_bytes, void* stream) {
  return settle_impl({cfg, packed_weights, tokens, pos, state_in, init_levels, states_out, batch, max_iters, 1, workspace,
                      workspace_bytes, stream}, tol, steps_out);
}

// glom_b200_forward_steps: a forward of max_steps steps in which image b stops after steps[b] (read on the device only)
GLOM_B200_API int glom_b200_forward_steps_workspace_bytes(const glom_b200_cfg* cfg, int batch, int max_steps, int return_all,
                                                          size_t* out_bytes) {
  return freeze_workspace_bytes(kForwardSteps, cfg, batch, max_steps, return_all, out_bytes);
}

GLOM_B200_API int glom_b200_forward_steps(const glom_b200_cfg* cfg, const void* packed_weights, const float* tokens,
                                          const float* pos, const float* state_in, const float* init_levels, float* state_out,
                                          int batch, const int32_t* steps, int max_steps, int return_all, void* workspace,
                                          size_t workspace_bytes, void* stream) {
  if (int r = check_freeze(kForwardSteps, cfg, batch, max_steps)) return r;
  if (int r = check_steps_ptr("forward_steps", "steps", steps)) return r;
  ForwardArgs a{cfg, packed_weights, tokens, pos, state_in, init_levels, state_out, batch, max_steps, return_all ? 1 : 0,
                workspace, workspace_bytes, stream};
  a.steps = steps;
  return forward_impl(a);
}

GLOM_B200_API int glom_b200_forward(const glom_b200_cfg* cfg, const void* packed_weights, const float* tokens, const float* pos,
                      const float* state_in, const float* init_levels, float* state_out, int batch, int iters,
                      int return_all, void* workspace, size_t workspace_bytes, void* stream) {
  return forward_impl({cfg, packed_weights, tokens, pos, state_in, init_levels, state_out, batch, iters, return_all, workspace,
                       workspace_bytes, stream});
}

GLOM_B200_API int glom_b200_forward_resume(const glom_b200_cfg* cfg, const void* packed_weights, const float* tokens,
                                           const float* pos, const float* state_in, float* state_out, int batch, int iters,
                                           int return_all, void* workspace, size_t workspace_bytes, void* stream,
                                           int shadow_parity, int* out_shadow_parity) {
  if (!cfg || cfg->precision != GLOM_B200_BF16) return fail(GLOM_B200_ERR_INVALID, "forward_resume: bf16 engine only");
  if (!state_in || (shadow_parity != 0 && shadow_parity != 1) || iters < 1)
    return fail(GLOM_B200_ERR_INVALID, "forward_resume: need state_in, shadow_parity in {0, 1} and iters >= 1");
  ForwardArgs a{cfg, packed_weights, tokens, pos, state_in, nullptr, state_out, batch, iters, return_all, workspace,
                workspace_bytes, stream};
  a.resume_parity = shadow_parity;
  const int r = forward_impl(a);
  if (r == 0 && out_shadow_parity) *out_shadow_parity = (shadow_parity + iters) & 1;
  return r;
}

// glom_b200_settle_queue_* and glom_b200_settle_video_*: the arguments shared by _begin and _run, checked in the same
// order as settle's.  settle_queue queues `items` = N images (frames = 1); settle_video queues `items` = S streams of
// `frames` frames each, and its images are the S * frames frames.
struct QueueMode { const char* name; const char* pre; const char* items; };
static const QueueMode kQueue{"settle_queue", "settle_queue: ", "images"}, kVideo{"settle_video", "settle_video: ", "streams"};

struct QueueArgs {
  const QueueMode& mode;
  const glom_b200_cfg* cfg; const float *tokens, *pos, *state_in, *init_levels; float* state_out; int32_t* steps_out;
  int items, frames, slots, max_iters; float tol; void* workspace; size_t workspace_bytes; void* stream;
};

static int check_queue_sizes(const QueueMode& m, const glom_b200_cfg* cfg, int items, int frames, int slots, int max_iters) {
  if (int r = check_cfg(cfg)) return r;
  if (cfg->precision != GLOM_B200_BF16) return fail(GLOM_B200_ERR_INVALID, "%s: bf16 engine only (precision fp32 given)", m.name);
  if (items < 1) return fail(GLOM_B200_ERR_INVALID, "%s: %s must be >= 1 (got %d)", m.name, m.items, items);
  if (frames < 1) return fail(GLOM_B200_ERR_INVALID, "%s: frames must be >= 1 (got %d)", m.name, frames);
  if ((int64_t)items * frames > INT32_MAX)
    return fail(GLOM_B200_ERR_INVALID, "%s: %s x frames must be < 2^31 (got %d x %d)", m.name, m.items, items, frames);
  if (slots < 1) return fail(GLOM_B200_ERR_INVALID, "%s: slots must be >= 1 (got %d)", m.name, slots);
  if (max_iters < 1) return fail(GLOM_B200_ERR_INVALID, "%s: max_iters must be >= 1 (got %d)", m.name, max_iters);
  return 0;
}

// -> 0 and the geometry / layout of the slots, after every argument check and the device query
static int check_queue(const QueueArgs& a, Geometry* g, QueueLayout* ql, DeviceInfo* di) {
  const char* fn = a.mode.name;
  if (int r = check_queue_sizes(a.mode, a.cfg, a.items, a.frames, a.slots, a.max_iters)) return r;
  if (a.tol != a.tol) return fail(GLOM_B200_ERR_INVALID, "%s: tol is NaN", fn);
  if (int r = check_steps_ptr(fn, "steps_out", a.steps_out)) return r;
  if (int r = check_tensors(a.mode.pre, false, nullptr, a.tokens, a.pos, a.state_in, a.init_levels, a.state_out, a.workspace))
    return r;
  *g = make_geometry(a.cfg, a.slots);
  *ql = queue_layout(*g, a.max_iters);
  if (!a.workspace || a.workspace_bytes < ql->total)
    return fail(GLOM_B200_ERR_WORKSPACE, "%s workspace: need %zu bytes, got %zu", fn, ql->total, a.workspace_bytes);
  return device_info(di);
}

static QueueSlots queue_slots(const QueueArgs& a, const QueueLayout& ql) {
  char* ws = static_cast<char*>(a.workspace);
  QueueSlots q{};
  q.slot_img = reinterpret_cast<int*>(ws + ql.slot_img_off);
  q.age = reinterpret_cast<int*>(ws + ql.age_off);
  q.pending = reinterpret_cast<int*>(ws + ql.pending_off);
  q.gather_img = reinterpret_cast<int*>(ws + ql.gather_off);
  q.fresh = reinterpret_cast<int*>(ws + ql.fresh_off);
  q.block_fresh = reinterpret_cast<int*>(ws + ql.block_fresh_off);
  q.head = reinterpret_cast<int*>(ws + ql.head_off);
  q.unfinished = reinterpret_cast<int*>(ws + ql.unfinished_off);
  q.images = a.items * a.frames;
  q.frames = a.frames;
  q.max_iters = a.max_iters;
  return q;
}

static int queue_begin(const QueueArgs& a) {
  Geometry g{}; QueueLayout ql{}; DeviceInfo di{};
  if (int r = check_queue(a, &g, &ql, &di)) return r;
  const SettleFlags fl = bind_settle_flags(ql.settle, a.workspace);
  Launch& ln = begin_launch(di.sms, a.stream);
  if (int r = launch_queue_init(g, queue_slots(a, ql), fl.frozen, fl.block_frozen, fl.done, ln))
    return fail(r, "%s init launch: %s", a.mode.name, ln.err);
  g_err[0] = 0;
  return 0;
}

// Global steps first_step .. first_step + num_steps - 1: schedule, fill, K1, K3, K2, convergence each.  num_steps == 0:
// the schedule and fill of step first_step without admissions, i.e. the hand-over of the images that stopped last.
static int queue_run(const QueueArgs& a, const void* packed_weights, int first_step, int num_steps, int32_t* remaining_out) {
  Geometry g{}; QueueLayout ql{}; DeviceInfo di{};
  const char* fn = a.mode.name;
  if (int r = check_queue_sizes(a.mode, a.cfg, a.items, a.frames, a.slots, a.max_iters)) return r;
  if (!packed_weights || misaligned(packed_weights, 1024))
    return fail(GLOM_B200_ERR_INVALID, "%s: packed weights NULL or not 1024-byte aligned", fn);
  if (first_step < 0 || num_steps < 0)
    return fail(GLOM_B200_ERR_INVALID, "%s: first_step and num_steps must be >= 0 (got %d, %d)", fn, first_step, num_steps);
  if (misaligned(remaining_out, 4)) return fail(GLOM_B200_ERR_INVALID, "%s: remaining_out must be 4-byte aligned", fn);
  if (int r = check_queue(a, &g, &ql, &di)) return r;
  char* ws = static_cast<char*>(a.workspace);
  const QueueSlots q = queue_slots(a, ql);
  float* slab[2] = {reinterpret_cast<float*>(ws + ql.slab_off[0]), reinterpret_cast<float*>(ws + ql.slab_off[1])};
  StepBuffers sbuf = bind_step_buffers(ql.settle.fwd, packed_layout(g.d, g.L, GLOM_B200_BF16), a.workspace, packed_weights, a.pos);
  const SettleFlags fl = bind_settle_flags(ql.settle, a.workspace);
  Bf16Buffers& b = sbuf.step;
  b.frozen = fl.frozen; b.block_frozen = fl.block_frozen; b.dsq_out = fl.dsq; b.block_fresh = q.block_fresh;
  Launch& ln = begin_launch(di.sms, a.stream);
  const int last = first_step + (num_steps > 0 ? num_steps : 1);
  for (int t = first_step; t < last; ++t) {
    const int p = t & 1;
    int r = launch_queue_schedule(g, q, num_steps > 0, fl.frozen, fl.block_frozen, ln);
    if (r == 0)
      r = launch_queue_fill(g, q, a.tokens, a.pos, a.state_in, a.init_levels, a.state_out, slab[p], sbuf.sb[p], sbuf.sp[p],
                            sbuf.nsq[p], sbuf.xb, ln);
    if (r) return fail(r, "%s slot launch before step %d: %s", fn, t, ln.err);
    if (num_steps == 0) break;
    b.s32_in = slab[p]; b.s32_out = slab[p ^ 1]; b.s32_in_bcast = 0;
    set_parity(sbuf, p);
    if (int r = step_bf16(g, b, t, ln)) return fail(r, "%s step %d: %s", fn, t, ln.err);
    if (int r = launch_settle_converge(g, t + 1, a.tol, fl.dsq, b.nsq_out, fl.frozen, fl.block_frozen, fl.done, fl.level_q,
                                       a.steps_out, ln, &q))
      return fail(r, "%s convergence launch after step %d: %s", fn, t, ln.err);
  }
  if (remaining_out) {
    if (int r = ln.launched(cudaMemcpyAsync(remaining_out, q.unfinished, sizeof(int32_t), cudaMemcpyDeviceToDevice, ln.st)))
      return fail(r, "%s count copy: %s", fn, ln.err);
  }
  g_err[0] = 0;
  return 0;
}

// Glom.settle_queue: N images through `slots` batch slots, see include/glom_b200.h
static int queue_workspace_bytes(const QueueMode& m, const glom_b200_cfg* cfg, int slots, int max_iters, size_t* out_bytes) {
  if (int r = check_queue_sizes(m, cfg, 1, 1, slots, max_iters)) return r;
  if (!out_bytes) return fail(GLOM_B200_ERR_INVALID, "out_bytes is NULL");
  *out_bytes = queue_layout(make_geometry(cfg, slots), max_iters).total;
  return 0;
}

GLOM_B200_API int glom_b200_settle_queue_workspace_bytes(const glom_b200_cfg* cfg, int slots, int max_iters, size_t* out_bytes) {
  return queue_workspace_bytes(kQueue, cfg, slots, max_iters, out_bytes);
}

GLOM_B200_API int glom_b200_settle_queue_begin(const glom_b200_cfg* cfg, const float* tokens, const float* pos,
                                               const float* state_in, const float* init_levels, float* state_out,
                                               int32_t* steps_out, int images, int slots, int max_iters, float tol,
                                               void* workspace, size_t workspace_bytes, void* stream) {
  return queue_begin({kQueue, cfg, tokens, pos, state_in, init_levels, state_out, steps_out, images, 1, slots, max_iters, tol,
                      workspace, workspace_bytes, stream});
}

GLOM_B200_API int glom_b200_settle_queue_run(const glom_b200_cfg* cfg, const void* packed_weights, const float* tokens,
                                             const float* pos, const float* state_in, const float* init_levels,
                                             float* state_out, int32_t* steps_out, int images, int slots, int max_iters,
                                             float tol, void* workspace, size_t workspace_bytes, void* stream, int first_step,
                                             int num_steps, int32_t* remaining_out) {
  return queue_run({kQueue, cfg, tokens, pos, state_in, init_levels, state_out, steps_out, images, 1, slots, max_iters, tol,
                    workspace, workspace_bytes, stream}, packed_weights, first_step, num_steps, remaining_out);
}

// Glom.settle_video: S streams of F frames through `slots` batch slots, see include/glom_b200.h
GLOM_B200_API int glom_b200_settle_video_workspace_bytes(const glom_b200_cfg* cfg, int slots, int max_iters, size_t* out_bytes) {
  return queue_workspace_bytes(kVideo, cfg, slots, max_iters, out_bytes);
}

GLOM_B200_API int glom_b200_settle_video_begin(const glom_b200_cfg* cfg, const float* tokens, const float* pos,
                                               const float* state_in, const float* init_levels, float* state_out,
                                               int32_t* steps_out, int streams, int frames, int slots, int max_iters,
                                               float tol, void* workspace, size_t workspace_bytes, void* stream) {
  return queue_begin({kVideo, cfg, tokens, pos, state_in, init_levels, state_out, steps_out, streams, frames, slots, max_iters,
                      tol, workspace, workspace_bytes, stream});
}

GLOM_B200_API int glom_b200_settle_video_run(const glom_b200_cfg* cfg, const void* packed_weights, const float* tokens,
                                             const float* pos, const float* state_in, const float* init_levels,
                                             float* state_out, int32_t* steps_out, int streams, int frames, int slots,
                                             int max_iters, float tol, void* workspace, size_t workspace_bytes, void* stream,
                                             int first_step, int num_steps, int32_t* remaining_out) {
  return queue_run({kVideo, cfg, tokens, pos, state_in, init_levels, state_out, steps_out, streams, frames, slots, max_iters,
                    tol, workspace, workspace_bytes, stream}, packed_weights, first_step, num_steps, remaining_out);
}

static int tok_kp(int patch) { return (3 * patch * patch + 63) / 64 * 64; }

// true unless the image is a batch of whole patches
static bool bad_patch_grid(int batch, int height, int width, int patch) {
  return batch < 1 || patch < 1 || height < patch || width < patch || height % patch || width % patch;
}

GLOM_B200_API int glom_b200_tokenize_workspace_bytes(int batch, int height, int width, int patch, int dim, int precision,
                                                     size_t* out_bytes) {
  if (!out_bytes || dim < 1 || bad_patch_grid(batch, height, width, patch))
    return fail(GLOM_B200_ERR_INVALID, "bad tokeniser geometry");
  if (precision == GLOM_B200_BF16) {
    const size_t rows = (size_t)batch * (height / patch) * (width / patch);
    *out_bytes = align_up(rows * tok_kp(patch) * 2, 1024) + align_up((size_t)dim * tok_kp(patch) * 2, 1024);
  } else {
    *out_bytes = 0;
  }
  return 0;
}

GLOM_B200_API int glom_b200_tokenize(const float* img, const float* weight, const float* bias, float* tokens, int batch, int height,
                       int width, int patch, int dim, int precision, void* workspace, size_t workspace_bytes, void* stream) {
  if (!img || !weight || !bias || !tokens) return fail(GLOM_B200_ERR_INVALID, "a required pointer is NULL");
  if (dim < 1 || bad_patch_grid(batch, height, width, patch))
    return fail(GLOM_B200_ERR_INVALID, "image %dx%d is not a positive multiple of patch %d", height, width, patch);
  if (precision != GLOM_B200_FP32 && precision != GLOM_B200_BF16) return fail(GLOM_B200_ERR_INVALID, "unknown precision %d", precision);
  DeviceInfo di{};
  if (int r = device_info(&di)) return r;
  Launch& ln = begin_launch(di.sms, stream);
  if (precision == GLOM_B200_FP32) {
    if (int r = launch_tokenize(img, weight, bias, tokens, batch, height, width, patch, dim, ln))
      return fail(r, "tokenize launch: %s", ln.err);
    return 0;
  }
  if (dim % 64) return fail(GLOM_B200_ERR_INVALID, "bf16 tokeniser needs dim %% 64 == 0 (got %d)", dim);
  size_t need = 0;
  glom_b200_tokenize_workspace_bytes(batch, height, width, patch, dim, precision, &need);
  if (!workspace || workspace_bytes < need || misaligned(workspace, 1024))
    return fail(GLOM_B200_ERR_WORKSPACE, "tokeniser workspace: need %zu bytes 1024-aligned, got %zu", need, workspace_bytes);
  const int kp = tok_kp(patch);
  const int rows = batch * (height / patch) * (width / patch);
  __nv_bfloat16* patches = static_cast<__nv_bfloat16*>(workspace);
  __nv_bfloat16* wtok = reinterpret_cast<__nv_bfloat16*>(static_cast<char*>(workspace) + align_up((size_t)rows * kp * 2, 1024));
  ProfScope scope(ln.prof, PROF_TOKENIZE, ln.st);
  if (int r = launch_patchify_bf16(img, weight, patches, wtok, batch, height, width, patch, dim, kp, ln))
    return fail(r, "patchify launch: %s", ln.err);
  if (int r = tokenize_tc(patches, wtok, bias, tokens, rows, dim, kp, ln)) return fail(r, "%s", ln.err);
  return 0;
}

GLOM_B200_API int glom_b200_tokenize_backward_workspace_bytes(int batch, int height, int width, int patch, int need_d_img,
                                                              size_t* out_bytes) {
  if (!out_bytes || bad_patch_grid(batch, height, width, patch))
    return fail(GLOM_B200_ERR_INVALID, "tokeniser backward: bad arguments");
  *out_bytes = tokenize_backward_workspace_bytes(batch, height, width, patch, need_d_img);
  return 0;
}

static int tokenize_backward_impl(const float* img, const float* weight, const float* d_tokens, float* d_weight,
                                  float* d_bias, float* d_img, int batch, int height, int width, int patch, int dim,
                                  int deterministic, void* workspace, size_t workspace_bytes, void* stream) {
  if (!img || !weight || !d_tokens) return fail(GLOM_B200_ERR_INVALID, "a required pointer is NULL");
  if (dim < 1 || bad_patch_grid(batch, height, width, patch))
    return fail(GLOM_B200_ERR_INVALID, "image %dx%d is not a positive multiple of patch %d", height, width, patch);
  DeviceInfo di{};
  if (int r = device_info(&di)) return r;
  const size_t need = tokenize_backward_workspace_bytes(batch, height, width, patch, d_img != nullptr);
  if ((d_weight || d_img) && (!workspace || workspace_bytes < need))
    return fail(GLOM_B200_ERR_WORKSPACE, "tokeniser backward workspace: need %zu bytes, got %zu", need, workspace_bytes);
  Launch& ln = begin_launch(di.sms, stream);
  if (int r = tokenize_backward(img, weight, d_tokens, d_weight, d_bias, d_img, batch, height, width, patch, dim, workspace, ln,
                                deterministic))
    return fail(r, "tokeniser backward: %s", ln.err);
  return 0;
}

GLOM_B200_API int glom_b200_tokenize_backward(const float* img, const float* weight, const float* d_tokens, float* d_weight,
                                              float* d_bias, float* d_img, int batch, int height, int width, int patch, int dim,
                                              void* workspace, size_t workspace_bytes, void* stream) {
  return tokenize_backward_impl(img, weight, d_tokens, d_weight, d_bias, d_img, batch, height, width, patch, dim, 0,
                                workspace, workspace_bytes, stream);
}

GLOM_B200_API int glom_b200_tokenize_backward_ex(const float* img, const float* weight, const float* d_tokens,
                                                 float* d_weight, float* d_bias, float* d_img, int batch, int height,
                                                 int width, int patch, int dim, int deterministic, void* workspace,
                                                 size_t workspace_bytes, void* stream) {
  if (deterministic != 0 && deterministic != 1)
    return fail(GLOM_B200_ERR_INVALID, "tokenize_backward_ex: deterministic must be 0 or 1 (got %d)", deterministic);
  return tokenize_backward_impl(img, weight, d_tokens, d_weight, d_bias, d_img, batch, height, width, patch, dim,
                                deterministic, workspace, workspace_bytes, stream);
}

GLOM_B200_API int glom_b200_backward_workspace_bytes(const glom_b200_cfg* cfg, int batch, size_t* out_bytes) {
  if (int r = check_cfg(cfg)) return r;
  if (batch < 1 || !out_bytes) return fail(GLOM_B200_ERR_INVALID, "bad batch/out_bytes");
  *out_bytes = backward_layout(make_geometry(cfg, batch), cfg->precision).total;
  return 0;
}

// The weight / gradient structs and tensor pointers of a backward, validated and gathered into `a`.  The explicit backward
// takes exactly one of d_state0 / d_init; the implicit one (`implicit`) neither
static int bind_backward(const glom_b200_weights_ref* w, const float* tokens, const float* pos, const float* states,
                         const float* grad_out, const glom_b200_grads* gr, bool implicit, int deterministic, BackwardArgs* a) {
  if (!w || w->struct_size != sizeof(glom_b200_weights_ref) || !gr || gr->struct_size != sizeof(glom_b200_grads))
    return fail(GLOM_B200_ERR_INVALID, "weights / grads struct missing or wrong size");
  if (!tokens || !pos || !states || !grad_out) return fail(GLOM_B200_ERR_INVALID, "a required pointer is NULL");
  if (!w->bu_w1 || !w->bu_b1 || !w->bu_w2 || !w->td_w1 || !w->td_b1 || !w->td_w2)
    return fail(GLOM_B200_ERR_INVALID, "a weight pointer is NULL");
  const bool outputs = gr->d_tokens && gr->d_pos && gr->d_bu_w1 && gr->d_bu_b1 && gr->d_bu_w2 && gr->d_bu_b2 && gr->d_td_w1 &&
                       gr->d_td_b1 && gr->d_td_w2 && gr->d_td_b2;
  if (!implicit && (!outputs || (!gr->d_state0 == !gr->d_init)))
    return fail(GLOM_B200_ERR_INVALID, "gradient pointers: all MLP/token/pos outputs and exactly one of d_state0 / d_init");
  if (implicit && !outputs) return fail(GLOM_B200_ERR_INVALID, "gradient pointers: all MLP/token/pos outputs are needed");
  if (implicit && (gr->d_state0 || gr->d_init))
    return fail(GLOM_B200_ERR_INVALID, "backward_implicit: d_state0 and d_init must be NULL (the fixed point does not "
                                       "depend on the start state)");
  *a = BackwardArgs{};
  a->tokens = tokens; a->pos = pos; a->states = states; a->grad_out = grad_out;
  a->bu_w1 = w->bu_w1; a->bu_b1 = w->bu_b1; a->bu_w2 = w->bu_w2; a->td_w1 = w->td_w1; a->td_b1 = w->td_b1; a->td_w2 = w->td_w2;
  a->d_tokens = gr->d_tokens; a->d_pos = gr->d_pos; a->d_state0 = gr->d_state0; a->d_init = gr->d_init;
  a->d_bu_w1 = gr->d_bu_w1; a->d_bu_b1 = gr->d_bu_b1; a->d_bu_w2 = gr->d_bu_w2; a->d_bu_b2 = gr->d_bu_b2;
  a->d_td_w1 = gr->d_td_w1; a->d_td_b1 = gr->d_td_b1; a->d_td_w2 = gr->d_td_w2; a->d_td_b2 = gr->d_td_b2;
  a->deterministic = deterministic;
  return 0;
}

// glom_b200_backward (steps == NULL) and glom_b200_backward_steps (per-image step counts, iters = max_steps)
static int backward_impl(const glom_b200_cfg* cfg, const glom_b200_weights_ref* w, const float* tokens, const float* pos,
                         const float* states, const float* grad_out, const glom_b200_grads* gr, int batch, int iters,
                         const int32_t* steps, int grad_all, void* workspace, size_t workspace_bytes, void* stream,
                         int deterministic = 0) {
  if (int r = check_cfg(cfg)) return r;
  if (batch < 1 || iters < 0) return fail(GLOM_B200_ERR_INVALID, "batch must be >= 1 and iters >= 0");
  BackwardArgs a{};
  if (int r = bind_backward(w, tokens, pos, states, grad_out, gr, false, deterministic, &a)) return r;
  DeviceInfo di{};
  if (int r = device_info(&di)) return r;
  const Geometry g = make_geometry(cfg, batch);
  const BackwardLayout wl = backward_layout(g, cfg->precision);
  if (!workspace || workspace_bytes < wl.total || misaligned(workspace, 1024))
    return fail(GLOM_B200_ERR_WORKSPACE, "backward workspace: need %zu bytes 1024-aligned, got %zu", wl.total, workspace_bytes);
  Launch& ln = begin_launch(di.sms, stream);
  if (int r = backward_run(g, a, cfg->precision, iters, grad_all, steps, workspace, ln)) return fail(r, "%s", ln.err);
  g_err[0] = 0;
  return 0;
}

GLOM_B200_API int glom_b200_backward(const glom_b200_cfg* cfg, const glom_b200_weights_ref* w, const float* tokens,
                                     const float* pos, const float* states, const float* grad_out,
                                     const glom_b200_grads* gr, int batch, int iters, int grad_all, void* workspace,
                                     size_t workspace_bytes, void* stream) {
  return backward_impl(cfg, w, tokens, pos, states, grad_out, gr, batch, iters, nullptr, grad_all, workspace,
                       workspace_bytes, stream);
}

GLOM_B200_API int glom_b200_backward_steps(const glom_b200_cfg* cfg, const glom_b200_weights_ref* w, const float* tokens,
                                           const float* pos, const float* states, const float* grad_out,
                                           const glom_b200_grads* gr, int batch, const int32_t* steps, int max_steps,
                                           int grad_all, void* workspace, size_t workspace_bytes, void* stream) {
  if (int r = check_steps_ptr("backward_steps", "steps", steps)) return r;
  if (max_steps < 0) return fail(GLOM_B200_ERR_INVALID, "backward_steps: max_steps must be >= 0 (got %d)", max_steps);
  return backward_impl(cfg, w, tokens, pos, states, grad_out, gr, batch, max_steps, steps, grad_all, workspace,
                       workspace_bytes, stream);
}

GLOM_B200_API int glom_b200_backward_ex(const glom_b200_cfg* cfg, const glom_b200_weights_ref* w, const float* tokens,
                                        const float* pos, const float* states, const float* grad_out,
                                        const glom_b200_grads* gr, int batch, const int32_t* steps, int max_steps,
                                        int grad_all, int deterministic, void* workspace, size_t workspace_bytes,
                                        void* stream) {
  if (deterministic != 0 && deterministic != 1)
    return fail(GLOM_B200_ERR_INVALID, "backward_ex: deterministic must be 0 or 1 (got %d)", deterministic);
  if (steps && misaligned(steps, 4)) return fail(GLOM_B200_ERR_INVALID, "backward_ex: steps must be 4-byte aligned");
  if (steps && max_steps < 0) return fail(GLOM_B200_ERR_INVALID, "backward_ex: max_steps must be >= 0 (got %d)", max_steps);
  return backward_impl(cfg, w, tokens, pos, states, grad_out, gr, batch, max_steps, steps, grad_all, workspace,
                       workspace_bytes, stream, deterministic);
}

GLOM_B200_API int glom_b200_backward_implicit_workspace_bytes(const glom_b200_cfg* cfg, int batch, size_t* out_bytes) {
  if (int r = check_cfg(cfg)) return r;
  if (cfg->precision != GLOM_B200_BF16) return fail(GLOM_B200_ERR_INVALID, "backward_implicit: bf16 engine only (precision fp32 given)");
  if (batch < 1 || !out_bytes) return fail(GLOM_B200_ERR_INVALID, "backward_implicit: bad batch/out_bytes");
  *out_bytes = implicit_layout(make_geometry(cfg, batch)).total;
  return 0;
}

GLOM_B200_API int glom_b200_backward_implicit(const glom_b200_cfg* cfg, const glom_b200_weights_ref* w, const float* tokens,
                                              const float* pos, const float* state, const float* grad_out,
                                              const glom_b200_grads* gr, int batch, int adjoint_iters, float adjoint_tol,
                                              int deterministic, int32_t* adjoint_steps_out, float* adjoint_q_out,
                                              void* workspace, size_t workspace_bytes, void* stream) {
  if (int r = check_cfg(cfg)) return r;
  if (cfg->precision != GLOM_B200_BF16) return fail(GLOM_B200_ERR_INVALID, "backward_implicit: bf16 engine only (precision fp32 given)");
  if (batch < 1) return fail(GLOM_B200_ERR_INVALID, "backward_implicit: batch must be >= 1 (got %d)", batch);
  if (adjoint_iters < 0)
    return fail(GLOM_B200_ERR_INVALID, "backward_implicit: adjoint_iters must be >= 0 (got %d)", adjoint_iters);
  if (adjoint_tol != adjoint_tol) return fail(GLOM_B200_ERR_INVALID, "backward_implicit: adjoint_tol is NaN");
  if (deterministic != 0 && deterministic != 1)
    return fail(GLOM_B200_ERR_INVALID, "backward_implicit: deterministic must be 0 or 1 (got %d)", deterministic);
  if (int r = check_steps_ptr("backward_implicit", "adjoint_steps_out", adjoint_steps_out)) return r;
  if (misaligned(adjoint_q_out, 4))
    return fail(GLOM_B200_ERR_INVALID, "backward_implicit: adjoint_q_out must be 4-byte aligned");
  BackwardArgs a{};
  if (int r = bind_backward(w, tokens, pos, state, grad_out, gr, true, deterministic, &a)) return r;
  DeviceInfo di{};
  if (int r = device_info(&di)) return r;
  const Geometry g = make_geometry(cfg, batch);
  const ImplicitLayout il = implicit_layout(g);
  if (!workspace || workspace_bytes < il.total || misaligned(workspace, 1024))
    return fail(GLOM_B200_ERR_WORKSPACE, "backward_implicit workspace: need %zu bytes 1024-aligned, got %zu", il.total,
                workspace_bytes);
  Launch& ln = begin_launch(di.sms, stream);
  if (int r = backward_implicit_run(g, a, adjoint_iters, adjoint_tol, adjoint_steps_out, adjoint_q_out, workspace, ln))
    return fail(r, "%s", ln.err);
  g_err[0] = 0;
  return 0;
}

GLOM_B200_API int glom_b200_islands(const float* states, int slabs, int side_h, int side_w, int levels, int dim, float threshold,
                                    float* cos_right, float* cos_down, float* agreement, int32_t* labels, int32_t* num_islands,
                                    void* stream) {
  if (!states || !cos_right || !cos_down || !agreement || !labels || !num_islands)
    return fail(GLOM_B200_ERR_INVALID, "a required pointer is NULL");
  if (slabs < 1 || slabs > 65535 || side_h < 1 || side_w < 1 || (long long)side_h * side_w > 8192 || levels < 1 ||
      levels > 65535 || dim < 4 || dim % 4)
    return fail(GLOM_B200_ERR_INVALID, "islands: need 1 <= slabs, levels <= 65535, side_h * side_w <= 8192, dim %% 4 == 0");
  if (misaligned(states, 16)) return fail(GLOM_B200_ERR_INVALID, "states must be 16-byte aligned");
  DeviceInfo di{};
  if (int r = device_info(&di)) return r;
  Launch& ln = begin_launch(di.sms, stream);
  if (int r = launch_islands(states, slabs, side_h, side_w, levels, dim, threshold, cos_right, cos_down, agreement, labels,
                             num_islands, ln))
    return fail(r, "islands launch: %s", ln.err);
  return 0;
}

GLOM_B200_API int glom_b200_island_tree(const int32_t* labels, const float* states, int slabs, int n, int levels, int dim,
                                        int32_t* size, int32_t* parent, float* containment, float* nested,
                                        float* embedding, float* member_cos, float* coherence, void* stream) {
  if (!labels || !size || !parent || !containment || (!nested && levels != 1))
    return fail(GLOM_B200_ERR_INVALID, "island_tree: a required pointer is NULL");
  if (!states != !embedding || !states != !member_cos || !states != !coherence)
    return fail(GLOM_B200_ERR_INVALID, "island_tree: states, embedding, member_cos and coherence are all NULL or all set");
  if (slabs < 1 || slabs > 65535 || n < 1 || n > 8192 || levels < 1 || levels > 65535 || dim < 4 || dim % 4)
    return fail(GLOM_B200_ERR_INVALID, "island_tree: need 1 <= slabs, levels <= 65535, 1 <= n <= 8192, dim %% 4 == 0");
  if (misaligned(states, 16) || misaligned(embedding, 16))
    return fail(GLOM_B200_ERR_INVALID, "island_tree: states and embedding must be 16-byte aligned");
  if (misaligned(labels, 4) || misaligned(size, 4) || misaligned(parent, 4) || misaligned(containment, 4) ||
      misaligned(nested, 4) || misaligned(member_cos, 4) || misaligned(coherence, 4))
    return fail(GLOM_B200_ERR_INVALID, "island_tree: labels and outputs must be 4-byte aligned");
  DeviceInfo di{};
  if (int r = device_info(&di)) return r;
  Launch& ln = begin_launch(di.sms, stream);
  if (int r = launch_island_tree(labels, states, slabs, n, levels, dim, size, parent, containment, nested, embedding,
                                 member_cos, coherence, ln))
    return fail(r, "island_tree launch: %s", ln.err);
  return 0;
}

GLOM_B200_API int glom_b200_island_track(const int32_t* labels, int outer, int times, int inner, int n, int levels,
                                         int32_t* prev, int32_t* overlap, int32_t* next, int32_t* track, void* stream) {
  if (!labels || !prev || !overlap || !next || !track)
    return fail(GLOM_B200_ERR_INVALID, "island_track: a required pointer is NULL");
  if (outer < 1 || times < 1 || inner < 1 || outer > 65535 || times > 65535 || inner > 65535 ||
      (long long)outer * times * inner > 65535 || n < 1 || n > 8192 || levels < 1 || levels > 65535)
    return fail(GLOM_B200_ERR_INVALID,
                "island_track: need 1 <= outer * times * inner <= 65535, 1 <= n <= 8192, 1 <= levels <= 65535");
  if (misaligned(labels, 4) || misaligned(prev, 4) || misaligned(overlap, 4) || misaligned(next, 4) ||
      misaligned(track, 4))
    return fail(GLOM_B200_ERR_INVALID, "island_track: labels and outputs must be 4-byte aligned");
  DeviceInfo di{};
  if (int r = device_info(&di)) return r;
  Launch& ln = begin_launch(di.sms, stream);
  if (int r = launch_island_track(labels, outer, times, inner, n, levels, prev, overlap, next, track, ln))
    return fail(r, "island_track launch: %s", ln.err);
  return 0;
}

GLOM_B200_API int glom_b200_clock_probe(uint64_t* out_cycles_ns, int spin_us, void* stream) {
  if (!out_cycles_ns || spin_us < 1 || spin_us > 100000) return fail(GLOM_B200_ERR_INVALID, "clock probe: bad arguments");
  cudaError_t e = launch_clock_probe(reinterpret_cast<unsigned long long*>(out_cycles_ns), (unsigned long long)spin_us * 1000ull,
                                     static_cast<cudaStream_t>(stream));
  if (e != cudaSuccess) return fail(GLOM_B200_ERR_CUDA, "clock probe launch: %s", cudaGetErrorString(e));
  return 0;
}

GLOM_B200_API int glom_b200_kernel_clocks(double* mhz_by_kind, double* ms_by_kind, double* wait_frac, int kinds, int reset) {
  if (!mhz_by_kind || !ms_by_kind || kinds < 1) return fail(GLOM_B200_ERR_INVALID, "kernel clocks: bad arguments");
  unsigned long long acc[PROF_KINDS][8];
  cudaError_t e = cudaDeviceSynchronize();
  if (e == cudaSuccess) e = tc_kernel_clocks(&acc[0][0], reset != 0);
  if (e != cudaSuccess) return fail(GLOM_B200_ERR_CUDA, "kernel clocks: %s", cudaGetErrorString(e));
  for (int i = 0; i < kinds; ++i) {
    const bool have = i < PROF_KINDS && acc[i][1] > 0;
    mhz_by_kind[i] = have ? 1e3 * (double)acc[i][0] / (double)acc[i][1] : 0.0;     // cycles per ns -> MHz
    ms_by_kind[i] = have ? 1e-6 * (double)acc[i][1] : 0.0;
    if (wait_frac)
      for (int j = 0; j < 6; ++j) wait_frac[6 * i + j] = have && acc[i][0] ? (double)acc[i][2 + j] / (double)acc[i][0] : 0.0;
  }
  return 0;
}

GLOM_B200_API int glom_b200_profile_begin(void) {
  g_prof.enabled = true;
  g_prof.used = 0;
  g_prof.spans.clear();
  return 0;
}

GLOM_B200_API int glom_b200_profile_end(double* ms_by_kind, int* launches_by_kind, int kinds) {
  if (!ms_by_kind || !launches_by_kind || kinds < 5) return fail(GLOM_B200_ERR_INVALID, "need room for at least 5 kinds");
  for (int i = 0; i < kinds; ++i) { ms_by_kind[i] = 0.0; launches_by_kind[i] = 0; }
  g_prof.enabled = false;
  for (const Profiler::Span& s : g_prof.spans) {
    cudaError_t e = cudaEventSynchronize(g_prof.ev[s.b]);
    float ms = 0.f;
    if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, g_prof.ev[s.a], g_prof.ev[s.b]);
    if (e != cudaSuccess) return fail(GLOM_B200_ERR_CUDA, "profile events: %s", cudaGetErrorString(e));
    if (s.kind >= kinds) continue;              // a caller built against an older header
    ms_by_kind[s.kind] += ms;
    launches_by_kind[s.kind] += 1;
  }
  g_prof.spans.clear();
  g_prof.used = 0;
  return 0;
}

}  // extern "C"
