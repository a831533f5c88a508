// Internal engine declarations shared by the C-ABI translation unit and the kernel files.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdarg.h>
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>
#include <mutex>
#include <vector>

#include "../../include/glom_b200.h"

namespace glom {

// Optional per-kernel CUDA-event timing (bench.py's roofline numbers).  Events are recorded on the
// launch stream around each kernel; nothing is synchronised until the caller reads them.
enum ProfKind { PROF_ATTN = 0, PROF_GEMM1 = 1, PROF_GEMM2 = 2, PROF_PREP = 3, PROF_TOKENIZE = 4, PROF_KINDS = 5 };
struct Profiler {
  bool enabled = false;
  std::vector<cudaEvent_t> ev;
  size_t used = 0;
  struct Span { int kind; size_t a, b; };
  std::vector<Span> spans;
  size_t mark(cudaStream_t st) {
    if (used == ev.size()) { cudaEvent_t e; cudaEventCreate(&e); ev.push_back(e); }
    cudaEventRecord(ev[used], st);
    return used++;
  }
};
struct ProfScope {   // RAII: events around one launch when profiling is on
  Profiler* p; int kind; cudaStream_t st; size_t a;
  ProfScope(Profiler* p_, int kind_, cudaStream_t st_) : p(p_ && p_->enabled ? p_ : nullptr), kind(kind_), st(st_), a(0) {
    if (p) a = p->mark(st);
  }
  ~ProfScope() { if (p) { const size_t b = p->mark(st); p->spans.push_back({kind, a, b}); } }
};

struct Geometry {
  int d, L, n, B;
  int rows;        // B * n   (columns of the batch = GEMM M)
  int G;           // 2L - 1  MLP groups, ordered bu_0, td_0, bu_1, td_1, ..., bu_{L-1}
  int hidden;      // 4d
  int attend_self, mask_side, mask_d2_max;
  int bn2;         // N tile of the second GEMM: 256 / 128 / 64 (largest dividing d)
  int part_w;      // columns covered by one squared-norm partial (one epilogue warp group)
  int nparts;      // squared-norm partials per (row, level) = d / part_w
};

// ---- packed weights -------------------------------------------------------------------------
// bf16 engine:  W1p [(G*4d) x d] bf16 | W2p [(L*d) x 8d] bf16 | b1p [G*4d] f32 | b2p [L*d] f32
// fp32 engine:  same shapes, all f32.
struct PackedLayout {
  size_t w1_off, w2_off, b1_off, b2_off, total;
};
PackedLayout packed_layout(int d, int L, int precision);

// ---- workspace ------------------------------------------------------------------------------
struct WorkspaceLayout {
  size_t s32_off;      // one fp32 state slab (ping-pong partner of state_out); 0 bytes if return_all
  size_t s32_bytes;
  size_t sb_off[2];    // bf16 shadow of the state           (rows, L, d)
  size_t sp_off[2];    // bf16 shadow of state[:, :, 1:] + pos (rows, L-1, d)
  size_t xb_off;       // bf16 tokens                        (rows, d)
  size_t h_off;        // hidden activations: bf16 engine = 16 KB blocks [G][rows/128][4d/64][128][64]; f32 = (rows, G*4d)
  size_t h_bytes;
  size_t c_off;        // consensus output                   (rows, L, d)   bf16 | f32
  size_t c_bytes;
  size_t nsq_off[2];   // squared-norm partials              (rows, L, nparts) f32
  size_t nsq_bytes;
  size_t attn_acc_off; // bf16 engine, n > 576 columns: fp32 output / (stabiliser, row sum) carried between the consensus kernel's key passes
  size_t attn_acc_bytes;
  size_t total;
};
WorkspaceLayout workspace_layout(const Geometry& g, int precision, int iters, int return_all);

// Glom.settle and the per-image step counts of glom_b200_forward_steps (bf16 engine): the forward workspace for
// (max_iters, return_all; settle: return_all = 0), followed by
struct SettleLayout {
  WorkspaceLayout fwd;
  size_t dsq_off;          // squared-change partials            (rows, L, nparts) f32
  size_t flags_off;        // zeroed at the start of a call:
  size_t frozen_off;       //   [B] int            1: the image has stopped
  size_t block_frozen_off; //   [ceil(rows/256)]   1: every row of the 256-row block belongs to a stopped image
  size_t done_off;         //   [1] unsigned       blocks of the convergence kernel that have finished
  size_t level_q_off;      //   [B * L] f32        the convergence kernel's per-(image, level) ratios
  size_t flags_bytes;
  size_t total;
};
SettleLayout settle_layout(const Geometry& g, int max_iters, int return_all = 0);

// Glom.settle_queue and Glom.settle_video (bf16 engine): B = slots.  The settle workspace for (slots, max_iters), whose
// fp32 slab is slab 0 of the two private slabs that hold S_t of the slots (slab t & 1), followed by slab 1 and the
// per-slot queue state.  settle_video's images are its frames, stream-major: image i = stream * frames + frame.
struct QueueLayout {
  SettleLayout settle;
  size_t slab_off[2];      // (B, n, L, d) f32 each
  size_t queue_off;        // initialised by glom_b200_settle_queue_begin / glom_b200_settle_video_begin:
  size_t slot_img_off;     //   [B] int   image in the slot, -1: none
  size_t age_off;          //   [B] int   steps the slot's image has run
  size_t pending_off;      //   [B] int   1: the image stopped; its final state waits in the slab for the next fill
  size_t gather_off;       //   [B] int   this step's fill hands the slot's final state to this image, -1: none
  size_t fresh_off;        //   [B] int   1: the slot admitted an image at this step
  size_t block_fresh_off;  //   [ceil(rows/256)] int   1: the block holds a slot admitted at this step
  size_t head_off;         //   [1] int   next queued stream (settle_queue: image)
  size_t unfinished_off;   //   [1] int   images queued or in flight
  size_t queue_bytes;
  size_t total;
};
QueueLayout queue_layout(const Geometry& g, int max_iters);

// device pointers into the queue state (QueueLayout), images = N (settle_video: streams * frames); frames = 1 for
// settle_queue; all NULL for Glom.settle
struct QueueSlots {
  int *slot_img, *age, *pending, *gather_img, *fresh, *block_fresh, *head, *unfinished;
  int images, frames, max_iters;
};

// ---- launchers (all asynchronous on the context's stream; -> 0 or the GLOM_B200_ERR_* code of the failure) -----------
struct Bf16Buffers {
  const float* s32_in;  float* s32_out;              // fp32 master state of step t / t+1
  int s32_in_bcast;                                   // 1: s32_in is init_levels (L, d) broadcast over the rows (step 0, no carried state)
  const __nv_bfloat16* sb_in;  __nv_bfloat16* sb_out;
  const __nv_bfloat16* sp_in;  __nv_bfloat16* sp_out;
  const __nv_bfloat16* xb;
  __nv_bfloat16* h;  __nv_bfloat16* c;
  float* attn_acc;                                    // n > 576 columns only: (rows, L, d) + (rows, L, 2) fp32 carried between key passes
  const float* nsq_in;  float* nsq_out;
  const float* pos;                                   // (n, d) fp32
  const __nv_bfloat16* w1;  const __nv_bfloat16* w2;  const float* b1;  const float* b2;
  // Glom.settle only (NULL for a forward): the step skips stopped images (SETTLE kernel instantiations)
  const int* frozen;                                  // [B] 1: the image has stopped
  const int* block_frozen;                            // [ceil(rows / 256)] 1: all rows of the block belong to stopped images
  float* dsq_out;                                     // (rows, L, nparts) squared-change partials |S_{t+1} - S_t|^2
  // Glom.settle_queue only (NULL otherwise): [ceil(rows / 256)] 1 = the block holds a slot admitted at this step; K1 then
  // runs MLP group 0 at every step, for these blocks only
  const int* block_fresh;
  // 1: a forward from init_levels at a step t < L (DESIGN.md, "Image-independent levels"): the work whose inputs are the
  // same in every image runs for the representative rows only
  int ii_reduce;
};

// The representative rows of image-independent work: the first lcm(n, 128) rows, whole images and whole 128-row H blocks,
// so 128-row block k holds the patches of block k % rep_h_blocks(n).  rep_row_blocks: the 256-row GEMM blocks covering them
static inline int rep_h_blocks(int n) {
  int a = n, b = 128;
  while (b) { const int r = a % b; a = b; b = r; }
  return n / a;
}
static inline int rep_row_blocks(int n) { return (rep_h_blocks(n) * 128 + 255) / 256; }

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// What every host-side launcher needs besides its own operands (the tensor-map encoder, the SM count to plan for, the
// stream, the optional profiler) and what it reports back: the launches it enqueued and the text of its failure.
struct Launch {
  EncodeTiledFn enc; int num_sms; cudaStream_t st; Profiler* prof;
  int launches;                 // kernels / async copies enqueued through this context
  char err[400];                // text of the failure
  // A kernel (or a counted async copy) was enqueued and the runtime answered `e`: count it, then as check()
  int launched(cudaError_t e, const char* what = nullptr) { ++launches; return check(e, what); }
  int launched(const char* what = nullptr) { return launched(cudaGetLastError(), what); }     // after kernel<<<...>>>
  // A runtime call that is no launch.  Failure -> GLOM_B200_ERR_CUDA, err = "[<what>: ]<the runtime's text>"
  int check(cudaError_t e, const char* what = nullptr) {
    if (e == cudaSuccess) return 0;
    return what ? fail(GLOM_B200_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e)) : fail(GLOM_B200_ERR_CUDA, "%s", cudaGetErrorString(e));
  }
  // -> code (GLOM_B200_ERR_INVALID: a shape the kernels do not support), err = the message.  The arguments may quote err
  // itself, to put a context in front of a callee's message
  int fail(int code, const char* fmt, ...) {
    char msg[sizeof(err)];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(msg, sizeof(msg), fmt, ap);
    va_end(ap);
    snprintf(err, sizeof(err), "%s", msg);
    return code;
  }
};
#define GLOM_TRY(x) do { if (const int r_ = (x)) return r_; } while (0)

// state prologue: S_0 -> fp32 master copy (dst may equal src => skipped), bf16 shadows, norms, bf16 tokens
int launch_prep(const Geometry& g, const float* state_in, const float* init_levels, const float* pos, const float* tokens,
                float* s32_dst, __nv_bfloat16* sb, __nv_bfloat16* sp, __nv_bfloat16* xb, float* nsq, Launch& ln);

// one Jacobi step on tensor cores, three launches: GEMM1+GELU -> H ; consensus -> C ; GEMM2+combine -> state t+1.
// step_index: position of the step inside the forward call.  The bottom-up net of level 0 reads the tokens, which do not
// change during a call (glom_pytorch.py:132-134), so its hidden activations (MLP group 0 of H) are computed by step 0 only
// and re-read by GEMM2 of the later steps.
int step_bf16(const Geometry& g, const Bf16Buffers& b, int step_index, Launch& ln);

// Glom.settle (settle_kernels.cu): the stopping rule after step `step` (one launch), and the copy of the stopped images
// whose final state is in the workspace slab into state_out (after the last step)
// settle queue (q != NULL): the rule is applied per running slot, which stops when it holds or its image has run
// q->max_iters steps; steps[image] = the image's step count
int launch_settle_converge(const Geometry& g, int step, float tol, const float* dsq, const float* nsq, int* frozen,
                           int* block_frozen, unsigned int* done, float* level_q, int32_t* steps, Launch& ln,
                           const QueueSlots* q = nullptr);
// Glom.settle_queue / Glom.settle_video (settle_kernels.cu).  init: the queue state of a new call (every slot empty, all
// images queued).  schedule, before step t: each finished or empty slot, in slot order, hands its stopped image over to
// the fill and, when `admit`, takes the next frame of its stream (settle_video) or else, while the queue is not empty,
// frame 0 of the next queued stream (settle_queue: the next queued image); writes frozen / block_frozen / block_fresh.
// fill, after the schedule: the handed-over images' final states from slab (S_t of the slots) into state_out, then S_0
// of each admitted image into slab (a continuing stream's S_0 is already there), its bf16 shadows sb / sp and norm
// partials nsq, and its bf16 token rows xb.
int launch_queue_init(const Geometry& g, const QueueSlots& q, int* frozen, int* block_frozen, unsigned int* done, Launch& ln);
int launch_queue_schedule(const Geometry& g, const QueueSlots& q, int admit, int* frozen, int* block_frozen, Launch& ln);
int launch_queue_fill(const Geometry& g, const QueueSlots& q, const float* tokens, const float* pos, const float* state_in,
                      const float* init_levels, float* state_out, float* slab, __nv_bfloat16* sb, __nv_bfloat16* sp,
                      float* nsq, __nv_bfloat16* xb, Launch& ln);
// s0 (nullable): where S_0 is when no step materialised it (the carried state, or init_levels broadcast if s0_bcast);
// images with steps[b] == 0 are copied from there
int launch_settle_gather(const Geometry& g, int max_iters, const int32_t* steps, const float* slab, float* state_out,
                         const float* s0, int s0_bcast, Launch& ln);
// glom_b200_forward_steps (settle_kernels.cu): the flags of step t from the given step counts (clamped to [0, max_steps]),
// one launch before every step; and, for return_all, the copy of slab steps[b] of each image into its slabs
// steps[b]+1 .. max_steps (after the last step)
int launch_steps_schedule(const Geometry& g, int t, int max_steps, const int32_t* steps, int* frozen, int* block_frozen,
                          Launch& ln);
int launch_steps_fill(const Geometry& g, int max_steps, const int32_t* steps, float* states, Launch& ln);
// return_all of a forward whose steps 0 .. L-2 ran image-independent levels for the representative rows only: level l >= s
// of slab s (1 <= s <= L-1) is copied from row r mod n into every row r >= n
int launch_level_fill(const Geometry& g, float* states, Launch& ln);

// fp32 consensus (attn_f32_kernel): a block of 16 queries keeps their rows (16 x dim) and logits (16 x n) as fp32 in
// shared memory, within the 227 KB a block may opt in to: dim + n <= 3632
constexpr int kAttnF32Queries = 16;
constexpr int kAttnF32MaxDimPlusN = (int)((227 * 1024) / (kAttnF32Queries * sizeof(float)));

struct F32Buffers {
  const float* s_in;  float* s_out;
  const float* x;  const float* pos;
  float* h;  float* c;
  const float* w1;  const float* w2;  const float* b1;  const float* b2;
};
int step_f32(const Geometry& g, const F32Buffers& b, Launch& ln);
int launch_broadcast_init(const Geometry& g, const float* state_in, const float* init_levels, float* dst, Launch& ln);

int launch_pack(int d, int L, int precision, const float* bu_w1, const float* bu_b1, const float* bu_w2, const float* bu_b2,
                const float* td_w1, const float* td_b1, const float* td_w2, const float* td_b2, void* packed, Launch& ln);

int launch_tokenize(const float* img, const float* w, const float* bias, float* tokens, int B, int H, int W, int p, int d,
                    Launch& ln);

// island analytics on state slabs (islands.cu)
int launch_islands(const float* states, int slabs, int side_h, int side_w, int L, int d, float threshold, float* cos_right,
                   float* cos_down, float* agreement, int* labels, int* num_islands, Launch& ln);
// part-whole trees over island labels (island_tree.cu); states == NULL: no embedding kernel
int launch_island_tree(const int* labels, const float* states, int slabs, int n, int L, int d, int* size, int* parent,
                       float* containment, float* nested, float* embedding, float* member_cos, float* coherence,
                       Launch& ln);
// island tracks through time over island labels (island_track.cu); labels (outer, times, inner, L, n)
int launch_island_track(const int* labels, int outer, int times, int inner, int n, int L, int* prev, int* overlap,
                        int* next, int* track, Launch& ln);

cudaError_t launch_clock_probe(unsigned long long* out, unsigned long long spin_ns, cudaStream_t st);
// (cycles, ns) sampled INSIDE the tensor-core kernels since the last reset, by ProfKind (tc_kernels.cu)
cudaError_t tc_kernel_clocks(unsigned long long* out /* [PROF_KINDS][8] */, bool reset);

// bf16 tokeniser: patchify + cast (CUDA cores), then the wgmma GEMM
int launch_patchify_bf16(const float* img, const float* w, __nv_bfloat16* patches, __nv_bfloat16* wtok, int B, int H, int W,
                         int p, int d, int kp, Launch& ln);
int tokenize_tc(const __nv_bfloat16* patches, const __nv_bfloat16* wtok, const float* bias, float* tokens, int rows,
                int d, int kp, Launch& ln);

// ---- backward (fp32, CUDA cores; bwd_kernels.cu) ---------------------------------------------------------
struct BackwardArgs {
  const float* tokens;   // (R, d)
  const float* pos;      // (n, d)
  const float* states;   // (T+1, R, L, d): S_0 .. S_T of the forward
  const float* grad_out; // (T+1, R, L, d) if grad_all else (R, L, d): dL/d(returned tensor)
  const float *bu_w1, *bu_b1, *bu_w2, *td_w1, *td_b1, *td_w2;   // reference layout, fp32 (second biases are not needed)
  // outputs, ACCUMULATED into (caller zero-initialises); d_state0 / d_init: exactly one is non-NULL
  float *d_tokens, *d_pos, *d_state0, *d_init;
  float *d_bu_w1, *d_bu_b1, *d_bu_w2, *d_bu_b2, *d_td_w1, *d_td_b1, *d_td_w2, *d_td_b2;
  // 1: every reduction runs in an order fixed by the shapes (no floating-point atomics): bit-reproducible gradients
  int deterministic;
  // Implicit gradients through settle (backward_implicit_run), all 0 for every other backward.  They apply to a one-step
  // call (iters = 1) at a state whose linearisation may already sit in the workspace:
  //   state_only: only dL/dS_t is wanted; no weight / bias / token / pos gradient is computed (the tensor-core DX still
  //               writes its token / pos rows, so d_tokens / d_pos must point at scratch)
  //   relin:      the workspace already holds everything of this state and these weights that does not depend on the
  //               cotangent (packed weights, bf16 tokens and shadows, BW_PRE's pre / h, khat / rnorm / khat_b, A / a_b)
  //               from an earlier call with relin = 0 and the same state: those stages are skipped
  //   skip_attn:  the consensus backward (it has no parameters) is skipped: dL/dS_t is incomplete
  int state_only, relin, skip_attn;
};
struct BackwardLayout {
  size_t g_off, gs_off, ds_off, khat_off, dkhat_off, rnorm_off, pre_off, h_off, dh_off, xp_off, dx_off, attn_off,
      dattn_off;
  // bf16 (tensor-core) MLP backward only
  size_t xb_off, sb_off, sp_off, gsb_off, w1p_off, w2t_off, w1t_off, b1p_off, bpre_off, bh_off, bdpre_off;
  size_t b1part_off;     // deterministic backward: BW_DH's bias partials (normally inside the unused fp32 pre / h / dh)
  size_t khatb_off, ab_off, dsimb_off;     // bf16 khat (state-like), probabilities and scaled dsim (Z, n, n)
  size_t blocked_bytes;
  size_t total;
};
// tensor-core MLP backward (tc_bwd_kernels.cu)
struct MlpBwdTc {
  const __nv_bfloat16 *xb, *sb, *sp, *gsb;      // bf16 shadows: tokens, S_t, S_t[:,1:]+pos, dL/dS_{t+1}/c
  const __nv_bfloat16 *w1p, *w2t, *w1t;        // (G*4d, d), (G*4d, d) = W2^T, (G*d, 4d) = W1^T, groups interleaved bu/td
  const float* b1p;                            // (G*4d)
  __nv_bfloat16 *pre, *h, *dpre;               // blocked (G, R_pad/128, 4d/64, 128, 64)
  float *ds, *d_tokens, *d_pos;                // input gradients of the groups are reduced straight into these:
                                               // dL/dS_t (R, L, d), dL/dtokens (R, d), dL/dpos (n, d)
  float *d_bu_w1, *d_bu_w2, *d_td_w1, *d_td_w2;
  float *d_bu_b1, *d_td_b1;                    // first-layer bias gradients, reduced in the DH epilogue
  // per-image step counts (glom_b200_backward_steps; NULL = every image runs every step): rows of images with
  // steps[b] <= t have gs = 0 at reverse step t, so row blocks made only of such rows are skipped
  const int32_t* steps;
  int t;
  // deterministic (1): no atomics.  DX stores the top-down groups' dx into dx_td (R, L-1, d) and DH the 32-row column
  // sums of dpre into b1_part [G][ceil(R/32)][4d]; the caller reduces both afterwards (backward_run)
  int deterministic;
  float *dx_td, *b1_part;
  // implicit gradients (BackwardArgs::relin / state_only): skip BW_PRE (pre / h already hold this state's), skip BW_DW
  int skip_pre, skip_dw;
};
int mlp_backward_tc(const Geometry& g, const MlpBwdTc& a, Launch& ln);

// One operand of the batched attention-backward GEMM: src is state-like (bf16 (B*n, L*d)) or attention-like (bf16
// (Z, n, n)); mn: see BwdParams
struct AttnBwdOperand { const void* src; int state, mn; };
// (a2 / b2: a second product accumulated into the same output tile, see tc_bwd_kernels.cu; a2.src == NULL: none)
// steps (nullable): the problems of images with steps[b] <= t are skipped and their output is left as it was
int attn_bwd_gemm_tc(const Geometry& g, AttnBwdOperand a, AttnBwdOperand b, int N, int K, int out_kind, float* out,
                     const int32_t* steps, int t, Launch& ln, AttnBwdOperand a2 = {}, AttnBwdOperand b2 = {});

BackwardLayout backward_layout(const Geometry& g, int precision);
// tokeniser backward (fp32, CUDA cores; bwd_kernels.cu): any of d_weight / d_bias / d_img may be NULL; all ACCUMULATED into
size_t tokenize_backward_workspace_bytes(int B, int H, int W, int p, int need_dimg);
// deterministic: d_bias by a fixed-order column sum instead of atomics (d_weight / d_img have no atomics)
int tokenize_backward(const float* img, const float* weight, const float* d_tokens, float* d_weight, float* d_bias,
                      float* d_img, int B, int H, int W, int p, int d, void* workspace, Launch& ln, int deterministic = 0);
// steps (nullable, device memory): per-image step counts; image b is the identity at every reverse step t >= steps[b]
int backward_run(const Geometry& g, const BackwardArgs& a, int precision, int iters, int grad_all, const int32_t* steps,
                 void* workspace, Launch& ln);

// Implicit gradients through settle (glom_b200_backward_implicit, bf16 engine): the backward workspace, followed by
struct ImplicitLayout {
  BackwardLayout bwd;
  size_t u_off;            // (rows, L, d) f32   the adjoint u
  size_t dsq_off;          // (rows, L, nparts) f32   |u_k - u_{k-1}|^2 partials
  size_t nsq_off;          // (rows, L, nparts) f32   |u_k|^2 partials
  size_t dtok_off;         // (rows, d) f32   token gradients of the adjoint passes (discarded)
  size_t dpos_off;         // (n, d) f32      pos gradients of the adjoint passes (discarded)
  size_t flags_off;        // zeroed at the start of a call:
  size_t frozen_off;       //   [B] int            1: the image's adjoint has stopped
  size_t block_frozen_off; //   [ceil(rows/256)]   (written by the convergence kernel, unused here)
  size_t done_off;         //   [1] unsigned       blocks of the convergence kernel that have finished
  size_t level_q_off;      //   [B * L] f32        the per-(image, level) ratios of each image's last adjoint pass
  size_t stop_off;         //   [B] int32          the backward's skip vector: 0 = stopped, 1 = running (step t = 0)
  size_t flags_bytes;
  size_t total;
};
ImplicitLayout implicit_layout(const Geometry& g);
// u_0 = grad_out; u_k = grad_out + J^T u_{k-1} at `state` for the running images, each stopped by settle's rule on u
// (adjoint_tol) or after adjoint_iters passes; then one VJP at `state` with cotangent u_K into the gradients of `a`
// (a.states = state, a.grad_out = grad_out; d_state0 / d_init NULL).  adjoint_steps (B) and adjoint_q (B, L, nullable)
// receive K_b and the last pass's ratios
int backward_implicit_run(const Geometry& g, const BackwardArgs& a, int adjoint_iters, float adjoint_tol,
                          int32_t* adjoint_steps, float* adjoint_q, void* workspace, Launch& ln);

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is per device and per function: remember, per device, the
// largest size already configured for one kernel (one instance of this per kernel template instantiation).
struct SmemOptIn {
  size_t configured[64] = {};
  std::mutex mu;
  template <typename K>
  cudaError_t ensure(K kernel, size_t bytes) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
    std::lock_guard<std::mutex> lk(mu);
    if (bytes <= configured[dev]) return cudaSuccess;
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e == cudaSuccess) configured[dev] = bytes;
    return e;
  }
};

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// glom_b200_set_sm_count_target (glom_api.cu): plan launches for at most this many SMs; 0 = the device's own count
extern std::atomic<int> g_sm_count_target;

// `device_sms` bounded by the SM-count target
static inline int planned_sms(int device_sms) {
  const int t = g_sm_count_target.load(std::memory_order_relaxed);
  return (t > 0 && t < device_sms) ? t : device_sms;
}

// SM count of the current device (bounded by the SM-count target): grid caps of the grid-stride CUDA-core kernels are a
// few waves of it
static inline int sm_count() {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n < 1)
    n = 132;
  return planned_sms(n);
}

}  // namespace glom
