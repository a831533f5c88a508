/*
 * glom_b200.h -- C ABI of the H100-native (sm_90a) GLOM column-update engine (libglom_b200.so).
 *
 * The reference (lucidrains/glom-pytorch) has no FFI: its hot path is the Python loop
 * glom_pytorch/glom_pytorch.py:131-145 calling GroupedFeedForward (:23-36) and
 * ConsensusAttention (:38-73).  This header is the boundary a maintainer would bind
 * instead of that loop (ctypes stub in INTEGRATION.md).  Conventions:
 *
 *   - plain C symbols, POD structs with a leading struct_size, no torch types;
 *   - every pointer is a DEVICE pointer owned by the caller (PyTorch's allocator);
 *     the library never allocates device memory, never synchronises the stream and
 *     never throws: 0 on success, a negative glom_b200_status otherwise, text via
 *     glom_b200_last_error() (thread-local);
 *   - all work is enqueued on `stream` (a cudaStream_t passed as void*) of the CURRENT
 *     device (caller does cudaSetDevice / torch.cuda.device);
 *   - state layout is the reference's: (B, n, L, d) contiguous, d fastest, fp32
 *     (the reference carries the state in fp32 even under autocast, SURVEY 5.1).
 */
#ifndef GLOM_B200_H_
#define GLOM_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GLOM_B200_ABI_VERSION 1

#if defined(__GNUC__)
#define GLOM_B200_API __attribute__((visibility("default")))
#else
#define GLOM_B200_API
#endif

typedef enum glom_b200_status {
  GLOM_B200_OK = 0,
  GLOM_B200_ERR_INVALID = -1,     /* bad argument / unsupported shape              */
  GLOM_B200_ERR_WORKSPACE = -2,   /* workspace or packed buffer too small          */
  GLOM_B200_ERR_CUDA = -3,        /* a CUDA runtime/driver call failed             */
  GLOM_B200_ERR_DEVICE = -4       /* device is not compute capability 9.x, sm_90a (no CPU / other-arch fallback) */
} glom_b200_status;

typedef enum glom_b200_precision {
  GLOM_B200_FP32 = 0,  /* CUDA-core fp32 path: matches the reference's fp32 forward     */
  GLOM_B200_BF16 = 1   /* wgmma tensor-core path: bf16 operands, fp32 accumulate, fp32 state --
                          the arithmetic of the reference under torch.autocast(bf16)     */
} glom_b200_precision;

/* Static description of one Glom module + one call geometry.
 * Mirrors Glom.__init__ kwargs (glom_pytorch.py:78-87) and ConsensusAttention (:39-54). */
typedef struct glom_b200_cfg {
  uint32_t struct_size;   /* = sizeof(glom_b200_cfg)                                     */
  int32_t dim;            /* d                                                           */
  int32_t levels;         /* L  (>= 2: the reference cannot build top_down for L == 1)    */
  int32_t n;              /* columns (patches) of THIS call, n <= num_patches (:115)     */
  int32_t attend_self;    /* consensus_self (:85); 0 => diagonal logit := -5e-4 (:11)    */
  int32_t mask_side;      /* patches per grid row for the radius mask; 0 => no mask      */
  int32_t mask_d2_max;    /* logits with (dh^2+dw^2) > mask_d2_max are masked (:44-54,
                             :67-69).  The host derives it from non_local_mask.          */
  int32_t precision;      /* glom_b200_precision                                         */
} glom_b200_cfg;

/* Device pointers to the reference's parameters in state_dict layout (fp32, contiguous):
 *   bottom_up.net.1.weight (L*4d, d, 1)   .bias (L*4d)      glom_pytorch.py:29
 *   bottom_up.net.3.weight (L*d, 4d, 1)   .bias (L*d)       glom_pytorch.py:31
 *   top_down.*  same with L-1 groups                         glom_pytorch.py:105   */
typedef struct glom_b200_weights_ref {
  uint32_t struct_size;
  const float* bu_w1; const float* bu_b1; const float* bu_w2; const float* bu_b2;
  const float* td_w1; const float* td_b1; const float* td_w2; const float* td_b2;
} glom_b200_weights_ref;

GLOM_B200_API int glom_b200_abi_version(void);

/* Thread-local text of the last error returned on this thread ("" if none). */
GLOM_B200_API const char* glom_b200_last_error(void);

/* Bytes of the packed-weight buffer for cfg (depends on dim, levels, precision). */
GLOM_B200_API int glom_b200_packed_weight_bytes(const glom_b200_cfg* cfg, size_t* out_bytes);

/* Repack the reference-layout MLP weights into the engine layout (per level: W1 rows of
 * bottom-up and top-down interleaved, W2 K-concatenated [bu | td], biases summed where the
 * combine adds them).  Replaces nothing in the reference: it is the one-time cost of
 * swapping GroupedFeedForward's Conv1d weights (:29, :31) for GEMM operands. */
GLOM_B200_API int glom_b200_pack_weights(const glom_b200_cfg* cfg, const glom_b200_weights_ref* w,
                           void* packed, size_t packed_bytes, void* stream);

/* Workspace bytes glom_b200_forward needs for (cfg, batch, iters, return_all). */
GLOM_B200_API int glom_b200_workspace_bytes(const glom_b200_cfg* cfg, int batch, int iters,
                              int return_all, size_t* out_bytes);

/* The hot path: `iters` Jacobi column updates.  Replaces glom_pytorch.py:123-148
 * (state init/carry, the loop :131-145, hiddens/return_all :147-148).
 *
 *   tokens      (B, n, d) fp32   image_to_tokens(img)                     (:114)
 *   pos         (n, d)    fp32   pos_emb.weight[:n]                       (:117)
 *   state_in    (B, n, L, d) fp32 contiguous, or NULL                     (:123)
 *   init_levels (L, d)    fp32   used (broadcast) when state_in == NULL   (:124)
 *   state_out   return_all ? (iters+1, B, n, L, d) : (B, n, L, d), fp32; slab 0 of the
 *               return_all form is S_0 (:126).  Must not alias state_in.
 */
GLOM_B200_API int glom_b200_forward(const glom_b200_cfg* cfg, const void* packed_weights,
                      const float* tokens, const float* pos, const float* state_in,
                      const float* init_levels, float* state_out, int batch, int iters,
                      int return_all, void* workspace, size_t workspace_bytes, void* stream);

/* Cross-call persistence.  Same as
 * glom_b200_forward with a carried-in state, for the case that `state_in` is bit for bit the FINAL state the previous
 * glom_b200_forward / _forward_resume call on this workspace wrote (same cfg, batch, and `pos`): the workspace then still
 * holds that state's bf16 shadows and norm partials in shadow buffer `shadow_parity` (0 after a plain forward with an even
 * number of steps, 1 after an odd one; in general what the previous _resume call returned), so the state prologue is
 * skipped and step 0 reads the fp32 master straight from `state_in`.  bf16 engine, iters >= 1.  *out_shadow_parity = the
 * buffer holding the new final state's shadows.  Passing a state that does not match the workspace gives wrong results;
 * the host side (glom.py) checks tensor identity and version before taking this path. */
GLOM_B200_API int glom_b200_forward_resume(const glom_b200_cfg* cfg, const void* packed_weights, const float* tokens,
                                           const float* pos, const float* state_in, float* state_out, int batch, int iters,
                                           int return_all, void* workspace, size_t workspace_bytes, void* stream,
                                           int shadow_parity, int* out_shadow_parity);

/* Inference until the columns settle (Glom.settle).  bf16 engine only.  Runs up to `max_iters` (>= 1) steps from the same
 * start as glom_b200_forward (state_in, or init_levels broadcast) and stops each image on its own, on the GPU and without
 * a host synchronisation.  After step k (k >= 1) image b has
 *   r_b(k) = max_l sqrt( sum_i |S_k[b,i,l] - S_{k-1}[b,i,l]|^2 / sum_i |S_k[b,i,l]|^2 )
 * (sums over the image's n columns, fp32, fixed order; 0/0 counts as 0, x/0 with x > 0 as inf).  The first k with
 * r_b(k) <= tol stops image b: state_out[b] = S_k and steps_out[b] = k.  An image that never meets it gets S_max_iters and
 * steps_out[b] = max_iters; a negative tol never stops an image.  state_out[b] is bit-identical to
 * glom_b200_forward(iters = steps_out[b]) on the same batch.
 *   state_out (B, n, L, d) fp32, must not alias state_in;  steps_out (B) int32, device memory, written on `stream`.
 * Later steps skip the stopped images' work (their launches stay enqueued).  NaN tol, max_iters < 1, precision fp32 and a
 * NULL steps_out are errors.  The workspace (1024-byte aligned) is the forward workspace for (batch, max_iters) plus the
 * stopping rule's partials and flags; a following glom_b200_forward_resume on it is not valid. */
GLOM_B200_API int glom_b200_settle_workspace_bytes(const glom_b200_cfg* cfg, int batch, int max_iters, size_t* out_bytes);
GLOM_B200_API int glom_b200_settle(const glom_b200_cfg* cfg, const void* packed_weights, const float* tokens, const float* pos,
                                   const float* state_in, const float* init_levels, float* state_out, int batch,
                                   int max_iters, float tol, int32_t* steps_out, void* workspace, size_t workspace_bytes,
                                   void* stream);
/* glom_b200_settle that keeps every state, for training through settle (its backward is glom_b200_backward_steps with
 * max_steps = max_iters and this call's steps_out) and for analysis of a settled run.  The stopping rule, steps_out and
 * the argument errors (reported before any device query) are those of glom_b200_settle.
 *   states_out (max_iters+1, B, n, L, d) fp32: slab t of image b is S_min(t, steps_out[b]), slab 0 is S_0 -- the
 *   return_all form of glom_b200_forward_steps.
 * The workspace (1024-byte aligned) is that of glom_b200_forward_steps(max_steps = max_iters, return_all = 1). */
GLOM_B200_API int glom_b200_settle_all_workspace_bytes(const glom_b200_cfg* cfg, int batch, int max_iters, size_t* out_bytes);
GLOM_B200_API int glom_b200_settle_all(const glom_b200_cfg* cfg, const void* packed_weights, const float* tokens,
                                       const float* pos, const float* state_in, const float* init_levels, float* states_out,
                                       int batch, int max_iters, float tol, int32_t* steps_out, void* workspace,
                                       size_t workspace_bytes, void* stream);

/* Per-image step counts.  bf16 engine only.  The forward of glom_b200_forward run for max_steps (>= 0) steps from the same
 * start (state_in, or init_levels broadcast), in which image b stops after steps[b] steps: its later steps skip its work
 * and store nothing.  steps (B) int32 is device memory, read on the device only; each entry is clamped on the device to
 * [0, max_steps].  With s_b = the clamped steps[b]:
 *   return_all = 0: state_out (B, n, L, d), state_out[b] = S_{s_b} of image b (S_0 when s_b == 0);
 *   return_all = 1: state_out (max_steps+1, B, n, L, d), slab t of image b = S_{min(t, s_b)}.
 * Image b's result is bit-identical to glom_b200_forward(iters = s_b, same return_all) on the same batch; each step is
 * the three-launch step.  The workspace (1024-byte aligned) is the forward workspace for (batch, max_steps, return_all)
 * plus the per-image and per-256-row-block flags; a following glom_b200_forward_resume on it is not valid.  Argument
 * errors (precision fp32, max_steps < 0, NULL steps) are reported before any device query. */
GLOM_B200_API int glom_b200_forward_steps_workspace_bytes(const glom_b200_cfg* cfg, int batch, int max_steps, int return_all,
                                                          size_t* out_bytes);
GLOM_B200_API int glom_b200_forward_steps(const glom_b200_cfg* cfg, const void* packed_weights, const float* tokens,
                                          const float* pos, const float* state_in, const float* init_levels, float* state_out,
                                          int batch, const int32_t* steps, int max_steps, int return_all, void* workspace,
                                          size_t workspace_bytes, void* stream);

/* A queue of images settled through fixed batch slots (Glom.settle_queue).  bf16 engine only.  `images` = N images run
 * through `slots` = B batch slots: each slot holds one image at a time and, on the step after its image stops, takes the
 * next queued image (open slots take queued images in slot order, so the assignment is deterministic).  Image i's result
 * is bit-identical to glom_b200_settle on the whole N-image batch with the same tol and max_iters: state_out[i] = S_k and
 * steps_out[i] = k, k the first step whose change criterion is <= tol, or max_iters.  The library never synchronises:
 * the caller loops on the host.
 *   tokens (N, n, d) fp32 (all images, tokenised up front);  pos (n, d);  state_in (N, n, L, d) or NULL with
 *   init_levels (L, d) broadcast;  state_out (N, n, L, d) fp32, must not alias state_in;  steps_out (N) int32 device.
 * _begin initialises the queue state in the workspace (every slot empty, all N images queued).  _run enqueues the global
 * steps first_step .. first_step + num_steps - 1 (first_step = the number of steps the earlier _run calls of this queue
 * enqueued), each a slot schedule, a slot fill (the final states of images that stopped at the previous step go to
 * state_out, S_0 of the admitted images into their slots), the three kernels of a settle step and the stopping rule;
 * then it copies the number of unfinished images (queued or in a slot) to *remaining_out (device int32, may be NULL).
 * When that count is 0, a _run with num_steps = 0 enqueues only the final hand-over of the images that stopped at the
 * last step; after it state_out and steps_out are complete.  A typical loop: begin; do { run(t, max_iters); t += max_iters;
 * read the count } while (count); run(t, 0).  Every call takes the same arguments.  Argument errors (precision fp32,
 * images < 1, slots < 1, max_iters < 1, NaN tol, NULL or misaligned steps_out) are reported before any device query.
 * The workspace (1024-byte aligned) depends on (slots, max_iters) only: the settle workspace of batch `slots`, a second
 * fp32 state slab and the per-slot queue state; a following glom_b200_forward_resume on it is not valid. */
GLOM_B200_API int glom_b200_settle_queue_workspace_bytes(const glom_b200_cfg* cfg, int slots, int max_iters, size_t* out_bytes);
GLOM_B200_API int glom_b200_settle_queue_begin(const glom_b200_cfg* cfg, const float* tokens, const float* pos,
                                               const float* state_in, const float* init_levels, float* state_out,
                                               int32_t* steps_out, int images, int slots, int max_iters, float tol,
                                               void* workspace, size_t workspace_bytes, void* stream);
GLOM_B200_API int glom_b200_settle_queue_run(const glom_b200_cfg* cfg, const void* packed_weights, const float* tokens,
                                             const float* pos, const float* state_in, const float* init_levels,
                                             float* state_out, int32_t* steps_out, int images, int slots, int max_iters,
                                             float tol, void* workspace, size_t workspace_bytes, void* stream, int first_step,
                                             int num_steps, int32_t* remaining_out);

/* Tokeniser, the step before the loop: replaces image_to_tokens
 * (glom_pytorch.py:94-97, call :114): patchify 'b c (h p1) (w p2) -> b (h w) (p1 p2 c)'
 * fused with the Linear(3*p*p -> d).
 *   img (B, 3, H, W) fp32;  weight (d, 3*p*p) fp32;  bias (d) fp32;  tokens (B, n, d) fp32
 * precision GLOM_B200_FP32: one CUDA-core fp32 kernel, no workspace.
 * precision GLOM_B200_BF16: gather + cast to a zero-padded bf16 operand, then a wgmma GEMM with
 *   fp32 accumulation (what autocast does to this Linear); needs the workspace below, 1024-aligned. */
GLOM_B200_API int glom_b200_tokenize_workspace_bytes(int batch, int height, int width, int patch,
                                                     int dim, int precision, size_t* out_bytes);
GLOM_B200_API int glom_b200_tokenize(const float* img, const float* weight, const float* bias,
                       float* tokens, int batch, int height, int width, int patch,
                       int dim, int precision, void* workspace, size_t workspace_bytes, void* stream);

/* Number of kernels the last glom_b200_forward / glom_b200_tokenize call on this thread
 * enqueued (bench.py reports it as gpu_launches). */
GLOM_B200_API int glom_b200_last_launch_count(void);

/* Diagnostics: byte offsets of intermediate buffers inside the workspace for the same
 * (cfg, batch, iters, return_all); tests use them to check single stages.
 * which: 0 = hidden activations H -- bf16 engine: 16 KB blocks [2L-1][ceil(rows/128)][4d/64][128][64]
 *            (group, 128-row block, 64-column block, row, column), fp32 engine: (rows, (2L-1)*4d);
 *        1 = consensus C (rows, L, d),
 *        2 = squared-norm partials. Returns GLOM_B200_ERR_INVALID for unknown ids. */
GLOM_B200_API int glom_b200_workspace_offset(const glom_b200_cfg* cfg, int batch, int iters, int return_all,
                               int which, size_t* out_offset, size_t* out_bytes);

/* Diagnostics: byte offsets of the settle buffers inside the workspace of glom_b200_settle (return_all = 0) or
 * glom_b200_settle_all (return_all = 1) for the same (cfg, batch, max_iters).  Each is 16-byte aligned and lies after
 * the forward layout, so H, C and the squared-norm partials are found with glom_b200_workspace_offset(iters = max_iters).
 * which: 0 = squared-change partials of the last step (rows, L, nparts) f32,
 *        1 = per-(image, level) ratios q (B, L) f32 of each image's last step,
 *        2 = frozen (B) int32, 1: the image met the stopping rule,
 *        3 = block_frozen (ceil(rows / 256)) int32, 1: every image with rows in the 256-row block is frozen.
 * Argument errors (those of glom_b200_settle_workspace_bytes, unknown ids) are reported before any device query. */
GLOM_B200_API int glom_b200_settle_workspace_offset(const glom_b200_cfg* cfg, int batch, int max_iters, int return_all,
                                                    int which, size_t* out_offset, size_t* out_bytes);

/* Backward of the column update: gradients of glom_b200_forward's loop
 * (glom_pytorch.py:123-148) with respect to tokens, pos, the initial state (or init_levels) and the
 * eight MLP tensors, given dL/d(output).  Per-step intermediates are recomputed from the saved states.  precision
 * GLOM_B200_BF16 with dim % 256 == 0: the MLP and consensus GEMMs of the reverse pass run on wgmma tensor cores (bf16
 * operands, fp32 accumulation), softmax / normalisation / bias reductions in fp32 on CUDA cores; otherwise everything
 * is fp32 on CUDA cores.  All d_* buffers are ACCUMULATED into (zero them first); weights and their
 * gradients use the reference's state_dict layout.
 *   states    (iters+1, B, n, L, d) fp32: S_0..S_T as returned by forward(return_all=1)
 *   grad_out  (iters+1, B, n, L, d) if grad_all else (B, n, L, d)
 *   d_state0  (B, n, L, d) or NULL;  d_init (L, d) or NULL  (the one matching how the forward was started) */
typedef struct glom_b200_grads {
  uint32_t struct_size;
  float* d_tokens; float* d_pos; float* d_state0; float* d_init;
  float* d_bu_w1; float* d_bu_b1; float* d_bu_w2; float* d_bu_b2;
  float* d_td_w1; float* d_td_b1; float* d_td_w2; float* d_td_b2;
} glom_b200_grads;
GLOM_B200_API int glom_b200_backward_workspace_bytes(const glom_b200_cfg* cfg, int batch, size_t* out_bytes);
GLOM_B200_API int glom_b200_backward(const glom_b200_cfg* cfg, const glom_b200_weights_ref* weights,
                       const float* tokens, const float* pos, const float* states, const float* grad_out,
                       const glom_b200_grads* grads, int batch, int iters, int grad_all,
                       void* workspace, size_t workspace_bytes, void* stream);
/* Backward of glom_b200_forward_steps(return_all = 1): the same as glom_b200_backward with iters = max_steps, for the
 * per-image program in which image b is the identity at every step t >= steps[b] (steps: the forward's (B) int32 device
 * array).  At such a step the image's upstream gradient passes through unchanged and it adds nothing to any parameter,
 * pos or token gradient; the MLP GEMMs of the tensor-core backward skip row blocks made only of such rows, and its
 * consensus-attention backward skips such images entirely.  `states` is the return_all output of forward_steps or
 * settle_all.  Same workspace as glom_b200_backward. */
GLOM_B200_API int glom_b200_backward_steps(const glom_b200_cfg* cfg, const glom_b200_weights_ref* weights,
                                           const float* tokens, const float* pos, const float* states, const float* grad_out,
                                           const glom_b200_grads* grads, int batch, const int32_t* steps, int max_steps,
                                           int grad_all, void* workspace, size_t workspace_bytes, void* stream);
/* glom_b200_backward (steps == NULL, iters = max_steps) or glom_b200_backward_steps (steps != NULL), with
 * deterministic = 1: bit-reproducible gradients.  No floating-point atomics run: every sum that the default path
 * accumulates with red.add / atomicAdd (the tensor-core MLP backward's dL/dS_t, dL/dpos and first-layer bias gradients,
 * the bias column sums, d_init) is computed in an order fixed by the shapes alone, independent of the grid and of the
 * SM count, so the same inputs give the same bits on every run on the same GPU model and build.  deterministic = 0 is
 * exactly the default entry points.  Same workspace as glom_b200_backward.  Argument errors (deterministic not 0 or 1,
 * misaligned steps, max_steps < 0, and those of glom_b200_backward) are reported before any device query. */
GLOM_B200_API int glom_b200_backward_ex(const glom_b200_cfg* cfg, const glom_b200_weights_ref* weights,
                                        const float* tokens, const float* pos, const float* states, const float* grad_out,
                                        const glom_b200_grads* grads, int batch, const int32_t* steps, int max_steps,
                                        int grad_all, int deterministic, void* workspace, size_t workspace_bytes,
                                        void* stream);

/* Backward of glom_b200_tokenize (image_to_tokens, glom_pytorch.py:94-97; SURVEY 8 rows f1 + f2), fp32 on CUDA cores:
 *   d_weight (dim, 3 patch^2) += d_tokens^T . patches,   d_bias (dim) += column sums of d_tokens,
 *   d_img (B, 3, H, W) += fold(d_tokens . weight).
 * Any of the three outputs may be NULL (skipped); they are ACCUMULATED into.  workspace: see _workspace_bytes
 * (need_d_img = whether d_img is requested). */
GLOM_B200_API int glom_b200_tokenize_backward_workspace_bytes(int batch, int height, int width, int patch, int need_d_img,
                                                              size_t* out_bytes);
GLOM_B200_API int glom_b200_tokenize_backward(const float* img, const float* weight, const float* d_tokens, float* d_weight,
                                              float* d_bias, float* d_img, int batch, int height, int width, int patch, int dim,
                                              void* workspace, size_t workspace_bytes, void* stream);
/* glom_b200_tokenize_backward with deterministic = 1: d_bias by a fixed-order column sum instead of atomics (d_weight
 * and d_img never use atomics), so all three are bit-reproducible.  deterministic must be 0 or 1 (checked before any
 * device query); same workspace. */
GLOM_B200_API int glom_b200_tokenize_backward_ex(const float* img, const float* weight, const float* d_tokens,
                                                 float* d_weight, float* d_bias, float* d_img, int batch, int height,
                                                 int width, int patch, int dim, int deterministic, void* workspace,
                                                 size_t workspace_bytes, void* stream);

/* Per-kernel device timing for the roofline report (bench.py).  Between _begin and _end every
 * kernel the forward/tokenize calls of THIS thread enqueue is bracketed by CUDA events on the
 * launch stream (no synchronisation is added to the calls).  _end waits for those events and
 * returns summed milliseconds and launch counts per kernel kind:
 *   0 consensus attention, 1 GEMM1+GELU, 2 GEMM2+combine, 3 state prologue, 4 tokeniser.
 * `kinds` is the capacity of both arrays (>= 5; kinds beyond the capacity are dropped). */
#define GLOM_B200_PROFILE_KINDS 5
GLOM_B200_API int glom_b200_profile_begin(void);
GLOM_B200_API int glom_b200_profile_end(double* ms_by_kind, int* launches_by_kind, int kinds);

/* Island analytics on column states.  states: `slabs` contiguous (side_h * side_w, levels, dim) fp32 state slabs, e.g. the (iters+1) * B slabs of
 * glom_b200_forward(return_all = 1).  Per (slab, level), on the patch grid (patch i = h * side_w + w):
 *   cos_right / cos_down (slabs, levels, n)  cosine similarity with the right / lower neighbour (0 where there is none)
 *   agreement            (slabs, levels, n)  mean cosine similarity with the existing 4-neighbours
 *   labels               (slabs, levels, n)  island id = smallest patch index of the 4-connected component in the graph
 *                                            of neighbour pairs with cosine similarity >= threshold
 *   num_islands          (slabs, levels)     number of such components
 * HBM-bound CUDA-core kernels (3 dot products per patch, no Gram matrix); all outputs device memory of the caller. */
GLOM_B200_API int glom_b200_islands(const float* states, int slabs, int side_h, int side_w, int levels, int dim, float threshold,
                                    float* cos_right, float* cos_down, float* agreement, int32_t* labels,
                                    int32_t* num_islands, void* stream);

/* Measurement aid (bench.py): one device thread spins for `spin_us` microseconds of %globaltimer and writes
 * {SM cycles elapsed, nanoseconds elapsed} to out_cycles_ns[0..1] (device memory, 16 bytes): cycles / ns is the SM
 * clock in GHz the device actually ran at when the probe executed.  Enqueued on `stream`; the caller synchronises. */
GLOM_B200_API int glom_b200_clock_probe(uint64_t* out_cycles_ns, int spin_us, void* stream);

/* Measurement aid (bench.py): the SM clock the tensor-core kernels ACTUALLY ran at.  One thread of block 0 of every
 * tensor-core kernel brackets the kernel's working phase with (clock64, %globaltimer); the deltas accumulate per kernel kind
 * (indices as in glom_b200_profile_end: 0 consensus, 1 GEMM1+GELU, 2 GEMM2+combine, 4 tokeniser GEMM).
 * Writes MHz (cycles per microsecond of in-kernel time) and the in-kernel milliseconds per kind since the last reset;
 * kinds without samples report 0.  wait_frac (may be NULL, else 6 doubles per kind): fractions of block 0's in-kernel
 * cycles in slots {0: GEMMs: consumer warp 0 waited for operands, 1: unused (0), 2: the TMA lane waited for a free ring
 * slot, 3: consensus: consumer warp 0 waited for operands, 4: GEMMs: consumer warp 0's epilogue work; consensus: its
 * softmax work, 5: consensus: its output work}; the accumulators live in the consumers' registers, so there is no
 * accumulator wait.  Filled by the diagnostic instantiations only
 * (environment variable GLOM_B200_WAIT_COUNTERS=1).
 * Synchronises the device; `reset` != 0 clears the accumulators. */
GLOM_B200_API int glom_b200_kernel_clocks(double* mhz_by_kind, double* ms_by_kind, double* wait_frac, int kinds, int reset);

#ifdef __cplusplus
}
#endif
#endif /* GLOM_B200_H_ */
