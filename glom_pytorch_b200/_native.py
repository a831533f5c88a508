"""ctypes binding of libglom_b200.so (include/glom_b200.h).  No torch types cross the ABI:
only raw device pointers, sizes and the stream handle.  There is no fallback: if the library
is missing or fails to load, importing the engine raises."""
import ctypes
import os

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("GLOM_B200_LIB") or os.path.join(_PKG, "libglom_b200.so")   # override: A/B timing of builds

ABI_VERSION = 1
PRECISION = {"fp32": 0, "bf16": 1}
PROFILE_KINDS = ("attention", "gemm1_gelu", "gemm2_combine", "prologue", "tokenize")


class Cfg(ctypes.Structure):
    _fields_ = [("struct_size", ctypes.c_uint32), ("dim", ctypes.c_int32), ("levels", ctypes.c_int32),
                ("n", ctypes.c_int32), ("attend_self", ctypes.c_int32), ("mask_side", ctypes.c_int32),
                ("mask_d2_max", ctypes.c_int32), ("precision", ctypes.c_int32)]


class WeightsRef(ctypes.Structure):
    _fields_ = [("struct_size", ctypes.c_uint32)] + [
        (k, ctypes.c_void_p) for k in ("bu_w1", "bu_b1", "bu_w2", "bu_b2", "td_w1", "td_b1", "td_w2", "td_b2")]


class Grads(ctypes.Structure):
    _fields_ = [("struct_size", ctypes.c_uint32)] + [
        (k, ctypes.c_void_p) for k in ("d_tokens", "d_pos", "d_state0", "d_init", "d_bu_w1", "d_bu_b1", "d_bu_w2",
                                       "d_bu_b2", "d_td_w1", "d_td_b1", "d_td_w2", "d_td_b2")]


_vp, _sz, _i32, _f32 = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_float
_CFG, _W, _G = ctypes.POINTER(Cfg), ctypes.POINTER(WeightsRef), ctypes.POINTER(Grads)
_SZP, _I32P = ctypes.POINTER(_sz), ctypes.POINTER(_i32)
_SETTLE = [_CFG, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _f32, _vp, _vp, _sz, _vp]

# every symbol of include/glom_b200.h: name -> (restype, argtypes)
SIGNATURES = {
    "glom_b200_abi_version": (_i32, []),
    "glom_b200_last_error": (ctypes.c_char_p, []),
    "glom_b200_packed_weight_bytes": (_i32, [_CFG, _SZP]),
    "glom_b200_pack_weights": (_i32, [_CFG, _W, _vp, _sz, _vp]),
    "glom_b200_workspace_bytes": (_i32, [_CFG, _i32, _i32, _i32, _SZP]),
    "glom_b200_forward": (_i32, [_CFG, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _vp, _sz, _vp]),
    "glom_b200_forward_resume": (_i32, [_CFG, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _vp, _sz, _vp, _i32, _I32P]),
    "glom_b200_settle_workspace_bytes": (_i32, [_CFG, _i32, _i32, _SZP]),
    "glom_b200_settle": (_i32, _SETTLE),
    "glom_b200_settle_all_workspace_bytes": (_i32, [_CFG, _i32, _i32, _SZP]),
    "glom_b200_settle_all": (_i32, _SETTLE),
    "glom_b200_settle_workspace_offset": (_i32, [_CFG, _i32, _i32, _i32, _i32, _SZP, _SZP]),
    "glom_b200_settle_queue_workspace_bytes": (_i32, [_CFG, _i32, _i32, _SZP]),
    "glom_b200_settle_queue_begin": (_i32, [_CFG, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _f32, _vp, _sz, _vp]),
    "glom_b200_settle_queue_run": (_i32, [_CFG, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _f32, _vp, _sz, _vp,
                                          _i32, _i32, _vp]),
    "glom_b200_settle_video_workspace_bytes": (_i32, [_CFG, _i32, _i32, _SZP]),
    "glom_b200_settle_video_begin": (_i32, [_CFG, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _f32, _vp, _sz,
                                            _vp]),
    "glom_b200_settle_video_run": (_i32, [_CFG, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _f32, _vp, _sz,
                                          _vp, _i32, _i32, _vp]),
    "glom_b200_forward_steps_workspace_bytes": (_i32, [_CFG, _i32, _i32, _i32, _SZP]),
    "glom_b200_forward_steps": (_i32, [_CFG, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _i32, _i32, _vp, _sz, _vp]),
    "glom_b200_tokenize_workspace_bytes": (_i32, [_i32, _i32, _i32, _i32, _i32, _i32, _SZP]),
    "glom_b200_tokenize": (_i32, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _sz, _vp]),
    "glom_b200_last_launch_count": (_i32, []),
    "glom_b200_workspace_offset": (_i32, [_CFG, _i32, _i32, _i32, _i32, _SZP, _SZP]),
    "glom_b200_backward_workspace_bytes": (_i32, [_CFG, _i32, _SZP]),
    "glom_b200_backward": (_i32, [_CFG, _W, _vp, _vp, _vp, _vp, _G, _i32, _i32, _i32, _vp, _sz, _vp]),
    "glom_b200_backward_steps": (_i32, [_CFG, _W, _vp, _vp, _vp, _vp, _G, _i32, _vp, _i32, _i32, _vp, _sz, _vp]),
    "glom_b200_backward_ex": (_i32, [_CFG, _W, _vp, _vp, _vp, _vp, _G, _i32, _vp, _i32, _i32, _i32, _vp, _sz, _vp]),
    "glom_b200_backward_implicit_workspace_bytes": (_i32, [_CFG, _i32, _SZP]),
    "glom_b200_backward_implicit": (_i32, [_CFG, _W, _vp, _vp, _vp, _vp, _G, _i32, _i32, _f32, _i32, _vp, _vp, _vp, _sz,
                                           _vp]),
    "glom_b200_tokenize_backward_workspace_bytes": (_i32, [_i32, _i32, _i32, _i32, _i32, _SZP]),
    "glom_b200_tokenize_backward": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp, _sz, _vp]),
    "glom_b200_tokenize_backward_ex": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _sz,
                                              _vp]),
    "glom_b200_profile_begin": (_i32, []),
    "glom_b200_profile_end": (_i32, [ctypes.POINTER(ctypes.c_double), _I32P, _i32]),
    "glom_b200_islands": (_i32, [_vp, _i32, _i32, _i32, _i32, _i32, _f32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "glom_b200_clock_probe": (_i32, [_vp, _i32, _vp]),
    "glom_b200_kernel_clocks": (_i32, [_vp, _vp, _vp, _i32, _i32]),
    "glom_b200_set_sm_count_target": (_i32, [_i32]),
}
EXPORTS = tuple(SIGNATURES)


class GlomB200Error(RuntimeError):
    pass


_lib = None


def load():
    """Load the shared library once; raise (never fall back) if it is absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise GlomB200Error(
            f"{LIB_PATH} not found: build it with `python -m glom_pytorch_b200.build` "
            "(nvcc, sm_90a). There is no CPU or PyTorch fallback for the GLOM column update.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes
    if lib.glom_b200_abi_version() != ABI_VERSION:
        raise GlomB200Error(f"libglom_b200 ABI {lib.glom_b200_abi_version()} != expected {ABI_VERSION}")
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        raise GlomB200Error(f"glom_b200 error {rc}: {load().glom_b200_last_error().decode()}")


def make_cfg(dim, levels, n, attend_self, mask_side, mask_d2_max, precision):
    return Cfg(ctypes.sizeof(Cfg), dim, levels, n, int(bool(attend_self)), mask_side, mask_d2_max,
               PRECISION[precision])


def _bytes(symbol, *args):
    """The size_t that a *_bytes entry point writes through its last argument."""
    out = ctypes.c_size_t()
    check(getattr(load(), symbol)(*args, ctypes.byref(out)))
    return out.value


def packed_weight_bytes(cfg):
    return _bytes("glom_b200_packed_weight_bytes", ctypes.byref(cfg))


def workspace_bytes(cfg, batch, iters, return_all):
    return _bytes("glom_b200_workspace_bytes", ctypes.byref(cfg), batch, iters, int(return_all))


def workspace_offset(cfg, batch, iters, return_all, which):
    off, nb = ctypes.c_size_t(), ctypes.c_size_t()
    check(load().glom_b200_workspace_offset(ctypes.byref(cfg), batch, iters, int(return_all), which,
                                            ctypes.byref(off), ctypes.byref(nb)))
    return off.value, nb.value


def settle_workspace_offset(cfg, batch, max_iters, return_all, which):
    """(offset, bytes) of settle buffer `which` (0 dsq, 1 level_q, 2 frozen, 3 block_frozen) in the settle workspace."""
    off, nb = ctypes.c_size_t(), ctypes.c_size_t()
    check(load().glom_b200_settle_workspace_offset(ctypes.byref(cfg), batch, max_iters, int(return_all), which,
                                                   ctypes.byref(off), ctypes.byref(nb)))
    return off.value, nb.value


def pack_weights(cfg, ptrs, packed_ptr, packed_bytes, stream):
    w = WeightsRef(ctypes.sizeof(WeightsRef), *ptrs)
    check(load().glom_b200_pack_weights(ctypes.byref(cfg), ctypes.byref(w), packed_ptr, packed_bytes, stream))


def forward(cfg, packed_ptr, tokens_ptr, pos_ptr, state_in_ptr, init_ptr, out_ptr, batch, iters,
            return_all, ws_ptr, ws_bytes, stream):
    check(load().glom_b200_forward(ctypes.byref(cfg), packed_ptr, tokens_ptr, pos_ptr, state_in_ptr, init_ptr,
                                   out_ptr, batch, iters, int(return_all), ws_ptr, ws_bytes, stream))


def tokenize_workspace_bytes(batch, height, width, patch, dim, precision):
    return _bytes("glom_b200_tokenize_workspace_bytes", batch, height, width, patch, dim, PRECISION[precision])


def tokenize(img_ptr, w_ptr, b_ptr, out_ptr, batch, height, width, patch, dim, precision, ws_ptr, ws_bytes, stream):
    check(load().glom_b200_tokenize(img_ptr, w_ptr, b_ptr, out_ptr, batch, height, width, patch, dim,
                                    PRECISION[precision], ws_ptr, ws_bytes, stream))


def last_launch_count():
    return load().glom_b200_last_launch_count()


def profile_begin():
    check(load().glom_b200_profile_begin())


def profile_end():
    """-> {kind: (milliseconds, launches)} for the kernels enqueued since profile_begin()."""
    k = len(PROFILE_KINDS)
    ms = (ctypes.c_double * k)()
    cnt = (ctypes.c_int * k)()
    check(load().glom_b200_profile_end(ms, cnt, k))
    return {name: (ms[i], cnt[i]) for i, name in enumerate(PROFILE_KINDS)}


def forward_resume(cfg, packed_ptr, tokens_ptr, pos_ptr, state_in_ptr, out_ptr, batch, iters, return_all, ws_ptr, ws_bytes,
                   stream, shadow_parity):
    """glom_b200_forward_resume: returns the shadow buffer index holding the new final state's shadows."""
    out_par = ctypes.c_int(0)
    check(load().glom_b200_forward_resume(ctypes.byref(cfg), packed_ptr, tokens_ptr, pos_ptr, state_in_ptr, out_ptr, batch, iters,
                                          int(bool(return_all)), ws_ptr, ws_bytes, stream, shadow_parity, ctypes.byref(out_par)))
    return out_par.value


def settle_workspace_bytes(cfg, batch, max_iters):
    return _bytes("glom_b200_settle_workspace_bytes", ctypes.byref(cfg), batch, max_iters)


def settle_all_workspace_bytes(cfg, batch, max_iters):
    return _bytes("glom_b200_settle_all_workspace_bytes", ctypes.byref(cfg), batch, max_iters)


def forward_steps_workspace_bytes(cfg, batch, max_steps, return_all):
    return _bytes("glom_b200_forward_steps_workspace_bytes", ctypes.byref(cfg), batch, max_steps, int(bool(return_all)))


def settle(cfg, packed_ptr, tokens_ptr, pos_ptr, state_in_ptr, init_ptr, out_ptr, batch, max_iters, return_all, tol,
           steps_ptr, ws_ptr, ws_bytes, stream):
    """glom_b200_settle: up to max_iters steps, each image stopped on the GPU; steps_ptr -> (batch,) int32 device words.
    return_all: glom_b200_settle_all, every state kept; out_ptr -> (max_iters+1, batch, n, L, d) fp32, slab t of image b
    = S_min(t, steps[b])."""
    lib = load()
    fn = lib.glom_b200_settle_all if return_all else lib.glom_b200_settle
    check(fn(ctypes.byref(cfg), packed_ptr, tokens_ptr, pos_ptr, state_in_ptr, init_ptr, out_ptr, batch, max_iters,
             float(tol), steps_ptr, ws_ptr, ws_bytes, stream))


def settle_queue_workspace_bytes(cfg, slots, max_iters):
    return _bytes("glom_b200_settle_queue_workspace_bytes", ctypes.byref(cfg), slots, max_iters)


def settle_queue_begin(cfg, tokens_ptr, pos_ptr, state_in_ptr, init_ptr, out_ptr, steps_ptr, images, slots, max_iters, tol,
                       ws_ptr, ws_bytes, stream):
    """glom_b200_settle_queue_begin: every slot empty, all `images` queued (enqueued on `stream`)."""
    check(load().glom_b200_settle_queue_begin(ctypes.byref(cfg), tokens_ptr, pos_ptr, state_in_ptr, init_ptr, out_ptr,
                                              steps_ptr, images, slots, max_iters, float(tol), ws_ptr, ws_bytes, stream))


def settle_queue_run(cfg, packed_ptr, tokens_ptr, pos_ptr, state_in_ptr, init_ptr, out_ptr, steps_ptr, images, slots,
                     max_iters, tol, ws_ptr, ws_bytes, stream, first_step, num_steps, remaining_ptr):
    """glom_b200_settle_queue_run: global steps first_step .. first_step + num_steps - 1, then the unfinished count into
    remaining_ptr (device int32); num_steps = 0 enqueues the final hand-over only."""
    check(load().glom_b200_settle_queue_run(ctypes.byref(cfg), packed_ptr, tokens_ptr, pos_ptr, state_in_ptr, init_ptr,
                                            out_ptr, steps_ptr, images, slots, max_iters, float(tol), ws_ptr, ws_bytes,
                                            stream, first_step, num_steps, remaining_ptr))


def settle_video_workspace_bytes(cfg, slots, max_iters):
    return _bytes("glom_b200_settle_video_workspace_bytes", ctypes.byref(cfg), slots, max_iters)


def settle_video_begin(cfg, tokens_ptr, pos_ptr, state_in_ptr, init_ptr, out_ptr, steps_ptr, streams, frames, slots,
                       max_iters, tol, ws_ptr, ws_bytes, stream):
    """glom_b200_settle_video_begin: every slot empty, all `streams` queued (enqueued on `stream`)."""
    check(load().glom_b200_settle_video_begin(ctypes.byref(cfg), tokens_ptr, pos_ptr, state_in_ptr, init_ptr, out_ptr,
                                              steps_ptr, streams, frames, slots, max_iters, float(tol), ws_ptr, ws_bytes,
                                              stream))


def settle_video_run(cfg, packed_ptr, tokens_ptr, pos_ptr, state_in_ptr, init_ptr, out_ptr, steps_ptr, streams, frames,
                     slots, max_iters, tol, ws_ptr, ws_bytes, stream, first_step, num_steps, remaining_ptr):
    """glom_b200_settle_video_run: as settle_queue_run; the count is of unfinished frames."""
    check(load().glom_b200_settle_video_run(ctypes.byref(cfg), packed_ptr, tokens_ptr, pos_ptr, state_in_ptr, init_ptr,
                                            out_ptr, steps_ptr, streams, frames, slots, max_iters, float(tol), ws_ptr,
                                            ws_bytes, stream, first_step, num_steps, remaining_ptr))


def forward_steps(cfg, packed_ptr, tokens_ptr, pos_ptr, state_in_ptr, init_ptr, out_ptr, batch, steps_ptr, max_steps,
                  return_all, ws_ptr, ws_bytes, stream):
    """glom_b200_forward_steps: image b runs steps[b] steps (steps_ptr -> (batch,) int32 device words, clamped on the
    device to [0, max_steps])."""
    check(load().glom_b200_forward_steps(ctypes.byref(cfg), packed_ptr, tokens_ptr, pos_ptr, state_in_ptr, init_ptr, out_ptr,
                                         batch, steps_ptr, max_steps, int(bool(return_all)), ws_ptr, ws_bytes, stream))


def backward_workspace_bytes(cfg, batch):
    return _bytes("glom_b200_backward_workspace_bytes", ctypes.byref(cfg), batch)


def backward(cfg, weight_ptrs, tokens_ptr, pos_ptr, states_ptr, grad_out_ptr, grad_ptrs, batch, iters, grad_all,
             ws_ptr, ws_bytes, stream, steps_ptr=None, deterministic=False):
    """weight_ptrs: the 8 reference-layout tensors; grad_ptrs: dict of the Grads fields (None allowed for
    d_state0 / d_init).  With steps_ptr (the forward's (batch,) int32 step vector, iters = max_steps):
    glom_b200_backward_steps, the backward of forward_steps / settle_all.  deterministic: glom_b200_backward_ex with
    its fixed-order reductions (bit-reproducible gradients)."""
    w = WeightsRef(ctypes.sizeof(WeightsRef), *weight_ptrs)
    g = Grads(ctypes.sizeof(Grads), *[grad_ptrs.get(k) for k, _ in Grads._fields_[1:]])
    lib = load()
    if deterministic:
        rc = lib.glom_b200_backward_ex(ctypes.byref(cfg), ctypes.byref(w), tokens_ptr, pos_ptr, states_ptr, grad_out_ptr,
                                       ctypes.byref(g), batch, steps_ptr, iters, int(grad_all), 1, ws_ptr, ws_bytes, stream)
    elif steps_ptr is None:
        rc = lib.glom_b200_backward(ctypes.byref(cfg), ctypes.byref(w), tokens_ptr, pos_ptr, states_ptr, grad_out_ptr,
                                    ctypes.byref(g), batch, iters, int(grad_all), ws_ptr, ws_bytes, stream)
    else:
        rc = lib.glom_b200_backward_steps(ctypes.byref(cfg), ctypes.byref(w), tokens_ptr, pos_ptr, states_ptr,
                                          grad_out_ptr, ctypes.byref(g), batch, steps_ptr, iters, int(grad_all), ws_ptr,
                                          ws_bytes, stream)
    check(rc)


def backward_implicit_workspace_bytes(cfg, batch):
    return _bytes("glom_b200_backward_implicit_workspace_bytes", ctypes.byref(cfg), batch)


def backward_implicit(cfg, weight_ptrs, tokens_ptr, pos_ptr, state_ptr, grad_out_ptr, grad_ptrs, batch, adjoint_iters,
                      adjoint_tol, adjoint_steps_ptr, adjoint_q_ptr, ws_ptr, ws_bytes, stream, deterministic=False):
    """glom_b200_backward_implicit: the implicit gradients of the settled state at state_ptr given its cotangent;
    grad_ptrs as in backward, with d_state0 / d_init absent or None.  adjoint_steps_ptr -> (batch,) int32 device words,
    adjoint_q_ptr -> (batch, L) fp32 device words or None."""
    w = WeightsRef(ctypes.sizeof(WeightsRef), *weight_ptrs)
    g = Grads(ctypes.sizeof(Grads), *[grad_ptrs.get(k) for k, _ in Grads._fields_[1:]])
    check(load().glom_b200_backward_implicit(ctypes.byref(cfg), ctypes.byref(w), tokens_ptr, pos_ptr, state_ptr,
                                             grad_out_ptr, ctypes.byref(g), batch, adjoint_iters, float(adjoint_tol),
                                             int(bool(deterministic)), adjoint_steps_ptr, adjoint_q_ptr, ws_ptr, ws_bytes,
                                             stream))


def tokenize_backward_workspace_bytes(batch, h, w, patch, need_d_img):
    return _bytes("glom_b200_tokenize_backward_workspace_bytes", batch, h, w, patch, int(bool(need_d_img)))


def tokenize_backward(img_ptr, weight_ptr, d_tokens_ptr, d_weight_ptr, d_bias_ptr, d_img_ptr, batch, h, w, patch, dim,
                      ws_ptr, ws_bytes, stream, deterministic=False):
    """Tokeniser backward; d_* pointers may be None (skipped); outputs are accumulated into.  deterministic:
    glom_b200_tokenize_backward_ex, d_bias by a fixed-order column sum."""
    if deterministic:
        check(load().glom_b200_tokenize_backward_ex(img_ptr, weight_ptr, d_tokens_ptr, d_weight_ptr, d_bias_ptr, d_img_ptr,
                                                    batch, h, w, patch, dim, 1, ws_ptr, ws_bytes, stream))
        return
    check(load().glom_b200_tokenize_backward(img_ptr, weight_ptr, d_tokens_ptr, d_weight_ptr, d_bias_ptr, d_img_ptr, batch, h, w,
                                             patch, dim, ws_ptr, ws_bytes, stream))


def clock_probe(out_ptr, spin_us, stream):
    """Enqueue the SM clock probe: out_ptr -> 2 x uint64 device words {cycles, ns} (read after a synchronize)."""
    check(load().glom_b200_clock_probe(out_ptr, spin_us, stream))


def kernel_clocks(reset=True):
    """{kind: (SM MHz inside the kernels, in-kernel ms, [6 cycle fractions of block 0, see glom_b200_kernel_clocks in
    include/glom_b200.h])} since the last reset."""
    k = len(PROFILE_KINDS)
    mhz, ms, wf = (ctypes.c_double * k)(), (ctypes.c_double * k)(), (ctypes.c_double * (6 * k))()
    check(load().glom_b200_kernel_clocks(mhz, ms, wf, k, int(bool(reset))))
    return {PROFILE_KINDS[i]: (mhz[i], ms[i], [round(wf[6 * i + j], 4) for j in range(6)]) for i in range(k) if ms[i] > 0}


def set_sm_count_target(sms):
    """Plan every later launch of this process for at most `sms` SMs (0: the device's own count) -> the previous
    target.  Grids change, results do not (glom_b200_set_sm_count_target)."""
    lib = load()
    prev = lib.glom_b200_set_sm_count_target(int(sms))
    if prev < 0:
        raise GlomB200Error(f"glom_b200 error {prev}: {lib.glom_b200_last_error().decode()}")
    return prev


def islands(states_ptr, slabs, side_h, side_w, levels, dim, threshold, cos_right_ptr, cos_down_ptr, agreement_ptr,
            labels_ptr, num_islands_ptr, stream):
    check(load().glom_b200_islands(states_ptr, slabs, side_h, side_w, levels, dim, threshold, cos_right_ptr, cos_down_ptr,
                                   agreement_ptr, labels_ptr, num_islands_ptr, stream))
