"""ctypes binding of liblion_b200.so (the C ABI declared in include/lion_b200.h).

There is no CPU or eager-PyTorch fallback: if the shared library is missing, or a call
returns a non-zero code, an exception is raised.
"""
import ctypes as C
import os
import threading

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "liblion_b200.so")


class LionError(RuntimeError):
    pass


_lib = None
_lock = threading.Lock()
c_f = C.c_void_p   # device pointers travel as integers


def _proto(lib):
    i, f, d, sz, vp = C.c_int, C.c_float, C.c_double, C.c_size_t, C.c_void_p
    P = lambda *a: list(a)
    sig = {
        "lion_version": ([], i),
        "lion_last_error": ([], C.c_char_p),
        "lion_ctx_create": (P(i, C.POINTER(vp)), i),
        "lion_ctx_destroy": (P(vp), i),
        "lion_ctx_last_launches": (P(vp), i),
        "lion_ctx_last_conv_group": (P(vp), i),
        "lion_ctx_last_conv_stage_taps": (P(vp), i),
        "lion_ctx_set_conv_whole_slabs": (P(vp, i), i),
        "lion_ctx_set_sparse_conv1_dense": (P(vp, i), i),
        "lion_ctx_set_conv2_class_mode": (P(vp, i), i),
        "lion_ctx_last_conv2_class_blocks": (P(vp, vp, vp), i),
        "lion_ctx_arena_bytes": (P(vp), sz),
        "lion_ctx_generation": (P(vp), C.c_uint),
        "lion_ctx_timeline": (P(vp, vp, vp, i), i),
        "lion_avg_voxelize": (P(vp, vp, vp, vp, vp, i, i, i, i, vp), i),
        "lion_trilinear_devoxelize": (P(vp, vp, vp, vp, vp, i, i, i, i, i, vp), i),
        "lion_furthest_point_sampling": (P(vp, vp, i, i, i, vp), i),
        "lion_gather": (P(vp, vp, vp, i, i, i, i, vp), i),
        "lion_ball_query": (P(vp, vp, vp, i, i, i, f, i, vp), i),
        "lion_grouping": (P(vp, vp, vp, i, i, i, i, i, vp), i),
        "lion_three_nn_interpolate": (P(vp, vp, vp, vp, vp, vp, i, i, i, i, vp), i),
        "lion_voxel_coords": (P(vp, vp, vp, i, i, i, i, f, vp), i),
        "lion_avg_voxelize_backward": (P(vp, vp, vp, vp, i, i, i, i, vp), i),
        "lion_trilinear_devoxelize_backward": (P(vp, vp, vp, vp, i, i, i, i, vp), i),
        "lion_grouping_backward": (P(vp, vp, vp, i, i, i, i, i, vp), i),
        "lion_three_nn_interpolate_backward": (P(vp, vp, vp, vp, i, i, i, i, vp), i),
        "lion_gather_backward": (P(vp, vp, vp, i, i, i, i, vp), i),
        "lion_model_create": (P(vp, i, C.POINTER(i), i, C.POINTER(vp), i, C.POINTER(vp)), i),
        "lion_model_destroy": (P(vp), i),
        "lion_model_refresh": (P(vp), i),
        "lion_unet_forward": (P(vp, vp, vp, vp, vp, vp, i, i, vp), i),
        "lion_unet_forward_flags": (P(vp, vp, vp, vp, vp, vp, i, i, i, vp), i),
        "lion_unet_cache_style": (P(vp, vp, vp, i, vp), i),
        "lion_style_encoder_forward": (P(vp, vp, vp, i, i, vp), i),
        "lion_pvconv_fwd": (P(vp, vp, vp, vp, vp, i, i, vp), i),
        "lion_sa_module_fwd": (P(vp, vp, vp, vp, vp, vp, i, i, vp), i),
        "lion_fp_module_fwd": (P(vp, vp, vp, vp, vp, vp, vp, i, i, i, vp), i),
        "lion_linear_attention_fwd": (P(vp, vp, vp, i, i, vp), i),
        "lion_shared_mlp_fwd": (P(vp, vp, vp, vp, i, i, vp), i),
        "lion_global_prior_forward": (P(vp, vp, vp, vp, vp, i, vp), i),
        "lion_adagn_fwd": (P(vp, vp, vp, vp, i, i, vp), i),
        "lion_se3d_fwd": (P(vp, vp, vp, vp, vp, i, i, i, vp), i),
        "lion_swish_fwd": (P(vp, vp, sz, vp), i),
        "lion_ddpm_update": (P(vp, vp, vp, vp, vp, vp, f, sz, vp, i, vp), i),
        "lion_ddpm_set_step": (P(vp, vp, i, i, vp), i),
        "lion_ddpm_next_step": (P(vp, vp, i, vp), i),
        "lion_ddpm_fetch_noise": (P(vp, vp, vp, sz, vp), i),
        "lion_conv3d_gn_fwd": (P(vp, vp, vp, vp, vp, i, vp), i),
        "lion_conv3d_gn_fwd_flags": (P(vp, vp, vp, vp, vp, i, i, vp), i),
        "lion_pvconv_conv1_probe": (P(vp, vp, vp, i, vp, vp, vp, C.POINTER(i), i, i, vp), i),
        "lion_pvconv_conv1_mask_probe": (P(vp, vp, vp, vp, vp, i, i, vp), i),
        "lion_sa_mlp_probe": (P(vp, vp, vp, vp, i, vp, vp, vp, vp, vp, vp, C.POINTER(i), i, i, vp), i),
        "lion_pvconv_probe": (P(vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, C.POINTER(i), i, i, vp), i),
        "lion_pvconv_probe_flags": (P(vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, C.POINTER(i), i, i, i, vp), i),
        "lion_attention_probe": (P(vp, vp, vp, vp, vp, i, i, vp), i),
        "lion_fp_probe": (P(vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, i, i, i, vp), i),
        "lion_unet_probe": (P(vp, vp, vp, vp, vp, vp, C.POINTER(vp), i, C.POINTER(i), i, i, i, vp), i),
        "lion_global_prior_step": (P(vp, vp, vp, vp, vp, i, vp), i),
        "lion_global_prior_probe": (P(vp, vp, vp, vp, vp, C.POINTER(vp), i, i, vp), i),
        "lion_global_prior_saved_floats": (P(vp, i), sz),
        "lion_global_prior_forward_train": (P(vp, vp, vp, vp, vp, vp, vp, i, vp), i),
        "lion_global_prior_backward": (P(vp, vp, vp, vp, vp, vp, C.POINTER(vp), i, i, vp), i),
        "lion_global_prior_backward_probe": (P(vp, vp, vp, vp, vp, vp, C.POINTER(vp), i, C.POINTER(vp), i, i, vp), i),
        "lion_workspace_bytes": (P(vp), sz),
        "lion_ddim_update": (P(vp, vp, vp, vp, vp, vp, sz, vp, vp), i),
        "lion_ddim_set_step": (P(vp, vp, vp, i, i, i, vp), i),
        "lion_ddim_next_step": (P(vp, vp, vp, i, i, vp), i),
        "lion_scheduler_step": (P(vp, vp, vp, vp, vp, vp, sz, vp), i),
        "lion_ode_state_bytes": ([], sz),
        "lion_ode_init": (P(vp, vp, vp, sz, d, d, d, d, i, vp), i),
        "lion_ode_stage": (P(vp, vp, vp, vp, sz, i, vp, vp, i, vp), i),
        "lion_ode_rhs": (P(vp, vp, vp, vp, sz, i, d, d, d, vp, vp), i),
        "lion_ode_norms": (P(vp, vp, vp, vp, sz, i, vp, vp), i),
        "lion_ode_control": (P(vp, vp, sz, i, vp), i),
        "lion_ode_commit": (P(vp, vp, vp, vp, sz, vp), i),
        "lion_ode_dense_end": (P(vp, vp, vp, sz, vp, vp), i),
        "lion_chamfer_forward": (P(vp, vp, vp, vp, vp, vp, i, i, i, vp), i),
        "lion_chamfer_pairwise": (P(vp, vp, vp, i, i, i, i, vp), i),
        "lion_chamfer_backward": (P(vp, vp, vp, vp, vp, vp, vp, vp, i, i, i, vp), i),
        "lion_emd_approx": (P(vp, vp, vp, i, i, i, vp), i),
        "lion_emd_approx_saved": (P(vp, vp, vp, vp, i, i, i, vp), i),
        "lion_emd_backward": (P(vp, vp, vp, vp, vp, vp, i, i, i, vp), i),
        "lion_emd_pairwise": (P(vp, vp, vp, i, i, i, i, vp), i),
        "lion_occupancy_grid": (P(vp, vp, i, i, i, vp, vp, vp), i),
        "lion_bench_conv": (P(vp, i, i, i, i, i, i, i, C.POINTER(f), C.POINTER(C.c_double), vp), i),
    }
    for name, (args, res) in sig.items():
        fn = getattr(lib, name)      # AttributeError if the library does not export it
        fn.argtypes = args
        fn.restype = res
    return sig


EXPORTS = None


def lib():
    """Load (once) and return the shared library; raises LionError when it is not built."""
    global _lib, EXPORTS
    if _lib is None:
        with _lock:
            if _lib is None:
                if not os.path.exists(LIB_PATH):
                    raise LionError(
                        "lion_b200: %s not found -- build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                        "or `make -C lion_b200/csrc`; there is no fallback path." % LIB_PATH)
                l = C.CDLL(LIB_PATH)
                EXPORTS = sorted(_proto(l).keys())
                _lib = l
    return _lib


def check(rc, what=""):
    if rc != 0:
        msg = lib().lion_last_error()
        raise LionError("lion_b200 %s failed (code %d): %s" % (what, rc, msg.decode() if msg else "?"))


def ptr(t):
    """Device pointer of a contiguous fp32/int32 CUDA tensor (or None)."""
    if t is None:
        return None
    if not t.is_cuda:
        raise LionError("lion_b200 needs CUDA tensors (got %s); there is no CPU path" % t.device)
    if not t.is_contiguous():
        raise LionError("lion_b200 needs contiguous tensors")
    return t.data_ptr()


def stream():
    return torch.cuda.current_stream().cuda_stream


FWD_CONV_FP16 = 1     # LION_FWD_CONV_FP16 (include/lion_b200.h)

# the device-resident RK45 (include/lion_b200.h: LionOdeState and the lion_ode_* entry points)
ODE_RUNNING, ODE_DONE, ODE_TOO_SMALL = 0, 1, 2
ODE_INIT_H0, ODE_INIT_H1, ODE_END, ODE_BEGIN = 0, 1, 2, 3
ODE_STAGE_PROBE = 7
ODE_PARTIALS = 2 * 256


class OdeState(C.Structure):
    _fields_ = [(k, C.c_double) for k in ("t", "t_bound", "direction", "rtol", "atol", "h_abs", "h", "t_new", "min_step",
                                          "h0", "d1", "err_norm")] + \
               [(k, C.c_int) for k in ("status", "nfe", "n_accepted", "n_rejected", "step_rejected", "new_step", "accepted",
                                       "negate")]


def forward_flags():
    """The forward flags of the current autocast state: FWD_CONV_FP16 inside torch.autocast("cuda", dtype=torch.float16)
    (what the reference's `autocast(enable_autocast)` enables), 0 otherwise.  Outputs stay fp32 either way."""
    if torch.is_autocast_enabled("cuda") and torch.get_autocast_dtype("cuda") == torch.float16:
        return FWD_CONV_FP16
    return 0


_ctxs = {}


def ctx(device=None):
    """One context (scratch arena) per CUDA device."""
    dev = torch.cuda.current_device() if device is None else torch.device(device).index
    if dev is None:
        dev = torch.cuda.current_device()
    h = _ctxs.get(dev)
    if h is None:
        out = C.c_void_p()
        check(lib().lion_ctx_create(dev, C.byref(out)), "ctx_create")
        h = out
        _ctxs[dev] = h
    return h


def last_launches(device=None):
    return lib().lion_ctx_last_launches(ctx(device))


KIND_UNET, KIND_PVCONV, KIND_SA, KIND_FP, KIND_ATTN, KIND_SHARED_MLP, KIND_GLOBAL_PRIOR, KIND_ADAGN, KIND_CONV3D, KIND_STYLE_ENC = 1, 2, 3, 4, 5, 6, 7, 8, 9, 10


def float_bits(x):
    import struct
    return struct.unpack("i", struct.pack("f", float(x)))[0]


class Model:
    """A packed network/block living in the library.  Re-created when the parameter tensors
    are replaced, re-packed (refresh) when they were modified in place."""

    def __init__(self, kind, desc, params):
        for p in params:
            if not (p.is_cuda and p.dtype == torch.float32 and p.is_contiguous()):
                raise LionError("lion_b200: parameters must be contiguous fp32 CUDA tensors (move the module with "
                                ".cuda() first); there is no CPU path")
        self.kind = kind
        self.device = params[0].device
        self.params = [p.detach() for p in params]           # keep storage alive
        self.sig = tuple(p.data_ptr() for p in self.params)
        self.versions = tuple(p._version for p in params)
        d = (C.c_int * len(desc))(*[int(v) for v in desc])
        pp = (C.c_void_p * len(params))(*[p.data_ptr() for p in self.params])
        out = C.c_void_p()
        with torch.cuda.device(self.device):
            check(lib().lion_model_create(ctx(self.device), kind, d, len(desc), pp, len(params), C.byref(out)),
                  "model_create(kind=%d)" % kind)
        self.h = out

    def __del__(self):
        try:
            if getattr(self, "h", None) is not None and _lib is not None:
                _lib.lion_model_destroy(self.h)
        except Exception:
            pass

    def refresh(self):
        with torch.cuda.device(self.device):
            check(lib().lion_model_refresh(self.h), "model_refresh")

    # The handle is a per-process device object: copies (copy.deepcopy(module) for an EMA twin, torch.save(module),
    # pickling) must not carry it.  The copy gets None in place of the Model and rebuilds lazily on its first forward.
    def __deepcopy__(self, memo):
        return None

    def __reduce__(self):
        return (type(None), ())


def model_for(module, kind, desc, params):
    """Cached Model of an nn.Module; tracks load_state_dict / .cuda() / in-place updates."""
    m = module.__dict__.get("_lion_model")
    sig = tuple(p.data_ptr() for p in params)
    if m is None or m.sig != sig or m.kind != kind:
        m = Model(kind, desc, params)
        module.__dict__["_lion_model"] = m
    else:
        vers = tuple(p._version for p in params)
        if vers != m.versions:
            m.refresh()
            m.versions = vers
            m.style_key = None        # cached AdaGN style Linears were computed with the old weights
    return m


class capture_graph:
    """`with capture_graph() as g: ...; g.replay()` -- CUDA-graph capture of the enclosed launches on a
    side stream, like `torch.cuda.graph`, minus its `gc.collect()` + `torch.cuda.empty_cache()` +
    device-wide synchronize on entry: with two captures per sampling pass those cost more than the
    capture itself (and empty_cache makes the next pass cudaMalloc its gigabyte of history again)."""

    def __init__(self):
        self.graph = torch.cuda.CUDAGraph()
        self.stream = torch.cuda.Stream()
        self.generation = None

    def __enter__(self):
        self.stream.wait_stream(torch.cuda.current_stream())
        self._ctx = torch.cuda.stream(self.stream)
        self._ctx.__enter__()
        self.graph.capture_begin()
        return self

    def __exit__(self, et, ev, tb):
        try:
            try:
                self.graph.capture_end()          # also on an exception: never leave the stream in capture mode
            except Exception:
                if et is None:
                    raise
        finally:
            self._ctx.__exit__(et, ev, tb)
        if et is None:
            torch.cuda.current_stream().wait_stream(self.stream)
            self.generation = lib().lion_ctx_generation(ctx())
        return False

    def replay(self):
        """The captured launches have the scratch-arena addresses baked in: refuse to replay once a later eager call
        re-allocated the arena (use-after-free otherwise)."""
        if lib().lion_ctx_generation(ctx()) != self.generation:
            raise LionError("lion_b200: the scratch arena was re-allocated after this CUDA graph was captured; capture it again")
        self.graph.replay()
