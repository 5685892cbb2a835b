"""
_ffi.py -- ctypes binding of libb200gp.so (include/b200gp.h).  The only module that touches the
C-ABI; everything numerical happens behind it on the GPU.  There is no CPU fallback: if the
library or a CUDA device is missing, importing works (so CPU-only hosts can run the host-logic
tests) but the first call raises `B200GPError`.
"""
import contextlib
import ctypes as C
import os
import threading

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libb200gp.so")

KERNEL_RBF, KERNEL_MATERN52, KERNEL_PERIODIC = 0, 1, 2
KERNEL_NNGP_ERF, KERNEL_NNGP_RELU = 3, 4
ACT_RELU, ACT_TANH = 0, 1
KIND = {"RBF": KERNEL_RBF, "Matern": KERNEL_MATERN52, "Periodic": KERNEL_PERIODIC,
        "NNGP_erf": KERNEL_NNGP_ERF, "NNGP_relu": KERNEL_NNGP_RELU}

FLAG_DEVICE_PTRS = 1 << 0
FLAG_LOWER_ONLY = 1 << 1
FLAG_F32 = 1 << 2
FLAG_KPP_DIAG = 1 << 3
OUT_MEAN, OUT_VAR, OUT_COV, OUT_SAMPLE = 1 << 4, 1 << 5, 1 << 6, 1 << 7
OUT_DMEAN, OUT_DVAR = 1 << 8, 1 << 9


class B200GPError(RuntimeError):
    pass


def _mlp_nparams(D, widths):
    """entries of the flat parameter layout of a network with input width D and layer widths `widths`"""
    n, i = 0, int(D)
    for w in widths:
        n += i * int(w) + int(w)
        i = int(w)
    return n


class Timing(C.Structure):
    _fields_ = [("total_ms", C.c_double), ("gram_ms", C.c_double), ("potrf_ms", C.c_double),
                ("trsm_ms", C.c_double), ("epilogue_ms", C.c_double), ("h2d_ms", C.c_double),
                ("d2h_ms", C.c_double), ("flops", C.c_double), ("gram_bytes", C.c_double),
                ("launches", C.c_int64), ("host_enqueue_ms", C.c_double)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int)
_vp = C.c_void_p

# every symbol include/b200gp.h declares: name -> (restype, argtypes)
SIGNATURES = {
    "b2gp_version": (C.c_int, []),
    "b2gp_ctx_create": (C.c_int, [C.c_int, C.POINTER(_vp)]),
    "b2gp_ctx_destroy": (C.c_int, [_vp]),
    "b2gp_last_error": (C.c_char_p, [_vp]),
    "b2gp_set_option": (C.c_int, [_vp, C.c_char_p, C.c_int64]),
    "b2gp_get_option": (C.c_int, [_vp, C.c_char_p, C.POINTER(C.c_int64)]),
    "b2gp_device_info": (C.c_int, [_vp, _ip, _ip, _ip, C.POINTER(C.c_size_t)]),
    "b2gp_last_timing": (C.c_int, [_vp, C.POINTER(Timing)]),
    "b2gp_dev_alloc": (C.c_int, [_vp, C.c_size_t, C.POINTER(_vp)]),
    "b2gp_dev_free": (C.c_int, [_vp, _vp]),
    "b2gp_host_alloc": (C.c_int, [_vp, C.c_size_t, C.POINTER(_vp)]),
    "b2gp_host_free": (C.c_int, [_vp, _vp]),
    "b2gp_h2d": (C.c_int, [_vp, _vp, _vp, C.c_size_t]),
    "b2gp_d2h": (C.c_int, [_vp, _vp, _vp, C.c_size_t]),
    "b2gp_sync": (C.c_int, [_vp]),
    "b2gp_gram": (C.c_int, [_vp, C.c_int, _vp, C.c_int64, _vp, C.c_int64, C.c_int, _vp, C.c_double, C.c_double,
                            C.c_double, C.c_int, _vp, C.c_int64, C.c_uint]),
    "b2gp_gram_multitask": (C.c_int, [_vp, C.c_int, _vp, _vp, C.c_int64, _vp, _vp, C.c_int64, C.c_int, _vp, C.c_double, C.c_double, _vp,
                                      C.c_int, _vp, C.c_double, C.c_int, C.c_int, _vp, C.c_int64, C.c_uint]),
    "b2gp_potrf": (C.c_int, [_vp, C.c_int64, _vp, C.c_int64, _ip, C.c_uint]),
    "b2gp_trsm_lower": (C.c_int, [_vp, C.c_int64, C.c_int64, _vp, C.c_int64, _vp, C.c_int64, C.c_uint]),
    "b2gp_gemm_nt": (C.c_int, [_vp, C.c_int64, C.c_int64, C.c_int64, C.c_double, _vp, C.c_int64, _vp, C.c_int64,
                               C.c_double, _vp, C.c_int64, C.c_int, C.c_uint]),
    "b2gp_posterior": (C.c_int, [_vp, C.c_int, _vp, C.c_int64, _vp, C.c_int64, _vp, C.c_int64, C.c_int, C.c_int64,
                                 _vp, C.c_int, C.c_double, C.c_uint, _vp, _vp, _vp, _vp, C.c_int64, _vp, _vp,
                                 C.POINTER(Timing)]),
    "b2gp_posterior_batch": (C.c_int, [_vp, C.c_int, _vp, C.c_int64, C.c_int64, _vp, C.c_int64, _vp, C.c_int64, C.c_int64, C.c_int,
                                       C.c_int64, _vp, _vp, C.c_int64, C.c_int, C.c_double, C.c_uint, _vp, _vp, _vp, _vp,
                                       C.c_int64, _vp, _vp, C.POINTER(Timing)]),
    "b2gp_posterior_grad": (C.c_int, [_vp, C.c_int, _vp, C.c_int64, _vp, C.c_int64, _vp, C.c_int64, C.c_int, C.c_int64,
                                      _vp, C.c_int, C.c_double, C.c_uint, _vp, _vp, _vp, _vp, _vp, C.POINTER(Timing)]),
    "b2gp_posterior_multitask": (C.c_int, [_vp, C.c_int, _vp, _vp, C.c_int64, _vp, C.c_int64, _vp, _vp, C.c_int64, C.c_int, C.c_int,
                                           C.c_int, C.c_int, C.c_int64, _vp, _vp, _vp, C.c_int, C.c_double, C.c_uint, _vp, _vp, _vp,
                                           _vp, C.c_int64, _vp, _vp, C.POINTER(Timing)]),
    "b2gp_posterior_multitask_grad": (C.c_int, [_vp, C.c_int, _vp, _vp, C.c_int64, _vp, C.c_int64, _vp, _vp, C.c_int64, C.c_int,
                                                C.c_int, C.c_int, C.c_int, C.c_int64, _vp, _vp, _vp, C.c_int, C.c_double, C.c_uint,
                                                _vp, _vp, _vp, _vp, _vp, C.POINTER(Timing)]),
    "b2gp_mll_multitask": (C.c_int, [_vp, C.c_int, _vp, _vp, C.c_int64, _vp, C.c_int, C.c_int, C.c_int, C.c_int, _vp, _vp, _vp,
                                     C.c_double, C.c_uint, _dp, _vp, _vp, _vp, _vp, _ip]),
    "b2gp_mll_v": (C.c_int, [_vp, C.c_int, _vp, C.c_int64, _vp, C.c_int, _vp, _vp, C.c_double, C.c_uint, _dp, _vp, _vp, _vp, _ip]),
    "b2gp_sparse_posterior": (C.c_int, [_vp, C.c_int, _vp, C.c_int64, _vp, C.c_int64, _vp, _vp, C.c_int64, C.c_int,
                                        _vp, C.c_int, C.c_double, C.c_uint, _vp, _vp, _vp, _vp, C.POINTER(Timing)]),
    "b2gp_mll": (C.c_int, [_vp, C.c_int, _vp, C.c_int64, _vp, C.c_int, _vp, C.c_double, C.c_uint, _dp, _vp, _vp, _ip]),
    "b2gp_mll_batch": (C.c_int, [_vp, C.c_int, _vp, C.c_int64, _vp, C.c_int, C.c_int64, _vp, C.c_double, C.c_uint, _vp, _vp, _vp,
                                 _vp, _vp]),
    "b2gp_mll_draws": (C.c_int, [_vp, C.c_int, _vp, C.c_int64, _vp, C.c_int64, C.c_int, C.c_int64, _vp, C.c_double, C.c_uint, _vp,
                                 _vp, _vp, _vp]),
    "b2gp_mll_draws_v": (C.c_int, [_vp, C.c_int, _vp, C.c_int64, _vp, C.c_int64, C.c_int, C.c_int64, _vp, _vp, C.c_int64, C.c_double,
                                   C.c_uint, _vp, _vp, _vp, _vp, _vp]),
    "b2gp_mll_gram": (C.c_int, [_vp, _vp, C.c_int64, C.c_int64, _vp, _vp, C.c_int64, C.c_int64, C.c_uint, _dp, _vp, _vp, _ip]),
    "b2gp_posterior_gram": (C.c_int, [_vp, _vp, C.c_int64, C.c_int64, _vp, C.c_int64, _vp, C.c_int64, C.c_int64, C.c_int64, _vp,
                                      C.c_int64, C.c_uint, _vp, _vp, _vp, _vp, C.c_int64, _vp, _vp, C.POINTER(Timing)]),
    "b2gp_mlp_forward": (C.c_int, [_vp, _vp, C.c_int64, C.c_int64, C.c_int, _vp, C.c_int, _vp, C.c_int64, C.c_int64, _vp, C.c_uint]),
    "b2gp_dkl_mll": (C.c_int, [_vp, C.c_int, _vp, C.c_int64, C.c_int64, _vp, C.c_int, _vp, C.c_int, _vp, _vp, C.c_double, C.c_uint,
                               _dp, _vp, _vp, _vp, _ip]),
    "b2gp_dkl_posterior_grad": (C.c_int, [_vp, C.c_int, _vp, C.c_int64, C.c_int64, _vp, C.c_int64, _vp, C.c_int64, C.c_int, _vp,
                                          C.c_int, _vp, C.c_int64, C.c_int64, _vp, C.c_int, C.c_double, C.c_uint, _vp, _vp, _vp,
                                          _vp, _vp]),
    "b2gp_mtdkl_mll": (C.c_int, [_vp, C.c_int, _vp, _vp, C.c_int64, C.c_int64, _vp, C.c_int, C.c_int, C.c_int, C.c_int, _vp, C.c_int,
                                 _vp, _vp, _vp, _vp, C.c_double, C.c_uint, _dp, _vp, _vp, _vp, _vp, _vp, _ip]),
    "b2gp_bnn_loglik": (C.c_int, [_vp, _vp, C.c_int64, C.c_int64, _vp, C.c_int64, C.c_int, _vp, C.c_int, _vp, C.c_double, C.c_uint,
                                  _dp, _dp, _vp]),
    "b2gp_bnn_loglik_draws": (C.c_int, [_vp, _vp, C.c_int64, C.c_int64, _vp, C.c_int64, C.c_int, _vp, C.c_int, C.c_int64, _vp,
                                        C.c_int64, _vp, C.c_uint, _vp, _vp, _vp]),
    "b2gp_bnn_predict":(C.c_int, [_vp, _vp, C.c_int64, C.c_int64, C.c_int, _vp, C.c_int, _vp, C.c_int64, C.c_int64, C.c_int64, _vp,
                                   _vp, C.c_int64, _vp, _vp, C.c_uint]),
    "b2gp_bnn_predict_grad": (C.c_int, [_vp, _vp, C.c_int64, C.c_int64, C.c_int, _vp, C.c_int, _vp, C.c_int64, C.c_int64, _vp, _vp,
                                        C.c_uint]),
    "b2gp_sparse_elbo": (C.c_int, [_vp, C.c_int, _vp, C.c_int64, _vp, C.c_int64, _vp, C.c_int, _vp, C.c_double, C.c_uint, _dp, _vp,
                                   _vp, _ip]),
    "b2gp_sparse_elbo_ex": (C.c_int, [_vp, C.c_int, _vp, C.c_int64, _vp, C.c_int64, _vp, C.c_int, _vp, C.c_double, C.c_uint, _dp,
                                      _vp, _vp, _vp, _ip]),
    "b2gp_sparse_elbo_gram": (C.c_int, [_vp, _vp, C.c_int64, _vp, C.c_int64, _vp, _vp, C.c_double, _vp, _vp, _vp, C.c_int64, _vp, _vp,
                                        C.c_int64, C.c_uint, _dp, _vp, _dp, _vp, _vp, _ip]),
    "b2gp_sparse_posterior_gram": (C.c_int, [_vp, _vp, C.c_int64, _vp, C.c_int64, _vp, C.c_double, _vp, _vp, C.c_int64, C.c_uint, _vp,
                                             _vp, _vp, _ip, C.POINTER(Timing)]),
    "b2gp_dist_unique_id": (C.c_int, [_vp]),
    "b2gp_dist_init": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_int, C.c_int]),
    "b2gp_dist_info": (C.c_int, [_vp, _ip, _ip, _ip, _ip]),
    "b2gp_dist_finalize": (C.c_int, [_vp]),
    "b2gp_dist_posterior": (C.c_int, [_vp, C.c_int, _vp, C.c_int64, _vp, _vp, C.c_int64, C.c_int, _vp, C.c_int, C.c_double,
                                      C.c_int64, C.c_uint, _vp, _vp, _ip, C.POINTER(Timing)]),
    "b2gp_dist_sparse_posterior": (C.c_int, [_vp, C.c_int, _vp, C.c_int64, _vp, C.c_int64, _vp, _vp, C.c_int64, C.c_int, _vp, C.c_int,
                                             C.c_double, C.c_uint, _vp, _vp, _ip, C.POINTER(Timing)]),
    "b2gp_dist_layout": (C.c_int, [C.c_int64, C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int64,
                                   C.POINTER(C.c_int64)]),
    "b2gp_sparse_partial": (C.c_int, [_vp, C.c_int, _vp, C.c_int64, _vp, C.c_int64, _vp, C.c_int, _vp, C.c_double, _vp,
                                      C.c_int64, _vp, _ip]),
    "b2gp_sparse_finish": (C.c_int, [_vp, C.c_int, _vp, C.c_int64, _vp, C.c_int64, _vp, _vp, C.c_int64, C.c_int, _vp, C.c_int,
                                     C.c_double, C.c_uint, _vp, _vp, _vp, _ip]),
    "b2gp_potrf_inv": (C.c_int, [_vp, C.c_int64, _vp, C.c_int64, _vp, _ip]),
    "b2gp_trsm_inv": (C.c_int, [_vp, C.c_int64, C.c_int64, _vp, C.c_int64, _vp, _vp, C.c_int64]),
    "b2gp_rowdot": (C.c_int, [_vp, C.c_int64, C.c_int64, _vp, C.c_int64, _vp, C.c_double, _vp, _vp, C.c_int]),
    "b2gp_mvn_sample": (C.c_int, [_vp, _vp, _vp, C.c_int64, C.c_int64, _vp, C.c_int64, _vp, _vp, C.c_uint]),
    "b2gp_acq_moments": (C.c_int, [_vp, C.c_int, _vp, _vp, C.c_int64, C.c_int64, C.c_int, C.c_double, C.c_double, C.c_int, _vp,
                                   C.c_uint]),
    "b2gp_acq_samples": (C.c_int, [_vp, C.c_int, _vp, C.c_int64, C.c_int64, C.c_int, C.c_double, C.c_double, C.c_int, _vp, _vp,
                                   _vp, C.c_uint]),
    "b2gp_kg": (C.c_int, [_vp, _vp, _vp, C.c_int64, _vp, C.c_int64, C.c_double, C.c_double, C.c_int, _vp, C.c_uint]),
    "b2gp_kg_v": (C.c_int, [_vp, _vp, _vp, C.c_int64, _vp, C.c_int64, _vp, _vp, C.c_int, _vp, C.c_uint]),
    "b2gp_copy2d": (C.c_int, [_vp, _vp, C.c_int64, _vp, C.c_int64, C.c_int64, C.c_int64]),
}

_lib = None
_lib_lock = threading.Lock()


def load_library():
    """dlopen libb200gp.so and bind every declared symbol (no CUDA call is made)."""
    global _lib
    with _lib_lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise B200GPError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(or `make -C gpax_b200/csrc`).  gpax_b200 has no CPU fallback.")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)   # AttributeError if the .so lacks a declared symbol
            fn.restype = res
            fn.argtypes = args
        _lib = lib
        return lib


def _ptr(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


def _f32(a, shape=None):
    a = np.ascontiguousarray(a, dtype=np.float32)
    if shape is not None:
        a = a.reshape(shape)
    return a


def _f64(a, shape=None):
    a = np.ascontiguousarray(a, dtype=np.float64)
    if shape is not None:
        a = a.reshape(shape)
    return a


class DeviceArray:
    """A device allocation owned by a Context (fp64 elements unless stated)."""

    def __init__(self, ctx, nbytes, shape=None):
        self.ctx, self.nbytes, self.shape = ctx, int(nbytes), shape
        p = C.c_void_p()
        ctx._check(ctx.lib.b2gp_dev_alloc(ctx.h, self.nbytes, C.byref(p)))
        self.ptr = p

    def upload(self, host):
        host = np.ascontiguousarray(host)
        assert host.nbytes <= self.nbytes
        self.ctx._check(self.ctx.lib.b2gp_h2d(self.ctx.h, self.ptr, _ptr(host), host.nbytes))
        return self

    def download(self, shape=None, dtype=np.float64):
        shape = shape if shape is not None else self.shape
        out = np.empty(shape, dtype=dtype)
        assert out.nbytes <= self.nbytes
        self.ctx._check(self.ctx.lib.b2gp_d2h(self.ctx.h, _ptr(out), self.ptr, out.nbytes))
        return out

    def free(self):
        if self.ptr is not None and self.ctx.h is not None:
            self.ctx.lib.b2gp_dev_free(self.ctx.h, self.ptr)
        self.ptr = None


class Context:
    """One per Python thread (a ctx is not thread-safe).  Owns streams, workspaces, the device."""

    def __init__(self, device=0, streams=None):
        self.lib = load_library()
        h = C.c_void_p()
        rc = self.lib.b2gp_ctx_create(int(device), C.byref(h))
        if rc != 0:
            raise B200GPError(f"b2gp_ctx_create(device={device}) failed with {rc}: no usable CUDA device "
                              "(gpax_b200 has no CPU fallback)")
        self.h = h
        self.device = device
        self._pinned = []          # pinned host blocks handed out by pinned(): released with the context
        if streams is not None:
            self.set_option("streams", streams)

    # ---- plumbing
    def _check(self, rc):
        if rc != 0:
            msg = self.lib.b2gp_last_error(self.h)
            raise B200GPError(f"libb200gp error {rc}: {msg.decode() if msg else ''}")

    def close(self):
        """destroy the context; pinned arrays obtained from pinned() must not be used afterwards"""
        if getattr(self, "h", None) is not None:
            for p in getattr(self, "_pinned", []):
                self.lib.b2gp_host_free(self.h, p)
            self._pinned = []
            self.lib.b2gp_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_option(self, key, value):
        self._check(self.lib.b2gp_set_option(self.h, key.encode(), int(value)))

    def get_option(self, key):
        v = C.c_int64()
        self._check(self.lib.b2gp_get_option(self.h, key.encode(), C.byref(v)))
        return v.value

    @contextlib.contextmanager
    def options(self, **kw):
        """set the given options for the duration of a `with` block, then restore the values they had before"""
        old = {k: self.get_option(k) for k in kw}
        try:
            for k, v in kw.items():
                self.set_option(k, v)
            yield self
        finally:
            for k, v in old.items():
                self.set_option(k, v)

    # cumulative counters of b2gp_debug_path_counts, in its order (PathCounter in csrc/common.cuh)
    PATHS = ("gemm_nt", "gemm_tma", "oz_mma", "oz_slice", "trsm_strip", "potrf_diag", "panel_solve", "trsm_tall", "potrf_tall",
             "potrf_tall_fp64", "mll_nngp_grad", "mll_gram_trace", "mll_batch_small", "potrf_tall_batch",
             "mll_draws_batch", "sparse_gram_trace")

    def path_counts(self):
        """development aid: how often each kernel was launched / each solver route entered on this context so far"""
        fn = self.lib.b2gp_debug_path_counts
        fn.restype, fn.argtypes = C.c_int, [_vp, C.POINTER(C.c_int64), C.c_int]
        out = (C.c_int64 * len(self.PATHS))()
        n = fn(self.h, out, len(self.PATHS))
        if n != len(self.PATHS):
            raise B200GPError(f"b2gp_debug_path_counts reports {n} counters, the binding knows {len(self.PATHS)}")
        return dict(zip(self.PATHS, out))

    def cache_hits(self):
        """development aid: posterior calls on this context that reused the cached factor (b2gp_debug_cache_hits)"""
        fn = self.lib.b2gp_debug_cache_hits
        fn.restype, fn.argtypes = C.c_int64, [_vp]
        return fn(self.h)

    def device_info(self):
        sm, ma, mi, mem = C.c_int(), C.c_int(), C.c_int(), C.c_size_t()
        self._check(self.lib.b2gp_device_info(self.h, C.byref(sm), C.byref(ma), C.byref(mi), C.byref(mem)))
        return {"sm_count": sm.value, "cc": (ma.value, mi.value), "mem_bytes": mem.value}

    def last_timing(self):
        t = Timing()
        self._check(self.lib.b2gp_last_timing(self.h, C.byref(t)))
        return t.as_dict()

    def sync(self):
        self._check(self.lib.b2gp_sync(self.h))

    def alloc(self, shape, dtype=np.float64):
        shape = tuple(np.atleast_1d(shape).tolist())
        return DeviceArray(self, int(np.prod(shape)) * np.dtype(dtype).itemsize, shape)

    def to_device(self, host):
        host = np.ascontiguousarray(host)
        return DeviceArray(self, host.nbytes, host.shape).upload(host)

    def pinned(self, shape, dtype=np.float64):
        """NumPy array over pinned (page-locked) host memory; the block lives until close()"""
        n = int(np.prod(shape)) * np.dtype(dtype).itemsize
        p = C.c_void_p()
        self._check(self.lib.b2gp_host_alloc(self.h, n, C.byref(p)))
        self._pinned.append(C.c_void_p(p.value))
        buf = (C.c_char * n).from_address(p.value)
        arr = np.frombuffer(buf, dtype=dtype).reshape(shape)
        return arr

    # ---- primitives (host arrays in / out)
    def gram(self, kind, X, Z, lengthscale, scale, period=1.0, diag_add=0.0, same_xz=None, lower_only=False, f32=False):
        """f32: X, Z are handed over as float32 and K comes back float32 (B2GP_FLAG_F32)"""
        cv, dt = (_f32, np.float32) if f32 else (_f64, np.float64)
        X, Z = cv(X), cv(Z)
        n, d = X.shape
        m = Z.shape[0]
        ell = _f64(np.broadcast_to(np.asarray(lengthscale, dtype=np.float64).reshape(-1), (d,)))
        if same_xz is None:
            same_xz = X.shape == Z.shape          # kernels.py:63
        K = np.zeros((n, m), dtype=dt) if lower_only else np.empty((n, m), dtype=dt)
        if n == 0 or m == 0:
            return K
        flags = (FLAG_LOWER_ONLY if lower_only else 0) | (FLAG_F32 if f32 else 0)
        self._check(self.lib.b2gp_gram(self.h, KIND[kind] if isinstance(kind, str) else kind, _ptr(X), n, _ptr(Z), m, d,
                                       _ptr(ell), float(scale), float(period), float(diag_add), int(bool(same_xz)),
                                       _ptr(K), m, flags))
        return K

    def gram_multitask(self, kind, X, tX, Z, tZ, lengthscale, scale, period, B, noise_task, jitter, same_xz, group=1):
        X, Z, B = _f64(X), _f64(Z), _f64(B)
        n, d = X.shape
        m = Z.shape[0]
        tX, tZ = np.ascontiguousarray(tX, dtype=np.int32), np.ascontiguousarray(tZ, dtype=np.int32)
        ell = _f64(np.broadcast_to(np.asarray(lengthscale, dtype=np.float64).reshape(-1), (d,)))
        nt = None if noise_task is None else _f64(noise_task)
        K = np.empty((n, m))
        self._check(self.lib.b2gp_gram_multitask(self.h, kind if isinstance(kind, int) else KIND[kind], _ptr(X), _ptr(tX), n, _ptr(Z), _ptr(tZ),
                                                 m, d, _ptr(ell), float(scale), float(period), _ptr(B), B.shape[0], _ptr(nt), float(jitter),
                                                 int(bool(same_xz)), int(group), _ptr(K), m, 0))
        return K

    def potrf(self, A):
        A = np.array(A, dtype=np.float64, order="C", copy=True)
        n = A.shape[0]
        info = C.c_int(0)
        self._check(self.lib.b2gp_potrf(self.h, n, _ptr(A), A.shape[1] if A.ndim == 2 else 1, C.byref(info), 0))
        return A, info.value

    def trsm_lower(self, L, B):
        """Rows of B are right-hand sides: returns B L^{-T} (row r = L^{-1} b_r).  Call right after potrf."""
        L = _f64(L)
        B = np.array(B, dtype=np.float64, order="C", copy=True)
        n = L.shape[0]
        self._check(self.lib.b2gp_trsm_lower(self.h, n, B.shape[0], _ptr(L), n, _ptr(B), B.shape[1], 0))
        return B

    def gemm_nt(self, A, B, C_in=None, alpha=1.0, beta=0.0, lower_only=False):
        A, B = _f64(A), _f64(B)
        m, k = A.shape
        n = B.shape[0]
        Cm = np.zeros((m, n)) if C_in is None else np.array(C_in, dtype=np.float64, order="C", copy=True)
        self._check(self.lib.b2gp_gemm_nt(self.h, m, n, k, float(alpha), _ptr(A), k, _ptr(B), k, float(beta), _ptr(Cm), n,
                                          int(lower_only), 0))
        return Cm

    # ---- the posterior (host arrays in / out)
    def posterior(self, kind, Xtr, yres, Xnew, theta, noiseless=False, jitter=1e-6, want=("mean", "cov"),
                  eps=None, timing=False, noise_vec=None, f32=False):
        """theta: [S, d+3] rows (lengthscale[d], k_scale, noise, period); yres [N] or [S, N].  Xtr [N, d] or per member
        [S, N, d]; Xnew [P, d] or [S, P, d]; noise_vec None, [N] or [S, N] (per-point noise variances on k_XX's diagonal).
        f32: the data arrays cross the boundary as float32 in both directions (B2GP_FLAG_F32), theta stays float64."""
        _f64 = _f32 if f32 else globals()["_f64"]      # noqa: F811  data arrays in the I/O precision
        odt = np.float32 if f32 else np.float64
        Xtr, Xnew = _f64(Xtr), _f64(Xnew)
        N, d = Xtr.shape[-2:]
        P = Xnew.shape[-2]
        theta = globals()["_f64"](theta).reshape(-1, d + 3)
        S = theta.shape[0]
        yres = _f64(yres)
        stride = 0 if yres.ndim == 1 else yres.shape[1]
        xs = 0 if Xtr.ndim == 2 else N * d
        xns = 0 if Xnew.ndim == 2 else P * d
        nv = None if noise_vec is None else _f64(noise_vec)
        nvs = 0 if nv is None or nv.ndim == 1 else N
        for a, n_ in ((Xtr, xs), (Xnew, xns), (nv, nvs)):
            if a is not None and n_ and a.shape[0] != S:
                raise ValueError("per-member arrays need a leading axis of length S = theta.shape[0]")
        flags = FLAG_F32 if f32 else 0
        mean = var = cov = samp = None
        if "mean" in want:
            flags |= OUT_MEAN
            mean = np.empty((S, P), dtype=odt)
        if "var" in want:
            flags |= OUT_VAR
            var = np.empty((S, P), dtype=odt)
        if "cov" in want:
            flags |= OUT_COV
            cov = np.empty((S, P, P), dtype=odt)
        n_samp = 0
        if eps is not None:
            eps = _f64(eps).reshape(S, -1, P)
            n_samp = eps.shape[1]
            flags |= OUT_SAMPLE
            samp = np.empty((S, n_samp, P), dtype=odt)
        info = np.zeros(S, dtype=np.int32)
        t = Timing()
        self._check(self.lib.b2gp_posterior_batch(
            self.h, KIND[kind] if isinstance(kind, str) else kind, _ptr(Xtr), xs, N, _ptr(yres), stride, _ptr(Xnew), xns, P, d, S,
            _ptr(theta), _ptr(nv), nvs, int(bool(noiseless)), float(jitter), flags, _ptr(mean), _ptr(var), _ptr(cov), _ptr(eps),
            n_samp, _ptr(samp), info.ctypes.data_as(_vp), C.byref(t) if timing else None))
        out = {"mean": mean, "var": var, "cov": cov, "y_sampled": samp, "info": info}
        if timing:
            out["timing"] = t.as_dict()
        return out

    def posterior_grad(self, kind, Xtr, yres, Xnew, theta, noiseless=False, jitter=1e-6,
                       want=("mean", "var", "dmean", "dvar"), timing=False):
        """The posterior mean / variance and their gradients w.r.t. the test inputs (b2gp_posterior_grad).  Xtr [N, d],
        Xnew [P, d], theta [S, d+3], yres [N] or [S, N]; fp64 host arrays.  Returns a dict with mean / var [S, P],
        dmean / dvar [S, P, d] (None where not in `want`) and info [S]."""
        Xtr, Xnew = _f64(Xtr), _f64(Xnew)
        N, d = Xtr.shape
        P = Xnew.shape[0]
        theta = _f64(theta).reshape(-1, d + 3)
        S = theta.shape[0]
        yres = _f64(yres)
        stride = 0 if yres.ndim == 1 else yres.shape[1]
        bits = {"mean": (OUT_MEAN, (S, P)), "var": (OUT_VAR, (S, P)), "dmean": (OUT_DMEAN, (S, P, d)), "dvar": (OUT_DVAR, (S, P, d))}
        flags, out = 0, {}
        for name, (bit, shape) in bits.items():
            out[name] = np.empty(shape) if name in want else None
            flags |= bit if name in want else 0
        info = np.zeros(S, dtype=np.int32)
        t = Timing()
        self._check(self.lib.b2gp_posterior_grad(
            self.h, KIND[kind] if isinstance(kind, str) else kind, _ptr(Xtr), N, _ptr(yres), stride, _ptr(Xnew), P, d, S,
            _ptr(theta), int(bool(noiseless)), float(jitter), flags, _ptr(out["mean"]), _ptr(out["var"]), _ptr(out["dmean"]),
            _ptr(out["dvar"]), info.ctypes.data_as(_vp), C.byref(t) if timing else None))
        out["info"] = info
        if timing:
            out["timing"] = t.as_dict()
        return out

    def mll(self, kind, X, yres, theta, jitter=1e-6, want_grad=True, want_alpha=False, noise_vec=None):
        """log marginal likelihood, its gradient w.r.t. log(lengthscale[d], k_scale, noise, period), alpha = K^-1 y.
        With noise_vec [N] (per-point noise variances on the diagonal) the return gains d value / d noise_vec."""
        X, yres = _f64(X), _f64(yres)
        N, d = X.shape
        theta = _f64(theta).reshape(d + 3)
        val = C.c_double(0.0)
        grad = np.zeros(d + 3) if want_grad else None
        alpha = np.zeros(N) if want_alpha else None
        info = C.c_int(0)
        if noise_vec is None:
            self._check(self.lib.b2gp_mll(self.h, KIND[kind] if isinstance(kind, str) else kind, _ptr(X), N, _ptr(yres), d,
                                          _ptr(theta), float(jitter), 0, C.byref(val), _ptr(grad), _ptr(alpha), C.byref(info)))
            return val.value, grad, alpha, info.value
        nv = _f64(noise_vec).reshape(N)
        gnv = np.zeros(N) if want_grad else None
        self._check(self.lib.b2gp_mll_v(self.h, KIND[kind] if isinstance(kind, str) else kind, _ptr(X), N, _ptr(yres), d,
                                        _ptr(theta), _ptr(nv), float(jitter), 0, C.byref(val), _ptr(grad), _ptr(alpha), _ptr(gnv),
                                        C.byref(info)))
        return val.value, grad, alpha, info.value, gnv

    def mll_batch(self, kind, X, yres, theta, jitter=1e-6, want_grad=True, want_alpha=False, want_grad_x=False):
        """B independent likelihoods (b2gp_mll_batch): member b is ctx.mll(kind, X[b], yres[b], theta[b]) and, with
        want_grad_x, d value / d X[b] as ctx.dkl_mll(n_layers=0).  X [B, N, d], yres [B, N], theta [B, d+3] (host arrays).
        Returns (value [B], grad [B, d+3] or None, alpha [B, N] or None, grad_x [B, N, d] or None, info [B])."""
        X, yres, theta = _f64(X), _f64(yres), _f64(theta)
        if X.ndim != 3:
            raise ValueError(f"X must be [B, N, d], got shape {X.shape}")
        B, N, d = X.shape
        if yres.shape != (B, N) or theta.shape != (B, d + 3):
            raise ValueError(f"yres must be [{B}, {N}] and theta [{B}, {d + 3}], got {yres.shape} and {theta.shape}")
        if want_grad_x and not want_grad:
            raise ValueError("want_grad_x needs want_grad")
        val = np.zeros(B)
        grad = np.zeros((B, d + 3)) if want_grad else None
        alpha = np.zeros((B, N)) if want_alpha else None
        gx = np.zeros((B, N, d)) if want_grad_x else None
        info = np.zeros(B, dtype=np.int32)
        self._check(self.lib.b2gp_mll_batch(self.h, KIND[kind] if isinstance(kind, str) else kind, _ptr(X), N, _ptr(yres), d, B,
                                            _ptr(theta), float(jitter), 0, _ptr(val), _ptr(grad), _ptr(alpha), _ptr(gx),
                                            _ptr(info)))
        return val, grad, alpha, gx, info

    def mll_draws(self, kind, X, yres, theta, jitter=1e-6, want_grad=True, want_alpha=False):
        """S likelihoods on one X in lock-step (b2gp_mll_draws): draw s is ctx.mll(kind, X, yres[s], theta[s]) bit for bit.
        X [N, d]; yres [N] (shared) or [S, N]; theta [S, d+3] (host arrays).
        Returns (value [S], grad [S, d+3] or None, alpha [S, N] or None, info [S])."""
        X, yres = _f64(X), _f64(yres)
        N, d = X.shape
        theta = _f64(theta).reshape(-1, d + 3)
        S = theta.shape[0]
        if yres.shape not in ((N,), (S, N)):
            raise ValueError(f"yres must be [{N}] or [{S}, {N}], got shape {yres.shape}")
        val = np.zeros(S)
        grad = np.zeros((S, d + 3)) if want_grad else None
        alpha = np.zeros((S, N)) if want_alpha else None
        info = np.zeros(S, dtype=np.int32)
        self._check(self.lib.b2gp_mll_draws(self.h, KIND[kind] if isinstance(kind, str) else kind, _ptr(X), N, _ptr(yres),
                                            0 if yres.ndim == 1 else N, d, S, _ptr(theta), float(jitter), 0, _ptr(val),
                                            _ptr(grad), _ptr(alpha), _ptr(info)))
        return val, grad, alpha, info

    def mll_draws_v(self, kind, X, yres, theta, noise_vec, jitter=1e-6, want_grad=True, want_alpha=False):
        """mll_draws with per-point noise variances (b2gp_mll_draws_v): draw s is ctx.mll(kind, X, yres[s], theta[s],
        noise_vec=noise_vec[s]) bit for bit.  noise_vec [N] (shared) or [S, N]; the rest as mll_draws.
        Returns (value [S], grad [S, d+3] or None, alpha [S, N] or None, grad_noise_vec [S, N] or None, info [S])."""
        X, yres, nv = _f64(X), _f64(yres), _f64(noise_vec)
        N, d = X.shape
        theta = _f64(theta).reshape(-1, d + 3)
        S = theta.shape[0]
        if yres.shape not in ((N,), (S, N)) or nv.shape not in ((N,), (S, N)):
            raise ValueError(f"yres and noise_vec must be [{N}] or [{S}, {N}], got shapes {yres.shape} and {nv.shape}")
        val = np.zeros(S)
        grad = np.zeros((S, d + 3)) if want_grad else None
        alpha = np.zeros((S, N)) if want_alpha else None
        gnv = np.zeros((S, N)) if want_grad else None
        info = np.zeros(S, dtype=np.int32)
        self._check(self.lib.b2gp_mll_draws_v(self.h, KIND[kind] if isinstance(kind, str) else kind, _ptr(X), N, _ptr(yres),
                                              0 if yres.ndim == 1 else N, d, S, _ptr(theta), _ptr(nv), 0 if nv.ndim == 1 else N,
                                              float(jitter), 0, _ptr(val), _ptr(grad), _ptr(alpha), _ptr(gnv), _ptr(info)))
        return val, grad, alpha, gnv, info

    def mll_gram(self, K, yres, dKs=(), want_grad=True, want_alpha=False):
        """log N(yres; 0, K) from a caller-supplied K [N, N] (factored as (K + K^T) / 2), the traces
        grad[j] = 1/2 sum (alpha alpha^T - K^-1) * dKs[j] for the N x N matrices in `dKs`, and alpha = K^-1 yres
        (b2gp_mll_gram).  K, yres and the dKs are all NumPy arrays, or all DeviceArrays (B2GP_FLAG_DEVICE_PTRS).
        Returns (value, grad [len(dKs)] or None, alpha [N] or None, info)."""
        dev = isinstance(K, DeviceArray)
        if dev:
            N = K.shape[0]
            if K.shape != (N, N) or tuple(yres.shape) != (N,) or any(tuple(D.shape) != (N, N) for D in dKs):
                raise ValueError("K and every dK must be [N, N] and yres [N]")
            Kp, yp, ptrs = K.ptr, yres.ptr, [D.ptr.value for D in dKs]
        else:
            K, yres = _f64(K), _f64(yres)
            N = K.shape[0]
            dKs = [_f64(D) for D in dKs]
            if K.shape != (N, N) or yres.shape != (N,) or any(D.shape != (N, N) for D in dKs):
                raise ValueError("K and every dK must be [N, N] and yres [N]")
            Kp, yp, ptrs = _ptr(K), _ptr(yres), [D.ctypes.data for D in dKs]
        p = len(ptrs) if want_grad else 0
        arr = (C.c_void_p * max(p, 1))(*ptrs[:p])
        val = C.c_double(0.0)
        grad = np.zeros(p) if want_grad else None
        alpha = np.zeros(N) if want_alpha else None
        info = C.c_int(0)
        self._check(self.lib.b2gp_mll_gram(self.h, Kp, N, N, yp, C.cast(arr, _vp), N, p, FLAG_DEVICE_PTRS if dev else 0,
                                           C.byref(val), _ptr(grad), _ptr(alpha), C.byref(info)))
        return val.value, grad, alpha, info.value

    def posterior_gram(self, Kxx, Kpx, Kpp, yres, want=("mean", "cov"), eps=None, kpp_diag=False, timing=False):
        """The batched posterior from caller-supplied Gram blocks (b2gp_posterior_gram): Kxx [S, N, N] or [N, N] (shared),
        Kpx [S, P, N] or [P, N], Kpp [S, P, P] or [P, P] -- or with kpp_diag its diagonal [S, P] or [P] (mean / var only) --
        and yres [N] or [S, N].  Host fp64 arrays; outputs as posterior()."""
        Kxx, Kpx, yres = _f64(Kxx), _f64(Kpx), _f64(yres)
        N = Kxx.shape[-1]
        P = Kpx.shape[-2]
        Kpp = None if Kpp is None else _f64(Kpp)
        pp = (P,) if kpp_diag else (P, P)
        S = max([1] + [a.shape[0] for a, nd in ((Kxx, 3), (Kpx, 3), (Kpp, len(pp) + 1), (yres, 2)) if a is not None and a.ndim == nd])
        for a, shp in ((Kxx, (N, N)), (Kpx, (P, N)), (Kpp, pp), (yres, (N,))):
            if a is not None and a.shape not in (shp, (S,) + shp):
                raise ValueError(f"Gram block of shape {a.shape}: expected {shp} or {(S,) + shp}")
        stride = lambda a, n: 0 if a is None or a.ndim == len(n) else int(np.prod(n))   # noqa: E731
        flags = FLAG_KPP_DIAG if kpp_diag else 0
        out = {"mean": None, "var": None, "cov": None, "y_sampled": None}
        for name, bit, shape in (("mean", OUT_MEAN, (S, P)), ("var", OUT_VAR, (S, P)), ("cov", OUT_COV, (S, P, P))):
            if name in want:
                flags |= bit
                out[name] = np.empty(shape)
        n_samp = 0
        if eps is not None:
            eps = _f64(eps).reshape(S, -1, P)
            n_samp = eps.shape[1]
            flags |= OUT_SAMPLE
            out["y_sampled"] = np.empty((S, n_samp, P))
        info = np.zeros(S, dtype=np.int32)
        t = Timing()
        self._check(self.lib.b2gp_posterior_gram(
            self.h, _ptr(Kxx), stride(Kxx, (N, N)), N, _ptr(Kpx), stride(Kpx, (P, N)), _ptr(Kpp), stride(Kpp, pp), P, S, _ptr(yres),
            stride(yres, (N,)), flags, _ptr(out["mean"]), _ptr(out["var"]), _ptr(out["cov"]), _ptr(eps), n_samp, _ptr(out["y_sampled"]),
            info.ctypes.data_as(_vp), C.byref(t) if timing else None))
        out["info"] = info
        if timing:
            out["timing"] = t.as_dict()
        return out

    def posterior_multitask(self, kind, Xtr, task_tr, yres, Xnew, task_new, theta, B, noise, group=1, noiseless=False, jitter=1e-6,
                            want=("mean", "cov"), eps=None, timing=False, flags=0):
        """The LCM posterior of MultiTaskGP / CoregGP (b2gp_posterior_multitask).  Xtr [N, d] and task_tr [N], Xnew [P, d] and
        task_new [P] count rows (the Kronecker form is expanded by the caller, group = T); theta [S, L, d+2] rows
        (lengthscale[d], k_scale, period), B [S, L, T, T], noise [S, T]; yres [N] or [S, N].  Outputs as posterior()."""
        Xtr, Xnew = _f64(Xtr), _f64(Xnew)
        N, d = Xtr.shape
        P = Xnew.shape[0]
        B = _f64(B)
        S, L, T = B.shape[0], B.shape[1], B.shape[2]
        theta, noise = _f64(theta, (S, L, d + 2)), _f64(noise, (S, T))
        ttr, tnew = np.ascontiguousarray(task_tr, dtype=np.int32), np.ascontiguousarray(task_new, dtype=np.int32)
        yres = _f64(yres)
        stride = 0 if yres.ndim == 1 else yres.shape[1]
        mean = var = cov = samp = None
        if "mean" in want:
            flags |= OUT_MEAN
            mean = np.empty((S, P))
        if "var" in want:
            flags |= OUT_VAR
            var = np.empty((S, P))
        if "cov" in want:
            flags |= OUT_COV
            cov = np.empty((S, P, P))
        n_samp = 0
        if eps is not None:
            eps = _f64(eps).reshape(S, -1, P)
            n_samp = eps.shape[1]
            flags |= OUT_SAMPLE
            samp = np.empty((S, n_samp, P))
        info = np.zeros(S, dtype=np.int32)
        t = Timing()
        self._check(self.lib.b2gp_posterior_multitask(
            self.h, KIND[kind] if isinstance(kind, str) else kind, _ptr(Xtr), _ptr(ttr), N, _ptr(yres), stride, _ptr(Xnew), _ptr(tnew),
            P, d, int(group), T, L, S, _ptr(theta), _ptr(B), _ptr(noise), int(bool(noiseless)), float(jitter), flags, _ptr(mean),
            _ptr(var), _ptr(cov), _ptr(eps), n_samp, _ptr(samp), info.ctypes.data_as(_vp), C.byref(t) if timing else None))
        out = {"mean": mean, "var": var, "cov": cov, "y_sampled": samp, "info": info}
        if timing:
            out["timing"] = t.as_dict()
        return out

    def posterior_multitask_grad(self, kind, Xtr, task_tr, yres, Xnew, task_new, theta, B, noise, group=1, noiseless=False,
                                 jitter=1e-6, want=("mean", "var", "dmean", "dvar"), timing=False, flags=0):
        """The LCM posterior and its gradients w.r.t. the test inputs (b2gp_posterior_multitask_grad).  Arguments as
        posterior_multitask().  Returns a dict with mean / var [S, P], dmean / dvar [S, P, d] (None where not in `want`)
        and info [S]."""
        Xtr, Xnew = _f64(Xtr), _f64(Xnew)
        N, d = Xtr.shape
        P = Xnew.shape[0]
        B = _f64(B)
        S, L, T = B.shape[0], B.shape[1], B.shape[2]
        theta, noise = _f64(theta, (S, L, d + 2)), _f64(noise, (S, T))
        ttr, tnew = np.ascontiguousarray(task_tr, dtype=np.int32), np.ascontiguousarray(task_new, dtype=np.int32)
        yres = _f64(yres)
        stride = 0 if yres.ndim == 1 else yres.shape[1]
        bits = {"mean": (OUT_MEAN, (S, P)), "var": (OUT_VAR, (S, P)), "dmean": (OUT_DMEAN, (S, P, d)), "dvar": (OUT_DVAR, (S, P, d))}
        out = {}
        for name, (bit, shape) in bits.items():
            out[name] = np.empty(shape) if name in want else None
            flags |= bit if name in want else 0
        info = np.zeros(S, dtype=np.int32)
        t = Timing()
        self._check(self.lib.b2gp_posterior_multitask_grad(
            self.h, KIND[kind] if isinstance(kind, str) else kind, _ptr(Xtr), _ptr(ttr), N, _ptr(yres), stride, _ptr(Xnew), _ptr(tnew),
            P, d, int(group), T, L, S, _ptr(theta), _ptr(B), _ptr(noise), int(bool(noiseless)), float(jitter), flags, _ptr(out["mean"]),
            _ptr(out["var"]), _ptr(out["dmean"]), _ptr(out["dvar"]), info.ctypes.data_as(_vp), C.byref(t) if timing else None))
        out["info"] = info
        if timing:
            out["timing"] = t.as_dict()
        return out

    def mll_multitask(self, kind, X, task, yres, theta, B, noise, group=1, jitter=1e-6, want_grad=True, want_alpha=False, flags=0):
        """The multi-task log marginal likelihood (b2gp_mll_multitask): X [N, d], task [N], theta [L, d+2], B [L, T, T],
        noise [T].  Returns (value, grad_theta [L, d+2] (d/dlog), grad_B [L, T, T], grad_noise [T] (d/dlog), alpha, info)."""
        X, yres, B = _f64(X), _f64(yres), _f64(B)
        N, d = X.shape
        L, T = B.shape[0], B.shape[1]
        theta, noise = _f64(theta, (L, d + 2)), _f64(noise, (T,))
        task = np.ascontiguousarray(task, dtype=np.int32)
        val, info = C.c_double(0.0), C.c_int(0)
        gt, gB, gn = (np.zeros((L, d + 2)), np.zeros((L, T, T)), np.zeros(T)) if want_grad else (None, None, None)
        alpha = np.zeros(N) if want_alpha else None
        self._check(self.lib.b2gp_mll_multitask(self.h, KIND[kind] if isinstance(kind, str) else kind, _ptr(X), _ptr(task), N,
                                                _ptr(yres), d, int(group), T, L, _ptr(theta), _ptr(B), _ptr(noise), float(jitter),
                                                flags, C.byref(val), _ptr(gt), _ptr(gB), _ptr(gn), _ptr(alpha), C.byref(info)))
        return val.value, gt, gB, gn, alpha, info.value

    def mlp_forward(self, X, widths, act, params):
        """Z [S, N, d] = MLP(X) for S weight sets (b2gp_mlp_forward).  X [N, D]: a host array or a DeviceArray; widths [L]:
        the layers' output widths; act ACT_RELU / ACT_TANH; params [S, P] or [P] in the flat layout (per layer W_l [in, out]
        row-major, then b_l)."""
        X, Xp, flags = self._arg(X)
        N, D = X.shape
        w = np.ascontiguousarray(widths, dtype=np.int64).reshape(-1)
        p = _f64(params)
        p = p.reshape(1, -1) if p.ndim == 1 else p
        S = p.shape[0]
        d = int(w[-1]) if w.size else D
        Z = np.empty((S, N, d))
        self._check(self.lib.b2gp_mlp_forward(self.h, Xp, N, D, int(w.size), _ptr(w), int(act), _ptr(p) if p.size else None, S,
                                              p.shape[1], _ptr(Z), flags))
        return Z

    def dkl_mll(self, kind, X, yres, widths, act, params, theta, jitter=1e-6, want_params=True, want_z=False):
        """log N(yres; 0, K(MLP(X))) and its gradients (b2gp_dkl_mll).  X [N, D] and yres [N]: both host arrays or both
        DeviceArrays; params [P] flat layout; theta [d+3].  Returns (value, grad_theta [d+3] (d/dlog), grad_params [P] or
        None, grad_z [N, d] or None, info)."""
        X, Xp, flags = self._arg(X)
        yres, yp, yflags = self._arg(yres)
        if flags != yflags:
            raise ValueError("X and yres must both be host arrays or both DeviceArrays")
        N, D = X.shape
        w = np.ascontiguousarray(widths, dtype=np.int64).reshape(-1)
        d = int(w[-1]) if w.size else D
        theta, p = _f64(theta).reshape(d + 3), _f64(params).reshape(-1)
        val, info = C.c_double(0.0), C.c_int(0)
        gt = np.zeros(d + 3)
        gp = np.zeros(p.size) if want_params else None
        gz = np.zeros((N, d)) if want_z else None
        self._check(self.lib.b2gp_dkl_mll(self.h, KIND[kind] if isinstance(kind, str) else kind, Xp, N, D, yp, int(w.size), _ptr(w),
                                          int(act), _ptr(p) if p.size else None, _ptr(theta), float(jitter), flags, C.byref(val),
                                          _ptr(gt), _ptr(gp), _ptr(gz), C.byref(info)))
        return val.value, gt, gp, gz, info.value

    def dkl_posterior_grad(self, kind, X, yres, Xnew, widths, act, params, theta, noiseless=False, jitter=1e-6,
                           want=("mean", "var", "dmean", "dvar")):
        """The posterior on z = MLP(X) and its gradients w.r.t. the raw test inputs (b2gp_dkl_posterior_grad).  X [N, D],
        Xnew [P, D], yres [N] or [S, N]; widths [L] and act as mlp_forward; params [S, P] or [P] in the flat layout;
        theta [S, d+3] or [d+3].  Host fp64 arrays.  Returns a dict with mean / var [S, P], dmean / dvar [S, P, D] (None
        where not in `want`) and info [S]."""
        X, Xnew = _f64(X), _f64(Xnew)
        N, D = X.shape
        P = Xnew.shape[0]
        w = np.ascontiguousarray(widths, dtype=np.int64).reshape(-1)
        d = int(w[-1]) if w.size else D
        p = _f64(params)
        p = p.reshape(1, -1) if p.ndim == 1 else p
        theta = _f64(theta).reshape(-1, d + 3)
        S = theta.shape[0]
        if w.size and p.shape[0] != S:
            raise ValueError(f"{p.shape[0]} weight sets for {S} theta rows")
        if w.size and p.shape[1] != _mlp_nparams(D, w):
            raise ValueError(f"params rows have {p.shape[1]} entries, the network D={D}, widths={w.tolist()} has "
                             f"{_mlp_nparams(D, w)}")
        yres = _f64(yres)
        stride = 0 if yres.ndim == 1 else yres.shape[1]
        bits = {"mean": (OUT_MEAN, (S, P)), "var": (OUT_VAR, (S, P)), "dmean": (OUT_DMEAN, (S, P, D)), "dvar": (OUT_DVAR, (S, P, D))}
        flags, out = 0, {}
        for name, (bit, shape) in bits.items():
            out[name] = np.empty(shape) if name in want else None
            flags |= bit if name in want else 0
        info = np.zeros(S, dtype=np.int32)
        self._check(self.lib.b2gp_dkl_posterior_grad(
            self.h, KIND[kind] if isinstance(kind, str) else kind, _ptr(X), N, D, _ptr(yres), stride, _ptr(Xnew), P, int(w.size),
            _ptr(w), int(act), _ptr(p) if p.size else None, S, p.shape[1], _ptr(theta), int(bool(noiseless)), float(jitter), flags,
            _ptr(out["mean"]), _ptr(out["var"]), _ptr(out["dmean"]), _ptr(out["dvar"]), info.ctypes.data_as(_vp)))
        out["info"] = info
        return out

    def mtdkl_mll(self, kind, X, task, yres, widths, act, params, theta, B, noise, group=1, jitter=1e-6, want_params=True,
                  want_z=False):
        """The multi-task likelihood on z = MLP(X) and its gradients (b2gp_mtdkl_mll).  X [N, D] (N points, no task column)
        and yres [N * group]: both host arrays or both DeviceArrays; task [N * group]; params [P] flat layout; theta [L, d+2],
        B [L, T, T], noise [T] as mll_multitask.  Returns (value, grad_theta [L, d+2] (d/dlog), grad_B [L, T, T],
        grad_noise [T] (d/dlog), grad_params [P] or None, grad_z [N, d] or None, info)."""
        X, Xp, flags = self._arg(X)
        yres, yp, yflags = self._arg(yres)
        if flags != yflags:
            raise ValueError("X and yres must both be host arrays or both DeviceArrays")
        N, D = X.shape
        w = np.ascontiguousarray(widths, dtype=np.int64).reshape(-1)
        d = int(w[-1]) if w.size else D
        B = _f64(B)
        L, T = B.shape[0], B.shape[1]
        theta, noise, p = _f64(theta, (L, d + 2)), _f64(noise, (T,)), _f64(params).reshape(-1)
        task = np.ascontiguousarray(task, dtype=np.int32)
        val, info = C.c_double(0.0), C.c_int(0)
        gt, gB, gn = np.zeros((L, d + 2)), np.zeros((L, T, T)), np.zeros(T)
        gp = np.zeros(p.size) if want_params else None
        gz = np.zeros((N, d)) if want_z else None
        self._check(self.lib.b2gp_mtdkl_mll(self.h, KIND[kind] if isinstance(kind, str) else kind, Xp, _ptr(task), N, D, yp,
                                            int(group), T, L, int(w.size), _ptr(w), int(act), _ptr(p) if p.size else None,
                                            _ptr(theta), _ptr(B), _ptr(noise), float(jitter), flags, C.byref(val), _ptr(gt),
                                            _ptr(gB), _ptr(gn), _ptr(gp), _ptr(gz), C.byref(info)))
        return val.value, gt, gB, gn, gp, gz, info.value

    def bnn_loglik(self, X, y, widths, act, params, sigma, want_params=True):
        """sum log N(y; MLP(X), sigma) and its gradients (b2gp_bnn_loglik).  X [N, D] and y [N, O]: both host arrays or both
        DeviceArrays; widths [L] with widths[-1] = O; params [P] flat layout.  Returns (value, d/dsigma, grad_params [P] or
        None)."""
        X, Xp, flags = self._arg(X)
        y, yp, yflags = self._arg(y)
        if flags != yflags:
            raise ValueError("X and y must both be host arrays or both DeviceArrays")
        N, D = X.shape
        w = np.ascontiguousarray(widths, dtype=np.int64).reshape(-1)
        p = _f64(params).reshape(-1)
        if p.size != _mlp_nparams(D, w):
            raise ValueError(f"params has {p.size} entries, the network D={D}, widths={w.tolist()} has {_mlp_nparams(D, w)}")
        if tuple(y.shape) != (N, int(w[-1])):
            raise ValueError(f"y has shape {tuple(y.shape)}, the network needs ({N}, {int(w[-1])})")
        val, gs = C.c_double(0.0), C.c_double(0.0)
        gp = np.zeros(p.size) if want_params else None
        self._check(self.lib.b2gp_bnn_loglik(self.h, Xp, N, D, yp, int(w[-1]), int(w.size), _ptr(w), int(act), _ptr(p),
                                             float(sigma), flags, C.byref(val), C.byref(gs), _ptr(gp)))
        return val.value, gs.value, gp

    def bnn_loglik_draws(self, X, y, widths, act, params, sigma, want_params=True):
        """bnn_loglik for S weight sets on one X and y (b2gp_bnn_loglik_draws): draw s is bnn_loglik(X, y, widths, act,
        params[s], sigma[s]) bit for bit.  X, y as in bnn_loglik; params [S, P] (rows may be a strided view's) and sigma
        [S].  Returns (values [S], d/dsigma [S], grad_params [S, P] or None)."""
        X, Xp, flags = self._arg(X)
        y, yp, yflags = self._arg(y)
        if flags != yflags:
            raise ValueError("X and y must both be host arrays or both DeviceArrays")
        N, D = X.shape
        w = np.ascontiguousarray(widths, dtype=np.int64).reshape(-1)
        p = np.asarray(params, dtype=np.float64)
        if p.ndim != 2 or p.shape[1] != _mlp_nparams(D, w):
            raise ValueError(f"params has shape {p.shape}, expected (S, {_mlp_nparams(D, w)}) for D={D}, widths={w.tolist()}")
        if p.strides[1] != 8 or p.strides[0] % 8 or p.strides[0] < 8 * p.shape[1]:
            p = np.ascontiguousarray(p)
        S = p.shape[0]
        sg = _f64(sigma).reshape(-1)
        if sg.size != S:
            raise ValueError(f"sigma has {sg.size} entries for {S} weight sets")
        if tuple(y.shape) != (N, int(w[-1])):
            raise ValueError(f"y has shape {tuple(y.shape)}, the network needs ({N}, {int(w[-1])})")
        val, gs = np.empty(S), np.empty(S)
        gp = np.empty((S, p.shape[1])) if want_params else None
        self._check(self.lib.b2gp_bnn_loglik_draws(self.h, Xp, N, D, yp, int(w[-1]), int(w.size), _ptr(w), int(act), S, _ptr(p),
                                                   p.strides[0] // 8, _ptr(sg), flags, _ptr(val), _ptr(gs), _ptr(gp)))
        return val, gs, gp

    def bnn_predict(self, X, widths, act, params, sigma=None, eps=None):
        """loc [S, P, O] = MLP(X) for S weight sets and, given eps [S, n, P, O] and sigma [S], y_sampled [S, P, O] =
        loc + sigma * mean_k eps (b2gp_bnn_predict).  X [P, D]: a host array or a DeviceArray; params [S, P] or [P].
        Returns (loc, y_sampled or None)."""
        X, Xp, flags = self._arg(X)
        Pn, D = X.shape
        w = np.ascontiguousarray(widths, dtype=np.int64).reshape(-1)
        p = _f64(params)
        p = p.reshape(1, -1) if p.ndim == 1 else p
        S, O = p.shape[0], int(w[-1])
        if p.shape[1] != _mlp_nparams(D, w):
            raise ValueError(f"params rows have {p.shape[1]} entries, the network D={D}, widths={w.tolist()} has "
                             f"{_mlp_nparams(D, w)}")
        loc = np.empty((S, Pn, O))
        ys, n, sg = None, 0, None
        if eps is not None:
            eps = _f64(eps)
            if eps.ndim != 4 or eps.shape[0] != S or eps.shape[2:] != (Pn, O):
                raise ValueError(f"eps has shape {eps.shape}, expected ({S}, n, {Pn}, {O})")
            n = eps.shape[1]
            sg = _f64(np.broadcast_to(np.asarray(sigma, dtype=np.float64).reshape(-1), (S,)))
            ys = np.empty((S, Pn, O))
        self._check(self.lib.b2gp_bnn_predict(self.h, Xp, Pn, D, int(w.size), _ptr(w), int(act), _ptr(p), S, p.shape[1], O,
                                              _ptr(sg), _ptr(eps), n, _ptr(loc), _ptr(ys), flags))
        return loc, ys

    def bnn_predict_grad(self, X, widths, act, params):
        """loc [S, P] = MLP(X) of a one-output network for S weight sets and dloc [S, P, D] = d loc / dX
        (b2gp_bnn_predict_grad).  X [P, D] and params [S, P] or [P]: both host arrays or both DeviceArrays, so that an
        optimisation can keep the weight sets on the device.  Returns (loc, dloc)."""
        X, Xp, flags = self._arg(X)
        p, pp, pflags = self._arg(params)
        if flags != pflags:
            raise ValueError("X and params must both be host arrays or both DeviceArrays")
        Pn, D = X.shape
        w = np.ascontiguousarray(widths, dtype=np.int64).reshape(-1)
        shape = tuple(p.shape)
        S, npar = (1, shape[0]) if len(shape) == 1 else shape
        if npar != _mlp_nparams(D, w):
            raise ValueError(f"params rows have {npar} entries, the network D={D}, widths={w.tolist()} has {_mlp_nparams(D, w)}")
        loc, dloc = np.empty((S, Pn)), np.empty((S, Pn, D))
        self._check(self.lib.b2gp_bnn_predict_grad(self.h, Xp, Pn, D, int(w.size), _ptr(w), int(act), pp, S, npar, _ptr(loc),
                                                   _ptr(dloc), flags))
        return loc, dloc

    @staticmethod
    def _arg(a):
        """(array, pointer, flags) of a host array (made C-contiguous fp64) or a DeviceArray"""
        if isinstance(a, DeviceArray):
            return a, a.ptr, FLAG_DEVICE_PTRS
        a = _f64(a)
        return a, _ptr(a), 0

    def sparse_elbo(self, kind, Xu, X, yres, theta, jitter=1e-6, want_alpha=False):
        """VFE bound of the sparse GP, its gradient w.r.t. log(lengthscale[d], k_scale, noise, period) and w.r.t. Xu:
        (value, grad_theta, grad_Xu, info), with alpha = (W^T W + noise I)^-1 yres = d value / d mean appended when
        want_alpha (b2gp_sparse_elbo_ex)"""
        Xu, X, yres = _f64(Xu), _f64(X), _f64(yres)
        M, d = Xu.shape
        N = X.shape[0]
        theta = _f64(theta).reshape(d + 3)
        val, info = C.c_double(0.0), C.c_int(0)
        g, gx = np.zeros(d + 3), np.zeros((M, d))
        alpha = np.zeros(N) if want_alpha else None
        self._check(self.lib.b2gp_sparse_elbo_ex(self.h, KIND[kind] if isinstance(kind, str) else kind, _ptr(Xu), M, _ptr(X), N,
                                                 _ptr(yres), d, _ptr(theta), float(jitter), 0, C.byref(val), _ptr(g), _ptr(gx),
                                                 _ptr(alpha), C.byref(info)))
        if want_alpha:
            return val.value, g, gx, info.value, alpha
        return val.value, g, gx, info.value

    def sparse_elbo_gram(self, Kuu, Kuf, kff_diag, yres, noise, dirs=(), rdirs=(), want_alpha=False, flags=0):
        """The VFE bound from caller-supplied blocks (b2gp_sparse_elbo_gram): Kuu [M, M], Kuf [M, N], kff_diag [N], yres [N].
        `dirs` is a list of (dKuu, dKuf, dkff) triples and `rdirs` of (rKuu, rKuf) pairs; any block may be None.  All
        arrays are NumPy, or all DeviceArrays (B2GP_FLAG_DEVICE_PTRS); `flags` adds further bits.  Returns a dict: value,
        grad [len(dirs)],
        grad_log_noise, grad_rows [len(rdirs), M], alpha [N] or None, info."""
        dev = isinstance(Kuu, DeviceArray)
        conv = (lambda a: a) if dev else (lambda a: None if a is None else _f64(a))
        Kuu, Kuf, kff_diag, yres = conv(Kuu), conv(Kuf), conv(kff_diag), conv(yres)
        dirs = [tuple(conv(b) for b in t) for t in dirs]
        rdirs = [tuple(conv(b) for b in t) for t in rdirs]
        M, N = Kuu.shape[0], Kuf.shape[1]
        shapes = [((M, M), (M, N), (N,))[t] for t in range(3)]
        for a, shp in [(Kuu, shapes[0]), (Kuf, shapes[1]), (kff_diag, shapes[2]), (yres, shapes[2])] + \
                [(b, shapes[t]) for tr in dirs for t, b in enumerate(tr)] + [(b, shapes[t]) for pr in rdirs for t, b in enumerate(pr)]:
            if a is not None and tuple(a.shape) != shp:
                raise ValueError(f"block of shape {tuple(a.shape)}: expected {shp}")
        ptr = (lambda a: None if a is None else a.ptr.value) if dev else (lambda a: None if a is None else a.ctypes.data)
        p, q = len(dirs), len(rdirs)
        tables = [(C.c_void_p * max(n, 1))(*[ptr(t[k]) for t in seq])
                  for seq, n, ks in ((dirs, p, 3), (rdirs, q, 2)) for k in range(ks)]
        val, gln, info = C.c_double(0.0), C.c_double(0.0), C.c_int(0)
        grad, rows = np.zeros(p), np.zeros((q, M))
        alpha = np.zeros(N) if want_alpha else None
        vp = (lambda a: a.ptr) if dev else _ptr
        self._check(self.lib.b2gp_sparse_elbo_gram(
            self.h, vp(Kuu), M, vp(Kuf), N, vp(kff_diag), vp(yres), float(noise), C.cast(tables[0], _vp), C.cast(tables[1], _vp),
            C.cast(tables[2], _vp), p, C.cast(tables[3], _vp), C.cast(tables[4], _vp), q, (FLAG_DEVICE_PTRS if dev else 0) | flags,
            C.byref(val), _ptr(grad), C.byref(gln), _ptr(rows), _ptr(alpha), C.byref(info)))
        return {"value": val.value, "grad": grad, "grad_log_noise": gln.value, "grad_rows": rows, "alpha": alpha,
                "info": info.value}

    def sparse_posterior_gram(self, Kuu, Kuf, yres, noise, Kus, Kss=None, want=("mean", "cov"), kss_diag=False):
        """The sparse posterior from caller-supplied blocks (b2gp_sparse_posterior_gram): Kuu [M, M], Kuf [M, N], Kus [M, P]
        and Kss [P, P] -- or with kss_diag its diagonal [P] (mean / var only) -- host fp64 arrays; outputs as
        sparse_posterior()."""
        Kuu, Kuf, Kus, yres = _f64(Kuu), _f64(Kuf), _f64(Kus), _f64(yres)
        M, N, P = Kuu.shape[0], Kuf.shape[1], Kus.shape[1]
        Kss = None if Kss is None else _f64(Kss)
        for a, shp in ((Kuu, (M, M)), (Kuf, (M, N)), (Kus, (M, P)), (yres, (N,)), (Kss, (P,) if kss_diag else (P, P))):
            if a is not None and a.shape != shp:
                raise ValueError(f"block of shape {a.shape}: expected {shp}")
        flags = FLAG_KPP_DIAG if kss_diag else 0
        out = {"mean": None, "var": None, "cov": None}
        for name, bit, shape in (("mean", OUT_MEAN, (P,)), ("var", OUT_VAR, (P,)), ("cov", OUT_COV, (P, P))):
            if name in want:
                flags |= bit
                out[name] = np.empty(shape)
        info = np.zeros(1, dtype=np.int32)
        t = Timing()
        self._check(self.lib.b2gp_sparse_posterior_gram(
            self.h, _ptr(Kuu), M, _ptr(Kuf), N, _ptr(yres), float(noise), _ptr(Kus), _ptr(Kss), P, flags, _ptr(out["mean"]),
            _ptr(out["var"]), _ptr(out["cov"]), info.ctypes.data_as(_ip), C.byref(t)))
        out["info"] = int(info[0])
        out["timing"] = t.as_dict()
        return out

    def sparse_posterior(self, kind, Xu, Xtr, yres, Xnew, theta, noiseless=False, jitter=1e-6, want=("mean", "cov")):
        Xu, Xtr, Xnew = _f64(Xu), _f64(Xtr), _f64(Xnew)
        M, d = Xu.shape
        N, P = Xtr.shape[0], Xnew.shape[0]
        theta = _f64(theta).reshape(d + 3)
        yres = _f64(yres).reshape(N)
        flags = 0
        mean = var = cov = None
        if "mean" in want:
            flags |= OUT_MEAN
            mean = np.empty(P)
        if "var" in want:
            flags |= OUT_VAR
            var = np.empty(P)
        if "cov" in want:
            flags |= OUT_COV
            cov = np.empty((P, P))
        info = np.zeros(1, dtype=np.int32)
        t = Timing()
        self._check(self.lib.b2gp_sparse_posterior(
            self.h, KIND[kind] if isinstance(kind, str) else kind, _ptr(Xu), M, _ptr(Xtr), N, _ptr(yres), _ptr(Xnew), P, d,
            _ptr(theta), int(bool(noiseless)), float(jitter), flags, _ptr(mean), _ptr(var), _ptr(cov),
            info.ctypes.data_as(_vp), C.byref(t)))
        return {"mean": mean, "var": var, "cov": cov, "info": int(info[0]), "timing": t.as_dict()}


ACQ = {"EI": 0, "UCB": 1, "UE": 2, "POI": 3}


def _acq_moments(self, kind, mean, var, best_f=None, param=0.0, maximize=False):
    """acquisition function `kind` on moments [P] or [R, P] (host arrays)"""
    var = _f64(var)
    shape = var.shape
    var = var.reshape(-1, shape[-1])
    mean = None if mean is None else _f64(mean).reshape(var.shape)
    out = np.empty_like(var)
    self._check(self.lib.b2gp_acq_moments(self.h, ACQ[kind], _ptr(mean), _ptr(var), var.shape[0], var.shape[1],
                                          int(best_f is not None), float(best_f or 0.0), float(param), int(bool(maximize)),
                                          _ptr(out), 0))
    return out.reshape(shape)


def _acq_samples(self, kind, y, best_f=None, param=0.0, maximize=False):
    """moments over the rows of y [R, P], then the acquisition function; returns (acq, mean, var)"""
    y = _f64(y)
    y = y.reshape(-1, y.shape[-1])
    R, P = y.shape
    out, mean, var = np.empty(P), np.empty(P), np.empty(P)
    self._check(self.lib.b2gp_acq_samples(self.h, ACQ[kind], _ptr(y), R, P, int(best_f is not None), float(best_f or 0.0),
                                          float(param), int(bool(maximize)), _ptr(out), _ptr(mean), _ptr(var), 0))
    return out, mean, var


def _kg(self, mean, cov, ysim, diag_sub, noise_plus_jitter, maximize=True):
    """diag_sub and noise_plus_jitter: scalars (b2gp_kg) or one value per candidate [P] (b2gp_kg_v)"""
    mean, cov, ysim = _f64(mean), _f64(cov), _f64(ysim)
    P = mean.shape[0]
    ysim = ysim.reshape(-1, P)
    out = np.empty(P)
    if np.ndim(diag_sub) == 0 and np.ndim(noise_plus_jitter) == 0:
        self._check(self.lib.b2gp_kg(self.h, _ptr(mean), _ptr(cov), P, _ptr(ysim), ysim.shape[0], float(diag_sub),
                                     float(noise_plus_jitter), int(bool(maximize)), _ptr(out), 0))
        return out
    ds = _f64(np.broadcast_to(np.asarray(diag_sub, dtype=np.float64), (P,)))
    nj = _f64(np.broadcast_to(np.asarray(noise_plus_jitter, dtype=np.float64), (P,)))
    self._check(self.lib.b2gp_kg_v(self.h, _ptr(mean), _ptr(cov), P, _ptr(ysim), ysim.shape[0], _ptr(ds), _ptr(nj),
                                   int(bool(maximize)), _ptr(out), 0))
    return out


def _mvn_sample(self, mean, cov, eps):
    """mean [S, P], cov [S, P, P], eps [S, n, P] -> (mean + chol(cov) eps [S, n, P], info [S])"""
    mean, cov, eps = _f64(mean), _f64(cov), _f64(eps)
    P = mean.shape[-1]
    mean, cov = mean.reshape(-1, P), cov.reshape(-1, P, P)
    S = mean.shape[0]
    eps = eps.reshape(S, -1, P)
    y = np.empty_like(eps)
    info = np.zeros(S, dtype=np.int32)
    self._check(self.lib.b2gp_mvn_sample(self.h, _ptr(mean), _ptr(cov), S, P, _ptr(eps), eps.shape[1], _ptr(y),
                                         info.ctypes.data_as(_vp), 0))
    return y, info


Context.acq_moments, Context.acq_samples, Context.kg, Context.mvn_sample = _acq_moments, _acq_samples, _kg, _mvn_sample

_default_ctx = None


def default_context():
    """Process-wide context on the device named by LOCAL_RANK / B200GP_DEVICE (default 0)."""
    global _default_ctx
    if _default_ctx is None or _default_ctx.h is None:
        dev = int(os.environ.get("B200GP_DEVICE", os.environ.get("LOCAL_RANK", "0")))
        _default_ctx = Context(dev)
    return _default_ctx
