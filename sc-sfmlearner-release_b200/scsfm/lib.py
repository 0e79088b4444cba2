"""ctypes binding of libscsfm.so (C ABI: include/scsfm.h).

There is NO fallback: if the shared library is missing or an entry point fails, an
exception is raised.  Kernels are enqueued on torch's current CUDA stream.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libscsfm.so")
MAX_JOBS = 16

WITH_SSIM, WITH_MASK, WITH_AUTO_MASK = 1, 2, 4
PAD_ZEROS, PAD_BORDER = 0, 1

c_float_p = ctypes.c_void_p


class PairJob(ctypes.Structure):
    _fields_ = [("tgt_img", ctypes.c_void_p), ("ref_img", ctypes.c_void_p), ("tgt_depth", ctypes.c_void_p),
                ("ref_depth", ctypes.c_void_p), ("pose", ctypes.c_void_p), ("grad_tgt_depth", ctypes.c_void_p),
                ("grad_ref_depth", ctypes.c_void_p), ("grad_pose", ctypes.c_void_p), ("tgt_shift", ctypes.c_int),
                ("ref_shift", ctypes.c_int)]


class PairMaps(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in ("warped", "valid", "proj_depth", "comp_depth", "mask", "diff_img",
                                               "diff_depth")]


class SmoothJob(ctypes.Structure):
    _fields_ = [("depth", ctypes.c_void_p), ("img", ctypes.c_void_p), ("grad_depth", ctypes.c_void_p)]


class EvalDepthImage(ctypes.Structure):
    _fields_ = [("gt_offset", ctypes.c_longlong), ("H", ctypes.c_int), ("W", ctypes.c_int), ("y1", ctypes.c_int), ("y2", ctypes.c_int),
                ("x1", ctypes.c_int), ("x2", ctypes.c_int)]


_lib = None


def load():
    """Load libscsfm.so; raises if it has not been built (python __graft_entry__.py / build.sh)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError("libscsfm.so not found at %s -- build it with sc-sfmlearner-release_b200/build.sh; "
                           "there is no CPU fallback" % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    lib.scsfm_last_error.restype = ctypes.c_char_p
    lib.scsfm_version.restype = ctypes.c_int
    lib.scsfm_launch_count.restype = ctypes.c_longlong
    lib.scsfm_pairwise_stats_bytes.restype = ctypes.c_size_t
    lib.scsfm_pairwise_stats_bytes.argtypes = [ctypes.c_int, ctypes.c_int]
    lib.scsfm_smooth_stats_bytes.restype = ctypes.c_size_t
    lib.scsfm_smooth_stats_bytes.argtypes = [ctypes.c_int, ctypes.c_int]
    I, P = ctypes.c_int, ctypes.c_void_p
    lib.scsfm_pairwise_fwd.argtypes = [ctypes.POINTER(PairJob), I, P, I, I, I, I, I, P, P, ctypes.POINTER(PairMaps), P]
    lib.scsfm_pairwise_bwd.argtypes = [ctypes.POINTER(PairJob), I, P, I, I, I, I, I, P, P, P]
    lib.scsfm_inverse_warp2_fwd.argtypes = [P, P, P, P, P, I, I, I, I, P, P, P, P, P]
    lib.scsfm_inverse_warp2_bwd.argtypes = [P, P, P, P, P, I, I, I, I, P, P, P, P, P, P, P, P]
    lib.scsfm_pairwise_intrinsics_grad.argtypes = [ctypes.POINTER(PairJob), I, P, I, P, P, P]
    lib.scsfm_inverse_warp2_intrinsics_grad.argtypes = [P, P, I, P, P, P]
    lib.scsfm_pose_vec2mat.argtypes = [P, I, I, P, P]
    lib.scsfm_smooth_fwd.argtypes = [ctypes.POINTER(SmoothJob), I, I, I, I, P, P, P]
    lib.scsfm_smooth_bwd.argtypes = [ctypes.POINTER(SmoothJob), I, I, I, I, P, P, P]
    lib.scsfm_eval_depth_workspace_bytes.restype = ctypes.c_size_t
    lib.scsfm_eval_depth_workspace_bytes.argtypes = [ctypes.POINTER(EvalDepthImage), I]
    lib.scsfm_eval_depth.argtypes = [P, I, I, I, P, I, ctypes.c_longlong, ctypes.POINTER(EvalDepthImage), ctypes.c_double,
                                     ctypes.c_double, P, ctypes.c_size_t, P, P]
    _lib = lib
    return lib


def check(rc, what):
    if rc != 0:
        msg = load().scsfm_last_error().decode()
        if rc == -1:
            raise ValueError("%s: %s" % (what, msg))
        raise RuntimeError("%s: %s" % (what, msg))


def stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def dev_f32(t, name):
    """Contiguous fp32 CUDA tensor or a loud error (no silent CPU path)."""
    if not t.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor: the H100 path has no CPU fallback" % name)
    if t.dtype != torch.float32:
        raise TypeError("%s must be float32, got %s" % (name, t.dtype))
    return t.contiguous()


# ----- launch accounting / optional per-family CUDA-event profiling (used by bench.py) -------------
def launch_count():
    """Kernels launched by libscsfm so far in this process (counted at every launch site inside the library)."""
    return int(load().scsfm_launch_count())


PROF = {"enabled": False, "only": None, "events": []}


TAG = {"next": None}      # optional shape label attached to the next profiled launch (tools/profile_layers.py)


def launch(fn, what, family, n_kernels, work, *args):
    """Call a C-ABI entry point; optionally bracket it with CUDA events on the launching stream.
    `work` = algorithmic FLOPs (convs) or bytes (HBM-bound ops) of the call; `n_kernels` is documentation only
    (the library counts its own launches: launch_count())."""
    if PROF["enabled"] and (PROF["only"] is None or family in PROF["only"]):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        rc = fn(*args)
        e1.record()
        PROF["events"].append((family, work, e0, e1, TAG["next"]))
        TAG["next"] = None
    else:
        rc = fn(*args)
    check(rc, what)
