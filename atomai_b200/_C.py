"""
ctypes binding of libatomai_b200.so (the C ABI declared in include/atomai_b200.h).

The library is the product: there is no Python/torch fallback for any entry
point.  Importing this module never needs a GPU (the driver's CPU-side checks
load the library and verify every exported symbol); calling a kernel without
one fails loudly.
"""
import ctypes as C
import os
import subprocess
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libatomai_b200.so")
CSRC = os.path.join(_HERE, "csrc")
SOURCES = ["api.cu", "conv_tc.cu", "conv_simt.cu", "wgrad_tc.cu", "elementwise.cu",
           "selftest_tma.cu", "vae.cu", "gram.cu", "frontend.cu", "augment.cu", "p2p.cu", "resnet.cu",
           "segloss.cu", "refine.cu", "jlatent.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo",
              "-std=c++17", "-Xcompiler", "-fPIC", "-shared"]

ACT_LRELU = 0
ACT_TANH = 1
MATH_FP32 = 0
MATH_TF32 = 1
MATH_TF32X3 = 2
WMODE_FWD = 0
WMODE_DGRAD = 1
REFINE_NONFINITE = -2    # AB_REFINE_NONFINITE of include/atomai_b200.h
JLAT_MAX_CONT = 32       # AB_JLAT_MAX_CONT
JLAT_MAX_DISC = 64       # AB_JLAT_MAX_DISC
JLAT_ALPHAS = 0
JLAT_SAMPLE = 1


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile every CUDA source for sm_90a into libatomai_b200.so (in-tree)."""
    srcs = [os.path.join(CSRC, s) for s in SOURCES]
    deps = srcs + [os.path.join(CSRC, "common.cuh"), os.path.join(CSRC, "wgmma.cuh"),
                   os.path.join(_HERE, "..", "include", "atomai_b200.h")]
    if not force and os.path.exists(LIB_PATH):
        t = os.path.getmtime(LIB_PATH)
        if all(os.path.getmtime(d) <= t for d in deps):
            return LIB_PATH
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + NVCC_FLAGS + ["-o", LIB_PATH] + srcs
    if verbose:
        print(" ".join(cmd), file=sys.stderr)
    subprocess.run(cmd, check=True)
    return LIB_PATH


class Src(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("scale", C.c_void_p), ("shift", C.c_void_p),
                ("C", C.c_int32), ("ld", C.c_int32), ("pool", C.c_int32),
                ("reserved", C.c_int32)]


class Conv(C.Structure):
    _fields_ = [("N", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("Cout", C.c_int32),
                ("ks_h", C.c_int32), ("ks_w", C.c_int32), ("dil", C.c_int32),
                ("nsrc", C.c_int32), ("src", Src * 2), ("lrelu", C.c_float),
                ("math", C.c_int32), ("out_nchw", C.c_int32), ("act", C.c_int32)]


class CoordLat(C.Structure):
    _fields_ = [("B", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("zdim", C.c_int32),
                ("hid", C.c_int32), ("tanh_act", C.c_int32),
                ("z", C.c_void_p), ("phi", C.c_void_p), ("dx", C.c_void_p),
                ("wc", C.c_void_p), ("bc", C.c_void_p), ("wz", C.c_void_p)]


class JLat(C.Structure):
    _fields_ = [("B", C.c_int32), ("Dc", C.c_int32), ("coord", C.c_int32), ("nheads", C.c_int32),
                ("heads", C.c_int32 * JLAT_MAX_DISC), ("tau", C.c_float), ("phi_prior", C.c_float),
                ("dx_prior", C.c_float)]


_vp, _i, _i64, _f, _d = C.c_void_p, C.c_int, C.c_int64, C.c_float, C.c_double

# name -> (restype, argtypes); mirrors include/atomai_b200.h one to one
SIGNATURES = {
    "atomai_b200_version": (C.c_char_p, []),
    "atomai_b200_last_error": (C.c_char_p, []),
    "atomai_b200_device_ok": (_i, [_i]),
    "atomai_b200_prep_weights_elems": (_i64, [_i, _i, _i, _i, _i, _i]),
    "atomai_b200_prep_weights": (_i, [_vp, _i, _i, _i, _i, _i, _i, _vp, _vp]),
    "atomai_b200_conv_fwd": (_i, [C.POINTER(Conv), _vp, _vp, _vp, _i, _vp, _vp]),
    "atomai_b200_conv_supported": (_i, [C.POINTER(Conv), _i]),
    "atomai_b200_conv_info": (_i, [C.POINTER(Conv), C.POINTER(_i), C.POINTER(_i), C.POINTER(_i)]),
    "atomai_b200_conv_wgrad": (_i, [C.POINTER(Conv), _vp, _i, _vp, _vp]),
    "atomai_b200_bn_finalize": (_i, [_vp, _i, _d, _vp, _vp, _vp, _vp, _f, _f, _i, _vp, _vp, _vp,
                                     _vp, _vp]),
    "atomai_b200_affine": (_i, [_vp, _i, _vp, _vp, _vp, _i, _i64, _i, _i, _vp]),
    "atomai_b200_bn_bwd_reduce": (_i, [_vp, _i, _vp, _i, _vp, _vp, _i64, _i, _vp, _vp]),
    "atomai_b200_bn_lrelu_bwd": (_i, [_vp, _i, _vp, _i, _vp, _vp, _vp, _vp, _d, _vp, _i, _i, _f,
                                      _vp, _i, _vp, _i64, _i, _vp]),
    "atomai_b200_pool2x2_fwd": (_i, [_vp, _i, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "atomai_b200_pool2x2_bwd": (_i, [_vp, _i, _vp, _i, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i,
                                     _vp]),
    "atomai_b200_pool2x2_bwd_bn": (_i, [_vp, _i, _vp, _i, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i,
                                     _vp, _vp, _vp, _vp]),
    "atomai_b200_affine_res_act": (_i, [_vp, _i, _vp, _vp, _vp, _i, _f, _vp, _i, _i64, _i, _vp]),
    "atomai_b200_lrelu_mask_bwd": (_i, [_vp, _i, _vp, _i, _f, _vp, _i, _i64, _i, _vp]),
    "atomai_b200_resize_fwd": (_i, [_vp, _i, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "atomai_b200_resize_bwd": (_i, [_vp, _i, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "atomai_b200_upsample2x_fwd": (_i, [_vp, _i, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "atomai_b200_upsample2x_bwd": (_i, [_vp, _i, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "atomai_b200_transpose": (_i, [_vp, _vp, _i, _i, _i, _vp]),
    "atomai_b200_add_slice": (_i, [_vp, _i, _vp, _i, _i, _i64, _i, _vp]),
    "atomai_b200_dilated_sum": (_i, [C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp), _i, _f, _vp,
                                     _i64, _i, _vp]),
    "atomai_b200_ce_fwd_bwd": (_i, [_vp, _i, _vp, _i64, _i, _vp, _vp, _i, _f, _vp, _vp]),
    "atomai_b200_pointwise_loss": (_i, [_vp, _vp, _i64, _i, _vp, _vp, _f, _vp, _vp]),
    "atomai_b200_dice_sums": (_i, [_vp, _i, _vp, _i, _i, _i, _i, _i, _vp, _vp]),
    "atomai_b200_dice_finalize": (_i, [_vp, _i, _f, _vp, _vp, _vp]),
    "atomai_b200_dice_bwd": (_i, [_vp, _i, _vp, _i, _i, _i, _i, _i, _vp, _vp, _i, _f, _vp, _vp]),
    "atomai_b200_focal_finalize": (_i, [_vp, _d, _f, _f, _vp, _vp, _vp]),
    "atomai_b200_iou_hist": (_i, [_vp, _i, _vp, _i, _i64, _i, _i, _f, _vp, _vp]),
    "atomai_b200_iou_finalize": (_i, [_vp, _i, _vp, _vp]),
    "atomai_b200_adam_multi": (_i, [_vp, _i, _i64, _f, _f, _f, _f, _f, _i, _f, _vp]),
    "atomai_b200_linear_fwd": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "atomai_b200_linear_bwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "atomai_b200_gemm": (_i, [_vp, _i64, _i64, _vp, _i64, _i64, _vp, _i64, _i, _i, _i, _vp, _i,
                              _f, _i, _i, _vp]),
    "atomai_b200_coord_latent_fwd": (_i, [C.POINTER(CoordLat), _vp, _vp]),
    "atomai_b200_coord_latent_bwd": (_i, [C.POINTER(CoordLat), _vp, _vp, _vp, _vp, _vp, _vp,
                                          _vp]),
    "atomai_b200_jlatent_fwd": (_i, [C.POINTER(JLat), _i, _vp, _vp, _vp, _vp, _vp, C.c_uint64, _vp,
                                     _vp, _vp, _vp, _vp, _vp]),
    "atomai_b200_jlatent_bwd": (_i, [C.POINTER(JLat), _i, _vp, _vp, _vp, _vp, _vp, C.c_uint64, _vp,
                                     _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "atomai_b200_sqerr_reduce": (_i, [_vp, _vp, _i64, _vp, _vp, _f, _vp, _vp]),
    "atomai_b200_gram_workspace_bytes": (_i64, [_i, _i, _i]),
    "atomai_b200_gram": (_i, [_vp, _vp, _vp, _f, _i, _i, _i, _i, _i, _vp, _i64, _vp, _i64, _vp]),
    "atomai_b200_prob_mask": (_i, [_vp, _i, _i64, _i, _i, _f, _vp, _i, _vp, _vp]),
    "atomai_b200_gather_windows": (_i, [_vp, _i, _i, _i, _i, _vp, _i, _i, _vp, _vp, _vp]),
    "atomai_b200_peak_refine": (_i, [_vp, _i, _i, _i, _vp, _i, _i, _vp, _vp, _vp, _vp]),
    "atomai_b200_rowloss": (_i, [_vp, _vp, _i, _i64, _i, _vp, _vp, _vp, _vp]),
    "atomai_b200_dropout": (_i, [_vp, _i, _i64, _i, _f, C.c_uint64, _vp, _vp]),
    "atomai_b200_augment": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _f, _f, C.c_uint64,
                                 _vp, _vp]),
    "atomai_b200_ipc_export": (_i, [_vp, _vp, C.POINTER(_i64)]),
    "atomai_b200_ipc_import": (_i, [_vp, _i64, C.POINTER(_vp)]),
    "atomai_b200_p2p_data_bytes": (_i64, [_i]),
    "atomai_b200_p2p_flag_bytes": (_i64, [_i]),
    "atomai_b200_p2p_allreduce": (_i, [_vp, _vp, _i, _i, C.c_uint64, _vp, _i, _vp]),
    "atomai_b200_p2p_bn_finalize": (_i, [_vp, _vp, _i, _i, C.c_uint64, _vp, _i, _d, _vp, _vp, _vp,
                                         _vp, _f, _f, _vp, _vp, _vp, _vp, _vp]),
    "atomai_b200_selftest_tma": (_i, [_vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp]),
}

_lib = None


def lib():
    """Load (once) and return the ctypes handle; raises if the native library is missing."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not built: run `python -c 'import __graft_entry__ as g; g.build()'`"
                " — atomai_b200 has no non-CUDA fallback")
        _lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(_lib, name)
            fn.restype = res
            fn.argtypes = args
    return _lib


class NativeError(RuntimeError):
    pass


_LAUNCHES = [0]


def check(status: int) -> None:
    """Every kernel-launching ABI call funnels through here (count = lower bound on launches)."""
    _LAUNCHES[0] += 1
    if status != 0:
        raise NativeError(lib().atomai_b200_last_error().decode())


def launch_count() -> int:
    return _LAUNCHES[0]


def ptr(t):
    """Device pointer of a torch tensor (None -> NULL)."""
    return None if t is None else t.data_ptr()


def stream_ptr():
    import torch
    return torch.cuda.current_stream().cuda_stream
