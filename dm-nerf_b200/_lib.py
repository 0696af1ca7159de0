"""ctypes binding of libdmnerf_b200.so (C ABI: include/dmnerf_b200.h).

No torch types cross the boundary: tensors are passed as raw device pointers (`tensor.data_ptr()`)
plus sizes and the current CUDA stream handle.  There is NO CPU fallback: if the shared library is
missing or a call fails, a RuntimeError is raised with the library's own message.
"""
import ctypes as C
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
# DMNERF_LIB_PATH: diagnostics builds of the same ABI (tools/kprof.py); the default is the in-tree product library
LIB_PATH = os.environ.get("DMNERF_LIB_PATH") or os.path.join(_HERE, "lib", "libdmnerf_b200.so")

ABI_VERSION = 1
N_PARAMS = 30
IMPL_AUTO, IMPL_SIMT, IMPL_UMMA = 0, 1, 2
FLAG_PERTURB, FLAG_WANT_RAW, FLAG_KEEP_INS = 1, 2, 4

_f32p = C.c_void_p


class RenderIO(C.Structure):
    """Mirror of `struct dmnerf_render_io`."""
    _fields_ = [
        ("rays_o", _f32p), ("rays_d", _f32p), ("z_coarse", _f32p), ("z_row_stride", C.c_int64),
        ("t_rand", _f32p), ("u", _f32p),
        ("rgb_coarse", _f32p), ("rgb_fine", _f32p), ("depth_coarse", _f32p), ("depth_fine", _f32p),
        ("acc_coarse", _f32p), ("acc_fine", _f32p), ("ins_coarse", _f32p), ("ins_fine", _f32p),
        ("z_vals_coarse", _f32p), ("z_vals_fine", _f32p), ("weights_coarse", _f32p), ("weights_fine", _f32p),
        ("raw_coarse", _f32p), ("raw_fine", _f32p),
    ]


# name -> (restype, argtypes); every symbol declared in include/dmnerf_b200.h
PROTOTYPES = {
    "dmnerf_abi_version": (C.c_int, []),
    "dmnerf_last_error": (C.c_char_p, []),
    "dmnerf_launch_count": (C.c_int64, []),
    "dmnerf_ctx_create": (C.c_int, [C.c_int, C.POINTER(C.c_void_p)]),
    "dmnerf_ctx_destroy": (C.c_int, [C.c_void_p]),
    "dmnerf_set_weights": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_void_p]),
    "dmnerf_posenc": (C.c_int, [_f32p, C.c_int64, C.c_int, _f32p, C.c_void_p]),
    "dmnerf_mlp_forward": (C.c_int, [C.c_void_p, C.c_int, _f32p, C.c_int64, _f32p, C.c_int, C.c_void_p]),
    "dmnerf_mlp_forward_rays": (C.c_int, [C.c_void_p, C.c_int, _f32p, _f32p, _f32p, C.c_int64, C.c_int, _f32p, C.c_int,
                                          C.c_void_p]),
    "dmnerf_composite": (C.c_int, [_f32p, _f32p, _f32p, C.c_int64, C.c_int, C.c_int, C.c_int, _f32p, _f32p, _f32p, _f32p,
                                   _f32p, C.c_void_p]),
    "dmnerf_sample_pdf": (C.c_int, [_f32p, _f32p, C.c_int64, C.c_int, C.c_int, _f32p, _f32p, C.c_void_p]),
    "dmnerf_sort_concat": (C.c_int, [_f32p, _f32p, C.c_int64, C.c_int, C.c_int, _f32p, C.c_void_p]),
    "dmnerf_get_rays": (C.c_int, [C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_int, C.c_int, _f32p, _f32p, C.c_void_p]),
    "dmnerf_get_rays_at": (C.c_int, [C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_int, C.c_int, C.c_void_p, C.c_int64, _f32p,
                                     _f32p, C.c_void_p]),
    "dmnerf_get_rays_at_dev": (C.c_int, [C.POINTER(C.c_float), C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_int64, _f32p,
                                         _f32p, C.c_void_p]),
    "dmnerf_select_pixels": (C.c_int, [C.c_uint64, C.c_int, C.c_int, C.c_int64, C.c_void_p, C.c_void_p]),
    "dmnerf_hungarian_costs": (C.c_int, [_f32p, C.c_void_p, C.c_int64, C.c_int, _f32p, _f32p, _f32p, _f32p, _f32p, C.c_void_p]),
    "dmnerf_ins_loss_backward": (C.c_int, [_f32p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_int, _f32p, _f32p, _f32p, _f32p,
                                           _f32p, C.c_void_p]),
    "dmnerf_ins_label_rows": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "dmnerf_hungarian_assign": (C.c_int, [_f32p, _f32p, _f32p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, _f32p, C.c_void_p]),
    "dmnerf_ins_loss_backward_dev": (C.c_int, [_f32p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, _f32p, _f32p, _f32p,
                                               _f32p, _f32p, C.c_void_p]),
    "dmnerf_ins_status_take": (C.c_int, []),
    "dmnerf_stratify": (C.c_int, [_f32p, C.c_int64, _f32p, C.c_int64, C.c_int, _f32p, C.c_void_p]),
    "dmnerf_hier_sample": (C.c_int, [_f32p, _f32p, _f32p, C.c_int64, C.c_int, C.c_int, _f32p, C.c_void_p]),
    "dmnerf_act_floats_per_sample": (C.c_int, []),
    "dmnerf_mlp_backward_scratch_floats": (C.c_int64, [C.c_int64]),
    "dmnerf_mlp_forward_train": (C.c_int, [C.c_void_p, C.c_int, _f32p, _f32p, _f32p, _f32p, C.c_int64, C.c_int, _f32p, _f32p,
                                           C.c_int, C.c_void_p]),
    "dmnerf_mlp_backward": (C.c_int, [C.c_void_p, C.c_int, _f32p, _f32p, C.c_int64, C.POINTER(C.c_void_p), _f32p, C.c_int,
                                      C.c_void_p]),
    "dmnerf_composite_backward": (C.c_int, [_f32p, _f32p, _f32p, C.c_int64, C.c_int, C.c_int, C.c_int, _f32p, _f32p, _f32p, _f32p,
                                            _f32p, _f32p, C.c_int, C.c_void_p]),
    "dmnerf_render_forward": (C.c_int, [C.c_void_p, C.POINTER(RenderIO), C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int,
                                        C.c_void_p]),
    "dmnerf_sync_check": (C.c_int, [C.c_void_p, C.c_void_p]),
    "dmnerf_render_frame_host": (C.c_int, [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_int, C.c_int, C.c_float,
                                          C.c_float, C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(RenderIO),
                                          C.c_void_p]),
    "dmnerf_mlp_forward_points": (C.c_int, [C.c_void_p, C.c_int, _f32p, _f32p, C.c_int64, _f32p, C.c_int, C.c_void_p]),
    "dmnerf_exchanger": (C.c_int, [_f32p, C.POINTER(C.c_void_p), _f32p, C.POINTER(C.c_void_p), C.POINTER(C.c_int), C.c_int, C.c_int64,
                                  C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "dmnerf_penalizer_state_bytes": (C.c_int64, []),
    "dmnerf_penalizer_forward": (C.c_int, [_f32p, _f32p, _f32p, _f32p, C.c_int64, C.c_int, C.c_int, C.c_float, C.c_float, C.c_void_p,
                                          _f32p, C.c_void_p]),
    "dmnerf_penalizer_backward": (C.c_int, [_f32p, _f32p, _f32p, _f32p, C.c_int64, C.c_int, C.c_int, C.c_float, C.c_float,
                                           C.c_void_p, _f32p, _f32p, C.c_int, C.c_void_p]),
    "dmnerf_profile_enable": (C.c_int, [C.c_void_p, C.c_int]),
    "dmnerf_profile_read": (C.c_int, [C.c_void_p, C.POINTER(C.c_float), C.c_int]),
    "dmnerf_render_forward_host": (C.c_int, [C.c_void_p, C.POINTER(RenderIO), C.c_int64, C.c_int, C.c_int, C.c_int,
                                             C.c_int, C.c_void_p]),
    "dmnerf_mesh_grid_points": (C.c_int, [C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_int, C.c_int64, C.c_int64, _f32p,
                                          C.c_void_p]),
    "dmnerf_mesh_occupancy": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_int, C.c_float,
                                        C.c_int64, _f32p, C.c_void_p]),
    "dmnerf_mesh_mc_count": (C.c_int, [C.c_void_p, _f32p, C.c_int, C.c_int, C.c_int, C.c_float, C.POINTER(C.c_int64), C.c_void_p]),
    "dmnerf_mesh_mc_emit": (C.c_int, [C.c_void_p, _f32p, C.c_int, C.c_int, C.c_int, C.c_float, _f32p, C.c_void_p, C.c_void_p]),
    "dmnerf_mesh_to_scene": (C.c_int, [_f32p, C.c_int64, C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_int, _f32p, C.c_void_p]),
    "dmnerf_mesh_normals": (C.c_int, [C.c_void_p, _f32p, C.c_int64, C.c_void_p, C.c_int64, _f32p, C.c_void_p]),
    "dmnerf_mesh_clusters": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "dmnerf_mesh_clean": (C.c_int, [C.c_void_p, _f32p, _f32p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int, _f32p, _f32p,
                                    C.c_void_p, C.POINTER(C.c_int64), C.c_void_p]),
    "dmnerf_mesh_label_rays": (C.c_int, [_f32p, _f32p, C.c_int64, C.c_float, _f32p, _f32p, C.c_void_p]),
    "dmnerf_argmax_rows": (C.c_int, [_f32p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p]),
}

_lib = None
_lock = threading.Lock()


def load():
    """dlopen the in-tree shared library (built by dmnerf_b200.build / __graft_entry__.build)."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                "libdmnerf_b200.so not found at %s -- run `python -m dmnerf_b200.build` (there is no CPU fallback)"
                % LIB_PATH)
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in PROTOTYPES.items():
            fn = getattr(lib, name)      # AttributeError if the .so does not export a declared symbol
            fn.restype, fn.argtypes = res, args
        got = lib.dmnerf_abi_version()
        if got != ABI_VERSION:
            raise RuntimeError("libdmnerf_b200.so ABI version %d != binding version %d" % (got, ABI_VERSION))
        _lib = lib
    return _lib


def check(rc, what):
    if rc != 0:
        msg = load().dmnerf_last_error()
        raise RuntimeError("%s failed (status %d): %s" % (what, rc, (msg or b"").decode("utf-8", "replace")))


def ptr(t):
    """Device (or host) pointer of a contiguous float32 tensor, or None."""
    if t is None:
        return None
    import torch
    if not t.is_contiguous() or t.dtype != torch.float32:
        raise RuntimeError("native call needs a contiguous float32 tensor (got %s, contiguous=%s): convert it into a local "
                           "first so the copy outlives the launch" % (t.dtype, t.is_contiguous()))
    return C.c_void_p(t.data_ptr())


def launch_count():
    return int(load().dmnerf_launch_count())
