"""ctypes binding of libdmnerf_b200.so (C ABI: include/dmnerf_b200.h).

No torch types cross the boundary: tensors are passed as raw pointers (`ptr` / `ptrs`, which check dtype and
contiguity: ctypes itself checks nothing) plus sizes and the current CUDA stream handle; host-side matrices and masks
are built by `floats` / `doubles` / `camera` / `keep_mask`.  There is NO CPU fallback: if the shared library is
missing or a call fails, a RuntimeError is raised with the library's own message.
"""
import ctypes as C
import os
import threading

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# DMNERF_LIB_PATH: diagnostics builds of the same ABI; the default is the in-tree product library
LIB_PATH = os.environ.get("DMNERF_LIB_PATH") or os.path.join(_HERE, "lib", "libdmnerf_b200.so")

ABI_VERSION = 4
N_PARAMS = 30
IMPL_AUTO, IMPL_SIMT, IMPL_UMMA, IMPL_UMMA_F16 = 0, 1, 2, 3
FLAG_PERTURB, FLAG_WANT_RAW, FLAG_KEEP_INS = 1, 2, 4
LABEL_WORDS = 2049           # DMNERF_LABEL_WORDS

_f32p = C.c_void_p


class RegionDesc(C.Structure):
    """Mirror of `struct dmnerf_region` (objects.Region.abi builds one)."""
    _fields_ = [("bits", C.c_void_p), ("dim", C.c_int32), ("outside_keep", C.c_int32), ("voxel_map", C.c_float * 12),
                ("applies", C.c_uint32 * 4)]


class Edit(C.Structure):
    """Mirror of `struct dmnerf_edit` (render.scene_edit builds one)."""
    _fields_ = [("keep", C.POINTER(C.c_uint32)), ("region", C.POINTER(RegionDesc)), ("appearance", C.POINTER(C.c_float)),
                ("appearance_labels", C.c_int32)]


class RenderIO(C.Structure):
    """Mirror of `struct dmnerf_render_io`."""
    _fields_ = [
        ("rays_o", _f32p), ("rays_d", _f32p), ("z_coarse", _f32p), ("z_row_stride", C.c_int64),
        ("t_rand", _f32p), ("u", _f32p),
        ("rgb_coarse", _f32p), ("rgb_fine", _f32p), ("depth_coarse", _f32p), ("depth_fine", _f32p),
        ("acc_coarse", _f32p), ("acc_fine", _f32p), ("ins_coarse", _f32p), ("ins_fine", _f32p),
        ("z_vals_coarse", _f32p), ("z_vals_fine", _f32p), ("weights_coarse", _f32p), ("weights_fine", _f32p),
        ("raw_coarse", _f32p), ("raw_fine", _f32p), ("edit", C.POINTER(Edit)),
    ]


MAX_MOVES = 8                # DMNERF_MAX_MOVES
MAX_CANDIDATES = 4096        # DMNERF_MAX_CANDIDATES
MAX_BASES = 64               # DMNERF_MAX_BASES


class Pieces(C.Structure):
    """Mirror of `struct dmnerf_pieces`."""
    _fields_ = [
        ("region", RegionDesc * MAX_MOVES), ("rest_drop", C.c_int32 * MAX_MOVES),
        ("ori_vote", C.c_void_p * MAX_MOVES), ("tar_vote", C.c_void_p * MAX_MOVES),
        ("ori_rays_o", _f32p), ("ori_rays_d", _f32p), ("ori_z", _f32p),
        ("tar_rays_o", _f32p * MAX_MOVES), ("tar_rays_d", _f32p * MAX_MOVES), ("tar_z", _f32p * MAX_MOVES),
    ]


class EditMove(C.Structure):
    """Mirror of `struct dmnerf_edit_move` (objects.edited_sweep builds them)."""
    _fields_ = [("label", C.c_int32), ("rest_drop", C.c_int32), ("trans", C.c_double * 12), ("box", C.c_int32 * 6),
                ("piece", RegionDesc)]


class RenderMoves(C.Structure):
    """Mirror of `struct dmnerf_render_moves` (objects.render_moves builds one)."""
    _fields_ = [("moves", C.POINTER(EditMove)), ("n_moves", C.c_int32), ("dim", C.c_int32), ("transform", C.c_double * 16),
                ("extents", C.c_double * 3), ("level", C.c_float), ("voxel", C.c_float)]


class Deformation(C.Structure):
    """Mirror of `struct dmnerf_deformation` (objects.Deformation.abi builds one)."""
    _fields_ = [("n_knots", C.c_int32), ("frame", C.c_double * 12), ("h0", C.c_double), ("dh", C.c_double),
                ("knots", C.POINTER(C.c_double))]


class Placement(C.Structure):
    """Mirror of `struct dmnerf_placement` (objects.placement_map builds one)."""
    _fields_ = [("piece", RegionDesc), ("obstacles", C.c_uint32 * 4), ("label", C.c_int32), ("rest_drop", C.c_int32),
                ("axis", C.c_int32), ("sign", C.c_int32), ("lift", C.c_int32)]


class PlacementInfo(C.Structure):
    """Mirror of `struct dmnerf_placement_info`."""
    _fields_ = [("offset_lo", C.c_int32 * 2), ("offsets", C.c_int32 * 2), ("height", C.c_int32 * 2), ("runs", C.c_int64),
                ("points", C.c_int64), ("sum", C.c_int64 * 3)]


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
    "dmnerf_composite": (C.c_int, [_f32p, _f32p, _f32p, C.c_int64, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_uint32), _f32p, _f32p,
                                   _f32p, _f32p, _f32p, C.c_void_p]),
    "dmnerf_sample_pdf": (C.c_int, [_f32p, _f32p, C.c_int64, C.c_int, C.c_int, _f32p, _f32p, C.c_void_p]),
    "dmnerf_sort_concat": (C.c_int, [_f32p, _f32p, C.c_int64, C.c_int, C.c_int, _f32p, C.c_void_p]),
    "dmnerf_get_rays": (C.c_int, [C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_int, C.c_int, _f32p, _f32p, C.c_void_p]),
    "dmnerf_get_rays_at": (C.c_int, [C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_int, C.c_int, C.c_void_p, C.c_int64, _f32p,
                                     _f32p, C.c_void_p]),
    "dmnerf_get_rays_at_dev": (C.c_int, [C.POINTER(C.c_float), C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_int64, _f32p,
                                         _f32p, C.c_void_p]),
    "dmnerf_select_pixels": (C.c_int, [C.c_uint64, C.c_int, C.c_int, C.c_int64, C.c_void_p, C.c_void_p]),
    "dmnerf_hungarian_costs": (C.c_int, [_f32p, C.c_void_p, C.c_int64, C.c_int, _f32p, _f32p, _f32p, _f32p, _f32p, C.c_void_p]),
    "dmnerf_ins_loss_backward": (C.c_int, [_f32p, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, _f32p, _f32p,
                                           _f32p, _f32p, _f32p, C.c_void_p]),
    "dmnerf_ins_label_rows": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "dmnerf_hungarian_assign": (C.c_int, [_f32p, _f32p, _f32p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, _f32p, C.c_void_p]),
    "dmnerf_ins_status_take": (C.c_int, []),
    "dmnerf_ins_label_bitmap": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "dmnerf_ins_label_rows_merged": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p,
                                               C.c_void_p]),
    "dmnerf_hungarian_partials": (C.c_int, [_f32p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p]),
    "dmnerf_hungarian_costs_merged": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, _f32p, _f32p, _f32p, _f32p, _f32p,
                                                C.c_void_p]),
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
                                  C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(Pieces), C.c_void_p]),
    "dmnerf_piece_vote": (C.c_int, [_f32p, _f32p, _f32p, _f32p, _f32p, C.c_int64, C.c_int, C.c_int, C.POINTER(C.c_int),
                                    C.POINTER(RegionDesc), C.c_int, C.c_void_p, C.c_void_p]),
    "dmnerf_penalizer_state_bytes": (C.c_int64, []),
    "dmnerf_penalizer_forward": (C.c_int, [_f32p, _f32p, _f32p, _f32p, C.c_int64, C.c_int, C.c_int, C.c_float, C.c_float, C.c_void_p,
                                          _f32p, C.c_void_p]),
    "dmnerf_penalizer_backward": (C.c_int, [_f32p, _f32p, _f32p, _f32p, C.c_int64, C.c_int, C.c_int, C.c_float, C.c_float,
                                           C.c_void_p, _f32p, _f32p, C.c_int, C.c_void_p]),
    "dmnerf_penalizer_partials_bytes": (C.c_int64, [C.c_int64, C.c_int, C.c_int]),
    "dmnerf_penalizer_merge": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, _f32p, C.c_void_p]),
    "dmnerf_profile_enable": (C.c_int, [C.c_void_p, C.c_int]),
    "dmnerf_profile_read": (C.c_int, [C.c_void_p, C.POINTER(C.c_float), C.c_int]),
    "dmnerf_render_forward_host": (C.c_int, [C.c_void_p, C.POINTER(RenderIO), C.c_int64, C.c_int, C.c_int, C.c_int,
                                             C.c_int, C.c_void_p]),
    "dmnerf_mesh_grid_points": (C.c_int, [C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_int, C.c_int64, C.c_int64, _f32p,
                                          C.c_void_p]),
    "dmnerf_mesh_occupancy": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_int, C.c_float,
                                        C.c_int64, C.POINTER(C.c_uint32), _f32p, C.c_void_p, C.c_void_p]),
    "dmnerf_mesh_mc_count": (C.c_int, [C.c_void_p, _f32p, C.c_int, C.c_int, C.c_int, C.c_float, C.POINTER(C.c_int64), C.c_void_p]),
    "dmnerf_mesh_mc_emit": (C.c_int, [C.c_void_p, _f32p, C.c_int, C.c_int, C.c_int, C.c_float, _f32p, C.c_void_p, C.c_void_p]),
    "dmnerf_mesh_to_scene": (C.c_int, [_f32p, C.c_int64, C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_int, _f32p, C.c_void_p]),
    "dmnerf_mesh_normals": (C.c_int, [C.c_void_p, _f32p, C.c_int64, C.c_void_p, C.c_int64, _f32p, C.c_void_p]),
    "dmnerf_mesh_clusters": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "dmnerf_mesh_clean": (C.c_int, [C.c_void_p, _f32p, _f32p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int, _f32p, _f32p,
                                    C.c_void_p, C.POINTER(C.c_int64), C.c_void_p]),
    "dmnerf_mesh_label_rays": (C.c_int, [_f32p, _f32p, C.c_int64, C.c_float, _f32p, _f32p, C.c_void_p]),
    "dmnerf_argmax_rows": (C.c_int, [_f32p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p]),
    "dmnerf_mesh_occupancy_edit": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_int, C.c_float,
                                             C.c_float, C.c_int64, C.POINTER(EditMove), C.c_int, _f32p, C.c_void_p,
                                             C.POINTER(C.c_int64), C.c_void_p]),
    "dmnerf_render_moved": (C.c_int, [C.c_void_p, C.POINTER(RenderIO), C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int,
                                      C.POINTER(RenderMoves), C.POINTER(C.c_int64), C.c_void_p]),
    "dmnerf_mesh_vertex_labels": (C.c_int, [_f32p, C.c_int64, _f32p, C.c_void_p, C.c_int, C.c_float, C.c_void_p, C.c_void_p]),
    "dmnerf_object_voxels": (C.c_int, [C.c_void_p, _f32p, C.c_void_p, C.c_int, C.c_float, C.c_int, C.POINTER(C.c_int32),
                                       C.POINTER(C.c_int64), C.POINTER(C.c_uint32), C.c_void_p]),
    "dmnerf_object_spans": (C.c_int, [C.c_void_p, _f32p, C.c_void_p, C.c_int, C.c_float, C.c_int, C.POINTER(C.c_int32),
                                      C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_void_p]),
    "dmnerf_move_overlap": (C.c_int, [C.c_void_p, _f32p, C.c_void_p, C.c_int, C.c_float, C.POINTER(C.c_double), C.POINTER(C.c_double),
                                      C.POINTER(EditMove), C.c_int, C.POINTER(C.c_uint32), C.POINTER(C.c_int64),
                                      C.POINTER(C.c_int64), C.c_void_p]),
    "dmnerf_object_contacts": (C.c_int, [C.c_void_p, _f32p, C.c_void_p, C.c_int, C.c_float, C.c_int, C.POINTER(C.c_int64),
                                         C.c_void_p]),
    "dmnerf_placement_map": (C.c_int, [C.c_void_p, _f32p, C.c_void_p, C.c_int, C.c_float, C.POINTER(C.c_double),
                                       C.POINTER(C.c_double), C.POINTER(Placement), C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.POINTER(PlacementInfo), C.c_void_p]),
    "dmnerf_placement_contacts": (C.c_int, [C.c_void_p, _f32p, C.c_void_p, C.c_int, C.c_float, C.POINTER(C.c_double),
                                            C.POINTER(C.c_double), C.POINTER(Placement), C.c_int, C.c_int, C.POINTER(C.c_int32),
                                            C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_int32), C.c_void_p]),
    "dmnerf_placement_maps": (C.c_int, [C.c_void_p, _f32p, C.c_void_p, C.c_int, C.c_float, C.POINTER(C.c_double),
                                        C.POINTER(C.c_double), C.POINTER(Placement), C.POINTER(C.c_double), C.POINTER(C.c_int32),
                                        C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(PlacementInfo), C.POINTER(C.c_int32),
                                        C.c_void_p]),
    "dmnerf_placement_contacts_moved": (C.c_int, [C.c_void_p, _f32p, C.c_void_p, C.c_int, C.c_float, C.POINTER(C.c_double),
                                                  C.POINTER(C.c_double), C.POINTER(Placement), C.POINTER(C.c_double),
                                                  C.POINTER(C.c_int32), C.c_int, C.c_int, C.POINTER(C.c_int32), C.c_int64,
                                                  C.POINTER(C.c_int64), C.POINTER(C.c_int32), C.c_void_p]),
    "dmnerf_grid_edit": (C.c_int, [C.c_void_p, _f32p, C.c_void_p, C.c_int, C.c_float, C.POINTER(C.c_double), C.POINTER(C.c_double),
                                   C.POINTER(EditMove), C.c_int, _f32p, C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64),
                                   C.c_void_p]),
    "dmnerf_placement_maps_in_scene": (C.c_int, [C.c_void_p, _f32p, C.c_void_p, _f32p, C.c_void_p, C.c_int, C.c_float,
                                                 C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(Placement),
                                                 C.POINTER(C.c_double), C.POINTER(C.c_int32), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                                 C.POINTER(PlacementInfo), C.POINTER(C.c_int32), C.c_void_p]),
    "dmnerf_placement_contacts_in_scene": (C.c_int, [C.c_void_p, _f32p, C.c_void_p, _f32p, C.c_void_p, C.c_int, C.c_float,
                                                     C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(Placement),
                                                     C.POINTER(C.c_double), C.POINTER(C.c_int32), C.c_int, C.c_int, C.POINTER(C.c_int32),
                                                     C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_int32), C.c_void_p]),
    "dmnerf_mesh_occupancy_edit_copies": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_int,
                                                    C.c_float, C.c_float, C.c_int64, C.POINTER(EditMove), C.POINTER(C.c_int32), C.c_int,
                                                    _f32p, C.c_void_p, C.POINTER(C.c_int64), C.c_void_p]),
    "dmnerf_grid_edit_copies": (C.c_int, [C.c_void_p, _f32p, C.c_void_p, C.c_int, C.c_float, C.POINTER(C.c_double),
                                          C.POINTER(C.c_double), C.POINTER(EditMove), C.POINTER(C.c_int32), C.c_int, _f32p, C.c_void_p,
                                          C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.c_void_p]),
    "dmnerf_render_moved_copies": (C.c_int, [C.c_void_p, C.POINTER(RenderIO), C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int,
                                             C.POINTER(RenderMoves), C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.c_void_p]),
    "dmnerf_move_overlap_copies": (C.c_int, [C.c_void_p, _f32p, C.c_void_p, C.c_int, C.c_float, C.POINTER(C.c_double),
                                             C.POINTER(C.c_double), C.POINTER(EditMove), C.POINTER(C.c_int32), C.c_int,
                                             C.POINTER(C.c_uint32), C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.c_void_p]),
    "dmnerf_placement_maps_in_scene_copy": (C.c_int, [C.c_void_p, _f32p, C.c_void_p, _f32p, C.c_void_p, C.c_int, C.c_float,
                                                      C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(Placement), C.c_int,
                                                      C.POINTER(C.c_double), C.POINTER(C.c_int32), C.c_int, C.c_void_p, C.c_void_p,
                                                      C.c_void_p, C.POINTER(PlacementInfo), C.POINTER(C.c_int32), C.c_void_p]),
    "dmnerf_placement_contacts_in_scene_copy": (C.c_int, [C.c_void_p, _f32p, C.c_void_p, _f32p, C.c_void_p, C.c_int, C.c_float,
                                                          C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(Placement), C.c_int,
                                                          C.POINTER(C.c_double), C.POINTER(C.c_int32), C.c_int, C.c_int,
                                                          C.POINTER(C.c_int32), C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_int32),
                                                          C.c_void_p]),
    "dmnerf_mesh_occupancy_edit_groups": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_int,
                                                    C.c_float, C.c_float, C.c_int64, C.POINTER(EditMove), C.POINTER(C.c_int32),
                                                    C.POINTER(C.c_uint32), C.c_int, _f32p, C.c_void_p, C.POINTER(C.c_int64), C.c_void_p]),
    "dmnerf_grid_edit_groups": (C.c_int, [C.c_void_p, _f32p, C.c_void_p, C.c_int, C.c_float, C.POINTER(C.c_double),
                                          C.POINTER(C.c_double), C.POINTER(EditMove), C.POINTER(C.c_int32), C.POINTER(C.c_uint32),
                                          C.c_int, _f32p, C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.c_void_p]),
    "dmnerf_render_moved_groups": (C.c_int, [C.c_void_p, C.POINTER(RenderIO), C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int,
                                             C.POINTER(RenderMoves), C.POINTER(C.c_int32), C.POINTER(C.c_uint32), C.POINTER(C.c_int64),
                                             C.c_void_p]),
    "dmnerf_move_overlap_groups": (C.c_int, [C.c_void_p, _f32p, C.c_void_p, C.c_int, C.c_float, C.POINTER(C.c_double),
                                             C.POINTER(C.c_double), C.POINTER(EditMove), C.POINTER(C.c_int32), C.POINTER(C.c_uint32),
                                             C.c_int, C.POINTER(C.c_uint32), C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.c_void_p]),
    "dmnerf_placement_maps_in_scene_group": (C.c_int, [C.c_void_p, _f32p, C.c_void_p, _f32p, C.c_void_p, C.c_int, C.c_float,
                                                       C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(Placement), C.c_int,
                                                       C.POINTER(C.c_uint32), C.POINTER(C.c_double), C.POINTER(C.c_int32), C.c_int,
                                                       C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(PlacementInfo),
                                                       C.POINTER(C.c_int32), C.c_void_p]),
    "dmnerf_placement_contacts_in_scene_group": (C.c_int, [C.c_void_p, _f32p, C.c_void_p, _f32p, C.c_void_p, C.c_int, C.c_float,
                                                           C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(Placement), C.c_int,
                                                           C.POINTER(C.c_uint32), C.POINTER(C.c_double), C.POINTER(C.c_int32), C.c_int,
                                                           C.c_int, C.POINTER(C.c_int32), C.c_int64, C.POINTER(C.c_int64),
                                                           C.POINTER(C.c_int32), C.c_void_p]),
    "dmnerf_mesh_occupancy_edit_deformed": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_int,
                                                      C.c_float, C.c_float, C.c_int64, C.POINTER(EditMove), C.POINTER(C.c_int32),
                                                      C.POINTER(C.c_uint32), C.POINTER(Deformation), C.c_int, _f32p, C.c_void_p,
                                                      C.POINTER(C.c_int64), C.c_void_p]),
    "dmnerf_grid_edit_deformed": (C.c_int, [C.c_void_p, _f32p, C.c_void_p, C.c_int, C.c_float, C.POINTER(C.c_double),
                                            C.POINTER(C.c_double), C.POINTER(EditMove), C.POINTER(C.c_int32), C.POINTER(C.c_uint32),
                                            C.POINTER(Deformation), C.c_int, _f32p, C.c_void_p, C.POINTER(C.c_int64),
                                            C.POINTER(C.c_int64), C.c_void_p]),
    "dmnerf_render_moved_deformed": (C.c_int, [C.c_void_p, C.POINTER(RenderIO), C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int,
                                               C.POINTER(RenderMoves), C.POINTER(C.c_int32), C.POINTER(C.c_uint32),
                                               C.POINTER(Deformation), C.POINTER(C.c_int64), C.c_void_p]),
    "dmnerf_move_overlap_deformed": (C.c_int, [C.c_void_p, _f32p, C.c_void_p, C.c_int, C.c_float, C.POINTER(C.c_double),
                                               C.POINTER(C.c_double), C.POINTER(EditMove), C.POINTER(C.c_int32), C.POINTER(C.c_uint32),
                                               C.POINTER(Deformation), C.c_int, C.POINTER(C.c_uint32), C.POINTER(C.c_int64),
                                               C.POINTER(C.c_int64), C.c_void_p]),
    "dmnerf_object_components": (C.c_int, [C.c_void_p, _f32p, C.c_void_p, C.c_int, C.c_float, C.c_int, C.c_int, C.c_void_p,
                                           C.POINTER(C.c_int64), C.c_void_p]),
    "dmnerf_component_table": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p]),
    "dmnerf_component_groups": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "dmnerf_grid_cast": (C.c_int, [C.c_void_p, _f32p, C.c_void_p, C.c_int, C.c_float, C.POINTER(C.c_double), C.POINTER(C.c_double),
                                   C.POINTER(C.c_uint32), _f32p, _f32p, C.c_int64, C.c_float, C.c_float, _f32p, C.c_void_p, C.c_void_p,
                                   _f32p, C.c_void_p]),
    "dmnerf_grid_edit_source": (C.c_int, [C.c_void_p, _f32p, C.c_void_p, _f32p, C.c_void_p, C.POINTER(RenderMoves), C.POINTER(C.c_int32),
                                          C.POINTER(C.c_uint32), C.POINTER(Deformation), _f32p, _f32p, _f32p, C.c_void_p, C.c_int64,
                                          C.c_void_p, _f32p, _f32p, C.POINTER(C.c_int64), C.c_void_p]),
    "dmnerf_region_pack": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "dmnerf_region_dilate": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "dmnerf_region_contains": (C.c_int, [C.POINTER(RegionDesc), _f32p, C.c_int64, C.c_void_p, C.c_void_p]),
    "dmnerf_eval_workspace_bytes": (C.c_int64, [C.c_int64, C.c_int, C.c_int, C.c_int]),
    "dmnerf_eval_image": (C.c_int, [_f32p, _f32p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "dmnerf_ins_eval": (C.c_int, [_f32p, C.c_int64, C.c_int, C.c_void_p, C.c_int, _f32p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_void_p]),
    "dmnerf_calculate_ap": (C.c_int, [_f32p, _f32p, C.c_int, C.c_int, _f32p, C.c_void_p]),
    "dmnerf_ins_dense_rows": (C.c_int, [_f32p, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "dmnerf_label_colors": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
}


class EvalResult(C.Structure):
    """Mirror of `struct dmnerf_eval_result`."""
    _fields_ = [("ap", C.c_float * 6), ("gt_num", C.c_int32), ("pred_num", C.c_int32), ("status", C.c_int32),
                ("reserved", C.c_int32), ("psnr", C.c_double), ("ssim", C.c_double), ("return_labels", C.c_int32 * 128)]

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


def _addr(t, dtype, strided=False):
    if t.dtype != dtype or not (strided or t.is_contiguous()):
        raise RuntimeError("native call needs a contiguous %s tensor (got %s, contiguous=%s): convert it into a local "
                           "first so the copy outlives the launch" % (str(dtype).replace("torch.", ""), t.dtype,
                                                                      t.is_contiguous()))
    return t.data_ptr()


def ptr(t, dtype=torch.float32, strided=False):
    """Device (or host) pointer of a contiguous `dtype` tensor, or None.  strided=True is for an argument whose row stride
    is passed to the entry point beside it: only the dtype is checked."""
    return None if t is None else C.c_void_p(_addr(t, dtype, strided))


def ptrs(tensors, dtype=torch.float32):
    """Host array of the pointers of `tensors` (each checked like `ptr`), for the entry points that take `T* const*`."""
    return (C.c_void_p * len(tensors))(*[_addr(t, dtype) for t in tensors])


def _host_array(ctype, dtype, a, n):
    a = np.asarray(a.detach().cpu().double().numpy() if torch.is_tensor(a) else a, dtype=dtype).reshape(-1)
    if a.size != n:
        raise ValueError("expected %d values, got %d" % (n, a.size))
    return (ctype * n)(*a.tolist())


def floats(a, n):
    """Host float array of the n values of `a` (array, nested list or tensor, read row-major); ValueError for another count."""
    return _host_array(C.c_float, np.float32, a, n)


def doubles(a, n):
    """`floats` in float64."""
    return _host_array(C.c_double, np.float64, a, n)


def camera(K, c2w):
    """Host arrays of a camera entry point: the intrinsics K (3x3: 9 values) and the top 3x4 of the pose c2w (12 values)."""
    pose = c2w.detach()[:3, :4] if torch.is_tensor(c2w) else np.asarray(c2w)[:3, :4]
    return floats(K, 9), floats(pose, 12)


def keep_mask(words):
    """The 4-word object-selection mask (objects.object_mask) as the ABI's host uint32[4]."""
    return (C.c_uint32 * 4)(*words)


# DMNERF_INFER_IMPL=f16: IMPL_AUTO of an INFERENCE call means the fp16 preview network (IMPL_UMMA_F16), so that unmodified
# scripts render previews.  Read here only; the training forward (backward._train_impl) never consults it.
INFER_IMPL = IMPL_UMMA_F16 if os.environ.get("DMNERF_INFER_IMPL", "").strip().lower() == "f16" else IMPL_AUTO


def infer_impl(impl):
    """The network an inference entry point runs for `impl`: IMPL_AUTO follows DMNERF_INFER_IMPL, anything else is kept."""
    return INFER_IMPL if impl == IMPL_AUTO else impl


def need_cuda(what, *ts):
    """RuntimeError unless every tensor of `ts` that is not None is a CUDA tensor."""
    for t in ts:
        if t is not None and not (torch.is_tensor(t) and t.is_cuda):
            raise RuntimeError("%s: expected CUDA tensors (no CPU fallback)" % what)


def launch_count():
    return int(load().dmnerf_launch_count())
