"""ctypes binding of libalignn_b200.so (C ABI declared in include/alignn_b200.h).

The shared library is the only coupling between the PyTorch host code and the CUDA
kernels: it is dlopen'ed here, no torch types cross the boundary (device pointers,
sizes, flags and the raw cudaStream_t only).  There is NO fallback: if the library
is missing or a call fails, a RuntimeError is raised.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libalignn_b200.so")

NORM_LAYER, NORM_AFFINE, NORM_STATS = 0, 1, 2
SUPPORTED_D = (32, 64, 128, 256)

_fp = C.c_void_p  # device pointers travel as void*


class EgcFwdArgs(C.Structure):
    _fields_ = [
        ("struct_size", C.c_size_t),
        ("Nn", C.c_int64), ("Ne", C.c_int64),
        ("d", C.c_int32), ("norm_nodes", C.c_int32), ("norm_edges", C.c_int32), ("residual", C.c_int32),
        ("gate_is_m", C.c_int32),
        ("gate_eps", C.c_float), ("ln_eps", C.c_float),
        ("x", _fp), ("y", _fp), ("G", _fp), ("P", _fp),
        ("src", _fp), ("in_ptr", _fp), ("in_eid", _fp),
        ("n_w", _fp), ("n_b", _fp), ("e_w", _fp), ("e_b", _fp),
        ("x_out", _fp), ("y_out", _fp), ("M", _fp), ("XP", _fp), ("S", _fp), ("H", _fp),
        ("partials", _fp),
        ("stream", _fp),
    ]


class EgcBwdArgs(C.Structure):
    _fields_ = [
        ("struct_size", C.c_size_t),
        ("Nn", C.c_int64), ("Ne", C.c_int64),
        ("d", C.c_int32), ("norm_nodes", C.c_int32), ("norm_edges", C.c_int32),
        ("gate_eps", C.c_float), ("ln_eps", C.c_float),
        ("P", _fp), ("M", _fp), ("XP", _fp), ("S", _fp), ("H", _fp),
        ("src", _fp), ("dst", _fp), ("in_ptr", _fp), ("in_eid", _fp), ("out_ptr", _fp), ("out_eid", _fp),
        ("n_w", _fp), ("n_b", _fp), ("n_mean", _fp), ("n_rstd", _fp),
        ("e_w", _fp), ("e_b", _fp), ("e_mean", _fp), ("e_rstd", _fp),
        ("n_c1", _fp), ("n_c2", _fp), ("e_c1", _fp), ("e_c2", _fp),
        ("gx_out", _fp), ("gy_out", _fp),
        ("GM", _fp), ("GP", _fp), ("GSh", _fp),
        ("partials", _fp), ("partials_src", _fp),
        ("parent_in_ptr", _fp), ("parent_in_eid", _fp), ("parent_out_ptr", _fp), ("parent_out_eid", _fp),
        ("parent_Nn", C.c_int64),
        ("stream", _fp),
    ]


class EgcBwdVjpArgs(C.Structure):
    _fields_ = [
        ("struct_size", C.c_size_t),
        ("Nn", C.c_int64), ("Ne", C.c_int64),
        ("d", C.c_int32), ("norm", C.c_int32),
        ("gate_eps", C.c_float), ("ln_eps", C.c_float),
        ("P", _fp), ("M", _fp), ("XP", _fp), ("S", _fp), ("H", _fp),
        ("src", _fp), ("dst", _fp), ("in_ptr", _fp), ("in_eid", _fp), ("out_ptr", _fp), ("out_eid", _fp),
        ("n_w", _fp), ("n_b", _fp), ("e_w", _fp), ("e_b", _fp),
        ("gx_out", _fp), ("gy_out", _fp), ("GSh", _fp),
        ("GPbar", _fp), ("GMbar", _fp), ("gx_bar_res", _fp), ("gy_bar_res", _fp),
        ("Pbar", _fp), ("Mbar", _fp), ("gx_out_bar", _fp), ("gy_out_bar", _fp), ("Gamma", _fp), ("Shbar", _fp),
        ("partials", _fp), ("partials_src", _fp),
        ("stream", _fp),
    ]


class GemmGatherArgs(C.Structure):
    _fields_ = [
        ("struct_size", C.c_size_t),
        ("M", C.c_int64), ("N", C.c_int32), ("K", C.c_int32),
        ("A", _fp), ("lda", C.c_int64),
        ("w_image", _fp), ("bias", _fp),
        ("add0", _fp), ("ld0", C.c_int64), ("idx0", _fp),
        ("add1", _fp), ("ld1", C.c_int64), ("idx1", _fp),
        ("C", _fp), ("ldc", C.c_int64),
        ("stats", _fp),
        ("stream", _fp),
        ("bn_R", _fp), ("ld_bn_R", C.c_int64),
        ("bn_scale", _fp), ("bn_shift", _fp), ("bn_mean", _fp), ("bn_rstd", _fp),
    ]


class WgradProblem(C.Structure):
    _fields_ = [("A", _fp), ("lda", C.c_int64), ("B", _fp), ("ldb", C.c_int64), ("K", C.c_int64), ("out", _fp), ("ld_out", C.c_int64)]


class ColsumProblem(C.Structure):
    _fields_ = [("a", _fp), ("rows", C.c_int64), ("stride", C.c_int64), ("cols", C.c_int), ("alpha", C.c_float), ("out", _fp)]


class ImageEntry(C.Structure):
    _fields_ = [("W", _fp), ("ldw", C.c_int64), ("rows", C.c_int32), ("cols", C.c_int32), ("transpose", C.c_int32),
                ("n_off", C.c_int32), ("k_off", C.c_int32), ("N", C.c_int32), ("K", C.c_int32), ("image", _fp)]


class BiasEntry(C.Structure):
    _fields_ = [("a", _fp), ("b", _fp), ("dst", _fp), ("n", C.c_int32)]


class CrystalBatch(C.Structure):
    _fields_ = [("cart_coords", _fp), ("shifts", _fp), ("cells", _fp), ("lattices", _fp), ("atom_offsets", _fp),
                ("shift_offsets", _fp), ("crystal_of_atom", _fp), ("cutoffs", _fp),
                ("num_crystals", C.c_int64), ("num_atoms", C.c_int64), ("num_images", C.c_int64), ("max_images", C.c_int64),
                ("atol", C.c_double)]


class FireParams(C.Structure):
    _fields_ = [("maxstep", C.c_double), ("dtmax", C.c_double), ("finc", C.c_double), ("fdec", C.c_double),
                ("astart", C.c_double), ("fa", C.c_double), ("fmax", C.c_double), ("n_min", C.c_int32),
                ("max_steps", C.c_int32), ("force_multiplier", C.c_float)]


class FireCellParams(C.Structure):
    _fields_ = [("fire", FireParams), ("stress_wt", C.c_float)]


class LbfgsParams(C.Structure):
    _fields_ = [("maxstep", C.c_double), ("alpha", C.c_double), ("damping", C.c_double), ("fmax", C.c_double),
                ("memory", C.c_int32), ("slots", C.c_int32), ("max_steps", C.c_int32), ("cell", C.c_int32),
                ("force_multiplier", C.c_float), ("stress_wt", C.c_float)]


class BfgsParams(C.Structure):
    _fields_ = [("maxstep", C.c_double), ("alpha", C.c_double), ("fmax", C.c_double), ("max_steps", C.c_int32),
                ("cell", C.c_int32), ("force_multiplier", C.c_float), ("stress_wt", C.c_float)]


class MdParams(C.Structure):
    _fields_ = [("dt", C.c_double), ("taut", C.c_double), ("kB", C.c_double), ("evaluation", C.c_int32),
                ("steps", C.c_int32), ("ensemble", C.c_int32), ("force_multiplier", C.c_float)]


class MdNptParams(C.Structure):
    _fields_ = [("dt", C.c_double), ("taut", C.c_double), ("taup", C.c_double), ("kB", C.c_double),
                ("evaluation", C.c_int32), ("steps", C.c_int32), ("phase", C.c_int32), ("force_multiplier", C.c_float),
                ("stress_wt", C.c_float)]


class MdNoseHooverParams(C.Structure):
    _fields_ = [("dt", C.c_double), ("kB", C.c_double), ("evaluation", C.c_int32), ("steps", C.c_int32),
                ("force_multiplier", C.c_float), ("stress_wt", C.c_float)]


class MdThermostatParams(C.Structure):
    _fields_ = [("dt", C.c_double), ("kB", C.c_double), ("friction", C.c_double), ("andersen_prob", C.c_double),
                ("sqrt_dt", C.c_double), ("dt_1_5", C.c_double), ("two_sqrt3", C.c_double), ("evaluation", C.c_int32),
                ("steps", C.c_int32), ("ensemble", C.c_int32), ("force_multiplier", C.c_float)]


# name -> (restype, argtypes); mirrors include/alignn_b200.h one to one
_SIGNATURES = {
    "alignn_b200_version": (C.c_int, []),
    "alignn_b200_strerror": (C.c_char_p, [C.c_int]),
    "alignn_b200_last_cuda_error": (C.c_int, []),
    "alignn_b200_launch_count": (C.c_uint64, []),
    "alignn_b200_egc_partial_rows": (C.c_int, [C.c_int64, C.c_int]),
    "alignn_b200_egc_forward": (C.c_int, [C.POINTER(EgcFwdArgs)]),
    "alignn_b200_bn_finalize": (C.c_int, [_fp, C.c_int, C.c_int, C.c_int, C.c_int64, C.c_int, _fp, _fp, C.c_float,
                                          C.c_float, _fp, _fp, _fp, _fp, _fp, _fp, _fp]),
    "alignn_b200_affine_silu_residual": (C.c_int, [_fp, _fp, _fp, _fp, _fp, C.c_int64, C.c_int, _fp]),
    "alignn_b200_egc_backward": (C.c_int, [C.POINTER(EgcBwdArgs)]),
    "alignn_b200_egc_backward_vjp": (C.c_int, [C.POINTER(EgcBwdVjpArgs)]),
    "alignn_b200_bn_backward_reduce": (C.c_int, [_fp, _fp, _fp, _fp, _fp, _fp, C.c_int64, C.c_int, _fp, C.c_int, _fp]),
    "alignn_b200_rowstats_partials": (C.c_int, [_fp, C.c_int64, C.c_int, _fp, C.c_int, _fp]),
    "alignn_b200_bn_backward_apply": (C.c_int, [_fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp, C.c_int64, C.c_int, _fp, _fp]),
    "alignn_b200_ln_silu_forward": (C.c_int, [_fp, _fp, _fp, C.c_float, C.c_int64, C.c_int, _fp, _fp, _fp]),
    "alignn_b200_ln_silu_backward": (C.c_int, [_fp, _fp, _fp, _fp, _fp, C.c_int64, C.c_int, _fp, _fp, C.c_int, _fp]),
    "alignn_b200_adamw_flat": (C.c_int, [_fp, _fp, _fp, _fp, C.c_int64, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float,
                                         C.c_int, _fp, _fp, _fp]),
    "alignn_b200_colsum_partials": (C.c_int, [_fp, C.c_int64, C.c_int, _fp, C.c_int, _fp]),
    "alignn_b200_colsum": (C.c_int, [_fp, C.c_int64, C.c_int, C.c_int64, C.c_float, _fp, _fp]),
    "alignn_b200_colsum_batch": (C.c_int, [C.POINTER(ColsumProblem), C.c_int, _fp]),
    "alignn_b200_gather_segment_sum": (C.c_int, [_fp, _fp, _fp, _fp, _fp, C.c_int64, C.c_int64, C.c_int, _fp, _fp, _fp]),
    "alignn_b200_gemm_weight_image_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "alignn_b200_gemm_prepare_table": (C.c_int, [_fp, C.c_int, C.c_int64, _fp, C.c_int, _fp]),
    "alignn_b200_gemm_nt": (C.c_int, [_fp, C.c_int64, _fp, C.c_int64, C.c_int, C.c_int, _fp, _fp, C.c_int64, _fp,
                                      C.c_int64, _fp]),
    "alignn_b200_gemm_gather": (C.c_int, [C.POINTER(GemmGatherArgs)]),
    "alignn_b200_gemm_gather_stat_rows": (C.c_int, [C.c_int64, C.c_int]),
    "alignn_b200_wgrad_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int, C.c_int, C.c_int]),
    "alignn_b200_wgrad_batch_workspace_bytes": (C.c_size_t, [C.POINTER(WgradProblem), C.c_int, C.c_int]),
    "alignn_b200_wgrad_batch": (C.c_int, [C.POINTER(WgradProblem), C.c_int, C.c_int, _fp, C.c_size_t, _fp]),
    "alignn_b200_wgrad": (C.c_int, [_fp, C.c_int64, _fp, C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_int, _fp, C.c_int64,
                                    _fp, C.c_size_t, _fp]),
    "alignn_b200_csr_build_host": (C.c_int, [_fp, _fp, C.c_int64, C.c_int64, _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp]),
    "alignn_b200_line_graph_count_host": (C.c_int64, [_fp, _fp, _fp, C.c_int64]),
    "alignn_b200_line_graph_build_host": (C.c_int, [_fp, _fp, _fp, C.c_int64, _fp, C.c_int64, C.c_int64, _fp, _fp, _fp]),
    "alignn_b200_radius_graph_count_host": (C.c_int64, [_fp, _fp, C.c_int64, C.c_int64, C.c_double, C.c_double]),
    "alignn_b200_radius_graph_build_host": (C.c_int, [_fp, _fp, C.c_int64, C.c_int64, C.c_double, C.c_double, C.c_int64, _fp,
                                                      _fp, _fp, _fp]),
    "alignn_b200_csr_build_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int64]),
    "alignn_b200_csr_build": (C.c_int, [_fp, _fp, C.c_int64, C.c_int64, _fp, _fp, _fp, _fp, _fp, _fp, C.c_size_t, _fp]),
    "alignn_b200_line_graph_workspace_bytes": (C.c_size_t, [C.c_int64]),
    "alignn_b200_line_graph_offsets": (C.c_int, [_fp, _fp, _fp, C.c_int64, _fp, _fp, C.c_size_t, _fp]),
    "alignn_b200_line_graph_fill": (C.c_int, [_fp, _fp, _fp, _fp, C.c_int64, _fp, _fp, _fp, _fp]),
    "alignn_b200_radius_graph_workspace_bytes": (C.c_size_t, [C.c_int64]),
    "alignn_b200_radius_graph_offsets": (C.c_int, [_fp, _fp, C.c_int64, C.c_int64, C.c_double, C.c_double, _fp, _fp, C.c_size_t, _fp]),
    "alignn_b200_radius_graph_fill": (C.c_int, [_fp, _fp, C.c_int64, C.c_int64, C.c_double, C.c_double, _fp, _fp, _fp, _fp, _fp, _fp]),
    "alignn_b200_crystal_scan_workspace_bytes": (C.c_size_t, [C.c_int64]),
    "alignn_b200_crystal_scan_count": (C.c_int, [C.POINTER(CrystalBatch), C.c_int, _fp, _fp, _fp, C.c_size_t, _fp]),
    "alignn_b200_crystal_radius_fill": (C.c_int, [C.POINTER(CrystalBatch), _fp, _fp, _fp, _fp, _fp, _fp]),
    "alignn_b200_knn_graph_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int64, C.c_int64]),
    "alignn_b200_knn_graph_select": (C.c_int, [C.POINTER(CrystalBatch), _fp, C.c_int64, C.c_int, _fp, _fp, C.c_size_t, _fp]),
    "alignn_b200_knn_graph_order": (C.c_int, [C.POINTER(CrystalBatch), _fp, _fp, C.c_int64, C.c_int64, _fp, _fp, C.c_size_t,
                                              _fp]),
    "alignn_b200_knn_graph_emit": (C.c_int, [C.POINTER(CrystalBatch), _fp, C.c_int64, C.c_int64, _fp, _fp, _fp, _fp, _fp,
                                             C.c_size_t, _fp]),
    "alignn_b200_pair_force_scatter": (C.c_int, [_fp, _fp, _fp, _fp, _fp, C.c_int64, C.c_int, _fp, _fp]),
    "alignn_b200_virial_stress": (C.c_int, [_fp, _fp, _fp, _fp, _fp, C.c_int64, C.c_float, _fp, _fp]),
    "alignn_b200_bond_cutoff_workspace_bytes": (C.c_size_t, [C.c_int64]),
    "alignn_b200_bond_cutoff_offsets": (C.c_int, [_fp, _fp, _fp, _fp, C.c_int64, C.c_float, _fp, _fp, _fp, C.c_size_t, _fp]),
    "alignn_b200_bond_cutoff_fill": (C.c_int, [_fp, _fp, _fp, _fp, _fp, _fp, C.c_int64, C.c_int64, _fp, _fp, _fp, _fp, _fp,
                                               _fp]),
    "alignn_b200_remove_net_torque_workspace_bytes": (C.c_size_t, [C.c_int64]),
    "alignn_b200_remove_net_torque": (C.c_int, [_fp, _fp, _fp, C.c_int64, C.c_int64, C.c_int, _fp, _fp, C.c_size_t, _fp]),
    "alignn_b200_remove_net_torque_per_crystal_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int64]),
    "alignn_b200_remove_net_torque_per_crystal": (C.c_int, [_fp, _fp, _fp, C.c_int64, C.c_int64, _fp, _fp, C.c_size_t,
                                                            _fp]),
    "alignn_b200_fire_step": (C.c_int, [C.POINTER(FireParams), _fp, C.c_int64, _fp, _fp, C.c_int64, _fp, C.c_int64, _fp, _fp,
                                        _fp, _fp, _fp, _fp]),
    "alignn_b200_fire_cell_step": (C.c_int, [C.POINTER(FireCellParams), _fp, C.c_int64, _fp, _fp, C.c_int64, _fp, C.c_int64,
                                             _fp, C.c_int64, _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp]),
    "alignn_b200_lbfgs_step": (C.c_int, [C.POINTER(LbfgsParams), _fp, C.c_int64, _fp, _fp, C.c_int64, _fp, C.c_int64, _fp,
                                         C.c_int64] + [_fp] * 15 + [_fp]),
    "alignn_b200_bfgs_update": (C.c_int, [C.POINTER(BfgsParams), _fp, C.c_int64, _fp, _fp, C.c_int64, C.c_int64, _fp,
                                          C.c_int64, _fp, C.c_int64] + [_fp] * 16 + [_fp]),
    "alignn_b200_bfgs_apply": (C.c_int, [C.POINTER(BfgsParams), _fp, C.c_int64, C.c_int64, _fp, _fp, _fp, C.c_int64,
                                         C.c_int64] + [_fp] * 11 + [_fp]),
    "alignn_b200_md_step": (C.c_int, [C.POINTER(MdParams), _fp, C.c_int64, _fp, C.c_int64, _fp, _fp, _fp, _fp, _fp, _fp, _fp,
                                      _fp, _fp]),
    "alignn_b200_md_thermostat_step": (C.c_int, [C.POINTER(MdThermostatParams), _fp, C.c_int64, _fp, C.c_int64, _fp, _fp,
                                                 _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp]),
    "alignn_b200_md_npt_step": (C.c_int, [C.POINTER(MdNptParams), _fp, C.c_int64, _fp, C.c_int64, _fp, _fp, _fp, _fp, _fp,
                                          _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp]),
    "alignn_b200_md_nose_hoover_step": (C.c_int, [C.POINTER(MdNoseHooverParams), _fp, C.c_int64, _fp, C.c_int64]
                                        + [_fp] * 19),
    "alignn_b200_md_noise": (C.c_int, [C.c_uint64, C.c_int32, C.c_int32, C.c_uint32, C.c_int64, C.c_int32, _fp, _fp, _fp,
                                       _fp]),
    "alignn_b200_phonon_force_constants": (C.c_int, [_fp, C.c_double, C.c_float, _fp, C.c_int64, _fp, _fp, C.c_int64, _fp,
                                                     _fp, C.c_int64, _fp, _fp, _fp, _fp]),
    "alignn_b200_phonon_dynamical_matrix": (C.c_int, [_fp, C.c_int64, _fp, _fp, C.c_int64, C.c_int64, _fp, _fp, C.c_int64,
                                                      _fp, _fp, _fp]),
    "alignn_b200_eos_fit": (C.c_int, [C.c_int32, _fp, _fp, C.c_int64, C.c_int32, _fp, _fp, _fp]),
    "alignn_b200_debug_egc_flags": (None, [C.c_int]),
    "alignn_b200_segment_mean": (C.c_int, [_fp, _fp, C.c_int64, C.c_int, _fp, _fp]),
    "alignn_b200_segment_mean_backward": (C.c_int, [_fp, _fp, C.c_int64, C.c_int, _fp, _fp]),
}

EXPORTED_SYMBOLS = tuple(_SIGNATURES)

_lib: Optional[C.CDLL] = None


def load() -> C.CDLL:
    """dlopen the library (once) and type every entry point.  Raises if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} not found: the CUDA extension is not built. Run `python -c 'import __graft_entry__ as g; "
            "g.build()'` (nvcc, sm_90a). alignn_b200 has no CPU or eager fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export what the header declares
        fn.restype, fn.argtypes = res, args
    if lib.alignn_b200_version() != 101:
        raise RuntimeError("libalignn_b200.so version mismatch; rebuild")
    _lib = lib
    return lib


def check(status: int, what: str) -> None:
    if status != 0:
        lib = load()
        msg = lib.alignn_b200_strerror(status).decode()
        extra = ""
        if status == -4:
            extra = f" (cudaError {lib.alignn_b200_last_cuda_error()})"
        raise RuntimeError(f"{what} failed: {msg}{extra}")


def launch_count() -> int:
    return int(load().alignn_b200_launch_count())


def ptr(t: Optional[torch.Tensor]):
    """Device pointer of a contiguous fp32/int32 CUDA tensor (None -> NULL)."""
    if t is None:
        return None
    return t.data_ptr()


def stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


def require_cuda(*tensors: torch.Tensor) -> None:
    for t in tensors:
        if t is None:
            continue
        if not t.is_cuda:
            raise RuntimeError("alignn_b200 kernels need CUDA tensors (no CPU path exists); got a tensor on "
                               f"{t.device}. Move the model and graphs to the GPU with .to('cuda').")
        if t.dtype not in (torch.float32, torch.int32):
            raise RuntimeError(f"alignn_b200 kernels are fp32/int32 only; got {t.dtype}")
        if not t.is_contiguous():
            raise RuntimeError("alignn_b200 kernels need contiguous tensors")
