"""ctypes binding of ``libani_b200.so`` (the C-ABI declared in ``include/ani_b200.h``).

There is exactly one compute path: the CUDA library.  If it is missing or does not load the
import fails loudly -- there is no CPU or PyTorch fallback.
"""
from __future__ import annotations

import ctypes as C
import os
import typing as tp

HERE = os.path.dirname(os.path.abspath(__file__))
# ANI_B200_LIB selects another build of the same library (e.g. the 3 x bf16 operand variant)
LIB_PATH = os.environ.get("ANI_B200_LIB") or os.path.join(HERE, "libani_b200.so")

ANI_MAX_SPECIES = 8
ANI_MAX_SHFR = 32
ANI_MAX_SHFA = 8
ANI_MAX_SHFZ = 8
ANI_MAX_MEMBERS = 16
ANI_TILE_ROWS = 128
ANI_MAX_ANG = 96
ANI_VIRIAL_SLOTS = 64
ACT_CELU = 0                # ani_mlp_model::activation
ACT_GELU = 1
DIPOLE_FRAMES = ("center_of_mass", "center_of_geometry", "origin")   # the frame argument of ani_b200_charges
ANI_LATTICE_STRIDE = 18   # floats per conformer of the lattice table of grid mode 3: cell, inverse

STATUS_NBR_OVERFLOW = 1
STATUS_ANG_OVERFLOW = 2
STATUS_CELL_TOO_SMALL = 4
STATUS_PAIR_OVERFLOW = 8
STATUS_OPERAND_RANGE = 16
STATUS_INTERNAL = 32


class AEVParams(C.Structure):
    _fields_ = [
        ("rcr", C.c_float), ("rca", C.c_float),
        ("eta_r", C.c_float), ("eta_a", C.c_float), ("zeta", C.c_float),
        ("n_shf_r", C.c_int32), ("n_shf_a", C.c_int32), ("n_shf_z", C.c_int32),
        ("num_species", C.c_int32), ("cutoff_kind", C.c_int32),
        ("shf_r", C.c_float * ANI_MAX_SHFR), ("shf_a", C.c_float * ANI_MAX_SHFA),
        ("cos_z", C.c_float * ANI_MAX_SHFZ), ("sin_z", C.c_float * ANI_MAX_SHFZ),
        ("ang_pad", C.c_int32),
    ]


class Grid(C.Structure):
    _fields_ = [
        ("cell", C.c_float * 9), ("inv", C.c_float * 9), ("origin", C.c_float * 3),
        ("dims", C.c_int32 * 3), ("pbc", C.c_int32), ("nbins", C.c_int32), ("mode", C.c_int32),
        ("n_per_conf", C.c_int32), ("n_real", C.c_int32),
    ]


class MLPSpecies(C.Structure):
    _fields_ = [("h1", C.c_int32), ("h2", C.c_int32), ("h3", C.c_int32), ("pad_", C.c_int32),
                ("w_scale", C.c_float * 4)] + [
        (k, C.c_void_p) for k in ("b1", "b2", "b3", "w4", "b4", "t_f1", "t_f2", "t_f3", "t_b3", "t_b2", "t_b1")
    ]


class MLPModel(C.Structure):
    _fields_ = [
        ("num_species", C.c_int32), ("num_members", C.c_int32), ("in_dim", C.c_int32), ("ldx", C.c_int32),
        ("h1_max", C.c_int32), ("h2_max", C.c_int32), ("h3_max", C.c_int32), ("activation", C.c_int32),
        ("celu_alpha", C.c_float), ("member_scale", C.c_float * ANI_MAX_MEMBERS),
        ("sp", MLPSpecies * ANI_MAX_SPECIES),
        ("b1_compact", C.c_void_p),
    ]


class PairParams(C.Structure):
    _fields_ = [
        ("kind", C.c_int32), ("cutoff_fn", C.c_int32), ("num_species", C.c_int32), ("pad_", C.c_int32),
        ("cutoff", C.c_float), ("to_bohr", C.c_float),
        ("a", C.c_float * ANI_MAX_SPECIES * ANI_MAX_SPECIES), ("b", C.c_float * ANI_MAX_SPECIES * ANI_MAX_SPECIES),
        ("c", C.c_float * ANI_MAX_SPECIES * ANI_MAX_SPECIES),
        ("screen_coeff", C.c_float * 4), ("screen_exp", C.c_float * 4),
    ]


ANI_HESSIAN_ROW_ALIGN = 64


class HessianChunk(C.Structure):
    _fields_ = [
        ("atom", C.c_void_p), ("row_off", C.c_void_p), ("block_off", C.c_void_p), ("row_slot", C.c_void_p),
        ("tile_species", C.c_void_p), ("n_slots", C.c_int32), ("rows", C.c_int32), ("max_count", C.c_int32),
        ("pad_", C.c_int32),
    ]


class HessianWeights(C.Structure):
    _fields_ = [("w1", C.c_void_p * ANI_MAX_SPECIES), ("w2", C.c_void_p * ANI_MAX_SPECIES),
                ("w3", C.c_void_p * ANI_MAX_SPECIES)]


ANI_MD_BLOCK = 256
ANI_MD_PARAMS = 8
ANI_MD_THERMO = 4
ANI_MD_BARO_PARAMS = 3
ANI_MD_BARO = 2
MD_VERLET = 0
MD_LANGEVIN = 1


class MDState(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in ("x", "v", "inv_mass", "params", "counter", "stop_step", "trigger", "thermo",
                                          "frames", "partials")] + [
        ("seed", C.c_uint64), ("accel", C.c_double), ("kb", C.c_double)] + [
        (k, C.c_int32) for k in ("n_conf", "n_per_conf", "integrator", "thermo_rows", "record_every", "frame_slots",
                                 "frame_velocities", "pad_")]


class MDBarostat(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in ("master", "params", "cell_out", "virial", "record", "frame_cells")] + [
        ("cell_stride", C.c_int32), ("virial_slots", C.c_int32)]


ANI_OPT_PARAMS = 9
ANI_OPT_SCALARS = 3
ANI_OPT_RECORD = 3


class OptState(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in ("x", "v", "force_scale", "params", "scalars", "counter", "conv_step", "record",
                                          "partials")] + [
        (k, C.c_int32) for k in ("n_conf", "n_per_conf", "record_rows", "pad_")]


ANI_OPT_CELL_MASTER = 27
ANI_OPT_CELL_PARAMS = 3
ANI_OPT_CELL_RECORD = 3


class OptCell(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in ("master", "h0", "params", "cell_out", "virial", "cell_force", "record")] + [
        (k, C.c_int32) for k in ("cell_stride", "virial_slots", "projection", "pad_")]


ANI_LBFGS_PARAMS = 4
ANI_LBFGS_RECORD = 3
ANI_LBFGS_MAX_MEMORY = 128
ANI_LBFGS_TILE = 32


def lbfgs_partials(n_conf: int, n_per_conf: int, memory: int) -> int:
    """ANI_LBFGS_PARTIALS: the doubles of the scratch of ani_b200_lbfgs_step."""
    return n_conf * -(-n_per_conf // ANI_LBFGS_TILE) * (4 * (memory + 1) + 2)


class LbfgsState(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in ("x", "x_prev", "g_prev", "s", "y", "sy", "yy", "coef", "p", "iter",
                                          "force_scale", "params", "counter", "conv_step", "record", "partials")] + [
        (k, C.c_int32) for k in ("n_conf", "n_per_conf", "memory", "record_rows")]


ANI_NEB_RECORD = 4
ANI_NEB_DOTS = 5
ANI_NEB_ASENEB = 0
ANI_NEB_IMPROVED_TANGENT = 1


class NebState(C.Structure):
    _fields_ = [("fire", OptState)] + [(k, C.c_void_p) for k in ("endpoints", "end_energies", "springs", "climb",
                                                                  "neb_force", "dots")] + [
        (k, C.c_int32) for k in ("n_images", "n_atoms", "method", "pad_")]


class D3Params(C.Structure):
    _fields_ = [
        ("cutoff_fn", C.c_int32), ("num_species", C.c_int32), ("cutoff", C.c_float), ("to_bohr", C.c_float),
        ("s6", C.c_float), ("s8", C.c_float), ("a1", C.c_float), ("a2", C.c_float),
        ("k1", C.c_float), ("k2", C.c_float), ("k3", C.c_float), ("pad_", C.c_float),
        ("rcov", C.c_float * ANI_MAX_SPECIES),
        ("damp6", C.c_float * ANI_MAX_SPECIES * ANI_MAX_SPECIES),
        ("damp8", C.c_float * ANI_MAX_SPECIES * ANI_MAX_SPECIES),
        ("c8_scale", C.c_float * ANI_MAX_SPECIES * ANI_MAX_SPECIES),
    ]


_P = C.c_void_p
_I = C.c_int
_F = C.c_float
_D3_ARGS = [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _F, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _P]
_PAIR_ARGS = [_P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _I, _P, _P, _P, _P, _P, _P, _P, _I]
_PAIR_SEARCH_ARGS = [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _F, _P, _P, _P, _P, _P, _P, _P, _I, _P]

_PROTOTYPES = {
    "ani_b200_abi_version": (C.c_int, []),
    "ani_b200_operand_format": (C.c_int, [_P, _P, _P]),
    "ani_b200_error_string": (C.c_char_p, [_I]),
    "ani_b200_last_cuda_error": (C.c_char_p, []),
    "ani_b200_build_cells": (C.c_int, [_P, _P, _I, _I, _P, _I, _I, _F, _I, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "ani_b200_species_layout": (C.c_int, [_P, _P, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P, _P]),
    "ani_b200_aev_forward": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _P, _P, _I, _I, _P, _P, _I, _P, _P]),
    "ani_b200_aev_backward": (C.c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _P, _P, _I, _P, _P, _I, _P, _P, _I, _P, _P]),
    "ani_b200_pairs_to_rows": (C.c_int, [_P, _P, _P, C.c_int64, _I, _I, _P, _P, _P, _P, _P, _P]),
    "ani_b200_full_nbrlist_to_rows": (C.c_int, [_P, _I, _P, _P, _P, _I, _F, _I, _P, _P, _P, _P, _P, _P]),
    "ani_b200_aev_forward_rows": (C.c_int, [_P, _P, _P, _P, _P, _P, _I, _P, _P, _I, _I, _I, _P, _P]),
    "ani_b200_aev_backward_rows": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _I, _P, _P, _I, _I, _P, _P, _P]),
    "ani_b200_prepare_step": (C.c_int, [_P, _P, _I, _I, _P, _I, _I, C.c_float, _I, _P, _P, _P, _P, _P, _P, _P,
                                        _I, _I, _I, _I, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _I, _P, _I, _P, _P, _P, _P]),
    "ani_b200_prepare_step_cells": (C.c_int, [_P, _P, _I, _I, _P, _I, _I, C.c_float, _I, _P, _P, _P, _P, _P, _P, _P,
                                              _I, _I, _I, _I, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _I, _P, _I, _P,
                                              _P, _P, _P, _P]),
    "ani_b200_aev_forward_cells": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _P, _P, _I, _I, _P, _P, _I, _P,
                                             _P, _P]),
    "ani_b200_aev_backward_cells": (C.c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _P, _P, _I, _P, _P, _I, _P, _P, _I, _P,
                                              _P, _P]),
    "ani_b200_aev_backward_members": (C.c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _P, _P, _I, C.c_longlong, _P, _I, _P,
                                                _P, _I, _P, _P, _I, _P]),
    "ani_b200_aev_backward_members_cells": (C.c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _P, _P, _I, C.c_longlong, _P, _I,
                                                      _P, _P, _I, _P, _P, _I, _P, _P]),
    "ani_b200_ensemble_qbc": (C.c_int, [_P, _P, _I, _P, _P, _P, _I, _I, _P, _P, _P, _P, _P]),
    "ani_b200_pair_potential": (C.c_int, _PAIR_ARGS + [_P]),
    "ani_b200_pair_potential_cells": (C.c_int, _PAIR_ARGS + [_P, _P]),
    "ani_b200_pair_potential_search": (C.c_int, _PAIR_SEARCH_ARGS + [_P]),
    "ani_b200_pair_potential_search_cells": (C.c_int, _PAIR_SEARCH_ARGS + [_P, _P]),
    "ani_b200_pair_potential_pairs": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, C.c_int64, _I, _I, _P, _P, _P, _P]),
    "ani_b200_dispersion_d3": (C.c_int, _D3_ARGS + [_P]),
    "ani_b200_dispersion_d3_cells": (C.c_int, _D3_ARGS + [_P, _P]),
    "ani_b200_dispersion_d3_pairs": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, C.c_int64, _I, _I, _P, _P, _P, _P, _P,
                                               _P]),
    "ani_b200_verlet_positions":(C.c_int, [_I, _P, _P, _P, _I, _F, _P, _P, _P, _P, _P, _I, _P, _I, _P]),
    "ani_b200_debug_gemm_trace": (C.c_int, [_P, _I]),
    "ani_b200_debug_aev_trace": (C.c_int, [_P]),
    "ani_b200_half_neighbor_count": (C.c_int, [_P, _P, _P, _P, _P, _I, _F, _P, _P]),
    "ani_b200_half_neighbor_fill": (C.c_int, [_P, _P, _P, _P, _P, _I, _F, _P, C.c_int64, _P, _P, _P, _P, _P, _P]),
    "ani_b200_mlp_forward_backward": (C.c_int, [_P, _P, _P, _I, _P, _P, _P, _P, _P, _P, _P, _I, _P, _P]),
    "ani_b200_mlp_step_windows": (C.c_int, [_P, _I]),
    "ani_b200_mlp_step": (C.c_int, [_P, _P, _P, _I, _P, _P, _P, _P, _P, _P, _P, _I, _P, _P, _P]),
    "ani_b200_mlp_step_resident": (C.c_int, [_P, _P, _P, _I, _P, _P, _P, _P, _P, _P, _P, _P]),
    "ani_b200_mlp_step_resident_members": (C.c_int, [_P, _P, _P, C.c_longlong, _I, _P, _P, _P, _P, _P, _P, _P, _P]),
    "ani_b200_mlp_forward": (C.c_int, [_P, _P, _I, _P, _P, _P, _P, _P, _P, _P, _I, _P, _P]),
    "ani_b200_zero_live_blocks": (C.c_int, [_P, _P, _P, _P, _P]),
    "ani_b200_mlp_backward": (C.c_int, [_P, _P, _I, _P, _P, _P, _P, _P, _P, _I, _P, _P]),
    "ani_b200_pack_b_operand": (C.c_int, [_P, _I, _I, _I, _I, _F, _I, C.c_longlong, _P, C.c_longlong, _P]),
    "ani_b200_comm_create": (C.c_int, [_I, _I, C.c_longlong, C.c_longlong, _P]),
    "ani_b200_comm_handle": (C.c_int, [_P, _P]),
    "ani_b200_comm_connect": (C.c_int, [_P, _P]),
    "ani_b200_comm_buffers": (C.c_int, [_P, _P, _P, _P]),
    "ani_b200_comm_allreduce": (C.c_int, [_P, _P, _P, _P]),
    "ani_b200_comm_destroy": (C.c_int, [_P]),
    "ani_b200_active_aev_blocks": (C.c_int, [_P, _P, _I, _I, _I, _I, _I, _I, _I, _P, _P, _P]),
    "ani_b200_reduce_energies": (C.c_int, [_P, _P, _I, _P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P]),
    "ani_b200_charges": (C.c_int, [_P, _P, _P, _P, _P, _I, _I, _P, _I, _I, _I, C.c_double, _P, _I, _P, _P, _P]),
    "ani_b200_hessian_hidden_max": (C.c_int, [_P]),
    "ani_b200_hessian_jacobian": (C.c_int, [_P, _P, _P, _P, _I, _P, _P, _I, _P]),
    "ani_b200_hessian_network": (C.c_int, [_P, _P, _P, _P, _P, _P, _I, _P, _P, _P, _P, _P]),
    "ani_b200_hessian_geometric": (C.c_int, [_P, _P, _P, _P, _I, _P, _P, _I, _P, _P, _P, _P]),
    "ani_b200_hessian_assemble": (C.c_int, [_P, _P, _I, _P, _P, _P, _I, _P, _P]),
    "ani_b200_md_init": (C.c_int, [_P, _P, _I, _I, _P, _P]),
    "ani_b200_md_step": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P]),
    "ani_b200_md_step_cells": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P]),
    "ani_b200_md_noise": (C.c_int, [C.c_uint64, C.c_longlong, _I, _P, _P]),
    "ani_b200_md_step_npt": (C.c_int, [_P, _P, _P, _P, _P, _P]),
    "ani_b200_md_cell_noise": (C.c_int, [C.c_uint64, C.c_longlong, _I, _P, _P]),
    "ani_b200_opt_init": (C.c_int, [_P, _P, _I, _I, _P, _P]),
    "ani_b200_opt_step": (C.c_int, [_P, _P, _P, _P, _P, _P]),
    "ani_b200_opt_step_cells": (C.c_int, [_P, _P, _P, _P, _P, _P]),
    "ani_b200_opt_cell_init": (C.c_int, [_P, _P, _I, _P, _P]),
    "ani_b200_opt_cell_step": (C.c_int, [_P, _P, _P, _P, _P, _P]),
    "ani_b200_lbfgs_init": (C.c_int, [_P, _P, _I, _I, _P, _P]),
    "ani_b200_lbfgs_step": (C.c_int, [_P, _P, _P, _P, _P, _P]),
    "ani_b200_lbfgs_step_cells": (C.c_int, [_P, _P, _P, _P, _P, _P]),
    "ani_b200_neb_init": (C.c_int, [_P, _P, _I, _I, _P, _P]),
    "ani_b200_neb_step": (C.c_int, [_P, _P, _P, _P, _P, _P]),
    "ani_b200_neb_step_cells": (C.c_int, [_P, _P, _P, _P, _P, _P]),
    "ani_b200_neb_project": (C.c_int, [_P, _P, _P, _P]),
}

EXPORTED_SYMBOLS = tuple(_PROTOTYPES)


class ANIB200Error(RuntimeError):
    pass


VARIANTS = ("", "bf16x3")   # "" = the default build (2 x fp16 operand pieces), "bf16x3" = 3 x bfloat16 pieces


def variant_path(variant: str = "") -> str:
    """Path of a build variant of the library (build.py: same sources, other operand format)."""
    if not variant:
        return LIB_PATH
    return os.path.join(os.path.dirname(LIB_PATH), f"libani_b200_{variant}.so")


def available(variant: str = "") -> bool:
    return os.path.exists(variant_path(variant))


def _load(path: str) -> C.CDLL:
    if not os.path.exists(path):
        raise ImportError(
            f"{path} is missing: build it with `python -m torchani_b200.build` "
            "(nvcc, sm_90a).  torchani_b200 has no CPU / PyTorch fallback."
        )
    lib = C.CDLL(path)   # RTLD_LOCAL: the variants export the same C symbols side by side
    for name, (res, args) in _PROTOTYPES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    if lib.ani_b200_abi_version() != 4:
        raise ImportError(f"{path}: ABI version mismatch")
    return lib


_libs: tp.Dict[str, C.CDLL] = {}


def lib(variant: tp.Optional[str] = None) -> C.CDLL:
    """The C-ABI library; ``variant`` selects another operand-format build of the same sources (both can be
    loaded at once -- the automatic fallback of models.ANI uses that)."""
    v = variant or ""
    if v not in _libs:
        _libs[v] = _load(variant_path(v))
    return _libs[v]


class OperandFormat(tp.NamedTuple):
    parts: int           # 16-bit pieces per value: 2 = IEEE half, 3 = bfloat16
    value_scale: float   # power-of-two scale of AEV / activation operands
    grad_scale: float    # power-of-two scale of gradient operands


_fmts: tp.Dict[str, OperandFormat] = {}


def operand_format(variant: tp.Optional[str] = None) -> OperandFormat:
    """The tiled-operand format a library build was compiled for (ani_b200_operand_format)."""
    v = variant or ""
    if v not in _fmts:
        parts, vs, gs = C.c_int32(0), C.c_float(0), C.c_float(0)
        check(lib(v).ani_b200_operand_format(C.byref(parts), C.byref(vs), C.byref(gs)), "operand_format")
        _fmts[v] = OperandFormat(int(parts.value), float(vs.value), float(gs.value))
    return _fmts[v]


class OperandRangeError(RuntimeError):
    """A value left the range of the half-precision GEMM operand pieces (ANI_STATUS_OPERAND_RANGE)."""


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        l = lib()
        msg = l.ani_b200_error_string(rc).decode()
        if rc == -3:
            msg += " -- " + l.ani_b200_last_cuda_error().decode()
        raise ANIB200Error(f"{what}: {msg}" if what else msg)


def forbid_create_graph(what: str) -> None:
    """Raise when a custom autograd Function's backward runs under ``create_graph=True`` (grad mode is on inside a
    backward only then): its gradient has no graph of its own, so a second derivative taken through it would silently
    miss its term.  Called first in those backwards."""
    import torch
    if torch.is_grad_enabled():
        raise NotImplementedError(
            f"second derivatives through {what} are not supported (its backward has no graph of its own); for "
            "Hessians convert the model with torchani_b200.models.from_torchani and use ANI.energies_forces_hessians "
            "or torchani_b200.grad, which differentiate the fused step analytically (open systems, no D3, no LJ or "
            "Coulomb terms, no external neighbour lists)")


def ptr(t) -> int:
    """Raw device pointer of a torch tensor (None -> NULL)."""
    return None if t is None else t.data_ptr()
