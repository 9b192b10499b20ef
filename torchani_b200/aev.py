"""``AEVComputer`` with the interface of ``torchani.AEVComputer`` (aev/_computer.py:42-272).

``forward(elem_idxs, coords, cell, pbc) -> (C, A, out_dim)`` runs the fused CUDA kernel
(neighbour search + radial + angular in one pass, ``ani_b200_aev_forward``) and carries an
autograd edge to ``coords`` whose backward is ``ani_b200_aev_backward``.  The only compute
strategy is ``"b200"``: the reference's ``pyaev`` / ``cuaev`` strings are rejected.
"""
from __future__ import annotations

import ctypes as C
import math
import typing as tp
import warnings

import torch
from torch import Tensor

from . import _lib
from ._lib import check, ptr
from .engine import AEVConstants, _linspace
from .neighbors import (BucketGrid, CellList, Neighbors, NeighborlistArg, _parse_neighborlist, _validate_inputs,
                        effective_periodic_cell, supercell_for_thin_cell)


class SpeciesAEV(tp.NamedTuple):
    species: Tensor
    aevs: Tensor


class _Term(torch.nn.Module):
    def __init__(self, cutoff: float, cutoff_fn: str = "cosine") -> None:
        super().__init__()
        if cutoff_fn not in ("cosine", "smooth"):
            raise ValueError(f"Unsupported cutoff fn for the CUDA kernels: {cutoff_fn}")
        self.cutoff = float(cutoff)
        self.cutoff_fn = cutoff_fn
        self.num_feats = 0


class ANIRadial(_Term):
    """Constants of the radial sub-AEV (aev/_terms.py:118-241).  Holds parameters only; the
    terms are evaluated inside the fused CUDA kernel."""

    def __init__(self, eta: float, shifts: tp.Sequence[float], cutoff: float, cutoff_fn: str = "cosine"):
        super().__init__(cutoff, cutoff_fn)
        self.register_buffer("eta", torch.tensor([eta], dtype=torch.float))
        self.register_buffer("shifts", torch.tensor(shifts, dtype=torch.float))
        self.num_feats = len(shifts)

    @classmethod
    def cover_linearly(cls, start: float = 0.9, cutoff: float = 5.2, eta: float = 19.7,
                       num_shifts: int = 16, cutoff_fn: str = "cosine"):
        return cls(eta, _linspace(start, cutoff, num_shifts), cutoff, cutoff_fn)

    @classmethod
    def like_1x(cls, cutoff_fn: str = "cosine"):
        return cls.cover_linearly(0.9, 5.2, 16.0, 16, cutoff_fn)

    @classmethod
    def like_2x(cls, cutoff_fn: str = "cosine"):
        return cls.cover_linearly(0.8, 5.1, 19.7, 16, cutoff_fn)


class ANIAngular(_Term):
    """Constants of the angular sub-AEV (aev/_terms.py:244-408)."""

    def __init__(self, eta: float, zeta: float, shifts: tp.Sequence[float], sections: tp.Sequence[float],
                 cutoff: float, cutoff_fn: str = "cosine"):
        super().__init__(cutoff, cutoff_fn)
        self.register_buffer("eta", torch.tensor([eta], dtype=torch.float))
        self.register_buffer("zeta", torch.tensor([zeta], dtype=torch.float))
        self.register_buffer("shifts", torch.tensor(shifts, dtype=torch.float))
        self.register_buffer("sections", torch.tensor(sections, dtype=torch.float))
        self.num_feats = len(shifts) * len(sections)

    @classmethod
    def cover_linearly(cls, start: float = 0.9, cutoff: float = 3.5, eta: float = 12.5, zeta: float = 14.1,
                       num_shifts: int = 8, num_sections: int = 4, cutoff_fn: str = "cosine"):
        angle_start = math.pi / num_sections / 2
        return cls(eta, zeta, _linspace(start, cutoff, num_shifts),
                   _linspace(angle_start, math.pi + angle_start, num_sections), cutoff, cutoff_fn)

    @classmethod
    def like_1x(cls, cutoff_fn: str = "cosine"):
        return cls.cover_linearly(0.9, 3.5, 8.0, 32.0, 4, 8, cutoff_fn)

    @classmethod
    def like_2x(cls, cutoff_fn: str = "cosine"):
        return cls.cover_linearly(0.8, 3.5, 12.5, 14.1, 8, 4, cutoff_fn)


class _AEVFunction(torch.autograd.Function):
    """coords -> AEVs through the fused kernel; backward = the force kernel."""

    @staticmethod
    def forward(ctx, coords: Tensor, species: Tensor, cell: tp.Optional[Tensor], pbc: bool,
                computer: "AEVComputer") -> Tensor:
        consts = computer.constants
        g = BucketGrid(species, coords, cell, pbc, consts.rcr)
        n = g.n
        dev = coords.device
        out = torch.zeros(n, consts.out_dim, dtype=torch.float32, device=dev)
        cap = computer.nbr_cap
        nbr_cnt = torch.zeros(n, dtype=torch.int32, device=dev)
        nbr_list = torch.zeros(n * cap, dtype=torch.int32, device=dev)
        params = computer._params()
        # rows of the output are the flat input indices: row_of == sorted_orig
        check(_lib.lib().ani_b200_aev_forward(C.byref(params), ptr(g.grid), ptr(g.bin_start), ptr(g.spos),
                                              ptr(g.sbin), None, None, None, n, 0, n, ptr(g.sorted_orig), ptr(out),
                                              consts.out_dim, 0, ptr(nbr_cnt), ptr(nbr_list), cap, ptr(g.status),
                                              g.stream), "aev_forward")
        ctx.g, ctx.nbr_cnt, ctx.nbr_list, ctx.computer = g, nbr_cnt, nbr_list, computer
        computer._last_grid = g
        return out.view(species.shape[0], species.shape[1], consts.out_dim)

    @staticmethod
    def backward(ctx, grad_aev: Tensor):
        _lib.forbid_create_graph("the CUDA AEV computer (_AEVFunction)")
        g, computer = ctx.g, ctx.computer
        consts = computer.constants
        grad_aev = grad_aev.reshape(g.n, consts.out_dim).to(torch.float32).contiguous()
        grad = torch.zeros(g.n, 3, dtype=torch.float32, device=grad_aev.device)
        params = computer._params()
        st = torch.cuda.current_stream(grad_aev.device).cuda_stream
        check(_lib.lib().ani_b200_aev_backward(C.byref(params), ptr(g.grid), ptr(g.spos), ptr(g.sorted_orig),
                                               None, g.n, 0, g.n, ptr(g.sorted_orig), ptr(grad_aev), consts.out_dim,
                                               ptr(ctx.nbr_cnt), ptr(ctx.nbr_list), computer.nbr_cap, ptr(grad),
                                               ptr(g.status), 0, None, st), "aev_backward")
        return grad.view(g.n_conf, g.n_per_conf, 3), None, None, None, None


class _AEVFromNeighbors(torch.autograd.Function):
    """AEVs from a caller-supplied half pair list (``Neighbors``), gradient to coords only."""

    @staticmethod
    def forward(ctx, coords: Tensor, species: Tensor, indices: Tensor, diff_vectors: Tensor,
                computer: "AEVComputer") -> Tensor:
        consts = computer.constants
        dev = coords.device
        n_conf, n_per_conf = species.shape
        n = n_conf * n_per_conf
        num_pairs = int(indices.shape[1])
        i32 = dict(dtype=torch.int32, device=dev)
        spos = torch.zeros(n, 4, dtype=torch.float32, device=dev)
        spos[:, 3] = species.reshape(-1).to(torch.int32).view(torch.float32)   # only the species is read
        grid = torch.zeros(C.sizeof(_lib.Grid) // 4, **i32)
        grid[_lib.Grid.n_real.offset // 4] = n
        ident = torch.arange(n, **i32)
        row_start = torch.zeros(n + 1, **i32)
        row_j = torch.zeros(max(2 * num_pairs, 1), **i32)
        row_d = torch.zeros(max(2 * num_pairs, 1), 4, dtype=torch.float32, device=dev)
        scratch = torch.zeros(2 * n, **i32)
        status = torch.zeros(1, **i32)
        idx = indices.to(torch.int64).contiguous()
        dv = diff_vectors.detach().to(torch.float32).contiguous()
        st = torch.cuda.current_stream(dev).cuda_stream
        L = _lib.lib()
        params = computer._params()
        cap = computer.nbr_cap
        check(L.ani_b200_pairs_to_rows(idx[0].data_ptr(), idx[1].data_ptr(), ptr(dv), num_pairs, n, cap,
                                       ptr(row_start), ptr(row_j), ptr(row_d), ptr(scratch), ptr(status), st),
              "pairs_to_rows")
        out = torch.zeros(n, consts.out_dim, dtype=torch.float32, device=dev)
        check(L.ani_b200_aev_forward_rows(C.byref(params), ptr(grid), ptr(spos), ptr(row_start), ptr(row_j),
                                          ptr(row_d), n, ptr(ident), ptr(out), consts.out_dim, 0, cap, ptr(status),
                                          st), "aev_forward_rows")
        ctx.saved = (grid, spos, ident, row_start, row_j, row_d, status)
        ctx.computer, ctx.shape = computer, (n_conf, n_per_conf)
        computer._last_status = status
        return out.view(n_conf, n_per_conf, consts.out_dim)

    @staticmethod
    def backward(ctx, grad_aev: Tensor):
        _lib.forbid_create_graph("the CUDA AEV computer with a caller-supplied neighbour list (_AEVFromNeighbors)")
        grid, spos, ident, row_start, row_j, row_d, status = ctx.saved
        computer = ctx.computer
        consts = computer.constants
        n_conf, n_per_conf = ctx.shape
        n = n_conf * n_per_conf
        g = grad_aev.reshape(n, consts.out_dim).to(torch.float32).contiguous()
        grad = torch.zeros(n, 3, dtype=torch.float32, device=g.device)
        st = torch.cuda.current_stream(g.device).cuda_stream
        params = computer._params()
        check(_lib.lib().ani_b200_aev_backward_rows(C.byref(params), ptr(grid), ptr(spos), ptr(ident), ptr(row_start),
                                                    ptr(row_j), ptr(row_d), n, ptr(ident), ptr(g), consts.out_dim,
                                                    computer.nbr_cap, ptr(grad), ptr(status), st),
              "aev_backward_rows")
        return grad.view(n_conf, n_per_conf, 3), None, None, None, None


class _AEVFromFullList(torch.autograd.Function):
    """AEVs of the atoms in ``ilist`` from a full neighbour list over local + ghost atoms (MD-engine format);
    gradient to all coordinates (csrc/cuaev.cpp:225-246)."""

    @staticmethod
    def forward(ctx, coords: Tensor, species: Tensor, ilist: Tensor, jlist: Tensor, numneigh: Tensor,
                computer: "AEVComputer") -> Tensor:
        consts = computer.constants
        dev = coords.device
        n = species.shape[1]
        i32 = dict(dtype=torch.int32, device=dev)
        spos = torch.zeros(n, 4, dtype=torch.float32, device=dev)
        spos[:, 3] = species.reshape(-1).to(torch.int32).view(torch.float32)
        grid = torch.zeros(C.sizeof(_lib.Grid) // 4, **i32)
        grid[_lib.Grid.n_real.offset // 4] = n
        ident = torch.arange(n, **i32)
        il, jl, nn_ = (t.to(torch.int32).contiguous() for t in (ilist, jlist, numneigh))
        n_i, cap_rows = int(il.shape[0]), max(int(jl.shape[0]), 1)
        row_start = torch.zeros(n + 1, **i32)
        row_j = torch.zeros(cap_rows, **i32)
        row_d = torch.zeros(cap_rows, 4, dtype=torch.float32, device=dev)
        scratch = torch.zeros(n + n_i + 2, **i32)
        status = torch.zeros(1, **i32)
        xyz = coords.detach().reshape(-1, 3).to(torch.float32).contiguous()
        st = torch.cuda.current_stream(dev).cuda_stream
        L = _lib.lib()
        params = computer._params()
        cap = computer.nbr_cap
        check(L.ani_b200_full_nbrlist_to_rows(ptr(xyz), n, ptr(il), ptr(nn_), ptr(jl), n_i, consts.rcr, cap,
                                              ptr(row_start), ptr(row_j), ptr(row_d), ptr(scratch), ptr(status), st),
              "full_nbrlist_to_rows")
        out = torch.zeros(n, consts.out_dim, dtype=torch.float32, device=dev)
        check(L.ani_b200_aev_forward_rows(C.byref(params), ptr(grid), ptr(spos), ptr(row_start), ptr(row_j),
                                          ptr(row_d), n, ptr(ident), ptr(out), consts.out_dim, 0, cap, ptr(status),
                                          st), "aev_forward_rows")
        ctx.saved = (grid, spos, ident, row_start, row_j, row_d, status)
        ctx.computer, ctx.n = computer, n
        computer._last_status = status
        return out.view(1, n, consts.out_dim)

    @staticmethod
    def backward(ctx, grad_aev: Tensor):
        _lib.forbid_create_graph("the CUDA AEV computer with a full neighbour list (_AEVFromFullList)")
        grid, spos, ident, row_start, row_j, row_d, status = ctx.saved
        computer, n = ctx.computer, ctx.n
        consts = computer.constants
        g = grad_aev.reshape(n, consts.out_dim).to(torch.float32).contiguous()
        grad = torch.zeros(n, 3, dtype=torch.float32, device=g.device)
        st = torch.cuda.current_stream(g.device).cuda_stream
        params = computer._params()
        check(_lib.lib().ani_b200_aev_backward_rows(C.byref(params), ptr(grid), ptr(spos), ptr(ident), ptr(row_start),
                                                    ptr(row_j), ptr(row_d), n, ptr(ident), ptr(g), consts.out_dim,
                                                    computer.nbr_cap, ptr(grad), ptr(status), st),
              "aev_backward_rows")
        return grad.view(1, n, 3), None, None, None, None, None


class AEVComputer(torch.nn.Module):
    r"""Computes atomic environment vectors on the GPU (interface of aev/_computer.py:42-272).

    Args:
        radial, angular: ``ANIRadial`` / ``ANIAngular`` (or ``"ani1x"`` / ``"ani2x"``)
        num_species: number of supported elements
        strategy: only ``"b200"`` (``"auto"`` is accepted as an alias)
        neighborlist: kept for interface compatibility; the fused kernel searches the bucket
            grid itself, the module is what ``model.neighborlist`` exposes to callers.
    """

    def __init__(self, radial: tp.Union[str, ANIRadial], angular: tp.Union[str, ANIAngular], num_species: int,
                 strategy: str = "b200", cutoff_fn: tp.Optional[str] = None,
                 neighborlist: NeighborlistArg = "cell_list", nbr_cap: int = 128):
        super().__init__()
        if isinstance(radial, str):
            radial = {"ani1x": ANIRadial.like_1x, "ani1ccx": ANIRadial.like_1x, "ani2x": ANIRadial.like_2x}[radial]()
        if isinstance(angular, str):
            angular = {"ani1x": ANIAngular.like_1x, "ani1ccx": ANIAngular.like_1x,
                       "ani2x": ANIAngular.like_2x}[angular]()
        if type(radial) is not ANIRadial or type(angular) is not ANIAngular:
            raise ValueError("the CUDA kernels implement ANIRadial / ANIAngular terms only")
        if radial.cutoff_fn != angular.cutoff_fn:
            raise ValueError("Cutoff fn must be the same for angular and radial terms")
        if angular.cutoff > radial.cutoff:
            raise ValueError(f"Angular cutoff {angular.cutoff} should be smaller than radial cutoff {radial.cutoff}")
        self.radial, self.angular = radial, angular
        self.num_species = num_species
        self.num_species_pairs = num_species * (num_species + 1) // 2
        self.radial_len = radial.num_feats * num_species
        self.angular_len = angular.num_feats * self.num_species_pairs
        self.out_dim = self.radial_len + self.angular_len
        self.register_buffer("triu_index", self._calculate_triu_index(num_species))
        self.neighborlist = _parse_neighborlist(neighborlist)
        self.nbr_cap = nbr_cap
        self._strategy = ""
        self.set_strategy(strategy)
        self._struct = None
        self._consts: tp.Optional[AEVConstants] = None
        self._last_grid: tp.Optional[BucketGrid] = None
        self._last_status: tp.Optional[Tensor] = None
        self.constants.to_struct()  # validates the configuration early

    # -- strategy strings (aev/_computer.py:120-149) ---------------------------------------
    @property
    def strategy(self) -> str:
        return self._strategy

    def set_strategy(self, strat: str) -> None:
        if strat in ("b200", "auto"):
            self._strategy = "b200"
        elif strat in ("pyaev", "cuaev", "cuaev-fused", "cuaev-interface"):
            raise ValueError(f"{strat} strategy is not available in torchani_b200 (only 'b200')")
        else:
            raise ValueError("Unknown compute strategy")

    @staticmethod
    def _calculate_triu_index(num_species: int) -> Tensor:
        # aev/_computer.py:184-191
        s1, s2 = torch.triu_indices(num_species, num_species).unbind(0)
        ret = torch.zeros(num_species, num_species, dtype=torch.long)
        ret[s1, s2] = torch.arange(s1.shape[0])
        ret[s2, s1] = torch.arange(s1.shape[0])
        return ret

    @property
    def constants(self) -> AEVConstants:
        if self._consts is None:  # reading the buffers costs a device sync: do it once
            self._consts = self._read_constants()
        return self._consts

    def _read_constants(self) -> AEVConstants:
        r, a = self.radial, self.angular
        return AEVConstants(self.num_species, r.cutoff, a.cutoff, float(r.eta.item()),
                            tuple(float(v) for v in r.shifts.tolist()), float(a.eta.item()),
                            float(a.zeta.item()), tuple(float(v) for v in a.shifts.tolist()),
                            tuple(float(v) for v in a.sections.tolist()), r.cutoff_fn)

    def _params(self):
        if self._struct is None:
            self._struct = self.constants.to_struct()
        return self._struct

    def forward(self, elem_idxs: Tensor, coords: tp.Optional[Tensor] = None, cell: tp.Optional[Tensor] = None,
                pbc: tp.Optional[Tensor] = None) -> Tensor:
        if isinstance(elem_idxs, tuple):  # legacy call form, aev/_computer.py:211-222
            warnings.warn("`aev_computer((species, coords), cell, pbc)` is the TorchANI 1 signature; "
                          "use `aev_computer(species, coords, cell, pbc)`")
            _idx, _coords = elem_idxs
            return SpeciesAEV(_idx, self(_idx, _coords, coords, cell))
        assert coords is not None
        assert elem_idxs.dim() == 2
        assert coords.shape == (elem_idxs.shape[0], elem_idxs.shape[1], 3)
        _validate_inputs(self.radial.cutoff, elem_idxs, coords, cell, pbc)
        sup = None if isinstance(self.neighborlist, CellList) else \
            supercell_for_thin_cell(elem_idxs, coords, cell, pbc, self.radial.cutoff)
        if sup is not None:   # periodic cell thinner than the cutoff: AEVs of the original atoms of a supercell
            return self(sup[0], sup[1], sup[2], pbc)[:, :elem_idxs.shape[1]]
        cell = effective_periodic_cell(coords, cell, pbc, self.radial.cutoff)   # PBC in some directions only
        aev = _AEVFunction.apply(coords, elem_idxs, cell, pbc is not None, self)
        if self._last_grid is not None:
            self._last_grid.raise_on_status()
        return aev

    def compute_from_neighbors(self, elem_idxs: Tensor, coords: Tensor, neighbors: Neighbors) -> Tensor:
        r"""Compute the AEVs from the result of a neighborlist calculation (aev/_computer.py:251-272).

        Like the reference's cuAEV half-neighbour-list path (csrc/cuaev.cpp:141-163) the pairs and
        ``diff_vectors`` are taken as given (pairs beyond the radial cutoff must already be gone) and
        the gradient goes to ``coords`` only."""
        assert elem_idxs.dim() == 2 and coords.shape == (elem_idxs.shape[0], elem_idxs.shape[1], 3)
        if coords.device.type != "cuda":
            raise ValueError("torchani_b200 runs on CUDA tensors only (there is no CPU path)")
        aev = _AEVFromNeighbors.apply(coords, elem_idxs, neighbors.indices, neighbors.diff_vectors, self)
        code = int(self._last_status.item())
        if code & _lib.STATUS_NBR_OVERFLOW:
            raise RuntimeError(f"an atom has more than nbr_cap={self.nbr_cap} neighbours in the given list")
        if code & _lib.STATUS_ANG_OVERFLOW:
            raise RuntimeError(f"an atom has more than {_lib.ANI_MAX_ANG} neighbours within the angular cutoff")
        return aev

    def compute_from_full_neighborlist(self, elem_idxs: Tensor, coords: Tensor, ilist_unique: Tensor, jlist: Tensor,
                                       numneigh: Tensor) -> Tensor:
        r"""AEVs from a FULL neighbour list with ghost atoms, the format MD engines (LAMMPS, pmemd) hand over --
        the reference's ``_compute_cuaev_with_full_nbrlist`` (aev/_computer.py:409-438 ->
        ``cuaev::run_with_full_nbrlist``, csrc/aev.cu:1048-1126,1868-1956):

        * ``elem_idxs (1, A)`` / ``coords (1, A, 3)`` hold local AND ghost atoms (ghosts at their image positions),
        * ``ilist_unique (nI,)`` the atoms whose AEV is wanted, ``numneigh (nI,)`` their neighbour counts,
          ``jlist (sum numneigh,)`` the neighbours of ``ilist[0], ilist[1], ...`` one after the other (indices into
          the A atoms; a list built with cutoff + skin is screened with the true cutoff here).

        Returns ``(1, A, out_dim)``: rows of ``ilist`` atoms filled, all others zero; autograd reaches the
        coordinates of local and ghost atoms alike (the MD engine folds ghost forces back).  Single molecule only,
        as the reference."""
        if coords.shape[0] != 1:
            raise ValueError("cuAEV with full neighborlist doesn't support batches")
        assert elem_idxs.dim() == 2 and coords.shape == (1, elem_idxs.shape[1], 3)
        if coords.device.type != "cuda":
            raise ValueError("torchani_b200 runs on CUDA tensors only (there is no CPU path)")
        aev = _AEVFromFullList.apply(coords, elem_idxs, ilist_unique, jlist, numneigh, self)
        code = int(self._last_status.item())
        if code & _lib.STATUS_NBR_OVERFLOW:
            raise RuntimeError(f"an atom has more than nbr_cap={self.nbr_cap} neighbours in the given list")
        if code & _lib.STATUS_ANG_OVERFLOW:
            raise RuntimeError(f"an atom has more than {_lib.ANI_MAX_ANG} neighbours within the angular cutoff")
        return aev

    _compute_cuaev_with_full_nbrlist = compute_from_full_neighborlist   # the reference's (private) name

    # -- constructors (aev/_computer.py:498-666) -------------------------------------------
    @classmethod
    def like_1x(cls, num_species: int = 4, strategy: str = "b200", cutoff_fn: str = "cosine",
                neighborlist: NeighborlistArg = "cell_list", **kw):
        return cls(ANIRadial.like_1x(cutoff_fn), ANIAngular.like_1x(cutoff_fn), num_species, strategy,
                   neighborlist=neighborlist, **kw)

    @classmethod
    def like_2x(cls, num_species: int = 7, strategy: str = "b200", cutoff_fn: str = "cosine",
                neighborlist: NeighborlistArg = "cell_list", **kw):
        return cls(ANIRadial.like_2x(cutoff_fn), ANIAngular.like_2x(cutoff_fn), num_species, strategy,
                   neighborlist=neighborlist, **kw)

    @classmethod
    def from_constants(cls, radial_cutoff: float, angular_cutoff: float, radial_eta: float,
                       radial_shifts: tp.Sequence[float], angular_eta: float, angular_zeta: float,
                       angular_shifts: tp.Sequence[float], sections: tp.Sequence[float], num_species: int,
                       strategy: str = "b200", cutoff_fn: str = "cosine",
                       neighborlist: NeighborlistArg = "cell_list"):
        return cls(ANIRadial(radial_eta, radial_shifts, radial_cutoff, cutoff_fn),
                   ANIAngular(angular_eta, angular_zeta, angular_shifts, sections, angular_cutoff, cutoff_fn),
                   num_species, strategy, neighborlist=neighborlist)

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs) -> None:
        self._consts = None
        self._struct = None
        super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)

    def extra_repr(self) -> str:
        return (f"out_dim={self.out_dim}, radial_len={self.radial_len}, angular_len={self.angular_len}, "
                f"num_species={self.num_species}, strategy={self._strategy}")
