"""Neighbour lists with the interface of ``torchani.neighbors`` (neighbors.py:13-18,140-166).

``CellList`` / ``AllPairs`` / ``AdaptiveList`` all run the same bucket-grid kernels
(``ani_b200_build_cells`` + ``ani_b200_half_neighbor_*``): one conformer is bucketed on a grid
(periodic or bounding box), an open batch uses one bucket per conformer, a periodic batch one
sub-grid of the shared cell per conformer.  The result has the
reference's format -- ``Neighbors(indices (2,P) int64 into the flattened atoms, distances (P,),
diff_vectors (P,3) = x[idx0] - x[idx1] + shift)`` -- and carries autograd to ``coords`` the same
way (neighbors.py:107-112).  Pair ORDER differs from the reference (it is not specified there
either: the reference's argsort is unstable); compare as sets.
"""
from __future__ import annotations

import ctypes as C
import math
import typing as tp

import torch
from torch import Tensor

from . import _lib
from ._lib import Grid, check, ptr


class Neighbors(tp.NamedTuple):
    r"""Holds pairs of atoms that are neighbors (neighbors.py:13-18)."""

    indices: Tensor  #: Long tensor with idxs of neighbor pairs. Shape ``(2, pairs)``
    distances: Tensor  #: The associated pair distances. Shape is ``(pairs,)``
    diff_vectors: Tensor  #: The associated difference vectors. Shape is ``(pairs, 3)``


def discard_outside_cutoff(neighbors: Neighbors, cutoff: float) -> Neighbors:
    r"""Discard neighbors with distances that lie outside of the given cutoff (neighbors.py:46-55)"""
    keep = (neighbors.distances <= cutoff).nonzero().flatten()
    return Neighbors(neighbors.indices.index_select(1, keep), neighbors.distances.index_select(0, keep),
                     neighbors.diff_vectors.index_select(0, keep))


def narrow_down(cutoff: float, elem_idxs: Tensor, coords: Tensor, neighbor_idxs: Tensor,
                shifts: tp.Optional[Tensor] = None) -> Neighbors:
    r"""Takes a set of potential neighbor idxs (e.g. the Verlet list of an MD engine, built with a skin) and
    narrows it down to true neighbors (neighbors.py:64-113): pairs with a dummy atom and pairs beyond the cutoff
    are dropped, ``diff_vectors = x[idx0] - x[idx1] + shift`` keeps its autograd edge to ``coords``.  Plain
    tensor glue (index_select over the candidate pairs), as in the reference -- the AEV kernels then consume the
    result through ``ani_b200_pairs_to_rows``."""
    import math
    mask = (elem_idxs == -1).view(-1)
    if bool(mask.any()):
        pair_mask = mask[neighbor_idxs.view(-1)].view(2, -1)
        keep = (~pair_mask.any(dim=0)).nonzero().flatten()
        neighbor_idxs = neighbor_idxs.index_select(1, keep)
        if shifts is not None:
            shifts = shifts.index_select(0, keep)
    flat = coords.view(-1, 3)
    if cutoff == math.inf:
        if shifts is not None:
            raise ValueError("PBC can't use an infinite cutoff")
    else:
        det = flat.detach()
        d = det.index_select(0, neighbor_idxs[0]) - det.index_select(0, neighbor_idxs[1])
        if shifts is not None:
            d = d + shifts
        keep = (d.norm(2, -1) <= cutoff).nonzero().flatten()
        neighbor_idxs = neighbor_idxs.index_select(1, keep)
        if shifts is not None:
            shifts = shifts.index_select(0, keep)
    diff = flat.index_select(0, neighbor_idxs[0]) - flat.index_select(0, neighbor_idxs[1])
    if shifts is not None:
        diff = diff + shifts
    return Neighbors(neighbor_idxs, diff.norm(2, -1), diff)


def _validate_inputs(cutoff: float, species: Tensor, coords: Tensor, cell: tp.Optional[Tensor],
                     pbc: tp.Optional[Tensor], supports_batches: bool = True, conformer_cells: bool = False) -> None:
    # neighbors.py:918-949
    if cutoff <= 0.0:
        raise ValueError("Cutoff must be a strictly positive float")
    if species.dim() != 2 or coords.shape != (species.shape[0], species.shape[1], 3):
        raise ValueError("species must be (C, A) and coords (C, A, 3)")
    if cell is not None and cell.dim() != 2:
        # one cell per conformer (C, 3, 3) is a models.ANI input (grid mode 3); the neighbour lists and the
        # AEVComputer take one (3, 3) cell
        if not conformer_cells:
            raise ValueError("one cell per conformer, (C, 3, 3), is supported by models.ANI only; neighbour lists "
                             "and AEVComputer take one (3, 3) cell")
        if cell.shape != (species.shape[0], 3, 3):
            raise ValueError(f"cell must be (3, 3) or one cell per conformer, ({species.shape[0]}, 3, 3); "
                             f"got {tuple(cell.shape)}")
        if pbc is not None and not bool(pbc.all()):
            raise ValueError("one cell per conformer needs PBC in all three directions")
    if not supports_batches and coords.shape[0] != 1:
        raise ValueError("This neighborlist doesn't support batches")
    if pbc is not None:
        if not bool(pbc.any()):
            raise ValueError(
                "pbc = torch.tensor([False, False, False]) is not supported anymore please use pbc = None"
            )
        if cell is None:
            raise ValueError("If pbc is not None, cell should be present")
    elif cell is not None:
        raise ValueError("Cell is not supported if not using pbc")
    if coords.device.type != "cuda":
        raise ValueError("torchani_b200 runs on CUDA tensors only (there is no CPU path)")
    if coords.dtype != torch.float32:
        raise ValueError("torchani_b200 kernels are float32; got " + str(coords.dtype))


def effective_periodic_cell(coords: Tensor, cell: tp.Optional[Tensor], pbc: tp.Optional[Tensor],
                            cutoff: float) -> tp.Optional[Tensor]:
    """PBC in only some directions (neighbors.py:214-275: the reference enumerates image shifts along the periodic
    lattice vectors only) -> an equivalent FULLY periodic cell for the bucket-grid kernels: every non-periodic lattice
    vector is replaced by one along the normal of the other two, long enough (extent of the atoms along it + cutoff +
    1 A) that no pair within the cutoff crosses it.  Same pair set, same shifts along the periodic vectors, zero
    shift along the others.  One host synchronisation (the extent), only in this case."""
    if pbc is not None and cutoff == math.inf:
        raise ValueError("PBC can't use an infinite cutoff")
    if pbc is None or cell is None or bool(pbc.all()):
        return cell
    c = cell.detach().to(torch.float64)
    x = coords.detach().reshape(-1, 3).to(torch.float64)
    new = c.clone()
    flags = [bool(v) for v in pbc.tolist()]
    for d in range(3):
        if flags[d]:
            continue
        a, b = (k for k in range(3) if k != d)
        n = torch.linalg.cross(new[a], new[b])
        n = n / n.norm()
        if float(torch.dot(n, c[d])) < 0:
            n = -n
        proj = x @ n
        new[d] = n * (float(proj.max() - proj.min()) + cutoff + 1.0)
    return new.to(cell.dtype)


def supercell_for_thin_cell(species: Tensor, coords: Tensor, cell: tp.Optional[Tensor], pbc: tp.Optional[Tensor],
                            cutoff: float):
    """A periodic cell THINNER than the cutoff (the reference's `all_pairs` pairs every atom with several lattice
    images, neighbors.py:245-275; the bucket grid needs one bucket per cutoff): replicate the cell n_d = ceil(cutoff /
    width_d) times along every too-thin direction.  Returns None if the cell is wide enough, else
    ``(species_rep (C, R*A), coords_rep (C, R*A, 3), cell_rep, R)``, every conformer replicated within its own row,
    with the original atoms first: every replica is
    translation-equivalent, so AEVs / atomic energies of the original atoms are those of the first A atoms, the energy
    is 1/R of the supercell's, and dE/dx of an original atom is the SUM over its R copies of the supercell gradient
    (which autograd does by itself through the replication below).  One host sync (the cell widths)."""
    if pbc is None or cell is None:
        return None
    if cutoff == math.inf:
        raise ValueError("PBC can't use an infinite cutoff")
    c = cell.detach().to(torch.float64).cpu()
    inv = torch.linalg.inv(c)
    widths = 1.0 / inv.norm(dim=0)          # distance between the lattice planes of direction d
    flags = [bool(v) for v in pbc.tolist()]
    reps = [int(-(-(cutoff + 1e-5) // float(widths[d]))) if flags[d] else 1 for d in range(3)]
    if max(reps) == 1:
        return None
    shifts = torch.tensor([[a, b, k] for a in range(reps[0]) for b in range(reps[1]) for k in range(reps[2])],
                          dtype=coords.dtype, device=coords.device)
    offs = shifts @ cell.to(coords.dtype)                               # (R, 3); the first one is zero
    R = offs.shape[0]
    coords_rep = (coords.unsqueeze(1) + offs.view(1, R, 1, 3)).reshape(coords.shape[0], -1, 3)
    species_rep = species.repeat(1, R)
    cell_rep = cell * torch.tensor(reps, dtype=cell.dtype, device=cell.device).view(3, 1)
    return species_rep, coords_rep, cell_rep, R


class BucketGrid:
    """Device buffers of one bucket-grid build (shared by the neighbour list and the AEV API)."""

    def __init__(self, species: Tensor, coords: Tensor, cell: tp.Optional[Tensor], pbc: bool, cutoff: float):
        dev = coords.device
        n_conf, n_per_conf = species.shape
        n = n_conf * n_per_conf
        self.n, self.n_conf, self.n_per_conf = n, n_conf, n_per_conf
        i32 = dict(dtype=torch.int32, device=dev)
        # one conformer: its own grid; an open batch: one bucket per conformer; a periodic batch (mode 2): one sub-grid
        # per conformer with the bucket capacity of a single system
        self.mode = 0 if n_conf == 1 else (2 if pbc else 1)
        if self.mode == 0:
            self.max_bins = max(64, n + 2)
        elif self.mode == 1:
            self.max_bins = n_conf + 2
        else:
            self.max_bins = n_conf * (max(64, n_per_conf + 2) - 1) + 1
        self.grid = torch.zeros(C.sizeof(Grid) // 4, **i32)
        self.status = torch.zeros(1, **i32)
        self.bin_start = torch.zeros(self.max_bins + 2, **i32)
        self.sorted_orig = torch.zeros(n, **i32)
        self.orig_to_sorted = torch.zeros(n, **i32)
        self.spos = torch.zeros(n, 4, dtype=torch.float32, device=dev)
        self.sbin = torch.zeros(n, **i32)
        scratch = torch.zeros(3 * n + self.max_bins + 2, **i32)
        self.species_i32 = species.reshape(-1).to(torch.int32).contiguous()
        coords_f = coords.detach().reshape(-1, 3).contiguous()
        cell_f = None if cell is None else cell.detach().to(torch.float32).reshape(-1).contiguous()
        self.stream = torch.cuda.current_stream(dev).cuda_stream
        check(_lib.lib().ani_b200_build_cells(
            ptr(coords_f), ptr(self.species_i32), n_conf, n_per_conf, ptr(cell_f), int(pbc),
            self.mode, float(cutoff), self.max_bins, ptr(self.grid), ptr(self.bin_start),
            ptr(self.sorted_orig), ptr(self.orig_to_sorted), ptr(self.spos), ptr(self.sbin), None, ptr(scratch),
            ptr(self.status), self.stream), "build_cells")

    def raise_on_status(self) -> None:
        code = int(self.status.item())
        if code & _lib.STATUS_CELL_TOO_SMALL:
            raise RuntimeError("Cell is too small to perform pbc calculations")  # neighbors.py:402-403
        if code & _lib.STATUS_NBR_OVERFLOW:
            raise RuntimeError("neighbour capacity exceeded (raise nbr_cap, <= 256)")
        if code & _lib.STATUS_ANG_OVERFLOW:
            raise RuntimeError(f"an atom has more than {_lib.ANI_MAX_ANG} neighbours within the angular cutoff")
        if code & _lib.STATUS_PAIR_OVERFLOW:
            raise RuntimeError("half neighbour list capacity exceeded")


def _half_list(cutoff: float, species: Tensor, coords: Tensor, cell: tp.Optional[Tensor],
               pbc: tp.Optional[Tensor]) -> Neighbors:
    # (a periodic batch, neighbors.py:187-212, is one grid with a sub-grid per conformer: the pair indices refer to the
    # flattened (C * A) atoms, conformer after conformer)
    cell = effective_periodic_cell(coords, cell, pbc, cutoff)
    g = BucketGrid(species, coords, cell, pbc is not None, cutoff)
    L = _lib.lib()
    n = g.n
    dev = coords.device
    pair_start = torch.zeros(2 * n + 2, dtype=torch.int32, device=dev)
    check(L.ani_b200_half_neighbor_count(ptr(g.grid), ptr(g.bin_start), ptr(g.spos), ptr(g.sbin),
                                         ptr(g.sorted_orig), n, float(cutoff), ptr(pair_start), g.stream),
          "half_neighbor_count")
    num_pairs = int(pair_start[n].item())  # the one host sync of this API (the reference has several)
    g.raise_on_status()
    idx = torch.empty(2, num_pairs, dtype=torch.int64, device=dev)
    dist = torch.empty(num_pairs, dtype=torch.float32, device=dev)
    diff = torch.empty(num_pairs, 3, dtype=torch.float32, device=dev)
    if num_pairs:
        check(L.ani_b200_half_neighbor_fill(ptr(g.grid), ptr(g.bin_start), ptr(g.spos), ptr(g.sbin),
                                            ptr(g.sorted_orig), n, float(cutoff), ptr(pair_start), num_pairs,
                                            idx[0].data_ptr(), idx[1].data_ptr(), ptr(dist), ptr(diff),
                                            ptr(g.status), g.stream), "half_neighbor_fill")
    if coords.requires_grad:
        # same autograd edge as neighbors.py:107-112: diff = x[i0] - x[i1] + (constant shift)
        flat = coords.reshape(-1, 3)
        raw = flat.index_select(0, idx[0]) - flat.index_select(0, idx[1])
        diff = raw + (diff - raw.detach())
        dist = diff.norm(2, -1)
    return Neighbors(idx, dist, diff)


def cell_list(cutoff: float, species: Tensor, coords: Tensor, cell: tp.Optional[Tensor] = None,
              pbc: tp.Optional[Tensor] = None) -> Neighbors:
    """neighbors.py:366-415 (single conformer)."""
    _validate_inputs(cutoff, species, coords, cell, pbc, supports_batches=False)
    return _half_list(cutoff, species, coords, cell, pbc)


def all_pairs(cutoff: float, species: Tensor, coords: Tensor, cell: tp.Optional[Tensor] = None,
              pbc: tp.Optional[Tensor] = None) -> Neighbors:
    """neighbors.py:187-212 (batches with or without PBC).  Same pair set as the
    reference's O(N^2) enumeration as long as the periodic cell is at least one cutoff wide."""
    _validate_inputs(cutoff, species, coords, cell, pbc, supports_batches=True)
    return _half_list(cutoff, species, coords, cell, pbc)


class Neighborlist(torch.nn.Module):
    r"""Base class for modules that compute pairs of neighbors (neighbors.py:140-166)."""

    def forward(self, cutoff: float, species: Tensor, coords: Tensor, cell: tp.Optional[Tensor] = None,
                pbc: tp.Optional[Tensor] = None) -> Neighbors:
        raise NotImplementedError("Must be implemented by subclasses")


class AllPairs(Neighborlist):
    def forward(self, cutoff, species, coords, cell=None, pbc=None) -> Neighbors:
        return all_pairs(cutoff, species, coords, cell, pbc)


class CellList(Neighborlist):
    def forward(self, cutoff, species, coords, cell=None, pbc=None) -> Neighbors:
        return cell_list(cutoff, species, coords, cell, pbc)


class AdaptiveList(Neighborlist):
    """neighbors.py:317-363: the reference switches algorithm by size; the bucket grid adapts by
    itself (one bucket for small systems), so this is the same kernel."""

    def __init__(self, threshold: int = 190, threshold_nopbc: int = 1770) -> None:
        super().__init__()
        self._thresh, self._thresh_nopbc = threshold, threshold_nopbc

    def forward(self, cutoff, species, coords, cell=None, pbc=None) -> Neighbors:
        _validate_inputs(cutoff, species, coords, cell, pbc, supports_batches=False)
        return _half_list(cutoff, species, coords, cell, pbc)


class VerletCellList(CellList):
    r"""Cell list with a Verlet skin (neighbors.py:759-884): the pairs within ``cutoff + skin`` are
    cached together with their lattice shifts and only re-screened with the true cutoff and the
    current coordinates, until an atom has moved ``skin / 2`` or the cell changes.  (The fused engine
    caches the bucket grid instead of a pair list: ``calculator.HostCalculator(skin=...)``.)"""

    def __init__(self, skin: float = 1.0):
        super().__init__()
        if skin <= 0.0:
            raise ValueError("skin must be a positive float")
        self.skin = skin
        self.reset_cached_values()

    def reset_cached_values(self) -> None:
        self._prev_idx: tp.Optional[Tensor] = None       # (2, P) pairs within cutoff + skin
        self._prev_shift: tp.Optional[Tensor] = None     # (P, 3) lattice shift of every cached pair
        self._prev_coords: tp.Optional[Tensor] = None
        self._prev_cell: tp.Optional[Tensor] = None
        self._prev_cutoff = 0.0
        self.rebuilds = 0

    def _can_use_prev_list(self, cutoff: float, coords: Tensor, cell: tp.Optional[Tensor]) -> bool:
        if self._prev_idx is None or self._prev_coords is None or self._prev_coords.shape != coords.shape:
            return False
        if cutoff > self._prev_cutoff or (cell is None) != (self._prev_cell is None):
            return False
        if cell is not None and not torch.equal(cell.detach(), self._prev_cell):
            return False
        moved2 = (coords.detach() - self._prev_coords).pow(2).sum(-1)
        return bool((moved2 < (self.skin / 2) ** 2).all())

    def forward(self, cutoff, species, coords, cell=None, pbc=None) -> Neighbors:
        _validate_inputs(cutoff, species, coords, cell, pbc, supports_batches=False)
        flat = coords.reshape(-1, 3)
        if not self._can_use_prev_list(cutoff, coords, cell):
            wide = _half_list(cutoff + self.skin, species, coords.detach(), cell, pbc)
            i0, i1 = wide.indices[0], wide.indices[1]
            # diff = x[i0] - x[i1] + shift (neighbors.py:107-111): the shift is what stays constant
            self._prev_shift = wide.diff_vectors - (flat.detach().index_select(0, i0) - flat.detach().index_select(0, i1))
            self._prev_idx = wide.indices
            self._prev_coords = coords.detach().clone()
            self._prev_cell = None if cell is None else cell.detach().clone()
            self._prev_cutoff = float(cutoff)
            self.rebuilds += 1
        idx, shift = self._prev_idx, self._prev_shift
        diff = flat.index_select(0, idx[0]) - flat.index_select(0, idx[1]) + shift
        dist = diff.norm(2, -1)
        keep = (dist.detach() <= cutoff).nonzero().flatten()      # narrow_down (neighbors.py:64-113)
        return Neighbors(idx.index_select(1, keep), dist.index_select(0, keep), diff.index_select(0, keep))


NeighborlistArg = tp.Union[str, Neighborlist]


def _parse_neighborlist(neighborlist: NeighborlistArg = "cell_list") -> Neighborlist:
    # neighbors.py:899-914
    if isinstance(neighborlist, Neighborlist):
        return neighborlist
    table = {"all_pairs": AllPairs, "cell_list": CellList, "adaptive": AdaptiveList,
             "fast_cell_list": CellList, "verlet_cell_list": VerletCellList, "base": Neighborlist}
    if neighborlist not in table:
        raise ValueError(f"Unsupported neighborlist: {neighborlist}")
    return table[neighborlist]()
