"""TEST INFRASTRUCTURE ONLY -- float64 restatement of the reference's D3(BJ) two-body dispersion, beside ``pair_oracle``.

``TwoBodyDispersionD3`` (potentials/dftd3.py:113-311) over the pair-potential wrapper of potentials/core.py:155-207, in
plain torch: coordination numbers, the C6 interpolation with its eps = 1e-35, the Becke-Johnson damping, the envelope,
the atomic split and the ghost weight; forces by autograd (so the coordination-number chain is included), and the
"scaling" stress of ase.py:110-121,170-173.  ``make_d3_golden.py`` pins it to the reference before any fixture is
written.  The reference's buffers are inputs (tests take them from ``tests/golden/d3_params.npz``).
"""
from __future__ import annotations

import math
import typing as tp

import torch
from torch import Tensor

from . import ani_oracle as orc

ANGSTROM_TO_BOHR = 1.8897261258369282   # units.py:41
K1, K2, K3 = 16.0, 4.0 / 3.0, 4.0       # dftd3.py:171-174
EPS = 1e-35                             # dftd3.py:177


class D3Spec(tp.NamedTuple):
    cutoff: float
    cutoff_fn: str                # "cosine" | "smooth"
    s6: float
    s8: float
    a1: float
    a2: float
    cutoff_radii: Tensor          # (S, S) Bohr, _damp_fn.cutoff_radii
    sqrt_charge_ab: Tensor        # (S, S)
    covalent_radii: Tensor        # (S,) Bohr
    coeff6: Tensor                # (S, S, 5, 5) precalc_coeff6
    coordnums_a: Tensor           # (S, S, 5, 5)
    coordnums_b: Tensor           # (S, S, 5, 5)


def spec_from_npz(z, cutoff: float, cutoff_fn: str) -> D3Spec:
    t = {k: torch.tensor(z[k], dtype=torch.float64) for k in
         ("cutoff_radii", "sqrt_charge_ab", "covalent_radii", "precalc_coeff6", "precalc_coordnums_a",
          "precalc_coordnums_b")}
    return D3Spec(cutoff, cutoff_fn, float(z["s6"]), float(z["s8"]), float(z["a1"]), float(z["a2"]),
                  t["cutoff_radii"], t["sqrt_charge_ab"], t["covalent_radii"], t["precalc_coeff6"],
                  t["precalc_coordnums_a"], t["precalc_coordnums_b"])


def coordnums(spec: D3Spec, species: Tensor, nb: orc.Neighbors) -> Tensor:
    """dftd3.py:251-272: every listed pair counts for both of its atoms, no envelope."""
    d = nb.distances * ANGSTROM_TO_BOHR
    s12 = species.reshape(-1)[nb.indices]
    rc = spec.covalent_radii[s12[0]] + spec.covalent_radii[s12[1]]
    count = 1 / (1 + torch.exp(-K1 * (K2 * rc / d - 1)))
    cn = d.new_zeros(species.numel())
    return cn.index_add(0, nb.indices[0], count).index_add(0, nb.indices[1], count)


def coeff6(spec: D3Spec, species: Tensor, cn: Tensor, nb: orc.Neighbors) -> Tensor:
    """dftd3.py:274-311."""
    s12 = species.reshape(-1)[nb.indices]
    c6 = spec.coeff6[s12[0], s12[1]].flatten(1, 2)
    cna = spec.coordnums_a[s12[0], s12[1]].flatten(1, 2)
    cnb = spec.coordnums_b[s12[0], s12[1]].flatten(1, 2)
    g = (cn[nb.indices[0]].view(-1, 1) - cna) ** 2 + (cn[nb.indices[1]].view(-1, 1) - cnb) ** 2
    L = torch.exp(-K3 * g).masked_fill(c6 <= 0.0, 0.0)
    return ((c6 * L).sum(-1) + EPS) / (L.sum(-1) + EPS)


def pair_energies(spec: D3Spec, species: Tensor, nb: orc.Neighbors, ghost_flags: tp.Optional[Tensor] = None,
                  chain: bool = True) -> Tensor:
    """Energy of every pair of the half list, envelope and ghost weight included (dftd3.py:221-246,
    potentials/core.py:155-178).  ``chain=False`` detaches the coordination numbers: the forces then miss the
    coordination-number chain (a check that the tests can tell the difference)."""
    cn = coordnums(spec, species, nb)
    if not chain:
        cn = cn.detach()
    d = nb.distances * ANGSTROM_TO_BOHR
    s12 = species.reshape(-1)[nb.indices]
    c6 = coeff6(spec, species, cn, nb)
    c8 = 3 * c6 * spec.sqrt_charge_ab[s12[0], s12[1]]
    damp = spec.a1 * spec.cutoff_radii[s12[0], s12[1]] + spec.a2
    e = -(spec.s6 * c6 / (d ** 6 + damp ** 6) + spec.s8 * c8 / (d ** 8 + damp ** 8))
    e = e * orc._cutoff(spec.cutoff_fn)(nb.distances, spec.cutoff)
    if ghost_flags is not None:
        g12 = ghost_flags.reshape(-1)[nb.indices]
        e = torch.where(g12[0] | g12[1], e * 0.5, e)
    return e


def energies_from_neighbors(spec: D3Spec, species: Tensor, nb: orc.Neighbors, atomic: bool = False,
                            ghost_flags: tp.Optional[Tensor] = None, chain: bool = True) -> Tensor:
    """potentials/core.py:181-207: (C,) energies, or (C, A) with every pair split between its two atoms."""
    e = pair_energies(spec, species, nb, ghost_flags, chain)
    C, A = species.shape
    if atomic:
        out = e.new_zeros(C * A)
        out = out.index_add(0, nb.indices[0], e / 2).index_add(0, nb.indices[1], e / 2)
        return out.view(C, A)
    return e.new_zeros(C).index_add(0, torch.div(nb.indices[0], A, rounding_mode="floor"), e)


def compute(spec: D3Spec, species: Tensor, coords: Tensor, cell: tp.Optional[Tensor] = None,
            pbc: tp.Optional[Tensor] = None, neighborlist: str = "all_pairs", stress: bool = False,
            chain: bool = True) -> tp.Dict[str, Tensor]:
    """energy (C,), atomic (C, A), forces (C, A, 3) and, with ``stress``, dE/d(scaling) / volume (Hartree / A^3)."""
    assert spec.cutoff != math.inf, "the neighbour lists of the oracle need a finite cutoff"
    coords_in = coords.detach().clone().requires_grad_(True)
    x, scaling = coords_in, None
    if stress:
        assert cell is not None and pbc is not None
        scaling = torch.eye(3, dtype=coords.dtype, requires_grad=True)
        x, cell = x @ scaling, cell @ scaling
    nb = orc.neighborlist(neighborlist, spec.cutoff, species, x, cell, pbc)
    atomic = energies_from_neighbors(spec, species, nb, atomic=True, chain=chain)
    energy = atomic.sum(-1)
    out = {"energy": energy.detach(), "atomic": atomic.detach(),
           "forces": -torch.autograd.grad(energy.sum(), coords_in, retain_graph=stress)[0]}
    if stress:
        out["stress"] = (torch.autograd.grad(energy.sum(), scaling)[0] / torch.det(cell.detach()).abs()).detach()
    return out
