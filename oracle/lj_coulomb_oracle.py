"""TEST INFRASTRUCTURE ONLY -- float64 restatement of the reference's Lennard-Jones and fixed-charge Coulomb pair
potentials, beside ``pair_oracle``.

``LennardJones`` / ``RepulsionLJ`` / ``DispersionLJ`` (potentials/lj.py:60-145) and ``FixedCoulomb`` / ``FixedMNOK``
(potentials/fixed_coulomb.py:13-81) on top of ``BasePairPotential`` (potentials/core.py:106-207), in plain torch:
the same atomic split, ghost weight, envelope and "scaling" stress as ``pair_oracle``.  Without a cutoff (the
reference's default, no envelope) the neighbour list is every pair of an open system.  ``make_lj_coulomb_golden.py``
pins it to the reference before any fixture is written.  The per-element parameters are inputs (tests take them from
the golden fixture).
"""
from __future__ import annotations

import math
import typing as tp

import torch
from torch import Tensor

from . import ani_oracle as orc

ANGSTROM_TO_BOHR = 1.8897261258369282   # units.py:41
KINDS = ("lj", "rep_lj", "disp_lj", "coulomb", "mnok")
# the names of the reference's classes, and of this project's
CLASSES = {"lj": "LennardJones", "rep_lj": "RepulsionLJ", "disp_lj": "DispersionLJ", "coulomb": "FixedCoulomb",
           "mnok": "FixedMNOK"}
# an open system's "every pair" list: a finite stand-in for the infinite cutoff of the neighbour lists
_ALL = 1e4


class Spec(tp.NamedTuple):
    kind: str                 # one of KINDS
    cutoff: float             # math.inf: no envelope, every pair (open systems)
    cutoff_fn: str            # "cosine" | "smooth" | "dummy"
    eps: Tensor               # (S,) Hartree                 (LJ kinds)
    sigma: Tensor             # (S,) Angstrom                (LJ kinds)
    charges: Tensor           # (S,) e                       (Coulomb kinds)
    eta: Tensor               # (S,)                         (FixedMNOK)
    dielectric: float = 1.0   # FixedCoulomb only: the reference's FixedMNOK does not divide by it


def pair_energies(spec: Spec, species: Tensor, nb: orc.Neighbors, ghost_flags: tp.Optional[Tensor] = None) -> Tensor:
    """Energy of every pair of the half list, envelope and ghost weight included (potentials/core.py:155-178)."""
    r = nb.distances
    s12 = species.reshape(-1)[nb.indices]
    if spec.kind in ("lj", "rep_lj", "disp_lj"):
        eps = spec.eps.to(r.dtype)
        sigma = spec.sigma.to(r.dtype)
        e_ab = torch.sqrt(eps[s12[0]] * eps[s12[1]])                        # lj.py:104-106, Berthelot
        s_ab = (sigma[s12[0]] + sigma[s12[1]]) / 2                          # lj.py:108-110, Lorentz
        x = s_ab / r.clamp(min=1e-7)                                        # lj.py:123, 133, 143
        e = {"lj": 4 * e_ab * (x ** 12 - x ** 6), "rep_lj": 4 * e_ab * x ** 12, "disp_lj": -4 * e_ab * x ** 6}[spec.kind]
    else:
        q = spec.charges.to(r.dtype)
        qq = q[s12[0]] * q[s12[1]]
        if spec.kind == "coulomb":
            e = qq / spec.dielectric / (r.clamp(min=1e-7) * ANGSTROM_TO_BOHR)   # fixed_coulomb.py:28-38
        else:
            eta = spec.eta.to(r.dtype)
            inv_eta = 2 / (eta[s12[0]] + eta[s12[1]])                       # fixed_coulomb.py:69-70
            d = r * ANGSTROM_TO_BOHR
            e = qq / (d ** 2 + inv_eta ** 2).sqrt()                         # fixed_coulomb.py:72-81
    if spec.cutoff_fn != "dummy":
        e = e * orc._cutoff(spec.cutoff_fn)(r, spec.cutoff)                # core.py:168
    if ghost_flags is not None:
        g12 = ghost_flags.reshape(-1)[nb.indices]
        e = torch.where(g12[0] | g12[1], e * 0.5, e)                       # core.py:170-177
    return e


def energies_from_neighbors(spec: Spec, species: Tensor, nb: orc.Neighbors, atomic: bool = False,
                            ghost_flags: tp.Optional[Tensor] = None) -> Tensor:
    """potentials/core.py:181-207: (C,) energies, or (C, A) with every pair split between its two atoms."""
    e = pair_energies(spec, species, nb, ghost_flags)
    C, A = species.shape
    if atomic:
        out = e.new_zeros(C * A)
        out = out.index_add(0, nb.indices[0], e / 2).index_add(0, nb.indices[1], e / 2)
        return out.view(C, A)
    return e.new_zeros(C).index_add(0, torch.div(nb.indices[0], A, rounding_mode="floor"), e)


def compute(spec: Spec, species: Tensor, coords: Tensor, cell: tp.Optional[Tensor] = None,
            pbc: tp.Optional[Tensor] = None, neighborlist: str = "all_pairs", stress: bool = False
            ) -> tp.Dict[str, Tensor]:
    """energy (C,), atomic (C, A), forces (C, A, 3) and, with ``stress``, dE/d(scaling) / volume (Hartree / A^3)."""
    if spec.cutoff == math.inf:
        assert pbc is None, "PBC can't use an infinite cutoff"
        neighborlist, search = "all_pairs", _ALL
    else:
        search = spec.cutoff
    coords_in = coords.detach().clone().requires_grad_(True)
    x, scaling = coords_in, None
    if stress:
        assert cell is not None and pbc is not None
        scaling = torch.eye(3, dtype=coords.dtype, requires_grad=True)
        x, cell = x @ scaling, cell @ scaling
    nb = orc.neighborlist(neighborlist, search, species, x, cell, pbc)
    atomic = energies_from_neighbors(spec, species, nb, atomic=True)
    energy = atomic.sum(-1)
    out = {"energy": energy.detach(), "atomic": atomic.detach(),
           "forces": -torch.autograd.grad(energy.sum(), coords_in, retain_graph=stress)[0]}
    if stress:
        out["stress"] = (torch.autograd.grad(energy.sum(), scaling)[0] / torch.det(cell.detach()).abs()).detach()
    return out


def spec_from_params(kind: str, cutoff: float, cutoff_fn: str, params) -> Spec:
    """A Spec from the parameter arrays of tests/golden/ljc_params.npz."""
    t = {k: torch.as_tensor(params[k], dtype=torch.float64) for k in ("eps", "sigma", "charges", "eta")}
    return Spec(kind, cutoff, cutoff_fn, t["eps"], t["sigma"], t["charges"], t["eta"], float(params["dielectric"]))
