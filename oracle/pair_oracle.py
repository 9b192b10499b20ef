"""TEST INFRASTRUCTURE ONLY -- float64 restatement of the reference's pair potentials, beside ``ani_oracle``.

``BasePairPotential`` (potentials/core.py:106-207) + the two repulsion forms (potentials/xtb.py:57-77,
potentials/zbl.py:68-81) in plain torch, with autograd forces, the atomic split, the ghost weight and the "scaling"
stress of ase.py:110-121,170-173.  ``make_pair_golden.py`` pins it to the reference before any fixture is written.
The per-element-pair parameter tensors are inputs (tests take them from the golden fixture).
"""
from __future__ import annotations

import math
import typing as tp

import torch
from torch import Tensor

from . import ani_oracle as orc

ANGSTROM_TO_BOHR = 1.8897261258369282   # units.py:41
ZBL_COEFFS = (0.18175, 0.50986, 0.28022, 0.02817)      # potentials/zbl.py:45-50 (universal screening function)
ZBL_EXPONENTS = (3.19980, 0.94229, 0.40290, 0.20162)


class PairSpec(tp.NamedTuple):
    kind: str                 # "xtb" | "zbl"
    cutoff: float
    cutoff_fn: str            # "cosine" | "smooth" | "dummy" (no envelope, cutoff = inf)
    # xtb: y_ab, sqrt_alpha_ab, k_rep_ab (S, S); zbl: eff_z (S,), then k, eff_exponent, coeffs, exponents
    tables: tp.Tuple[Tensor, ...]
    k: float = 0.8853
    eff_exponent: float = 0.23
    coeffs: tp.Tuple[float, ...] = ZBL_COEFFS
    exponents: tp.Tuple[float, ...] = ZBL_EXPONENTS


def zbl_spec(symbols: tp.Sequence[str], cutoff: float, cutoff_fn: str) -> PairSpec:
    z = torch.tensor([float(orc.ATOMIC_NUMBERS[s]) for s in symbols], dtype=torch.float64)
    return PairSpec("zbl", cutoff, cutoff_fn, (z,))


def pair_energies(spec: PairSpec, species: Tensor, nb: orc.Neighbors,
                  ghost_flags: tp.Optional[Tensor] = None) -> Tensor:
    """Energy of every pair of the half list, envelope and ghost weight included (potentials/core.py:155-178)."""
    d = nb.distances.clamp(min=1e-7) * ANGSTROM_TO_BOHR                    # core.py:137-139, xtb.py:64
    s12 = species.reshape(-1)[nb.indices]
    if spec.kind == "xtb":
        y, sa, k = (t.to(d.dtype)[s12[0], s12[1]] for t in spec.tables)
        e = (y / d) * torch.exp(-sa * d ** k)                              # xtb.py:77
    else:
        z = spec.tables[0].to(d.dtype)
        za, zb = z[s12[0]], z[s12[1]]
        red = d * (za ** spec.eff_exponent + zb ** spec.eff_exponent) / spec.k   # zbl.py:76
        # the reference keeps the screening constants as float32 buffers (zbl.py:59-64)
        c = torch.tensor(spec.coeffs, dtype=torch.float32).to(d.dtype).view(1, -1)
        x = torch.tensor(spec.exponents, dtype=torch.float32).to(d.dtype).view(1, -1)
        e = za * zb / d * (c * torch.exp(-x * red.view(-1, 1))).sum(-1)           # zbl.py:75-81
    if spec.cutoff_fn != "dummy":
        e = e * orc._cutoff(spec.cutoff_fn)(nb.distances, spec.cutoff)      # core.py:168
    if ghost_flags is not None:
        g12 = ghost_flags.reshape(-1)[nb.indices]
        e = torch.where(g12[0] | g12[1], e * 0.5, e)                       # core.py:170-177
    return e


def energies_from_neighbors(spec: PairSpec, species: Tensor, nb: orc.Neighbors, atomic: bool = False,
                            ghost_flags: tp.Optional[Tensor] = None) -> Tensor:
    """potentials/core.py:181-207: (C,) energies, or (C, A) with every pair split between its two atoms."""
    e = pair_energies(spec, species, nb, ghost_flags)
    C, A = species.shape
    if atomic:
        out = e.new_zeros(C * A)
        out = out.index_add(0, nb.indices[0], e / 2).index_add(0, nb.indices[1], e / 2)
        return out.view(C, A)
    return e.new_zeros(C).index_add(0, torch.div(nb.indices[0], A, rounding_mode="floor"), e)


def compute(spec: PairSpec, species: Tensor, coords: Tensor, cell: tp.Optional[Tensor] = None,
            pbc: tp.Optional[Tensor] = None, neighborlist: str = "all_pairs", stress: bool = False
            ) -> tp.Dict[str, Tensor]:
    """energy (C,), atomic (C, A), forces (C, A, 3) and, with ``stress``, dE/d(scaling) / volume (Hartree / A^3)."""
    assert spec.cutoff != math.inf, "the neighbour lists of the oracle need a finite cutoff"
    coords_in = coords.detach().clone().requires_grad_(True)
    x, scaling = coords_in, None
    if stress:
        assert cell is not None and pbc is not None
        scaling = torch.eye(3, dtype=coords.dtype, requires_grad=True)
        x, cell = x @ scaling, cell @ scaling
    nb = orc.neighborlist(neighborlist, spec.cutoff, species, x, cell, pbc)
    atomic = energies_from_neighbors(spec, species, nb, atomic=True)
    energy = atomic.sum(-1)
    out = {"energy": energy.detach(), "atomic": atomic.detach(),
           "forces": -torch.autograd.grad(energy.sum(), coords_in, retain_graph=stress)[0]}
    if stress:
        out["stress"] = (torch.autograd.grad(energy.sum(), scaling)[0] / torch.det(cell.detach()).abs()).detach()
    return out
