"""Forces, Hessians and harmonic vibrational analysis through ``torch.autograd``, with the signatures, mode kinds and
units of ``torchani.grad``.

A model from ``torchani_b200.models`` returns energies whose gradient is produced by the fused step; when that
gradient is taken with ``create_graph=True`` the step's analytic Hessian (``Engine.hessian``, csrc/hessian.cu) is
computed once and the second backward is the product with it, so ``hessians`` costs one Hessian per forward however
many components it differentiates.  ``models.ANI.energies_forces_hessians`` gives the same three results without the
autograd round trip.

Units: energies in Hartree, lengths in Angstrom, masses in AMU (given by the caller: no mass table is shipped).
Frequencies come out in cm^-1 or meV, force constants in mDyne/Angstrom, reduced masses in AMU; imaginary frequencies
are returned as negative numbers.
"""
from __future__ import annotations

import math
import typing as tp

import torch
from torch import Tensor

__all__ = ["forces", "hessians", "forces_and_hessians", "energies_and_forces", "energies_forces_and_hessians",
           "vibrational_analysis", "VibAnalysis", "EnergiesForces", "EnergiesForcesHessians",
           "ForcesHessians"]

# ---- unit constants from the CODATA 2014 recommended values (the values ASE uses) ----
_C = 299792458.0                      # speed of light, m / s (exact)
_MU0 = 4e-7 * math.pi                 # vacuum permeability, N / A^2 (exact in CODATA 2014)
_EPS0 = 1.0 / (_MU0 * _C * _C)        # vacuum permittivity, F / m
_H = 6.626070040e-34                  # Planck constant, J s
_HBAR = _H / (2.0 * math.pi)
_ME = 9.10938356e-31                  # electron mass, kg
_E = 1.6021766208e-19                 # elementary charge, C
_AMU = 1.660539040e-27                # atomic mass unit, kg
HARTREE_TO_EV = _ME * _E ** 3 / (16.0 * math.pi ** 2 * _EPS0 ** 2 * _HBAR ** 2)
HARTREE_TO_JOULE = HARTREE_TO_EV * _E
INVCM_TO_EV = 100.0 * _C * _H / _E    # photon energy of 1 cm^-1
# sqrt(Hartree / (AMU A^2)) -> s^-1 (sqrt(J / kg) / m) -> wavenumber in cm^-1 (/ c, / 100)
SQRT_MHESSIAN_TO_INVCM = math.sqrt(HARTREE_TO_JOULE / _AMU) / 1e-10 / _C / 100.0
SQRT_MHESSIAN_TO_MILLIEV = SQRT_MHESSIAN_TO_INVCM * INVCM_TO_EV * 1000.0
# Hartree / A^2 -> N / m -> mDyne / A (1 N = 1e8 mDyne, 1 m = 1e10 A)
MHESSIAN_TO_FCONST = HARTREE_TO_JOULE * 1e8 / 1e-10
# 1 bar = 1e5 Pa = 1e5 J / m^3 in Hartree / A^3 (1 m^3 = 1e30 A^3)
BAR_TO_HARTREE_A3 = 1e5 / HARTREE_TO_JOULE / 1e30


class EnergiesForces(tp.NamedTuple):
    energies: Tensor
    forces: Tensor


class ForcesHessians(tp.NamedTuple):
    forces: Tensor
    hessians: Tensor


class EnergiesForcesHessians(tp.NamedTuple):
    energies: Tensor
    forces: Tensor
    hessians: Tensor


class VibAnalysis(tp.NamedTuple):
    """Frequencies (3A,), normal modes (3A, A, 3), force constants (3A,) and reduced masses (3A,), ascending in the
    eigenvalues of the mass-weighted Hessian."""
    freqs: Tensor
    modes: Tensor
    fconstants: Tensor
    rmasses: Tensor


def _leaf_requiring_grad(coordinates: Tensor, fn: str) -> None:
    if not coordinates.requires_grad:
        raise ValueError(f"'coordinates' passed to {fn} must require grad")
    if not coordinates.is_leaf:
        raise ValueError(f"'coordinates' passed to {fn} must be a leaf tensor (not the result of an operation)")


def forces(energies: Tensor, coordinates: Tensor, retain_graph: tp.Optional[bool] = None,
           create_graph: bool = False) -> Tensor:
    """-dE/dx of the summed energies with respect to the leaf ``coordinates``."""
    _leaf_requiring_grad(coordinates, "forces")
    (g,) = torch.autograd.grad([energies.sum()], [coordinates], retain_graph=retain_graph, create_graph=create_graph)
    return -g


def hessians(forces: Tensor, coordinates: Tensor, retain_graph: tp.Optional[bool] = None) -> Tensor:
    """(C, 3A, 3A) d^2E/dx^2 from ``forces`` that were computed with ``create_graph=True``: one backward per force
    component, each giving one row of every conformer's Hessian."""
    _leaf_requiring_grad(coordinates, "hessians")
    n_conf, n_atoms, _ = forces.shape
    flat = forces.reshape(n_conf, 3 * n_atoms)
    rows = []
    for k in range(3 * n_atoms):
        keep = True if k < 3 * n_atoms - 1 else retain_graph
        (g,) = torch.autograd.grad([flat[:, k].sum()], [coordinates], retain_graph=keep)
        rows.append(g.reshape(n_conf, 1, 3 * n_atoms))
    return -torch.cat(rows, dim=1)


def forces_and_hessians(energies: Tensor, coordinates: Tensor,
                        retain_graph: tp.Optional[bool] = None) -> ForcesHessians:
    f = forces(energies, coordinates, retain_graph=True, create_graph=True)
    return ForcesHessians(f, hessians(f, coordinates, retain_graph=retain_graph))


def energies_and_forces(model, species: Tensor, coordinates: Tensor, cell: tp.Optional[Tensor] = None,
                        pbc: tp.Optional[Tensor] = None, retain_graph: tp.Optional[bool] = None,
                        create_graph: bool = False) -> EnergiesForces:
    """Energies of ``model((species, coordinates), cell, pbc)`` and their forces; ``coordinates`` must be a leaf (its
    ``requires_grad`` flag is restored afterwards)."""
    saved = coordinates.requires_grad
    coordinates.requires_grad_(True)
    try:
        if not coordinates.is_leaf:
            raise ValueError("'coordinates' must be a leaf tensor (not the result of an operation)")
        energies = model((species, coordinates), cell, pbc).energies
        f = forces(energies, coordinates, retain_graph=retain_graph, create_graph=create_graph)
    finally:
        coordinates.requires_grad_(saved)
    return EnergiesForces(energies, f)


def energies_forces_and_hessians(model, species: Tensor, coordinates: Tensor,
                                 retain_graph: bool = False) -> EnergiesForcesHessians:
    """Energies, forces and Hessians of an open system through autograd (one Hessian computation of the fused step for
    a ``torchani_b200.models`` model)."""
    saved = coordinates.requires_grad
    coordinates.requires_grad_(True)
    try:
        energies, f = energies_and_forces(model, species, coordinates, retain_graph=True, create_graph=True)
        h = hessians(f, coordinates, retain_graph=retain_graph)
    finally:
        coordinates.requires_grad_(saved)
    return EnergiesForcesHessians(energies, f, h)


ModeKind = tp.Literal["mdu", "mdn", "mwn"]
UnitKind = tp.Literal["cm^-1", "meV"]
_MODE_KINDS = {"mdu": "mdu", "mass-deweighted-unnormalized": "mdu", "mdn": "mdn",
               "mass-deweighted-normalized": "mdn", "mwn": "mwn", "mass-weighted-normalized": "mwn"}


def vibrational_analysis(masses: Tensor, hessian: Tensor, mode_kind: ModeKind = "mdu",
                         unit: UnitKind = "cm^-1") -> VibAnalysis:
    """Harmonic analysis of ONE molecule: ``masses`` (1, A) in AMU, ``hessian`` (1, 3A, 3A) in Hartree / A^2.

    The generalised problem H q = w^2 M q is solved as the eigenproblem of M^-1/2 H M^-1/2.  Its eigenvectors are the
    mass-weighted normalised modes ("mwn", orthonormal); M^-1/2 times them are the mass-deweighted modes, unnormalised
    ("mdu", as ASE) or normalised to unit length ("mdn", as Gaussian and ORCA).  The reduced mass of a mode is
    1 / |mdu mode|^2 and its force constant the eigenvalue times that reduced mass."""
    if unit == "cm^-1":
        to_unit = SQRT_MHESSIAN_TO_INVCM
    elif unit == "meV":
        to_unit = SQRT_MHESSIAN_TO_MILLIEV
    else:
        raise ValueError("unit must be 'cm^-1' or 'meV'")
    kind = _MODE_KINDS.get(mode_kind.lower())
    if kind is None:
        raise ValueError(f"Incorrect mode kind {mode_kind}: expected 'mdu', 'mdn' or 'mwn'")
    if hessian.dim() != 3 or hessian.shape[0] != 1 or masses.shape[0] != 1:
        raise ValueError("vibrational_analysis takes one molecule at a time: masses (1, A), hessian (1, 3A, 3A)")
    w = masses.to(hessian.dtype).rsqrt().repeat_interleave(3, dim=1)[0]          # (3A,) 1 / sqrt(m)
    mw_hessian = hessian[0] * w.view(-1, 1) * w.view(1, -1)
    eigenvalues, vectors = torch.linalg.eigh(mw_hessian)
    mwn = vectors.t()                                                            # one mode per row
    mdu = mwn * w.view(1, -1)
    inv_norm = 1.0 / torch.linalg.norm(mdu, dim=1)
    rmasses = inv_norm ** 2
    fconstants = eigenvalues * MHESSIAN_TO_FCONST * rmasses
    n = eigenvalues.numel()
    modes = {"mdu": mdu, "mdn": mdu * inv_norm.view(-1, 1), "mwn": mwn}[kind].reshape(n, -1, 3)
    freqs = torch.sign(eigenvalues) * eigenvalues.abs().sqrt() / (2.0 * math.pi) * to_unit
    return VibAnalysis(freqs, modes, fconstants, rmasses)
