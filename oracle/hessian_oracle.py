"""TEST INFRASTRUCTURE ONLY -- float64 Hessians of the oracle models by double backward, and a float64 restatement of
the harmonic vibrational analysis.

The energy is that of ``ani_oracle`` (CELU networks) or ``gelu_oracle`` (GELU bias-free networks) plus any
``pair_oracle`` terms (xTB, ZBL) over an all-pairs neighbour list of open systems; self energies are constant and do
not enter.  ``hessian`` differentiates the forces once per component, as ``torchani.grad.hessians`` does; ``hvp``
gives Hessian-vector products for systems too large for a dense float64 Hessian on the CPU.
``make_hessian_golden.py`` pins these to the reference's ``torchani.grad`` before any fixture is written.
"""
from __future__ import annotations

import math
import typing as tp

import numpy as np
import torch
from torch import Tensor

from . import ani_oracle as orc
from . import gelu_oracle as gor
from . import pair_oracle as porc

# CODATA 2014 (the reference's units.py values): sqrt(Hartree / (AMU A^2)) -> cm^-1 and meV, Hartree / A^2 -> mDyne / A
_HARTREE_J = 27.211386024367243 * 1.6021766208e-19
SQRT_MHESSIAN_TO_INVCM = math.sqrt(_HARTREE_J / 1.660539040e-27) / 1e-10 / 299792458.0 / 100.0
SQRT_MHESSIAN_TO_MILLIEV = SQRT_MHESSIAN_TO_INVCM * 0.0001239841973964072 * 1000.0
MHESSIAN_TO_FCONST = _HARTREE_J * 1e8 / 1e-10


def energy_fn(model: orc.Model, species: Tensor, networks: str = "celu", pairs: tp.Sequence[porc.PairSpec] = (),
              members: tp.Optional[tp.List[int]] = None) -> tp.Callable[[Tensor], Tensor]:
    """coords (C, A, 3) -> (C,) energies without the self energies (ensemble mean of ``members``, all by default)."""
    ens = orc.ensemble_atomic_energies if networks == "celu" else gor.ensemble_atomic_energies

    def energy(coords: Tensor) -> Tensor:
        nb = orc.neighborlist("all_pairs", model.spec.rcr, species, coords)
        aev = orc.aev_from_neighbors(model.spec, species, nb)
        e = ens(model.symbols, model.weights, species, aev, members).mean(0).sum(-1)
        for p in pairs:
            nbp = orc.neighborlist("all_pairs", p.cutoff, species, coords)
            e = e + porc.energies_from_neighbors(p, species, nbp)
        return e
    return energy


def center_aev(spec: orc.AEVSpec, s_center: int, s_nbrs: tp.Sequence[int], vectors: Tensor) -> Tensor:
    """The AEV (out_dim,) of one central atom of element ``s_center`` as a function of its neighbour vectors ``vectors``
    (n, 3) = r_n - r_i (elements ``s_nbrs``), in the column order of ``aev_from_neighbors``: radial terms of the
    neighbours within Rcr, angular terms of every pair of neighbours within Rca (both inclusive, the cosine's
    denominator clamped at 1e-10).  Every neighbour and pair is summed in the order given, so the per-stage references
    are ``torch.func`` derivatives of this function with respect to ``vectors``.  ``s_center`` does not enter (an AEV
    row holds the neighbours' elements only); it is kept for the symmetry of the call with ``center_pair_energy``."""
    S = spec.num_species
    sp = torch.as_tensor(list(s_nbrs), dtype=torch.long).view(-1)
    d = vectors.norm(dim=-1)
    nr = len(spec.shf_r)
    radial = vectors.new_zeros(S, nr)
    r_in = d.detach() <= spec.rcr
    if bool(r_in.any()):
        radial = radial.index_add(0, sp[r_in], orc.radial_terms(spec, d[r_in]))
    npairs = S * (S + 1) // 2
    angular = vectors.new_zeros(npairs, spec.angular_sub)
    close = torch.nonzero(d.detach() <= spec.rca).view(-1)
    if close.numel() >= 2:
        ja, jb = torch.triu_indices(close.numel(), close.numel(), 1)
        a, b = close[ja], close[jb]
        terms = orc.angular_terms(spec, d[a], d[b], vectors[a], vectors[b])
        angular = angular.index_add(0, orc.triu_index(S)[sp[a], sp[b]], terms)
    return torch.cat([radial.reshape(-1), angular.reshape(-1)])


def center_pair_energy(pair: porc.PairSpec, s_center: int, s_nbrs: tp.Sequence[int], vectors: Tensor) -> Tensor:
    """Half of the pair energy E(R) fc(R) of one central atom (element ``s_center``) with each of its neighbours
    (``vectors`` (n, 3) = r_n - r_i, elements ``s_nbrs``) within the term's cutoff (inclusive): the atomic split of a
    full neighbour list, a scalar.  Summed over every atom of a system it is ``pair_oracle.energies_from_neighbors``."""
    n = vectors.shape[0]
    species = torch.tensor([[int(s_center)] + [int(s) for s in s_nbrs]], dtype=torch.long)
    d = vectors.norm(dim=-1)
    keep = d.detach() <= pair.cutoff
    idx = torch.stack([torch.zeros(n, dtype=torch.long), torch.arange(1, n + 1)])[:, keep]
    nb = orc.Neighbors(idx, d[keep], vectors[keep])
    return 0.5 * porc.pair_energies(pair, species, nb).sum()


def hessian(energy: tp.Callable[[Tensor], Tensor], coords: Tensor) -> Tensor:
    """(C, 3A, 3A) d^2E/dx^2 in the dtype of ``coords`` (conformers are independent: one backward per component)."""
    x = coords.detach().clone().requires_grad_(True)
    (g,) = torch.autograd.grad(energy(x).sum(), x, create_graph=True)
    C, A, _ = x.shape
    flat = g.reshape(C, 3 * A)
    rows = []
    for k in range(3 * A):
        (r,) = torch.autograd.grad(flat[:, k].sum(), x, retain_graph=True, allow_unused=True)
        rows.append(torch.zeros_like(x).reshape(C, 1, -1) if r is None else r.reshape(C, 1, -1))
    return torch.cat(rows, 1).detach()


def hvp(energy: tp.Callable[[Tensor], Tensor], coords: Tensor, vectors: Tensor) -> Tensor:
    """H v for each of ``vectors`` (K, C, A, 3) -> (K, C, A, 3)."""
    x = coords.detach().clone().requires_grad_(True)
    (g,) = torch.autograd.grad(energy(x).sum(), x, create_graph=True)
    out = [torch.autograd.grad((g * v).sum(), x, retain_graph=True)[0] for v in vectors]
    return torch.stack(out).detach()


def vibrational_analysis(masses: np.ndarray, hess: np.ndarray, mode_kind: str = "mdu", unit: str = "cm^-1"
                         ) -> tp.Dict[str, np.ndarray]:
    """One molecule (masses (A,) AMU, hess (3A, 3A) Hartree / A^2), float64 numpy: frequencies, modes (3A, A, 3),
    force constants (mDyne / A), reduced masses (AMU), modes of kind "mdu" / "mdn" / "mwn"."""
    w = np.repeat(1.0 / np.sqrt(np.asarray(masses, dtype=np.float64)), 3)
    lam, vec = np.linalg.eigh(hess * w[:, None] * w[None, :])
    mwn = vec.T
    mdu = mwn * w[None, :]
    red = 1.0 / np.sum(mdu * mdu, axis=1)
    modes = {"mdu": mdu, "mdn": mdu * np.sqrt(red)[:, None], "mwn": mwn}[mode_kind]
    conv = SQRT_MHESSIAN_TO_INVCM if unit == "cm^-1" else SQRT_MHESSIAN_TO_MILLIEV
    return {"freqs": np.sign(lam) * np.sqrt(np.abs(lam)) / (2 * math.pi) * conv,
            "modes": modes.reshape(len(lam), -1, 3), "fconstants": lam * MHESSIAN_TO_FCONST * red, "rmasses": red}
