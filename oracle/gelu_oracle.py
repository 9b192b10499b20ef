"""TEST INFRASTRUCTURE ONLY -- float64 restatement of the reference's GELU bias-free networks (ANI-2xr style).

The networks of ``torchani.arch.simple_ani`` and the ANI-2xr / ANI-2dr models (nn/_core.py:117-172,
``ANINetworks.default`` / ``like_dr``): ``torch.nn.GELU()`` (exact erf, approximate="none") after every hidden layer,
and no biases in any layer.  Everything else -- neighbour lists, AEV, self energies, forces and the "scaling" stress
-- is ``ani_oracle``'s; this module only replaces the networks, so ``compute`` returns what ``ani_oracle.compute``
returns for a model whose ``weights`` come from ``make_weights`` below.
"""
from __future__ import annotations

import math
import typing as tp

import numpy as np
import torch
from torch import Tensor

from oracle import ani_oracle as orc

SYMBOLS = ("H", "C", "N", "O", "F", "S", "Cl")   # the reference's SYMBOLS_2X_ZNUM_ORDER (simple_ani's element order)
RCR = 5.2                                        # simple_ani's radial cutoff (and the xTB repulsion's)


def gelu_spec(num_species: int = 7) -> orc.AEVSpec:
    """simple_ani's AEV (arch.py:1031-1047): cover_linearly radial 0.9-5.2 A x 16, angular 0.9-3.5 A x 8, 4 sections,
    smooth cutoff."""
    a0 = math.pi / 4 / 2
    return orc.AEVSpec(num_species, RCR, 3.5, 19.7, orc._linspace(0.9, RCR, 16), 12.5, 14.1,
                       orc._linspace(0.9, 3.5, 8), orc._linspace(a0, math.pi + a0, 4), "smooth")


def make_weights(symbols: tp.Sequence[str], dims: tp.Dict[str, tp.Tuple[int, ...]], in_dim: int, members: int,
                 seed: int = 1234, dtype: torch.dtype = torch.float32
                 ) -> tp.List[tp.Dict[str, tp.List[tp.Tuple[Tensor, None]]]]:
    """weights[member][symbol] = [(W [out,in], None) for each of the 4 Linear layers]: bias-free networks.  W is
    uniform in +-1/sqrt(fan_in), drawn from numpy's PCG64 stream (stable across numpy versions)."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(members):
        per_sym = {}
        for s in symbols:
            layer_dims = (in_dim,) + tuple(dims[s]) + (1,)
            per_sym[s] = [(torch.tensor(rng.uniform(-1.0 / math.sqrt(i), 1.0 / math.sqrt(i), size=(o, i)), dtype=dtype),
                           None) for i, o in zip(layer_dims[:-1], layer_dims[1:])]
        out.append(per_sym)
    return out


def atomic_network(x: Tensor, layers) -> Tensor:
    # nn/_core.py:146-149 with activation = torch.nn.GELU() and bias=False
    for w, _ in layers[:-1]:
        x = torch.nn.functional.gelu(x @ w.t(), approximate="none")
    return x @ layers[-1][0].t()


def ensemble_atomic_energies(symbols, weights, species: Tensor, aev: Tensor, members=None) -> Tensor:
    """(M_active, C, A) per-member atomic energies (nn/_containers.py:407-421,638-651)."""
    C, A = species.shape
    flat = species.reshape(-1)
    x = aev.reshape(C * A, -1)
    members = list(range(len(weights))) if members is None else members
    out = []
    for j in members:
        e = torch.zeros(C * A, dtype=aev.dtype)
        for i, s in enumerate(symbols):
            sel = torch.nonzero(flat == i).view(-1)
            if sel.numel():
                layers = [(w.to(aev.dtype), None) for w, _ in weights[j][s]]
                e = e.index_add(0, sel, atomic_network(x[sel], layers).view(-1))
        out.append(e.view(C, A))
    return torch.stack(out)


def compute(model: orc.Model, species: Tensor, coords: Tensor, cell: tp.Optional[Tensor] = None,
            pbc: tp.Optional[Tensor] = None, forces: bool = True, members: tp.Optional[tp.List[int]] = None,
            stress: bool = False) -> tp.Dict[str, Tensor]:
    """``ani_oracle.compute`` for a model with GELU bias-free networks (``model.weights`` from ``make_weights``)."""
    coords = coords.detach().clone().requires_grad_(forces)
    coords_in, scaling = coords, None
    if stress:
        assert cell is not None and pbc is not None, "stress needs a periodic cell"
        scaling = torch.eye(3, dtype=coords.dtype, requires_grad=True)
        coords = coords @ scaling
        cell = cell @ scaling
    nb = orc.neighborlist(model.neighborlist, model.spec.rcr, species, coords, cell, pbc)
    aev = orc.aev_from_neighbors(model.spec, species, nb)
    e_m = ensemble_atomic_energies(model.symbols, model.weights, species, aev, members)
    atomic_nn = e_m.mean(0)
    e_nn = atomic_nn.sum(-1)
    e_sae = orc.self_energies(model.symbols, model.sae, species, coords.dtype).sum(-1)
    out = {"aev": aev.detach(), "member_atomic": e_m.detach(), "atomic_nn": atomic_nn.detach(),
           "energy_nn": e_nn.detach(), "energy": (e_nn + e_sae).detach(), "num_pairs": torch.tensor(nb.indices.shape[1])}
    if forces:
        out["forces"] = -torch.autograd.grad(e_nn.sum(), coords_in, retain_graph=stress)[0]
    if stress:
        volume = torch.det(cell.detach()).abs()
        out["stress"] = (torch.autograd.grad(e_nn.sum(), scaling)[0] / volume).detach()   # Hartree / A^3
    return out
