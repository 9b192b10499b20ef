"""TEST INFRASTRUCTURE ONLY -- float64 restatement of the charge part of the reference's ANIq models.

* Charge networks (potentials/nnp.py:75-102, nn/_internal.py:69-90): per-element GELU bias-free networks with the
  ANI-2x widths on the model's AEV; ``out_dim = 2`` of which column 1 is the charge (``_ANINetworksDiscardFirstScalar``,
  ANImbis) or ``out_dim = 1`` (``ANINetworks``, simple_aniq).  0 for padding atoms.
* ``normalize`` (electro.py:29-93, ChargeNormalizer.forward): q = q_raw + (Q - sum q_raw) w / sum w, w = W[e]
  (* q_raw^2), 0 for padding.
* ``dipole`` (electro.py:96-156, DipoleComputer): sum_i q_i (r_i - r_ref) over the real atoms, r_ref the centre of
  mass (per-element masses), of geometry or the origin.

The energies are ``ani_oracle`` (CELU ensembles) or ``gelu_oracle`` (GELU bias-free ensembles).
"""
from __future__ import annotations

import math
import typing as tp

import numpy as np
import torch
from torch import Tensor

from oracle import ani_oracle as orc
from oracle import gelu_oracle as gor

FRAMES = ("center_of_mass", "center_of_geometry", "origin")


def make_charge_weights(symbols: tp.Sequence[str], dims: tp.Dict[str, tp.Tuple[int, ...]], in_dim: int, out_dim: int,
                        seed: int, dtype: torch.dtype = torch.float32
                        ) -> tp.Dict[str, tp.List[Tensor]]:
    """weights[symbol] = [W (out, in) for the 4 bias-free Linear layers], the last with ``out_dim`` rows; uniform in
    +-1/sqrt(fan_in) from numpy's PCG64 stream."""
    rng = np.random.default_rng(seed)
    out = {}
    for s in symbols:
        layer_dims = (in_dim,) + tuple(dims[s]) + (out_dim,)
        out[s] = [torch.tensor(rng.uniform(-1.0 / math.sqrt(i), 1.0 / math.sqrt(i), size=(o, i)), dtype=dtype)
                  for i, o in zip(layer_dims[:-1], layer_dims[1:])]
    return out


def raw_charges(symbols, weights, species: Tensor, aev: Tensor, kept: int) -> Tensor:
    """(C, A) raw charges: column ``kept`` of every element's network output, 0 for padding."""
    C, A = species.shape
    flat = species.reshape(-1)
    x = aev.reshape(C * A, -1)
    q = torch.zeros(C * A, dtype=aev.dtype)
    for i, s in enumerate(symbols):
        sel = torch.nonzero(flat == i).view(-1)
        if sel.numel():
            layers = [(w.to(aev.dtype), None) for w in weights[s]]
            h = x[sel]
            for w, _ in layers[:-1]:
                h = torch.nn.functional.gelu(h @ w.t(), approximate="none")
            q = q.index_add(0, sel, (h @ layers[-1][0].t())[:, kept])
    return q.view(C, A)


def normalize(species: Tensor, q_raw: Tensor, weights: tp.Sequence[float], scale_by_q2: bool,
              total_charge: float = 0.0) -> Tensor:
    w = torch.tensor(list(weights), dtype=q_raw.dtype)[species.clamp(min=0)].masked_fill(species < 0, 0.0)
    if scale_by_q2:
        w = w * q_raw ** 2
    excess = total_charge - q_raw.sum(-1, keepdim=True)
    return q_raw + excess * w / w.sum(-1, keepdim=True)


def dipole(species: Tensor, coords: Tensor, q: Tensor, frame: str, masses: tp.Optional[tp.Sequence[float]] = None
           ) -> Tensor:
    real = (species >= 0).to(coords.dtype)
    if frame == "origin":
        ref = torch.zeros(coords.shape[0], 1, 3, dtype=coords.dtype)
    else:
        if frame == "center_of_mass":
            m = torch.tensor(list(masses), dtype=coords.dtype)[species.clamp(min=0)] * real
        else:
            m = real
        ref = (m.unsqueeze(-1) * coords).sum(1, keepdim=True) / m.sum(1).view(-1, 1, 1)
    return ((q * real).unsqueeze(-1) * (coords - ref)).sum(1)


class ChargeModel(tp.NamedTuple):
    energy: orc.Model                       # the energy part (its weights: ani_oracle or gelu_oracle form)
    gelu_energy: bool                       # True: GELU bias-free energy networks (gelu_oracle)
    charge_weights: tp.Dict[str, tp.List[Tensor]]
    kept: int                               # output column of the charge networks
    norm_weights: tp.Tuple[float, ...]
    scale_by_q2: bool
    masses: tp.Tuple[float, ...]            # per element, for the centre-of-mass frame


def compute(model: ChargeModel, species: Tensor, coords: Tensor, cell: tp.Optional[Tensor] = None,
            pbc: tp.Optional[Tensor] = None, forces: bool = True) -> tp.Dict[str, Tensor]:
    """Energies / forces of the energy part, raw and normalised charges and the dipoles in the three frames."""
    e = (gor.compute if model.gelu_energy else orc.compute)(model.energy, species, coords, cell, pbc, forces=forces)
    q_raw = raw_charges(model.energy.symbols, model.charge_weights, species, e["aev"], model.kept)
    q = normalize(species, q_raw, model.norm_weights, model.scale_by_q2)
    out = dict(e)
    out["raw_charges"] = q_raw
    out["charges"] = q
    for f in FRAMES:
        out["dipole_" + f] = dipole(species, coords.detach(), q, f, model.masses)
    return out
