"""Atomic charges and dipoles with the interface of ``torchani.electro`` (electro.py:1-180).

``ChargeNormalizer`` makes raw atomic charges add up to a total charge, ``DipoleComputer`` / ``compute_dipole``
give the dipole sum_i q_i (r_i - r_ref) in e * Angstrom.  Both run the CUDA kernel ``ani_b200_charges`` (the one a
charge model's fused step uses, ``engine.Engine._charge_pass``) on CUDA tensors.

Tables.  The reference fills electronegativities, hardnesses and atomic masses from its literature tables
(``torchani.constants``).  They are not shipped here: ``ChargeNormalizer.from_electronegativity_and_hardness`` and a
centre-of-mass ``DipoleComputer`` raise ``ValueError`` unless the values are passed.  ``models.from_torchani`` reads
them from a reference model.
"""
from __future__ import annotations

import ctypes as C
import typing as tp

import torch
from torch import Tensor

from . import _lib
from ._lib import check, ptr
from .nn import ATOMIC_NUMBER

__all__ = ["BaseChargeNormalizer", "ChargeNormalizer", "DipoleComputer", "compute_dipole"]

Reference = tp.Literal["center_of_mass", "center_of_geometry", "origin"]


def frame_index(reference: str) -> int:
    """The ``frame`` argument of ``ani_b200_charges`` for a reference point name of the reference's DipoleComputer."""
    if reference not in _lib.DIPOLE_FRAMES:
        raise ValueError(f"unknown dipole reference {reference!r}; expected one of {_lib.DIPOLE_FRAMES}")
    return _lib.DIPOLE_FRAMES.index(reference)


def run_charges(elem_idxs: Tensor, q: Tensor, coords: tp.Optional[Tensor], weights: tp.Optional[tp.Sequence[float]],
                scale_by_q2: bool, normalize: bool, total_charge: float, masses: tp.Optional[tp.Sequence[float]],
                frame: int, want_dipoles: bool) -> tp.Tuple[Tensor, tp.Optional[Tensor]]:
    """One ``ani_b200_charges`` launch on plain (C, A) inputs in input order: (charges f32 (C, A), dipoles f64 (C, 3)
    or None).  ``elem_idxs`` are indices into ``weights`` / ``masses`` (-1 = padding)."""
    if q.device.type != "cuda":
        raise ValueError("torchani_b200 runs on CUDA tensors only (there is no CPU path)")
    if elem_idxs.dim() != 2 or q.shape != elem_idxs.shape:
        raise ValueError("element indices and charges must both have shape (C, A)")
    n_conf, n_per_conf = elem_idxs.shape
    S = max(len(weights or ()), len(masses or ()), 1)
    if S > _lib.ANI_MAX_SPECIES:
        raise ValueError(f"at most {_lib.ANI_MAX_SPECIES} elements per call")
    dev = q.device
    sp = elem_idxs.to(device=dev, dtype=torch.int32).contiguous()
    qf = q.detach().to(torch.float32).contiguous()
    out = torch.empty(n_conf, n_per_conf, dtype=torch.float32, device=dev)
    dip = torch.empty(n_conf, 3, dtype=torch.float64, device=dev) if want_dipoles else None
    co = None
    if want_dipoles:
        assert coords is not None and coords.shape == (n_conf, n_per_conf, 3)
        co = coords.detach().to(device=dev, dtype=torch.float32).contiguous()
    w = None if weights is None else (C.c_float * len(weights))(*weights)
    m = None if masses is None else (C.c_float * len(masses))(*masses)
    if n_conf * n_per_conf == 0:
        return out, (dip.zero_() if dip is not None else None)
    with torch.cuda.device(dev):
        st = torch.cuda.current_stream(dev).cuda_stream
        check(_lib.lib().ani_b200_charges(ptr(qf), None, None, ptr(sp), ptr(co), n_conf, n_per_conf, w, S,
                                          int(scale_by_q2), int(normalize), float(total_charge), m, frame, ptr(out),
                                          ptr(dip), st), "charges")
    return out, dip


class BaseChargeNormalizer(torch.nn.Module):
    """The identity normaliser (electro.py:22-26): raw charges are returned as they are."""

    def forward(self, elem_idxs: Tensor, raw_charges: Tensor, charge: int = 0) -> Tensor:
        return raw_charges


class ChargeNormalizer(BaseChargeNormalizer):
    r"""Normalise raw charges so that they add up to a total charge (electro.py:29-93):
    ``q_i = q_raw_i + (Q - sum q_raw) w_i / sum w`` with ``w_i = weights[e_i]`` (times ``q_raw_i^2`` with
    ``scale_weights_by_charges_squared``) and 0 for padding atoms."""

    atomic_numbers: Tensor
    weights: Tensor

    def __init__(self, symbols: tp.Sequence[str], weights: tp.Sequence[float] = (),
                 scale_weights_by_charges_squared: bool = False):
        super().__init__()
        self.atomic_numbers = torch.tensor([ATOMIC_NUMBER[e] for e in symbols], dtype=torch.long)
        if not weights:
            weights = [1.0] * len(symbols)
        if len(weights) != len(symbols):
            raise ValueError("one weight per symbol is required")
        self.register_buffer("weights", torch.tensor(list(weights), dtype=torch.float), persistent=False)
        self.scale_weights_by_charges_squared = bool(scale_weights_by_charges_squared)

    @classmethod
    def from_electronegativity_and_hardness(cls, symbols: tp.Sequence[str], electronegativity: tp.Sequence[float] = (),
                                            hardness: tp.Sequence[float] = (),
                                            scale_weights_by_charges_squared: bool = False) -> "ChargeNormalizer":
        """weights = (electronegativity / hardness)^2 per element.  The literature tables the reference falls back to
        are not shipped: pass both sequences (one value per symbol), or convert a reference model with
        ``models.from_torchani``, which reads its normaliser's weights."""
        if not electronegativity or not hardness:
            raise ValueError("electronegativities and hardnesses are not shipped with torchani_b200: pass both (one "
                             "value per symbol), or convert a reference model with models.from_torchani, which reads "
                             "its normaliser's weights")
        if len(electronegativity) != len(symbols) or len(hardness) != len(symbols):
            raise ValueError("one electronegativity and one hardness per symbol are required")
        weights = [(e / h) ** 2 for e, h in zip(electronegativity, hardness)]
        return cls(symbols, weights, scale_weights_by_charges_squared)

    def params(self) -> tp.Tuple[tp.Tuple[float, ...], bool]:
        """(weights as float32 values, scaling flag): what ``ani_b200_charges`` takes."""
        return tuple(float(w) for w in self.weights.float().cpu().tolist()), self.scale_weights_by_charges_squared

    def factor(self, elem_idxs: Tensor, raw_charges: Tensor) -> Tensor:
        weights = self.weights.to(raw_charges.device)[elem_idxs.clamp(min=0)].masked_fill(elem_idxs == -1, 0.0)
        if self.scale_weights_by_charges_squared:
            weights = weights * raw_charges ** 2
        return weights / torch.sum(weights, dim=-1, keepdim=True)

    def forward(self, elem_idxs: Tensor, raw_charges: Tensor, charge: int = 0) -> Tensor:
        """Normalised charges (C, A) in the dtype of ``raw_charges`` (computed in float32 with float64 sums)."""
        w, q2 = self.params()
        out, _ = run_charges(elem_idxs, raw_charges, None, w, q2, True, float(charge), None, 2, False)
        return out.to(raw_charges.dtype)


def _element_masses(atomic_nums: Tensor, masses: tp.Sequence[float]) -> tp.Tuple[Tensor, tp.List[float]]:
    """Atomic numbers (C, A) -> (element indices into the returned per-element masses, those masses).  ``masses`` is
    indexed by atomic number, as the reference's ``AtomicNumbersToMasses``."""
    znums = sorted(int(z) for z in torch.unique(atomic_nums).tolist() if z >= 0)
    if any(z == 0 for z in znums):
        raise ValueError("Input should be atomic numbers")
    if len(znums) > _lib.ANI_MAX_SPECIES:
        raise ValueError(f"at most {_lib.ANI_MAX_SPECIES} elements per call")
    table = torch.full((max(znums + [0]) + 2,), -1, dtype=torch.long)
    for i, z in enumerate(znums):
        table[z] = i
    elem = table.to(atomic_nums.device)[atomic_nums.clamp(min=0)].masked_fill(atomic_nums < 0, -1)
    el_masses = [float(masses[z]) for z in znums] if masses else []
    return elem, el_masses


class DipoleComputer(torch.nn.Module):
    r"""Dipoles in e * Angstrom (electro.py:96-156): ``sum_i q_i (r_i - r_ref)`` over the real atoms, with ``r_ref``
    the centre of mass, the centre of geometry or the origin.  ``masses`` are indexed by atomic number (as the
    reference's ``AtomicNumbersToMasses``); the reference's mass table is not shipped, so the centre-of-mass frame
    needs them."""

    def __init__(self, masses: tp.Iterable[float] = (), reference: Reference = "center_of_mass", device=None,
                 dtype=None) -> None:
        super().__init__()
        self._masses = [float(m) for m in masses]
        self._frame = frame_index(reference)
        if self._frame == 0 and not self._masses:
            raise ValueError("atomic masses are not shipped with torchani_b200: pass masses (indexed by atomic "
                             "number) for the center_of_mass reference, or use 'center_of_geometry' / 'origin'")
        self._atomic_masses = torch.tensor(self._masses, device=device, dtype=dtype)
        self._center_of_mass = self._frame == 0
        self._skip = self._frame == 2

    def forward(self, atomic_nums: Tensor, coordinates: Tensor, charges: Tensor) -> Tensor:
        """atomic_nums (C, A) (-1 = padding), coordinates (C, A, 3), charges (C, A) -> dipoles (C, 3) in the dtype of
        ``coordinates``."""
        assert atomic_nums.shape == charges.shape == coordinates.shape[:-1]
        elem, el_masses = _element_masses(atomic_nums, self._masses)
        _, dip = run_charges(elem, charges, coordinates, None, False, False, 0.0,
                             el_masses if self._frame == 0 else None, self._frame, True)
        return dip.to(coordinates.dtype)


def compute_dipole(species: Tensor, coordinates: Tensor, charges: Tensor, reference: Reference = "center_of_mass",
                   masses: tp.Sequence[float] = ()) -> Tensor:
    """Dipoles in e * Angstrom (electro.py:159-180).  ``masses`` (indexed by atomic number) are needed for the
    centre-of-mass frame: the reference's table is not shipped."""
    return DipoleComputer(masses, reference, species.device, coordinates.dtype)(species, coordinates, charges)
