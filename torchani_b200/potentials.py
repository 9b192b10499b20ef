"""Pair potentials with the interface of ``torchani.potentials`` (potentials/core.py:106-207): the short-range
repulsion terms ``RepulsionXTB`` (potentials/xtb.py) and ``RepulsionZBL`` (potentials/zbl.py), the Lennard-Jones
terms ``LennardJones``, ``RepulsionLJ`` and ``DispersionLJ`` (potentials/lj.py), the fixed-charge Coulomb terms
``FixedCoulomb`` and ``FixedMNOK`` (potentials/fixed_coulomb.py), and the D3(BJ) two-body dispersion
``TwoBodyDispersionD3`` (potentials/dftd3.py).

Inside a model (``models.ANI(..., potentials={...})``) the repulsion terms are evaluated by the fused step over the
neighbour list the AEV kernel has just built (``ani_b200_pair_potential``), which is why their cutoff may not exceed
the radial AEV cutoff.  The LJ and Coulomb terms run over a neighbour search of their own cutoff on the step's bucket
grid (``ani_b200_pair_potential_search``), at any cutoff; without a cutoff (the reference's default) on open systems
only.  On its own a module evaluates a half pair list (``compute_from_neighbors``, ``forward``) through
``ani_b200_pair_potential_pairs``.  CUDA float32 only; there is no CPU path.

D3 has a cutoff beyond Rcr (8 A in the reference's models) and coordination numbers that make it many-body: inside a
model it runs its own neighbour search over the step's bucket grid (``ani_b200_dispersion_d3``, three launches).

The reference's per-element xTB ``alpha`` / ``yeff`` defaults, its D3 tables (C6 references, covalent radii,
empirical charges) and its ff19SB LJ table are not shipped; neither are atomic charges or hardnesses for the Coulomb
terms: pass them, or convert a reference module (``from_torchani``), which reads its buffers.
"""
from __future__ import annotations

import math
import typing as tp

import torch
from torch import Tensor

from . import _lib
from ._lib import D3Params, PairParams, check, ptr
from .neighbors import Neighbors, all_pairs
from .nn import ATOMIC_NUMBER

ANGSTROM_TO_BOHR = 1.8897261258369282   # units.py:41
HARTREE_TO_KCALPERMOL = 627.5094738898777   # units.py:51
_CUTOFF_FNS = {"cosine": 0, "smooth": 1, "dummy": 2}


def _cutoff_fn_name(cutoff_fn: tp.Any) -> str:
    """'cosine' / 'smooth' from a name or a reference cutoff module (cutoffs.py: CutoffCosine, CutoffSmooth with
    order 2 and eps 1e-10, CutoffDummy)."""
    if isinstance(cutoff_fn, str):
        name = cutoff_fn
    else:
        name = {"CutoffCosine": "cosine", "CutoffSmooth": "smooth", "CutoffDummy": "dummy"}.get(
            type(cutoff_fn).__name__, type(cutoff_fn).__name__)
        if name == "smooth" and (getattr(cutoff_fn, "order", 2) != 2 or getattr(cutoff_fn, "eps", 1e-10) != 1e-10):
            raise ValueError("only the smooth cutoff with order=2, eps=1e-10 is supported by the CUDA kernels")
    if name not in ("cosine", "smooth", "dummy"):
        raise ValueError(f"cutoff function {name!r} is not supported by the CUDA kernels")
    return name


class _HalfListEnergy(torch.autograd.Function):
    """coords -> (energies (C,) float64, atomic energies (C, A)) of a term over a half pair list.  ``launch(species,
    idx, dist, diff, ghost, atomic, energies, grad, stream)`` runs the term's half-list entry point; dE/dcoords is
    produced by that forward launch (gradients reach ``coords`` only, as in ``AEVComputer.compute_from_neighbors``)."""

    @staticmethod
    def forward(ctx, coords: Tensor, elem_idxs: Tensor, neighbors: Neighbors, ghost_flags: tp.Optional[Tensor],
                launch: tp.Callable[..., None]):
        n_conf, n_per_conf = elem_idxs.shape
        dev = coords.device
        species = elem_idxs.reshape(-1).to(torch.int32).contiguous()
        idx = neighbors.indices.to(torch.int64).contiguous()
        dist = neighbors.distances.detach().to(torch.float32).contiguous()
        diff = neighbors.diff_vectors.detach().to(torch.float32).contiguous()
        ghost = None if ghost_flags is None else ghost_flags.reshape(-1).to(torch.uint8).contiguous()
        want_grad = bool(coords.requires_grad)
        atomic = torch.zeros(n_conf, n_per_conf, dtype=torch.float32, device=dev)
        energies = torch.zeros(n_conf, dtype=torch.float64, device=dev)
        grad = torch.zeros(n_conf, n_per_conf, 3, dtype=torch.float32, device=dev) if want_grad else None
        with torch.cuda.device(dev):
            launch(species, idx, dist, diff, ghost, atomic, energies, grad, torch.cuda.current_stream(dev).cuda_stream)
        ctx.want_grad = want_grad
        if want_grad:
            ctx.save_for_backward(grad)
        return energies, atomic

    @staticmethod
    def backward(ctx, g_energy, g_atomic):
        _lib.forbid_create_graph("the CUDA pair potentials over a half neighbour list (_HalfListEnergy)")
        if not ctx.want_grad:
            raise RuntimeError("energies were computed without forces (coords.requires_grad was False)")
        (grad,) = ctx.saved_tensors
        out = torch.zeros_like(grad)
        if g_energy is not None:
            out = out + grad * g_energy.to(grad.dtype).view(-1, 1, 1)
        if g_atomic is not None and bool((g_atomic != 0).any()):
            if not bool((g_atomic == g_atomic[:, :1]).all()):
                raise NotImplementedError("per-atom upstream gradients that differ inside a conformer are not supported")
            out = out + grad * g_atomic[:, :1].to(grad.dtype).unsqueeze(-1)
        return out, None, None, None, None


class PairPotential(torch.nn.Module):
    """Base of the pair potentials (potentials/core.py:106-207, ``BasePairPotential``).  Subclasses fill the
    element-pair tables of ``ani_pair_params`` in ``_fill``."""

    kind = -1
    _to_bohr = ANGSTROM_TO_BOHR   # the length unit of the kernel's d (the LJ kinds work in A)

    def __init__(self, symbols: tp.Sequence[str], *, cutoff: float = math.inf, cutoff_fn: tp.Any = "smooth"):
        super().__init__()
        if not 1 <= len(symbols) <= _lib.ANI_MAX_SPECIES:
            raise ValueError(f"the CUDA kernels support 1..{_lib.ANI_MAX_SPECIES} elements")
        self.symbols = tuple(symbols)
        self.register_buffer("atomic_numbers", torch.tensor([ATOMIC_NUMBER[s] for s in symbols], dtype=torch.long),
                             persistent=False)
        self.cutoff = float(cutoff)
        if not self.cutoff > 0:
            raise ValueError("cutoff must be positive")
        # potentials/core.py:132-135: without a cutoff there is no envelope
        self.cutoff_fn = "dummy" if self.cutoff == math.inf else _cutoff_fn_name(cutoff_fn)
        if self.cutoff != math.inf and self.cutoff_fn == "dummy":
            raise ValueError("a finite cutoff needs the cosine or the smooth envelope")
        self._enabled = True

    def _fill(self, p: PairParams) -> None:
        raise NotImplementedError

    def params(self) -> PairParams:
        """The ``ani_pair_params`` of this potential (built from its current buffers)."""
        p = PairParams()
        p.kind, p.cutoff_fn, p.num_species = self.kind, _CUTOFF_FNS[self.cutoff_fn], len(self.symbols)
        p.cutoff = self.cutoff if self.cutoff != math.inf else 0.0
        p.to_bohr = self._to_bohr
        self._fill(p)
        return p

    def _table(self, dst, values: Tensor) -> None:
        v = values.detach().to("cpu", torch.float64)
        if not bool(torch.isfinite(v).all()):
            raise ValueError("pair-potential parameters contain inf/NaN")
        for a in range(v.shape[0]):
            for b in range(v.shape[1]):
                dst[a][b] = float(v[a, b])

    def _half_list_launch(self, device: torch.device) -> tp.Callable[..., None]:
        """The launch of this term over a half pair list, for ``_HalfListEnergy``."""
        p = self.params()

        def launch(species, idx, dist, diff, ghost, atomic, energies, grad, stream):
            check(_lib.lib().ani_b200_pair_potential_pairs(
                _lib.C.byref(p), ptr(species), idx[0].data_ptr(), idx[1].data_ptr(), ptr(dist), ptr(diff), ptr(ghost),
                idx.shape[1], *atomic.shape, ptr(atomic), ptr(energies), ptr(grad), stream), "pair_potential_pairs")
        return launch

    def compute_from_neighbors(self, elem_idxs: Tensor, coords: Tensor, neighbors: Neighbors, charge: int = 0,
                               atomic: bool = False, ensemble_values: bool = False,
                               ghost_flags: tp.Optional[Tensor] = None) -> Tensor:
        """Energies ``(C,)`` or ``(C, A)`` of the given half pair list (potentials/core.py:181-207; pairs beyond the
        cutoff are ignored, pairs that touch a ghost atom count half; ``ensemble_values`` is disregarded as in the
        reference).  D3 (dftd3.py:221-246) counts every listed pair in the coordination numbers."""
        assert elem_idxs.dim() == 2 and coords.shape == (elem_idxs.shape[0], elem_idxs.shape[1], 3)
        if coords.device.type != "cuda":
            raise ValueError("torchani_b200 runs on CUDA tensors only (there is no CPU path)")
        if ghost_flags is not None and ghost_flags.numel() != elem_idxs.numel():
            raise ValueError("ghost_flags and species should have the same number of elements")
        energies, atomic_e = _HalfListEnergy.apply(coords, elem_idxs, neighbors, ghost_flags,
                                                   self._half_list_launch(coords.device))
        return atomic_e.to(coords.dtype) if atomic else energies.to(coords.dtype)

    def forward(self, species: Tensor, coords: Tensor, cell: tp.Optional[Tensor] = None,
                pbc: tp.Optional[Tensor] = None, atomic: bool = False, ensemble_values: bool = False,
                atomic_nums_input: bool = True) -> Tensor:
        """potentials/core.py:37-67: the energies of this potential alone, with a neighbour list of its own."""
        if self.cutoff == math.inf:
            raise ValueError("forward() needs a finite cutoff (the neighbour list is a bucket grid); "
                             "use compute_from_neighbors with a list of your own")
        elem_idxs = species
        if atomic_nums_input:
            conv = torch.full((int(self.atomic_numbers.max()) + 2,), -1, dtype=torch.long, device=species.device)
            conv[self.atomic_numbers.to(species.device)] = torch.arange(len(self.symbols), device=species.device)
            elem_idxs = conv[species]
        neighbors = all_pairs(self.cutoff, elem_idxs, coords, cell, pbc)
        return self.compute_from_neighbors(elem_idxs, coords, neighbors, 0, atomic, ensemble_values)


class RepulsionXTB(PairPotential):
    r"""xTB repulsion (potentials/xtb.py:16-77): ``E = y_ab / d * exp(-sqrt_alpha_ab * d^k_ab)``, d in Bohr, ``k_ab =
    krep`` except H-H (``krep_hydrogen``).  ``alpha`` and ``yeff`` (one value per symbol) are required."""

    kind = 0

    def __init__(self, symbols: tp.Sequence[str], krep_hydrogen: float = 1.0, krep: float = 1.5,
                 alpha: tp.Sequence[float] = (), yeff: tp.Sequence[float] = (), *, cutoff: float = math.inf,
                 cutoff_fn: tp.Any = "smooth"):
        super().__init__(symbols, cutoff=cutoff, cutoff_fn=cutoff_fn)
        for name, seq in (("alpha", alpha), ("yeff", yeff)):
            if not len(seq):
                raise ValueError(
                    f"RepulsionXTB needs `{name}` (one value per symbol): the reference's per-element xTB parameter "
                    "table is not shipped with torchani_b200; pass the values or convert a reference module "
                    "(potentials.from_torchani / models.from_torchani), which reads its buffers")
            if len(seq) != len(symbols):
                raise ValueError(f"`{name}` needs one value per symbol")
        k_rep_ab = torch.full((len(symbols), len(symbols)), float(krep))
        if "H" in self.symbols:
            h = self.symbols.index("H")
            k_rep_ab[h, h] = float(krep_hydrogen)
        _yeff = torch.tensor(list(yeff), dtype=torch.float32)
        _alpha = torch.tensor(list(alpha), dtype=torch.float32)
        self.register_buffer("y_ab", torch.outer(_yeff, _yeff))
        self.register_buffer("sqrt_alpha_ab", torch.outer(_alpha, _alpha).sqrt())
        self.register_buffer("k_rep_ab", k_rep_ab)

    def _fill(self, p: PairParams) -> None:
        self._table(p.a, self.y_ab)
        self._table(p.b, self.sqrt_alpha_ab)
        self._table(p.c, self.k_rep_ab)


class RepulsionZBL(PairPotential):
    r"""Ziegler-Biersack-Littmark screened nuclear repulsion (potentials/zbl.py:14-81):
    ``E = Z_a Z_b / d * sum_q c_q exp(-x_q * d * (Z_a^p + Z_b^p) / k)``, d in Bohr.  The defaults are the published
    universal screening function (the coefficient set LAMMPS uses, which sums to 1); effective Z = atomic number."""

    kind = 1

    def __init__(self, symbols: tp.Sequence[str], k: float = 0.8853,
                 screen_coeffs: tp.Sequence[float] = (0.18175, 0.50986, 0.28022, 0.02817),
                 screen_exponents: tp.Sequence[float] = (3.19980, 0.94229, 0.40290, 0.20162),
                 eff_exponent: float = 0.23, eff_atomic_nums: tp.Sequence[float] = (), *, cutoff: float = math.inf,
                 cutoff_fn: tp.Any = "smooth"):
        super().__init__(symbols, cutoff=cutoff, cutoff_fn=cutoff_fn)
        if len(screen_exponents) != len(screen_coeffs):
            raise ValueError("screen_exponents and screen_coeffs must have the same len")
        if len(screen_coeffs) != 4:
            raise ValueError("the CUDA kernel evaluates exactly four screening terms")
        if not math.isclose(sum(screen_coeffs), 1.0, abs_tol=1e-6):   # (float32 buffers of a converted module)
            raise ValueError("Screen coeffs must sum to 1")
        if not len(eff_atomic_nums):
            eff_atomic_nums = [float(ATOMIC_NUMBER[s]) for s in symbols]
        if len(eff_atomic_nums) != len(symbols):
            raise ValueError("`eff_atomic_nums` needs one value per symbol")
        self.register_buffer("_eff_atomic_nums", torch.tensor(list(eff_atomic_nums), dtype=torch.float32),
                             persistent=False)
        self.register_buffer("_coeffs", torch.tensor(list(screen_coeffs), dtype=torch.float32).view(1, -1),
                             persistent=False)
        self.register_buffer("_exponents", torch.tensor(list(screen_exponents), dtype=torch.float32).view(1, -1),
                             persistent=False)
        self._k = float(k)
        self._kz = float(eff_exponent)

    def _fill(self, p: PairParams) -> None:
        z = self._eff_atomic_nums.detach().to("cpu", torch.float64)
        self._table(p.a, torch.outer(z, z))
        zp = z ** self._kz
        self._table(p.b, (zp.view(-1, 1) + zp.view(1, -1)) / self._k)
        for q in range(4):
            p.screen_coeff[q] = float(self._coeffs.view(-1)[q])
            p.screen_exp[q] = float(self._exponents.view(-1)[q])


def _per_symbol(cls_name: str, name: str, seq: tp.Sequence[float], symbols: tp.Sequence[str]) -> Tensor:
    """One float32 value per symbol (the reference keeps these as float32 buffers, potentials/lj.py:84-88)."""
    if not len(seq):
        raise ValueError(f"{cls_name} needs `{name}` (one value per symbol): it has no default in torchani_b200; pass "
                         "the values or convert a reference module (potentials.from_torchani / models.from_torchani), "
                         "which reads its buffers")
    if len(seq) != len(symbols):
        raise ValueError(f"`{name}` needs one value per symbol")
    return torch.tensor([float(v) for v in seq], dtype=torch.float32)


class _LJ(PairPotential):
    r"""Lennard-Jones style potentials (potentials/lj.py:60-115): ``eps`` in Hartree and ``sigma`` in Angstrom, one
    value per symbol, combined by the Berthelot (``sqrt(eps_a eps_b)``) and Lorentz (``(sigma_a + sigma_b) / 2``)
    rules.  The defaults are the reference's: sigma = 1.5 A and eps = 0.1 kcal/mol for every element."""

    _to_bohr = 1.0

    def __init__(self, symbols: tp.Sequence[str], eps: tp.Sequence[float] = (), sigma: tp.Sequence[float] = (), *,
                 trainable: tp.Sequence[str] = (), cutoff: float = math.inf, cutoff_fn: tp.Any = "smooth"):
        super().__init__(symbols, cutoff=cutoff, cutoff_fn=cutoff_fn)
        if len(trainable):
            raise ValueError(f"{type(self).__name__}: trainable pair-potential parameters are not supported by the "
                             "CUDA kernels")
        name = type(self).__name__
        S = len(symbols)
        eps = eps if len(eps) else [0.1 / HARTREE_TO_KCALPERMOL] * S
        sigma = sigma if len(sigma) else [1.5] * S
        self.register_buffer("_eps", _per_symbol(name, "eps", eps, symbols), persistent=False)
        self.register_buffer("_sigma", _per_symbol(name, "sigma", sigma, symbols), persistent=False)

    def _fill(self, p: PairParams) -> None:
        eps = self._eps.detach().to("cpu", torch.float64)
        sigma = self._sigma.detach().to("cpu", torch.float64)
        self._table(p.a, torch.outer(eps, eps).sqrt())
        self._table(p.b, (sigma.view(-1, 1) + sigma.view(1, -1)) / 2)


class LennardJones(_LJ):
    r"""``E = 4 eps_ab (x^12 - x^6)``, ``x = sigma_ab / max(R, 1e-7)`` (potentials/lj.py:138-145)."""

    kind = 2


class RepulsionLJ(_LJ):
    r"""``E = 4 eps_ab x^12`` (potentials/lj.py:128-135)."""

    kind = 3


class DispersionLJ(_LJ):
    r"""``E = -4 eps_ab x^6`` (potentials/lj.py:118-125)."""

    kind = 4


class FixedCoulomb(PairPotential):
    r"""Coulomb energy of fixed per-element charges (potentials/fixed_coulomb.py:13-38):
    ``E = q_a q_b / (dielectric * max(R, 1e-7) * to_bohr)``.  ``charges`` (e, one value per symbol) are required."""

    kind = 5

    def __init__(self, symbols: tp.Sequence[str], dielectric: float = 1.0, charges: tp.Sequence[float] = (), *,
                 cutoff: float = math.inf, cutoff_fn: tp.Any = "smooth"):
        super().__init__(symbols, cutoff=cutoff, cutoff_fn=cutoff_fn)
        self._dielectric = float(dielectric)
        self.register_buffer("_charges", _per_symbol("FixedCoulomb", "charges", charges, symbols), persistent=False)

    def _fill(self, p: PairParams) -> None:
        q = self._charges.detach().to("cpu", torch.float64)
        self._table(p.a, torch.outer(q, q) / self._dielectric)


class FixedMNOK(PairPotential):
    r"""Mataga-Nishimoto-Ohno-Klopman screened Coulomb energy of fixed per-element charges
    (potentials/fixed_coulomb.py:49-81): ``E = q_a q_b / sqrt((R to_bohr)^2 + (2 / (eta_a + eta_b))^2)``, R not
    clamped.  As in the reference, ``dielectric`` is stored but does not enter the energy.  ``charges`` and ``eta`` (one
    value per symbol) are required."""

    kind = 6

    def __init__(self, symbols: tp.Sequence[str], dielectric: float = 1.0, charges: tp.Sequence[float] = (),
                 eta: tp.Sequence[float] = (), *, cutoff: float = math.inf, cutoff_fn: tp.Any = "smooth"):
        super().__init__(symbols, cutoff=cutoff, cutoff_fn=cutoff_fn)
        self._dielectric = float(dielectric)
        self.register_buffer("_charges", _per_symbol("FixedMNOK", "charges", charges, symbols), persistent=False)
        self.register_buffer("_eta", _per_symbol("FixedMNOK", "eta", eta, symbols), persistent=False)

    def _fill(self, p: PairParams) -> None:
        q = self._charges.detach().to("cpu", torch.float64)
        eta = self._eta.detach().to("cpu", torch.float64)
        self._table(p.a, torch.outer(q, q))
        self._table(p.b, 2 / (eta.view(-1, 1) + eta.view(1, -1)))


class _BeckeJohnsonDamp(torch.nn.Module):
    """Holds the damping radii of D3(BJ) under the reference's state-dict key ``_damp_fn.cutoff_radii``
    (potentials/dftd3.py:45-110): ``cutoff_radii = sqrt(3 outer(sqrt_q, sqrt_q))`` in Bohr, and ``_a1``, ``_a2``."""

    def __init__(self, a1: float, a2: float, sqrt_empirical_charge: Tensor):
        super().__init__()
        self.register_buffer("cutoff_radii", torch.sqrt(3 * torch.outer(sqrt_empirical_charge, sqrt_empirical_charge)))
        self._a1 = float(a1)
        self._a2 = float(a2)


class TwoBodyDispersionD3(PairPotential):
    r"""DFT-D3 two-body dispersion with Becke-Johnson damping (potentials/dftd3.py:113-311): coordination numbers,
    C6 interpolated between the tabulated references, ``C8 = 3 C6 sqrt_q_a sqrt_q_b``, and
    ``E = -(s6 C6 / (d^6 + (a1 R0 + a2)^6) + s8 C8 / (d^8 + (a1 R0 + a2)^8))`` per pair, times the envelope.

    ``sqrt_empirical_charge`` and ``covalent_radii`` (Angstrom) are one value per symbol; ``coeff6``,
    ``coordnums_a``, ``coordnums_b`` are the reference's ``precalc_*`` tables for these symbols, shape ``(S, S, 5,
    5)``, -1 where a reference is missing.  None of them is shipped: pass them, or convert a reference module
    (``potentials.from_torchani``), or pass the buffers of a reference state dict (the keys are the reference's,
    ``load_state_dict`` accepts its legacy ``_damp_fn_6`` / ``_damp_fn_8`` keys)."""

    def __init__(self, symbols: tp.Sequence[str], s6: float, s8: float, damp_a1: float, damp_a2: float,
                 sqrt_empirical_charge: tp.Sequence[float] = (), covalent_radii: tp.Sequence[float] = (), *,
                 coeff6: tp.Optional[tp.Any] = None, coordnums_a: tp.Optional[tp.Any] = None,
                 coordnums_b: tp.Optional[tp.Any] = None, cutoff_fn: tp.Any = "smooth", cutoff: float = math.inf):
        super().__init__(symbols, cutoff=cutoff, cutoff_fn=cutoff_fn)
        S = len(symbols)
        named = {"sqrt_empirical_charge": sqrt_empirical_charge, "covalent_radii": covalent_radii,
                 "coeff6": coeff6, "coordnums_a": coordnums_a, "coordnums_b": coordnums_b}
        for name, val in named.items():
            if val is None or (not isinstance(val, Tensor) and not len(val)):
                raise ValueError(
                    f"TwoBodyDispersionD3 needs `{name}`: the reference's D3 tables (c6.h5, atomic constants) are not "
                    "shipped with torchani_b200; pass them (e.g. the precalc_* buffers of a reference state dict, "
                    "then load_state_dict), or convert a reference module with potentials.from_torchani")
        sq = torch.as_tensor(sqrt_empirical_charge, dtype=torch.float32).reshape(-1)
        rc = torch.as_tensor(covalent_radii, dtype=torch.float32).reshape(-1)
        if sq.numel() != S or rc.numel() != S:
            raise ValueError("sqrt_empirical_charge and covalent_radii need one value per symbol")
        tabs = [torch.as_tensor(t, dtype=torch.float32) for t in (coeff6, coordnums_a, coordnums_b)]
        for t in tabs:
            if t.shape != (S, S, 5, 5):
                raise ValueError(f"the D3 reference tables must have shape ({S}, {S}, 5, 5), got {tuple(t.shape)}")
        self._damp_fn = _BeckeJohnsonDamp(damp_a1, damp_a2, sq)
        self._s6 = float(s6)
        self._s8 = float(s8)
        self._k1, self._k2, self._k3 = 16, 4 / 3, 4      # dftd3.py:171-174
        self.register_buffer("precalc_coeff6", tabs[0].clone())
        self.register_buffer("precalc_coordnums_a", tabs[1].clone())
        self.register_buffer("precalc_coordnums_b", tabs[2].clone())
        self.register_buffer("sqrt_charge_ab", torch.outer(sq, sq))
        self.register_buffer("covalent_radii", rc * ANGSTROM_TO_BOHR)   # Bohr, dftd3.py:162-163
        self._device_tables: tp.Dict[str, tp.Tuple[tp.Any, Tensor]] = {}

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs) -> None:
        # dftd3.py:127-138: older files hold `_damp_fn_6` (dropped) and `_damp_fn_8` (= `_damp_fn`)
        for k in list(state_dict.keys()):
            if not k.startswith(prefix):
                continue
            if "damp_fn_6" in k:
                state_dict.pop(k)
            elif "damp_fn_8" in k:
                state_dict[k.replace("damp_fn_8", "damp_fn")] = state_dict.pop(k)
        super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)

    def _versions(self) -> tp.Tuple[tp.Any, ...]:
        bufs = (self.precalc_coeff6, self.precalc_coordnums_a, self.precalc_coordnums_b)
        return tuple((b._version, b.data_ptr()) for b in bufs)

    def params(self) -> D3Params:
        """The ``ani_d3_params`` of this term (built from its current buffers)."""
        p = D3Params()
        S = len(self.symbols)
        p.cutoff_fn, p.num_species = _CUTOFF_FNS[self.cutoff_fn], S
        p.cutoff = self.cutoff if self.cutoff != math.inf else 0.0
        p.to_bohr = ANGSTROM_TO_BOHR
        p.s6, p.s8, p.a1, p.a2 = self._s6, self._s8, self._damp_fn._a1, self._damp_fn._a2
        p.k1, p.k2, p.k3 = float(self._k1), float(self._k2), float(self._k3)
        rcov = self.covalent_radii.detach().to("cpu", torch.float64)
        r0 = self._damp_fn.cutoff_radii.detach().to("cpu", torch.float64)
        q = self.sqrt_charge_ab.detach().to("cpu", torch.float64)
        for t in (rcov, r0, q):
            if not bool(torch.isfinite(t).all()):
                raise ValueError("D3 parameters contain inf/NaN")
        damp = self._damp_fn._a1 * r0 + self._damp_fn._a2
        for a in range(S):
            p.rcov[a] = float(rcov[a])
            for b in range(S):
                p.damp6[a][b] = float(damp[a, b] ** 6)
                p.damp8[a][b] = float(damp[a, b] ** 8)
                p.c8_scale[a][b] = float(3.0 * q[a, b])
        return p

    def tables(self, device: torch.device) -> Tensor:
        """The reference tables as the kernels read them: f32 (S, S, 25, 4) = {C6ref, CNa, CNb, 0} on ``device``
        (cached while the buffers are unchanged)."""
        key = str(device)
        hit = self._device_tables.get(key)
        if hit is not None and hit[0] == self._versions():
            return hit[1]
        S = len(self.symbols)
        t = torch.zeros(S, S, 25, 4, dtype=torch.float32)
        for k, buf in enumerate((self.precalc_coeff6, self.precalc_coordnums_a, self.precalc_coordnums_b)):
            t[..., k] = buf.detach().to("cpu", torch.float32).reshape(S, S, 25)
        if not bool(torch.isfinite(t).all()):
            raise ValueError("D3 reference tables contain inf/NaN")
        t = t.to(device)
        self._device_tables[key] = (self._versions(), t)
        return t

    def _half_list_launch(self, device: torch.device) -> tp.Callable[..., None]:
        p, tables = self.params(), self.tables(device)

        def launch(species, idx, dist, diff, ghost, atomic, energies, grad, stream):
            cn = torch.empty(atomic.numel(), dtype=torch.float32, device=device)
            dedcn = torch.empty_like(cn) if grad is not None else None
            check(_lib.lib().ani_b200_dispersion_d3_pairs(
                _lib.C.byref(p), ptr(tables), ptr(species), idx[0].data_ptr(), idx[1].data_ptr(), ptr(dist),
                ptr(diff), ptr(ghost), idx.shape[1], *atomic.shape, ptr(cn), ptr(dedcn), ptr(atomic), ptr(energies),
                ptr(grad), stream), "dispersion_d3_pairs")
        return launch


def _buffer_values(ref_pot, key: str) -> tp.List[float]:
    """A per-element buffer of a reference module; trainable parameters are refused (not supported by the kernels)."""
    v = getattr(ref_pot, key)
    if isinstance(v, torch.nn.Parameter):
        raise ValueError(f"{type(ref_pot).__name__}: trainable pair-potential parameters ({key}) are not supported by "
                         "the CUDA kernels")
    return [float(x) for x in v.detach().to("cpu", torch.float32).tolist()]


def from_torchani(ref_pot) -> PairPotential:
    """A reference ``RepulsionXTB`` / ``RepulsionZBL`` / ``LennardJones`` / ``RepulsionLJ`` / ``DispersionLJ`` /
    ``FixedCoulomb`` / ``FixedMNOK`` / ``TwoBodyDispersionD3`` module -> the CUDA module with the same parameters (read
    from the module's buffers).  Any other potential raises ``ValueError``."""
    name = type(ref_pot).__name__
    symbols = tuple(ref_pot.symbols)
    cutoff_fn = ref_pot.cutoff_fn
    lj = {"LennardJones": LennardJones, "RepulsionLJ": RepulsionLJ, "DispersionLJ": DispersionLJ}
    if name in lj:
        out: PairPotential = lj[name](symbols, eps=_buffer_values(ref_pot, "_eps"),
                                      sigma=_buffer_values(ref_pot, "_sigma"), cutoff=ref_pot.cutoff,
                                      cutoff_fn=cutoff_fn)
    elif name == "FixedCoulomb":
        out = FixedCoulomb(symbols, float(ref_pot._dielectric), _buffer_values(ref_pot, "_charges"),
                           cutoff=ref_pot.cutoff, cutoff_fn=cutoff_fn)
    elif name == "FixedMNOK":
        out = FixedMNOK(symbols, float(ref_pot._dielectric), _buffer_values(ref_pot, "_charges"),
                        _buffer_values(ref_pot, "_eta"), cutoff=ref_pot.cutoff, cutoff_fn=cutoff_fn)
    elif name == "RepulsionXTB":
        out = RepulsionXTB(symbols, alpha=[1.0] * len(symbols), yeff=[1.0] * len(symbols),
                                          cutoff=ref_pot.cutoff, cutoff_fn=cutoff_fn)
        for key in ("y_ab", "sqrt_alpha_ab", "k_rep_ab"):
            getattr(out, key).copy_(getattr(ref_pot, key).detach().to("cpu", torch.float32))
    elif name == "RepulsionZBL":
        out = RepulsionZBL(symbols, k=ref_pot._k, screen_coeffs=ref_pot._coeffs.view(-1).tolist(),
                           screen_exponents=ref_pot._exponents.view(-1).tolist(), eff_exponent=ref_pot._kz,
                           eff_atomic_nums=ref_pot._eff_atomic_nums.tolist(), cutoff=ref_pot.cutoff,
                           cutoff_fn=cutoff_fn)
    elif name == "TwoBodyDispersionD3":
        S = len(symbols)
        damp = ref_pot._damp_fn
        # (sqrt_charge_ab = outer(sqrt_q, sqrt_q); the diagonal gives sqrt_q back.  The buffers are then copied as they
        # are, so nothing is recomputed from them)
        sq = ref_pot.sqrt_charge_ab.detach().double().diagonal().sqrt().tolist()
        out = TwoBodyDispersionD3(symbols, float(ref_pot._s6), float(ref_pot._s8), float(damp._a1), float(damp._a2),
                                  sq, [1.0] * S, coeff6=ref_pot.precalc_coeff6.detach().cpu(),
                                  coordnums_a=ref_pot.precalc_coordnums_a.detach().cpu(),
                                  coordnums_b=ref_pot.precalc_coordnums_b.detach().cpu(), cutoff=ref_pot.cutoff,
                                  cutoff_fn=cutoff_fn)
        for key in ("sqrt_charge_ab", "covalent_radii"):
            getattr(out, key).copy_(getattr(ref_pot, key).detach().to("cpu", torch.float32))
        out._damp_fn.cutoff_radii.copy_(damp.cutoff_radii.detach().to("cpu", torch.float32))
        out._k1, out._k2, out._k3 = ref_pot._k1, ref_pot._k2, ref_pot._k3
    else:
        raise ValueError(f"potential {name} has no CUDA counterpart (RepulsionXTB, RepulsionZBL, LennardJones, "
                         "RepulsionLJ, DispersionLJ, FixedCoulomb, FixedMNOK and TwoBodyDispersionD3 do)")
    out._enabled = bool(ref_pot._enabled)
    return out
