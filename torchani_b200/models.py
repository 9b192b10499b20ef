"""ANI model assembly with the interface of ``torchani.arch.ANI`` / ``torchani.models``.

``ANI.forward((species, coords), cell, pbc, charge, atomic, ensemble_values)`` mirrors
arch.py:302-349 and returns ``SpeciesEnergies``; energies carry an autograd edge to ``coords``,
so ``torch.autograd.grad(energy, coords)`` (ase.py:159-162, grad.py:57-62) works unchanged.  For
the plain energy(+force) call the whole step runs through the fused ``Engine`` (one launch
sequence, forces produced in the forward pass and stashed for backward); ``atomic=True`` /
``ensemble_values=True`` use the same engine outputs.

Pretrained ANI parameters are not shipped (the reference downloads them, arch.py:1185-1220):
``ANI2x()`` / ``ANI1x()`` build the published architectures with seeded random weights, and
``load_state_dict`` accepts the reference's state-dict keys.  ``from_torchani(model)`` converts
an existing ``torchani.arch.ANI`` instance (weights, AEV constants, self energies).
"""
from __future__ import annotations

import math
import typing as tp

import torch
from torch import Tensor

from . import _lib
from .aev import AEVComputer
from .engine import Engine, StepResult, check_pair_cutoff
from .neighbors import (CellList, Neighbors, NeighborlistArg, _validate_inputs, discard_outside_cutoff,
                        effective_periodic_cell, narrow_down, supercell_for_thin_cell)
from .nn import (ANINetworks, ATOMIC_NUMBER, AtomicContainer, AtomicNetwork, Ensemble, SpeciesConverter,
                 SpeciesEnergies, fall_back_to_bf16x3)
from .potentials import PairPotential, TwoBodyDispersionD3
from . import potentials as _potentials

SYMBOLS_1X = ("H", "C", "N", "O")
SYMBOLS_2X = ("H", "C", "N", "O", "S", "F", "Cl")
# constants.py:88-96 (wb97x-631gd ground-state atomic energies, Hartree)
GSAES_WB97X_631GD = {"H": -0.4993212, "C": -37.8338334, "N": -54.5732825, "O": -75.0424519,
                     "S": -398.0814169, "F": -99.6949007, "Cl": -460.1167008}


class SpeciesForces(tp.NamedTuple):        # tuples.py of the reference
    species: Tensor
    energies: Tensor
    forces: Tensor


class SpeciesEnergiesQBC(tp.NamedTuple):
    species: Tensor
    energies: Tensor
    qbcs: Tensor


class AtomicStdev(tp.NamedTuple):
    species: Tensor
    energies: Tensor
    stdev_atomic_energies: Tensor


class ForceMagnitudes(tp.NamedTuple):
    species: Tensor
    magnitudes: Tensor


class ForceStdev(tp.NamedTuple):
    species: Tensor
    magnitudes: Tensor
    relative_stdev: Tensor
    relative_range: Tensor


class SelfEnergy(torch.nn.Module):
    """Constant per-element energies (sae.py:16-64).  The fused engine adds them in float64."""

    def __init__(self, symbols: tp.Sequence[str], self_energies: tp.Sequence[float]):
        super().__init__()
        if len(symbols) != len(self_energies):
            raise ValueError("one self energy per symbol is required")
        self.symbols = tuple(symbols)
        self.register_buffer("self_energies", torch.tensor(list(self_energies), dtype=torch.float64))
        self._enabled = True

    @classmethod
    def with_gsaes(cls, symbols: tp.Sequence[str], functional: str = "wb97x", basis_set: str = "631gd"):
        if (functional.lower(), basis_set.lower()) != ("wb97x", "631gd"):
            raise ValueError("only the wb97x-631gd GSAEs are bundled")
        return cls(symbols, [GSAES_WB97X_631GD[s] for s in symbols])

    def forward(self, elem_idxs: Tensor, atomic: bool = False) -> Tensor:
        e = self.self_energies.to(elem_idxs.device)[elem_idxs.clamp(min=0)].masked_fill(elem_idxs == -1, 0.0)
        return e if atomic else e.sum(dim=-1)


class _FusedEnergy(torch.autograd.Function):
    """coords -> (energies (C,), atomic NN energies (C, A), member atomic (M, C, A)); the
    gradient of the ensemble-mean energy is produced by the forward launch sequence.

    Under ``create_graph=True`` the backward returns that gradient through ``_HessianProduct``: it re-runs the step on
    the saved coordinates (the workspace may have been reused since the forward), computes the analytic Hessian once
    (``Engine.hessian``) and differentiates the gradient as the product with it."""

    @staticmethod
    def forward(ctx, coords: Tensor, species: Tensor, cell: tp.Optional[Tensor], pbc: bool, engine: Engine,
                want_grad: bool):
        res: StepResult = engine.step(species, coords.detach(), cell, pbc, want_grad=want_grad, check=True)
        ctx.want_grad = want_grad
        if want_grad:
            ctx.save_for_backward(res.grad.clone(), coords)
            ctx.step_args = (species, cell, pbc, engine)
        ctx.mark_non_differentiable(res.member_atomic)
        return res.energies.clone(), res.atomic_energies.clone(), res.member_atomic.clone()

    @staticmethod
    def backward(ctx, g_energy, g_atomic, g_member):
        if not ctx.want_grad:
            raise RuntimeError("energies were computed without forces (coords.requires_grad was False)")
        grad, coords = ctx.saved_tensors
        if g_atomic is not None and bool((g_atomic != 0).any()):
            raise NotImplementedError("per-atom upstream gradients are not supported by the fused engine; "
                                      "use AEVComputer + Ensemble modules directly")
        if g_energy is None:
            return None, None, None, None, None, None
        if torch.is_grad_enabled():   # create_graph=True: a gradient that can be differentiated again
            species, cell, pbc, engine = ctx.step_args
            hess = _step_hessian(engine, species, coords, cell, pbc)
            return _HessianProduct.apply(coords, g_energy, grad, hess), None, None, None, None, None
        return grad * g_energy.to(grad.dtype).view(-1, 1, 1), None, None, None, None, None


def _step_hessian(engine: Engine, species: Tensor, coords: Tensor, cell: tp.Optional[Tensor], pbc: bool) -> Tensor:
    """(C, 3A, 3A) float32 Hessian of one step on ``coords`` (eager launches; open systems only)."""
    if pbc:
        raise ValueError("Hessians of periodic systems are not supported (open molecules and conformer batches only)")
    engine.step(species, coords.detach(), cell, False, want_grad=True, check=True)
    return engine.hessian(engine.workspace(*species.shape))


class _HessianProduct(torch.autograd.Function):
    """(coords, g_energy) -> g_energy * dE/dcoords with the step's gradient and Hessian precomputed: the backward is
    the batched product with the Hessian (one per conformer), so every component of a Hessian taken through autograd
    reuses the one Hessian computation of the step."""

    @staticmethod
    def forward(ctx, coords: Tensor, g_energy: Tensor, grad: Tensor, hess: Tensor):
        ctx.save_for_backward(g_energy, grad, hess)
        ctx.coords_dtype = coords.dtype
        return grad * g_energy.to(grad.dtype).view(-1, 1, 1)

    @staticmethod
    def backward(ctx, v: Tensor):
        if torch.is_grad_enabled():
            raise NotImplementedError("third derivatives of the fused step are not supported")
        g_energy, grad, hess = ctx.saved_tensors
        n_conf = v.shape[0]
        hv = torch.bmm(hess, v.reshape(n_conf, -1, 1).to(hess.dtype)).view_as(v)
        d_coords = hv * g_energy.to(hv.dtype).view(-1, 1, 1)
        d_g = (grad.to(v.dtype) * v).sum((1, 2)).to(g_energy.dtype)
        return d_coords.to(ctx.coords_dtype), d_g, None, None


def _per_conformer(cell: tp.Optional[Tensor]) -> bool:
    """One cell per conformer, (C, 3, 3): a periodic batch in grid mode 3."""
    return cell is not None and cell.dim() == 3


class ANI(torch.nn.Module):
    r"""ANI-style neural network interatomic potential (interface of arch.py:90-381)."""

    def __init__(self, symbols: tp.Sequence[str], aev_computer: AEVComputer, neural_networks: AtomicContainer,
                 energy_shifter: SelfEnergy, periodic_table_index: bool = True,
                 potentials: tp.Optional[tp.Mapping[str, PairPotential]] = None):
        """``potentials``: pair potentials evaluated next to the networks (arch.py:116-127), e.g.
        ``{"repulsion_xtb": RepulsionXTB(...)}``.  The repulsion terms (xTB, ZBL) run inside the fused step over the
        AEV's own neighbour list, so each needs ``cutoff <=`` the radial AEV cutoff; the LJ and Coulomb terms run a
        neighbour search of their own cutoff over the step's bucket grid, at any cutoff (``math.inf``: open systems
        only); a ``TwoBodyDispersionD3`` (at most one, any name, a finite cutoff) runs its own neighbour search too.
        ``self.cutoff`` is the largest cutoff of the networks and the potentials (arch.py:125)."""
        super().__init__()
        self.register_buffer("atomic_numbers", torch.tensor([ATOMIC_NUMBER[e] for e in symbols], dtype=torch.long))
        assert len(energy_shifter.self_energies) == len(symbols)
        assert aev_computer.num_species == len(symbols)
        assert neural_networks.num_species == len(symbols)
        self.symbols = tuple(symbols)
        self.aev_computer = aev_computer
        self.neural_networks = neural_networks
        self.neighborlist = aev_computer.neighborlist
        self.energy_shifter = energy_shifter
        self.species_converter = SpeciesConverter(symbols)
        self.cutoff = aev_computer.radial.cutoff
        n_d3 = 0
        for name, pot in (potentials or {}).items():
            if name == "nnp" or not isinstance(pot, PairPotential):
                raise ValueError(f"potential {name!r}: expected a torchani_b200.potentials.PairPotential under a name "
                                 "other than 'nnp' (the networks)")
            if tuple(pot.symbols) != tuple(symbols):
                raise ValueError(f"potential {name!r} was built for other symbols")
            if isinstance(pot, TwoBodyDispersionD3):
                n_d3 += 1
                if pot.cutoff == math.inf:
                    raise ValueError(f"potential {name!r}: D3 in a model needs a finite cutoff (its neighbour search "
                                     "runs on the step's bucket grid)")
            elif pot.kind in (0, 1):
                check_pair_cutoff(pot.cutoff, self.cutoff)
        if n_d3 > 1:
            raise ValueError("a model takes at most one TwoBodyDispersionD3")
        self.cutoff = max([self.cutoff] + [float(p.cutoff) for p in (potentials or {}).values()])
        # (the networks are the "nnp" potential of the reference and come first; they stay direct attributes here)
        self.potentials = torch.nn.ModuleDict(dict(potentials or {}))
        self.periodic_table_index = periodic_table_index
        self._engine: tp.Optional[Engine] = None
        self._engine_key: tp.Any = None

    # -- reference conveniences (arch.py:132-146,253-275) ----------------------------------
    def set_active_members(self, idxs: tp.List[int]) -> None:
        self.neural_networks.set_active_members(idxs)

    def set_strategy(self, strategy: str) -> None:
        self.aev_computer.set_strategy(strategy)

    def __len__(self) -> int:
        return self.neural_networks.get_active_members_num()

    def __getitem__(self, idx: int) -> "ANI":
        import copy
        nets = self.neural_networks
        if not isinstance(nets, Ensemble):
            raise ValueError("Only ensembles can be indexed")
        return ANI(self.symbols, copy.deepcopy(self.aev_computer), copy.deepcopy(nets[idx]),
                   copy.deepcopy(self.energy_shifter), self.periodic_table_index,
                   {k: copy.deepcopy(p) for k, p in self.potentials.items()})

    def set_enabled(self, key: str, val: bool = True) -> None:
        """arch.py:136-142: switch the energy shifter or a pair potential on or off."""
        if key == "energy_shifter":
            self.energy_shifter._enabled = val
        else:
            self.potentials[key]._enabled = val

    def _enabled_potentials(self) -> tp.List[PairPotential]:
        return [p for p in self.potentials.values() if p._enabled]

    def _enabled_dispersion(self) -> tp.Optional[TwoBodyDispersionD3]:
        d3 = [p for p in self._enabled_potentials() if isinstance(p, TwoBodyDispersionD3)]
        return d3[0] if d3 else None

    def to_infer_model(self, use_mnp: bool = False) -> "ANI":
        return self

    def ase(self, overwrite: bool = False, stress_kind: str = "scaling", jit: bool = False, skin: float = 0.0):
        """An ASE ``Calculator`` that uses this model (arch.py:219-241).  ``jit`` is accepted for interface
        compatibility and ignored (the hot path is a CUDA graph already)."""
        from .ase import Calculator
        return Calculator(self, overwrite=overwrite, stress_kind=stress_kind, skin=skin)

    # -- fused engine ----------------------------------------------------------------------
    def engine(self, device: torch.device) -> Engine:
        # (the layer-1 operands are packed in the AEV kernels' internal column order: 32-aligned angular block)
        c = self.aev_computer.constants
        self.neural_networks._radial_len = c.num_species * len(c.shf_r)
        nets = self.neural_networks.packed(device)
        shifter = self.energy_shifter
        # the engine bakes the self energies and the pair-potential tables in: key it on their values (edits,
        # `_enabled` toggles)
        pairs = [p.params() for p in self._enabled_potentials() if not isinstance(p, TwoBodyDispersionD3)]
        d3 = self._enabled_dispersion()
        disp = None if d3 is None else (d3.params(), d3.tables(device))
        key = (str(device), id(nets), bool(shifter._enabled), shifter.self_energies._version,
               shifter.self_energies.data_ptr(), tuple(bytes(p) for p in pairs))
        if disp is not None:   # (the device tables are rebuilt when the reference tables change: key on them too)
            key = key + (bytes(disp[0]), disp[1].data_ptr())
        if self._engine is None or self._engine_key != key:
            sae = self.energy_shifter.self_energies.tolist() if self.energy_shifter._enabled else None
            kw = {} if disp is None else {"dispersion": disp}
            self._engine = Engine(self.aev_computer.constants, nets, sae, nbr_cap=self.aev_computer.nbr_cap,
                                  pairs=pairs, **kw)
            self._engine_key = key
        return self._engine

    def _guarded(self, fn: tp.Callable[[], tp.Any]) -> tp.Any:
        """Run an engine call; if a value left the range of the 2 x fp16 operand pieces
        (ANI_STATUS_OPERAND_RANGE), switch the networks to the 3 x bfloat16 build of the library -- same kernels,
        6 instead of 4 bytes per operand element, no range limit -- and redo the call."""
        try:
            return fn()
        except _lib.OperandRangeError:
            if not fall_back_to_bf16x3(self.neural_networks):
                raise
            return fn()

    @staticmethod
    def _check_inputs(elem_idxs: Tensor, coords: Tensor, charge: int = 0) -> None:
        assert elem_idxs.dim() == 2
        assert coords.shape == (elem_idxs.shape[0], elem_idxs.shape[1], 3)
        assert charge == 0, "Model only supports neutral molecules"

    def forward(self, species_coordinates: tp.Tuple[Tensor, Tensor], cell: tp.Optional[Tensor] = None,
                pbc: tp.Optional[Tensor] = None, charge: int = 0, atomic: bool = False,
                ensemble_values: bool = False) -> SpeciesEnergies:
        species, coords = species_coordinates
        self._check_inputs(species, coords, charge)
        elem_idxs = self.species_converter(species, nop=not self.periodic_table_index)
        _validate_inputs(self.cutoff, elem_idxs, coords, cell, pbc, conformer_cells=True)
        # (a periodic batch -- C conformers in one shared cell, or one (C, 3, 3) cell per conformer -- is one engine
        # step: one sub-grid per conformer)
        # (with a cell-list neighbour list the reference raises "Cell is too small" instead, neighbors.py:402-403: so
        # does the engine; all_pairs / adaptive models take the supercell route -- for a shared cell only: a thin cell
        # of one conformer of a (C, 3, 3) batch raises too)
        sup = None if (isinstance(self.neighborlist, CellList) or _per_conformer(cell)) else \
            supercell_for_thin_cell(species, coords, cell, pbc, self.cutoff)
        if sup is not None:
            # periodic cell thinner than the cutoff (neighbors.py:245-275): evaluate a supercell of R translation-
            # equivalent copies; atomic energies of the original atoms are the first A, the energy is 1/R of the whole
            sp_rep, co_rep, cell_rep, R = sup
            a = elem_idxs.shape[1]
            if atomic:
                out = self((sp_rep, co_rep), cell_rep, pbc, charge, True, ensemble_values).energies[..., :a]
            else:
                out = self((sp_rep, co_rep), cell_rep, pbc, charge, False, ensemble_values).energies / R
            return SpeciesEnergies(elem_idxs, out)
        cell = effective_periodic_cell(coords, cell, pbc, self.cutoff)   # PBC in some directions only
        e, e_atomic, e_member = self._guarded(lambda: _FusedEnergy.apply(
            coords, elem_idxs, cell, pbc is not None, self.engine(coords.device), bool(coords.requires_grad)))
        energies: Tensor
        if ensemble_values:
            active = self.neural_networks.active_members_idxs
            energies = e_member[active].to(coords.dtype)
            if self.energy_shifter._enabled:
                energies = energies + self.energy_shifter(elem_idxs, atomic=True).to(coords.dtype)
            if not atomic:
                energies = energies.sum(-1)
        elif atomic:
            energies = e_atomic.to(coords.dtype)
            if self.energy_shifter._enabled:
                energies = energies + self.energy_shifter(elem_idxs, atomic=True).to(coords.dtype)
        else:
            energies = e.to(coords.dtype)
        return SpeciesEnergies(elem_idxs, energies)

    # -- entry point with a caller-supplied neighbour list (arch.py:354-381, potentials/nnp.py:20-32) ----
    def compute_from_neighbors(self, elem_idxs: Tensor, coords: Tensor, neighbors: Neighbors, charge: int = 0,
                               atomic: bool = False, ensemble_values: bool = False) -> Tensor:
        """Energies from element indices, coordinates and the result of a neighbour-list calculation
        (pairs beyond the radial cutoff are discarded first, as ``discard_outside_cutoff`` does for
        every potential of the reference).  Shape: (C,), (C, A), (M, C) or (M, C, A)."""
        self._check_inputs(elem_idxs, coords, charge)
        neighbors = discard_outside_cutoff(neighbors, self.cutoff)
        rcr = self.aev_computer.radial.cutoff
        aevs = self.aev_computer.compute_from_neighbors(
            elem_idxs, coords, neighbors if self.cutoff <= rcr else discard_outside_cutoff(neighbors, rcr))
        energies = self.neural_networks(elem_idxs, aevs, atomic, ensemble_values)
        for pot in self._enabled_potentials():   # (C,) / (C, A): broadcast over the members, arch.py:365-378
            energies = energies + pot.compute_from_neighbors(
                elem_idxs, coords, discard_outside_cutoff(neighbors, pot.cutoff), charge, atomic,
                ensemble_values).to(energies.dtype)
        if self.energy_shifter._enabled:
            energies = energies + self.energy_shifter(elem_idxs, atomic=atomic).to(energies.dtype)
        return energies

    def compute_from_external_neighbors(self, species: Tensor, coords: Tensor, neighbor_idxs: Tensor,
                                        shifts: tp.Optional[Tensor], charge: int = 0, atomic: bool = False,
                                        ensemble_values: bool = False) -> Tensor:
        r"""Entry point for an EXTERNAL neighbour list (arch.py:171-206), e.g. the Verlet list of an MD engine:
        ``neighbor_idxs (2, P)`` candidate pairs (possibly built with a skin) and their lattice ``shifts (P, 3)``
        (None without PBC); pairs beyond the cutoff and pairs with dummy atoms are screened out first
        (``narrow_down``).  IMPORTANT, as in the reference: coords must be mapped to the central cell."""
        self._check_inputs(species, coords, charge)
        elem_idxs = self.species_converter(species, nop=not self.periodic_table_index)
        neighbors = narrow_down(self.cutoff, elem_idxs, coords, neighbor_idxs, shifts)
        return self.compute_from_neighbors(elem_idxs, coords, neighbors, charge, atomic, ensemble_values)

    def compute_from_full_neighborlist(self, species: Tensor, coords: Tensor, ilist_unique: Tensor, jlist: Tensor,
                                       numneigh: Tensor, atomic: bool = False, ensemble_values: bool = False) -> Tensor:
        r"""Energies of the LOCAL atoms (``ilist_unique``) of a local + ghost atom set with the full neighbour list
        of an MD engine (LAMMPS ``ilist / jlist / numneigh``; csrc/cuaev.cpp:225-246 + the network pass of
        potentials/nnp.py:20-32).  Ghost atoms contribute as neighbours only: their energies are masked out, and
        ``torch.autograd.grad`` of the result gives dE/dx for local and ghost coordinates alike."""
        self._check_inputs(species, coords, 0)
        if self._enabled_potentials():
            raise NotImplementedError("pair potentials are not evaluated over a full neighbour list with ghost atoms; "
                                      "disable them (set_enabled) or use compute_from_external_neighbors")
        elem_idxs = self.species_converter(species, nop=not self.periodic_table_index)
        aevs = self.aev_computer.compute_from_full_neighborlist(elem_idxs, coords, ilist_unique, jlist, numneigh)
        local = torch.zeros_like(elem_idxs, dtype=torch.bool).view(-1)
        local[ilist_unique.long()] = True
        masked = torch.where(local.view_as(elem_idxs), elem_idxs, torch.full_like(elem_idxs, -1))
        energies = self.neural_networks(masked, aevs, atomic, ensemble_values)
        if self.energy_shifter._enabled:
            energies = energies + self.energy_shifter(masked, atomic=atomic).to(energies.dtype)
        return energies

    # -- ensemble statistics (arch.py:385-576; query-by-committee active learning) ---------------------
    def atomic_energies(self, species_coordinates: tp.Tuple[Tensor, Tensor], cell: tp.Optional[Tensor] = None,
                        pbc: tp.Optional[Tensor] = None, charge: int = 0,
                        ensemble_values: bool = False) -> SpeciesEnergies:
        return self(species_coordinates, cell, pbc, charge, True, ensemble_values)

    def members_forces(self, species_coordinates: tp.Tuple[Tensor, Tensor], cell: tp.Optional[Tensor] = None,
                       pbc: tp.Optional[Tensor] = None, charge: int = 0) -> SpeciesForces:
        """Energies (M, C) and forces (M, C, A, 3) of every active ensemble member (arch.py:403-436).
        The reference differentiates each member's energy by autograd; here ONE pass of the engine
        (``Engine.step_members``, the query-by-committee step): the MLP launch writes one dE_m/dAEV slab per member
        instead of their sum, and ONE force-kernel launch contracts all of them, inside a captured CUDA graph."""
        species, coords = species_coordinates
        self._check_inputs(species, coords, charge)
        elem_idxs = self.species_converter(species, nop=not self.periodic_table_index)
        _validate_inputs(self.cutoff, elem_idxs, coords, cell, pbc, conformer_cells=True)
        cell = effective_periodic_cell(coords, cell, pbc, self.cutoff)

        def run():
            eng = self.engine(coords.device)
            out = eng.step_members(elem_idxs, coords.detach(), cell, pbc is not None)
            eng.check_status()
            return out
        e_m, g_m = self._guarded(run)
        return SpeciesForces(elem_idxs, e_m.to(coords.dtype), -g_m)

    def energies_qbcs(self, species_coordinates: tp.Tuple[Tensor, Tensor], cell: tp.Optional[Tensor] = None,
                      pbc: tp.Optional[Tensor] = None, unbiased: bool = True, charge: int = 0) -> SpeciesEnergiesQBC:
        """Mean energies and query-by-committee factors std_m(E_m) / sqrt(num_atoms) (arch.py:439-485)."""
        elem_idxs, energies = self(species_coordinates, cell, pbc, charge, False, True)
        if energies.shape[0] == 1:
            qbc = torch.zeros_like(energies).squeeze(0)
        else:
            qbc = energies.std(0, unbiased=unbiased)
        qbc = qbc / (elem_idxs >= 0).sum(dim=1, dtype=energies.dtype).sqrt()
        return SpeciesEnergiesQBC(elem_idxs, energies.mean(dim=0), qbc)

    def atomic_stdev(self, species_coordinates: tp.Tuple[Tensor, Tensor], cell: tp.Optional[Tensor] = None,
                     pbc: tp.Optional[Tensor] = None, charge: int = 0, ensemble_values: bool = False,
                     unbiased: bool = True) -> AtomicStdev:
        elem_idxs, energies = self(species_coordinates, cell, pbc, charge, True, True)
        stdev = torch.zeros_like(energies).squeeze(0) if energies.shape[0] == 1 else energies.std(0, unbiased=unbiased)
        if not ensemble_values:
            energies = energies.mean(0)
        return AtomicStdev(elem_idxs, energies, stdev)

    def force_magnitudes(self, species_coordinates: tp.Tuple[Tensor, Tensor], cell: tp.Optional[Tensor] = None,
                         pbc: tp.Optional[Tensor] = None, ensemble_values: bool = False) -> ForceMagnitudes:
        species, _, members_forces = self.members_forces(species_coordinates, cell, pbc)
        magnitudes = members_forces.norm(dim=-1)
        if not ensemble_values:
            magnitudes = magnitudes.mean(0)
        return ForceMagnitudes(species, magnitudes)

    def force_qbc(self, species_coordinates: tp.Tuple[Tensor, Tensor], cell: tp.Optional[Tensor] = None,
                  pbc: tp.Optional[Tensor] = None, ensemble_values: bool = False, unbiased: bool = True) -> ForceStdev:
        """Mean force magnitudes, relative std and relative range across the ensemble (arch.py:543-576)."""
        species, mags = self.force_magnitudes(species_coordinates, cell, pbc, True)
        eps = 1e-8
        mean_mags = mags.mean(0)
        if mags.shape[0] == 1:
            relative_std = torch.zeros_like(mags).squeeze(0)
            relative_range = torch.ones_like(mags).squeeze(0)
        else:
            relative_std = (mags.std(0, unbiased=unbiased) + eps) / (mean_mags + eps)
            relative_range = ((mags.max(dim=0).values - mags.min(dim=0).values) + eps) / (mean_mags + eps)
        if not ensemble_values:
            mags = mean_mags
        return ForceStdev(species, mags, relative_std, relative_range)

    def energies_f64(self, species_coordinates: tp.Tuple[Tensor, Tensor], cell: tp.Optional[Tensor] = None,
                     pbc: tp.Optional[Tensor] = None) -> Tensor:
        """Total energies in float64 as accumulated on the device (the float32 tensor returned by
        ``forward`` loses ~3e-3 Ha at |E| ~ 2.5e4 Ha, see BASELINE.md)."""
        species, coords = species_coordinates
        elem_idxs = self.species_converter(species, nop=not self.periodic_table_index)
        if _per_conformer(cell):
            _validate_inputs(self.cutoff, elem_idxs, coords, cell, pbc, conformer_cells=True)
        cell = effective_periodic_cell(coords, cell, pbc, self.cutoff)
        return self._guarded(lambda: self.engine(coords.device).step(
            elem_idxs, coords.detach(), cell, pbc is not None, want_grad=False, check=True).energies.clone())

    def energies_and_forces(self, species: Tensor, coords: Tensor, cell: tp.Optional[Tensor] = None,
                            pbc: tp.Optional[Tensor] = None) -> tp.Tuple[Tensor, Tensor]:
        """grad.py:263-290 without the autograd round trip: (energies f64 (C,), forces f32 (C,A,3))."""
        elem_idxs = self.species_converter(species, nop=not self.periodic_table_index)
        if _per_conformer(cell):
            _validate_inputs(self.cutoff, elem_idxs, coords, cell, pbc, conformer_cells=True)
        cell = effective_periodic_cell(coords, cell, pbc, self.cutoff)
        res = self._guarded(lambda: self.engine(coords.device).step(
            elem_idxs, coords.detach(), cell, pbc is not None, want_grad=True, check=True))
        return res.energies.clone(), -res.grad

    def energies_forces_hessians(self, species: Tensor, coords: Tensor) -> tp.Tuple[Tensor, Tensor, Tensor]:
        """(energies f64 (C,), forces f32 (C, A, 3), Hessians d^2E/dx^2 f32 (C, 3A, 3A)) of open molecules or conformer
        batches (grad.py:239-260 without the autograd round trip): one step with gradients and its analytic Hessian
        (``Engine.hessian``).  Padding atoms get zero rows and columns.  Periodic input, D3, Lennard-Jones and Coulomb
        terms are not supported; the xTB and ZBL repulsion terms are included.  A charge model gives the Hessian of its
        energy (the charges are not differentiated)."""
        elem_idxs = self.species_converter(species, nop=not self.periodic_table_index)
        _validate_inputs(self.cutoff, elem_idxs, coords, None, None)

        def run():
            eng = self.engine(coords.device)
            res = eng.step(elem_idxs, coords.detach(), None, False, want_grad=True, check=True)
            e, f = res.energies.clone(), -res.grad
            return e, f, eng.hessian(eng.workspace(*elem_idxs.shape))
        return self._guarded(run)

    def energies_forces_stress(self, species: Tensor, coords: Tensor, cell: Tensor,
                               pbc: tp.Optional[Tensor] = None) -> tp.Tuple[Tensor, Tensor, Tensor]:
        """(energies f64 (C,), forces f32 (C, A, 3), stress f64 in Hartree/A^3) of periodic systems in one cell: (3, 3)
        for one system, (C, 3, 3) for a batch of C conformers.  The stress is the "f dot r" virial of ase.py:164-168 -- sum over the pairs of
        (dE/dDelta)_a Delta_b, accumulated by the force kernel -- divided by the cell volume; it equals
        the strain derivative dE/d(scaling)/V of ase.py:170-173 and, unlike that one, does not need the
        atoms to be wrapped into the cell.  With one cell per conformer, ``cell`` (C, 3, 3), conformer c's stress is
        its virial over the volume of its own cell."""
        elem_idxs = self.species_converter(species, nop=not self.periodic_table_index)
        if _per_conformer(cell):   # (periodic in all directions whether or not pbc is given)
            full = torch.ones(3, dtype=torch.bool, device=coords.device) if pbc is None else pbc
            _validate_inputs(self.cutoff, elem_idxs, coords, cell, full, conformer_cells=True)
        res = self._guarded(lambda: self.engine(coords.device).step(
            elem_idxs, coords.detach(), cell, True, want_grad=True, want_virial=True, check=True))
        volume = torch.det(cell.detach().double()).abs()
        if _per_conformer(cell):
            volume = volume.view(-1, 1, 1)
            if res.virial.dim() == 2:   # a batch of one conformer
                return res.energies.clone(), -res.grad, res.virial.unsqueeze(0) / volume
        return res.energies.clone(), -res.grad, res.virial / volume

    # -- state dicts of the reference (arch.py:278-290) ------------------------------------
    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs) -> None:
        for old in list(state_dict.keys()):
            new = old.replace("potentials.nnp.aev_computer.", "aev_computer.")
            new = new.replace("potentials.nnp.neural_networks.", "neural_networks.")
            if new.startswith(prefix + "potentials.0."):   # legacy numbered potentials, arch.py:278-290
                new = new.replace("potentials.0.", "potentials.dispersion_d3.", 1)
            elif new.startswith(prefix + "potentials.1."):
                new = new.replace("potentials.1.", "potentials.repulsion_xtb.", 1)
            elif new.startswith(prefix + "potentials.2."):
                new = new.replace("potentials.2.", "", 1)
            new = new.replace("radial_terms", "radial").replace("angular_terms", "angular")
            new = new.replace(".EtaR", ".eta").replace(".ShfR", ".shifts").replace(".EtaA", ".eta")
            new = new.replace(".Zeta", ".zeta").replace(".ShfA", ".shifts").replace(".ShfZ", ".sections")
            if new != old:
                state_dict[new] = state_dict.pop(old).reshape(-1) if any(
                    new.endswith(k) for k in (".eta", ".zeta", ".shifts", ".sections")) else state_dict.pop(old)
        super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)


def _assemble(symbols, aev_ctor, net_ctor, ensemble_size: int, neighborlist: NeighborlistArg,
              periodic_table_index: bool, seed: tp.Optional[int], device) -> ANI:
    if seed is not None:
        torch.manual_seed(seed)
    aevc = aev_ctor(num_species=len(symbols), neighborlist=neighborlist)
    members = [net_ctor(symbols, aevc.out_dim) for _ in range(ensemble_size)]
    nets: AtomicContainer = Ensemble(members) if ensemble_size > 1 else members[0]
    model = ANI(symbols, aevc, nets, SelfEnergy.with_gsaes(symbols), periodic_table_index)
    model.requires_grad_(False)
    return model.to(device) if device is not None else model


def ANI2x(model_index: tp.Optional[int] = None, neighborlist: NeighborlistArg = "cell_list",
          periodic_table_index: bool = True, device=None, seed: tp.Optional[int] = 0) -> ANI:
    """ANI-2x architecture (models.py:165-198): 7 elements, 1008-dim AEV, 8-member ensemble.
    Weights are seeded random (no download in this environment)."""
    model = _assemble(SYMBOLS_2X, AEVComputer.like_2x, ANINetworks.like_2x, 8, neighborlist,
                      periodic_table_index, seed, device)
    return model if model_index is None else model[model_index]


def ANI1x(model_index: tp.Optional[int] = None, neighborlist: NeighborlistArg = "cell_list",
          periodic_table_index: bool = True, device=None, seed: tp.Optional[int] = 0) -> ANI:
    """ANI-1x architecture (models.py:105-131): 4 elements, 384-dim AEV, 8-member ensemble."""
    model = _assemble(SYMBOLS_1X, AEVComputer.like_1x, ANINetworks.like_1x, 8, neighborlist,
                      periodic_table_index, seed, device)
    return model if model_index is None else model[model_index]


def from_weight_lists(kind: str, weights, device=None, neighborlist: NeighborlistArg = "cell_list",
                      periodic_table_index: bool = False) -> ANI:
    """Build an ANI-1x / ANI-2x shaped model from ``weights[member][symbol] = [(W, b) x 4]``."""
    symbols = SYMBOLS_2X if kind == "2x" else SYMBOLS_1X
    aev_ctor = AEVComputer.like_2x if kind == "2x" else AEVComputer.like_1x
    net_ctor = ANINetworks.like_2x if kind == "2x" else ANINetworks.like_1x
    model = _assemble(symbols, aev_ctor, net_ctor, len(weights), neighborlist, periodic_table_index, None, None)
    members = model.neural_networks.member_networks()
    with torch.no_grad():
        for net, w_m in zip(members, weights):
            for s in symbols:
                for (w_dst, b_dst), (w, b) in zip(net.atomics[s].linear_pairs(), w_m[s]):
                    w_dst.copy_(w)
                    b_dst.copy_(b)
    return model.to(device) if device is not None else model


def aev_computer_from_torchani(aevr, neighborlist: NeighborlistArg = "cell_list") -> AEVComputer:
    """``torchani.aev.AEVComputer`` (standard ANIRadial / ANIAngular terms, cosine or smooth cutoff:
    what its own ``_check_cuaev_avail`` accepts, aev/_computer.py:151-168) -> the CUDA module with the
    same constants."""
    cutoff_fn = getattr(aevr, "_cuaev_cutoff_fn", "") or getattr(aevr.radial.cutoff_fn, "_cuaev_name", "") or ""
    if cutoff_fn not in ("cosine", "smooth"):
        raise ValueError("only the cosine and smooth(order=2, eps=1e-10) cutoffs are supported")
    return AEVComputer.from_constants(
        aevr.radial.cutoff, aevr.angular.cutoff, float(aevr.radial.eta), aevr.radial.shifts.tolist(),
        float(aevr.angular.eta), float(aevr.angular.zeta), aevr.angular.shifts.tolist(),
        aevr.angular.sections.tolist(), aevr.num_species, cutoff_fn=cutoff_fn, neighborlist=neighborlist)


def networks_from_torchani(netr) -> AtomicContainer:
    """``torchani.nn.Ensemble`` / ``ANINetworks`` / ``BmmEnsemble`` (nn/_containers.py:319-660,
    nn/_infer.py:61-216) -> the CUDA container with the same weights, activation and active members: CELU networks
    with biases (ANI-1x / 2x) or GELU networks without (ANI-2xr / 2dr, ``simple_ani``)."""
    first = next(iter(netr.atomics.values())) if hasattr(netr, "atomics") else None
    # (BmmEnsemble does not carry atomic_numbers: the keys of `atomics` are the symbols everywhere)
    symbols = tuple(netr.atomics.keys()) if first is not None else tuple(netr.members[0].atomics.keys())
    per_member: tp.List[tp.Dict[str, tp.List[tp.Tuple[Tensor, tp.Optional[Tensor]]]]] = []
    if hasattr(netr, "members"):
        activation = netr.members[0].atomics[symbols[0]].activation
        for rm in netr.members:
            per_member.append({s: [(l.weight, l.bias) for l in list(rm.atomics[s].layers) + [rm.atomics[s].final_layer]]
                               for s in symbols})
    elif first is not None and hasattr(first, "_num_batched_networks"):
        # BmmAtomicNetwork: weights stacked as (members, in, out), biases (members, 1, out); _beta == 0: no bias
        activation = first.activation
        for m in range(int(first._num_batched_networks)):
            per_member.append({s: [(l.weight[m].t(), l.bias[m, 0] if l._beta else None)
                                   for l in list(netr.atomics[s].layers) + [netr.atomics[s].final_layer]]
                               for s in symbols})
    else:
        activation = first.activation
        per_member.append({s: [(l.weight, l.bias) for l in list(netr.atomics[s].layers) + [netr.atomics[s].final_layer]]
                           for s in symbols})
    members = []
    for layers in per_member:
        mods = {}
        for s in symbols:
            dims = [layers[s][0][0].shape[1]] + [w.shape[0] for w, _ in layers[s]]
            biases = {b is not None for _, b in layers[s]}
            if len(biases) != 1:
                raise ValueError("networks with biases in some layers only are not supported")
            an = AtomicNetwork(dims, activation, bias=biases.pop())   # raises for unsupported kinds
            with torch.no_grad():
                for (w_dst, b_dst), (w, b) in zip(an.linear_pairs(), layers[s]):
                    w_dst.copy_(w)
                    if b_dst is not None:
                        b_dst.copy_(b)
            mods[s] = an
        members.append(ANINetworks(mods))
    nets: AtomicContainer = Ensemble(members) if len(members) > 1 else members[0]
    if hasattr(netr, "members"):
        nets.set_active_members(list(netr.active_members_idxs))
    nets.requires_grad_(False)
    return nets


def charge_networks_from_torchani(netr) -> "ChargeNetworks":
    """The charge container of a reference ``SeparateChargesNNPotential`` -- ``ANINetworks`` with ``out_dim = 1`` or
    ``_ANINetworksDiscardFirstScalar`` with ``out_dim = 2`` (column 1 kept) -- as a ``ChargeNetworks`` with the same
    weights."""
    from .nn import ChargeNetworks
    if hasattr(netr, "members") or not hasattr(netr, "atomics"):
        raise ValueError("charge networks: only one ANINetworks-style container is supported (no ensembles, SingleNN "
                         "or shared networks)")
    kept = 1 if type(netr).__name__ == "_ANINetworksDiscardFirstScalar" else 0
    plain = networks_from_torchani(netr)
    return ChargeNetworks(dict(plain.atomics.items()), kept_output=kept).requires_grad_(False)


def charge_normalizer_from_torchani(norm, symbols):
    """A reference ``ChargeNormalizer`` (its non-persistent ``weights`` buffer and scaling flag) or
    ``BaseChargeNormalizer``."""
    from .electro import BaseChargeNormalizer, ChargeNormalizer
    name = type(norm).__name__
    if name == "ChargeNormalizer":
        return ChargeNormalizer(symbols, norm.weights.detach().double().cpu().tolist(),
                                bool(norm.scale_weights_by_charges_squared))
    if name == "BaseChargeNormalizer":
        return BaseChargeNormalizer()
    raise ValueError(f"charge normalizer {name!r} is not supported")


def from_torchani(ref_model, device=None) -> ANI:
    """Convert a ``torchani.arch.ANI`` instance (reference, e.g. ``torchani.models.ANI2x()``) into
    the CUDA model: same symbols, AEV constants, network weights and self energies."""
    aevr = ref_model.potentials["nnp"].aev_computer
    netr = ref_model.potentials["nnp"].neural_networks
    symbols = tuple(ref_model.symbols)
    aevc = aev_computer_from_torchani(aevr)
    nets = networks_from_torchani(netr)
    sae = SelfEnergy(symbols, ref_model.energy_shifter.self_energies.double().tolist())
    sae._enabled = bool(ref_model.energy_shifter._enabled)
    # every other potential of the reference model is converted or refused, never dropped
    extra = {}
    for name, pot in ref_model.potentials.items():
        if name == "nnp":
            continue
        try:
            extra[name] = _potentials.from_torchani(pot)
        except ValueError as exc:
            raise ValueError(f"cannot convert potential {name!r} of the reference model: {exc}; a converted model "
                             "without it would compute other energies and forces") from None
    nnp = ref_model.potentials["nnp"]
    if type(nnp).__name__ == "MergedChargesNNPotential":
        raise ValueError("merged charge networks (MergedChargesNNPotential) are not supported: their energy networks "
                         "have out_dim = 2, which the fused backward does not run")
    if hasattr(nnp, "charge_networks"):   # SeparateChargesNNPotential (arch.ANIq)
        model: ANI = ANIq(symbols, aevc, nets, sae, extra, ref_model.periodic_table_index,
                          charge_networks_from_torchani(nnp.charge_networks),
                          charge_normalizer_from_torchani(nnp.charge_normalizer, symbols))
    else:
        model = ANI(symbols, aevc, nets, sae, ref_model.periodic_table_index, extra)
    model.requires_grad_(False)
    if device is None:
        device = ref_model.energy_shifter.self_energies.device
    return model.to(device)


def accelerate_torchani_(ref_model):
    """Swap the CUDA modules INTO an existing ``torchani.arch.ANI`` in place -- its three plug-in points
    (arch.py:116-127, 208-217, 264-275): ``model.neighborlist``, ``model.potentials["nnp"].aev_computer`` and
    ``model.potentials["nnp"].neural_networks`` -- and return it.  Everything else of the reference model
    (species converter, energy shifter, extra pair potentials, its ``forward`` / ``compute_from_neighbors``
    / ``ase()``) keeps running unchanged on top of them; CUDA float32 only."""
    nnp = ref_model.potentials["nnp"]
    dev = ref_model.energy_shifter.self_energies.device
    aevc = aev_computer_from_torchani(nnp.aev_computer).to(dev)
    nets = networks_from_torchani(nnp.neural_networks).to(dev)
    nnp.aev_computer = aevc
    nnp.neural_networks = nets
    if type(nnp).__name__ == "MergedChargesNNPotential":
        raise ValueError("merged charge networks (MergedChargesNNPotential) are not supported")
    if hasattr(nnp, "charge_networks"):   # SeparateChargesNNPotential: same AEV, forward-only charge networks
        nnp.charge_networks = charge_networks_from_torchani(nnp.charge_networks).to(dev)
    ref_model.neighborlist = aevc.neighborlist
    # the pair potentials with a CUDA counterpart run through the CUDA pair-list kernels; any other potential stays as
    # it is
    for name, pot in list(ref_model.potentials.items()):
        if name != "nnp" and type(pot).__name__ in _CONVERTED_POTENTIALS:
            ref_model.potentials[name] = _DropInPairPotential(_potentials.from_torchani(pot).to(dev))
    return ref_model


_CONVERTED_POTENTIALS = ("RepulsionXTB", "RepulsionZBL", "LennardJones", "RepulsionLJ", "DispersionLJ", "FixedCoulomb",
                         "FixedMNOK", "TwoBodyDispersionD3")


class _DropInPairPotential(torch.nn.Module):
    """A CUDA pair potential in a reference model's ``potentials``: the reference's call convention
    (``compute_from_neighbors(...) -> EnergiesScalars``-like object with ``.energies``) around ``PairPotential``."""

    class _Energies(tp.NamedTuple):
        energies: Tensor
        scalars: tp.Optional[Tensor] = None

    def __init__(self, potential: PairPotential):
        super().__init__()
        self.potential = potential
        self.cutoff = potential.cutoff

    @property
    def _enabled(self) -> bool:
        return self.potential._enabled

    @_enabled.setter
    def _enabled(self, val: bool) -> None:
        self.potential._enabled = val

    def compute_from_neighbors(self, elem_idxs: Tensor, coords: Tensor, neighbors, charge: int = 0,
                               atomic: bool = False, ensemble_values: bool = False,
                               ghost_flags: tp.Optional[Tensor] = None):
        return self._Energies(self.potential.compute_from_neighbors(
            elem_idxs, coords, Neighbors(neighbors.indices, neighbors.distances, neighbors.diff_vectors), charge,
            atomic, ensemble_values, ghost_flags))


# -- charge models (arch.py:579-680, models.py:201-252) -------------------------------------------------------------
class SpeciesEnergiesAtomicCharges(tp.NamedTuple):   # tuples.py of the reference
    species: Tensor
    energies: Tensor
    atomic_charges: Tensor


class EnergiesScalars(tp.NamedTuple):
    energies: Tensor
    scalars: tp.Optional[Tensor] = None


class _FusedEnergyCharges(torch.autograd.Function):
    """``_FusedEnergy`` with the charge pass: coords -> (energies, atomic NN energies, member atomic, charges (C, A),
    dipoles (C, 3)) from one step.  Charges and dipoles carry no gradient: a nonzero upstream gradient on them
    raises."""

    @staticmethod
    def forward(ctx, coords: Tensor, species: Tensor, cell: tp.Optional[Tensor], pbc: bool, engine: Engine,
                want_grad: bool):
        res: StepResult = engine.step(species, coords.detach(), cell, pbc, want_grad=want_grad, check=True,
                                      want_charges=True)
        ws = engine.workspace(*species.shape)
        q = engine.charges_result(ws)
        ctx.want_grad = want_grad
        if want_grad:   # (what _FusedEnergy.backward reads)
            ctx.save_for_backward(res.grad.clone(), coords)
        ctx.mark_non_differentiable(res.member_atomic)
        return (res.energies.clone(), res.atomic_energies.clone(), res.member_atomic.clone(), q.charges.clone(),
                q.dipoles.clone())

    @staticmethod
    def backward(ctx, g_energy, g_atomic, g_member, g_charges, g_dipoles):
        _lib.forbid_create_graph("the fused step with charges (_FusedEnergyCharges)")
        for g in (g_charges, g_dipoles):
            if g is not None and bool((g != 0).any()):
                raise NotImplementedError("gradients of atomic charges and dipoles are not computed by the fused "
                                          "engine (the charge networks run forward only)")
        out, *_ = _FusedEnergy.backward(ctx, g_energy, g_atomic, g_member)
        return out, None, None, None, None, None


class ANIq(ANI):
    r"""ANI-style model that computes atomic charges next to the energies (interface of arch.py:579-680), with
    separate charge networks that read the energy networks' AEV (potentials/nnp.py:75-102,
    ``SeparateChargesNNPotential``).

    The charge networks run forward-only inside the fused step, on the AEVs it already built, and one more kernel
    normalises the charges per conformer (``charge_normalizer``) and forms the dipoles.  Energies and forces are those
    of an ``ANI`` with the same energy networks.  Merged charge networks (one container with ``out_dim = 2`` for
    energies and charges) are not supported."""

    def __init__(self, symbols: tp.Sequence[str], aev_computer: AEVComputer, neural_networks: AtomicContainer,
                 energy_shifter: SelfEnergy, potentials: tp.Optional[tp.Mapping[str, PairPotential]] = None,
                 periodic_table_index: bool = True, charge_networks: tp.Optional[AtomicContainer] = None,
                 charge_normalizer: tp.Optional[torch.nn.Module] = None):
        super().__init__(symbols, aev_computer, neural_networks, energy_shifter, periodic_table_index, potentials)
        from .electro import BaseChargeNormalizer, ChargeNormalizer
        from .nn import ChargeNetworks
        if charge_networks is None:
            raise ValueError("merged charge networks (MergedChargesNNPotential: energies and charges from one container "
                             "with out_dim = 2) are not supported; pass separate charge_networks")
        if not isinstance(charge_networks, ChargeNetworks):
            raise ValueError("charge_networks must be a torchani_b200.nn.ChargeNetworks (one container, no ensemble)")
        if charge_networks.num_species != len(symbols) or charge_networks.in_dim != neural_networks.member_networks()[0].in_dim:
            raise ValueError("the charge networks must take the model's elements and AEV")
        if charge_normalizer is None:
            charge_normalizer = ChargeNormalizer(symbols)
        if not isinstance(charge_normalizer, BaseChargeNormalizer):
            raise ValueError("charge_normalizer must be a torchani_b200.electro.ChargeNormalizer or BaseChargeNormalizer")
        self.charge_networks = charge_networks
        self.charge_normalizer = charge_normalizer
        # dipole frame of the step's charge pass (ANIq.dipoles sets it); forward reads only the charges
        self._dipole_params: tp.Tuple[int, tp.Optional[tp.Tuple[float, ...]]] = (2, None)

    def __getitem__(self, idx: int) -> "ANIq":
        import copy
        base = ANI.__getitem__(self, idx)
        return ANIq(self.symbols, base.aev_computer, base.neural_networks, base.energy_shifter, dict(base.potentials),
                    self.periodic_table_index, copy.deepcopy(self.charge_networks),
                    copy.deepcopy(self.charge_normalizer))

    def _charge_params(self):
        from .electro import ChargeNormalizer
        from .engine import ChargeParams
        norm = self.charge_normalizer
        frame, masses = self._dipole_params
        if isinstance(norm, ChargeNormalizer):
            w, q2 = norm.params()
            return ChargeParams(w, q2, True, masses, frame)
        return ChargeParams(tuple(1.0 for _ in self.symbols), False, False, masses, frame)

    def engine(self, device: torch.device) -> Engine:
        # the charge networks follow the energy networks' operand format (models.ANI._guarded switches both)
        qnets = self.charge_networks
        if qnets._variant != self.neural_networks._variant:
            qnets.use_variant(self.neural_networks._variant)
        eng = super().engine(device)
        c = self.aev_computer.constants
        qnets._radial_len = c.num_species * len(c.shf_r)
        eng.set_charges((qnets.packed(device), self._charge_params()))
        return eng

    def _guarded(self, fn: tp.Callable[[], tp.Any]) -> tp.Any:
        try:
            return fn()
        except _lib.OperandRangeError:
            if not fall_back_to_bf16x3(self.neural_networks, self.charge_networks):
                raise
            return fn()

    def _step_with_charges(self, species_coordinates, cell, pbc, charge: int, want_grad: tp.Optional[bool] = None):
        """(elem_idxs, energies, atomic NN energies, member atomic, charges, dipoles) of one fused step, or, for a
        periodic cell thinner than the cutoff, of a supercell (then normalised over the supercell; the first A atoms'
        outputs are returned and the dipole is formed from their charges and the original coordinates)."""
        species, coords = species_coordinates
        self._check_inputs(species, coords, charge)
        elem_idxs = self.species_converter(species, nop=not self.periodic_table_index)
        _validate_inputs(self.cutoff, elem_idxs, coords, cell, pbc, conformer_cells=True)
        sup = None if (isinstance(self.neighborlist, CellList) or _per_conformer(cell)) else \
            supercell_for_thin_cell(species, coords, cell, pbc, self.cutoff)
        if sup is not None:
            sp_rep, co_rep, cell_rep, R = sup
            a = elem_idxs.shape[1]
            _, e, e_at, e_m, q, _ = self._step_with_charges((sp_rep, co_rep), cell_rep, pbc, charge, want_grad)
            q = q[:, :a]
            frame, masses = self._dipole_params
            from .electro import run_charges
            _, dip = run_charges(elem_idxs, q, coords, None, False, False, 0.0, masses, frame, True)
            return elem_idxs, e / R, e_at[..., :a], e_m[..., :a], q, dip
        cell = effective_periodic_cell(coords, cell, pbc, self.cutoff)
        wg = bool(coords.requires_grad) if want_grad is None else want_grad
        e, e_atomic, e_member, q, dip = self._guarded(lambda: _FusedEnergyCharges.apply(
            coords, elem_idxs, cell, pbc is not None, self.engine(coords.device), wg))
        return elem_idxs, e, e_atomic, e_member, q, dip

    def forward(self, species_coordinates: tp.Tuple[Tensor, Tensor], cell: tp.Optional[Tensor] = None,
                pbc: tp.Optional[Tensor] = None, charge: int = 0, atomic: bool = False,
                ensemble_values: bool = False) -> SpeciesEnergiesAtomicCharges:
        """arch.py:640-680: energies as ``ANI.forward`` and the normalised atomic charges (C, A) of the same step."""
        coords = species_coordinates[1]
        elem_idxs, e, e_atomic, e_member, q, _ = self._step_with_charges(species_coordinates, cell, pbc, charge)
        if ensemble_values:
            energies = e_member[self.neural_networks.active_members_idxs].to(coords.dtype)
            if self.energy_shifter._enabled:
                energies = energies + self.energy_shifter(elem_idxs, atomic=True).to(coords.dtype)
            if not atomic:
                energies = energies.sum(-1)
        elif atomic:
            energies = e_atomic.to(coords.dtype)
            if self.energy_shifter._enabled:
                energies = energies + self.energy_shifter(elem_idxs, atomic=True).to(coords.dtype)
        else:
            energies = e.to(coords.dtype)
        return SpeciesEnergiesAtomicCharges(elem_idxs, energies, q.to(coords.dtype))

    def dipoles(self, species_coordinates: tp.Tuple[Tensor, Tensor], cell: tp.Optional[Tensor] = None,
                pbc: tp.Optional[Tensor] = None, charge: int = 0, reference: str = "center_of_mass",
                masses: tp.Sequence[float] = ()) -> Tensor:
        """Dipoles (C, 3) in e * Angstrom, ``sum_i q_i (r_i - r_ref)`` over the real atoms of the normalised charges of
        the same fused step (electro.py:96-156, DipoleComputer), in the coordinates as given (not wrapped into the
        cell).  ``masses``: one per symbol of the model, needed for ``reference="center_of_mass"`` (the reference's
        mass table is not shipped)."""
        from .electro import frame_index
        frame = frame_index(reference)
        if frame == 0 and len(masses) != len(self.symbols):
            raise ValueError("the center_of_mass reference needs one mass per symbol of the model (masses=...): atomic "
                             "masses are not shipped with torchani_b200")
        self._dipole_params = (frame, tuple(float(m) for m in masses) if frame == 0 else None)
        try:
            coords = species_coordinates[1]
            *_, dip = self._step_with_charges(species_coordinates, cell, pbc, charge, want_grad=False)
        finally:
            self._dipole_params = (2, None)
        return dip.to(coords.dtype)

    def compute_from_neighbors(self, elem_idxs: Tensor, coords: Tensor, neighbors: Neighbors, charge: int = 0,
                               atomic: bool = False, ensemble_values: bool = False) -> EnergiesScalars:
        """arch.py:620-660: energies as ``ANI.compute_from_neighbors`` and the normalised charges (C, A) of the charge
        networks on the same AEVs."""
        self._check_inputs(elem_idxs, coords, charge)
        neighbors = discard_outside_cutoff(neighbors, self.cutoff)
        rcr = self.aev_computer.radial.cutoff
        aevs = self.aev_computer.compute_from_neighbors(
            elem_idxs, coords, neighbors if self.cutoff <= rcr else discard_outside_cutoff(neighbors, rcr))
        energies = self.neural_networks(elem_idxs, aevs, atomic, ensemble_values)
        for pot in self._enabled_potentials():
            energies = energies + pot.compute_from_neighbors(
                elem_idxs, coords, discard_outside_cutoff(neighbors, pot.cutoff), charge, atomic,
                ensemble_values).to(energies.dtype)
        if self.energy_shifter._enabled:
            energies = energies + self.energy_shifter(elem_idxs, atomic=atomic).to(energies.dtype)
        if self.charge_networks._variant != self.neural_networks._variant:
            self.charge_networks.use_variant(self.neural_networks._variant)
        qs = self.charge_normalizer(elem_idxs, self.charge_networks(elem_idxs, aevs, atomic=True), charge)
        return EnergiesScalars(energies, qs.to(coords.dtype))

    def compute_from_full_neighborlist(self, *args, **kwargs):
        raise NotImplementedError("charges over a full neighbour list with ghost atoms are not supported: the "
                                  "normaliser needs every atom of the system")

    def members_forces(self, *args, **kwargs):
        raise ValueError("the query-by-committee step of an ANIq model computes no charges; call forward for the "
                         "charges, or build an ANI from the same energy networks for the member forces")

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs) -> None:
        for old in list(state_dict.keys()):
            if old.startswith(prefix + "potentials.nnp.charge_networks."):
                state_dict[old.replace("potentials.nnp.charge_networks.", "charge_networks.", 1)] = state_dict.pop(old)
        super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)


def ANImbis(model_index: tp.Optional[int] = None, neighborlist: NeighborlistArg = "cell_list",
            periodic_table_index: bool = True, device=None, seed: tp.Optional[int] = 0,
            electronegativity: tp.Sequence[float] = (), hardness: tp.Sequence[float] = ()) -> ANIq:
    """The ANImbis architecture (models.py:201-252): ANI-2x energies (AEV, 8-member CELU ensemble, self energies) and
    one set of charge networks with ANI-2x widths, GELU, no biases and ``out_dim = 2`` (column 1 is the charge), with a
    ``ChargeNormalizer`` of weights (electronegativity / hardness)^2 scaled by the squared raw charges.  Weights are
    seeded random (no download).  The electronegativities and hardnesses (one per symbol, ANI-2x order) are not
    shipped: pass them, or convert a reference model with ``from_torchani``."""
    from .electro import ChargeNormalizer
    from .nn import ChargeNetworks
    normalizer = ChargeNormalizer.from_electronegativity_and_hardness(
        SYMBOLS_2X, electronegativity, hardness, scale_weights_by_charges_squared=True)
    base = _assemble(SYMBOLS_2X, AEVComputer.like_2x, ANINetworks.like_2x, 8, neighborlist, periodic_table_index,
                     seed, None)
    qnets = ChargeNetworks.like_2x(SYMBOLS_2X, base.aev_computer.out_dim)
    model = ANIq(SYMBOLS_2X, base.aev_computer, base.neural_networks, base.energy_shifter, None, periodic_table_index,
                 qnets, normalizer)
    model.requires_grad_(False)
    if model_index is not None:
        model = model[model_index]
    return model.to(device) if device is not None else model
