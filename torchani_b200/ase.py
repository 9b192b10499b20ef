r"""ASE ``Calculator`` for the CUDA path -- the counterpart of ``torchani.ase.Calculator`` (ase.py:32-173).

    calc = model.ase()                 # torchani_b200.models.ANI.ase(overwrite, stress_kind)
    atoms.calc = calc                  # energy / free_energy / forces / stress, ASE units (eV, eV/A, eV/A^3)

The reference converts numpy -> tensors -> GPU on every call, runs the model under autograd and reads the
energy and the forces back with two blocking copies.  Here ``calculate`` hands the positions to a persistent
``calculator.HostCalculator`` (pinned staging buffers, the whole step -- H2D, kernels, D2H -- one captured CUDA
graph, one synchronisation); a new one is built only when the atomic numbers or the periodicity change.

``stress_kind`` (ase.py:52-55,142-156): ``"fdotr"`` and ``"scaling"`` both come from the virial the force kernel
accumulates (sum over pairs of dE/dDelta (x) Delta, divided by the volume -- for a potential that depends on the
pair vectors only, the strain derivative of ``"scaling"`` IS that virial, DESIGN.md / tests/test_gpu_api.py);
``"numerical"`` uses ASE's own finite-difference ``calculate_numerical_stress``.

``ase`` is imported lazily and only here, exactly as in the reference: without it this module raises the
reference's ImportError and ``ANI.ase()`` is unavailable -- nothing else in the package depends on it.
"""
from __future__ import annotations

import typing as tp
import warnings

import numpy as np

try:
    import ase.units
    from ase.calculators.calculator import Calculator as AseCalculator, all_changes
except ImportError:
    raise ImportError(
        "Error when trying to import 'torchani_b200.ase':"
        " The ASE package could not be found. 'torchani_b200.ase' and the '*.ase()' methods"
        " of models won't be available. Please install ase if you want to use them."
    ) from None

from .calculator import HostCalculator
from .nn import ATOMIC_NUMBER

StressKind = str   # "scaling" | "fdotr" | "numerical"  (annotations.py of the reference)


class Calculator(AseCalculator):
    """TorchANI CUDA calculator for ASE (same constructor and results as ase.py:32-173)."""

    implemented_properties = ["energy", "free_energy", "forces", "stress"]

    def __init__(self, model, overwrite: bool = False, stress_kind: StressKind = "scaling", skin: float = 0.0,
                 qbc: bool = False):
        """``qbc=True``: every calculation also reports the ensemble's disagreement (query-by-committee active
        learning; HostCalculator.calculate_with_qbc): ``results["energy_qbc"]`` (eV), ``"force_magnitudes"`` (eV/A,
        per atom), ``"force_relative_stdev"`` and ``"force_relative_range"`` (per atom, dimensionless).  A calculation
        that also asks for the virial stress (``"scaling"`` / ``"fdotr"``) runs the stress step and then the QBC step on
        the same positions: the results carry both, at the cost of a second evaluation."""
        super().__init__()
        self.model = model
        buf = next(model.buffers())
        self.device = buf.device
        if not model.periodic_table_index:
            raise ValueError("ASE models must have periodic_table_index=True")
        if stress_kind not in ("scaling", "fdotr", "numerical"):
            raise ValueError(f"Unsupported stress kind {stress_kind}")
        self.overwrite = overwrite
        self.stress_kind = stress_kind
        self.skin = skin
        self.qbc = bool(qbc)
        if self.qbc:
            self.implemented_properties = list(Calculator.implemented_properties) + [
                "energy_qbc", "force_magnitudes", "force_relative_stdev", "force_relative_range"]
        # a charge model (models.ANIq): atomic charges (e) and the dipole about the centre of mass (e * A, ASE's unit)
        self._charges = hasattr(model, "charge_networks")
        if self._charges:
            self.implemented_properties = list(self.implemented_properties) + ["charges", "dipole"]
        self._host: tp.Optional[HostCalculator] = None
        self._host_key: tp.Any = None

    def _host_calculator(self, numbers: np.ndarray, periodic: bool, cell) -> HostCalculator:
        key = (numbers.tobytes(), periodic)
        if self._host is None or self._host_key != key:
            self._host = HostCalculator(self.model, numbers, cell if periodic else None, pbc=periodic, skin=self.skin)
            self._host_key = key
        return self._host

    def calculate(self, atoms=None, properties=["energy"], system_changes=all_changes):
        super().calculate(atoms, properties, system_changes)
        assert self.atoms is not None
        needs_stress = "stress" in properties
        numbers = np.asarray(self.atoms.get_atomic_numbers(), dtype=np.int64)
        positions = np.asarray(self.atoms.get_positions(), dtype=np.float64)
        cell = np.asarray(self.atoms.get_cell(complete=True).array if hasattr(self.atoms.get_cell(complete=True), "array")
                          else self.atoms.get_cell(complete=True), dtype=np.float64)
        pbc = np.asarray(self.atoms.get_pbc(), dtype=bool)
        periodic = bool(pbc.any())
        if periodic and not pbc.all():
            # PBC in some directions only (slabs, wires): an equivalent fully periodic cell whose non-periodic
            # lattice vectors are long enough that no pair within the cutoff crosses them (neighbors.py:214-275
            # enumerates image shifts along the periodic vectors only -- same pair set)
            import torch
            from .neighbors import effective_periodic_cell
            cell = effective_periodic_cell(torch.from_numpy(positions), torch.from_numpy(cell), torch.from_numpy(pbc),
                                           float(self.model.cutoff)).numpy()
        if periodic and self.overwrite:
            warnings.warn("'overwrite' set, info about crossing PBC *will be lost*")
            frac = positions @ np.linalg.inv(cell)
            positions = (frac - np.floor(frac)) @ cell            # utils.py:237-255 (map_to_central)
            self.atoms.set_positions(positions)
        host = self._host_calculator(numbers, periodic, cell)
        if periodic and (host.h_cell.numpy().reshape(3, 3) != cell.astype(np.float32)).any():
            host.set_cell(cell)
        ha = ase.units.Hartree
        if needs_stress and self.stress_kind in ("scaling", "fdotr"):
            if not periodic:
                raise ValueError("the stress needs a periodic cell")
            e, f, stress = host.calculate_with_stress(positions)
            self.results["stress"] = stress * ha
            if self.qbc:
                _, _, q = host.calculate_with_qbc(positions)
                self._store_qbc(q, ha)
        elif self.qbc:
            e, f, q = host.calculate_with_qbc(positions)
            self._store_qbc(q, ha)
        elif self._charges:
            self._set_masses(host)
            e, f, charges, dipole = host.calculate_with_charges(positions)
            self._store_charges(charges, dipole)
        else:
            e, f = host.calculate(positions)
        if self._charges and (needs_stress or self.qbc) and ("charges" in properties or "dipole" in properties):
            self._set_masses(host)
            _, _, charges, dipole = host.calculate_with_charges(positions)
            self._store_charges(charges, dipole)
        self.results["energy"] = e * ha
        self.results["free_energy"] = e * ha
        self.results["forces"] = f.astype(np.float64) * ha
        if needs_stress and self.stress_kind == "numerical":
            self.results["stress"] = self.calculate_numerical_stress(self.atoms)

    def _set_masses(self, host: HostCalculator) -> None:
        """The dipole is taken about the centre of mass of the Atoms: one mass per element of the model."""
        numbers = np.asarray(self.atoms.get_atomic_numbers())
        masses = np.asarray(self.atoms.get_masses(), dtype=np.float64)
        per_symbol = []
        for s in self.model.symbols:
            m = masses[numbers == ATOMIC_NUMBER[s]]
            if m.size and not np.all(m == m[0]):
                raise ValueError(f"the atoms of element {s} carry different masses: the dipole kernel takes one mass "
                                 "per element")
            per_symbol.append(float(m[0]) if m.size else 1.0)
        host.set_dipole_reference("center_of_mass", per_symbol)

    def _store_charges(self, charges: np.ndarray, dipole: np.ndarray) -> None:
        self.results["charges"] = charges.astype(np.float64)
        self.results["dipole"] = dipole.astype(np.float64)

    def _store_qbc(self, q, ha: float) -> None:
        self.results["energy_qbc"] = q.energy_qbc * ha
        self.results["force_magnitudes"] = q.force_magnitudes.astype(np.float64) * ha
        self.results["force_relative_stdev"] = q.force_relative_stdev.astype(np.float64)
        self.results["force_relative_range"] = q.force_relative_range.astype(np.float64)
