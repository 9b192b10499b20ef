"""Host-buffer calculator: the CUDA counterpart of ``torchani.ase.Calculator.calculate``
(ase.py:75-173) without the ``ase`` dependency.

An MD driver owns positions on the HOST (numpy / pinned torch tensors).  Per step the
reference converts numpy -> tensors, copies to the GPU, runs the model, calls ``energy.item()``
and ``forces.cpu().numpy()`` (two blocking D2H syncs).  Here the positions go straight into the
engine's persistent input buffer (one async H2D), the captured CUDA graph of the step is
replayed, energy and forces come back through pinned buffers (async D2H) and ONE stream
synchronisation ends the step.  After a few eager steps the copies themselves are captured too
(the pinned host buffers are persistent): a step is then ONE graph launch + ONE synchronisation.
"""
from __future__ import annotations

import typing as tp

import numpy as np
import torch
from torch import Tensor

from . import _lib
from .models import ANI
from .nn import fall_back_to_bf16x3

HARTREE_TO_EV = 27.211386024367243  # units.py (CODATA 2014, as used by the reference's ASE interface)


class QBC(tp.NamedTuple):
    """Ensemble disagreement of one ``HostCalculator.calculate_with_qbc`` call (arch.py:439-576 of the reference).
    Shapes are those of a single system; a batch adds a leading conformer axis."""
    energy_qbc: tp.Any                  # float (Hartree), or (C,) float64: std_m(E_m) / sqrt(real atoms)
    force_magnitudes: np.ndarray        # (A,) / (C, A) float32 [Hartree/A]: mean over the members of |F_m|
    force_relative_stdev: np.ndarray    # (A,) / (C, A): (std_m |F_m| + 1e-8) / (mean + 1e-8), unbiased std
    force_relative_range: np.ndarray    # (A,) / (C, A): (max_m |F_m| - min_m |F_m| + 1e-8) / (mean + 1e-8)


class HostCalculator:
    """Energy + forces for a fixed set of atoms from host coordinates.

    A BATCH of C systems of A atoms each (replicas, the frames of a trajectory, a screened dataset) is one step
    too: ``atomic_numbers`` (C, A) (-1 pads a shorter system), ``cell`` one (3, 3) cell shared by all or one cell per
    conformer (C, 3, 3); ``calculate`` then takes positions (C, A, 3) and returns energies (C,) and forces (C, A, 3)
    with the same single H2D and D2H copy per step, inside the same captured graph.

    Args:
        model: a ``torchani_b200.models.ANI`` on a CUDA device
        atomic_numbers: (A,) or (1, A) integer array (atomic numbers, or element indices if the
            model was built with ``periodic_table_index=False``), or (C, A) for a batch
        cell: (3, 3) lattice vectors as rows, (C, 3, 3) one cell per conformer of a batch, or None for a non-periodic
            system
        pbc: periodic in all three directions (partial periodicity is not supported)
        skin: > 0 switches on Verlet-skin reuse of the bucket grid (the counterpart of
            ``torchani.neighbors.VerletCellList``, neighbors.py:759-884): the grid is built for
            cutoff + skin and reused -- only the positions inside it are refreshed -- until an atom has
            moved more than 70 % of skin/2 from where it was binned; a step in which an atom left its
            skin/2 sphere is recomputed after a rebuild, so the results are always those of a fresh
            grid.  Pays off when consecutive calls move the atoms by a small fraction of ``skin``.
    """

    def __init__(self, model: ANI, atomic_numbers, cell=None, pbc: bool = False, shard: tp.Tuple[int, int] = (0, 1),
                 skin: float = 0.0, sharded: tp.Any = None):
        dev = next(model.buffers()).device
        if dev.type != "cuda":
            raise ValueError("HostCalculator needs a model on a CUDA device")
        self.model, self.device, self.pbc, self.shard = model, dev, bool(pbc), shard
        z = np.asarray(atomic_numbers)
        self.n_conf = z.shape[0] if z.ndim == 2 else 1
        self.batch = self.n_conf > 1
        z = torch.as_tensor(z).reshape(self.n_conf, -1).to(dev)
        self.elem_idxs = model.species_converter(z, nop=not model.periodic_table_index)   # validated once
        self.n = z.shape[1]
        self.engine = model.engine(dev)
        self.skin = float(skin)
        if self.skin < 0:
            raise ValueError("skin must be >= 0")
        if self.batch and (self.skin > 0 or sharded is not None):
            raise ValueError("a batch of systems runs on one GPU with a freshly built grid: no skin, no sharding")
        self.conformer_cells = False   # one cell per conformer of a batch (grid mode 3)
        if self.skin > 0:
            self.engine.skin = self.skin   # buckets for cutoff + skin (shared by every user of this engine)
        # multi-GPU (one process per GPU): `sharded` = parallel.ShardedEngine over this model's engine.  This rank
        # evaluates its slice of the atoms; the partial forces / energies are summed over the ranks ON THE DEVICE
        # (peer-memory reduction inside the captured graph) before the single D2H copy, so every rank returns the
        # full result
        self.sharded = sharded
        if sharded is not None:
            if sharded.engine is not self.engine:
                raise ValueError("`sharded` must wrap this model's engine")
            if self.skin > 0:
                raise ValueError("Verlet-skin reuse is not combined with multi-GPU sharding")
            self.shard = shard = (sharded.rank, sharded.world)
            self.ws = sharded.attach(1, self.n)
            self.ws.species_i32.copy_(self.elem_idxs.reshape(-1))
        else:
            self.ws = self._workspace()
        # pinned mirrors of the workspace's two transfer blocks (engine.Workspace.in_block / out_block): ONE H2D copy of
        # [cell(s) | coords] and ONE D2H copy of [energies | status | gradient] per step
        C_ = self.n_conf
        self.h_in = torch.zeros(self.ws.in_block.numel(), dtype=torch.float32).pin_memory()
        # (out_full: out_block followed by what the query-by-committee step adds; calculate copies out_block only)
        self.h_out_full = torch.zeros(self.ws.out_full.numel(), dtype=torch.uint8).pin_memory()
        self.h_out = self.h_out_full[:self.ws.out_block.numel()]
        shape = (C_, self.n, 3) if self.batch else (self.n, 3)
        self.h_coords = self.h_in[self.ws.in_coords_off:].view(shape)
        self.h_cell = self.h_in[:9]
        self.h_cells = self.h_in[:9 * C_].view(C_, 9)
        off = self.ws._out_grad_off
        self.h_grad = self.h_out[off:].view(torch.float32).view(shape)
        self.h_energy = self.h_out[:8 * C_].view(torch.float64)
        self.h_status = self.h_out[8 * C_:8 * C_ + 4].view(torch.int32)
        q0, s0 = self.ws._out_qbc_off, self.ws._out_stats_off
        M = self.engine.nets.num_members
        self.h_energy_qbc = self.h_out_full[q0 + 8 * M * C_:q0 + 8 * (M + 1) * C_].view(torch.float64)
        self.h_atom_stats = self.h_out_full[s0:s0 + 12 * C_ * self.n].view(torch.float32).view((3,) + shape[:-1])
        c0 = self.ws._out_chg_off
        self.h_dipoles = self.h_out_full[c0:c0 + 24 * C_].view(torch.float64).view(C_, 3)
        self.h_charges = self.h_out_full[c0 + 24 * C_:].view(torch.float32).view(shape[:-1])
        self._dipole: tp.Tuple[int, tp.Optional[tp.Tuple[float, ...]]] = (2, None)   # origin (set_dipole_reference)
        self.h_moved = torch.zeros(1, dtype=torch.int32).pin_memory()
        self._have_grid = False       # a grid built with the skin exists and may be reused
        self.rebuilds = 0             # steps that built the grid
        self.redone = 0               # reuse steps that had to be recomputed (an atom left its skin/2 sphere)
        self.h2d_bytes = self.h_in.numel() * 4
        self.d2h_bytes = self.h_out.numel()
        self.graph_after = 3          # eager host-driven steps before copies + kernels are captured as one graph
        self._calls = 0
        self._graphs: tp.Dict[tp.Any, torch.cuda.CUDAGraph] = {}   # reuse flag (or ("qbc", reuse)) -> captured step
        self._mode_calls = {False: 0, True: 0}
        self._graph_version: tp.Any = None
        if pbc and cell is None:
            raise ValueError("If pbc is not None, cell should be present")
        if cell is not None:
            self.set_cell(cell)

    def _workspace(self):
        ws = self.engine.workspace(self.n_conf, self.n)
        if self.batch and self.pbc:
            ws.make_periodic()
        ws.species_i32.copy_(self.elem_idxs.reshape(-1))
        return ws

    def set_cell(self, cell) -> None:
        c = torch.as_tensor(np.asarray(cell, dtype=np.float32))
        per = c.dim() == 3
        if per and not self.batch:
            c, per = c.reshape(3, 3), False   # (1, 3, 3): the cell of the one system
        if per:
            if c.shape != (self.n_conf, 3, 3):
                raise ValueError(f"cell must be (3, 3) or ({self.n_conf}, 3, 3); got {tuple(c.shape)}")
            self.h_cells.copy_(c.reshape(self.n_conf, 9))
        else:
            self.h_cell.copy_(c.reshape(-1))
        if per != self.conformer_cells:   # another kind of cell: other kernels, other captured graphs
            self.conformer_cells = per
            self._graphs = {}
            self._mode_calls = {False: 0, True: 0}
        self._have_grid = False   # a grid belongs to one cell

    def calculate_with_stress(self, positions, cell=None) -> tp.Tuple[float, np.ndarray, np.ndarray]:
        """(energy [Ha], forces (A, 3) [Ha/A], stress (3, 3) [Ha/A^3]) of a periodic system: the "f dot r"
        virial of ase.py:164-168 accumulated by the force kernel, divided by the cell volume.  Runs the
        step eagerly with a freshly built grid (the virial slots are not part of the captured graph)."""
        if not self.pbc:
            raise ValueError("the stress needs a periodic cell")
        if cell is not None:
            self.set_cell(cell)
        self._set_positions(positions)
        with torch.cuda.device(self.device):
            self._copies_in(False)
            res = self.engine.run(self.ws, True, want_grad=True, shard=self.shard, want_virial=True,
                                  conformer_cells=self.conformer_cells)
            self._copies_out(False)
            virial = res.virial.cpu().numpy()
        self._have_grid = False
        if int(self.h_status[0]) and self._check_or_switch():
            return self.calculate_with_stress(positions)
        if self.batch:
            cells = (self.h_cells.numpy().reshape(-1, 3, 3) if self.conformer_cells
                     else self.h_cell.numpy().reshape(1, 3, 3))
            volume = np.abs(np.linalg.det(cells.astype(np.float64))).reshape(-1, 1, 1)
            return self.h_energy.numpy().copy(), np.negative(self.h_grad.numpy()), virial / volume
        volume = abs(float(np.linalg.det(self.h_cell.numpy().reshape(3, 3).astype(np.float64))))
        return float(self.h_energy[0]), np.negative(self.h_grad.numpy()), virial / volume

    def _set_positions(self, positions) -> None:
        shape = tuple(self.h_coords.shape)
        if isinstance(positions, Tensor):
            self.h_coords.copy_(positions.reshape(shape))
        else:
            self.h_coords.numpy()[...] = np.asarray(positions, dtype=np.float32).reshape(shape)

    def calculate(self, positions, cell=None) -> tp.Tuple[float, np.ndarray]:
        """positions: (A, 3) float array on the host (Angstrom).  Returns (energy [Hartree],
        forces (A, 3) [Hartree/Angstrom]) -- multiply by HARTREE_TO_EV for ASE units.  A batch: positions (C, A, 3),
        energies (C,) float64 and forces (C, A, 3); ``cell`` (3, 3) or (C, 3, 3) replaces the cell(s)."""
        if cell is not None:
            self.set_cell(cell)
        self._set_positions(positions)
        eng = self.engine
        self._calls += 1
        if self._graphs and self._graph_version != eng.nets.active_key:
            self._graphs = {}   # the active ensemble members changed: the captured scales are stale
        reuse = self.skin > 0 and self._have_grid
        self._run(reuse)
        if reuse and (int(self.h_moved[0]) & 1):
            # an atom left its skin/2 sphere: the refreshed grid may have missed pairs -> rebuild, redo
            self.redone += 1
            self._run(False)
        elif reuse and int(self.h_moved[0]):
            self._have_grid = False   # close to the limit: rebuild before the next step
        if int(self.h_status[0]) and self._check_or_switch():   # came back with the results
            return self.calculate(positions)
        # a fresh array: h_grad is the persistent pinned D2H buffer and is overwritten by the next call
        if self.batch:
            return self.h_energy.numpy().copy(), np.negative(self.h_grad.numpy())
        return float(self.h_energy[0]), np.negative(self.h_grad.numpy())

    def calculate_with_qbc(self, positions, cell=None) -> tp.Tuple[tp.Any, np.ndarray, QBC]:
        """``calculate`` plus the ensemble's disagreement, for query-by-committee active learning: (energy [Hartree],
        forces [Hartree/A], ``QBC``).  One step evaluates every active member's forces (one AEV-backward launch for
        all of them) and the statistics on the device; like ``calculate`` it is one H2D and one D2H copy per call and,
        after a few calls, its own captured CUDA graph.  Energy and forces are the ensemble mean, as from
        ``calculate``.  Works with ``skin > 0`` and with batches; not with multi-GPU sharding."""
        if self.sharded is not None or tuple(self.shard) != (0, 1):
            raise ValueError("calculate_with_qbc runs on one GPU: no sharding")
        if cell is not None:
            self.set_cell(cell)
        self._set_positions(positions)
        eng = self.engine
        self._calls += 1
        if self._graphs and self._graph_version != eng.nets.active_key:
            self._graphs = {}   # the active ensemble members changed: the captured launches are stale
        reuse = self.skin > 0 and self._have_grid
        self._run(reuse, members=True)
        if reuse and (int(self.h_moved[0]) & 1):
            self.redone += 1   # an atom left its skin/2 sphere: rebuild, redo
            self._run(False, members=True)
        elif reuse and int(self.h_moved[0]):
            self._have_grid = False
        if int(self.h_status[0]) and self._check_or_switch():
            return self.calculate_with_qbc(positions)
        stats = self.h_atom_stats.numpy().copy()
        eq = self.h_energy_qbc.numpy().copy() if self.batch else float(self.h_energy_qbc[0])
        qbc = QBC(eq, stats[0], stats[1], stats[2])
        if self.batch:
            return self.h_energy.numpy().copy(), np.negative(self.h_grad.numpy()), qbc
        return float(self.h_energy[0]), np.negative(self.h_grad.numpy()), qbc

    def set_dipole_reference(self, reference: str = "origin", masses: tp.Optional[tp.Sequence[float]] = None) -> None:
        """Reference point of the dipoles of ``calculate_with_charges``: "origin" (default), "center_of_geometry" or
        "center_of_mass", which needs one mass per symbol of the model."""
        from .electro import frame_index
        frame = frame_index(reference)
        if frame == 0 and (masses is None or len(masses) != len(self.model.symbols)):
            raise ValueError("the center_of_mass reference needs one mass per symbol of the model")
        self._dipole = (frame, tuple(float(m) for m in masses) if frame == 0 else None)

    def calculate_with_charges(self, positions, cell=None) -> tp.Tuple[tp.Any, np.ndarray, np.ndarray, np.ndarray]:
        """``calculate`` plus the atomic charges of a charge model (``models.ANIq``): (energy [Hartree], forces
        [Hartree/A], charges (A,) [e], dipole (3,) [e * A], about the point of ``set_dipole_reference``).  One step
        computes everything; like ``calculate`` it is one H2D and one D2H copy per call and, after a few calls, its own
        captured CUDA graph.  Works with ``skin > 0`` and with batches (then (C,), (C, A, 3), (C, A), (C, 3)); not
        with multi-GPU sharding: the normaliser needs every atom's raw charge."""
        if getattr(self.engine, "charges", None) is None:
            raise ValueError("calculate_with_charges needs a charge model (models.ANIq)")
        if self.sharded is not None or tuple(self.shard) != (0, 1):
            raise ValueError("calculate_with_charges runs on one GPU: no sharding")
        if cell is not None:
            self.set_cell(cell)
        self._set_positions(positions)
        eng = self.engine
        self._calls += 1
        if self._graphs and self._graph_version != eng.nets.active_key:
            self._graphs = {}
        reuse = self.skin > 0 and self._have_grid
        self._run(reuse, charges=True)
        if reuse and (int(self.h_moved[0]) & 1):
            self.redone += 1   # an atom left its skin/2 sphere: rebuild, redo
            self._run(False, charges=True)
        elif reuse and int(self.h_moved[0]):
            self._have_grid = False
        if int(self.h_status[0]) and self._check_or_switch():
            return self.calculate_with_charges(positions)
        q, dip = self.h_charges.numpy().copy(), self.h_dipoles.numpy().copy()
        if self.batch:
            return self.h_energy.numpy().copy(), np.negative(self.h_grad.numpy()), q, dip
        return float(self.h_energy[0]), np.negative(self.h_grad.numpy()), q, dip[0]

    def _check_or_switch(self) -> bool:
        """Raise what the reference raises for the status word of the last step.  If the 2 x fp16 operand format ran
        out of range, rebuild on the 3 x bfloat16 build of the library instead and return True: the caller redoes the
        step."""
        try:
            self.engine.check_status(self.ws)
        except _lib.OperandRangeError:
            if self.sharded is not None or not fall_back_to_bf16x3(self.model.neural_networks):
                raise
            self.engine = self.model.engine(self.device)
            self.engine.skin = self.skin
            self.ws = self._workspace()
            self._graphs, self._have_grid = {}, False
            self._mode_calls = {False: 0, True: 0}
            return True
        return False

    def _run(self, reuse: bool, members: bool = False, charges: bool = False) -> None:
        """One step (H2D, kernels, D2H, synchronise); after a few eager uses of a mode its whole sequence
        is captured into one CUDA graph.  ``members``: the query-by-committee step (Engine.run(..., members=True)).
        ``charges``: the step with the charge pass (Engine.run(..., charges=True))."""
        with torch.cuda.device(self.device):   # the C-ABI launches on the current device's stream
            if members:
                self._run_members(reuse)
            elif charges:
                self._run_charges(reuse)
            else:
                self._run_on_device(reuse)

    def _run_members(self, reuse: bool) -> None:
        ws, eng = self.ws, self.engine
        key = ("qbc", reuse)
        self._mode_calls[key] = self._mode_calls.get(key, 0) + 1
        if not reuse:
            self.rebuilds += 1
        eng.members_buffers(ws)
        graph = self._graphs.get(key)
        if graph is None and eng.cuda_graph and not eng.profile and self._mode_calls[key] > self.graph_after:
            eng.note_composition(ws)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                self._copies_in(reuse)
                eng._launch(ws, self.pbc, True, 0, ws.n, reuse, conformer_cells=self.conformer_cells, members=True)
                self._copies_out(reuse, members=True)
            self._graphs[key], self._graph_version = graph, eng.nets.active_key
        if graph is not None:
            graph.replay()
        else:
            self._copies_in(reuse)
            eng.run(ws, self.pbc, want_grad=True, reuse=reuse, conformer_cells=self.conformer_cells, members=True)
            self._copies_out(reuse, members=True)
        torch.cuda.current_stream(self.device).synchronize()
        if not reuse:
            self._have_grid = self.skin > 0

    def _run_charges(self, reuse: bool) -> None:
        ws, eng = self.ws, self.engine
        qn, qp = eng.charges
        qp = qp._replace(frame=self._dipole[0], masses=self._dipole[1])
        eng.set_charges((qn, qp))   # (the model's own calls may have left other dipole parameters on the engine)
        key = ("charges", reuse, qn, qp)
        self._mode_calls[key] = self._mode_calls.get(key, 0) + 1
        if not reuse:
            self.rebuilds += 1
        eng.charge_buffers(ws)
        graph = self._graphs.get(key)
        if graph is None and eng.cuda_graph and not eng.profile and self._mode_calls[key] > self.graph_after:
            eng.note_composition(ws)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                self._copies_in(reuse)
                eng._launch(ws, self.pbc, True, 0, ws.n, reuse, conformer_cells=self.conformer_cells, charges=True)
                self._copies_out(reuse, members=True)
            self._graphs[key], self._graph_version = graph, eng.nets.active_key
        if graph is not None:
            graph.replay()
        else:
            self._copies_in(reuse)
            eng.run(ws, self.pbc, want_grad=True, reuse=reuse, conformer_cells=self.conformer_cells, charges=True)
            self._copies_out(reuse, members=True)
        torch.cuda.current_stream(self.device).synchronize()
        if not reuse:
            self._have_grid = self.skin > 0

    def _run_on_device(self, reuse: bool) -> None:
        ws, eng = self.ws, self.engine
        self._mode_calls[reuse] += 1
        if not reuse:
            self.rebuilds += 1
        graph = self._graphs.get(reuse)
        nccl_fallback = self.sharded is not None and self.sharded.world > 1 and self.sharded.mode == "nccl"
        if nccl_fallback:
            # peer memory could not be mapped: eager step, library all-reduce of the partials on the device
            import torch.distributed as dist
            self._copies_in(reuse)
            eng.run(ws, self.pbc, want_grad=True, shard=self.shard, reuse=reuse)
            dist.all_reduce(ws.grad, group=self.sharded.group)
            dist.all_reduce(ws.energies, group=self.sharded.group)
            self._copies_out(reuse)
            torch.cuda.current_stream(self.device).synchronize()
            return
        if graph is None and eng.cuda_graph and not eng.profile and self._mode_calls[reuse] > self.graph_after:
            rank, world = self.shard
            lo, hi = (ws.n * rank) // world, (ws.n * (rank + 1)) // world   # (all atoms of a batch)
            eng.note_composition(ws)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                self._copies_in(reuse)
                eng._launch(ws, self.pbc, True, lo, hi, reuse, conformer_cells=self.conformer_cells)
                self._copies_out(reuse)
            self._graphs[reuse], self._graph_version = graph, eng.nets.active_key
        if graph is not None:
            graph.replay()
        else:
            self._copies_in(reuse)
            eng.run(ws, self.pbc, want_grad=True, shard=self.shard, reuse=reuse, conformer_cells=self.conformer_cells)
            self._copies_out(reuse)
        torch.cuda.current_stream(self.device).synchronize()
        if not reuse:
            self._have_grid = self.skin > 0

    def _copies_in(self, reuse: bool = False) -> None:
        if reuse:
            self.ws.moved.zero_()
        self.ws.in_block.copy_(self.h_in, non_blocking=True)

    def _copies_out(self, reuse: bool = False, members: bool = False) -> None:
        # (members: the whole of out_full, with the query-by-committee and the charge outputs behind out_block)
        if members:
            self.h_out_full.copy_(self.ws.out_full, non_blocking=True)
        else:
            self.h_out.copy_(self.ws.out_block, non_blocking=True)
        if reuse:
            self.h_moved.copy_(self.ws.moved, non_blocking=True)

    def check_status(self) -> None:
        self.engine.check_status(self.ws)
