"""Molecular dynamics on the device: velocity Verlet (NVE), Langevin (BAOAB, NVT) and Langevin with stochastic cell
rescaling (NPT) loops whose positions, velocities and cells stay in device memory, with K whole MD steps -- the
integrator launches of csrc/md.cu and the fused force step -- captured into one CUDA graph.  The host touches the GPU
once per K steps: one replay, one copy of the replay's thermo records and frames into pinned memory, one
synchronisation.

    dyn = md.Langevin(model, atomic_numbers, positions, masses, dt=0.5, temperature=300.0, friction=0.02, seed=0)
    dyn.run(10_000)
    dyn.positions, dyn.velocities, dyn.thermo, dyn.frames

Units: Angstrom, fs, amu, Hartree, K.  ``friction`` is in fs^-1: ASE's ``Langevin(..., friction=f)`` takes f in units
of the inverse ASE time unit (``ASE_TIME_FS`` = 10.1805 fs), so ASE's ``friction=0.2`` is ``0.2 / ASE_TIME_FS`` =
0.0196 fs^-1 here.  The BAOAB splitting samples the same distribution as ASE's Langevin but is not the same trajectory
(another scheme, other random numbers).

Every MD step rebuilds the bucket grid (no Verlet skin).  ``VelocityVerlet`` and ``Langevin`` keep the cell fixed, and
the system fully periodic or open; ``LangevinNPT`` rescales the cell of every conformer of a fully periodic system.
Pressures are in bar and compressibilities in 1 / bar (``BAR_TO_HARTREE_A3`` converts).
"""
from __future__ import annotations

import ctypes as C
import math
import typing as tp

import numpy as np
import torch
from torch import Tensor

from . import _lib
from ._lib import check, ptr
from .engine import conformer_cells
from .grad import BAR_TO_HARTREE_A3, HARTREE_TO_JOULE, _AMU, _E
from .nn import fall_back_to_bf16x3

__all__ = ["VelocityVerlet", "Langevin", "LangevinNPT", "maxwell_boltzmann", "Thermo", "Frames", "NPT", "ACCEL", "KB",
           "ASE_TIME_FS", "BAR_TO_HARTREE_A3"]

K_B_JOULE = 1.38064852e-23                     # Boltzmann constant, J / K (CODATA 2014)
ACCEL = HARTREE_TO_JOULE / _AMU * 1e-10        # Hartree / (amu A^2) in fs^-2: acceleration = -dE/dx / m * ACCEL
KB = K_B_JOULE / HARTREE_TO_JOULE              # k_B in Hartree / K
ASE_TIME_FS = 1e5 * math.sqrt(_AMU / _E)       # ASE's time unit, A sqrt(amu / eV), in fs


class Thermo(tp.NamedTuple):
    """One record per step and conformer (steps ascending)."""
    step: np.ndarray          # (S,) int64
    potential: np.ndarray     # (S, C) Hartree: the model's energy
    kinetic: np.ndarray       # (S, C) Hartree
    temperature: np.ndarray   # (S, C) K: 2 E_kin / (3 N_real k_B), as ASE reports it


class Frames(tp.NamedTuple):
    step: np.ndarray                    # (F,) int64: the recorded steps (multiples of record_every)
    positions: np.ndarray               # (F, C, A, 3) float64, unwrapped
    velocities: tp.Optional[np.ndarray]  # (F, C, A, 3) float64 with record_velocities, else None


class NPT(tp.NamedTuple):
    """One barostat record per step and conformer (``LangevinNPT``; steps ascending, those of ``Thermo``)."""
    step: np.ndarray          # (S,) int64
    volume: np.ndarray        # (S, C) A^3: the cell of the step
    pressure: np.ndarray      # (S, C) bar: the internal pressure (2 E_kin - tr W) / (3 V), W the force step's virial


def _host(x, dtype=None) -> np.ndarray:
    """An input as a numpy array (a tensor is copied to the host)."""
    return np.asarray(x.detach().cpu() if isinstance(x, Tensor) else x, dtype=dtype)


def _per_conf(x, n: int) -> np.ndarray:
    """A scalar or one value per conformer as (n,) float64."""
    return np.broadcast_to(np.asarray(x, dtype=np.float64).reshape(-1), (n,))


def maxwell_boltzmann(masses, temperature, seed: int = 0) -> np.ndarray:
    """Velocities (..., A, 3) float64 in A / fs drawn from the Maxwell-Boltzmann distribution at ``temperature`` (K; a
    scalar, or one per conformer for masses (C, A)), with the centre-of-mass momentum of every conformer set to zero.
    Atoms with mass 0 (padding) get zero velocity."""
    m = np.asarray(masses, dtype=np.float64)
    batch = m.ndim == 2
    m2 = m.reshape(-1, m.shape[-1])
    T = np.broadcast_to(np.asarray(temperature, dtype=np.float64).reshape(-1, 1), (m2.shape[0], 1))
    if (T <= 0).any() or (m2 < 0).any():
        raise ValueError("temperature must be > 0 and masses >= 0")
    real = m2 > 0
    inv = np.where(real, 1.0 / np.where(real, m2, 1.0), 0.0)
    rng = np.random.default_rng(seed)
    v = rng.standard_normal(m2.shape + (3,)) * np.sqrt(KB * T * ACCEL * inv)[..., None]
    p = (m2[..., None] * v).sum(1, keepdims=True)
    v = np.where(real[..., None], v - p / m2.sum(1, keepdims=True)[..., None], 0.0)
    return v if batch else v[0]


class _DeviceLoop:
    """The machinery every device loop shares (the MD integrators here, FIRE in ``optimize``): the model's engine with a
    workspace of its own, the initial force step, the status check with the switch to the 3 x bfloat16 build and the
    redo of the work from a saved state, and K steps -- the loop's own launches (``_integrate``) and the fused force
    step -- captured into one CUDA graph.

    A subclass lays out its float64 buffer with ``_layout`` and defines ``_init_launch(reset)`` (the coordinates of the
    current state and, with ``reset``, its initial values) and ``_integrate()``."""

    isobaric = False   # the force step accumulates the virial, and the cells are the loop's (LangevinNPT)
    qbc = False        # the force step is the query-by-committee step
    _what = "the device MD loop"

    def _set_system(self, model, atomic_numbers, cell, pbc, steps_per_replay: int) -> tp.Optional[np.ndarray]:
        """Model, device, species, PBC and the fixed cell (``per_conf``, ``_cell32``); returns the float64 cell."""
        dev = next(model.buffers()).device
        if dev.type != "cuda":
            raise ValueError(f"{self._what} needs a model on a CUDA device")
        self.model, self.device = model, dev
        pb = _host(pbc, bool).reshape(-1)
        if pb.size not in (1, 3) or (pb.any() and not pb.all()):
            raise ValueError("partial PBC is not supported: the system is fully periodic or open")
        self.pbc = bool(pb.all())
        if self.pbc and cell is None:
            raise ValueError("If pbc is not None, cell should be present")
        z = torch.as_tensor(_host(atomic_numbers))
        C_ = z.shape[0] if z.dim() == 2 else 1
        z = z.reshape(C_, -1).to(dev)
        self.n_conf, self.n_per_conf = C_, z.shape[1]
        self.species = model.species_converter(z, nop=not model.periodic_table_index)
        self.K = int(steps_per_replay)
        # the cell, in the form the engine takes it
        self.per_conf = False
        self._cell32 = None
        if not self.pbc:
            return None
        c64 = _host(cell, np.float64)
        c = torch.as_tensor(c64.astype(np.float32))
        if c.dim() == 3 and C_ == 1:
            c = c.reshape(3, 3)
        self.per_conf = conformer_cells(c, C_)
        self._cell32 = c.to(dev)
        return c64

    def _layout(self, head, flags, records) -> tp.Dict[str, Tensor]:
        """Lay out the float64 buffer ``_buf`` from named segments (name, shape[, dtype]) in this order: ``head``, the
        state a redone replay restores (``_head``, saved in ``_backup``); ``flags``, the stop or convergence words, -1
        until set, which end the head and start what a replay copies to the host (``_rec`` to ``_h_rec``); and
        ``records``, the record rings and frames ``_collect`` gathers.  Returns the device views by name."""
        segs = [(s[0], s[1], s[2] if len(s) > 2 else torch.float64) for s in (*head, *flags, *records)]
        ends = np.cumsum([math.prod(shape) for _, shape, _ in segs]).tolist()
        n_head, r0 = ends[len(head) + len(flags) - 1], ends[len(head) - 1]
        self._buf = torch.zeros(ends[-1], dtype=torch.float64, device=self.device)
        self._head, self._rec = self._buf[:n_head], self._buf[r0:]
        self._backup = torch.empty_like(self._head)
        self._h_rec = torch.zeros(self._rec.numel(), dtype=torch.float64).pin_memory()
        self._h_status = torch.zeros(1, dtype=torch.int32).pin_memory()
        views, host = {}, {}
        for (name, shape, dtype), b in zip(segs, ends):
            a = b - math.prod(shape)
            views[name] = self._buf[a:b].view(dtype).view(shape)
            if a >= r0:
                host[name] = self._h_rec[a - r0:b - r0].view(dtype).view(shape).numpy()
        for s in flags:
            views[s[0]].fill_(-1)
        self._h_flags = self._h_rec[:n_head - r0].view(torch.int64).numpy()
        self._flags = np.full(self._h_flags.shape, -1, dtype=np.int64)   # as of the last replay
        self._h_records = {s[0]: host[s[0]] for s in records}
        self._records: tp.Dict[str, tp.List[np.ndarray]] = {s[0]: [] for s in records}
        self.step = 0   # steps done (the device counter, mirrored)
        self._graph: tp.Optional[torch.cuda.CUDAGraph] = None
        return views

    def _rows(self, name: str, t0: int, k: int) -> tp.List[int]:
        """The rows of record segment ``name`` that steps t0 .. t0 + k - 1 wrote: those of a ring of K rows."""
        return [(t0 + i) % self.K for i in range(k)]

    def _collect(self, t0: int, k: int) -> None:
        for name, h in self._h_records.items():
            self._records[name].append(h[self._rows(name, t0, k)].copy())
        self._flags = self._h_flags.copy()

    def _joined(self, name: str, last: bool = False) -> np.ndarray:
        """The collected rows of record segment ``name`` (``last``: of the last replay only), steps ascending."""
        parts = self._records[name][-1:] if last else self._records[name]
        return np.concatenate([np.zeros((0,) + self._h_records[name].shape[1:])] + parts)

    def _run(self, steps: int, callback, args: tp.Callable[[], tuple],
             start: tp.Optional[tp.Callable[[], None]] = None) -> bool:
        """``start()``, then ``steps`` steps: replays of ``steps_per_replay`` steps, the remainder as eager launches of
        the same sequence (bitwise the same result), each followed by ``callback(step, *args())``; the run ends early
        once every flag word is set.  Returns whether they all are."""
        steps = int(steps)
        if steps < 0:
            raise ValueError("steps must be >= 0")
        with torch.cuda.device(self.device):
            if start is not None:
                start()
            done = 0
            while done < steps:
                k = min(self.K, steps - done)
                self._advance(k)
                done += k
                if callback is not None:
                    callback(self.step, *args())
                if bool((self._flags >= 0).all()):
                    break
        return bool((self._flags >= 0).all())

    def _init_cell(self) -> tuple:
        """(cell pointer, cell_mode) of the init entry points: cell_mode 0 open, 1 one cell, 2 one per conformer."""
        return ptr(self.ws.cell) if self.pbc else None, 2 if self.per_conf else (1 if self.pbc else 0)

    def _step_call(self, name: str, *args) -> None:
        """ani_b200_<name>(state, grad, energies, *args, cell, coords, stream) with the fixed cell, or its ``_cells``
        twin with the lattice table of one cell per conformer."""
        ws, L = self.ws, self.engine.lib
        if self.per_conf:
            fn, cell = getattr(L, f"ani_b200_{name}_cells"), ptr(ws.lattice)
        else:
            fn, cell = getattr(L, f"ani_b200_{name}"), ptr(ws.cell) if self.pbc else None
        check(fn(C.byref(self._state), ptr(ws.grad), ptr(ws.energies), *args, cell, ptr(ws.coords), self._stream()),
              name)

    # -- engine and workspace ----------------------------------------------------------------
    def _attach_engine(self) -> None:
        eng = self.model.engine(self.device)
        if eng.skin > 0:
            raise ValueError(f"{self._what} rebuilds the bucket grid every step: Verlet-skin reuse "
                             "(Engine.skin > 0) is not supported")
        if any(w.reducer is not None for w in eng._ws.values()):
            raise ValueError(f"{self._what} runs on one GPU: this engine is sharded")
        eng.check_pair_cutoffs(self.pbc)
        # a workspace of its own: between two runs it holds the forces of the current positions
        ws = eng.new_workspace(self.n_conf, self.n_per_conf)
        if self.pbc and self.n_conf > 1:
            ws.make_periodic()
        ws.species_i32.copy_(self.species.reshape(-1))
        if self.isobaric:
            pass   # the float32 cell(s) of the current master cell, written by _begin
        elif self.per_conf:
            ws.cells.copy_(self._cell32.reshape(self.n_conf, 9))
        elif self.pbc:
            ws.cell.copy_(self._cell32.reshape(-1))
        self.engine, self.ws = eng, ws
        self._graph = None
        self._attached()

    def _attached(self) -> None:
        """What a loop adds to a newly attached engine and workspace."""

    def _begin(self, reset: bool) -> None:
        """Write the float32 coordinates of the current positions and run the force step there (eagerly); on an operand
        range overflow switch to the 3 x bfloat16 build, restore the state and start again."""
        while True:
            self._backup.copy_(self._head)
            self._init_launch(reset)
            self._force_step()
            self._h_status.copy_(self.ws.status, non_blocking=True)
            torch.cuda.current_stream(self.device).synchronize()
            if not self._switched():
                return
            self._head.copy_(self._backup)

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    def _switched(self) -> bool:
        """Raise for the status word of the last force steps as Engine.check_status does; if the 2 x fp16 operand
        format ran out of range, move to the 3 x bfloat16 build instead and return True (the caller redoes the work)."""
        if int(self._h_status[0]) == 0:
            return False
        try:
            self.engine.check_status(self.ws)
        except _lib.OperandRangeError:
            if not fall_back_to_bf16x3(self.model.neural_networks):
                raise
            self._attach_engine()
            return True
        return False

    # -- the loop -------------------------------------------------------------------------------
    def _force_step(self) -> None:
        self.engine._launch(self.ws, self.pbc, True, 0, self.ws.n, False, want_virial=self.isobaric,
                            conformer_cells=self.per_conf, members=self.qbc)

    def _body(self, k: int) -> None:
        """k steps on the stream (graph-capturable): save the state, k x (the loop's launches, force step), copies
        out."""
        self._backup.copy_(self._head)
        for _ in range(k):
            self._integrate()
            self._force_step()
        self._h_rec.copy_(self._rec, non_blocking=True)
        self._h_status.copy_(self.ws.status, non_blocking=True)

    def _advance(self, k: int) -> None:
        """k steps: one replay of the captured K-step graph (k == K) or eager launches of the same sequence."""
        while True:
            if k == self.K and self.engine.cuda_graph:
                if self._graph is None:
                    self.engine.note_composition(self.ws)
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g):
                        self._body(k)
                    self._graph = g
                self._graph.replay()
            else:
                self._body(k)
            torch.cuda.current_stream(self.device).synchronize()
            if not self._switched():
                break
            self._head.copy_(self._backup)   # redo the replay on the new build from the state it started with
            self._begin(False)
        self._collect(self.step, k)
        self.step += k


class _Dynamics(_DeviceLoop):
    """The device MD loop shared by ``VelocityVerlet`` and ``Langevin`` (see the module docstring)."""

    integrator = _lib.MD_VERLET

    def __init__(self, model, atomic_numbers, positions, masses, dt: float, temperature, friction, seed: int,
                 cell, pbc, velocities, steps_per_replay: int, record_every: int, record_velocities: bool,
                 qbc_stop, zero_momentum: bool, barostat: tp.Optional[tp.Tuple[np.ndarray, float, np.ndarray]] = None):
        if not (math.isfinite(dt) and dt > 0):
            raise ValueError(f"dt must be > 0 fs, got {dt}")
        self.isobaric = barostat is not None
        c64 = self._set_system(model, atomic_numbers, cell, pbc, steps_per_replay)
        dev, C_, A = self.device, self.n_conf, self.n_per_conf
        real = (self.species >= 0).cpu().numpy()
        m = np.asarray(masses, dtype=np.float64)
        m = np.broadcast_to(m.reshape(-1, A), (C_, A))
        if not (np.isfinite(m[real]) & (m[real] > 0)).all():
            raise ValueError("masses must be > 0 (amu) for every real atom")
        n_real = real.sum(1)
        if (n_real == 0).any():
            raise ValueError("every conformer needs at least one real atom")
        T, g = _per_conf(temperature, C_), _per_conf(friction, C_)
        if self.integrator == _lib.MD_LANGEVIN:
            if not (np.isfinite(T) & (T > 0)).all():
                raise ValueError("temperature must be > 0 K")
            if not (np.isfinite(g) & (g >= 0)).all():
                raise ValueError("friction must be >= 0 (1 / fs)")
        self.qbc = qbc_stop is not None
        e_thr, f_thr = (None, None) if qbc_stop is None else qbc_stop
        e_thr = _per_conf(math.inf if e_thr is None else e_thr, C_)
        f_thr = _per_conf(math.inf if f_thr is None else f_thr, C_)
        self.record_every = int(record_every)
        if self.K < 1 or self.record_every < 0:
            raise ValueError("steps_per_replay must be >= 1 and record_every >= 0")
        self.dt = float(dt)

        if self.isobaric and self.pbc:
            if C_ > 1 and not self.per_conf:   # every replica's box evolves on its own: grid mode 3
                self._cell32, self.per_conf = self._cell32.expand(C_, 3, 3).contiguous(), True
            c64 = np.broadcast_to(c64.reshape(-1, 3, 3), (C_, 3, 3))
            if not (np.isfinite(c64).all() and (np.abs(np.linalg.det(c64)) > 0).all()):
                raise ValueError("constant pressure needs a finite cell of volume > 0 for every conformer")

        f64 = dict(dtype=torch.float64, device=dev)
        self.frame_slots = -(-self.K // self.record_every) if self.record_every else 0
        self.frame_f = 2 if record_velocities else 1
        npt = self.isobaric
        seg = self._layout(
            [("x", (C_, A, 3)), ("v", (C_, A, 3)), ("counter", (2,), torch.int64)] +
            ([("master", (2, C_, 3, 3))] if npt else []),
            [("stop", (C_,), torch.int64)],
            [("thermo", (self.K, C_, _lib.ANI_MD_THERMO)), ("frames", (self.frame_slots, self.frame_f, C_, A, 3))] +
            ([("npt", (self.K, C_, _lib.ANI_MD_BARO)), ("frame_cells", (self.frame_slots, C_, 3, 3))] if npt else []))
        self.x, self.v, self._counter, self._stop = seg["x"], seg["v"], seg["counter"], seg["stop"]
        self._master = seg.get("master")
        self._seg = seg
        if npt:
            self._master[0].copy_(torch.from_numpy(np.array(c64)).to(dev))
        self.x.copy_(torch.from_numpy(_host(positions, np.float64)).reshape(C_, A, 3).to(dev))
        if velocities is not None:
            self.v.copy_(torch.from_numpy(_host(velocities, np.float64)).reshape(C_, A, 3).to(dev))
        inv = np.where(real, 1.0 / np.where(real, m, 1.0), 0.0)
        self.inv_mass = torch.from_numpy(np.ascontiguousarray(inv)).to(**f64).reshape(-1)
        params = np.zeros((C_, _lib.ANI_MD_PARAMS))
        params[:, 0], params[:, 1], params[:, 2], params[:, 3], params[:, 4] = self.dt, T, g, e_thr, f_thr
        params[:, 5] = 3 * n_real
        self.params = torch.from_numpy(params).to(**f64)
        if self.isobaric:
            p0, tau, beta = barostat
            bp = np.zeros((C_, _lib.ANI_MD_BARO_PARAMS))
            bp[:, 0], bp[:, 1], bp[:, 2] = p0, tau, beta
            self.baro_params = torch.from_numpy(bp).to(**f64)
        self.trigger = torch.zeros(2, C_, A, 3, **f64) if self.qbc else None
        nb = -(-A // _lib.ANI_MD_BLOCK)
        self._partials = torch.zeros(C_ * nb * 2, **f64)
        st = _lib.MDState()
        st.x, st.v, st.inv_mass, st.params = ptr(self.x), ptr(self.v), ptr(self.inv_mass), ptr(self.params)
        st.counter, st.stop_step, st.trigger = ptr(self._counter), ptr(self._stop), ptr(self.trigger)
        st.thermo, st.frames, st.partials = ptr(seg["thermo"]), ptr(seg["frames"]), ptr(self._partials)
        st.seed = int(seed) & (2 ** 64 - 1)
        st.accel, st.kb = ACCEL, KB
        st.n_conf, st.n_per_conf, st.integrator = C_, A, self.integrator
        st.thermo_rows, st.record_every = self.K, self.record_every
        st.frame_slots, st.frame_velocities = self.frame_slots, int(self.frame_f == 2)
        self._state = st
        self._zero_momentum = bool(zero_momentum)
        with torch.cuda.device(dev):
            self._attach_engine()
            self._begin(True)

    def _attached(self) -> None:
        ws = self.ws
        if self.qbc:
            self.engine.members_buffers(ws)
        if self.isobaric:
            b = _lib.MDBarostat()
            b.master, b.params, b.virial = ptr(self._master), ptr(self.baro_params), ptr(ws.virial)
            b.cell_out, b.cell_stride = ptr(ws.cells) if self.per_conf else ptr(ws.cell), 9
            b.record, b.frame_cells = ptr(self._seg["npt"]), ptr(self._seg["frame_cells"])
            b.virial_slots = _lib.ANI_VIRIAL_SLOTS
            self._baro = b

    def _init_launch(self, reset: bool) -> None:
        """ani_b200_md_init (with the momentum removal when asked for, at the start only)."""
        if self.isobaric:   # the float32 cell(s) of the current step's master cell
            h = self._master[self.step % 2]
            if self.per_conf:
                self.ws.cells.copy_(h.reshape(self.n_conf, 9))
            else:
                self.ws.cell.copy_(h.reshape(-1))
        check(self.engine.lib.ani_b200_md_init(C.byref(self._state), *self._init_cell(),
                                               int(reset and self._zero_momentum), ptr(self.ws.coords),
                                               self._stream()), "md_init")

    def _integrate(self) -> None:
        """The integrator launches of one step (ani_b200_md_step: finish step t, start step t + 1)."""
        ws = self.ws
        if self.isobaric:
            check(self.engine.lib.ani_b200_md_step_npt(C.byref(self._state), C.byref(self._baro), ptr(ws.grad),
                                                       ptr(ws.energies), ptr(ws.coords), self._stream()), "md_step_npt")
        else:
            self._step_call("md_step", ptr(ws.qbc) if self.qbc else None, ptr(ws.atom_stats[1]) if self.qbc else None)

    def _rows(self, name: str, t0: int, k: int) -> tp.List[int]:
        if name in ("frames", "frame_cells"):   # the slot of every recorded step
            re = self.record_every
            return [(t // re) % self.frame_slots for t in range(t0, t0 + k) if t % re == 0] if re else []
        return super()._rows(name, t0, k)

    def run(self, steps: int, callback: tp.Optional[tp.Callable[..., tp.Any]] = None) -> None:
        """Run ``steps`` MD steps: replays of ``steps_per_replay`` steps, the remainder as eager launches of the same
        sequence (bitwise the same result).  ``callback(step, positions, velocities, thermo)`` runs after every replay
        (``thermo``: that replay's records).  With ``qbc_stop`` the run ends early once every conformer has stopped;
        the force steps of stopped conformers go on to the end of their replay (at most K - 1 wasted steps each)."""
        self._run(steps, callback, lambda: (self.positions, self.velocities, self._as_thermo(self._joined("thermo", True))))

    # -- results ----------------------------------------------------------------------------------
    @property
    def cell(self) -> tp.Optional[Tensor]:
        """The fixed cell in the form the engine takes it: (3, 3) or, one per conformer, (C, 3, 3) float32 (device);
        None for an open system."""
        return self._cell32

    @property
    def positions(self) -> Tensor:
        """(C, A, 3) float64 master positions of the current step, unwrapped (device)."""
        return self.x

    @property
    def velocities(self) -> Tensor:
        """(C, A, 3) float64 velocities of the current step t (device): the stored velocities lack the final half kick
        of step t until the next step applies it, so it is applied here from the forces of the last force step (not at
        t = 0 and not for stopped conformers, whose velocities are those of their stop step)."""
        if self.step == 0:
            return self.v.clone()
        h = (0.5 * self.params[:, 0] * ACCEL).view(-1, 1, 1) * self.inv_mass.view(self.n_conf, -1, 1)
        kicked = self.v - h * self.ws.grad.view(self.n_conf, self.n_per_conf, 3).double()
        stopped = (self._stop >= 0).view(-1, 1, 1)
        return torch.where(stopped, self.v, kicked)

    @staticmethod
    def _as_thermo(th: np.ndarray) -> Thermo:
        return Thermo(th[:, 0, 0].astype(np.int64), th[..., 1].copy(), th[..., 2].copy(), th[..., 3].copy())

    @property
    def thermo(self) -> Thermo:
        return self._as_thermo(self._joined("thermo"))

    @property
    def frames(self) -> Frames:
        f = self._joined("frames")
        steps = np.arange(0, self.step, self.record_every) if self.record_every else np.zeros(0, dtype=np.int64)
        return Frames(steps, f[:, 0], f[:, 1] if self.frame_f == 2 else None)

    @property
    def stop_step(self) -> np.ndarray:
        """(C,) int64: the step at which each conformer stopped, -1 while it runs (``qbc_stop``)."""
        return self._stop.cpu().numpy()

    @property
    def stopped(self) -> np.ndarray:
        return self.stop_step >= 0

    @property
    def trigger_frame(self) -> tp.Tuple[Tensor, Tensor]:
        """(positions, velocities), each (C, A, 3) float64 on the device, of every conformer at its stop step (zeros
        for a conformer that has not stopped); ``qbc_stop`` only."""
        if self.trigger is None:
            raise ValueError("no qbc_stop was given")
        return self.trigger[0], self.trigger[1]


class VelocityVerlet(_Dynamics):
    """NVE: B(dt/2) A(dt) forces B(dt/2), as ASE's ``VelocityVerlet``.

    Args:
        model: a ``torchani_b200.models.ANI`` on a CUDA device
        atomic_numbers: (A,) or (C, A) (element indices if the model has ``periodic_table_index=False``); -1 pads
        positions: (A, 3) or (C, A, 3) Angstrom; masses: (A,) or (C, A) amu (ignored for padding)
        dt: time step, fs
        cell: None, (3, 3) shared or (C, 3, 3) one per conformer; pbc: fully periodic (True) or open
        velocities: initial velocities (A / fs), default zero (see ``maxwell_boltzmann``)
        steps_per_replay: K, the MD steps of one CUDA graph replay
        record_every: a frame every so many steps (0: none); record_velocities: frames hold the velocities too
        qbc_stop: None, or (energy QBC threshold, force relative-stdev threshold) -- scalars or one per conformer, None
            for a check that is not wanted: a conformer stops, and its x and v freeze, at the first step whose ensemble
            disagreement exceeds either (``stopped``, ``stop_step``, ``trigger_frame``); the steps run the
            query-by-committee force step
        zero_momentum: remove the centre-of-mass momentum of every conformer at the start
    """

    integrator = _lib.MD_VERLET

    def __init__(self, model, atomic_numbers, positions, masses, dt: float = 0.5, cell=None, pbc=False,
                 velocities=None, steps_per_replay: int = 20, record_every: int = 10, record_velocities: bool = False,
                 qbc_stop=None, zero_momentum: bool = False):
        super().__init__(model, atomic_numbers, positions, masses, dt, 0.0, 0.0, 0, cell, pbc, velocities,
                         steps_per_replay, record_every, record_velocities, qbc_stop, zero_momentum)


class Langevin(_Dynamics):
    """NVT: BAOAB (Leimkuhler-Matthews), B(dt/2) A(dt/2) O(dt) A(dt/2) forces B(dt/2), with
    O: v = c v + sqrt((1 - c^2) k_B T / m) xi, c = exp(-friction dt), and xi from a counter-based generator keyed on
    (seed, step, atom, component): the noise does not depend on K or on replay boundaries.  ``temperature`` (K) and
    ``friction`` (1 / fs) may be one per conformer (replicas at different temperatures in one batch).  The other
    arguments are those of ``VelocityVerlet``."""

    integrator = _lib.MD_LANGEVIN

    def __init__(self, model, atomic_numbers, positions, masses, dt: float = 0.5, temperature=300.0,
                 friction=0.02, seed: int = 0, cell=None, pbc=False, velocities=None, steps_per_replay: int = 20,
                 record_every: int = 10, record_velocities: bool = False, qbc_stop=None, zero_momentum: bool = False):
        super().__init__(model, atomic_numbers, positions, masses, dt, temperature, friction, seed, cell, pbc,
                         velocities, steps_per_replay, record_every, record_velocities, qbc_stop, zero_momentum)


class LangevinNPT(_Dynamics):
    """NPT: ``Langevin`` (BAOAB) with isotropic stochastic cell rescaling (C-rescale; Bernetti & Bussi, J. Chem. Phys.
    153, 114107 (2020)).  With eps = ln V, per conformer and step t:

        P_int = (2 E_kin - tr W) / (3 V)                 W = sum (dE/dDelta)_a Delta_b, the force step's virial
        d eps = -(beta_T / tau_p) (P0 - P_int) dt + sqrt(2 k_B T beta_T dt / (V tau_p)) xi
        mu    = exp(d eps / 3):   h <- mu h,   x <- mu x,   v <- v / mu

    (Euler-Maruyama in eps.  The paper's k_B T / V drift term belongs to its volume form, dV = ...; in eps it cancels
    against the Ito correction; keeping it would sample Gamma(N + 2) instead of Gamma(N + 1), whose mean is
    1 / (N + 1) = 1.5 % larger for an ideal gas of 64 atoms.)

    P_int is formed from E_kin, W and V of step t; the rescaling follows the B A O A moves of the step, so the next force
    step sees the positions and the cell it is used with.  The noise xi is keyed on (seed, step, conformer) apart from
    the atoms' (``cell_noise``).  Isotropic scaling keeps the cell's shape (triclinic cells included).  The sampled
    volume distribution is that of the isothermal-isobaric ensemble (an ideal gas of N atoms: Gamma(N + 1, k_B T / P0)).

    Args: those of ``Langevin`` without ``pbc`` (always fully periodic); ``qbc_stop`` is rejected (the
    query-by-committee step computes no virial); and
        cell: (3, 3) or (C, 3, 3) lattice vectors as rows; a shared cell of a batch becomes one cell per conformer, since
            every replica's box evolves on its own
        pressure: P0, bar (scalar or one per conformer)
        tau_p: the barostat's relaxation time, fs
        compressibility: beta_T, 1 / bar (scalar or one per conformer; 4.5e-5 is water's)
    A box that shrinks below the cutoff raises ``ANI_STATUS_CELL_TOO_SMALL`` at the end of the replay, as does a
    neighbour-list overflow as the density rises.
    """

    integrator = _lib.MD_LANGEVIN

    def __init__(self, model, atomic_numbers, positions, masses, cell, dt: float = 0.5, temperature=300.0,
                 friction=0.02, pressure=1.01325, tau_p: float = 1000.0, compressibility=4.5e-5, seed: int = 0,
                 velocities=None, steps_per_replay: int = 20, record_every: int = 10, record_velocities: bool = False,
                 qbc_stop=None, zero_momentum: bool = False):
        if cell is None:
            raise ValueError("constant pressure needs a fully periodic cell")
        if qbc_stop is not None:
            raise ValueError("qbc_stop is not supported at constant pressure: the query-by-committee step computes no "
                             "virial")
        n_conf = np.shape(atomic_numbers)[0] if np.ndim(atomic_numbers) == 2 else 1
        p0, beta = _per_conf(pressure, n_conf), _per_conf(compressibility, n_conf)
        tau_p = float(tau_p)
        if not np.isfinite(p0).all():
            raise ValueError("pressure must be finite (bar)")
        if not (math.isfinite(tau_p) and tau_p > 0):
            raise ValueError(f"tau_p must be > 0 fs, got {tau_p}")
        if not (np.isfinite(beta) & (beta > 0)).all():
            raise ValueError("compressibility must be > 0 (1 / bar)")
        super().__init__(model, atomic_numbers, positions, masses, dt, temperature, friction, seed, cell, True,
                         velocities, steps_per_replay, record_every, record_velocities, None, zero_momentum,
                         (p0 * BAR_TO_HARTREE_A3, tau_p, beta / BAR_TO_HARTREE_A3))

    @property
    def cell(self) -> Tensor:
        """(C, 3, 3) float64 cell of the current step, lattice vectors as rows: a copy on the device (the master cells
        are rewritten by every step)."""
        return self._master[self.step % 2].clone()

    @property
    def volume(self) -> Tensor:
        """(C,) float64 volume of the current cell, A^3 (device)."""
        return torch.linalg.det(self._master[self.step % 2]).abs()

    @property
    def npt(self) -> NPT:
        r = self._joined("npt")
        return NPT(self.thermo.step, r[..., 0].copy(), r[..., 1] / BAR_TO_HARTREE_A3)

    @property
    def frame_cells(self) -> np.ndarray:
        """(F, C, 3, 3) float64: the cell of every frame of ``frames``."""
        return self._joined("frame_cells")


def noise(seed: int, step: int, n: int, device) -> Tensor:
    """(n, 3) float64: the standard normals the Langevin O step of ``step`` draws for atoms 0..n-1 (flat index over
    the conformers), from ani_b200_md_noise."""
    out = torch.empty(n, 3, dtype=torch.float64, device=device)
    with torch.cuda.device(out.device):
        check(_lib.lib().ani_b200_md_noise(int(seed) & (2 ** 64 - 1), int(step), int(n), ptr(out),
                                           torch.cuda.current_stream(out.device).cuda_stream), "md_noise")
    return out


def cell_noise(seed: int, step: int, n_conf: int, device) -> Tensor:
    """(n_conf,) float64: the standard normals the cell rescaling of ``step`` draws for conformers 0..n_conf-1, from
    ani_b200_md_cell_noise."""
    out = torch.empty(n_conf, dtype=torch.float64, device=device)
    with torch.cuda.device(out.device):
        check(_lib.lib().ani_b200_md_cell_noise(int(seed) & (2 ** 64 - 1), int(step), int(n_conf), ptr(out),
                                                torch.cuda.current_stream(out.device).cuda_stream), "md_cell_noise")
    return out
