"""Geometry optimisation on the device: FIRE or L-BFGS for every conformer of a batch at once, with the positions and
the optimiser's state in device memory, and K whole optimisation steps -- the launches of csrc/opt.cu (FIRE) or
csrc/lbfgs.cu (L-BFGS) and the fused force step -- captured into one CUDA graph.  The host touches the GPU once per K
steps: one replay, one copy of the replay's records into pinned memory, one synchronisation.

    opt = optimize.FIRE(model, atomic_numbers, positions)
    done = opt.run(fmax=0.05, steps=1000)
    opt.positions, opt.energies, opt.forces, opt.converged, opt.log

FIRE is ASE's ``ase.optimize.FIRE`` (Bitzek et al., PRL 97, 170201 (2006)) without its ``downhill_check``, with ASE's
parameters and defaults, and each conformer runs its own optimisation.  Per conformer and step t, with the forces f in
eV / A (zero for fixed and padding atoms):

    fmax(t) = max_i |f_i| < fmax:  converged at t; x, v, dt, a, n never change again
    P = f.v, F2 = f.f, V2 = v.v
    t > 0, P > 0:   c1 = 1 - a, c2 = a sqrt(V2 / F2);  if n > n_min: dt = min(dt finc, dtmax), a = a fa;  n += 1
    t > 0, P <= 0:  c1 = c2 = 0, a = astart, dt = dt fdec, n = 0
    t = 0:          c1 = 1, c2 = 0          (ASE's first step: v = dt f, no shrinking of dt)
    v' = c1 v + (c2 + dt) f,   x(t+1) = x(t) + dt v' min(1, maxstep / |dt v'|)

The step of a conformer is clamped as a whole (ASE's global norm), not atom by atom.

Units: ``fmax`` and ``log.fmax`` are in eV / A, ASE's unit, so ASE's thresholds and FIRE parameters keep their meaning
(``maxstep`` in A).  ``energies`` is in Hartree and ``forces`` in Hartree / A, like every other output of the package.

Every step rebuilds the bucket grid (no Verlet skin).  ``FIRE`` keeps the cell fixed; ``CellFIRE`` relaxes the lattice
vectors with the atoms, as ASE's ``FIRE(FrechetCellFilter(atoms))`` does (see its docstring).  ``LBFGS`` is ASE's
``LBFGS`` without its line search, with the inputs, ``run`` and results of ``FIRE`` (see its docstring).  ``NEB`` is
ASE's nudged elastic band under FIRE, one FIRE optimisation per band, with the interior images of every band in one
force step (csrc/neb.cu; see its docstring).
"""
from __future__ import annotations

import ctypes as C
import math
import typing as tp
import warnings

import numpy as np
import torch
from torch import Tensor

from . import _lib
from ._lib import check, ptr
from .grad import BAR_TO_HARTREE_A3, HARTREE_TO_EV
from .md import _DeviceLoop, _host, _per_conf
from .nn import fall_back_to_bf16x3

__all__ = ["FIRE", "CellFIRE", "LBFGS", "NEB", "interpolate", "Log", "CellLog", "NEBLog", "HARTREE_TO_EV",
           "BAR_TO_HARTREE_A3"]


class Log(tp.NamedTuple):
    """One record per step and conformer (steps ascending)."""
    step: np.ndarray     # (S,) int64
    energy: np.ndarray   # (S, C) Hartree: the energy at the step's positions
    fmax: np.ndarray     # (S, C) eV / A: the largest force on a movable atom there


class CellLog(tp.NamedTuple):
    """One record per step and conformer of ``CellFIRE`` (steps ascending)."""
    step: np.ndarray       # (S,) int64
    energy: np.ndarray     # (S, C) Hartree
    fmax: np.ndarray       # (S, C) eV / A: the largest row norm of the atom and cell forces (FrechetCellFilter's)
    volume: np.ndarray     # (S, C) A^3
    pressure: np.ndarray   # (S, C) bar: -tr W / (3 V), the virial pressure of the force step
    enthalpy: np.ndarray   # (S, C) Hartree: E + p0 V


def _fixed_mask(fixed, n: int, A: int) -> np.ndarray:
    """``fixed`` (None, or an (A,) or (n, A) boolean mask) as an (n, A) mask."""
    fix = np.zeros((n, A), dtype=bool)
    if fixed is not None:
        f = _host(fixed)
        if f.dtype != bool or f.shape not in ((A,), (n, A)):
            raise ValueError(f"fixed must be a boolean mask of shape ({A},) or ({n}, {A}), got {f.dtype} {f.shape}")
        fix[:] = f
    return fix


class _Optimizer(_DeviceLoop):
    """What the device optimisers share: the system, the fixed mask and ``force_scale``, one float64 buffer
    [x | the optimiser's state | conv_step O | log K O R | further records], ``run`` and the results.  O is the number
    of optimisations (``_n_opt``: one per conformer, one per band for ``NEB``) and R the words of a record
    (``_record_words``).  A subclass lists its state (``_state_segments``) and further records (``_record_segments``)
    and names its parameter column of the fmax threshold (``_fmax_col``)."""

    _fmax_col = 0
    _record_words = _lib.ANI_OPT_RECORD

    @property
    def _n_opt(self) -> int:
        return self.n_conf

    def _state_segments(self) -> tp.List[tuple]:
        raise NotImplementedError

    def _record_segments(self) -> tp.List[tuple]:
        return []

    def _allocate(self, model, atomic_numbers, positions, cell, pbc, fixed, steps_per_replay):
        """The system and the buffer; returns the float64 cell and the buffer's views by name."""
        if int(steps_per_replay) < 1:
            raise ValueError("steps_per_replay must be >= 1")
        c64 = self._set_system(model, atomic_numbers, cell, pbc, steps_per_replay)
        C_, A = self.n_conf, self.n_per_conf
        self.fixed = _fixed_mask(fixed, C_, A)
        seg = self._layout([("x", (C_, A, 3))] + self._state_segments(), [("conv", (self._n_opt,), torch.int64)],
                           [("log", (self.K, self._n_opt, self._record_words))] + self._record_segments())
        self.x, self._conv = seg["x"], seg["conv"]
        self.x.copy_(torch.from_numpy(_host(positions, np.float64)).reshape(C_, A, 3).to(self.device))
        real = (self.species >= 0).cpu().numpy()
        scale = np.where(real & ~self.fixed, HARTREE_TO_EV, 0.0)
        self.force_scale = torch.from_numpy(scale).to(dtype=torch.float64, device=self.device).reshape(-1)
        return c64, seg

    def _start(self) -> None:
        with torch.cuda.device(self.device):
            self._attach_engine()
            self._begin(True)

    def run(self, fmax: float = 0.05, steps: int = 1000,
            callback: tp.Optional[tp.Callable[..., tp.Any]] = None) -> bool:
        """Optimise until every conformer has max_i |f_i| < ``fmax`` (eV / A) or ``steps`` steps have run: replays of
        ``steps_per_replay`` steps, the remainder as eager launches of the same sequence.  Returns True when every
        conformer converged.  A new ``run`` starts a new convergence check and keeps the optimiser's state (FIRE's v,
        dt, a, n; L-BFGS's history), so a second ``run`` with a smaller ``fmax`` continues the optimisation, as ASE's
        does.  ``callback(step, positions, log)`` runs after every replay (``log``: that replay's records)."""
        fmax = float(fmax)
        if not (math.isfinite(fmax) and fmax >= 0):
            raise ValueError(f"fmax must be >= 0 eV/A, got {fmax}")

        def start() -> None:
            self.params[:, self._fmax_col].fill_(fmax)
            self._conv.fill_(-1)
            self._flags[:] = -1

        return self._run(steps, callback, lambda: (self.positions, self._as_log(self._log_rows(True))), start)

    def _log_rows(self, last: bool = False) -> np.ndarray:
        """The collected records of ``log`` (``last``: of the last replay only)."""
        return self._joined("log", last)

    # -- results ----------------------------------------------------------------------------------
    @property
    def positions(self) -> Tensor:
        """(C, A, 3) float64 positions of the current step, unwrapped (device)."""
        return self.x

    @property
    def energies(self) -> Tensor:
        """(C,) float64 energies (Hartree) of the last force step: at the current positions (device, a copy)."""
        return self.ws.energies.clone()

    @property
    def forces(self) -> Tensor:
        """(C, A, 3) float32 forces -dE/dx (Hartree / A) of the last force step, fixed atoms included (device, a
        copy)."""
        return -self.ws.grad.view(self.n_conf, self.n_per_conf, 3)

    @property
    def converged_step(self) -> np.ndarray:
        """(O,) int64: the step at which each optimisation (conformer, or band of ``NEB``) converged in the current
        ``run``, -1 if it has not."""
        return self._conv.cpu().numpy()

    @property
    def converged(self) -> np.ndarray:
        return self.converged_step >= 0

    @staticmethod
    def _as_log(r: np.ndarray) -> Log:
        return Log(r[:, 0, 0].astype(np.int64), r[..., 1].copy(), r[..., 2].copy())

    @property
    def log(self) -> Log:
        return self._as_log(self._log_rows())


def _fire_params(dt, maxstep, dtmax, n_min, finc, fdec, astart, fa) -> tp.Tuple[float, ...]:
    """ASE's FIRE parameters, checked: the first eight columns of the parameter row of ani_opt_state."""
    dt, maxstep, dtmax, n_min = float(dt), float(maxstep), float(dtmax), float(n_min)
    finc, fdec, astart, fa = float(finc), float(fdec), float(astart), float(fa)
    par = (dt, maxstep, dtmax, n_min, finc, fdec, astart, fa)
    if not all(math.isfinite(p) for p in par):
        raise ValueError("the FIRE parameters must be finite")
    if not (dt > 0 and maxstep > 0 and dtmax > 0):
        raise ValueError("dt, maxstep and dtmax must be > 0")
    if not (0 < fdec < 1 <= finc):
        raise ValueError("FIRE needs 0 < fdec < 1 <= finc")
    if not (0 < fa <= 1 and 0 <= astart <= 1):
        raise ValueError("FIRE needs 0 < fa <= 1 and 0 <= astart <= 1")
    if n_min < 0:
        raise ValueError("n_min must be >= 0")
    return par


class FIRE(_Optimizer):
    """FIRE on the device (see the module docstring).

    Args:
        model: a ``torchani_b200.models.ANI`` on a CUDA device
        atomic_numbers: (A,) or (C, A) (element indices if the model has ``periodic_table_index=False``); -1 pads
        positions: (A, 3) or (C, A, 3) Angstrom
        cell: None, (3, 3) shared or (C, 3, 3) one per conformer (fixed); pbc: fully periodic (True) or open
        fixed: None, or an (A,) or (C, A) boolean mask of atoms that never move (ASE's ``FixAtoms``); they are left
            out of fmax
        dt, maxstep, dtmax, n_min, finc, fdec, astart, fa: ASE's FIRE parameters (maxstep in A), with
            0 < fdec < 1 <= finc, 0 < fa <= 1, dt, maxstep, dtmax > 0, n_min >= 0 and 0 <= astart <= 1
        steps_per_replay: K, the steps of one CUDA graph replay

    ``run`` returns after the replay in which the last conformer converged: the force steps of a converged conformer
    go on to the end of that replay (at most K - 1 steps each), while its positions stay where they converged.
    """

    _what = "the device optimiser"
    _fmax_col = 8

    def __init__(self, model, atomic_numbers, positions, cell=None, pbc=False, fixed=None, dt: float = 0.1,
                 maxstep: float = 0.2, dtmax: float = 1.0, n_min: int = 5, finc: float = 1.1, fdec: float = 0.5,
                 astart: float = 0.1, fa: float = 0.99, steps_per_replay: int = 20):
        par = _fire_params(dt, maxstep, dtmax, n_min, finc, fdec, astart, fa)
        c64, seg = self._allocate(model, atomic_numbers, positions, cell, pbc, fixed, steps_per_replay)
        self._state = self._fire_state(par, seg)
        self._setup(c64, seg)
        self._start()

    def _state_segments(self) -> tp.List[tuple]:
        return [("v", (self.n_conf, self.n_per_conf, 3)), ("scalars", (2, self._n_opt, _lib.ANI_OPT_SCALARS)),
                ("counter", (2,), torch.int64)]

    def _fire_state(self, par: tp.Tuple[float, ...], seg: tp.Dict[str, Tensor]) -> _lib.OptState:
        """FIRE's views of the buffer, parameters and scratch, and its ani_opt_state: one optimisation over the rows
        of each conformer (or of each band's interior images)."""
        C_, A, O = self.n_conf, self.n_per_conf, self._n_opt
        f64 = dict(dtype=torch.float64, device=self.device)
        self.v, self._scalars, self._counter = seg["v"], seg["scalars"], seg["counter"]
        params = np.zeros((O, _lib.ANI_OPT_PARAMS))
        params[:, :8] = par
        self.params = torch.from_numpy(params).to(**f64)
        self._partials = torch.zeros(C_ * -(-A // _lib.ANI_MD_BLOCK) * 4, **f64)
        st = _lib.OptState()
        st.x, st.v, st.force_scale, st.params = ptr(self.x), ptr(self.v), ptr(self.force_scale), ptr(self.params)
        st.scalars, st.counter, st.conv_step = ptr(self._scalars), ptr(self._counter), ptr(self._conv)
        st.record, st.partials = ptr(seg["log"]), ptr(self._partials)
        st.n_conf, st.n_per_conf, st.record_rows = O, C_ // O * A, self.K
        return st

    def _setup(self, cell64: tp.Optional[np.ndarray], seg: tp.Dict[str, Tensor]) -> None:
        """What a subclass adds to the state before the engine is attached."""

    # -- the device loop ------------------------------------------------------------------------
    def _init_launch(self, reset: bool) -> None:
        """ani_b200_opt_init (v = 0 and the initial scalars at the start only)."""
        check(self.engine.lib.ani_b200_opt_init(C.byref(self._state), *self._init_cell(), int(reset),
                                                ptr(self.ws.coords), self._stream()), "opt_init")

    def _integrate(self) -> None:
        """The FIRE launches of one step (ani_b200_opt_step: step t to x(t+1))."""
        self._step_call("opt_step")


class CellFIRE(FIRE):
    """FIRE over positions and lattice vectors: ASE's ``FIRE(FrechetCellFilter(atoms, scalar_pressure=...))`` on the
    device, one relaxation per conformer of a fully periodic batch.

    Per conformer, with h0 the cell at construction (rows are lattice vectors), F the deformation gradient (the cell is
    h = h0 F^T), c = ``cell_factor`` and p0 = ``pressure``, FIRE runs over A + 3 rows:

        atom rows   u_i = F^-1 r_i,        forces g_i = F^T f_i              (f = -dE/dr, eV / A)
        cell rows   d = c logm F,          forces Phi = D_expm(L^T)[G] / c,  L = d / c,  G = -(W + p0 V I) F^-T
        enthalpy    H = E + p0 V,          V = |det h|

    W is the force step's virial (eV here), D_expm the Frechet derivative of the matrix exponential; g and Phi are
    -dH/du and -dH/dd.  P, F2, V2, fmax and the maxstep clamp of ``FIRE`` include the cell rows, so ``fmax`` means what
    it means for ASE's filtered ``Atoms``; a converged conformer keeps its positions and cell.

    Args: those of ``FIRE`` (pbc is always fully periodic, and ``fixed`` is rejected: ASE's ``FixAtoms`` acts on
    Cartesian positions, which the filter's coordinates do not express), and
        cell: (3, 3) or (C, 3, 3) lattice vectors as rows; a shared cell of a batch becomes one cell per conformer
        pressure: p0, bar (scalar or one per conformer; 1 eV / A^3 = 1.6021766208e6 bar)
        cell_factor: c (scalar or one per conformer); default the number of real atoms, as ASE's
        hydrostatic_strain: keep only the isotropic part (tr Phi / 3) I of the cell force: the shape is kept
        constant_volume: keep only its traceless part: det F = 1
    A box that shrinks below the cutoff raises ``ANI_STATUS_CELL_TOO_SMALL`` at the end of the replay.
    """

    isobaric = True   # the force step accumulates the virial, and the cells are the loop's
    _what = "the device cell optimiser"

    def __init__(self, model, atomic_numbers, positions, cell, pbc=True, pressure=0.0, cell_factor=None,
                 hydrostatic_strain: bool = False, constant_volume: bool = False, fixed=None, **fire):
        pb = _host(pbc, bool).reshape(-1)
        if cell is None or pb.size not in (1, 3) or not pb.all():
            raise ValueError("variable-cell relaxation needs a fully periodic cell")
        if fixed is not None:
            raise ValueError("fixed atoms are not supported with a variable cell: the filter's coordinates do not "
                             "express Cartesian constraints")
        if hydrostatic_strain and constant_volume:
            raise ValueError("hydrostatic_strain and constant_volume are mutually exclusive")
        z = _host(atomic_numbers)
        n_conf = z.shape[0] if z.ndim == 2 else 1
        h = _host(cell, np.float64)
        if h.shape not in ((3, 3), (n_conf, 3, 3)) and not (n_conf == 1 and h.shape == (1, 3, 3)):
            raise ValueError(f"cell must be (3, 3) or ({n_conf}, 3, 3), got {h.shape}")
        h = np.broadcast_to(h.reshape(-1, 3, 3), (n_conf, 3, 3))
        if not (np.isfinite(h).all() and (np.abs(np.linalg.det(h)) > 0).all()):
            raise ValueError("variable-cell relaxation needs a finite cell of volume > 0 for every conformer")
        p0 = _per_conf(pressure, n_conf)
        if not np.isfinite(p0).all():
            raise ValueError("pressure must be finite (bar)")
        n_real = (z.reshape(n_conf, -1) >= 0).sum(1).astype(np.float64)
        cf = n_real if cell_factor is None else _per_conf(cell_factor, n_conf)
        if not (np.isfinite(cf) & (cf > 0)).all():
            raise ValueError("cell_factor must be > 0 (and every conformer needs a real atom)")
        self._p0 = p0 * BAR_TO_HARTREE_A3
        self._cell_factor = np.array(cf)
        self._projection = 1 if hydrostatic_strain else (2 if constant_volume else 0)
        # every conformer's cell evolves on its own: a batch always runs one cell per conformer (grid mode 3)
        super().__init__(model, atomic_numbers, positions, cell=np.array(h, order="C") if n_conf > 1 else cell,
                         pbc=True, **fire)

    def _state_segments(self) -> tp.List[tuple]:
        return super()._state_segments() + [("master", (2, self.n_conf, _lib.ANI_OPT_CELL_MASTER))]

    def _record_segments(self) -> tp.List[tuple]:
        return [("cell_log", (self.K, self.n_conf, _lib.ANI_OPT_CELL_RECORD))]

    def _setup(self, cell64, seg) -> None:
        dev, C_ = self.device, self.n_conf
        f64 = dict(dtype=torch.float64, device=dev)
        # (a C-order copy: numpy's default copy of a broadcast keeps the conformer axis innermost)
        self.h0 = torch.from_numpy(np.array(np.broadcast_to(cell64.reshape(-1, 3, 3), (C_, 3, 3)), order="C")).to(**f64)
        par = np.stack([self._p0, self._cell_factor, np.full(C_, HARTREE_TO_EV)], 1)
        self.cell_params = torch.from_numpy(par).to(**f64)
        self._cell_force = torch.zeros(C_, 9, **f64)
        self._master, self._cell_log_dev = seg["master"], seg["cell_log"]

    def _attached(self) -> None:
        q = _lib.OptCell()
        q.master, q.h0, q.params = ptr(self._master), ptr(self.h0), ptr(self.cell_params)
        q.cell_out, q.cell_stride = (ptr(self.ws.cells) if self.per_conf else ptr(self.ws.cell)), 9
        q.virial, q.virial_slots = ptr(self.ws.virial), _lib.ANI_VIRIAL_SLOTS
        q.cell_force, q.record, q.projection = ptr(self._cell_force), ptr(self._cell_log_dev), self._projection
        self._cell = q

    def _init_launch(self, reset: bool) -> None:
        """ani_b200_opt_cell_init: (with reset, v = 0, the initial scalars and F = I,) the float32 cell and coordinates
        of the current state."""
        check(self.engine.lib.ani_b200_opt_cell_init(C.byref(self._state), C.byref(self._cell), int(reset),
                                                     ptr(self.ws.coords), self._stream()), "opt_cell_init")

    def _integrate(self) -> None:
        """The launches of one step (ani_b200_opt_cell_step: u(t), d(t) to u(t+1), d(t+1))."""
        ws = self.ws
        check(self.engine.lib.ani_b200_opt_cell_step(C.byref(self._state), C.byref(self._cell), ptr(ws.grad),
                                                     ptr(ws.energies), ptr(ws.coords), self._stream()),
              "opt_cell_step")

    def _log_rows(self, last: bool = False) -> np.ndarray:
        return np.concatenate([self._joined("log", last), self._joined("cell_log", last)], -1)

    # -- results ----------------------------------------------------------------------------------
    @property
    def deformation(self) -> Tensor:
        """(C, 3, 3) float64 deformation gradient F of the current step (device, a copy)."""
        return self._master[self.step % 2, :, 18:].reshape(self.n_conf, 3, 3).clone()

    @property
    def positions(self) -> Tensor:
        """(C, A, 3) float64 Cartesian positions r = F u of the current step, unwrapped (device)."""
        return self.x @ self.deformation.transpose(1, 2)

    @property
    def cell(self) -> Tensor:
        """(C, 3, 3) float64 cell h0 F^T of the current step, lattice vectors as rows (device)."""
        return self.h0 @ self.deformation.transpose(1, 2)

    @property
    def volume(self) -> Tensor:
        """(C,) float64 volume of the current cell, A^3 (device)."""
        return torch.linalg.det(self.cell).abs()

    @property
    def stress(self) -> Tensor:
        """(C, 3, 3) float64 W / V (Hartree / A^3) of the last force step, at the current positions and cell: the
        convention of ``HostCalculator.calculate_with_stress``."""
        w = self.ws.virial.view(self.n_conf, -1, 9).sum(1).view(self.n_conf, 3, 3)
        return w / self.volume.view(-1, 1, 1)

    @property
    def enthalpies(self) -> Tensor:
        """(C,) float64 E + p0 V (Hartree) of the current step (device)."""
        return self.ws.energies + torch.from_numpy(self._p0).to(self.device) * self.volume

    @staticmethod
    def _as_log(r: np.ndarray) -> CellLog:
        return CellLog(r[:, 0, 0].astype(np.int64), r[..., 1].copy(), r[..., 2].copy(), r[..., 3].copy(),
                       r[..., 4] / BAR_TO_HARTREE_A3, r[..., 5].copy())


class LBFGS(_Optimizer):
    """L-BFGS on the device: ASE's ``ase.optimize.LBFGS(atoms, maxstep, memory, damping, alpha)`` without its line
    search, one optimisation per conformer of a batch.  Per conformer and step t, with f the forces in eV / A (zero for
    fixed and padding atoms), g = -f and H0 = 1 / alpha:

        fmax(t) = max_i |f_i| < fmax:  converged at t; nothing of the conformer changes again
        k >= 1:   s = x(t) - x(t-1), y = g(t) - g(t-1) join the history; the oldest pair leaves when more than
                  ``memory`` are kept
        p = -H g  (H the inverse BFGS matrix of the kept pairs with H0: the two-loop recursion's p; p = f / alpha at
                  k = 0)
        x(t+1) = x(t) + damping p min(1, maxstep / max_i |p_i|)   (the factor applies when max_i |p_i| >= maxstep:
                  the longest atom step, not FIRE's global norm);   k += 1

    One deviation from ASE: a pair with y.s == 0 exactly, where ASE divides by zero, is skipped.  Pairs with y.s < 0
    are kept, as ASE keeps them.  The device forms p from the compact representation of H (Byrd, Nocedal & Schnabel,
    Math. Prog. 63 (1994)) in four launches (csrc/lbfgs.cu), not by the two-loop recursion; both give the same p up to
    rounding.

    Args: those of ``FIRE`` without FIRE's parameters, and ASE's
        maxstep: the longest atom step, A (> 1 warns, as ASE does)
        memory: the pairs kept, 1 .. 128
        damping: the factor of every step
        alpha: the initial Hessian guess 1 / H0, eV / A^2
    The history is C x memory x 3A x 2 doubles on the device (and as much again for the copy a 3 x bfloat16 redo
    restores).  A second ``run`` keeps the history and k, as ASE's optimiser does.
    """

    _what = "the device optimiser"
    _fmax_col = 3

    def __init__(self, model, atomic_numbers, positions, cell=None, pbc=False, fixed=None, maxstep: float = 0.2,
                 memory: int = 100, damping: float = 1.0, alpha: float = 70.0, steps_per_replay: int = 20):
        maxstep, damping, alpha = float(maxstep), float(damping), float(alpha)
        for name, v in (("maxstep", maxstep), ("damping", damping), ("alpha", alpha)):
            if not (math.isfinite(v) and v > 0):
                raise ValueError(f"{name} must be finite and > 0, got {v}")
        if int(memory) != memory or not 1 <= int(memory) <= _lib.ANI_LBFGS_MAX_MEMORY:
            raise ValueError(f"memory must be an integer in 1..{_lib.ANI_LBFGS_MAX_MEMORY}, got {memory}")
        if maxstep > 1.0:
            warnings.warn(f"a much too large maximum step size for L-BFGS: {maxstep:.1f} A")
        self.memory = int(memory)
        _, seg = self._allocate(model, atomic_numbers, positions, cell, pbc, fixed, steps_per_replay)
        dev, C_, A = self.device, self.n_conf, self.n_per_conf
        self.x_prev, self.g_prev, self._s, self._y = seg["x_prev"], seg["g_prev"], seg["s"], seg["y"]
        self._sy, self._yy, self._iter, self._counter = seg["sy"], seg["yy"], seg["iter"], seg["counter"]
        f64 = dict(dtype=torch.float64, device=dev)
        params = np.zeros((C_, _lib.ANI_LBFGS_PARAMS))
        params[:, :3] = (maxstep, damping, 1.0 / alpha)
        self.params = torch.from_numpy(params).to(**f64)
        self._coef = torch.zeros(C_, 2, self.memory, **f64)
        self._p = torch.zeros(C_, A, 3, **f64)
        self._partials = torch.zeros(_lib.lbfgs_partials(C_, A, self.memory), **f64)
        st = _lib.LbfgsState()
        st.x, st.x_prev, st.g_prev = ptr(self.x), ptr(self.x_prev), ptr(self.g_prev)
        st.s, st.y, st.sy, st.yy = ptr(self._s), ptr(self._y), ptr(self._sy), ptr(self._yy)
        st.coef, st.p, st.iter = ptr(self._coef), ptr(self._p), ptr(self._iter)
        st.force_scale, st.params, st.counter = ptr(self.force_scale), ptr(self.params), ptr(self._counter)
        st.conv_step, st.record, st.partials = ptr(self._conv), ptr(seg["log"]), ptr(self._partials)
        st.n_conf, st.n_per_conf, st.memory, st.record_rows = C_, A, self.memory, self.K
        self._state = st
        self._start()

    def _state_segments(self) -> tp.List[tuple]:
        C_, A, M = self.n_conf, self.n_per_conf, self.memory + 1
        return [("x_prev", (C_, A, 3)), ("g_prev", (C_, A, 3)), ("s", (C_, M, A, 3)), ("y", (C_, M, A, 3)),
                ("sy", (C_, M, M)), ("yy", (C_, M, M)), ("iter", (C_, 2), torch.int64), ("counter", (2,), torch.int64)]

    def _init_launch(self, reset: bool) -> None:
        """ani_b200_lbfgs_init (x_prev = x, g_prev = 0 and an empty history at the start only)."""
        check(self.engine.lib.ani_b200_lbfgs_init(C.byref(self._state), *self._init_cell(), int(reset),
                                                  ptr(self.ws.coords), self._stream()), "lbfgs_init")

    def _integrate(self) -> None:
        """The L-BFGS launches of one step (ani_b200_lbfgs_step: step t to x(t+1))."""
        self._step_call("lbfgs_step")

    @property
    def iteration(self) -> np.ndarray:
        """(C,) int64: the steps each conformer has taken (ASE's ``iteration``)."""
        return self._iter[:, 0].cpu().numpy()

    def _history(self) -> tp.Tuple[Tensor, Tensor]:
        """(S, Y), each (C, L, A, 3) float64 on the device: the kept pairs of every conformer in chronological order,
        L = min(memory, pairs stored) of the conformer with the fewest (a copy)."""
        head = self._iter[:, 1].cpu().numpy()
        M = self.memory + 1
        L = int(min(self.memory, head.min()))
        idx = torch.as_tensor(np.stack([(h - L + np.arange(L)) % M for h in head]), device=self.device)
        take = idx.view(self.n_conf, L, 1, 1).expand(-1, -1, self.n_per_conf, 3)
        return torch.gather(self._s, 1, take), torch.gather(self._y, 1, take)


class NEBLog(tp.NamedTuple):
    """One record per step and band of ``NEB`` (steps ascending)."""
    step: np.ndarray   # (S,) int64
    emax: np.ndarray   # (S, B) Hartree: the largest interior energy at the step, E_imax
    fmax: np.ndarray   # (S, B) eV / A: the largest NEB force on a movable atom of the band's interior images
    imax: np.ndarray   # (S, B) int64: the image of E_imax (1 .. n - 2)


_NEB_METHODS = {"aseneb": _lib.ANI_NEB_ASENEB, "improvedtangent": _lib.ANI_NEB_IMPROVED_TANGENT}


class NEB(FIRE):
    """A nudged elastic band relaxed by FIRE on the device: ASE's ``FIRE(NEB(images, k, climb, method))`` for every
    band of a batch, with the interior images of all bands evaluated by one force step.

    A band has images 0 .. n - 1 (n >= 3); the endpoints never move.  Interior image i of band b is conformer
    b (n - 2) + i - 1 of the force step.  Per interior image, with F its forces (eV / A; zero for fixed and padding
    atoms), t- = x_i - x_{i-1}, t+ = x_{i+1} - x_i (zero on those atoms), k- = k_{i-1}, k+ = k_i and imax = 1 + the
    first index of the largest of E_1 .. E_{n-2}, the tangent is tau = alpha t- + beta t+ and

        method="aseneb" (ASE's default): (alpha, beta) = (0, 1) below imax, (1, 0) above it and (1, 1) at imax;
            m = tau.tau (1 if 0); climbing image f = F - 2 (F.tau / m) tau, every other image
            f = F - ((F.tau + (k- t- - k+ t+).tau) / m) tau
        method="improvedtangent" (Henkelman & Jonsson, J. Chem. Phys. 113, 9978 (2000)): (0, 1) where the energy rises
            through the image, (1, 0) where it falls, else weights |dE| max / min by the higher neighbour;
            u = tau / |tau|; climbing image f = F - 2 (F.u) u, every other image f = F - (F.u) u + (k+ |t+| - k- |t-|) u

    The one deviation from ASE: |tau| = 0 with "improvedtangent", where ASE divides by zero, gives u = 0.  The climbing
    image (Henkelman, Uberuaga & Jonsson, J. Chem. Phys. 113, 9901 (2000)) is image imax of each band when ``climb``
    is set; ``neb.climb = True`` before a second ``run`` continues with the FIRE state kept, as ASE's second
    ``opt.run()`` does.  FIRE (that of ``FIRE``) runs per band over the rows of its interior images: P, F2, V2, the
    maxstep clamp and fmax = max_i |f_i| (row norms of the NEB forces, as ASE 3.22's ``Optimizer.converged``) are the
    band's; a converged band's positions freeze.  The endpoint energies come from one force step at construction.

    Args:
        model: a ``torchani_b200.models.ANI`` on a CUDA device
        atomic_numbers: (A,) or (B, A); -1 pads
        images: (n, A, 3) or (B, n, A, 3) Angstrom, endpoints included (``interpolate`` makes a linear band)
        cell: None, (3, 3) shared by every band, or (B, 3, 3) one per band (fixed); pbc: fully periodic or open
        fixed: None, or an (A,) or (B, A) boolean mask of atoms that never move; their positions must be the same in
            every image of a band
        k: spring constants, eV / A^2: a scalar, (n - 1,) or (B, n - 1); spring j joins images j and j + 1
        climb: the climbing image; method: "aseneb" or "improvedtangent"
        dt, maxstep, dtmax, n_min, finc, fdec, astart, fa, steps_per_replay: those of ``FIRE``
    ASE's ``remove_rotation_and_translation`` and ``precon`` are rejected, as are its "eb", "spline" and "string"
    methods.
    """

    _what = "the device NEB"
    _record_words = _lib.ANI_NEB_RECORD

    def __init__(self, model, atomic_numbers, images, cell=None, pbc=False, fixed=None, k=0.1, climb: bool = False,
                 method: str = "aseneb", dt: float = 0.1, maxstep: float = 0.2, dtmax: float = 1.0, n_min: int = 5,
                 finc: float = 1.1, fdec: float = 0.5, astart: float = 0.1, fa: float = 0.99,
                 steps_per_replay: int = 20, remove_rotation_and_translation: bool = False, precon=None):
        if method not in _NEB_METHODS:
            raise ValueError(f"method must be 'aseneb' or 'improvedtangent', got {method!r} (ASE's 'eb', 'spline' and "
                             "'string' are not supported)")
        if remove_rotation_and_translation:
            raise ValueError("remove_rotation_and_translation is not supported")
        if precon is not None:
            raise ValueError("preconditioned NEB is not supported")
        par = _fire_params(dt, maxstep, dtmax, n_min, finc, fdec, astart, fa)
        x = _host(images, np.float64)
        if x.ndim == 3:
            x = x[None]
        if x.ndim != 4 or x.shape[-1] != 3:
            raise ValueError(f"images must be (n, A, 3) or (B, n, A, 3), got {x.shape}")
        B, n, A = x.shape[:3]
        if n < 3:
            raise ValueError(f"a band needs n >= 3 images, got {n}")
        m = n - 2
        if B * m > 65535:
            raise ValueError(f"B (n - 2) = {B * m} interior images exceed 65535")
        if not np.isfinite(x).all():
            raise ValueError("images must be finite")
        z = _host(atomic_numbers)
        if z.shape not in ((A,), (B, A)):
            raise ValueError(f"atomic_numbers must be ({A},) or ({B}, {A}), got {z.shape}")
        z = np.broadcast_to(z.reshape(-1, A), (B, A))
        fix = _fixed_mask(fixed, B, A)
        for b in range(B):   # t is zeroed on fixed atoms: ASE's result only if they sit still along the band
            if not (x[b][:, fix[b]] == x[b, 0][fix[b]]).all():
                raise ValueError(f"fixed atoms must have the same positions in every image of a band (band {b})")
        kk = np.asarray(k, dtype=np.float64)
        if kk.shape not in ((), (n - 1,), (B, n - 1)):
            raise ValueError(f"k must be a scalar, ({n - 1},) or ({B}, {n - 1}), got {kk.shape}")
        kk = np.array(np.broadcast_to(kk, (B, n - 1)), order="C")   # (numpy's copy of a broadcast is not C-order)
        if not (np.isfinite(kk) & (kk > 0)).all():
            raise ValueError("k must be finite and > 0 (eV / A^2)")
        # the cell of the force step: shared (grid mode 2) or one per interior image (grid mode 3)
        fcell = None
        if cell is not None:
            h = _host(cell, np.float64)
            if h.shape not in ((3, 3), (B, 3, 3)):
                raise ValueError(f"cell must be (3, 3) or ({B}, 3, 3), got {h.shape}")
            fcell = h.reshape(3, 3) if h.ndim == 2 or B == 1 else np.repeat(h, m, 0)
        self.n_bands, self.n_images, self.method = B, n, method
        self._climb = bool(climb)
        _, seg = self._allocate(model, np.repeat(z, m, 0), x[:, 1:-1].reshape(B * m, A, 3), fcell, pbc,
                                np.repeat(fix, m, 0), steps_per_replay)
        C_, f64 = self.n_conf, dict(dtype=torch.float64, device=self.device)
        st = _lib.NebState()
        st.fire = self._fire_state(par, seg)
        nb = -(-A // _lib.ANI_MD_BLOCK)
        self._dots = torch.zeros(C_ * nb * _lib.ANI_NEB_DOTS, **f64)
        self._neb_force = torch.zeros(C_, A, 3, **f64)
        self.endpoints = torch.from_numpy(np.ascontiguousarray(x[:, [0, n - 1]])).to(**f64)
        self.end_energies = torch.zeros(B, 2, **f64)
        self.springs = torch.from_numpy(kk).to(**f64)
        self._climb_dev = torch.full((B,), 1.0 if self._climb else 0.0, **f64)
        st.endpoints, st.end_energies, st.springs = ptr(self.endpoints), ptr(self.end_energies), ptr(self.springs)
        st.climb, st.neb_force, st.dots = ptr(self._climb_dev), ptr(self._neb_force), ptr(self._dots)
        st.n_images, st.n_atoms, st.method = n, A, _NEB_METHODS[method]
        self._state = st
        self._endpoint_energies()
        self._start()

    @property
    def _n_opt(self) -> int:
        return self.n_bands

    def _endpoint_energies(self) -> None:
        """One force step on the 2B endpoint conformers, at float32 coordinates wrapped as the loop writes them."""
        B, A, dev = self.n_bands, self.n_per_conf, self.device
        m = self.n_images - 2
        z = self.species.view(B, m, A)[:, :1].expand(B, 2, A).reshape(2 * B, A)
        xe = self.endpoints.reshape(2 * B, A, 3)
        cell = None
        if self.pbc:
            h = self._cell32.double().view(-1, 3, 3)
            h = h[::m].repeat_interleave(2, 0) if self.per_conf else h.expand(2 * B, 3, 3)
            xe = xe - torch.floor(xe @ torch.linalg.inv(h)) @ h
            cell = self._cell32.view(-1, 3, 3)[::m].repeat_interleave(2, 0) if self.per_conf else self._cell32
        with torch.cuda.device(dev):
            while True:
                try:
                    r = self.model.engine(dev).step(z, xe.float(), cell, self.pbc, check=True)
                    break
                except _lib.OperandRangeError:
                    if not fall_back_to_bf16x3(self.model.neural_networks):
                        raise
            self.end_energies.copy_(r.energies.view(B, 2))
        self._end_variant = self.model.neural_networks._variant

    def _attached(self) -> None:
        if self.model.neural_networks._variant != self._end_variant:   # switched to 3 x bfloat16: endpoints too
            self._endpoint_energies()

    @property
    def climb(self) -> bool:
        """Whether image imax of every band climbs.  Setting it writes the device word the next step and
        ``neb_forces`` read, so ``neb.climb = True; neb.run(...)`` continues with the FIRE state kept."""
        return self._climb

    @climb.setter
    def climb(self, value: bool) -> None:
        self._climb = bool(value)
        self._climb_dev.fill_(1.0 if self._climb else 0.0)

    # -- the device loop ------------------------------------------------------------------------
    def _init_launch(self, reset: bool) -> None:
        """ani_b200_neb_init (v = 0 and the initial scalars at the start only)."""
        check(self.engine.lib.ani_b200_neb_init(C.byref(self._state), *self._init_cell(), int(reset),
                                                ptr(self.ws.coords), self._stream()), "neb_init")

    def _integrate(self) -> None:
        """The NEB launches of one step (ani_b200_neb_step: step t to x(t+1))."""
        self._step_call("neb_step")

    # -- results ----------------------------------------------------------------------------------
    @property
    def positions(self) -> Tensor:
        """(B, n, A, 3) float64 positions of the current step, endpoints included, unwrapped (device, a copy)."""
        B, m, A = self.n_bands, self.n_images - 2, self.n_per_conf
        e = self.endpoints
        return torch.cat([e[:, :1], self.x.view(B, m, A, 3), e[:, 1:]], 1)

    @property
    def energies(self) -> Tensor:
        """(B, n) float64 energies (Hartree) of the images at the current positions (device, a copy)."""
        B, m = self.n_bands, self.n_images - 2
        return torch.cat([self.end_energies[:, :1], self.ws.energies.view(B, m), self.end_energies[:, 1:]], 1)

    @property
    def forces(self) -> Tensor:
        """(B, n - 2, A, 3) float32 forces -dE/dx (Hartree / A) of the interior images at the current positions,
        fixed atoms included (device, a copy)."""
        return -self.ws.grad.view(self.n_bands, self.n_images - 2, self.n_per_conf, 3)

    @property
    def neb_forces(self) -> Tensor:
        """(B, n - 2, A, 3) float64 NEB forces (eV / A) at the current positions: ani_b200_neb_project of the last
        force step (device, a copy)."""
        with torch.cuda.device(self.device):
            check(self.engine.lib.ani_b200_neb_project(C.byref(self._state), ptr(self.ws.grad),
                                                       ptr(self.ws.energies), self._stream()), "neb_project")
        return self._neb_force.view(self.n_bands, self.n_images - 2, self.n_per_conf, 3).clone()

    @property
    def imax(self) -> np.ndarray:
        """(B,) int64: the image of the largest interior energy at the current positions (the first of equal ones)."""
        e = self.ws.energies.view(self.n_bands, self.n_images - 2).cpu().numpy()
        return 1 + np.argmax(e, 1)

    @property
    def barrier(self) -> np.ndarray:
        """(B,) float64: E_imax - E_0 (Hartree) at the current positions."""
        e = self.energies.cpu().numpy()
        return e[np.arange(self.n_bands), self.imax] - e[:, 0]

    @staticmethod
    def _as_log(r: np.ndarray) -> NEBLog:
        return NEBLog(r[:, 0, 0].astype(np.int64), r[..., 1].copy(), r[..., 2].copy(), r[..., 3].astype(np.int64))


def interpolate(initial, final, n_images: int, cell=None, mic: bool = False) -> np.ndarray:
    """ASE's linear ``NEB.interpolate()`` on the host: (n_images, A, 3) float64 images from ``initial`` to ``final``
    (each (A, 3)), endpoints included.  With ``mic`` the displacement of every atom is taken to its nearest periodic
    image under ``cell`` (rows are lattice vectors), as ASE's ``interpolate(mic=True)``."""
    a = np.asarray(initial, dtype=np.float64)
    d = np.asarray(final, dtype=np.float64) - a
    if int(n_images) < 2 or a.shape != d.shape or a.ndim != 2 or a.shape[1] != 3:
        raise ValueError("interpolate needs n_images >= 2 and initial, final of the same (A, 3) shape")
    if mic:
        if cell is None:
            raise ValueError("mic needs a cell")
        h = np.asarray(cell, dtype=np.float64).reshape(3, 3)
        f = d @ np.linalg.inv(h)
        d = (f - np.round(f)) @ h
    s = np.arange(int(n_images)).reshape(-1, 1, 1) / (int(n_images) - 1)
    return a[None] + s * d[None]
