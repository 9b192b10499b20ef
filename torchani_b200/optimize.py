"""Geometry optimisation on the device: FIRE for every conformer of a batch at once, with the positions, the FIRE
velocities and the per-conformer scalars in device memory, and K whole optimisation steps -- the two launches of
csrc/opt.cu and the fused force step -- captured into one CUDA graph.  The host touches the GPU once per K steps: one
replay, one copy of the replay's records into pinned memory, one synchronisation.

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

Every step rebuilds the bucket grid (no Verlet skin), and the cell stays fixed.
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
from .grad import HARTREE_TO_EV
from .md import _DeviceLoop

__all__ = ["FIRE", "Log", "HARTREE_TO_EV"]


class Log(tp.NamedTuple):
    """One record per step and conformer (steps ascending)."""
    step: np.ndarray     # (S,) int64
    energy: np.ndarray   # (S, C) Hartree: the energy at the step's positions
    fmax: np.ndarray     # (S, C) eV / A: the largest force on a movable atom there


class FIRE(_DeviceLoop):
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

    def __init__(self, model, atomic_numbers, positions, cell=None, pbc=False, fixed=None, dt: float = 0.1,
                 maxstep: float = 0.2, dtmax: float = 1.0, n_min: int = 5, finc: float = 1.1, fdec: float = 0.5,
                 astart: float = 0.1, fa: float = 0.99, steps_per_replay: int = 20):
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
        if int(steps_per_replay) < 1:
            raise ValueError("steps_per_replay must be >= 1")
        self._set_system(model, atomic_numbers, cell, pbc, steps_per_replay)
        dev, C_, A = self.device, self.n_conf, self.n_per_conf
        n = C_ * A
        real = (self.species >= 0).cpu().numpy()
        fix = np.zeros((C_, A), dtype=bool)
        if fixed is not None:
            f = np.asarray(fixed if not isinstance(fixed, Tensor) else fixed.cpu())
            if f.dtype != bool or f.shape not in ((A,), (C_, A)):
                raise ValueError(f"fixed must be a boolean mask of shape ({A},) or ({C_}, {A}), got {f.dtype} "
                                 f"{f.shape}")
            fix[:] = f
        self.fixed = fix

        f64 = dict(dtype=torch.float64, device=dev)
        # [x 3n | v 3n | scalars 2 C 3 | counter 2 | conv_step C | records K C 3]: the head up to conv_step is what a
        # redone replay restores, the tail from conv_step on is what a replay copies to the host
        ns = 2 * C_ * _lib.ANI_OPT_SCALARS
        head = 6 * n + ns + 2 + C_
        self._buf = torch.zeros(head + self.K * C_ * _lib.ANI_OPT_RECORD, **f64)
        self.x = self._buf[:3 * n].view(C_, A, 3)
        self.v = self._buf[3 * n:6 * n].view(C_, A, 3)
        self._scalars = self._buf[6 * n:6 * n + ns].view(2, C_, _lib.ANI_OPT_SCALARS)
        self._counter = self._buf[6 * n + ns:6 * n + ns + 2].view(torch.int64)
        self._conv = self._buf[head - C_:head].view(torch.int64)
        self._rec = self._buf[head - C_:]
        self._head = self._buf[:head]
        self._backup = torch.empty_like(self._head)
        self._record_dev = self._buf[head:]
        self._h_rec = torch.zeros(self._rec.numel(), dtype=torch.float64).pin_memory()
        self._h_status = torch.zeros(1, dtype=torch.int32).pin_memory()
        pos = torch.as_tensor(positions if not isinstance(positions, Tensor) else positions.detach().cpu()
                              ).to(torch.float64).reshape(C_, A, 3)
        self.x.copy_(pos.to(dev))
        self._conv.fill_(-1)
        scale = np.where(real & ~fix, HARTREE_TO_EV, 0.0)
        self.force_scale = torch.from_numpy(scale).to(**f64).reshape(-1)
        params = np.zeros((C_, _lib.ANI_OPT_PARAMS))
        params[:, :8] = par
        self.params = torch.from_numpy(params).to(**f64)
        self._partials = torch.zeros(C_ * -(-A // _lib.ANI_MD_BLOCK) * 4, **f64)
        st = _lib.OptState()
        st.x, st.v, st.force_scale, st.params = ptr(self.x), ptr(self.v), ptr(self.force_scale), ptr(self.params)
        st.scalars, st.counter, st.conv_step = ptr(self._scalars), ptr(self._counter), ptr(self._conv)
        st.record, st.partials = ptr(self._record_dev), ptr(self._partials)
        st.n_conf, st.n_per_conf, st.record_rows = C_, A, self.K
        self._state = st
        self.step = 0   # steps done (the device counter, mirrored)
        self._conv_host = np.full(C_, -1, dtype=np.int64)
        self._log: tp.List[np.ndarray] = []
        self._graph: tp.Optional[torch.cuda.CUDAGraph] = None
        with torch.cuda.device(dev):
            self._attach_engine()
            self._begin(True)

    # -- the device loop ------------------------------------------------------------------------
    def _init_launch(self, reset: bool) -> None:
        """ani_b200_opt_init (v = 0 and the initial scalars at the start only)."""
        mode = 2 if self.per_conf else (1 if self.pbc else 0)
        check(self.engine.lib.ani_b200_opt_init(
            C.byref(self._state), ptr(self.ws.cell) if self.pbc else None, mode,
            int(reset), ptr(self.ws.coords), self._stream()), "opt_init")

    def _integrate(self) -> None:
        """The FIRE launches of one step (ani_b200_opt_step: step t to x(t+1))."""
        ws, L = self.ws, self.engine.lib
        if self.per_conf:
            rc = L.ani_b200_opt_step_cells(C.byref(self._state), ptr(ws.grad), ptr(ws.energies), ptr(ws.lattice),
                                           ptr(ws.coords), self._stream())
        else:
            rc = L.ani_b200_opt_step(C.byref(self._state), ptr(ws.grad), ptr(ws.energies),
                                     ptr(ws.cell) if self.pbc else None, ptr(ws.coords), self._stream())
        check(rc, "opt_step")

    def _collect(self, t0: int, k: int) -> None:
        C_ = self.n_conf
        h = self._h_rec.numpy()
        rows = [(t0 + i) % self.K for i in range(k)]
        self._log.append(h[C_:].reshape(self.K, C_, _lib.ANI_OPT_RECORD)[rows].copy())
        self._conv_host = h[:C_].view(np.int64).copy()

    def run(self, fmax: float = 0.05, steps: int = 1000,
            callback: tp.Optional[tp.Callable[..., tp.Any]] = None) -> bool:
        """Optimise until every conformer has max_i |f_i| < ``fmax`` (eV / A) or ``steps`` steps have run: replays of
        ``steps_per_replay`` steps, the remainder as eager launches of the same sequence.  Returns True when every
        conformer converged.  A new ``run`` starts a new convergence check and keeps the FIRE state (v, dt, a, n), so
        a second ``run`` with a smaller ``fmax`` continues the optimisation, as ASE's does.  ``callback(step,
        positions, log)`` runs after every replay (``log``: that replay's records)."""
        fmax, steps = float(fmax), int(steps)
        if not (math.isfinite(fmax) and fmax >= 0):
            raise ValueError(f"fmax must be >= 0 eV/A, got {fmax}")
        if steps < 0:
            raise ValueError("steps must be >= 0")
        with torch.cuda.device(self.device):
            self.params[:, 8].fill_(fmax)
            self._conv.fill_(-1)
            self._conv_host[:] = -1
            done = 0
            while done < steps:
                k = min(self.K, steps - done)
                self._advance(k)
                done += k
                if callback is not None:
                    callback(self.step, self.positions, self._as_log(self._log[-1]))
                if bool((self._conv_host >= 0).all()):
                    break
        return bool((self._conv_host >= 0).all())

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
        """(C,) int64: the step at which each conformer converged in the current ``run``, -1 if it has not."""
        return self._conv.cpu().numpy()

    @property
    def converged(self) -> np.ndarray:
        return self.converged_step >= 0

    @staticmethod
    def _as_log(r: np.ndarray) -> Log:
        return Log(r[:, 0, 0].astype(np.int64), r[..., 1].copy(), r[..., 2].copy())

    @property
    def log(self) -> Log:
        if not self._log:
            z = np.zeros((0, self.n_conf))
            return Log(np.zeros(0, dtype=np.int64), z, z.copy())
        return self._as_log(np.concatenate(self._log))
