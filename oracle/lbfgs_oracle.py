"""Float64 restatement of the device L-BFGS step (csrc/lbfgs.cu, torchani_b200/optimize.py): ASE's
ase.optimize.LBFGS (``step``, ``update`` and ``determine_step`` of ase/optimize/lbfgs.py, without the line search),
one conformer at a time, with list histories as ASE keeps them.  The one deviation from ASE: a pair with y.s == 0
exactly (ASE divides by it) is skipped, as on the device.  ``compact_direction`` restates the device's algebra (the
compact representation of the same inverse BFGS matrix), so the tests can size their bars from the spread between the
two forms."""
import math

import numpy as np

from oracle.fire_oracle import E_LJ13, HARTREE_EV, icosahedron, lj

PARAMS = ("maxstep", "damping", "H0", "fmax")


def params(fmax, maxstep=0.2, damping=1.0, alpha=70.0) -> np.ndarray:
    """The per-conformer parameter row of ani_lbfgs_state (ASE's defaults)."""
    return np.array([maxstep, damping, 1.0 / alpha, fmax], dtype=np.float64)


class State:
    """One conformer's L-BFGS state: ASE's ``iteration``, ``s``, ``y``, ``rho``, ``r0`` and ``f0`` (here g0 = -f0)."""

    def __init__(self, memory=100):
        self.memory = memory
        self.iteration = 0
        self.s, self.y, self.rho = [], [], []
        self.r0 = self.g0 = None


def update(st: State, x, g) -> None:
    """ASE's ``update``: append the pair of the last step (skipped when y.s == 0) and keep the last ``memory``."""
    if st.iteration > 0:
        s0, y0 = (x - st.r0).reshape(-1), (g - st.g0).reshape(-1)
        ys = float(np.dot(y0, s0))
        if ys != 0.0:
            st.s.append(s0)
            st.y.append(y0)
            st.rho.append(1.0 / ys)
    if len(st.s) > st.memory:
        st.s.pop(0)
        st.y.pop(0)
        st.rho.pop(0)


def two_loop(s, y, rho, g, H0) -> np.ndarray:
    """ASE's two-loop recursion: p = -H g (flat)."""
    L = len(s)
    a = np.empty(L)
    q = np.array(g, dtype=np.float64).reshape(-1)
    for i in range(L - 1, -1, -1):
        a[i] = rho[i] * np.dot(s[i], q)
        q = q - a[i] * y[i]
    z = H0 * q
    for i in range(L):
        b = rho[i] * np.dot(y[i], z)
        z = z + s[i] * (a[i] - b)
    return -z


def compact_direction(S, Y, g, H0) -> np.ndarray:
    """p = -H g from the compact representation (Byrd, Nocedal & Schnabel 1994, Thm 2.2), S, Y (L, n) chronological:
    r = R^-1 u, a = R^-T ((D + H0 Y^T Y) r - H0 w), b = -H0 r, p = -(H0 g + S^T a + Y^T b)."""
    g = np.asarray(g, dtype=np.float64).reshape(-1)
    S, Y = np.asarray(S, dtype=np.float64).reshape(-1, g.size), np.asarray(Y, dtype=np.float64).reshape(-1, g.size)
    if len(S) == 0:
        return -H0 * g
    R = np.triu(S @ Y.T)
    D = np.diag(np.diag(R))
    u, w = S @ g, Y @ g
    r = _back(R, u)
    a = _forward(R.T, (D + H0 * (Y @ Y.T)) @ r - H0 * w)
    return -(H0 * g + S.T @ a + Y.T @ (-H0 * r))


def _back(U, b):
    x = np.zeros_like(b)
    for i in range(len(b) - 1, -1, -1):
        x[i] = (b[i] - U[i, i + 1:] @ x[i + 1:]) / U[i, i]
    return x


def _forward(Lo, b):
    x = np.zeros_like(b)
    for i in range(len(b)):
        x[i] = (b[i] - Lo[i, :i] @ x[:i]) / Lo[i, i]
    return x


def determine_step(p, maxstep):
    """ASE's ``determine_step``: scale the whole step so that the longest atom step is maxstep, when it is >=
    maxstep."""
    longest = math.sqrt((p * p).sum(1).max()) if p.size else 0.0
    return p * (maxstep / longest) if longest >= maxstep else p


def step(st: State, x, grad, force_scale, par, converged=False):
    """One L-BFGS step of one conformer at its current state: x (A, 3); grad (A, 3) dE/dx (Hartree / A, or any unit with
    force_scale 1); force_scale (A,) (eV per Hartree for movable atoms, 0 for fixed and padding atoms); par a ``params``
    row; converged: the conformer converged at an earlier step.  Updates st; returns x(t+1), fmax(t) and whether the
    conformer converges now."""
    g = np.asarray(grad, dtype=np.float64) * np.asarray(force_scale, dtype=np.float64)[:, None]
    fmax = math.sqrt((g * g).sum(1).max())
    if converged or fmax < par[3]:
        return x, fmax, not converged
    update(st, x, g)
    p = two_loop(st.s, st.y, st.rho, g, par[2]).reshape(-1, 3)
    dr = determine_step(p, par[0]) * par[1]
    st.r0, st.g0 = x.copy(), g.copy()
    st.iteration += 1
    return x + dr, fmax, False


def run(x, energy_grad, par, steps, memory=100, force_scale=None):
    """Optimise one conformer from a fresh state: returns (x, E, the step it converged at or -1)."""
    force_scale = np.ones(len(x)) if force_scale is None else force_scale
    st = State(memory)
    for t in range(steps):
        e, g = energy_grad(x)
        x, _, conv = step(st, x, g, force_scale, par)
        if conv:
            return x, e, t
    return x, energy_grad(x)[0], -1


__all__ = ["PARAMS", "E_LJ13", "HARTREE_EV", "params", "State", "update", "two_loop", "compact_direction",
           "determine_step", "step", "run", "lj", "icosahedron"]
