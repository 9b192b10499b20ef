"""Float64 restatement of the device FIRE step (csrc/opt.cu, torchani_b200/optimize.py): ASE's ase.optimize.FIRE
(Bitzek et al., PRL 97, 170201 (2006)) without its downhill check, one conformer at a time.  Also the 13-atom
Lennard-Jones cluster, whose global minimum (the icosahedron, E = -44.326801 eps) is the known answer the tests
optimise to."""
import math

import numpy as np

from oracle.md_oracle import HARTREE_EV

PARAMS = ("dt0", "maxstep", "dtmax", "n_min", "finc", "fdec", "astart", "fa", "fmax")
E_LJ13 = -44.326801   # eps: the global minimum of LJ13


def params(fmax, dt=0.1, maxstep=0.2, dtmax=1.0, n_min=5, finc=1.1, fdec=0.5, astart=0.1, fa=0.99) -> np.ndarray:
    """The per-conformer parameter row of ani_opt_state (ASE's defaults)."""
    return np.array([dt, maxstep, dtmax, n_min, finc, fdec, astart, fa, fmax], dtype=np.float64)


def init(par) -> np.ndarray:
    """The scalars {dt, a, n} of step 0."""
    return np.array([par[0], par[6], 0.0])


def step(x, v, scalars, grad, force_scale, par, t, converged=False):
    """One FIRE step of one conformer at step t: x, v (A, 3); scalars {dt, a, n}; grad (A, 3) dE/dx (Hartree / A, or
    any unit with force_scale 1); force_scale (A,) (eV per Hartree for movable atoms, 0 for fixed and padding atoms);
    par a ``params`` row; converged: the conformer converged at an earlier step.
    Returns x(t+1), v', the scalars of t + 1, fmax(t) and whether the conformer converges at t."""
    f = -np.asarray(grad, dtype=np.float64) * np.asarray(force_scale, dtype=np.float64)[:, None]
    fmax = math.sqrt((f * f).sum(1).max())
    if converged or fmax < par[8]:
        return x, v, scalars, fmax, not converged
    dt, a, n = scalars
    p, f2, v2 = (f * v).sum(), (f * f).sum(), (v * v).sum()
    c1, c2 = 1.0, 0.0
    if t > 0:
        if p > 0:
            c1, c2 = 1.0 - a, a * math.sqrt(v2 / f2)
            if n > par[3]:
                dt, a = min(dt * par[4], par[2]), a * par[7]
            n += 1.0
        else:
            c1, a, dt, n = 0.0, par[6], dt * par[5], 0.0
    cf = c2 + dt
    v1 = c1 * v + cf * f
    dr = dt * math.sqrt(c1 * c1 * v2 + 2.0 * c1 * cf * p + cf * cf * f2)   # = |dt v1|
    x1 = x + dt * (par[1] / dr if dr > par[1] else 1.0) * v1
    return x1, v1, np.array([dt, a, n]), fmax, False


def run(x, energy_grad, par, steps, force_scale=None):
    """Optimise one conformer from v = 0 at step 0: returns (x, E, the step it converged at or -1)."""
    force_scale = np.ones(len(x)) if force_scale is None else force_scale
    v, sc = np.zeros_like(x), init(par)
    for t in range(steps):
        e, g = energy_grad(x)
        x, v, sc, _, conv = step(x, v, sc, g, force_scale, par, t)
        if conv:
            return x, e, t
    return x, energy_grad(x)[0], -1


def lj(x, sigma=1.0, eps=1.0):
    """Lennard-Jones energy and gradient dE/dx of the cluster x (A, 3)."""
    d = x[:, None] - x[None]
    r2 = (d ** 2).sum(-1)
    np.fill_diagonal(r2, 1.0)
    s6 = (sigma * sigma / r2) ** 3
    e = 4.0 * eps * (s6 * s6 - s6)
    np.fill_diagonal(e, 0.0)
    g = 4.0 * eps * (-12.0 * s6 * s6 + 6.0 * s6) / r2
    np.fill_diagonal(g, 0.0)
    return 0.5 * e.sum(), (g[..., None] * d).sum(1)


def icosahedron(sigma=1.0) -> np.ndarray:
    """LJ13 at its minimum's shape: a centre and 12 vertices at the pair-minimum distance 2^(1/6) sigma."""
    p = (1.0 + math.sqrt(5.0)) / 2.0
    v = []
    for a in (-1.0, 1.0):
        for b in (-1.0, 1.0):
            v += [(0.0, a, b * p), (a, b * p, 0.0), (b * p, 0.0, a)]
    v = np.array(v)
    v /= np.linalg.norm(v[0])
    return np.vstack([np.zeros(3), v * 2.0 ** (1.0 / 6.0) * sigma])


__all__ = ["PARAMS", "E_LJ13", "HARTREE_EV", "params", "init", "step", "run", "lj", "icosahedron"]
