"""Float64 restatement of the device variable-cell FIRE step (csrc/opt.cu ani_b200_opt_cell_step,
torchani_b200/optimize.py CellFIRE): FIRE on the degrees of freedom of ASE's ``FrechetCellFilter``, one conformer at a
time.  The FIRE step itself is ``fire_oracle.step``, unchanged, on the (A + 3)-row vector this module builds.

Per conformer, with h0 the cell at construction (rows are lattice vectors), F the deformation gradient (h = h0 F^T), c
the cell factor and p0 the target pressure:

    atom rows   u_i = F^-1 r_i                   g_i = F^T f_i        (f = -dE/dr; row form g = f @ F)
    cell rows   d = c L,  L = logm F             Phi = D_expm(L^T)[G] / c,   G = -(W + p0 V I) F^-T
    enthalpy    H = E(r, h) + p0 V,  V = |det h|

W_ab = sum over pairs (dE/dDelta)_a Delta_b is the force step's virial.  g and Phi are -dH/du and -dH/dd.  The adjoint
of the Frechet derivative of expm is the Frechet derivative at the transpose: sum_ab G_ab [D_expm(L)[E_mn]]_ab =
[D_expm(L^T)[G]]_mn (``nine_directions`` is the left side, for the tests).  Projections: ``HYDROSTATIC`` keeps the
isotropic part (tr Phi / 3) I, ``CONSTANT_VOLUME`` the traceless part.
"""
import numpy as np
from scipy.linalg import expm, expm_frechet, logm

from oracle import fire_oracle
from oracle.md_oracle import HARTREE_EV

NONE, HYDROSTATIC, CONSTANT_VOLUME = 0, 1, 2


def deformation(d, c):
    """F = expm(d / c)."""
    return expm(np.asarray(d, dtype=np.float64) / c)


def cell_coordinates(F, c):
    """d = c logm(F) (real for the F of a relaxation, near the identity)."""
    return c * np.real(logm(F))


def adjoint_frechet(L, G):
    """The adjoint of D_expm(L) applied to G: D_expm(L^T)[G]."""
    return expm_frechet(np.asarray(L).T, np.asarray(G), compute_expm=False)


def nine_directions(L, G):
    """The same by its definition: entry (m, n) is sum_ab G_ab [D_expm(L)[E_mn]]_ab."""
    out = np.zeros((3, 3))
    for m in range(3):
        for n in range(3):
            E = np.zeros((3, 3))
            E[m, n] = 1.0
            out[m, n] = (np.asarray(G) * expm_frechet(np.asarray(L), E, compute_expm=False)).sum()
    return out


def project(phi, projection):
    tr3 = np.trace(phi) / 3.0
    if projection == HYDROSTATIC:
        return tr3 * np.eye(3)
    if projection == CONSTANT_VOLUME:
        return phi - tr3 * np.eye(3)
    return phi


def cell_force(d, W, p0, h0, c, projection=NONE):
    """Phi (3, 3) in the unit of W (energy), with p0 in energy / A^3; also V."""
    L = np.asarray(d, dtype=np.float64) / c
    F = expm(L)
    vol = abs(np.linalg.det(h0 @ F.T))
    G = -(np.asarray(W, dtype=np.float64) + p0 * vol * np.eye(3)) @ np.linalg.inv(F).T
    return project(adjoint_frechet(L, G) / c, projection), vol


def positions(u, F):
    """r = F u (row form u @ F^T)."""
    return np.asarray(u) @ F.T


def step(u, v, d, vc, scalars, grad, W, energy, h0, p0, c, par, t, force_scale, projection=NONE, converged=False,
         unit=HARTREE_EV):
    """One variable-cell FIRE step of one conformer at step t.

    u, v (A, 3) atom rows and their FIRE velocities; d, vc (3, 3) cell rows and theirs; scalars {dt, a, n}; grad (A, 3)
    dE/dr at r = u F^T in cell h0 F^T, W (3, 3) the virial there and energy E (Hartree, or any energy unit); p0 in that
    energy unit / A^3; c the cell factor; par a ``fire_oracle.params`` row; force_scale (A,) (``unit`` for real atoms, 0
    for padding); unit: eV per energy unit of the cell rows.

    Returns u, v, d, vc, scalars of t + 1, fmax(t) over the A + 3 rows, whether the conformer converges at t, and the
    record (V, -tr W / (3 V), E + p0 V) of step t."""
    F = deformation(d, c)
    f = -np.asarray(grad, dtype=np.float64) * np.asarray(force_scale, dtype=np.float64)[:, None]
    phi, vol = cell_force(d, np.asarray(W, dtype=np.float64) * unit, p0 * unit, h0, c, projection)
    x = np.vstack([u, d])
    vv = np.vstack([v, vc])
    g = -np.vstack([f @ F, phi])   # fire_oracle.step takes dE/dx: minus the forces, with force_scale 1
    x1, v1, sc, fmax, conv = fire_oracle.step(x, vv, scalars, g, np.ones(len(x)), par, t, converged)
    A = len(u)
    rec = np.array([vol, -np.trace(W) / (3.0 * vol), energy + p0 * vol])
    return x1[:A], v1[:A], x1[A:], v1[A:], sc, fmax, conv, rec


def run(u, h0, energy_grad_virial, par, steps, c, p0=0.0, projection=NONE, unit=1.0):
    """Relax one conformer from v = 0 at step 0 (energy_grad_virial(r, h) -> E, dE/dr, W): returns (r, h, H, the step
    it converged at or -1)."""
    v, d, vc, sc = np.zeros_like(u), np.zeros((3, 3)), np.zeros((3, 3)), fire_oracle.init(par)
    scale = np.full(len(u), unit)
    for t in range(steps):
        F = deformation(d, c)
        r, h = positions(u, F), h0 @ F.T
        e, g, W = energy_grad_virial(r, h)
        u, v, d, vc, sc, _, conv, rec = step(u, v, d, vc, sc, g, W, e, h0, p0, c, par, t, scale, projection,
                                             unit=unit)
        if conv:
            return r, h, rec[2], t
    F = deformation(d, c)
    r, h = positions(u, F), h0 @ F.T
    return r, h, energy_grad_virial(r, h)[0] + p0 * abs(np.linalg.det(h)), -1


__all__ = ["NONE", "HYDROSTATIC", "CONSTANT_VOLUME", "HARTREE_EV", "deformation", "cell_coordinates",
           "adjoint_frechet", "nine_directions", "project", "cell_force", "positions", "step", "run"]
