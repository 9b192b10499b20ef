"""Float64 numpy restatement of the device barostat (csrc/md.cu, torchani_b200/md.py LangevinNPT): isotropic stochastic
cell rescaling (Bernetti & Bussi, J. Chem. Phys. 153, 114107 (2020)), beside the integrator steps of md_oracle.  It is a
module of its own so that md_oracle, the restatement the NVE / NVT tests are pinned to, stays as it is.  Test
infrastructure only: the reference has no integrator.

One device step t at constant pressure is md_oracle's ``finish`` and ``start`` followed by ``cell_rescale``, whose
internal pressure uses the kinetic energy after ``finish`` and the virial of the forces at x(t).  Units: Angstrom, fs,
amu, Hartree, K.
"""
import numpy as np

from oracle.md_oracle import HARTREE_J, KB

BAR = 1e5 * 1e-30 / HARTREE_J   # 1 bar (1e5 J / m^3) in Hartree / A^3


def cell_rescale(x, v, cell, ekin, virial, temperature, p0, tau_p, beta, dt, xi):
    """One isotropic C-rescale step per conformer, Euler-Maruyama in eps = ln V:

        P_int = (2 E_kin - tr W) / (3 V)
        d eps = -(beta_T / tau_p) (P0 - P_int) dt + sqrt(2 k_B T beta_T dt / (V tau_p)) xi,   mu = exp(d eps / 3)

    (the k_B T / V term of the paper's volume form, dV = -(beta_T V / tau_p) (P0 - P_int - k_B T / V) dt + ..., cancels
    against the Ito correction of the change of variable).  x, v (C, A, 3) after B A (O A); cell (C, 3, 3) rows of step t; ekin
    (C,) Hartree after the final half kick of step t; virial (C, 3, 3) sum (dE/dDelta)_a Delta_b at x(t), Hartree;
    temperature (K), p0 (Hartree / A^3), beta (A^3 / Hartree) and xi (standard normals): (C,) or scalars; tau_p, dt
    fs.  Returns (mu x, v / mu, mu cell, V, P_int), with V (A^3) and P_int (Hartree / A^3) of step t."""
    vol = np.abs(np.linalg.det(cell))
    p_int = (2.0 * ekin - np.trace(virial, axis1=-2, axis2=-1)) / (3.0 * vol)
    kt = KB * np.asarray(temperature, dtype=np.float64)
    bt = np.asarray(beta, dtype=np.float64) / tau_p
    de = -bt * (p0 - p_int) * dt + np.sqrt(2.0 * kt * bt * dt / vol) * xi
    mu = np.exp(de / 3.0)[..., None, None]
    return x * mu, v / mu, cell * mu, vol, p_int
