"""Float64 numpy restatement of the device MD integrators (csrc/md.cu, torchani_b200/md.py), given the forces and the
Langevin noise, with the unit constants derived from CODATA 2014 on their own.  Test infrastructure only: the
reference has no integrator (its MD runs ASE's on the host), so nothing here is pinned to it.

Units: Angstrom, fs, amu, Hartree, K.  State: x, v (..., 3); grad = dE/dx (Hartree / A); inv_mass (...,) with 0 for
atoms that never move.  One device step t is ``finish`` (the final half kick with the forces at x(t), none at t = 0)
followed by ``start`` (the move to x(t + 1) with the same forces).
"""
import math

import numpy as np

# CODATA 2014
C_LIGHT = 299792458.0
MU0 = 4e-7 * math.pi
EPS0 = 1.0 / (MU0 * C_LIGHT ** 2)
H_PLANCK = 6.626070040e-34
HBAR = H_PLANCK / (2.0 * math.pi)
M_E = 9.10938356e-31
E_CHARGE = 1.6021766208e-19
AMU = 1.660539040e-27
K_B = 1.38064852e-23

HARTREE_J = M_E * E_CHARGE ** 4 / (16.0 * math.pi ** 2 * EPS0 ** 2 * HBAR ** 2)
HARTREE_EV = HARTREE_J / E_CHARGE
ACCEL = HARTREE_J / AMU / 1e-20 * 1e-30     # Hartree / (amu A^2) -> fs^-2
KB = K_B / HARTREE_J                         # Hartree / K
ASE_FS = 1e-15 * 1e10 * math.sqrt(E_CHARGE / AMU)   # ASE's units.fs (its time unit is A sqrt(amu / eV))
ASE_KB = K_B / E_CHARGE                             # ASE's units.kB, eV / K

VERLET, LANGEVIN = 0, 1


_PHILOX_M = (np.uint64(0xD2511F53), np.uint64(0xCD9E8D57))
_PHILOX_W = (np.uint32(0x9E3779B9), np.uint32(0xBB67AE85))
_LO32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(counter, key) -> np.ndarray:
    """Philox4x32-10 (Salmon et al., SC'11, as in Random123): counter (..., 4) and key (..., 2) uint32 words, broadcast
    against each other; returns the (..., 4) uint32 output block."""
    c = np.asarray(counter, dtype=np.uint32)
    k = np.asarray(key, dtype=np.uint32)
    lead = np.broadcast_shapes(c.shape[:-1], k.shape[:-1])
    c = [np.broadcast_to(c[..., j], lead).astype(np.uint64) for j in range(4)]
    k0 = np.broadcast_to(k[..., 0], lead).astype(np.uint32)
    k1 = np.broadcast_to(k[..., 1], lead).astype(np.uint32)
    with np.errstate(over="ignore"):
        for _ in range(10):
            p0, p1 = _PHILOX_M[0] * c[0], _PHILOX_M[1] * c[2]
            c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0.astype(np.uint64), p1 & _LO32,
                 (p0 >> np.uint64(32)) ^ c[3] ^ k1.astype(np.uint64), p0 & _LO32]
            k0 = k0 + _PHILOX_W[0]
            k1 = k1 + _PHILOX_W[1]
    return np.stack([w.astype(np.uint32) for w in c], -1)


def unit_open(a, b) -> np.ndarray:
    """A uniform double in (0, 1) from the top 53 bits of the words (a, b): (m + 1/2) 2^-53."""
    m = ((np.asarray(a, dtype=np.uint64) << np.uint64(32)) | np.asarray(b, dtype=np.uint64)) >> np.uint64(11)
    return (m.astype(np.float64) + 0.5) * 2.0 ** -53


def normal(seed, step, atom, comp) -> np.ndarray:
    """The device's standard normal of (seed, step, atom, component), broadcast over its arguments: one Philox4x32-10
    block with counter (step low, step high, atom, component) and key (seed low, seed high), two uniforms from its
    words (0, 1) and (2, 3), and the cosine branch of Box-Muller."""
    step = np.asarray(step, dtype=np.int64).astype(np.uint64)
    seed = np.asarray(seed, dtype=np.uint64)
    atom = np.asarray(atom, dtype=np.int64).astype(np.uint32)
    comp = np.asarray(comp, dtype=np.int64).astype(np.uint32)
    step, seed, atom, comp = np.broadcast_arrays(step, seed, atom, comp)
    ctr = np.stack([(step & _LO32).astype(np.uint32), (step >> np.uint64(32)).astype(np.uint32), atom, comp], -1)
    key = np.stack([(seed & _LO32).astype(np.uint32), (seed >> np.uint64(32)).astype(np.uint32)], -1)
    w = philox4x32_10(ctr, key)
    u1, u2 = unit_open(w[..., 0], w[..., 1]), unit_open(w[..., 2], w[..., 3])
    return np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)


def kick(v, grad, inv_mass, dt):
    """B(dt/2): v + dt/2 a, a = -grad / m * ACCEL."""
    h = (0.5 * dt * ACCEL * inv_mass)[..., None]
    return v - h * grad


def finish(v, grad, inv_mass, dt, t):
    return v if t == 0 else kick(v, grad, inv_mass, dt)


def start(x, v, grad, inv_mass, dt, integrator, temperature=0.0, friction=0.0, noise=None):
    """B(dt/2) A(dt) (velocity Verlet) or B(dt/2) A(dt/2) O(dt) A(dt/2) (BAOAB, ``noise`` standard normals like x)."""
    moving = (inv_mass > 0)[..., None]
    v1 = kick(v, grad, inv_mass, dt)
    if integrator == VERLET:
        x1 = x + dt * v1
    else:
        hd = 0.5 * dt
        x1 = x + hd * v1
        c = math.exp(-friction * dt)
        s = np.sqrt((1.0 - c * c) * KB * temperature * ACCEL * inv_mass)[..., None]
        v1 = c * v1 + s * noise
        x1 = x1 + hd * v1
    return np.where(moving, x1, x), np.where(moving, v1, v)


def kinetic(v, inv_mass):
    """Hartree, summed over the last two axes' atoms (per conformer for (C, A, 3))."""
    real = inv_mass > 0
    m = np.where(real, 1.0 / np.where(real, inv_mass, 1.0), 0.0)
    return 0.5 * (m[..., None] * v * v).sum((-1, -2)) / ACCEL


def temperature(ekin, n_real):
    return 2.0 * ekin / (3.0 * n_real * KB)


def wrap(x, cell):
    """x (..., 3) into the cell (rows are lattice vectors): fractional coordinates minus their floor."""
    frac = x @ np.linalg.inv(cell)
    return x - np.floor(frac) @ cell


def run(x, v, force, inv_mass, dt, steps, integrator=VERLET, temperature=0.0, friction=0.0, rng=None):
    """A whole trajectory with forces ``force(x) -> grad``: returns the positions and velocities of steps 0..steps
    (arrays (steps + 1, ...)).  Langevin noise from ``rng.standard_normal``."""
    xs, vs = [x], [v]
    g = force(x)
    for _ in range(steps):
        nz = rng.standard_normal(x.shape) if integrator == LANGEVIN else None
        x, v = start(x, v, g, inv_mass, dt, integrator, temperature, friction, nz)
        g = force(x)
        v = kick(v, g, inv_mass, dt)
        xs.append(x)
        vs.append(v)
    return np.stack(xs), np.stack(vs)
