"""Float64 restatement of the device NEB (csrc/neb.cu, torchani_b200/optimize.py NEB): ASE's ``NEB.get_forces`` per
image for the methods "aseneb" and "improvedtangent", with and without the climbing image, written literally as ASE's
loop over images (``get_forces``), and the alpha / beta / gamma form the device uses (``get_forces_dots``); FIRE over
the concatenated rows of a band's interior images reuses ``fire_oracle.step``.  Also the known answers the tests relax
to: the Mueller-Brown surface and the collinear LJ3 saddle.

A band is x (n, A, 3) with the endpoints x[0], x[n - 1]; forces F (n - 2, A, 3) eV / A of the interior images (zero on
fixed and padding atoms, scale == 0, where t is zeroed too); energies E (n,); springs k (n - 1,)."""
import math

import numpy as np

from oracle import fire_oracle

METHODS = ("aseneb", "improvedtangent")


def imax_of(energies) -> int:
    """1 + the first index of the largest interior energy (ASE's argsort(...)[-1] leaves ties unspecified)."""
    return 1 + int(np.argmax(np.asarray(energies)[1:-1]))


def springs(x, scale):
    """t[j] = x[j + 1] - x[j] (ASE's Spring.t), zeroed on atoms with scale == 0."""
    t = np.diff(np.asarray(x, dtype=np.float64), axis=0)
    return np.where((np.asarray(scale) != 0)[None, :, None], t, 0.0)


def get_forces(x, energies, forces, k, method="aseneb", climb=False, scale=None):
    """ASE's NEB.get_forces loop, image by image (the contract of DESIGN §4.15; |tau| = 0 gives u = 0)."""
    x = np.asarray(x, dtype=np.float64)
    n = len(x)
    scale = np.ones(x.shape[1]) if scale is None else np.asarray(scale)
    t = springs(x, scale)
    E = np.asarray(energies, dtype=np.float64)
    k = np.broadcast_to(np.asarray(k, dtype=np.float64), (n - 1,))
    imax = imax_of(E)
    out = np.array(forces, dtype=np.float64)
    for i in range(1, n - 1):
        t1, t2, k1, k2 = t[i - 1], t[i], k[i - 1], k[i]
        if method == "aseneb":
            tangent = t2.copy() if i < imax else (t1.copy() if i > imax else t1 + t2)
        else:
            if E[i + 1] > E[i] > E[i - 1]:
                tangent = t2.copy()
            elif E[i + 1] < E[i] < E[i - 1]:
                tangent = t1.copy()
            else:
                dmax = max(abs(E[i + 1] - E[i]), abs(E[i - 1] - E[i]))
                dmin = min(abs(E[i + 1] - E[i]), abs(E[i - 1] - E[i]))
                tangent = t2 * dmax + t1 * dmin if E[i + 1] > E[i - 1] else t2 * dmin + t1 * dmax
            nrm = np.linalg.norm(tangent)
            tangent = tangent / nrm if nrm > 0 else np.zeros_like(tangent)
        f = out[i - 1]
        tf = np.vdot(f, tangent)
        if climb and i == imax:
            if method == "aseneb":
                f -= 2 * tf / (np.vdot(tangent, tangent) or 1.0) * tangent
            else:
                f -= 2 * tf * tangent
        elif method == "aseneb":
            factor = tangent / (np.vdot(tangent, tangent) or 1.0)
            f -= tf * factor
            f -= np.vdot(t1 * k1 - t2 * k2, tangent) * factor
        else:
            f -= tf * tangent
            f += (np.linalg.norm(t2) * k2 - np.linalg.norm(t1) * k1) * tangent
    return out


def coefficients(i, imax, e0, e1, e2, method):
    """(alpha, beta) of tau = alpha t- + beta t+ at image i with energies e0, e1, e2 of images i - 1, i, i + 1."""
    if method == "aseneb":
        return (0.0 if i < imax else 1.0), (0.0 if i > imax else 1.0)
    if e2 > e1 > e0:
        return 0.0, 1.0
    if e2 < e1 < e0:
        return 1.0, 0.0
    dmax, dmin = max(abs(e2 - e1), abs(e0 - e1)), min(abs(e2 - e1), abs(e0 - e1))
    return (dmin, dmax) if e2 > e0 else (dmax, dmin)


def gammas(dots, alpha, beta, km, kp, method, climbing):
    """(gamma-, gamma+) of f = F + gamma- t- + gamma+ t+ from {a, b, c, p, q} = {t-.t-, t+.t+, t-.t+, F.t-, F.t+}."""
    a, b, c, p, q = dots
    ft = alpha * p + beta * q
    tt = alpha * alpha * a + 2.0 * alpha * beta * c + beta * beta * b
    if method == "aseneb":
        m = tt if tt != 0.0 else 1.0
        g = -2.0 * ft / m if climbing else -(ft + km * (alpha * a + beta * c) - kp * (alpha * c + beta * b)) / m
    elif tt > 0.0:
        g = -2.0 * ft / tt if climbing else -ft / tt + (kp * math.sqrt(b) - km * math.sqrt(a)) / math.sqrt(tt)
    else:
        g = 0.0
    return g * alpha, g * beta


def get_forces_dots(x, energies, forces, k, method="aseneb", climb=False, scale=None, branches=None):
    """The device's form of ``get_forces``: five dot products per image, then f = F + gamma- t- + gamma+ t+.
    ``branches`` (a set) collects the tangent branch of every image: "up", "down", "max", "min", "flat", "zero"."""
    x = np.asarray(x, dtype=np.float64)
    n = len(x)
    scale = np.ones(x.shape[1]) if scale is None else np.asarray(scale)
    t = springs(x, scale)
    E = np.asarray(energies, dtype=np.float64)
    k = np.broadcast_to(np.asarray(k, dtype=np.float64), (n - 1,))
    imax = imax_of(E)
    F = np.asarray(forces, dtype=np.float64)
    out = np.empty_like(F)
    for i in range(1, n - 1):
        tm, tp, f = t[i - 1], t[i], F[i - 1]
        dots = ((tm * tm).sum(), (tp * tp).sum(), (tm * tp).sum(), (f * tm).sum(), (f * tp).sum())
        al, be = coefficients(i, imax, E[i - 1], E[i], E[i + 1], method)
        if branches is not None:
            e0, e1, e2 = E[i - 1], E[i], E[i + 1]
            branches.add("up" if e2 > e1 > e0 else "down" if e2 < e1 < e0 else "flat" if e0 == e1 == e2 else
                         "max" if e1 >= max(e0, e2) else "min")
            if al * al * dots[0] + 2 * al * be * dots[2] + be * be * dots[1] == 0.0:
                branches.add("zero")
        gm, gp = gammas(dots, al, be, k[i - 1], k[i], method, climb and i == imax)
        out[i - 1] = f + gm * tm + gp * tp
    return out


def fmax(f) -> float:
    """The band's fmax: the largest row norm of its NEB forces."""
    return math.sqrt((np.asarray(f) ** 2).sum(-1).max())


def step(x, v, scalars, energies, forces, k, par, t, method="aseneb", climb=False, scale=None, converged=False):
    """One device NEB step of one band: x (n, A, 3) with endpoints, v (n - 2, A, 3), FIRE scalars {dt, a, n}, the
    interior forces (n - 2, A, 3) eV / A and all n energies.  FIRE is ``fire_oracle.step`` over the band's rows.
    Returns x(t+1) (n, A, 3), v', the scalars of t + 1, fmax(t), whether the band converges at t, and imax."""
    f = get_forces(x, energies, forces, k, method, climb, scale)
    m, A = f.shape[:2]
    x1, v1, sc, fm, conv = fire_oracle.step(np.asarray(x[1:-1]).reshape(-1, 3), np.asarray(v).reshape(-1, 3),
                                            scalars, -f.reshape(-1, 3), np.ones(m * A), par, t, converged)
    xn = np.array(x, dtype=np.float64)
    xn[1:-1] = x1.reshape(m, A, 3)
    return xn, v1.reshape(m, A, 3), sc, fm, conv, imax_of(energies)


def run(x, energy_grad, k, par, steps, method="aseneb", climb=False, scale=None):
    """Relax one band (x (n, A, 3)) from v = 0 under FIRE; energy_grad(x_i) -> (E, dE/dx) in eV and eV / A.
    Returns (x, E (n,), the step it converged at or -1)."""
    x = np.array(x, dtype=np.float64)
    n = len(x)
    scale = np.ones(x.shape[1]) if scale is None else np.asarray(scale)
    v, sc = np.zeros_like(x[1:-1]), fire_oracle.init(par)
    e_end = [energy_grad(x[0])[0], energy_grad(x[-1])[0]]
    E = np.zeros(n)
    for t in range(steps):
        eg = [energy_grad(xi) for xi in x[1:-1]]
        E = np.array([e_end[0]] + [e for e, _ in eg] + [e_end[1]])
        F = -np.stack([g for _, g in eg]) * scale[None, :, None]
        x, v, sc, _, conv, _ = step(x, v, sc, E, F, k, par, t, method, climb, scale)
        if conv:
            return x, E, t
    return x, E, -1


# -- Mueller-Brown (Mueller & Brown, Theor. Chim. Acta 53, 75 (1979)): one atom in the z = 0 plane -------------------
MB_A = np.array([-200.0, -100.0, -170.0, 15.0])
MB_a = np.array([-1.0, -1.0, -6.5, 0.7])
MB_b = np.array([0.0, 0.0, 11.0, 0.6])
MB_c = np.array([-10.0, -10.0, -6.5, 0.7])
MB_X = np.array([1.0, 0.0, -0.5, -1.0])
MB_Y = np.array([0.0, 0.5, 1.5, 1.0])


def muller_brown(p):
    """Energy and gradient (3,) of the Mueller-Brown surface at the (x, y) of p (any leading shape (..., 3))."""
    p = np.asarray(p, dtype=np.float64)
    x, y = p[..., 0:1], p[..., 1:2]
    dx, dy = x - MB_X, y - MB_Y
    e = MB_A * np.exp(MB_a * dx * dx + MB_b * dx * dy + MB_c * dy * dy)
    gx = (e * (2 * MB_a * dx + MB_b * dy)).sum(-1)
    gy = (e * (MB_b * dx + 2 * MB_c * dy)).sum(-1)
    return e.sum(-1), np.stack([gx, gy, np.zeros_like(gx)], -1)


def mb_energy_grad(xi):
    """energy_grad of ``run`` for a one-atom image on the Mueller-Brown surface (the z component held at 0)."""
    e, g = muller_brown(xi[0])
    return float(e), g.reshape(1, 3)


# -- LJ3: the collinear saddle of three Lennard-Jones atoms ----------------------------------------------------------
def lj_pair(r, sigma=1.0, eps=1.0):
    s6 = (sigma / r) ** 6
    return 4.0 * eps * (s6 * s6 - s6)


def lj3_saddle(sigma=1.0, eps=1.0):
    """(E*, r*): the collinear LJ3 saddle, min over r of 2 V(r) + V(2 r)."""
    from scipy.optimize import minimize_scalar
    res = minimize_scalar(lambda r: 2 * lj_pair(r, sigma, eps) + lj_pair(2 * r, sigma, eps),
                          bounds=(0.9 * sigma, 1.3 * sigma), method="bounded", options={"xatol": 1e-12})
    return float(res.fun), float(res.x)


__all__ = ["METHODS", "imax_of", "springs", "get_forces", "coefficients", "gammas", "get_forces_dots", "fmax", "step",
           "run", "muller_brown", "mb_energy_grad", "lj_pair", "lj3_saddle"]
