"""The float64 variable-cell FIRE oracle (oracle/cell_fire_oracle.py) against autograd of the enthalpy and against a
lattice constant known from a one-dimensional minimisation, its projections, and the cell entry points of the C-ABI and
the CellFIRE driver without a GPU (struct layout, argument checks that return before any CUDA call)."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest
import torch
from scipy.optimize import minimize_scalar

import oracle.ani_oracle as orc
import oracle.cell_fire_oracle as co
import oracle.fire_oracle as fo
import oracle.lj_coulomb_oracle as ljo
from helpers import ROOT

RC = 2.5   # sigma: the smooth envelope's cutoff of the reduced-unit LJ crystal


def spec(rc=RC):
    one, zero = torch.ones(1, dtype=torch.float64), torch.zeros(1, dtype=torch.float64)
    return ljo.Spec("lj", rc, "smooth", one, one, zero, zero)


def fcc(a, reps=(1, 1, 1)):
    base = np.array([[0, 0, 0], [0, 0.5, 0.5], [0.5, 0, 0.5], [0.5, 0.5, 0]])
    cells = np.array([(i, j, k) for i in range(reps[0]) for j in range(reps[1]) for k in range(reps[2])])
    return a * (cells[:, None] + base[None]).reshape(-1, 3), a * np.diag(np.asarray(reps, dtype=np.float64))


def energy_grad_virial(r, h, sp=None):
    """E, dE/dr and W_ab = sum (dE/dDelta)_a Delta_b of the reduced-unit LJ crystal (lj_coulomb_oracle)."""
    A = len(r)
    species = torch.zeros(1, A, dtype=torch.long)
    out = ljo.compute(sp or spec(), species, torch.as_tensor(r)[None], torch.as_tensor(h),
                      torch.ones(3, dtype=torch.bool), neighborlist="all_pairs", stress=True)
    vol = abs(np.linalg.det(h))
    return (float(out["energy"][0]), -out["forces"][0].numpy(), (out["stress"].numpy() * vol).T)


def enthalpy_torch(u, d, h0, c, p0, sp=None):
    """H(u, d) = E(u F^T, h0 F^T) + p0 V with F = expm(d / c), differentiable in u and d (float64)."""
    F = torch.matrix_exp(d / c)
    r, h = u @ F.T, h0 @ F.T
    species = torch.zeros(1, len(u), dtype=torch.long)
    nb = orc.all_pairs(RC, species, r[None], h, torch.ones(3, dtype=torch.bool))
    return ljo.energies_from_neighbors(sp or spec(), species, nb).sum() + p0 * torch.det(h).abs()


def sheared_crystal(seed=0, noise=0.03):
    rng = np.random.default_rng(seed)
    r, h = fcc(1.6, (2, 1, 1))
    shear = np.array([[1.02, 0.05, -0.03], [0.0, 0.97, 0.04], [0.02, 0.0, 1.03]])
    h0 = h @ shear
    return r @ shear + noise * rng.standard_normal(r.shape), h0


# ------------------------------------------------------------------------------------------------------------------
# the forces are -dH
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p0,d_scale", [(0.0, 0.0), (0.0, 0.03), (1.5, 0.03), (-0.7, 0.05)])
def test_forces_are_minus_grad_enthalpy(p0, d_scale):
    """g = F^T f and Phi = D_expm(L^T)[G] / c equal -dH/du and -dH/dd from autograd of H(u, d), for a sheared 8-atom
    cell with displaced atoms, at d = 0 and d != 0 (a strained and rotated F), at p0 = 0 and p0 != 0."""
    rng = np.random.default_rng(7)
    r0, h0 = sheared_crystal()
    c = 8.0
    d = d_scale * c * rng.standard_normal((3, 3))
    F = co.deformation(d, c)
    u = r0 @ np.linalg.inv(F).T
    ut = torch.tensor(u, requires_grad=True)
    dt = torch.tensor(d, requires_grad=True)
    H = enthalpy_torch(ut, dt, torch.tensor(h0), c, p0)
    gu, gd = torch.autograd.grad(H, (ut, dt))
    r, h = co.positions(u, F), h0 @ F.T
    e, grad, W = energy_grad_virial(r, h)
    g = -grad @ F
    phi, vol = co.cell_force(d, W, p0, h0, c)
    assert vol == pytest.approx(abs(np.linalg.det(h)), rel=1e-14)
    assert float(H.detach()) == pytest.approx(e + p0 * vol, rel=1e-13)
    assert np.abs(g + gu.numpy()).max() <= 1e-10 * np.abs(g).max()
    assert np.abs(phi + gd.numpy()).max() <= 1e-10 * np.abs(phi).max()
    assert np.abs(phi).max() > 1e-3   # a cell force to compare


def test_adjoint_frechet_is_the_nine_direction_sum():
    rng = np.random.default_rng(1)
    for scale in (1e-3, 0.1, 0.8):
        L, G = scale * rng.standard_normal((3, 3)), rng.standard_normal((3, 3))
        ref = co.nine_directions(L, G)
        assert np.abs(co.adjoint_frechet(L, G) - ref).max() <= 1e-13 * np.abs(ref).max()
    # the transpose matters: for a non-normal L the plain derivative at L is another matrix
    L = np.array([[0.0, 0.6, 0.0], [0.0, 0.0, 0.3], [0.1, 0.0, 0.0]])
    assert np.abs(expm_frechet_plain(L, G) - co.nine_directions(L, G)).max() > 1e-3


def expm_frechet_plain(L, G):
    from scipy.linalg import expm_frechet
    return expm_frechet(L, G, compute_expm=False)


# ------------------------------------------------------------------------------------------------------------------
# projections
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("projection", [co.HYDROSTATIC, co.CONSTANT_VOLUME])
def test_projections(projection):
    """40 steps on the sheared crystal at p0 = 0.5: hydrostatic strain keeps L a multiple of I (the shape of h0, h h^T
    proportional to h0 h0^T); constant volume keeps tr L = 0, so det F = 1."""
    r0, h0 = sheared_crystal(seed=3)
    c, p0 = 8.0, 0.5
    par = fo.params(0.0, maxstep=0.05)
    u, v, d, vc, sc = r0.copy(), np.zeros_like(r0), np.zeros((3, 3)), np.zeros((3, 3)), fo.init(par)
    for t in range(40):
        F = co.deformation(d, c)
        e, g, W = energy_grad_virial(co.positions(u, F), h0 @ F.T)
        u, v, d, vc, sc, _, _, _ = co.step(u, v, d, vc, sc, g, W, e, h0, p0, c, par, t, np.ones(len(u)),
                                            projection, unit=1.0)
    L = d / c
    F = co.deformation(d, c)
    if projection == co.HYDROSTATIC:
        assert abs(L[0, 0]) > 1e-3, "the cell did not move"
        assert np.abs(L - L[0, 0] * np.eye(3)).max() <= 1e-15
        h = h0 @ F.T
        gram, gram0 = h @ h.T, h0 @ h0.T
        assert np.abs(gram / gram[0, 0] - gram0 / gram0[0, 0]).max() <= 1e-13
    else:
        assert np.abs(L - np.diag(np.diag(L))).max() > 1e-3, "the cell did not move"
        assert abs(np.trace(L)) <= 1e-15
        assert abs(np.linalg.det(F) - 1.0) <= 1e-13


def test_projection_is_the_isotropic_or_traceless_part():
    rng = np.random.default_rng(2)
    phi = rng.standard_normal((3, 3))
    iso, dev = co.project(phi, co.HYDROSTATIC), co.project(phi, co.CONSTANT_VOLUME)
    assert np.allclose(iso + dev, phi, rtol=0, atol=1e-15) and abs(np.trace(dev)) <= 1e-15
    assert np.array_equal(co.project(phi, co.NONE), phi)


# ------------------------------------------------------------------------------------------------------------------
# a known lattice constant
# ------------------------------------------------------------------------------------------------------------------
def lattice_minimum(p0):
    """The fcc lattice constant minimising E(a) + p0 a^3 per conventional cell (4 atoms)."""
    def h(a):
        r, cell = fcc(a)
        return energy_grad_virial(r, cell)[0] + p0 * a ** 3
    res = minimize_scalar(h, bracket=(1.45, 1.55, 1.65), tol=1e-12)
    return res.x


@pytest.mark.parametrize("p0", [0.0, 2.0])
def test_sheared_fcc_relaxes_to_the_cubic_lattice_constant(p0):
    """A strained and sheared 4-atom fcc cell with displaced atoms relaxes (fmax 1e-9 in reduced units) to a cubic cell:
    its Gram matrix h h^T is a^2 I with a the one-dimensional minimum of E(a) + p0 a^3 (the same smooth envelope),
    to 1e-6 relative (minimize_scalar's own precision is ~1e-8)."""
    a_ref = lattice_minimum(p0)
    rng = np.random.default_rng(5)
    r, h = fcc(1.52)
    shear = np.array([[1.04, 0.06, 0.0], [-0.02, 0.97, 0.03], [0.01, 0.0, 1.02]])
    h0 = h @ shear
    u = r @ shear + 0.02 * rng.standard_normal(r.shape)
    par = fo.params(1e-9, maxstep=0.1)
    rf, hf, H, t = co.run(u, h0, energy_grad_virial, par, 3000, 4.0, p0)
    assert 0 < t < 3000, t
    gram = hf @ hf.T
    assert np.abs(gram / a_ref ** 2 - np.eye(3)).max() <= 2e-6, (gram, a_ref)
    e_ref = energy_grad_virial(*fcc(a_ref))[0] + p0 * a_ref ** 3
    assert H == pytest.approx(e_ref, rel=1e-9)
    if p0 > 0:
        assert a_ref < lattice_minimum(0.0) - 1e-3   # compressed


# ------------------------------------------------------------------------------------------------------------------
# the C-ABI and the driver without a GPU
# ------------------------------------------------------------------------------------------------------------------
def test_opt_cell_layout_matches_header(tmp_path):
    from torchani_b200 import _lib
    prog = tmp_path / "cell.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "ani_b200.h"\n'
                    'int main(){printf("%zu %zu %zu %zu %zu %zu %d %d %d\\n", sizeof(ani_opt_cell),'
                    ' offsetof(ani_opt_cell, record), offsetof(ani_opt_cell, cell_stride),'
                    ' offsetof(ani_opt_cell, virial_slots), offsetof(ani_opt_cell, projection),'
                    ' offsetof(ani_opt_cell, pad_), ANI_OPT_CELL_MASTER, ANI_OPT_CELL_PARAMS,'
                    ' ANI_OPT_CELL_RECORD);return 0;}\n')
    exe = tmp_path / "cell"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    out = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    S = _lib.OptCell
    assert out == [C.sizeof(S), S.record.offset, S.cell_stride.offset, S.virial_slots.offset, S.projection.offset,
                   S.pad_.offset, _lib.ANI_OPT_CELL_MASTER, _lib.ANI_OPT_CELL_PARAMS, _lib.ANI_OPT_CELL_RECORD]


def test_opt_cell_argument_validation_without_gpu():
    """Bad arguments are rejected before any CUDA call (the pointers are host dummies)."""
    from torchani_b200 import _lib
    L = _lib.lib()
    buf = (C.c_char * 4096)()
    h = C.cast(buf, C.c_void_p).value

    def state(**kw):
        s = _lib.OptState()
        for k in ("x", "v", "force_scale", "params", "scalars", "counter", "conv_step", "record", "partials"):
            setattr(s, k, h)
        s.n_conf, s.n_per_conf, s.record_rows = 1, 4, 4
        for k, v in kw.items():
            setattr(s, k, v)
        return s

    def cell(**kw):
        q = _lib.OptCell()
        for k in ("master", "h0", "params", "cell_out", "virial", "cell_force", "record"):
            setattr(q, k, h)
        q.cell_stride, q.virial_slots, q.projection = 9, _lib.ANI_VIRIAL_SLOTS, 0
        for k, v in kw.items():
            setattr(q, k, v)
        return q

    def step(s=None, q=None, grad=h, energies=h, coords=h):
        return L.ani_b200_opt_cell_step(C.byref(s or state()), C.byref(q or cell()), grad, energies, coords, None)

    for bad in ({"master": None}, {"h0": None}, {"params": None}, {"cell_out": None}, {"virial": None},
                {"cell_force": None}, {"record": None}, {"cell_stride": 8}, {"virial_slots": 0}, {"projection": 3},
                {"projection": -1}):
        assert step(q=cell(**bad)) == -1, bad
        assert L.ani_b200_opt_cell_init(C.byref(state()), C.byref(cell(**bad)), 1, h, None) == -1, bad
    for bad in ({"x": None}, {"conv_step": None}, {"record": None}, {"partials": None}, {"n_conf": 0},
                {"record_rows": 0}):
        assert step(s=state(**bad)) == -1, bad
    assert step(grad=None) == -1 and step(energies=None) == -1 and step(coords=None) == -1
    assert step(s=state(n_conf=70000)) != 0
    assert L.ani_b200_opt_cell_step(C.byref(state()), None, h, h, h, None) == -1
    assert L.ani_b200_opt_cell_init(C.byref(state()), None, 1, h, None) == -1
    assert L.ani_b200_opt_cell_init(C.byref(state()), C.byref(cell()), 1, None, None) == -1


class _CpuModel:
    def buffers(self):
        yield torch.zeros(1)


@pytest.mark.parametrize("kw,match", [
    (dict(cell=None), "periodic"), (dict(pbc=False), "periodic"), (dict(pbc=[True, True, False]), "periodic"),
    (dict(fixed=np.zeros(3, dtype=bool)), "fixed"), (dict(pressure=math.nan), "pressure"),
    (dict(pressure=[1.0, math.inf]), "pressure"), (dict(cell_factor=0.0), "cell_factor"),
    (dict(cell_factor=-1.0), "cell_factor"), (dict(hydrostatic_strain=True, constant_volume=True), "exclusive"),
    (dict(cell=np.diag([10.0, 10.0, 0.0])), "volume"), (dict(cell=np.full((3, 3), math.nan)), "volume"),
    (dict(cell=np.eye(2)), "cell must be"), (dict(dt=0.0), "dt"), (dict(steps_per_replay=0), "steps_per_replay"),
    (dict(), "CUDA")])
def test_cell_fire_rejections_without_gpu(kw, match):
    from torchani_b200 import optimize
    args = dict(cell=np.eye(3) * 10.0)
    args.update(kw)
    sp = np.zeros(3, dtype=np.int64) if "pressure" not in kw or np.ndim(kw["pressure"]) == 0 else \
        np.zeros((2, 3), dtype=np.int64)
    with pytest.raises(ValueError, match=match):
        optimize.CellFIRE(_CpuModel(), sp, np.zeros(sp.shape + (3,)), **args)


def test_bar_constant():
    """1 eV / A^3 = 1.6021766208e6 bar (CODATA 2014, the value ASE's units give)."""
    from torchani_b200 import optimize
    ev_a3_in_bar = 1.0 / (optimize.BAR_TO_HARTREE_A3 * optimize.HARTREE_TO_EV)
    assert ev_a3_in_bar == pytest.approx(1.6021766208e6, rel=1e-12)
