"""The NEB oracle (oracle/neb_oracle.py) and the NEB entry points without a GPU: ASE's per-image loop against the
alpha / beta / gamma form the device uses, the Mueller-Brown saddles, the improved tangent's equal spacing, the LJ3
saddle, ``optimize.interpolate``, the struct layout and argument checks that return before any CUDA call."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
from scipy.optimize import root

import oracle.fire_oracle as fo
import oracle.neb_oracle as no
from helpers import ROOT


def _random_band(rng, n, A, energies):
    x = rng.standard_normal((n, A, 3))
    F = rng.standard_normal((n - 2, A, 3))
    scale = np.ones(A)
    scale[::4] = 0.0
    F[:, scale == 0] = 0.0
    x[:, scale == 0] = x[0, scale == 0]
    return x, F, scale, energies


@pytest.mark.parametrize("method", no.METHODS)
def test_the_two_forms_agree(method):
    """Random bands whose energies reach every tangent branch (rising and falling through an image, maxima, minima,
    equal energies), coincident images (a zero tangent), per-spring k and fixed atoms: 1e-12 relative."""
    rng = np.random.default_rng(5)
    cases = []
    for _ in range(20):
        n = int(rng.integers(3, 10))
        cases.append(_random_band(rng, n, 9, rng.standard_normal(n)))
    x, F, s, _ = _random_band(rng, 7, 9, None)
    cases.append((x, F, s, np.array([0.0, 1.0, 1.0, 1.0, 2.0, 2.0, 0.5])))       # equal energies
    x, F, s, _ = _random_band(rng, 6, 9, None)
    x[3] = x[1]                                                                  # x_{i+1} = x_{i-1} at i = 2
    cases.append((x, F, s, np.array([0.0, 1.0, 3.0, 1.0, 0.5, 0.0])))
    x, F, s, _ = _random_band(rng, 5, 9, None)
    cases.append((x, F, s, np.array([0.0, 1.0, 1.0, 1.0, 0.0])))                  # flat: |tau| = 0 (improved)
    branches = set()
    for x, F, s, E in cases:
        n = len(x)
        for k in (0.1, rng.uniform(0.05, 2.0, n - 1)):
            for climb in (False, True):
                ref = no.get_forces(x, E, F, k, method, climb, s)
                got = no.get_forces_dots(x, E, F, k, method, climb, s, branches)
                assert np.abs(got - ref).max() <= 1e-12 * np.abs(ref).max()
                assert (got[:, s == 0] == 0).all()
    assert branches >= {"up", "down", "max", "min", "flat", "zero"}, branches


def _mb_band(a, b, n):
    x = np.zeros((n, 1, 3))
    s = np.linspace(0.0, 1.0, n)
    x[:, 0, 0] = a[0] + s * (b[0] - a[0])
    x[:, 0, 1] = a[1] + s * (b[1] - a[1])
    return x


def _mb_saddle(guess):
    r = root(lambda p: no.muller_brown(np.array([p[0], p[1], 0.0]))[1][:2], guess, tol=1e-12)
    assert np.abs(r.fun).max() < 1e-9
    return r.x, float(no.muller_brown(np.array([r.x[0], r.x[1], 0.0]))[0])


@pytest.mark.parametrize("method", no.METHODS)
@pytest.mark.parametrize("ends,guess,known", [
    (((-0.5582, 1.4417), (0.6235, 0.0280)), (-0.82, 0.62), (-0.82200, 0.62431, -40.66484)),
    (((-0.0500, 0.4667), (0.6235, 0.0280)), (0.21, 0.29), (0.21249, 0.29299, -72.24894))])
def test_mueller_brown_saddles(method, ends, guess, known):
    """A 9-image band relaxed to 0.05, then climbing to 1e-3: the climbing image sits on the saddle that
    scipy.optimize.root finds on grad V."""
    p, e = _mb_saddle(guess)
    assert np.abs(p - known[:2]).max() < 1e-5 and abs(e - known[2]) < 1e-5
    x = _mb_band(*ends, 9)
    x, E, c = no.run(x, no.mb_energy_grad, 1.0, fo.params(0.05, maxstep=0.05), 3000, method)
    assert c >= 0
    x, E, c = no.run(x, no.mb_energy_grad, 1.0, fo.params(1e-3, maxstep=0.05), 6000, method, climb=True)
    assert c >= 0
    i = no.imax_of(E)
    assert np.abs(x[i, 0, :2] - p).max() < 1e-4
    assert abs(E[i] - e) < 1e-6


def test_improved_tangent_spaces_images_equally():
    """Without climbing, equal springs leave |t+| = |t-| at convergence and the perpendicular force below fmax."""
    x = _mb_band((-0.5582, 1.4417), (0.6235, 0.0280), 7)
    x, E, c = no.run(x, no.mb_energy_grad, 5.0, fo.params(1e-4, maxstep=0.05), 20000, "improvedtangent")
    assert c >= 0
    t = np.linalg.norm(np.diff(x[:, 0], axis=0), axis=1)
    assert np.abs(t - t.mean()).max() <= 1e-3 * t.mean()
    F = -np.stack([no.mb_energy_grad(xi)[1] for xi in x[1:-1]])
    f = no.get_forces(x, E, F, 5.0, "improvedtangent")
    assert no.fmax(f) < 1e-4


def test_lj3_climbing_image_reaches_the_collinear_saddle():
    """Three LJ atoms in the z = 0 plane: atom 1 moves from one side of the 0-2 axis to its mirror image; the climbing
    image reaches E* = min_r [2 V(r) + V(2 r)] with equal, collinear bonds."""
    es, rs = no.lj3_saddle()
    assert abs(es + 2.031124) < 1e-6 and abs(rs - 1.121030) < 1e-6

    def eg(x):
        return fo.lj(x)
    r0 = 2.0 ** (1.0 / 6.0)
    a = np.array([[0.0, 0.0, 0.0], [0.5 * r0, 0.8660254 * r0, 0.0], [r0, 0.0, 0.0]])
    b = a.copy()
    b[1, 1] *= -1.0
    x = a[None] + np.linspace(0.0, 1.0, 8)[:, None, None] * (b - a)[None]
    x, E, c = no.run(x, eg, 0.1, fo.params(1e-5, maxstep=0.05), 20000, "aseneb", climb=True)
    assert c >= 0
    i = no.imax_of(E)
    assert abs(E[i] - es) < 1e-6
    d01, d12 = np.linalg.norm(x[i, 1] - x[i, 0]), np.linalg.norm(x[i, 2] - x[i, 1])
    assert abs(d01 - d12) < 1e-4 and abs(np.linalg.norm(x[i, 2] - x[i, 0]) - d01 - d12) < 1e-6


def test_interpolate():
    from torchani_b200.optimize import interpolate
    a, b = np.zeros((2, 3)), np.array([[1.0, 2.0, 3.0], [9.5, 0.0, 0.0]])
    im = interpolate(a, b, 5)
    assert im.shape == (5, 2, 3) and np.array_equal(im[0], a) and np.allclose(im[-1], b)
    assert np.allclose(im[2], 0.5 * b)
    cell = np.eye(3) * 10.0
    im = interpolate(a, b, 3, cell=cell, mic=True)
    assert np.allclose(im[-1, 1], [-0.5, 0.0, 0.0])
    with pytest.raises(ValueError):
        interpolate(a, b, 1)


def test_struct_layout_and_argument_checks(tmp_path):
    from torchani_b200 import _lib
    S = _lib.NebState
    prog = tmp_path / "neb.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "ani_b200.h"\n'
                    'int main(){printf("%zu %zu %zu %zu %d %d\\n", sizeof(ani_neb_state), offsetof(ani_neb_state, '
                    'endpoints), offsetof(ani_neb_state, dots), offsetof(ani_neb_state, method), ANI_NEB_RECORD, '
                    'ANI_NEB_DOTS);return 0;}\n')
    exe = tmp_path / "neb"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    out = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert out == [C.sizeof(S), S.endpoints.offset, S.dots.offset, S.method.offset, _lib.ANI_NEB_RECORD,
                   _lib.ANI_NEB_DOTS]
    L = _lib.lib()
    st = S()
    assert L.ani_b200_neb_step(None, None, None, None, None, None) == -1
    assert L.ani_b200_neb_step(C.byref(st), None, None, None, None, None) == -1
    assert L.ani_b200_neb_project(C.byref(st), None, None, None) == -1
    assert L.ani_b200_neb_init(C.byref(st), None, 0, 1, None, None) == -1
    assert L.ani_b200_neb_step_cells(C.byref(st), None, None, None, None, None) == -1


def test_near_folded_band_error_is_bounded_by_the_cancellation():
    """Where t+ is close to -t- and alpha close to beta, tau.tau = alpha^2 a + 2 alpha beta c + beta^2 b cancels: the
    five-dot form then agrees with ASE's loop to eps (alpha^2 a + beta^2 b + 2 |alpha beta c|) / tau.tau relative (times a
    small constant), not to 1e-12.  Both sides of that statement are checked."""
    rng = np.random.default_rng(9)
    eps = np.finfo(np.float64).eps
    worst = 0.0
    for fold in (1e-2, 1e-4, 1e-6):
        x, F, s, _ = _random_band(rng, 5, 9, None)
        x[3] = x[1] + fold * rng.standard_normal(x[1].shape) * (s != 0)[:, None]
        E = np.array([0.0, 1.0, 2.0, 1.0 + 1e-3, 0.5])   # improved tangent at i = 2: alpha = 1, beta = 1 - 1e-3
        ref = no.get_forces(x, E, F, 0.1, "improvedtangent", False, s)
        got = no.get_forces_dots(x, E, F, 0.1, "improvedtangent", False, s)
        t = no.springs(x, s)
        al, be = no.coefficients(2, no.imax_of(E), E[1], E[2], E[3], "improvedtangent")
        a, b, c = (t[1] * t[1]).sum(), (t[2] * t[2]).sum(), (t[1] * t[2]).sum()
        tt = al * al * a + 2 * al * be * c + be * be * b
        cond = (al * al * a + be * be * b + 2 * abs(al * be * c)) / tt
        err = np.abs(got[1] - ref[1]).max() / np.abs(ref).max()
        assert err <= 64 * eps * cond, (fold, err, cond)
        worst = max(worst, err)
    assert worst > 1e-12   # the limit is real: the most folded band is beyond the 1e-12 of well-conditioned images
