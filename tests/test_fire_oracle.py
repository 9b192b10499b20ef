"""The float64 FIRE oracle (oracle/fire_oracle.py) on a problem with a known answer and on the rules it restates, the
device optimiser's constants, and the opt entry points of the C-ABI and the Python driver without a GPU (struct layout,
argument checks that return before any CUDA call)."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import oracle.fire_oracle as fo
from helpers import ROOT


def _lj13(n, seed=0, noise=0.08):
    rng = np.random.default_rng(seed)
    return [fo.icosahedron() + noise * rng.standard_normal((13, 3)) for _ in range(n)]


def test_hartree_to_ev_is_the_oracles():
    from torchani_b200 import grad, optimize
    assert optimize.HARTREE_TO_EV == grad.HARTREE_TO_EV
    assert grad.HARTREE_TO_EV == pytest.approx(fo.HARTREE_EV, rel=1e-15)


def test_lj13_reaches_the_global_minimum():
    """Eight perturbed icosahedra (reduced units, noise 0.08 sigma) reach E = -44.326801 eps at fmax 1e-4; near the
    minimum E - E_min ~ fmax^2 / (2 k), far below the 1e-6 the known value is given to."""
    for x0 in _lj13(8):
        x, e, t = fo.run(x0, fo.lj, fo.params(1e-4), 5000)
        assert 0 < t < 1000, t
        assert e == pytest.approx(fo.E_LJ13, abs=1e-6)
        assert np.sqrt((fo.lj(x)[1] ** 2).sum(1)).max() < 1e-4


def test_first_step_does_not_shrink_dt():
    """At t = 0 FIRE only does v = dt f: with v = 0 the power P is 0, which at t > 0 would mean an uphill step (dt *=
    fdec, a = astart)."""
    x = _lj13(1, seed=1)[0]
    par = fo.params(0.0)
    g = fo.lj(x)[1]
    sc0 = fo.init(par)
    x1, v1, sc, _, _ = fo.step(x, np.zeros_like(x), sc0, g, np.ones(13), par, 0)
    assert np.array_equal(sc, sc0)
    assert np.allclose(v1, -par[0] * g, rtol=1e-15, atol=0)
    _, _, sc_later, _, _ = fo.step(x, np.zeros_like(x), sc0, g, np.ones(13), par, 1)
    assert sc_later[0] == par[0] * par[5] and sc_later[1] == par[6] and sc_later[2] == 0.0


def test_maxstep_clamp_and_three_sum_norm():
    """The step's norm from the sums P, F2, V2 equals the direct |dt v'| (to 1e-12), and the whole conformer's step is
    scaled down to maxstep when longer (a global norm, not atom by atom)."""
    rng = np.random.default_rng(3)
    x = rng.standard_normal((13, 3))
    v = rng.standard_normal((13, 3))
    g = -v - 0.3 * rng.standard_normal((13, 3))   # P > 0
    par = fo.params(0.0, maxstep=10.0)
    sc = np.array([0.1, 0.1, 0.0])
    x1, v1, sc1, _, _ = fo.step(x, v, sc, g, np.ones(13), par, 5)
    f = -g
    dt, a = sc1[0], sc[1]
    c1, cf = 1 - a, a * math.sqrt((v * v).sum() / (f * f).sum()) + dt
    direct = np.linalg.norm(dt * v1)
    three = dt * math.sqrt(c1 * c1 * (v * v).sum() + 2 * c1 * cf * (f * v).sum() + cf * cf * (f * f).sum())
    assert three == pytest.approx(direct, rel=1e-12)
    assert np.abs(x1 - x - dt * v1).max() <= 1e-14   # below maxstep: unclamped (bar: rounding of x1 - x)
    small = fo.params(0.0, maxstep=0.1 * direct)
    x2, v2, _, _, _ = fo.step(x, v, sc, g, np.ones(13), small, 5)
    assert np.linalg.norm(x2 - x) == pytest.approx(0.1 * direct, rel=1e-12)
    assert np.allclose((x2 - x) / np.linalg.norm(x2 - x), v2 / np.linalg.norm(v2), rtol=1e-12, atol=1e-15)


def test_fixed_atoms_and_batch_equals_single():
    """Atoms with force scale 0 never move and are left out of fmax; conformers are independent, so running them in
    any company gives each the same steps (here: two conformers stepped alongside each other and alone)."""
    xs = _lj13(2, seed=4)
    scale = np.ones(13)
    scale[[0, 5]] = 0.0
    par = fo.params(1e-3)
    x, v, sc, conv = [c.copy() for c in xs], [np.zeros((13, 3))] * 2, [fo.init(par)] * 2, [False, False]
    for t in range(200):
        for c in range(2):
            g = fo.lj(x[c])[1]
            x[c], v[c], sc[c], fm, now = fo.step(x[c], v[c], sc[c], g, scale, par, t, conv[c])
            conv[c] = conv[c] or now
            if not conv[c]:
                f = np.sqrt((g ** 2).sum(1))
                assert fm == pytest.approx(f[scale > 0].max(), rel=1e-15)
    for c in range(2):
        assert np.array_equal(x[c][[0, 5]], xs[c][[0, 5]])
        alone, _, _ = fo.run(xs[c], fo.lj, par, 200, scale)
        assert np.array_equal(alone, x[c])


def test_opt_state_layout_matches_header(tmp_path):
    from torchani_b200 import _lib
    prog = tmp_path / "opt.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "ani_b200.h"\n'
                    'int main(){printf("%zu %zu %zu %zu %zu %d %d %d\\n", sizeof(ani_opt_state),'
                    ' offsetof(ani_opt_state, partials), offsetof(ani_opt_state, n_conf),'
                    ' offsetof(ani_opt_state, record_rows), offsetof(ani_opt_state, pad_), ANI_OPT_PARAMS,'
                    ' ANI_OPT_SCALARS, ANI_OPT_RECORD);return 0;}\n')
    exe = tmp_path / "opt"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    out = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    S = _lib.OptState
    assert out == [C.sizeof(S), S.partials.offset, S.n_conf.offset, S.record_rows.offset, S.pad_.offset,
                   _lib.ANI_OPT_PARAMS, _lib.ANI_OPT_SCALARS, _lib.ANI_OPT_RECORD]
    assert len(fo.PARAMS) == _lib.ANI_OPT_PARAMS


def test_opt_argument_validation_without_gpu():
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

    def step(s, grad=h, energies=h, coords=h):
        return L.ani_b200_opt_step(C.byref(s), grad, energies, None, coords, None)

    for bad in ({"x": None}, {"v": None}, {"force_scale": None}, {"params": None}, {"scalars": None},
                {"counter": None}, {"conv_step": None}, {"record": None}, {"partials": None}, {"n_conf": 0},
                {"n_per_conf": 0}, {"record_rows": 0}):
        assert step(state(**bad)) == -1, bad
    assert step(state(), grad=None) == -1
    assert step(state(), energies=None) == -1
    assert step(state(), coords=None) == -1
    assert step(state(n_conf=70000)) != 0   # more conformers than a grid dimension holds
    assert L.ani_b200_opt_step_cells(C.byref(state()), h, h, None, h, None) == -1   # no lattice table
    assert L.ani_b200_opt_init(C.byref(state()), None, 1, 1, h, None) == -1   # a periodic mode without its cell
    assert L.ani_b200_opt_init(C.byref(state()), h, 3, 1, h, None) == -1
    assert L.ani_b200_opt_init(C.byref(state()), None, 0, 1, None, None) == -1
    assert L.ani_b200_opt_init(C.byref(state(x=None)), None, 0, 1, h, None) == -1


class _CpuModel:
    """Enough of a model for the driver's checks that come before any device work."""

    def buffers(self):
        import torch
        yield torch.zeros(1)


@pytest.mark.parametrize("kw,match", [
    (dict(dt=0.0), "dt"), (dict(maxstep=-0.1), "maxstep"), (dict(dtmax=0.0), "dtmax"), (dict(fdec=1.0), "fdec"),
    (dict(fdec=0.0), "fdec"), (dict(finc=0.9), "finc"), (dict(fa=0.0), "fa"), (dict(fa=1.5), "fa"),
    (dict(astart=-0.1), "astart"), (dict(n_min=-1), "n_min"), (dict(dt=math.nan), "finite"),
    (dict(steps_per_replay=0), "steps_per_replay")])
def test_fire_parameter_rejections_without_gpu(kw, match):
    from torchani_b200 import optimize
    with pytest.raises(ValueError, match=match):
        optimize.FIRE(_CpuModel(), np.zeros(3, dtype=np.int64), np.zeros((3, 3)), **kw)


def test_fire_rejects_a_cpu_model():
    from torchani_b200 import optimize
    with pytest.raises(ValueError, match="CUDA"):
        optimize.FIRE(_CpuModel(), np.zeros(3, dtype=np.int64), np.zeros((3, 3)))
