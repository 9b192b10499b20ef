"""The float64 barostat oracle (oracle/npt_oracle.py) on an ideal gas, whose isothermal-isobaric volume distribution is
known; the bar-to-Hartree constant against CODATA 2014; and, without a GPU, the barostat struct's layout, the argument
checks of ani_b200_md_step_npt / ani_b200_md_cell_noise and the rejections of md.LangevinNPT that come before any
device work."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import oracle.md_oracle as mo
import oracle.npt_oracle as no
from helpers import ROOT

HARTREE_J_CODATA2014 = 4.359744650e-18   # the tabulated Hartree energy, J


def test_bar_constant():
    bar = 1e5 / HARTREE_J_CODATA2014 / 1e30
    assert no.BAR == pytest.approx(bar, rel=1e-9)
    assert no.BAR == pytest.approx(2.2937e-8, rel=1e-4)
    from torchani_b200 import grad, md
    assert grad.BAR_TO_HARTREE_A3 == pytest.approx(no.BAR, rel=1e-15)
    assert md.BAR_TO_HARTREE_A3 is grad.BAR_TO_HARTREE_A3


def test_ideal_gas_volume_distribution():
    """64 replicas of 64 free atoms (forces and virial zero) under BAOAB + C-rescale: V is Gamma(N + 1, k_B T / P0), so
    <V> = (N + 1) k_B T / P0 and Var(V) / <V>^2 = 1 / (N + 1).  A Berendsen barostat (no noise term) gets the mean but
    a far smaller variance; a k_B T / V drift term in the eps update would give Gamma(N + 2), whose mean is
    1 / (N + 1) = 1.5 % larger here.  With beta_T = 1 / P0 (the ideal gas's compressibility) V relaxes in ~tau_p = 200 fs, so
    20 ps per replica holds ~100 relaxation times: the standard error of <V> is ~0.2 % and that of the variance ratio
    ~2 %, against bars of 1 % and 15 %.  dt / tau_p = 0.005 keeps the first-order splitting's bias well below both."""
    C_, A, T, dt, tau, gamma = 64, 64, 300.0, 1.0, 200.0, 0.05
    p0 = 65 * mo.KB * T / 27000.0           # <V> = 27 000 A^3
    beta = 1.0 / p0
    rng = np.random.default_rng(3)
    inv = np.full((C_, A), 1.0 / 16.0)
    x = rng.uniform(0.0, 30.0, (C_, A, 3))
    v = np.sqrt(mo.KB * T * mo.ACCEL * inv)[..., None] * rng.standard_normal((C_, A, 3))
    cell = np.tile(np.eye(3) * 30.0, (C_, 1, 1))
    g = np.zeros_like(x)
    zero = np.zeros((C_, 3, 3))
    vols = []
    for t in range(22000):
        ek = mo.kinetic(v, inv)
        x, v = mo.start(x, v, g, inv, dt, mo.LANGEVIN, T, gamma, rng.standard_normal(x.shape))
        x, v, cell, vol, _ = no.cell_rescale(x, v, cell, ek, zero, T, p0, tau, beta, dt, rng.standard_normal(C_))
        if t >= 2000:
            vols.append(vol)
    V = np.array(vols)                      # (steps, replicas)
    target = (A + 1) * mo.KB * T / p0
    assert abs(V.mean() / target - 1) < 0.01, V.mean() / target
    ratio = V.var() / V.mean() ** 2
    assert abs(ratio * (A + 1) - 1) < 0.15, ratio * (A + 1)
    # the replicas' own means scatter by the standard error the docstring assumes
    assert V.mean(0).std(ddof=1) / math.sqrt(C_) < 0.004 * target


def test_cell_rescale_scales_isotropically():
    rng = np.random.default_rng(1)
    cell = np.array([[[10.0, 0, 0], [2.0, 9.0, 0], [1.0, 1.0, 8.0]]])
    x, v = rng.standard_normal((1, 5, 3)), rng.standard_normal((1, 5, 3))
    w = rng.standard_normal((1, 3, 3))
    x1, v1, c1, vol, p = no.cell_rescale(x, v, cell, np.array([0.01]), w, 300.0, 1e-6, 1e3, 500.0, 0.5,
                                         np.array([0.3]))
    mu = np.cbrt(np.linalg.det(c1) / np.linalg.det(cell))
    assert np.allclose(c1, mu[:, None, None] * cell, rtol=1e-14)
    assert np.allclose(x1, mu * x, rtol=1e-14) and np.allclose(v1, v / mu, rtol=1e-14)
    assert vol[0] == pytest.approx(abs(np.linalg.det(cell[0])), rel=1e-14)
    assert p[0] == pytest.approx((0.02 - np.trace(w[0])) / (3 * vol[0]), rel=1e-14)


def test_md_barostat_layout_matches_header(tmp_path):
    from torchani_b200 import _lib
    prog = tmp_path / "baro.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "ani_b200.h"\n'
                    'int main(){printf("%zu %zu %zu %d %d\\n", sizeof(ani_md_barostat),'
                    ' offsetof(ani_md_barostat, frame_cells), offsetof(ani_md_barostat, virial_slots),'
                    ' ANI_MD_BARO_PARAMS, ANI_MD_BARO);return 0;}\n')
    exe = tmp_path / "baro"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    out = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    B = _lib.MDBarostat
    assert out == [C.sizeof(B), B.frame_cells.offset, B.virial_slots.offset, _lib.ANI_MD_BARO_PARAMS,
                   _lib.ANI_MD_BARO]


def test_md_step_npt_argument_validation_without_gpu():
    """Bad arguments are rejected before any CUDA call (the pointers are host dummies)."""
    from torchani_b200 import _lib
    L = _lib.lib()
    buf = (C.c_char * 4096)()
    h = C.cast(buf, C.c_void_p).value

    def state(**kw):
        s = _lib.MDState()
        for k in ("x", "v", "inv_mass", "params", "counter", "stop_step", "thermo", "partials"):
            setattr(s, k, h)
        s.n_conf, s.n_per_conf, s.integrator, s.thermo_rows, s.accel, s.kb = 1, 4, 1, 4, mo.ACCEL, mo.KB
        for k, v in kw.items():
            setattr(s, k, v)
        return s

    def baro(**kw):
        b = _lib.MDBarostat()
        for k in ("master", "params", "cell_out", "virial", "record"):
            setattr(b, k, h)
        b.cell_stride, b.virial_slots = 9, _lib.ANI_VIRIAL_SLOTS
        for k, v in kw.items():
            setattr(b, k, v)
        return b

    def step(s, b, grad=h):
        return L.ani_b200_md_step_npt(C.byref(s), C.byref(b) if b is not None else None, grad, h, h, None)

    assert step(state(), None) == -1
    for bad in ({"integrator": 0}, {"x": None}, {"params": None}, {"n_conf": 0}, {"thermo_rows": 0}, {"kb": 0.0},
                {"record_every": 5, "frames": h, "frame_slots": 1}):
        assert step(state(**bad), baro()) == -1, bad
    for bad in ({"master": None}, {"params": None}, {"cell_out": None}, {"virial": None}, {"record": None},
                {"cell_stride": 8}, {"virial_slots": 0}):
        assert step(state(), baro(**bad)) == -1, bad
    assert step(state(), baro(), grad=None) == -1
    assert L.ani_b200_md_cell_noise(0, 0, 0, h, None) == -1
    assert L.ani_b200_md_cell_noise(0, 0, 4, None, None) == -1


def test_langevin_npt_rejections_without_gpu():
    """The barostat's own inputs are checked before the model is touched."""
    from torchani_b200 import md
    sp, co, m, cell = np.zeros(3, dtype=np.int64), np.zeros((3, 3)), np.ones(3), np.eye(3) * 20.0
    with pytest.raises(ValueError, match="periodic"):
        md.LangevinNPT(None, sp, co, m, None)
    with pytest.raises(ValueError, match="qbc_stop"):
        md.LangevinNPT(None, sp, co, m, cell, qbc_stop=(1.0, None))
    for bad in (math.nan, math.inf, -math.inf):
        with pytest.raises(ValueError, match="pressure"):
            md.LangevinNPT(None, sp, co, m, cell, pressure=bad)
    for bad in (0.0, -5.0, math.nan):
        with pytest.raises(ValueError, match="tau_p"):
            md.LangevinNPT(None, sp, co, m, cell, tau_p=bad)
    for bad in (0.0, -1e-5, math.inf):
        with pytest.raises(ValueError, match="compressibility"):
            md.LangevinNPT(None, sp, co, m, cell, compressibility=bad)
