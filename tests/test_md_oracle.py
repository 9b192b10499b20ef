"""The float64 MD oracle (oracle/md_oracle.py) on problems with known answers, its unit constants against CODATA 2014 and
ASE's published values, the device-MD driver's constants and host helpers, and the md entry points of the C-ABI
without a GPU (struct layout, argument checks that return before any CUDA call)."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import oracle.md_oracle as mo
from helpers import ROOT

# ASE 3.22 with its default CODATA 2014 set: units.fs, units.kB (eV / K), units.Hartree (eV)
ASE_FS = 0.09822694788464063
ASE_KB = 8.617330337217213e-05
ASE_HARTREE = 27.211386024367243
K_B_CODATA2014 = 1.38064852e-23


def test_unit_constants():
    assert mo.K_B == K_B_CODATA2014
    assert mo.ASE_FS == pytest.approx(ASE_FS, rel=1e-15)
    assert mo.ASE_KB == pytest.approx(ASE_KB, rel=1e-15)
    assert mo.HARTREE_EV == pytest.approx(ASE_HARTREE, rel=1e-14)
    # 1 eV / (amu A^2) is (1 / ASE time unit)^2 = units.fs^2 per fs^2; k_B in Hartree / K is units.kB / Hartree
    assert mo.ACCEL == pytest.approx(ASE_HARTREE * ASE_FS ** 2, rel=1e-14)
    assert mo.ACCEL == pytest.approx(0.26255, rel=1e-4)
    assert mo.KB == pytest.approx(ASE_KB / ASE_HARTREE, rel=1e-14)
    from torchani_b200 import md
    assert md.ACCEL == pytest.approx(mo.ACCEL, rel=1e-15)
    assert md.KB == pytest.approx(mo.KB, rel=1e-15)
    # the friction conversion of the documentation: ASE's friction=0.2 (per ASE time unit) is 0.0196 / fs
    assert md.ASE_TIME_FS == pytest.approx(1.0 / ASE_FS, rel=1e-15)
    assert 0.2 / md.ASE_TIME_FS == pytest.approx(0.0196, abs=5e-5)


K_SPRING = 0.5          # Hartree / A^2
MASS = 1.0              # amu


def _oscillators(n: int):
    inv = np.full(n, 1.0 / MASS)
    return inv, (lambda x: K_SPRING * x)


def test_velocity_verlet_energy_error_is_second_order():
    """Velocity Verlet on a harmonic oscillator conserves a shadow energy E + O(dt^2): the largest deviation of E over
    many periods scales with dt^2.  The O(dt^4) term moves the ratio by about (omega dt)^2 / 4 < 1 % here."""
    inv, force = _oscillators(1)
    omega = math.sqrt(K_SPRING * mo.ACCEL / MASS)
    assert omega * 0.5 < 0.2
    errs = []
    for dt in (0.5, 0.25):
        steps = int(round(400.0 / dt))   # ~20 periods
        xs, vs = mo.run(np.array([[0.1, 0.0, 0.0]]), np.zeros((1, 3)), force, inv, dt, steps)
        e = 0.5 * K_SPRING * (xs ** 2).sum((-1, -2)) + mo.kinetic(vs, inv)
        errs.append(np.abs(e - e[0]).max())
    assert errs[0] / errs[1] == pytest.approx(4.0, rel=0.10), errs


@pytest.mark.parametrize("dt", [1.0, 0.5])
def test_baoab_samples_the_harmonic_boltzmann_distribution(dt):
    """BAOAB's configurational sampling is exact for a harmonic potential at any stable dt: <x^2> = k_B T / k per
    component.  The error bar comes from the data: 1500 independent oscillators x 3 components, each time-averaged; the
    standard error of the mean of those averages, and the check at 5 of them."""
    T, gamma = 300.0, 0.1
    n = 1500
    inv, force = _oscillators(n)
    rng = np.random.default_rng(7)
    x0 = np.zeros((n, 3))
    steps = int(round(1500.0 / dt))
    burn = int(round(100.0 / dt))
    xs, _ = mo.run(x0, np.zeros((n, 3)), force, inv, dt, steps, mo.LANGEVIN, T, gamma, rng)
    per = (xs[burn:] ** 2).mean(0).reshape(-1)          # time average per oscillator component
    mean, sem = per.mean(), per.std(ddof=1) / math.sqrt(per.size)
    target = mo.KB * T / K_SPRING
    assert abs(mean - target) < 5 * sem, (mean, target, sem)
    assert sem < 0.02 * target   # the check is sharp enough to see a 10 % error


def test_wrap_and_temperature_helpers():
    cell = np.array([[10.0, 0, 0], [2.0, 9.0, 0], [0, 1.0, 8.0]])
    x = np.array([[25.3, -4.0, 17.1]])
    w = mo.wrap(x, cell)
    frac = w @ np.linalg.inv(cell)
    assert ((frac >= 0) & (frac < 1)).all()
    n = np.linalg.solve(cell.T, (x - w).T).T
    assert np.allclose(n, np.round(n), atol=1e-12)
    assert mo.temperature(1.5 * mo.KB * 300.0 * 4, 4) == pytest.approx(300.0)


def test_maxwell_boltzmann():
    from torchani_b200 import md
    m = np.tile(np.array([16.0, 1.0, 1.0] * 200), (2, 1))
    m[1, -3:] = 0.0                                  # padding
    v = md.maxwell_boltzmann(m, [300.0, 600.0], seed=3)
    assert v.shape == (2, 600, 3)
    assert np.abs((m[..., None] * v).sum(1)).max() < 1e-12
    assert (v[1, -3:] == 0).all()
    inv = np.where(m > 0, 1.0 / np.where(m > 0, m, 1.0), 0.0)
    T = mo.temperature(mo.kinetic(v, inv), (m > 0).sum(1))
    # 3 N - 3 degrees of freedom after the momentum removal: the sample's T has a relative spread of sqrt(2 / 3N)
    assert np.all(np.abs(T / np.array([300.0, 600.0]) - 1) < 5 * math.sqrt(2 / 1800)), T
    with pytest.raises(ValueError):
        md.maxwell_boltzmann(m, 0.0)


@pytest.mark.parametrize("counter, key, out", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_philox_known_answers(counter, key, out):
    """The Philox4x32-10 restatement against the Random123 known-answer vectors (counter -> output, key words last),
    one at a time and broadcast over a batch."""
    assert tuple(int(w) for w in mo.philox4x32_10(counter, key)) == out
    batch = mo.philox4x32_10(np.tile(np.array(counter, dtype=np.uint32), (3, 1)), key)
    assert batch.shape == (3, 4) and (batch == np.array(out, dtype=np.uint32)).all()


def test_normal_counter_layout():
    """``normal`` draws from the block of counter (step low, step high, atom, component) and key (seed low, seed
    high): each word changes the draw, the step's high word included, and the words (0, 1) and (2, 3) of the block
    give the two uniforms of Box-Muller's cosine branch."""
    seed, step = 0x0123456789ABCDEF, (5 << 32) + 7
    z = mo.normal(seed, step, 11, 2)
    w = mo.philox4x32_10((7, 5, 11, 2), (0x89ABCDEF, 0x01234567))
    u1, u2 = mo.unit_open(w[0], w[1]), mo.unit_open(w[2], w[3])
    assert 0.0 < u1 < 1.0 and 0.0 < u2 < 1.0
    assert z == pytest.approx(math.sqrt(-2.0 * math.log(u1)) * math.cos(2.0 * math.pi * u2), rel=1e-15, abs=1e-15)
    others = [mo.normal(seed ^ 1, step, 11, 2), mo.normal(seed ^ (1 << 32), step, 11, 2), mo.normal(seed, step + 1, 11, 2),
              mo.normal(seed, step + (1 << 32), 11, 2), mo.normal(seed, step, 12, 2), mo.normal(seed, step, 11, 3)]
    assert len({float(z)} | {float(o) for o in others}) == 7
    assert mo.unit_open(0, 0) == 2.0 ** -54 and mo.unit_open(0, 0x800) == 1.5 * 2.0 ** -53
    # moments of a large batch: mean 0 and variance 1 to a few standard errors
    zs = mo.normal(seed, np.arange(4)[:, None, None], np.arange(5000)[None, :, None], np.arange(4)[None, None, :])
    assert abs(zs.mean()) < 5.0 / math.sqrt(zs.size) and abs(zs.var() - 1.0) < 5.0 * math.sqrt(2.0 / zs.size)


def test_md_state_layout_matches_header(tmp_path):
    from torchani_b200 import _lib
    prog = tmp_path / "md.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "ani_b200.h"\n'
                    'int main(){printf("%zu %zu %zu %zu %d %d %d\\n", sizeof(ani_md_state), offsetof(ani_md_state, seed),'
                    ' offsetof(ani_md_state, n_conf), offsetof(ani_md_state, pad_), ANI_MD_BLOCK, ANI_MD_PARAMS,'
                    ' ANI_MD_THERMO);return 0;}\n')
    exe = tmp_path / "md"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    out = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    S = _lib.MDState
    assert out == [C.sizeof(S), S.seed.offset, S.n_conf.offset, S.pad_.offset, _lib.ANI_MD_BLOCK, _lib.ANI_MD_PARAMS,
                   _lib.ANI_MD_THERMO]


def test_md_argument_validation_without_gpu():
    """Bad arguments are rejected before any CUDA call (the pointers are host dummies)."""
    from torchani_b200 import _lib
    L = _lib.lib()
    buf = (C.c_char * 4096)()
    h = C.cast(buf, C.c_void_p).value

    def state(**kw):
        s = _lib.MDState()
        for k in ("x", "v", "inv_mass", "params", "counter", "stop_step", "thermo", "partials"):
            setattr(s, k, h)
        s.n_conf, s.n_per_conf, s.integrator, s.thermo_rows, s.accel, s.kb = 1, 4, 0, 4, mo.ACCEL, mo.KB
        for k, v in kw.items():
            setattr(s, k, v)
        return s

    def step(s, qbc=None, stdev=None, grad=h):
        return L.ani_b200_md_step(C.byref(s), grad, h, qbc, stdev, None, h, None)

    for bad in ({"x": None}, {"v": None}, {"inv_mass": None}, {"params": None}, {"counter": None},
                {"stop_step": None}, {"thermo": None}, {"partials": None}, {"n_conf": 0}, {"n_per_conf": 0},
                {"integrator": 2}, {"thermo_rows": 0}, {"record_every": -1}, {"record_every": 5},
                {"record_every": 5, "frames": h}, {"accel": 0.0}, {"kb": -1.0}):
        assert step(state(**bad)) == -1, bad
    assert step(state(), qbc=h) == -1          # QBC without the force statistics
    assert step(state(), stdev=h) == -1
    assert step(state(), grad=None) == -1
    assert L.ani_b200_md_step_cells(C.byref(state()), h, h, None, None, None, h, None) == -1   # no lattice table
    assert L.ani_b200_md_init(C.byref(state()), None, 1, 0, h, None) == -1   # a periodic mode without its cell
    assert L.ani_b200_md_init(C.byref(state()), h, 3, 0, h, None) == -1
    assert L.ani_b200_md_init(C.byref(state(x=None)), None, 0, 0, h, None) == -1
    assert L.ani_b200_md_noise(0, 0, 0, h, None) == -1
    assert L.ani_b200_md_noise(0, 0, 4, None, None) == -1
