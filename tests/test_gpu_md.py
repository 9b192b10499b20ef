"""The device MD loop (csrc/md.cu, torchani_b200/md.py) on the H100: one integrator step against the float64 oracle,
the device loop against a host loop of Engine.step + oracle steps, determinism across replay shapes, energy
conservation, the Langevin temperature, periodic boxes, batches, the QBC stop, the operand-range fallback, and the
rejected inputs.

The bars, and where they come from:
* one step: the integration is float64 and the forces are inputs, so x and v agree with the oracle to float64 rounding
  of a few operations (1e-12 relative);
* longer runs: the integrator is bitwise reproducible (test_integrator_is_bitwise_reproducible), but the force step
  is not: the AEV backward adds float32 contributions with atomics, whose order may differ between two runs.  Such a
  difference (~1e-7 relative of a force) reaches the float32 coordinates after a few steps and then grows with the
  divergence of nearby trajectories: on water30_pbc two device runs of the same input were measured 3e-9 A apart
  after 60 steps and 1e-6 A after 200 steps (a doubling about every 8 fs).  TRAJ_BAR is sized from that.
"""
import math

import numpy as np
import pytest
import torch

import oracle.md_oracle as mo
from helpers import F_ATOL, golden_inputs, load_golden

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
TRAJ_BAR = {60: 1e-7, 100: 1e-7, 200: 1e-5}   # A, by number of steps (see above)
MASSES_2X = np.array([1.008, 12.011, 14.007, 15.999, 32.06, 18.998, 35.45])   # H C N O S F Cl, amu


def _model():
    from torchani_b200 import models
    base = models.ANI2x(seed=0)
    return models.ANI(base.symbols, base.aev_computer, base.neural_networks, base.energy_shifter, False).to(DEV)


_MODEL = {}


def model():
    if "m" not in _MODEL:
        _MODEL["m"] = _model()
    return _MODEL["m"]


def system(name):
    sp, co, cell, pbc = golden_inputs(load_golden(name))
    sp = sp.numpy()
    return sp, co.numpy(), None if cell is None else cell.numpy(), bool(pbc is not None and bool(pbc.all())), \
        MASSES_2X[np.maximum(sp, 0)] * (sp >= 0)


def make(kind="verlet", name="water30_pbc_ani2x", T=300.0, seed=0, **kw):
    from torchani_b200 import md
    sp, co, cell, pbc, m = system(name)
    kw.setdefault("velocities", md.maxwell_boltzmann(m, T, seed=11))
    if kind == "verlet":
        return md.VelocityVerlet(model(), sp, co, m, cell=cell, pbc=pbc, **kw), m
    return md.Langevin(model(), sp, co, m, temperature=T, seed=seed, cell=cell, pbc=pbc, **kw), m


def inv_mass(m):
    return np.where(m > 0, 1.0 / np.where(m > 0, m, 1.0), 0.0)


def np64(t):
    return t.detach().double().cpu().numpy()


# ------------------------------------------------------------------------------------------------------------------
# 1. one step against the oracle
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["verlet", "langevin"])
@pytest.mark.parametrize("name", ["water30_pbc_ani2x", "small264_nopbc_ani2x"])
def test_one_step_vs_oracle(kind, name):
    from torchani_b200 import md
    dyn, m = make(kind, name, steps_per_replay=1, record_every=0, friction=0.05) if kind == "langevin" else \
        make(kind, name, steps_per_replay=1, record_every=0)
    im = inv_mass(m).reshape(dyn.n_conf, -1)
    integ = mo.LANGEVIN if kind == "langevin" else mo.VERLET
    x, v = np64(dyn.x), np64(dyn.v)
    for t in range(2):
        g = np64(dyn.ws.grad).reshape(x.shape)
        v = mo.finish(v, g, im, 0.5, t)
        noise = np64(md.noise(0, t, x.size // 3, DEV)).reshape(x.shape) if kind == "langevin" else None
        x, v_next = mo.start(x, v, g, im, 0.5, integ, 300.0, 0.05, noise)
        ek = mo.kinetic(v, im)
        e_pot = float(dyn.ws.energies[0])
        dyn.run(1)
        th = dyn.thermo
        assert th.step[-1] == t
        assert abs(th.kinetic[-1, 0] - ek[0]) <= 1e-12 * abs(ek[0])
        assert th.temperature[-1, 0] == pytest.approx(mo.temperature(ek[0], int((m > 0).sum())), rel=1e-12)
        assert th.potential[-1, 0] == e_pot
        v = v_next
        for got, ref, what in ((np64(dyn.x), x, "x"), (np64(dyn.v), v, "v")):
            err = np.abs(got - ref).max()
            assert err <= 1e-12 * np.abs(ref).max(), f"{what} step {t}: {err:.3e}"
    # the f32 coordinates of the next force step are x, wrapped into the cell
    c = np64(dyn.ws.coords).reshape(x.shape)
    _, _, cell, pbc, _ = system(name)
    ref = mo.wrap(x, cell) if pbc else x
    assert np.abs(c - ref.astype(np.float32)).max() <= 4e-6


# ------------------------------------------------------------------------------------------------------------------
# 2. the device loop against a host loop
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,name", [("verlet", "water30_pbc_ani2x"), ("langevin", "small264_nopbc_ani2x")])
def test_device_loop_vs_host_loop(kind, name):
    """200 steps on the device against Engine.step + oracle steps on the same float32 coordinates.  Bar TRAJ_BAR[200]
    = 1e-5 A rather than 1e-6: two device runs of the same input already drift 1e-6 A apart in 200 steps (the force
    step's atomics, module docstring), and so does a host loop."""
    from torchani_b200 import md
    kw = dict(friction=0.05) if kind == "langevin" else {}
    dyn, m = make(kind, name, steps_per_replay=20, record_every=0, **kw)
    sp, co, cell, pbc, _ = system(name)
    im = inv_mass(m).reshape(1, -1)
    integ = mo.LANGEVIN if kind == "langevin" else mo.VERLET
    x, v = np64(dyn.x), np64(dyn.v)
    eng = model().engine(torch.device(DEV))
    species = torch.as_tensor(sp).to(DEV)
    cell_t = None if cell is None else torch.tensor(cell, dtype=torch.float32, device=DEV)

    def force(x):
        xc = mo.wrap(x, cell) if pbc else x
        r = eng.step(species, torch.tensor(xc, dtype=torch.float32, device=DEV), cell_t, pbc)
        return np64(r.grad)

    g = force(x)
    for t in range(200):
        v = mo.finish(v, g, im, 0.5, t)
        noise = np64(md.noise(0, t, x.size // 3, DEV)).reshape(x.shape) if kind == "langevin" else None
        x, v = mo.start(x, v, g, im, 0.5, integ, 300.0, 0.05, noise)
        g = force(x)
    dyn.run(200)
    err = np.abs(np64(dyn.x) - x).max()
    assert err <= TRAJ_BAR[200], err


# ------------------------------------------------------------------------------------------------------------------
# 3. determinism
# ------------------------------------------------------------------------------------------------------------------
def _trajectory(K, steps=60, seed=0):
    dyn, _ = make("langevin", steps_per_replay=K, record_every=5, seed=seed, friction=0.05)
    dyn.run(steps)
    return np64(dyn.x), np64(dyn.velocities), dyn.thermo, dyn.frames


def test_integrator_is_bitwise_reproducible():
    """The same state and forces give the same bits: the integrator launches of one step, twice from a saved state,
    for a Langevin batch with frames and the QBC stop check."""
    from torchani_b200 import md
    sp, co, cell, pbc, m = system("water30_pbc_ani2x")
    sp3, co3, m3 = np.repeat(sp, 3, 0), np.repeat(co, 3, 0), np.repeat(m, 3, 0)
    dyn = md.Langevin(model(), sp3, co3, m3, temperature=[250.0, 300.0, 350.0], friction=0.05, cell=cell, pbc=True,
                      velocities=md.maxwell_boltzmann(m3, 300.0, seed=4), steps_per_replay=4, record_every=2,
                      record_velocities=True, qbc_stop=(math.inf, math.inf))
    dyn.run(6)
    saved = dyn._buf.clone(), dyn.ws.coords.clone()
    outs = []
    for _ in range(2):
        dyn._buf.copy_(saved[0])
        dyn._integrate()
        dyn._integrate()
        torch.cuda.synchronize()
        outs.append((dyn._buf.clone().view(torch.int64), dyn.ws.coords.clone().view(torch.int32)))   # (bit patterns)
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert not torch.equal(outs[0][0], saved[0].view(torch.int64))


def test_replay_shapes_agree():
    """60 steps as eager launches (the remainder path: K = 64 > 60), as 6 replays of 10 and 3 of 20: the same
    sequence of launches, so the same trajectory up to the force step's atomics (TRAJ_BAR[60])."""
    runs = [_trajectory(64), _trajectory(10), _trajectory(20)]
    x0, v0, th0, fr0 = runs[0]
    assert list(th0.step) == list(range(60)) and list(fr0.step) == list(range(0, 60, 5))
    for x, v, th, fr in runs[1:]:
        assert np.abs(x - x0).max() <= TRAJ_BAR[60] and np.abs(v - v0).max() <= TRAJ_BAR[60]
        assert np.array_equal(th.step, th0.step)
        assert np.abs(th.kinetic - th0.kinetic).max() <= 1e-6 * np.abs(th0.kinetic).max()
        assert np.abs(th.potential - th0.potential).max() <= 1e-5
        assert np.abs(fr.positions - fr0.positions).max() <= TRAJ_BAR[60]


def test_seed_reproduces_and_changes_the_trajectory():
    """Another seed moves the atoms by the thermostat's noise, sqrt((1 - c^2) k_B T / m) dt / 2 ~ 1e-3 A per step."""
    a, b, c = _trajectory(20, 20, 1), _trajectory(20, 20, 1), _trajectory(20, 20, 2)
    assert np.abs(a[0] - b[0]).max() <= TRAJ_BAR[60]
    assert np.abs(a[0] - c[0]).max() > 1e-3


def test_noise_moments():
    """10^6 normals: mean 0 (standard error 1e-3) and variance 1 (standard error sqrt(2) 1e-3) within 5 sigma; steps,
    atoms and components give different numbers."""
    from torchani_b200 import md
    z = np64(md.noise(123, 7, 333_334, DEV)).reshape(-1)[:1_000_000]
    assert abs(z.mean()) < 5e-3
    assert abs(z.var() - 1.0) < 5 * math.sqrt(2) * 1e-3
    z2 = np64(md.noise(123, 8, 10, DEV))
    assert not np.array_equal(z2, np64(md.noise(123, 7, 10, DEV)))
    assert np.array_equal(np64(md.noise(123, 7, 10, DEV)).reshape(-1), z[:30])


# ------------------------------------------------------------------------------------------------------------------
# 4. NVE
# ------------------------------------------------------------------------------------------------------------------
def test_nve_energy_error_scales_with_dt_squared():
    """Velocity Verlet over 0.2 ps: the largest drift of E_pot + E_kin falls by (0.5 / 0.25)^2 = 4 when dt halves;
    2.5 .. 5.5 leaves room for the O(dt^4) term and the float32 noise of E_pot (~1e-6 Ha here)."""
    errs = []
    for dt in (0.5, 0.25):
        dyn, _ = make("verlet", dt=dt, steps_per_replay=50, record_every=0)
        dyn.run(int(round(200 / dt)))
        th = dyn.thermo
        e = th.potential[:, 0] + th.kinetic[:, 0]
        errs.append(np.abs(e - e[0]).max())
    assert 2.5 <= errs[0] / errs[1] <= 5.5, errs


def test_nve_momentum_of_an_open_molecule():
    """Zero centre-of-mass momentum at the start; the forces sum to zero up to float32 rounding of n terms of size
    |F|, so the momentum may change by at most steps * dt * ACCEL * n * 2^-23 * max|F| (amu A / fs)."""
    dyn, m = make("verlet", "small264_nopbc_ani2x", steps_per_replay=25, record_every=0, zero_momentum=True)
    p0 = (m.reshape(-1, 1) * np64(dyn.v).reshape(-1, 3)).sum(0)
    assert np.abs(p0).max() < 1e-12
    fmax = float(dyn.ws.grad.abs().max())
    dyn.run(100)
    p = (m.reshape(-1, 1) * np64(dyn.velocities).reshape(-1, 3)).sum(0)
    bar = 100 * 0.5 * mo.ACCEL * m.size * 2.0 ** -23 * 4 * fmax
    assert np.abs(p).max() <= bar, (p, bar)


# ------------------------------------------------------------------------------------------------------------------
# 5. Langevin temperature
# ------------------------------------------------------------------------------------------------------------------
def _mean_t_and_error(T):
    """Mean and standard error (from 100-fs block averages, longer than the ~10 fs correlation time at gamma 0.05)."""
    blocks = T[: len(T) // 200 * 200].reshape(-1, 200).mean(1)
    return T.mean(), blocks.std(ddof=1) / math.sqrt(len(blocks))


def test_langevin_temperature():
    """300 K, gamma 0.05 / fs, 12 ps at 0.5 fs: the mean temperature of the last 10 ps within 2 % of the target.  With
    90 degrees of freedom T fluctuates by sqrt(2 / 90) = 15 %; over ~1000 correlation times its mean has a standard
    error of ~0.5 % (measured: 0.56 % from 100-fs blocks), so 2 % is about 3.6 standard errors; the test also checks
    that the measured error stays below 0.8 %."""
    dyn, _ = make("langevin", T=300.0, friction=0.05, steps_per_replay=50, record_every=0)
    dyn.run(24000)
    T = dyn.thermo.temperature[4000:, 0]
    mean, se = _mean_t_and_error(T)
    assert abs(mean / 300.0 - 1) < 0.02, (mean, se)
    assert se < 0.008 * 300.0, se


def test_langevin_replicas_at_three_temperatures():
    from torchani_b200 import md
    sp, co, cell, pbc, m = system("water30_pbc_ani2x")
    Ts = np.array([250.0, 300.0, 350.0])
    sp3, co3, m3 = np.repeat(sp, 3, 0), np.repeat(co, 3, 0), np.repeat(m, 3, 0)
    dyn = md.Langevin(model(), sp3, co3, m3, temperature=Ts, friction=0.05, cell=cell, pbc=True,
                      velocities=md.maxwell_boltzmann(m3, Ts, seed=5), steps_per_replay=50, record_every=0)
    dyn.run(24000)
    T = dyn.thermo.temperature[4000:]
    for c in range(3):
        mean, se = _mean_t_and_error(T[:, c])
        assert abs(mean / Ts[c] - 1) < 0.02, (c, mean, se)
        assert se < 0.008 * Ts[c], (c, se)


# ------------------------------------------------------------------------------------------------------------------
# 6. periodic boxes
# ------------------------------------------------------------------------------------------------------------------
def test_periodic_wrapping_and_lattice_shift():
    sp, co, cell, pbc, m = system("water30_pbc_ani2x")
    dyn, _ = make("langevin", steps_per_replay=20, record_every=1, friction=0.05, T=600.0)
    dyn.run(400)
    frac = np64(dyn.ws.coords).reshape(-1, 3) @ np.linalg.inv(cell)
    assert frac.min() >= -1e-6 and frac.max() <= 1 + 1e-6
    xs = dyn.frames.positions[:, 0]
    assert np.abs(np.diff(xs, axis=0)).max() < 0.3, "the master trajectory jumps"
    # the same run on positions shifted by a lattice vector: the same forces and thermo
    from torchani_b200 import md
    v0 = md.maxwell_boltzmann(m, 600.0, seed=11)
    a = md.Langevin(model(), sp, co, m, temperature=600.0, friction=0.05, cell=cell, pbc=True, velocities=v0,
                    steps_per_replay=20, record_every=0)
    b = md.Langevin(model(), sp, co + cell[0] - cell[2], m, temperature=600.0, friction=0.05, cell=cell, pbc=True,
                    velocities=v0, steps_per_replay=20, record_every=0)
    ga = np64(a.ws.grad)
    gb = np64(b.ws.grad)
    assert np.abs(ga - gb).max() <= 1e-5
    a.run(40)
    b.run(40)
    assert np.abs(a.thermo.potential - b.thermo.potential).max() <= 1e-5
    assert np.abs(a.thermo.kinetic - b.thermo.kinetic).max() <= 1e-5 * np.abs(a.thermo.kinetic).max()
    assert np.abs(np64(b.x) - (cell[0] - cell[2]) - np64(a.x)).max() <= 1e-5


def test_per_conformer_cells():
    from torchani_b200 import md
    sp, co, cell, pbc, m = system("water30_pbc_ani2x")
    cells = np.stack([cell, cell * 1.02])
    sp2, co2, m2 = np.repeat(sp, 2, 0), np.repeat(co, 2, 0), np.repeat(m, 2, 0)
    dyn = md.Langevin(model(), sp2, co2, m2, temperature=400.0, friction=0.05, cell=cells, pbc=True,
                      velocities=md.maxwell_boltzmann(m2, 400.0, seed=3), steps_per_replay=20, record_every=0)
    assert dyn.per_conf
    dyn.run(200)
    c = np64(dyn.ws.coords).reshape(2, -1, 3)
    for k in range(2):
        frac = c[k] @ np.linalg.inv(cells[k])
        assert frac.min() >= -1e-6 and frac.max() <= 1 + 1e-6
    assert np.isfinite(dyn.thermo.potential).all()


# ------------------------------------------------------------------------------------------------------------------
# 7. batch against single
# ------------------------------------------------------------------------------------------------------------------
def test_batch_vs_single():
    """Conformer c of an open padded batch against its own single-system run over 20 steps of 0.5 fs.  The engine
    computes the batch and the single system to within F_ATOL of each other (its batch-vs-single bar); a force
    difference dF held over t = 10 fs moves an atom of mass m by at most t^2 / 2 * ACCEL * dF / m."""
    from torchani_b200 import md, synthetic
    sp, co = synthetic.conformer_batch(4, seed=5)
    sp, co = sp.numpy(), co.double().numpy()
    m = MASSES_2X[np.maximum(sp, 0)] * (sp >= 0)
    v = md.maxwell_boltzmann(m, 300.0, seed=9)
    batch = md.VelocityVerlet(model(), sp, co, m, velocities=v, steps_per_replay=10, record_every=0)
    batch.run(20)
    bar = 0.5 * 10.0 ** 2 * mo.ACCEL * F_ATOL / MASSES_2X[0]
    for c in range(4):
        n = int((sp[c] >= 0).sum())
        one = md.VelocityVerlet(model(), sp[c, :n], co[c, :n], m[c, :n], velocities=v[c, :n], steps_per_replay=10,
                                record_every=0)
        one.run(20)
        assert np.abs(np64(batch.x)[c, :n] - np64(one.x)[0]).max() <= bar
        assert np.abs(batch.thermo.potential[:, c] - one.thermo.potential[:, 0]).max() <= 1e-4


# ------------------------------------------------------------------------------------------------------------------
# 8. stop on ensemble disagreement
# ------------------------------------------------------------------------------------------------------------------
def test_qbc_stop():
    """Run 100 steps with the query-by-committee step and no threshold, reading the energy QBC of every step; pick a
    step s where it sets a new running maximum and a threshold between the two; the rerun stops at s."""
    inf = math.inf
    first, _ = make("langevin", friction=0.05, steps_per_replay=1, record_every=1, record_velocities=True,
                    qbc_stop=(inf, inf))
    q = [float(first.ws.qbc[0])]
    for _ in range(100):
        first.run(1)
        q.append(float(first.ws.qbc[0]))
    q = np.array(q[:100])
    records = [s for s in range(10, 100) if q[s] > q[:s].max()]
    assert records, "no new running maximum of the energy QBC in 100 steps"
    s = records[0]
    thr = 0.5 * (q[:s].max() + q[s])
    again, _ = make("langevin", friction=0.05, steps_per_replay=10, record_every=1, record_velocities=True,
                    qbc_stop=(thr, None))
    again.run(100)
    assert int(again.stop_step[0]) == s and bool(again.stopped[0])
    tx, tv = again.trigger_frame
    fr = first.frames
    k = list(fr.step).index(s)
    assert np.abs(np64(tx) - fr.positions[k]).max() <= TRAJ_BAR[100]
    assert np.abs(np64(tv) - fr.velocities[k]).max() <= TRAJ_BAR[100]
    x_stop, v_stop = np64(again.x), np64(again.velocities)
    assert np.array_equal(x_stop, np64(tx)) and np.array_equal(v_stop, np64(tv))
    again.run(10)   # frozen: nothing moves (the run returns at once: every conformer has stopped)
    assert np.array_equal(np64(again.x), x_stop) and np.array_equal(np64(again.v), np64(tv))


# ------------------------------------------------------------------------------------------------------------------
# 9. operand-range fallback
# ------------------------------------------------------------------------------------------------------------------
def test_operand_range_fallback_matches_a_bf16x3_loop():
    """A hydrogen with 48 neighbours 0.8 A away: its angular AEV exceeds the 2 x fp16 operand range.  The loop built on
    that build switches to 3 x bfloat16 at its first force step and restores its state; it then runs the launches a
    loop built on 3 x bfloat16 from the start runs (equal up to the force step's atomics: TRAJ_BAR[60])."""
    from torchani_b200 import _lib, md
    from test_gpu_operand_range import cap_system
    if not _lib.available("bf16x3"):
        pytest.skip("the 3 x bfloat16 build is missing")
    s = cap_system(48)
    sp, co = s.species.numpy(), s.coords.double().numpy()
    m = np.full(sp.shape, 1.008)
    runs = []
    for variant in ("", "bf16x3"):
        mdl = _model()
        if variant:
            mdl.neural_networks.use_variant("bf16x3")
        ctx = pytest.warns(UserWarning, match="bfloat16") if not variant else _nothing()
        with ctx:
            dyn = md.VelocityVerlet(mdl, sp, co, m, dt=0.01, steps_per_replay=5, record_every=1)
            dyn.run(12)
        assert mdl.neural_networks._variant == "bf16x3"
        runs.append((np64(dyn.x), np64(dyn.v), dyn.thermo))
    assert np.abs(runs[0][0] - runs[1][0]).max() <= TRAJ_BAR[60]
    assert np.abs(runs[0][1] - runs[1][1]).max() <= TRAJ_BAR[60]
    assert np.abs(runs[0][2].potential - runs[1][2].potential).max() <= 1e-5


class _nothing:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


# ------------------------------------------------------------------------------------------------------------------
# 10. rejections and launches
# ------------------------------------------------------------------------------------------------------------------
def test_rejections():
    from torchani_b200 import md, models, potentials
    sp, co, cell, pbc, m = system("water30_pbc_ani2x")
    M = model()
    with pytest.raises(ValueError, match="dt"):
        md.VelocityVerlet(M, sp, co, m, dt=0.0, cell=cell, pbc=True)
    with pytest.raises(ValueError, match="masses"):
        md.VelocityVerlet(M, sp, co, m * 0, cell=cell, pbc=True)
    with pytest.raises(ValueError, match="temperature"):
        md.Langevin(M, sp, co, m, temperature=-1.0, cell=cell, pbc=True)
    with pytest.raises(ValueError, match="friction"):
        md.Langevin(M, sp, co, m, friction=-0.1, cell=cell, pbc=True)
    with pytest.raises(ValueError, match="partial PBC"):
        md.VelocityVerlet(M, sp, co, m, cell=cell, pbc=[True, True, False])
    eng = M.engine(torch.device(DEV))
    eng.skin = 1.0
    try:
        with pytest.raises(ValueError, match="Verlet-skin"):
            md.VelocityVerlet(M, sp, co, m, cell=cell, pbc=True)
    finally:
        eng.skin = 0.0
    ws = eng.workspace(1, sp.shape[1])
    ws.reducer = object()
    try:
        with pytest.raises(ValueError, match="sharded"):
            md.VelocityVerlet(M, sp, co, m, cell=cell, pbc=True)
    finally:
        ws.reducer = None
    base = models.ANI2x(seed=0)
    lj = models.ANI(base.symbols, base.aev_computer, base.neural_networks, base.energy_shifter, False,
                    {"lj": potentials.LennardJones(base.symbols)}).to(DEV)
    with pytest.raises(ValueError, match="infinite cutoff"):
        md.VelocityVerlet(lj, sp, co, m, cell=cell, pbc=True)


def test_engine_launches_unchanged_after_md():
    sp, co, cell, pbc, m = system("water30_pbc_ani2x")
    eng = model().engine(torch.device(DEV))
    args = (torch.as_tensor(sp).to(DEV), torch.tensor(co, dtype=torch.float32, device=DEV),
            torch.tensor(cell, dtype=torch.float32, device=DEV), True)
    r0 = eng.step(*args)
    before, e0 = eng.launches_per_step, float(r0.energies[0])
    dyn, _ = make("langevin", friction=0.05, steps_per_replay=10, qbc_stop=(math.inf, math.inf))
    dyn.run(20)
    r1 = eng.step(*args)
    assert eng.launches_per_step == before
    assert float(r1.energies[0]) == pytest.approx(e0, abs=1e-6)
