"""Constant-pressure MD on the device (md.LangevinNPT: csrc/md.cu ani_b200_md_step_npt) on the H100: one step against
the float64 oracles, the cell the force step sees, the sign and units of the internal pressure, the ideal gas's volume
distribution, replay shapes, the operand-range fallback, shared-cell batches, rejections, and the launches of the
other step forms.

The bars are those of tests/test_gpu_md.py: one integrator step is float64 given the forces (1e-12 relative); longer
runs differ by the force step's float32 atomics (TRAJ_BAR); energies from two force steps on the same float32 input
agree to 1e-5 Hartree.
"""
import math

import numpy as np
import pytest
import torch

import oracle.md_oracle as mo
import oracle.npt_oracle as no
from test_gpu_md import DEV, MASSES_2X, TRAJ_BAR, inv_mass, model, np64, system

pytestmark = pytest.mark.gpu

E_BAR = 1e-5   # Hartree: two force steps on the same float32 input (the AEV backward's atomics)


def npt(name="water30_pbc_ani2x", T=300.0, seed=0, sp=None, co=None, cell=None, m=None, mdl=None, **kw):
    from torchani_b200 import md
    if sp is None:
        sp, co, cell, _, m = system(name)
    kw.setdefault("velocities", md.maxwell_boltzmann(m, T, seed=11))
    kw.setdefault("friction", 0.05)
    return md.LangevinNPT(mdl or model(), sp, co, m, cell, temperature=T, seed=seed, **kw), m


def perturbed_batch(name, n=4, seed=2):
    """n copies of a periodic golden system, each in its own cell (scaled by 1 + 1 % per copy, the positions with it)
    with 0.02 A of noise."""
    sp, co, cell, _, m = system(name)
    rng = np.random.default_rng(seed)
    s = 1.0 + 0.01 * np.arange(n)
    cells = cell[None] * s[:, None, None] if cell.ndim == 2 else cell[0][None] * s[:, None, None]
    cos = co[0][None] * s[:, None, None] + 0.02 * rng.standard_normal((n,) + co.shape[1:])
    return np.repeat(sp, n, 0), cos, cells, np.repeat(m, n, 0)


def virial(dyn):
    return np64(dyn.ws.virial).reshape(dyn.n_conf, -1, 9).sum(1).reshape(-1, 3, 3)


def f32_cells(dyn):
    return np64(dyn.ws.cells if dyn.per_conf else dyn.ws.cell).reshape(dyn.n_conf, 3, 3)


# ------------------------------------------------------------------------------------------------------------------
# 1. one step against the oracle
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("batch", [False, True])
def test_one_step_vs_oracle(batch):
    """water999 (grid mode 0) and 4 perturbed copies in their own cells (mode 3): two steps of the device against
    md_oracle's finish / start and npt_oracle's cell_rescale, on the device's own forces, energies, virial and noise."""
    from torchani_b200 import md
    if batch:
        sp, co, cell, m = perturbed_batch("water999_pbc_ani2x")
    else:
        sp, co, cell, _, m = system("water999_pbc_ani2x")
    P0, tau, beta, T, gamma, dt = 200.0, 50.0, 4.5e-5, 300.0, 0.05, 0.5
    dyn, _ = npt(sp=sp, co=co, cell=cell, m=m, pressure=P0, tau_p=tau, compressibility=beta, steps_per_replay=1,
                 record_every=1)
    assert dyn.per_conf == batch
    C_ = dyn.n_conf
    im = inv_mass(m).reshape(C_, -1)
    x, v, h = np64(dyn.x), np64(dyn.v), np64(dyn.cell)
    for t in range(2):
        g = np64(dyn.ws.grad).reshape(x.shape)
        W = virial(dyn)
        e_pot = np64(dyn.ws.energies)
        v = mo.finish(v, g, im, dt, t)
        ek = mo.kinetic(v, im)
        noise = np64(md.noise(0, t, x.size // 3, DEV)).reshape(x.shape)
        x1, v1 = mo.start(x, v, g, im, dt, mo.LANGEVIN, T, gamma, noise)
        xi = np64(md.cell_noise(0, t, C_, DEV))
        x2, v2, h2, vol, p_int = no.cell_rescale(x1, v1, h, ek, W, T, P0 * no.BAR, tau, beta / no.BAR, dt, xi)
        h_dev = np64(dyn.cell)   # the device's master cell of step t (from t = 1 on within 1e-12 of the oracle's h)
        dyn.run(1)
        r = dyn.npt
        assert r.step[-1] == t and np.array_equal(dyn.thermo.potential[-1], e_pot)
        assert np.abs(r.volume[-1] - vol).max() <= 1e-12 * vol.max()
        p_scale = (2 * ek + np.abs(np.trace(W, axis1=1, axis2=2))) / (3 * vol)
        assert np.all(np.abs(r.pressure[-1] * no.BAR - p_int) <= 1e-12 * p_scale), (r.pressure[-1], p_int / no.BAR)
        assert np.array_equal(dyn.frame_cells[-1], h_dev)   # the frame holds the cell of its step, copied
        x, v, h = x2, v2, h2
        for got, ref, what in ((np64(dyn.x), x, "x"), (np64(dyn.v), v, "v"), (np64(dyn.cell), h, "cell")):
            err = np.abs(got - ref).max()
            assert err <= 1e-12 * np.abs(ref).max(), f"{what} step {t}: {err:.3e}"
        assert np.abs(np64(dyn.volume) - np.abs(np.linalg.det(h))).max() <= 1e-12 * vol.max()
    assert not np.allclose(h, dyn.frame_cells[0], rtol=1e-9, atol=0)   # the cell moved
    # the float32 cell of the next force step, and the coordinates wrapped into it
    h32 = h.astype(np.float32)
    assert np.all(np.abs(f32_cells(dyn) - h32) <= np.abs(h32) * 2.0 ** -23)
    c = np64(dyn.ws.coords).reshape(x.shape)
    ref = np.stack([mo.wrap(x[k], f32_cells(dyn)[k]) for k in range(C_)])
    assert np.abs(c - ref.astype(np.float32)).max() <= 4e-6


# ------------------------------------------------------------------------------------------------------------------
# 2. the force step sees the new cell
# ------------------------------------------------------------------------------------------------------------------
def test_graph_sees_the_new_cell():
    """100 steps at K = 10, a frame every step: the energy and virial the loop recorded at step 99 are those of a fresh
    HostCalculator.calculate_with_stress at that frame's positions and cell, and the energy the loop holds for step
    100 is that of the final positions in the final cell."""
    from torchani_b200.calculator import HostCalculator
    sp, co, cell, _, m = system("water999_pbc_ani2x")
    dyn, _ = npt(sp=sp, co=co, cell=cell, m=m, pressure=100.0, steps_per_replay=10, record_every=1)
    dyn.run(100)
    h = np64(dyn.cell)[0]
    assert np.abs(np64(dyn.volume)[0] - abs(np.linalg.det(h))) <= 1e-12 * abs(np.linalg.det(h))
    assert abs(np.linalg.det(h) / np.linalg.det(cell.reshape(3, 3)) - 1) > 1e-6, "the cell did not move"
    calc = HostCalculator(model(), sp[0], cell=cell.reshape(3, 3), pbc=True)
    fc = dyn.frame_cells[-1, 0]
    assert dyn.frames.step[-1] == 99
    e, _, stress = calc.calculate_with_stress(mo.wrap(dyn.frames.positions[-1, 0], fc), fc.astype(np.float32))
    r, th = dyn.npt, dyn.thermo
    assert th.step[-1] == 99 and abs(th.potential[-1, 0] - e) <= E_BAR
    p_vir = r.pressure[-1, 0] * no.BAR - 2 * th.kinetic[-1, 0] / (3 * r.volume[-1, 0])
    ref = -np.trace(stress) / 3
    assert abs(p_vir - ref) <= 1e-4 * np.abs(stress).max() + 1e-10, (p_vir, ref)
    e_end, _, _ = calc.calculate_with_stress(np64(dyn.ws.coords), h.astype(np.float32))
    assert abs(float(dyn.ws.energies[0]) - e_end) <= E_BAR


# ------------------------------------------------------------------------------------------------------------------
# 3. sign and units of the pressure
# ------------------------------------------------------------------------------------------------------------------
def _xtb_d3_model():
    import test_gpu_dispersion as td3
    return td3.model(xtb="smooth")


@pytest.mark.parametrize("which", ["ani2x", "xtb_d3"])
def test_pressure_is_minus_dE_dV(which):
    """With v = 0 the first step's P_int is the virial pressure -tr W / (3 V), which must be -dE/dV: central
    differences of the energy at the cell scaled by 1 +- 1e-3 with the fractional coordinates fixed.  The bar is sized
    from the float32 energy noise, measured as the spread of the energy over rigid translations of the whole box."""
    from torchani_b200.calculator import HostCalculator
    mdl = model() if which == "ani2x" else _xtb_d3_model()
    sp, co, cell, _, m = system("water999_pbc_ani2x")
    h = cell.reshape(3, 3)
    dyn, _ = npt(sp=sp, co=co, cell=h, m=m, mdl=mdl, velocities=np.zeros_like(co), steps_per_replay=1)
    dyn.run(1)
    p = dyn.npt.pressure[0, 0] * no.BAR
    calc = HostCalculator(mdl, sp[0], cell=h, pbc=True)

    def energy(s, shift=(0.0, 0.0, 0.0)):
        hc = h * (1 + s)
        e, _ = calc.calculate(mo.wrap(co[0] * (1 + s) + np.asarray(shift), hc).astype(np.float32))
        return float(e)

    calc.set_cell(h.astype(np.float32))
    e0 = [energy(0.0, sh) for sh in ([0, 0, 0], [0.31, 0.17, 0.05], [1.3, -0.7, 2.1], [-2.2, 0.4, -0.9])]
    noise = max(np.std(e0, ddof=1), 1e-9)
    s = 1e-3
    ep, em = [], []
    for sign, out in ((1, ep), (-1, em)):
        calc.set_cell((h * (1 + sign * s)).astype(np.float32))
        out.append(energy(sign * s))
    vol = abs(np.linalg.det(h))
    dv = vol * ((1 + s) ** 3 - (1 - s) ** 3)
    ref = -(ep[0] - em[0]) / dv
    bar = 6 * math.sqrt(2) * noise / dv + 1e-5 * abs(ref)
    assert abs(p - ref) <= bar, (p / no.BAR, ref / no.BAR, bar / no.BAR)
    assert abs(ref) > 3 * bar, "the pressure is lost in the noise: no check of its sign"


# ------------------------------------------------------------------------------------------------------------------
# 4. ideal gas
# ------------------------------------------------------------------------------------------------------------------
def zero_output_model():
    """Seeded ANI-2x-shaped networks whose output layers are zero: E is constant, F and W are zero."""
    import oracle.ani_oracle as orc
    from torchani_b200 import models
    w = orc.make_weights(orc.SYMBOLS_2X, orc.DIMS_2X, 1008, 1, 1234, torch.float32)
    w = [{s: list(layers[:-1]) + [(layers[-1][0] * 0, layers[-1][1] * 0)] for s, layers in wm.items()} for wm in w]
    base = models.from_weight_lists("2x", w, periodic_table_index=False)
    return models.ANI(base.symbols, base.aev_computer, base.neural_networks, base.energy_shifter, False).to(DEV)


def test_ideal_gas_volume_distribution():
    """64 replicas of 64 free atoms at P0 and 64 at 2 P0, each in its own cell, V ~ 27 000 A^3 at P0: V is
    Gamma(N + 1, k_B T / P0), so <V> = (N + 1) k_B T / P0 and Var(V) / <V>^2 = 1 / (N + 1).  beta_T = 1 / P (the
    ideal gas's compressibility) makes V relax in ~tau_p = 500 fs; 2 k steps of equilibration, then 20 k steps (20
    relaxation times per replica).  <V> within max(4 standard errors of the replica means, 1 %), the variance ratio
    within 15 % (its standard error is ~4 %), the mean temperature within 2 % (test_langevin_temperature's bar)."""
    from torchani_b200 import md
    C_, A, T = 128, 64, 300.0
    p0 = 65 * mo.KB * T / 27000.0 / no.BAR        # bar
    P = np.where(np.arange(C_) < 64, p0, 2 * p0)
    rng = np.random.default_rng(5)
    L = 30.0 * (1 + 0.01 * (np.arange(C_) % 5))
    cells = L[:, None, None] * np.eye(3)
    co = rng.uniform(0, 1, (C_, A, 3)) * L[:, None, None]
    sp = np.zeros((C_, A), dtype=np.int64)
    m = np.full((C_, A), 16.0)
    dyn = md.LangevinNPT(zero_output_model(), sp, co, m, cells, temperature=T, friction=0.05, pressure=P,
                         tau_p=500.0, compressibility=1.0 / P, velocities=md.maxwell_boltzmann(m, T, seed=2),
                         steps_per_replay=50, record_every=0)
    assert float(dyn.ws.grad.abs().max()) == 0.0 and np.abs(virial(dyn)).max() == 0.0
    dyn.run(22000)
    V = dyn.npt.volume[2000:]
    Tm = dyn.thermo.temperature[2000:].mean()
    assert abs(Tm / T - 1) < 0.02, Tm
    for grp, p in ((slice(0, 64), p0), (slice(64, 128), 2 * p0)):
        v = V[:, grp]
        target = (A + 1) * mo.KB * T / (p * no.BAR)
        se = v.mean(0).std(ddof=1) / math.sqrt(v.shape[1])
        assert abs(v.mean() - target) <= max(4 * se, 0.01 * target), (p, v.mean() / target, se / target)
        ratio = v.var() / v.mean() ** 2 * (A + 1)
        assert abs(ratio - 1) < 0.15, (p, ratio)


# ------------------------------------------------------------------------------------------------------------------
# 5. replay shapes
# ------------------------------------------------------------------------------------------------------------------
def test_replay_shapes_agree():
    """60 steps as one eager remainder (K = 64), as 60 replays of 1 and as 6 of 10: the same (x, v, cell)."""
    runs = []
    for K in (64, 1, 10):
        dyn, _ = npt(pressure=500.0, steps_per_replay=K, record_every=5)
        dyn.run(60)
        runs.append((np64(dyn.x), np64(dyn.velocities), np64(dyn.cell), dyn.npt))
    x0, v0, h0, r0 = runs[0]
    assert list(r0.step) == list(range(60))
    for x, v, h, r in runs[1:]:
        assert np.abs(x - x0).max() <= TRAJ_BAR[60] and np.abs(v - v0).max() <= TRAJ_BAR[60]
        assert np.abs(h - h0).max() <= TRAJ_BAR[60]
        assert np.abs(r.volume - r0.volume).max() <= 1e-6 * r0.volume.max()


# ------------------------------------------------------------------------------------------------------------------
# 6. operand-range fallback
# ------------------------------------------------------------------------------------------------------------------
def test_operand_range_fallback_matches_a_bf16x3_loop():
    """The cap system of test_gpu_md's fallback test in a 20 A box: the loop built on the 2 x fp16 build switches to
    3 x bfloat16 at its first force step, restores its state (master cells included) and then runs what a loop built on
    3 x bfloat16 runs."""
    from torchani_b200 import _lib, md
    from test_gpu_md import _model, _nothing
    from test_gpu_operand_range import cap_system
    if not _lib.available("bf16x3"):
        pytest.skip("the 3 x bfloat16 build is missing")
    s = cap_system(48)
    sp, co = s.species.numpy(), s.coords.double().numpy() + 5.0
    m = np.full(sp.shape, 1.008)
    cell = np.eye(3) * 20.0
    runs = []
    for variant in ("", "bf16x3"):
        mdl = _model()
        if variant:
            mdl.neural_networks.use_variant("bf16x3")
        ctx = pytest.warns(UserWarning, match="bfloat16") if not variant else _nothing()
        with ctx:
            dyn = md.LangevinNPT(mdl, sp, co, m, cell, dt=0.01, tau_p=10.0, pressure=1e4, steps_per_replay=5,
                                 record_every=1)
            dyn.run(12)
        assert mdl.neural_networks._variant == "bf16x3"
        runs.append((np64(dyn.x), np64(dyn.v), np64(dyn.cell), dyn.thermo))
    for k in range(3):
        assert np.abs(runs[0][k] - runs[1][k]).max() <= TRAJ_BAR[60], k
    assert np.abs(runs[0][3].potential - runs[1][3].potential).max() <= E_BAR
    assert not np.array_equal(runs[0][2][0], cell)


# ------------------------------------------------------------------------------------------------------------------
# 7. shared cell of a batch
# ------------------------------------------------------------------------------------------------------------------
def test_shared_cell_batch_gets_a_cell_per_conformer():
    sp, co, cell, _, m = system("water30_pbc_ani2x")
    sp3, co3, m3 = np.repeat(sp, 3, 0), np.repeat(co, 3, 0), np.repeat(m, 3, 0)
    dyn, _ = npt(sp=sp3, co=co3, cell=cell.reshape(3, 3), m=m3, pressure=500.0, steps_per_replay=10, record_every=0)
    assert dyn.per_conf and tuple(dyn.cell.shape) == (3, 3, 3)
    dyn.run(50)
    h = np64(dyn.cell)
    assert not np.array_equal(h[0], h[1]) and not np.array_equal(h[1], h[2])
    for k in range(3):   # each conformer's coordinates are wrapped into its own float32 cell
        frac = np64(dyn.ws.coords).reshape(3, -1, 3)[k] @ np.linalg.inv(f32_cells(dyn)[k])
        assert frac.min() >= -1e-6 and frac.max() <= 1 + 1e-6


# ------------------------------------------------------------------------------------------------------------------
# 8. rejections
# ------------------------------------------------------------------------------------------------------------------
def test_rejections():
    from torchani_b200 import md
    sp, co, cell, _, m = system("water30_pbc_ani2x")
    M = model()
    with pytest.raises(ValueError, match="periodic"):
        md.LangevinNPT(M, sp, co, m, None)
    with pytest.raises(ValueError, match="volume"):
        md.LangevinNPT(M, sp, co, m, np.diag([10.0, 10.0, 0.0]))
    with pytest.raises(ValueError, match="qbc_stop"):
        md.LangevinNPT(M, sp, co, m, cell, qbc_stop=(math.inf, math.inf))
    with pytest.raises(ValueError, match="pressure"):
        md.LangevinNPT(M, sp, co, m, cell, pressure=math.nan)
    with pytest.raises(ValueError, match="tau_p"):
        md.LangevinNPT(M, sp, co, m, cell, tau_p=0.0)
    with pytest.raises(ValueError, match="compressibility"):
        md.LangevinNPT(M, sp, co, m, cell, compressibility=-1.0)
    with pytest.raises(ValueError, match="temperature"):
        md.LangevinNPT(M, sp, co, m, cell, temperature=0.0)
    with pytest.raises(ValueError, match="dt"):
        md.LangevinNPT(M, sp, co, m, cell, dt=-0.5)


# ------------------------------------------------------------------------------------------------------------------
# 9. the other step forms are unchanged
# ------------------------------------------------------------------------------------------------------------------
def test_engine_and_nvt_launches_unchanged_after_npt():
    """Engine.step, an NVE and an NVT loop issue the same launches and give the same results before and after an NPT
    run on the same engine."""
    from test_gpu_md import make
    sp, co, cell, pbc, m = system("water30_pbc_ani2x")
    eng = model().engine(torch.device(DEV))
    args = (torch.as_tensor(sp).to(DEV), torch.tensor(co, dtype=torch.float32, device=DEV),
            torch.tensor(cell, dtype=torch.float32, device=DEV), True)

    def others():
        r = eng.step(*args)
        out = [eng.launches_per_step, float(r.energies[0])]
        for kind in ("verlet", "langevin"):
            dyn, _ = make(kind, friction=0.05, steps_per_replay=10) if kind == "langevin" else \
                make(kind, steps_per_replay=10)
            dyn.run(20)
            out += [eng.launches_per_step, np64(dyn.x)]
        return out

    before = others()
    dyn, _ = npt(pressure=500.0, steps_per_replay=10)
    dyn.run(20)
    after = others()
    assert before[0] == after[0] and before[2] == after[2] and before[4] == after[4]
    assert after[1] == pytest.approx(before[1], abs=1e-6)
    assert np.abs(after[3] - before[3]).max() <= TRAJ_BAR[60]
    assert np.abs(after[5] - before[5]).max() <= TRAJ_BAR[60]
