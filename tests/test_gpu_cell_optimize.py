"""Variable-cell FIRE on the device (optimize.CellFIRE: csrc/opt.cu ani_b200_opt_cell_step) on the H100: one to three
steps against the float64 oracle, bitwise reproducibility, the device loop against a host loop, the cell force against
central differences of the enthalpy, a known lattice constant (fcc Lennard-Jones) at zero and high pressure, the
projections, batches, a second run, the operand-range fallback, the rejections and the launches of the other step forms.

The bars are those of tests/test_gpu_optimize.py: one step is float64 given the forces and the virial (1e-12
relative); trajectories differ by the force step's float32 atomics and run TRAJ_STEPS steps (TRAJ_BAR).
"""
import math

import numpy as np
import pytest
import torch
from scipy.linalg import expm

import oracle.cell_fire_oracle as co
import oracle.fire_oracle as fo
import oracle.lj_coulomb_oracle as ljo
import oracle.md_oracle as mo
import oracle.npt_oracle as no
from test_gpu_optimize import DEV, TRAJ_BAR, TRAJ_STEPS, _nothing, model, np64, system

pytestmark = pytest.mark.gpu

LJ_SIGMA, LJ_EPS, LJ_RC = 2.5, 0.5, 6.25   # A, eV, A: the crystal's LJ and its smooth envelope's cutoff
_MODELS = {}


def lj_cut_model():
    """test_gpu_optimize's pure Lennard-Jones model (zero networks, no self energies) with a finite smooth cutoff."""
    if "lj" not in _MODELS:
        from torchani_b200 import models, potentials
        base = models.ANI2x(seed=0)
        with torch.no_grad():
            for p in base.neural_networks.parameters():
                p.zero_()
        S = len(base.symbols)
        lj = potentials.LennardJones(base.symbols, eps=[LJ_EPS / mo.HARTREE_EV] * S, sigma=[LJ_SIGMA] * S,
                                     cutoff=LJ_RC, cutoff_fn="smooth")
        _MODELS["lj"] = models.ANI(base.symbols, base.aev_computer, base.neural_networks,
                                   models.SelfEnergy(base.symbols, [0.0] * S), False, {"lj": lj}).to(DEV)
    return _MODELS["lj"]


def fcc(a, n=4):
    base = np.array([[0, 0, 0], [0, 0.5, 0.5], [0.5, 0, 0.5], [0.5, 0.5, 0]])
    cells = np.array([(i, j, k) for i in range(n) for j in range(n) for k in range(n)])
    return a * (cells[:, None] + base[None]).reshape(-1, 3), a * n * np.eye(3)


SHEAR = np.array([[1.03, 0.04, 0.0], [-0.02, 0.98, 0.03], [0.01, 0.0, 1.02]])


def strained_crystal(a=1.56 * LJ_SIGMA, seed=0, shear=SHEAR):
    rng = np.random.default_rng(seed)
    r, h = fcc(a)
    return r @ shear + 0.02 * rng.standard_normal(r.shape), h @ shear


def lattice_constant(p0_bar):
    """The fcc lattice constant minimising E(a) + p0 a^3 per conventional cell, from lj_coulomb_oracle (float64)."""
    from scipy.optimize import minimize_scalar
    one, zero = torch.ones(1, dtype=torch.float64), torch.zeros(1, dtype=torch.float64)
    spec = ljo.Spec("lj", LJ_RC, "smooth", one * LJ_EPS / mo.HARTREE_EV, one * LJ_SIGMA, zero, zero)
    p0 = p0_bar * no.BAR

    def h(a):
        r, cell = fcc(a, 1)
        out = ljo.compute(spec, torch.zeros(1, 4, dtype=torch.long), torch.as_tensor(r)[None], torch.as_tensor(cell),
                          torch.ones(3, dtype=torch.bool), neighborlist="all_pairs")
        return float(out["energy"][0]) + p0 * a ** 3
    return minimize_scalar(h, bracket=(1.50 * LJ_SIGMA, 1.55 * LJ_SIGMA, 1.60 * LJ_SIGMA), tol=1e-12).x


def virial(opt):
    return np64(opt.ws.virial).reshape(opt.n_conf, -1, 9).sum(1).reshape(-1, 3, 3)


def master(opt, slot):
    m = np64(opt._master[slot])
    return m[:, :9].reshape(-1, 3, 3), m[:, 9:18].reshape(-1, 3, 3), m[:, 18:].reshape(-1, 3, 3)


def f32_cells(opt):
    return np64(opt.ws.cells if opt.per_conf else opt.ws.cell).reshape(opt.n_conf, 3, 3)


def perturbed_batch(name, n=3, seed=2):
    sp, co_, cell, _ = system(name)
    rng = np.random.default_rng(seed)
    s = 1.0 + 0.01 * np.arange(n)
    cells = cell[None] * s[:, None, None]
    pos = co_[0][None] * s[:, None, None] + 0.02 * rng.standard_normal((n,) + co_.shape[1:])
    return np.repeat(sp, n, 0), pos, cells


# ------------------------------------------------------------------------------------------------------------------
# 1. one to three steps against the oracle
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["water30_pbc_ani2x", "benzene_pbc_ani2x", "batch"])
def test_three_steps_vs_oracle(name):
    """u, v, d, v_cell, F, the cell, fmax and the records against cell_fire_oracle.step on the device's own grad,
    energies and virial (1e-12 relative), at p0 = 5 kbar; the float32 cell and coordinates of the next force step."""
    from torchani_b200 import optimize
    if name == "batch":
        sp, pos, cell = perturbed_batch("water30_pbc_ani2x")
    else:
        sp, pos, cell, _ = system(name)
    P0 = 5000.0
    opt = optimize.CellFIRE(model(), sp, pos, cell, pressure=P0, steps_per_replay=1, maxstep=0.05)
    assert opt.per_conf == (name == "batch")
    C_ = opt.n_conf
    h0 = np.broadcast_to(np.asarray(cell).reshape(-1, 3, 3), (C_, 3, 3))
    c = (sp >= 0).sum(-1).reshape(C_).astype(np.float64)
    scale = np.where(sp.reshape(C_, -1) >= 0, fo.HARTREE_EV, 0.0)
    par = fo.params(0.0, maxstep=0.05)
    p0 = P0 * no.BAR
    u, v = np64(opt.x), np.zeros_like(np64(opt.x))
    d, vc = np.zeros((C_, 3, 3)), np.zeros((C_, 3, 3))
    sc = [fo.init(par) for _ in range(C_)]
    for t in range(3):
        g = np64(opt.ws.grad).reshape(u.shape)
        e, W = np64(opt.ws.energies), virial(opt)
        fmax, rec = np.zeros(C_), np.zeros((C_, 3))
        for k in range(C_):
            u[k], v[k], d[k], vc[k], sc[k], fmax[k], _, rec[k] = co.step(
                u[k], v[k], d[k], vc[k], sc[k], g[k], W[k], e[k], h0[k], p0, c[k], par, t, scale[k])
        assert not opt.run(fmax=0.0, steps=1)
        log = opt.log
        assert log.step[-1] == t and np.array_equal(log.energy[-1], e)
        assert np.abs(log.fmax[-1] - fmax).max() <= 1e-12 * fmax.max()
        for got, ref in ((log.volume[-1], rec[:, 0]), (log.pressure[-1] * no.BAR, rec[:, 1]),
                         (log.enthalpy[-1], rec[:, 2])):
            assert np.abs(got - ref).max() <= 1e-12 * np.abs(ref).max()
        F = np.stack([expm(d[k] / c[k]) for k in range(C_)])
        md, mv, mF = master(opt, (t + 1) % 2)
        for got, ref, what in ((np64(opt.x), u, "u"), (np64(opt.v), v, "v"), (md, d, "d"), (mv, vc, "v_cell"),
                               (mF, F, "F"), (np64(opt.cell), h0 @ F.transpose(0, 2, 1), "cell"),
                               (np64(opt.positions), u @ F.transpose(0, 2, 1), "positions")):
            err = np.abs(got - ref).max()
            assert err <= 1e-12 * max(np.abs(ref).max(), 1e-300), f"{what} step {t}: {err:.3e}"
        assert np.abs(d).max() > 0   # the cell moved
    h = h0 @ F.transpose(0, 2, 1)
    h32 = h.astype(np.float32)
    assert np.all(np.abs(f32_cells(opt) - h32) <= np.abs(h32) * 2.0 ** -23)
    cc = np64(opt.ws.coords).reshape(u.shape)
    ref = np.stack([mo.wrap(u[k] @ F[k].T, f32_cells(opt)[k]) for k in range(C_)])
    assert np.abs(cc - ref.astype(np.float32)).max() <= 4e-6
    # the properties of the current state
    assert np.abs(np64(opt.volume) - np.abs(np.linalg.det(h))).max() <= 1e-12 * np.abs(np.linalg.det(h)).max()
    W = virial(opt)
    vol = np.abs(np.linalg.det(h))
    assert np.abs(np64(opt.stress) - W / vol[:, None, None]).max() <= 1e-12 * np.abs(W / vol[:, None, None]).max()
    assert np.abs(np64(opt.enthalpies) - (np64(opt.energies) + p0 * vol)).max() <= 1e-9


def test_cell_launches_are_bitwise_reproducible():
    from torchani_b200 import optimize
    sp, pos, cell = perturbed_batch("water30_pbc_ani2x")
    opt = optimize.CellFIRE(model(), sp, pos, cell, pressure=1000.0, steps_per_replay=4)
    opt.run(0.0, 6)
    saved = opt._buf.clone()
    outs = []
    for _ in range(2):
        opt._buf.copy_(saved)
        opt._integrate()
        torch.cuda.synchronize()
        outs.append((opt._buf.clone().view(torch.int64), opt.ws.coords.clone().view(torch.int32),
                     opt.ws.cells.clone().view(torch.int32), opt._cell_force.clone().view(torch.int64)))
    for a, b in zip(*outs):
        assert torch.equal(a, b)
    assert not torch.equal(outs[0][0], saved.view(torch.int64))


# ------------------------------------------------------------------------------------------------------------------
# 2. the device loop against a host loop
# ------------------------------------------------------------------------------------------------------------------
def test_device_loop_vs_host_loop():
    """TRAJ_STEPS steps on the device against HostCalculator.calculate_with_stress + oracle steps on the same float32
    coordinates and cells (TRAJ_BAR for the positions and the cell)."""
    from torchani_b200 import optimize
    from torchani_b200.calculator import HostCalculator
    sp, pos, cell, _ = system("water30_pbc_ani2x")
    P0 = 2000.0
    opt = optimize.CellFIRE(model(), sp, pos, cell, pressure=P0, steps_per_replay=10)
    calc = HostCalculator(model(), sp[0], cell=cell, pbc=True)
    c, p0 = float((sp >= 0).sum()), P0 * no.BAR
    par = fo.params(0.0)
    scale = np.where(sp[0] >= 0, fo.HARTREE_EV, 0.0)
    u, v, d, vc, sc = pos[0].copy(), np.zeros_like(pos[0]), np.zeros((3, 3)), np.zeros((3, 3)), fo.init(par)
    for t in range(TRAJ_STEPS):
        F = expm(d / c)
        h32 = (cell @ F.T).astype(np.float32)
        e, f, stress = calc.calculate_with_stress(mo.wrap(u @ F.T, h32).astype(np.float32), h32)
        W = np.asarray(stress, dtype=np.float64) * abs(np.linalg.det(h32.astype(np.float64)))
        u, v, d, vc, sc, _, _, _ = co.step(u, v, d, vc, sc, -np.asarray(f, dtype=np.float64), W, e, cell, p0, c, par,
                                            t, scale)
    opt.run(0.0, TRAJ_STEPS)
    F = expm(d / c)
    assert np.abs(np64(opt.positions)[0] - u @ F.T).max() <= TRAJ_BAR
    assert np.abs(np64(opt.cell)[0] - cell @ F.T).max() <= TRAJ_BAR
    assert np.abs(d).max() > 1e-3


# ------------------------------------------------------------------------------------------------------------------
# 3. the cell force is -dH/dd
# ------------------------------------------------------------------------------------------------------------------
def _xtb_d3_model():
    import test_gpu_dispersion as td3
    return td3.model(xtb="smooth")


@pytest.mark.parametrize("which", ["ani2x", "xtb_d3"])
def test_cell_force_is_minus_dH_dd(which):
    """The first step's Phi (eV) along a direction D that strains and shears the cell equals -dH/ds of
    H(s) = E(r0 expm(s D / c)^T, h0 expm(s D / c)^T) + p0 V by central differences through the model API, at p0 = 20 kbar.
    The bar is sized from the float32 energy noise, the spread of E over rigid translations of the whole box."""
    from torchani_b200 import optimize
    from torchani_b200.calculator import HostCalculator
    mdl = model() if which == "ani2x" else _xtb_d3_model()
    sp, pos, cell, _ = system("water999_pbc_ani2x")
    h0 = cell.reshape(3, 3)
    P0 = 20000.0
    opt = optimize.CellFIRE(mdl, sp, pos, h0, pressure=P0, steps_per_replay=1)
    opt.run(0.0, 1)
    phi = np64(opt._cell_force)[0].reshape(3, 3)
    c, p0 = float((sp >= 0).sum()), P0 * no.BAR
    D = np.array([[1.0, 0.4, -0.2], [0.4, -0.5, 0.3], [-0.2, 0.3, 0.7]])
    calc = HostCalculator(mdl, sp[0], cell=h0, pbc=True)

    def enthalpy(s, shift=(0.0, 0.0, 0.0)):
        F = expm(s * D / c)
        h = (h0 @ F.T).astype(np.float32)
        calc.set_cell(h)
        e, _ = calc.calculate(mo.wrap(pos[0] @ F.T + np.asarray(shift), h).astype(np.float32))
        return float(e) + p0 * abs(np.linalg.det(h.astype(np.float64)))

    e0 = [enthalpy(0.0, sh) for sh in ([0, 0, 0], [0.31, 0.17, 0.05], [1.3, -0.7, 2.1], [-2.2, 0.4, -0.9])]
    noise = max(np.std(e0, ddof=1), 1e-9)
    s = 1e-3 * c
    ref = -(enthalpy(s) - enthalpy(-s)) / (2 * s) * fo.HARTREE_EV
    got = float((phi * D).sum())
    bar = 6 * math.sqrt(2) * noise / (2 * s) * fo.HARTREE_EV + 1e-4 * abs(ref)
    assert abs(got - ref) <= bar, (got, ref, bar)
    assert abs(ref) > 3 * bar, "the cell force is lost in the noise"


# ------------------------------------------------------------------------------------------------------------------
# 4. a known lattice constant: 256-atom fcc Lennard-Jones
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P0", [0.0, 10000.0])
def test_fcc_relaxes_to_the_lattice_constant(P0):
    """From a strained and sheared start the crystal converges (fmax 5e-4 eV / A) to a cubic cell: its Gram matrix
    h h^T is (4 a)^2 I with a the oracle's one-dimensional minimum of E(a) + p0 a^3, to 1e-4 relative in a (the filter may
    rotate the cell, the Gram matrix does not see it); W / V + p0 I is within the bound fmax implies, ~c fmax / V."""
    from torchani_b200 import optimize
    r, h = strained_crystal()
    sp = np.zeros(len(r), dtype=np.int64)
    fmax = 5e-4
    opt = optimize.CellFIRE(lj_cut_model(), sp, r, h, pressure=P0, steps_per_replay=50)
    assert opt.run(fmax=fmax, steps=3000), opt.log.fmax[-5:]
    a = lattice_constant(P0)
    hf = np64(opt.cell)[0]
    gram = hf @ hf.T / (4 * a) ** 2
    assert np.abs(gram - np.eye(3)).max() <= 2e-4, (gram, a)
    if P0 > 0:   # (10 kbar compresses this crystal, B ~ 2.4 eV / A^3, by ~1e-4 in a: the stress check below sees p0)
        assert a < lattice_constant(0.0)
    vol = float(np64(opt.volume)[0])
    dev = np64(opt.stress)[0] + P0 * no.BAR * np.eye(3)
    bound = 2 * len(r) * fmax / fo.HARTREE_EV / vol
    assert np.abs(dev).max() <= bound, (dev, bound)
    assert opt.log.enthalpy[-1, 0] < opt.log.enthalpy[0, 0]


@pytest.mark.parametrize("kind", ["hydrostatic_strain", "constant_volume"])
def test_projections_on_the_device(kind):
    """hydrostatic_strain keeps the cell's shape (h h^T proportional to h0 h0^T); constant_volume keeps V to 1e-12."""
    from torchani_b200 import optimize
    r, h = strained_crystal(seed=1)
    sp = np.zeros(len(r), dtype=np.int64)
    opt = optimize.CellFIRE(lj_cut_model(), sp, r, h, pressure=5000.0, steps_per_replay=20, **{kind: True})
    opt.run(0.0, 100)
    hf = np64(opt.cell)[0]
    v0 = abs(np.linalg.det(h))
    if kind == "hydrostatic_strain":
        g, g0 = hf @ hf.T, h @ h.T
        assert np.abs(g / g[0, 0] - g0 / g0[0, 0]).max() <= 1e-12
        assert abs(np.linalg.det(hf) / v0 - 1) > 1e-3
    else:
        assert abs(np.linalg.det(hf) / v0 - 1) <= 1e-12
        assert np.abs(hf - h).max() > 1e-3
        assert np.abs(np64(opt.volume)[0] / v0 - 1) <= 1e-12


# ------------------------------------------------------------------------------------------------------------------
# 5. batches and a second run
# ------------------------------------------------------------------------------------------------------------------
def test_batch_vs_single_and_a_second_run():
    """Three perturbed copies of water30 in one shared cell (which becomes one cell per conformer), TRAJ_STEPS steps at
    2 kbar: each as it is alone (TRAJ_BAR); then a crystal relaxed to fmax 0.05 and again to 1e-3 eV / A: the second
    run continues from the first's state (steps, FIRE scalars, cell)."""
    from torchani_b200 import optimize
    sp, pos, cells = perturbed_batch("water30_pbc_ani2x")
    h = cells[0]
    batch = optimize.CellFIRE(model(), sp, pos, h, pressure=2000.0, steps_per_replay=10)
    assert batch.per_conf
    batch.run(0.0, TRAJ_STEPS)
    for k in range(3):
        one = optimize.CellFIRE(model(), sp[k], pos[k], h, pressure=2000.0, steps_per_replay=10)
        one.run(0.0, TRAJ_STEPS)
        assert np.abs(np64(batch.positions)[k] - np64(one.positions)[0]).max() <= TRAJ_BAR
        assert np.abs(np64(batch.cell)[k] - np64(one.cell)[0]).max() <= TRAJ_BAR
    assert not np.array_equal(np64(batch.cell)[0], np64(batch.cell)[1])
    r, hc = strained_crystal()
    opt = optimize.CellFIRE(lj_cut_model(), np.zeros(len(r), dtype=np.int64), r, hc, steps_per_replay=10)
    assert opt.run(fmax=0.05, steps=1000)
    s1, h1 = opt.step, np64(opt.cell)
    assert opt.run(fmax=1e-3, steps=2000)
    assert opt.log.step[0] == 0 and opt.log.step[-1] == opt.step - 1 and (opt.converged_step >= s1).all()
    assert opt.log.fmax[-1, 0] < 1e-3 and not np.array_equal(np64(opt.cell), h1)


# ------------------------------------------------------------------------------------------------------------------
# 6. operand-range fallback
# ------------------------------------------------------------------------------------------------------------------
def test_operand_range_fallback_matches_a_bf16x3_loop():
    """The cap system of the FIRE fallback test in a 20 A box: the loop built on 2 x fp16 switches to 3 x bfloat16 at
    its first force step, restores its state (the master cell included) and then runs what a loop built on 3 x bfloat16
    from the start runs."""
    from torchani_b200 import _lib, optimize
    from test_gpu_md import _model
    from test_gpu_operand_range import cap_system
    if not _lib.available("bf16x3"):
        pytest.skip("the 3 x bfloat16 build is missing")
    s = cap_system(48)
    sp, pos = s.species.numpy(), s.coords.double().numpy() + 5.0
    cell = np.eye(3) * 20.0
    runs = []
    for variant in ("", "bf16x3"):
        mdl = _model()
        if variant:
            mdl.neural_networks.use_variant("bf16x3")
        ctx = pytest.warns(UserWarning, match="bfloat16") if not variant else _nothing()
        with ctx:
            opt = optimize.CellFIRE(mdl, sp, pos, cell, pressure=1e4, maxstep=0.01, steps_per_replay=5)
            opt.run(0.0, 12)
        assert mdl.neural_networks._variant == "bf16x3"
        runs.append((np64(opt.positions), np64(opt.cell), opt.log))
    assert np.abs(runs[0][0] - runs[1][0]).max() <= TRAJ_BAR
    assert np.abs(runs[0][1] - runs[1][1]).max() <= TRAJ_BAR
    assert np.abs(runs[0][2].energy - runs[1][2].energy).max() <= 1e-5
    assert not np.array_equal(runs[0][1][0], cell)


# ------------------------------------------------------------------------------------------------------------------
# 7. rejections and launches
# ------------------------------------------------------------------------------------------------------------------
def test_rejections():
    from torchani_b200 import models, optimize, potentials
    sp, pos, cell, _ = system("water30_pbc_ani2x")
    M = model()
    with pytest.raises(ValueError, match="periodic"):
        optimize.CellFIRE(M, sp, pos, None)
    with pytest.raises(ValueError, match="periodic"):
        optimize.CellFIRE(M, sp, pos, cell, pbc=[True, False, True])
    with pytest.raises(ValueError, match="fixed"):
        optimize.CellFIRE(M, sp, pos, cell, fixed=np.zeros(sp.shape[1], dtype=bool))
    with pytest.raises(ValueError, match="pressure"):
        optimize.CellFIRE(M, sp, pos, cell, pressure=math.nan)
    with pytest.raises(ValueError, match="cell_factor"):
        optimize.CellFIRE(M, sp, pos, cell, cell_factor=0.0)
    with pytest.raises(ValueError, match="exclusive"):
        optimize.CellFIRE(M, sp, pos, cell, hydrostatic_strain=True, constant_volume=True)
    with pytest.raises(ValueError, match="volume"):
        optimize.CellFIRE(M, sp, pos, np.diag([8.0, 8.0, 0.0]))
    opt = optimize.CellFIRE(M, sp, pos, cell)
    with pytest.raises(ValueError, match="fmax"):
        opt.run(-0.05, 10)
    eng = M.engine(torch.device(DEV))
    eng.skin = 1.0
    try:
        with pytest.raises(ValueError, match="Verlet-skin"):
            optimize.CellFIRE(M, sp, pos, cell)
    finally:
        eng.skin = 0.0
    base = models.ANI2x(seed=0)
    lj = models.ANI(base.symbols, base.aev_computer, base.neural_networks, base.energy_shifter, False,
                    {"lj": potentials.LennardJones(base.symbols)}).to(DEV)
    with pytest.raises(ValueError, match="infinite cutoff"):
        optimize.CellFIRE(lj, sp, pos, cell)
    # a box that shrinks below the cutoff: 8 free atoms (zero forces and virial) at 10 kbar, each step clamped to
    # |dL| = 0.5 / sqrt(3) per diagonal entry, so the 30 A box is thinner than the AEV cutoff after ~6 steps: the status
    # error of the step, at the end of the replay
    from test_gpu_npt import zero_output_model
    rng = np.random.default_rng(3)
    sq = optimize.CellFIRE(zero_output_model(), np.zeros(8, dtype=np.int64), rng.uniform(0, 30, (8, 3)),
                           30.0 * np.eye(3), pressure=1e4, cell_factor=1.0, maxstep=0.5, steps_per_replay=10)
    with pytest.raises(RuntimeError, match="too small"):
        sq.run(0.0, 20)


def test_other_launches_unchanged_after_a_cell_optimisation():
    """Engine.step, FIRE, NVE, NVT, NPT and HostCalculator issue the same launches and give the same results before and
    after a CellFIRE run on the same engine."""
    from torchani_b200 import md, optimize
    from torchani_b200.calculator import HostCalculator
    sp, pos, cell, _ = system("water30_pbc_ani2x")
    eng = model().engine(torch.device(DEV))
    args = (torch.as_tensor(sp).to(DEV), torch.tensor(pos, dtype=torch.float32, device=DEV),
            torch.tensor(cell, dtype=torch.float32, device=DEV), True)
    m = np.where(sp >= 0, 1.008, 0.0)
    calc = HostCalculator(model(), sp, cell=cell, pbc=True)

    def others():
        r = eng.step(*args)
        out = [eng.launches_per_step, float(r.energies[0])]
        fire = optimize.FIRE(model(), sp, pos, cell=cell, pbc=True, steps_per_replay=10)
        fire.run(0.0, 20)
        out += [eng.launches_per_step, np64(fire.x)]
        for dyn in (md.VelocityVerlet(model(), sp, pos, m, cell=cell, pbc=True, steps_per_replay=5, record_every=0),
                    md.Langevin(model(), sp, pos, m, cell=cell, pbc=True, steps_per_replay=5, record_every=0),
                    md.LangevinNPT(model(), sp, pos, m, cell, pressure=500.0, steps_per_replay=5, record_every=0)):
            dyn.run(10)
            out += [eng.launches_per_step, np64(dyn.x)]
        out += [np.asarray(calc.calculate(pos[0])[1], dtype=np.float64)]
        return out

    before = others()
    opt = optimize.CellFIRE(model(), sp, pos, cell, pressure=1000.0, steps_per_replay=10)
    opt.run(0.05, 20)
    after = others()
    for k in (0, 2, 4, 6, 8):
        assert before[k] == after[k], k
    assert after[1] == pytest.approx(before[1], abs=1e-6)
    for k in (3, 5, 7, 9):
        assert np.abs(after[k] - before[k]).max() <= TRAJ_BAR, k
    assert np.abs(after[10] - before[10]).max() <= 1e-5
