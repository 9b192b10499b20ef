"""The device FIRE loop (csrc/opt.cu, torchani_b200/optimize.py) on the H100: one to three steps against the float64
oracle, the device loop against a host loop of Engine.step + oracle steps, a known minimum (LJ13) through the fused
step, convergence and freezing, fixed atoms, replay shapes, periodic input, the operand-range fallback and the rejected
inputs.

The bars, and where they come from:
* one to three steps: FIRE is float64 and the forces are inputs, so x, v, the scalars and the record agree with the
  oracle to float64 rounding of a few operations (1e-12 relative);
* longer runs: the FIRE launches are bitwise reproducible, the force step is not (the AEV backward adds float32
  contributions with atomics), and a difference in the last bits of a force then grows along the optimisation.
  TRAJ_BAR is sized from two device runs of the same input on the H100 (see its comment).
"""
import math

import numpy as np
import pytest
import torch

import oracle.fire_oracle as fo
import oracle.md_oracle as mo
from helpers import golden_inputs, load_golden

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
# two device runs of the same input, TRAJ_STEPS steps of small264_nopbc_ani2x, water30_pbc_ani2x and randbatch_ani2x,
# were measured at most 7e-7 A apart on an H100 (the force step's atomics, module docstring).  Over longer runs FIRE's
# discrete choices (a step with P <= 0 halves dt and zeroes v) amplify such differences fast: the same pairs of runs
# were 1.5e-4 A apart after 60 steps and 1.7e-2 A after 100 on water30_pbc.  So every trajectory comparison runs
# TRAJ_STEPS steps, and the bar leaves a factor of 14 over the measured spread.
TRAJ_STEPS = 30
TRAJ_BAR = 1e-5
LJ_SIGMA, LJ_EPS = 2.5, 0.5   # A, eV: forces of O(1) eV / A at 0.08 sigma from the minimum


def _model():
    from torchani_b200 import models
    base = models.ANI2x(seed=0)
    return models.ANI(base.symbols, base.aev_computer, base.neural_networks, base.energy_shifter, False).to(DEV)


_MODEL = {}


def model():
    if "m" not in _MODEL:
        _MODEL["m"] = _model()
    return _MODEL["m"]


def lj_model():
    """A pure Lennard-Jones model: every network weight and bias zero, no self energies, and one LJ term without a
    cutoff (its envelope is then none)."""
    if "lj" not in _MODEL:
        from torchani_b200 import models, potentials
        base = models.ANI2x(seed=0)
        with torch.no_grad():
            for p in base.neural_networks.parameters():
                p.zero_()
        S = len(base.symbols)
        lj = potentials.LennardJones(base.symbols, eps=[LJ_EPS / mo.HARTREE_EV] * S, sigma=[LJ_SIGMA] * S,
                                     cutoff=math.inf)
        assert lj.cutoff_fn == "dummy"
        _MODEL["lj"] = models.ANI(base.symbols, base.aev_computer, base.neural_networks,
                                  models.SelfEnergy(base.symbols, [0.0] * S), False, {"lj": lj}).to(DEV)
    return _MODEL["lj"]


def lj13_batch(n, seed=2024):
    rng = np.random.default_rng(seed)
    return np.stack([fo.icosahedron(LJ_SIGMA) + 0.08 * LJ_SIGMA * rng.standard_normal((13, 3)) for _ in range(n)])


def system(name):
    sp, co, cell, pbc = golden_inputs(load_golden(name))
    return sp.numpy(), co.numpy(), None if cell is None else cell.numpy(), bool(pbc is not None and bool(pbc.all()))


def make(name, **kw):
    from torchani_b200 import optimize
    sp, co, cell, pbc = system(name)
    return optimize.FIRE(model(), sp, co, cell=cell, pbc=pbc, **kw)


def np64(t):
    return t.detach().double().cpu().numpy()


# ------------------------------------------------------------------------------------------------------------------
# 1. one, two and three steps against the oracle
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["water30_pbc_ani2x", "small264_nopbc_ani2x", "randbatch_ani2x"])
def test_three_steps_vs_oracle(name):
    opt = make(name, steps_per_replay=1, maxstep=0.05)
    sp, _, cell, pbc = system(name)
    scale = np.where(sp >= 0, fo.HARTREE_EV, 0.0)
    par = fo.params(0.0, maxstep=0.05)
    C_ = opt.n_conf
    x, v = np64(opt.x), np.zeros_like(np64(opt.x))
    sc = [fo.init(par) for _ in range(C_)]
    for t in range(3):
        g = np64(opt.ws.grad).reshape(x.shape)
        e = np64(opt.ws.energies)
        fmax = np.zeros(C_)
        for c in range(C_):
            x[c], v[c], sc[c], fmax[c], _ = fo.step(x[c], v[c], sc[c], g[c], scale[c], par, t)
        assert not opt.run(fmax=0.0, steps=1)
        log = opt.log
        assert log.step[-1] == t
        assert np.array_equal(log.energy[-1], e)
        assert np.abs(log.fmax[-1] - fmax).max() <= 1e-12 * fmax.max()
        for got, ref, what in ((np64(opt.x), x, "x"), (np64(opt.v), v, "v")):
            err = np.abs(got - ref).max()
            assert err <= 1e-12 * max(np.abs(ref).max(), 1e-300), f"{what} step {t}: {err:.3e}"
        got_sc = np64(opt._scalars[(t + 1) % 2])
        assert np.abs(got_sc - np.stack(sc)).max() <= 1e-12 * np.abs(np.stack(sc)).max(), t
    c32 = np64(opt.ws.coords).reshape(x.shape)
    ref = np.stack([mo.wrap(x[c], cell) for c in range(C_)]) if pbc else x
    assert np.abs(c32 - ref.astype(np.float32)).max() <= 4e-6
    assert opt.step == 3 and not opt.converged.any()


def test_fire_launches_are_bitwise_reproducible():
    """The same state and forces give the same bits: the FIRE launches of one step, twice from a saved state."""
    opt = make("randbatch_ani2x", steps_per_replay=4)
    opt.run(0.0, 6)
    saved = opt._buf.clone()
    outs = []
    for _ in range(2):
        opt._buf.copy_(saved)
        opt._integrate()
        torch.cuda.synchronize()
        outs.append((opt._buf.clone().view(torch.int64), opt.ws.coords.clone().view(torch.int32)))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert not torch.equal(outs[0][0], saved.view(torch.int64))


# ------------------------------------------------------------------------------------------------------------------
# 2. the device loop against a host loop
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["water30_pbc_ani2x", "small264_nopbc_ani2x"])
def test_device_loop_vs_host_loop(name):
    """TRAJ_STEPS steps on the device against Engine.step + oracle steps on the same float32 coordinates (TRAJ_BAR)."""
    opt = make(name, steps_per_replay=20)
    sp, co, cell, pbc = system(name)
    scale = np.where(sp[0] >= 0, fo.HARTREE_EV, 0.0)
    par = fo.params(0.0)
    eng = model().engine(torch.device(DEV))
    species = torch.as_tensor(sp).to(DEV)
    cell_t = None if cell is None else torch.tensor(cell, dtype=torch.float32, device=DEV)
    x, v, sc = np64(opt.x)[0], np.zeros_like(np64(opt.x)[0]), fo.init(par)
    for t in range(TRAJ_STEPS):
        xc = mo.wrap(x, cell) if pbc else x
        g = np64(eng.step(species, torch.tensor(xc[None], dtype=torch.float32, device=DEV), cell_t, pbc).grad)
        x, v, sc, _, _ = fo.step(x, v, sc, g.reshape(x.shape), scale, par, t)
    opt.run(0.0, TRAJ_STEPS)
    err = np.abs(np64(opt.x)[0] - x).max()
    assert err <= TRAJ_BAR, err


# ------------------------------------------------------------------------------------------------------------------
# 3.-5. a known minimum through the fused step; convergence; freezing
# ------------------------------------------------------------------------------------------------------------------
def test_lj13_batch_reaches_the_global_minimum():
    """64 perturbed LJ13 icosahedra (sigma 2.5 A, eps 0.5 eV, noise 0.08 sigma; the float64 oracle takes 71-118 steps
    for each) all converge to fmax 1e-3 eV / A, each at E = -44.326801 eps.  Bar 1e-4 eps: the float32 pair kernel
    rounds each of the 78 pair energies (|e| <= eps) to 2^-24 relative and the atoms' sums likewise, < 1e-5 eps in all;
    at fmax 1e-3 eV / A the distance to the minimum adds (fmax^2 / 2k) < 1e-6 eps.

    Then: a fresh energies_and_forces at the positions has max |F| < fmax (eV / A) within float32 slack; a conformer's
    positions are bitwise constant from its convergence step on while others continue; and a budget too small
    reports converged = False."""
    from torchani_b200 import optimize
    M = lj_model()
    x0 = lj13_batch(64)
    sp = np.zeros((64, 13), dtype=np.int64)
    frames = []
    opt = optimize.FIRE(M, sp, x0, steps_per_replay=10)
    done = opt.run(fmax=1e-3, steps=1000, callback=lambda step, pos, log: frames.append((step, np64(pos))))
    assert done and opt.converged.all()
    conv = opt.converged_step
    assert conv.max() < 400, conv
    e = np64(opt.energies) * mo.HARTREE_EV / LJ_EPS
    assert np.abs(e - fo.E_LJ13).max() <= 1e-4, e
    assert (opt.log.fmax[conv, np.arange(64)] < 1e-3).all()
    # a fresh force evaluation at the final positions
    spt = torch.as_tensor(sp).to(DEV)
    _, f = M.energies_and_forces(spt, opt.positions.float())
    fm = np64(f).reshape(64, 13, 3)
    assert (np.sqrt((fm ** 2).sum(-1)).max(1) * mo.HARTREE_EV < 1e-3 + 1e-5).all()
    # freezing: after its convergence step a conformer's positions are those of the end, bitwise
    final = np64(opt.positions)
    early = int(np.argmin(conv))
    assert conv[early] < conv.max() - 10
    for step, pos in frames:
        if step > conv[early]:
            assert np.array_equal(pos[early], final[early])
    moved = [s for s, pos in frames if s > conv[early] and not np.array_equal(pos[conv.argmax()],
                                                                              final[conv.argmax()])]
    assert moved, "the last conformer did not continue"
    # a budget too small
    short = optimize.FIRE(M, sp[:4], x0[:4], steps_per_replay=10)
    assert not short.run(fmax=1e-3, steps=15)
    assert not short.converged.any() and (short.converged_step == -1).all() and short.step == 15


def test_batch_vs_single_and_a_second_run():
    """A conformer's result in a batch equals its result alone (TRAJ_BAR), and a second run with a smaller fmax
    continues from the first's FIRE state."""
    from torchani_b200 import optimize
    M = lj_model()
    x0 = lj13_batch(4, seed=7)
    sp = np.zeros((4, 13), dtype=np.int64)
    batch = optimize.FIRE(M, sp, x0, steps_per_replay=10)
    batch.run(fmax=0.0, steps=TRAJ_STEPS)
    for c in range(4):
        one = optimize.FIRE(M, sp[c], x0[c], steps_per_replay=10)
        one.run(fmax=0.0, steps=TRAJ_STEPS)
        assert np.abs(np64(batch.positions)[c] - np64(one.positions)[0]).max() <= TRAJ_BAR
    # 0.05 then 1e-3: the second run goes on from v, dt, a, n of the first (the record's steps continue)
    opt = optimize.FIRE(M, sp, x0, steps_per_replay=10)
    assert opt.run(fmax=0.05, steps=500)
    s1 = opt.step
    dt_a_n = np64(opt._scalars[s1 % 2])
    assert (dt_a_n[:, 2] > 0).any()   # some conformer had a run of downhill steps
    assert opt.run(fmax=1e-3, steps=500)
    assert opt.log.step[0] == 0 and opt.log.step[-1] == opt.step - 1 and (opt.converged_step >= s1).all()


# ------------------------------------------------------------------------------------------------------------------
# 6. fixed atoms; replay shapes
# ------------------------------------------------------------------------------------------------------------------
def test_fixed_atoms_do_not_move():
    sp, co, cell, pbc = system("small264_nopbc_ani2x")
    fixed = np.zeros(sp.shape[1], dtype=bool)
    fixed[::3] = True
    opt = make("small264_nopbc_ani2x", fixed=fixed, steps_per_replay=7)
    x0 = np64(opt.x)
    opt.run(0.0, 30)
    x = np64(opt.x)
    assert np.array_equal(x[0, fixed], x0[0, fixed])
    assert np.abs(x[0, ~fixed] - x0[0, ~fixed]).max() > 1e-3
    assert (np64(opt.v)[0, fixed] == 0).all()
    # fmax of the next step is that of the movable atoms at the current positions
    f = np64(opt.forces)[0] * fo.HARTREE_EV
    opt.run(0.0, 1)
    assert opt.log.fmax[-1, 0] == pytest.approx(np.sqrt((f[~fixed] ** 2).sum(-1)).max(), rel=1e-12)


def test_replay_shapes_agree():
    """TRAJ_STEPS = 30 steps as replays of 1, of 7 (+ a remainder of 2) and of 20 (+ 10): the same launches, so the
    same result up to the force step's atomics (TRAJ_BAR)."""
    runs = []
    for K in (1, 7, 20):
        opt = make("randbatch_ani2x", steps_per_replay=K)
        opt.run(0.0, TRAJ_STEPS)
        runs.append((np64(opt.x), opt.log))
    for x, log in runs[1:]:
        assert np.abs(x - runs[0][0]).max() <= TRAJ_BAR
        assert np.array_equal(log.step, np.arange(TRAJ_STEPS))
        assert np.abs(log.energy - runs[0][1].energy).max() <= 1e-4


# ------------------------------------------------------------------------------------------------------------------
# 7. periodic input
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("per_conf", [False, True])
def test_periodic_batch(per_conf):
    from torchani_b200 import optimize
    sp, co, cell, pbc = system("water30_pbc_ani2x")
    cells = np.stack([cell, cell * 1.02]) if per_conf else cell
    sp2, co2 = np.repeat(sp, 2, 0), np.repeat(co, 2, 0)
    co2[1] += cell[0] - cell[2]   # a lattice shift: the same system, unwrapped elsewhere
    opt = optimize.FIRE(model(), sp2, co2, cell=cells, pbc=True, steps_per_replay=10)
    assert opt.per_conf == per_conf
    e0 = np64(opt.energies)
    opt.run(0.0, TRAJ_STEPS)
    x = np64(opt.x)
    c = np64(opt.ws.coords).reshape(2, -1, 3)
    cs = cells if per_conf else np.stack([cell, cell])
    for k in range(2):
        assert np.abs(c[k] - mo.wrap(x[k], cs[k]).astype(np.float32)).max() <= 4e-6
    if not per_conf:   # the shifted copy stays unwrapped: the same trajectory, one lattice vector apart
        assert np.abs(x[1] - (cell[0] - cell[2]) - x[0]).max() <= TRAJ_BAR
    assert (opt.log.energy[-1] < e0).all()


# ------------------------------------------------------------------------------------------------------------------
# 8. operand-range fallback
# ------------------------------------------------------------------------------------------------------------------
def test_operand_range_fallback_matches_a_bf16x3_loop():
    """A hydrogen with 48 neighbours 0.8 A away exceeds the 2 x fp16 operand range: the optimiser built on that build
    switches to 3 x bfloat16 at its first force step and restores its state; it then runs what an optimiser built on
    3 x bfloat16 from the start runs (TRAJ_BAR)."""
    from torchani_b200 import _lib, optimize
    from test_gpu_operand_range import cap_system
    if not _lib.available("bf16x3"):
        pytest.skip("the 3 x bfloat16 build is missing")
    s = cap_system(48)
    sp, co = s.species.numpy(), s.coords.double().numpy()
    runs = []
    for variant in ("", "bf16x3"):
        mdl = _model()
        if variant:
            mdl.neural_networks.use_variant("bf16x3")
        ctx = pytest.warns(UserWarning, match="bfloat16") if not variant else _nothing()
        with ctx:
            opt = optimize.FIRE(mdl, sp, co, maxstep=0.01, steps_per_replay=5)
            opt.run(0.0, 12)
        assert mdl.neural_networks._variant == "bf16x3"
        runs.append((np64(opt.x), opt.log))
    assert np.abs(runs[0][0] - runs[1][0]).max() <= TRAJ_BAR
    assert np.abs(runs[0][1].energy - runs[1][1].energy).max() <= 1e-5


class _nothing:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


# ------------------------------------------------------------------------------------------------------------------
# 9. rejections and launches
# ------------------------------------------------------------------------------------------------------------------
def test_rejections():
    from torchani_b200 import models, optimize, potentials
    sp, co, cell, pbc = system("water30_pbc_ani2x")
    M = model()
    with pytest.raises(ValueError, match="partial PBC"):
        optimize.FIRE(M, sp, co, cell=cell, pbc=[True, True, False])
    with pytest.raises(ValueError, match="cell"):
        optimize.FIRE(M, sp, co, pbc=True)
    with pytest.raises(ValueError, match="fixed"):
        optimize.FIRE(M, sp, co, cell=cell, pbc=True, fixed=np.zeros(5, dtype=bool))
    with pytest.raises(ValueError, match="fixed"):
        optimize.FIRE(M, sp, co, cell=cell, pbc=True, fixed=np.zeros(sp.shape[1]))
    opt = optimize.FIRE(M, sp, co, cell=cell, pbc=True)
    with pytest.raises(ValueError, match="steps"):
        opt.run(0.05, -1)
    with pytest.raises(ValueError, match="fmax"):
        opt.run(-0.05, 10)
    eng = M.engine(torch.device(DEV))
    eng.skin = 1.0
    try:
        with pytest.raises(ValueError, match="Verlet-skin"):
            optimize.FIRE(M, sp, co, cell=cell, pbc=True)
    finally:
        eng.skin = 0.0
    ws = eng.workspace(1, sp.shape[1])
    ws.reducer = object()
    try:
        with pytest.raises(ValueError, match="sharded"):
            optimize.FIRE(M, sp, co, cell=cell, pbc=True)
    finally:
        ws.reducer = None
    base = models.ANI2x(seed=0)
    lj = models.ANI(base.symbols, base.aev_computer, base.neural_networks, base.energy_shifter, False,
                    {"lj": potentials.LennardJones(base.symbols)}).to(DEV)
    with pytest.raises(ValueError, match="infinite cutoff"):
        optimize.FIRE(lj, sp, co, cell=cell, pbc=True)


def test_launches_unchanged_after_an_optimisation():
    from torchani_b200 import md
    from torchani_b200.calculator import HostCalculator
    sp, co, cell, pbc = system("water30_pbc_ani2x")
    eng = model().engine(torch.device(DEV))
    args = (torch.as_tensor(sp).to(DEV), torch.tensor(co, dtype=torch.float32, device=DEV),
            torch.tensor(cell, dtype=torch.float32, device=DEV), True)
    m = np.where(sp >= 0, 1.008, 0.0)

    def md_run():
        dyn = md.VelocityVerlet(model(), sp, co, m, cell=cell, pbc=True, steps_per_replay=5, record_every=0)
        dyn.run(10)
        return dyn.thermo.potential, eng.launches_per_step

    r0 = eng.step(*args)
    before, e0 = eng.launches_per_step, float(r0.energies[0])
    calc = HostCalculator(model(), sp, cell=cell, pbc=True)
    h0 = calc.calculate(co)
    md0, md_launches0 = md_run()
    opt = make("water30_pbc_ani2x", steps_per_replay=10)
    opt.run(0.05, 20)
    r1 = eng.step(*args)
    assert eng.launches_per_step == before
    assert float(r1.energies[0]) == pytest.approx(e0, abs=1e-6)
    md1, md_launches1 = md_run()
    assert md_launches1 == md_launches0
    assert np.abs(md1 - md0).max() <= 1e-5
    h1 = calc.calculate(co)
    for a, b in zip(h0, h1):
        assert np.abs(np.asarray(a, dtype=np.float64) - np.asarray(b, dtype=np.float64)).max() <= 1e-5
