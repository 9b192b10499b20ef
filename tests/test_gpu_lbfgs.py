"""The device L-BFGS loop (csrc/lbfgs.cu, torchani_b200/optimize.py) on the H100: three steps and a wrapped ring
against the float64 oracle (ASE's two-loop recursion), bitwise reproducible launches, the device loop against a host
loop, a known minimum (LJ13) through the fused step, freezing and fixed atoms, replay shapes, periodic batches and a
second run, the operand-range fallback, the rejected inputs and the launches of the other loops.

The bars, and where they come from:
* a few steps: L-BFGS is float64 and the forces are inputs, so x, the record and k agree with the oracle to float64
  rounding (1e-12 relative); the device's compact form and the oracle's two-loop recursion differ by less (the CPU
  tests bound their spread by 1e-12 on random histories);
* longer runs: the L-BFGS launches are bitwise reproducible, the force step is not (the AEV backward adds float32
  contributions with atomics), and a difference in the last bits of a force then grows along the optimisation.
  TRAJ_BAR is sized from two device runs of the same input on the H100 (see its comment).
"""
import numpy as np
import pytest
import torch

import oracle.fire_oracle as fo
import oracle.lbfgs_oracle as lo
import oracle.md_oracle as mo
from test_gpu_optimize import LJ_EPS, LJ_SIGMA, _model, _nothing, lj13_batch, lj_model, model, np64, system

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
# three device runs of the same input were measured on an H100 (the largest difference from the first run): after
# TRAJ_STEPS = 10 steps 1.0e-6 A on small264_nopbc_ani2x and 3.9e-6 A on water30_pbc_ani2x, after 20 steps 3.2e-6 A on
# small264_nopbc_ani2x.  L-BFGS carries such differences forward faster than FIRE: water30_pbc_ani2x was 1.2e-4 A apart
# after 15 steps and 1.9e-3 A after 20, and randbatch_ani2x (atoms far from any minimum, every step clamped) 4.8e-4 A
# after 10.  So trajectory comparisons run TRAJ_STEPS steps on water30 and 20 on small264, and the bar leaves a factor
# of 10 over the measured spread.
TRAJ_STEPS = 10
TRAJ_BAR = 4e-5
# the operand-range system (a hydrogen with 48 neighbours 0.8 A away) after 12 steps of maxstep 0.01 A: an optimiser
# switched to 3 x bfloat16 and one built on it were measured 6.3e-5 A apart on an H100; the bar leaves a factor of 16
FALLBACK_BAR = 1e-3


def make(name, **kw):
    from torchani_b200 import optimize
    sp, co, cell, pbc = system(name)
    return optimize.LBFGS(model(), sp, co, cell=cell, pbc=pbc, **kw)


def _oracle_steps(opt, name, steps, memory, maxstep, check_history=False):
    """``steps`` single steps of the device, each against oracle steps fed the device's own gradient."""
    sp, _, cell, pbc = system(name)
    scale = np.where(sp >= 0, fo.HARTREE_EV, 0.0)
    par = lo.params(0.0, maxstep=maxstep)
    C_ = opt.n_conf
    x = np64(opt.x)
    st = [lo.State(memory) for _ in range(C_)]
    for t in range(steps):
        g = np64(opt.ws.grad).reshape(x.shape)
        e = np64(opt.ws.energies)
        fmax = np.zeros(C_)
        for c in range(C_):
            x[c], fmax[c], _ = lo.step(st[c], x[c], g[c], scale[c], par)
        assert not opt.run(fmax=0.0, steps=1)
        log = opt.log
        assert log.step[-1] == t
        assert np.array_equal(log.energy[-1], e)
        assert np.abs(log.fmax[-1] - fmax).max() <= 1e-12 * fmax.max()
        err = np.abs(np64(opt.x) - x).max()
        assert err <= 1e-12 * np.abs(x).max(), f"x step {t}: {err:.3e}"
        assert (opt.iteration == [s.iteration for s in st]).all()
        if check_history and t > 0:
            S, Y = opt._history()
            for c in range(C_):
                assert len(st[c].s) == S.shape[1]
                for j in range(S.shape[1]):
                    for got, ref in ((S[c, j], st[c].s[j]), (Y[c, j], st[c].y[j])):
                        assert np.abs(np64(got).reshape(-1) - ref).max() <= 1e-12 * max(np.abs(ref).max(), 1e-300)
    return x, cell, pbc


# ------------------------------------------------------------------------------------------------------------------
# 1.-3. steps against the oracle; the ring; reproducibility
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["water30_pbc_ani2x", "small264_nopbc_ani2x", "randbatch_ani2x"])
def test_three_steps_vs_oracle(name):
    opt = make(name, steps_per_replay=1, maxstep=0.05)
    x, cell, pbc = _oracle_steps(opt, name, 3, 100, 0.05)
    c32 = np64(opt.ws.coords).reshape(x.shape)
    ref = np.stack([mo.wrap(x[c], cell) for c in range(opt.n_conf)]) if pbc else x
    assert np.abs(c32 - ref.astype(np.float32)).max() <= 4e-6
    assert opt.step == 3 and not opt.converged.any()


def test_ring_of_three_against_the_oracle():
    """memory = 3 over eight steps: the slot order, the drop of the oldest pair and the incremental SY / YY."""
    opt = make("randbatch_ani2x", steps_per_replay=1, maxstep=0.05, memory=3)
    _oracle_steps(opt, "randbatch_ani2x", 8, 3, 0.05, check_history=True)
    assert (opt._iter[:, 1].cpu().numpy() == 7).all()   # seven pairs stored, three kept


def test_lbfgs_launches_are_bitwise_reproducible():
    """The same state and forces give the same bits: the L-BFGS launches of one step, twice from a saved state."""
    opt = make("randbatch_ani2x", steps_per_replay=4)
    opt.run(0.0, 6)
    saved = opt._buf.clone()
    outs = []
    for _ in range(2):
        opt._buf.copy_(saved)
        opt._integrate()
        torch.cuda.synchronize()
        outs.append((opt._buf.clone().view(torch.int64), opt.ws.coords.clone().view(torch.int32),
                     opt._coef.clone().view(torch.int64)))
    for a, b in zip(*outs):
        assert torch.equal(a, b)
    assert not torch.equal(outs[0][0], saved.view(torch.int64))


# ------------------------------------------------------------------------------------------------------------------
# 4. the device loop against a host loop
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["water30_pbc_ani2x", "small264_nopbc_ani2x"])
def test_device_loop_vs_host_loop(name):
    """TRAJ_STEPS steps on the device against Engine.step + oracle steps on the same float32 coordinates (TRAJ_BAR)."""
    opt = make(name, steps_per_replay=20)
    sp, co, cell, pbc = system(name)
    scale = np.where(sp[0] >= 0, fo.HARTREE_EV, 0.0)
    par = lo.params(0.0)
    eng = model().engine(torch.device(DEV))
    species = torch.as_tensor(sp).to(DEV)
    cell_t = None if cell is None else torch.tensor(cell, dtype=torch.float32, device=DEV)
    x, st = np64(opt.x)[0], lo.State()
    for t in range(TRAJ_STEPS):
        xc = mo.wrap(x, cell) if pbc else x
        g = np64(eng.step(species, torch.tensor(xc[None], dtype=torch.float32, device=DEV), cell_t, pbc).grad)
        x, _, _ = lo.step(st, x, g.reshape(x.shape), scale, par)
    opt.run(0.0, TRAJ_STEPS)
    err = np.abs(np64(opt.x)[0] - x).max()
    assert err <= TRAJ_BAR, err


# ------------------------------------------------------------------------------------------------------------------
# 5.-6. a known minimum through the fused step; freezing; fixed atoms
# ------------------------------------------------------------------------------------------------------------------
def test_lj13_batch_reaches_the_global_minimum():
    """64 perturbed LJ13 icosahedra (sigma 2.5 A, eps 0.5 eV, noise 0.08 sigma; the float64 oracle takes 26-47 steps)
    all converge to fmax 1e-3 eV / A, each at E = -44.326801 eps (bar 1e-4 eps: the float32 pair kernel's rounding,
    as for FIRE) within twice the oracle's steps for that cluster.  A conformer's positions are bitwise constant from
    its convergence step on while others continue."""
    from torchani_b200 import optimize
    M = lj_model()
    x0 = lj13_batch(64)
    sp = np.zeros((64, 13), dtype=np.int64)
    frames = []
    opt = optimize.LBFGS(M, sp, x0, steps_per_replay=10)
    done = opt.run(fmax=1e-3, steps=1000, callback=lambda step, pos, log: frames.append((step, np64(pos))))
    assert done and opt.converged.all()
    conv = opt.converged_step

    def eg(x):
        return fo.lj(x, LJ_SIGMA, LJ_EPS)
    ref = np.array([lo.run(x, eg, lo.params(1e-3), 1000)[2] for x in x0])
    assert (ref > 0).all() and (conv <= 2 * ref).all(), (conv, ref)
    e = np64(opt.energies) * mo.HARTREE_EV / LJ_EPS
    assert np.abs(e - fo.E_LJ13).max() <= 1e-4, e
    assert (opt.log.fmax[conv, np.arange(64)] < 1e-3).all()
    final = np64(opt.positions)
    early = int(np.argmin(conv))
    assert conv[early] < conv.max()
    for step, pos in frames:
        if step > conv[early]:
            assert np.array_equal(pos[early], final[early])
    # the iteration count stops with the conformer
    assert (opt.iteration == conv).all()


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
    S, Y = opt._history()
    assert (np64(S)[0][:, fixed] == 0).all() and (np64(Y)[0][:, fixed] == 0).all()
    f = np64(opt.forces)[0] * fo.HARTREE_EV
    opt.run(0.0, 1)
    assert opt.log.fmax[-1, 0] == pytest.approx(np.sqrt((f[~fixed] ** 2).sum(-1)).max(), rel=1e-12)


# ------------------------------------------------------------------------------------------------------------------
# 7.-8. replay shapes; batches and runs
# ------------------------------------------------------------------------------------------------------------------
def test_replay_shapes_agree():
    """20 steps as replays of 1, of 7 (+ a remainder of 6) and of 20: the same launches, so the same result up to the
    force step's atomics (TRAJ_BAR)."""
    runs = []
    for K in (1, 7, 20):
        opt = make("small264_nopbc_ani2x", steps_per_replay=K)
        opt.run(0.0, 20)
        runs.append((np64(opt.x), opt.log))
    for x, log in runs[1:]:
        assert np.abs(x - runs[0][0]).max() <= TRAJ_BAR
        assert np.array_equal(log.step, np.arange(20))
        assert np.abs(log.energy - runs[0][1].energy).max() <= 1e-4


@pytest.mark.parametrize("per_conf", [False, True])
def test_periodic_batch_matches_single_runs(per_conf):
    from torchani_b200 import optimize
    sp, co, cell, pbc = system("water30_pbc_ani2x")
    cells = np.stack([cell, cell * 1.02]) if per_conf else cell
    sp2, co2 = np.repeat(sp, 2, 0), np.repeat(co, 2, 0)
    co2[1] += 0.05 * np.sin(np.arange(co2[1].size)).reshape(co2[1].shape)
    opt = optimize.LBFGS(model(), sp2, co2, cell=cells, pbc=True, steps_per_replay=10)
    assert opt.per_conf == per_conf
    e0 = np64(opt.energies)
    opt.run(0.0, TRAJ_STEPS)
    x = np64(opt.x)
    c = np64(opt.ws.coords).reshape(2, -1, 3)
    cs = cells if per_conf else np.stack([cell, cell])
    for k in range(2):
        assert np.abs(c[k] - mo.wrap(x[k], cs[k]).astype(np.float32)).max() <= 4e-6
        one = optimize.LBFGS(model(), sp, co2[k], cell=cs[k], pbc=True, steps_per_replay=10)
        one.run(0.0, TRAJ_STEPS)
        assert np.abs(np64(one.x)[0] - x[k]).max() <= TRAJ_BAR
    assert (opt.log.energy[-1] < e0).all()


def test_a_second_run_continues_the_history():
    """0.05 then 1e-3 eV / A: the second run keeps k and the pairs of the first (the record's steps continue), and
    reaches the end as one run with the same budget does."""
    from torchani_b200 import optimize
    M = lj_model()
    x0 = lj13_batch(4, seed=7)
    sp = np.zeros((4, 13), dtype=np.int64)
    opt = optimize.LBFGS(M, sp, x0, steps_per_replay=10)
    assert opt.run(fmax=0.05, steps=500)
    s1, k1 = opt.step, opt.iteration.copy()
    assert (k1 == opt.converged_step).all()
    assert opt.run(fmax=1e-3, steps=500)
    assert opt.log.step[0] == 0 and opt.log.step[-1] == opt.step - 1 and (opt.converged_step >= s1).all()
    assert (opt.iteration > k1).all()
    e = np64(opt.energies) * mo.HARTREE_EV / LJ_EPS
    assert np.abs(e - fo.E_LJ13).max() <= 1e-4


# ------------------------------------------------------------------------------------------------------------------
# 9. operand-range fallback
# ------------------------------------------------------------------------------------------------------------------
def test_operand_range_fallback_matches_a_bf16x3_loop():
    """The optimiser built on the 2 x fp16 build switches to 3 x bfloat16 at its first force step and restores its
    state (the history included); it then runs what an optimiser built on 3 x bfloat16 from the start runs
    (FALLBACK_BAR)."""
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
            opt = optimize.LBFGS(mdl, sp, co, maxstep=0.01, steps_per_replay=5)
            opt.run(0.0, 12)
        assert mdl.neural_networks._variant == "bf16x3"
        runs.append((np64(opt.x), opt.log, opt.iteration))
    assert np.abs(runs[0][0] - runs[1][0]).max() <= FALLBACK_BAR
    assert np.abs(runs[0][1].energy - runs[1][1].energy).max() <= 1e-3
    assert (runs[0][2] == 12).all() and (runs[1][2] == 12).all()


# ------------------------------------------------------------------------------------------------------------------
# 10.-11. rejections and launches
# ------------------------------------------------------------------------------------------------------------------
def test_rejections():
    from torchani_b200 import optimize
    sp, co, cell, pbc = system("water30_pbc_ani2x")
    M = model()
    with pytest.raises(ValueError, match="partial PBC"):
        optimize.LBFGS(M, sp, co, cell=cell, pbc=[True, True, False])
    with pytest.raises(ValueError, match="cell"):
        optimize.LBFGS(M, sp, co, pbc=True)
    with pytest.raises(ValueError, match="fixed"):
        optimize.LBFGS(M, sp, co, cell=cell, pbc=True, fixed=np.zeros(5, dtype=bool))
    for kw in (dict(memory=0), dict(memory=129), dict(alpha=-1.0), dict(damping=0.0), dict(maxstep=float("nan"))):
        with pytest.raises(ValueError):
            optimize.LBFGS(M, sp, co, cell=cell, pbc=True, **kw)
    opt = optimize.LBFGS(M, sp, co, cell=cell, pbc=True, memory=128)
    with pytest.raises(ValueError, match="steps"):
        opt.run(0.05, -1)
    with pytest.raises(ValueError, match="fmax"):
        opt.run(-0.05, 10)
    opt.run(0.0, 3)   # the largest memory: R of 128 x 128 doubles in shared memory
    eng = M.engine(torch.device(DEV))
    eng.skin = 1.0
    try:
        with pytest.raises(ValueError, match="Verlet-skin"):
            optimize.LBFGS(M, sp, co, cell=cell, pbc=True)
    finally:
        eng.skin = 0.0


def test_launches_unchanged_after_an_lbfgs_run():
    from torchani_b200 import md, optimize
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

    def fire_run():
        opt = optimize.FIRE(model(), sp, co, cell=cell, pbc=True, steps_per_replay=5)
        opt.run(0.0, 10)
        return np64(opt.x)

    r0 = eng.step(*args)
    before, e0 = eng.launches_per_step, float(r0.energies[0])
    calc = HostCalculator(model(), sp, cell=cell, pbc=True)
    h0 = calc.calculate(co)
    md0, md_launches0 = md_run()
    f0 = fire_run()
    opt = make("water30_pbc_ani2x", steps_per_replay=10)
    opt.run(0.05, 20)
    r1 = eng.step(*args)
    assert eng.launches_per_step == before
    assert float(r1.energies[0]) == pytest.approx(e0, abs=1e-6)
    md1, md_launches1 = md_run()
    assert md_launches1 == md_launches0
    assert np.abs(md1 - md0).max() <= 1e-5
    assert np.abs(fire_run() - f0).max() <= 1e-5
    h1 = calc.calculate(co)
    for a, b in zip(h0, h1):
        assert np.abs(np.asarray(a, dtype=np.float64) - np.asarray(b, dtype=np.float64)).max() <= 1e-5
