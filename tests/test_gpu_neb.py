"""The device NEB (csrc/neb.cu, torchani_b200/optimize.py NEB) on the H100: the projection and three steps against the
float64 oracle (ASE's per-image loop, fed the device's own forces), bitwise reproducible launches, the LJ3 saddle
through the fused step, what never moves, continuation and replay shapes, the rejections and the launches of the other
loops.

The bars: the NEB launches are float64 and the forces are inputs, so the NEB forces, x, v and the records agree with
the oracle to float64 rounding (1e-12 relative).  Runs longer than a few steps differ in the last bits of the force
step (its atomics); they are compared by energies against bars in eps, as the FIRE tests do.
"""
import numpy as np
import pytest
import torch

import oracle.fire_oracle as fo
import oracle.md_oracle as mo
import oracle.neb_oracle as no
from test_gpu_optimize import LJ_EPS, LJ_SIGMA, lj_model, model, np64, system

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def band_of(name, n, seed=0, amp=0.05):
    """n images of a golden system: the system, a displaced copy, and interior images on the line between them with
    noise of ``amp`` A, so that every image has its own energy and tangents of every direction."""
    sp, co, cell, pbc = system(name)
    rng = np.random.default_rng(seed)
    end = co + 0.3 * rng.standard_normal(co.shape) * (sp >= 0)[..., None]
    s = np.linspace(0.0, 1.0, n).reshape(1, n, 1, 1)
    x = co[:, None] + s * (end - co)[:, None]
    x[:, 1:-1] += amp * rng.standard_normal(x[:, 1:-1].shape) * (sp >= 0)[:, None, :, None]
    return sp, x, cell, pbc


def make(name, n=5, **kw):
    from torchani_b200 import optimize
    sp, x, cell, pbc = band_of(name, n)
    return optimize.NEB(model(), sp, x, cell=cell, pbc=pbc, **kw), sp


def oracle_forces(neb, sp, fixed=None):
    """The oracle's NEB forces (B, n - 2, A, 3) of every band from the device's positions, energies and forces."""
    x, E = np64(neb.positions), np64(neb.energies)
    F = np64(neb.forces) * mo.HARTREE_EV
    k = np64(neb.springs)
    out = []
    for b in range(neb.n_bands):
        scale = ((sp[b] >= 0) & (True if fixed is None else ~fixed[b])).astype(np.float64)
        out.append(no.get_forces(x[b], E[b], F[b] * scale[None, :, None], k[b], neb.method, neb.climb, scale))
    return np.stack(out)


@pytest.mark.parametrize("method", no.METHODS)
@pytest.mark.parametrize("climb", [False, True])
@pytest.mark.parametrize("name", ["small264_nopbc_ani2x", "randbatch_ani2x"])
def test_projection_vs_oracle(name, method, climb):
    """Fixed atoms, padding and per-spring k (given as one (n - 1,) row for every band).  An exactly zero tangent is
    covered by the CPU tests of the two forms: here the float32 energies of two equal images need not be equal, and
    t+ = -t- with alpha close to beta is where the five-dot form loses precision (DESIGN §4.15)."""
    from torchani_b200 import optimize
    sp, x, cell, pbc = band_of(name, 7)
    sp = sp[:3]
    x = x[:3]
    fixed = np.zeros(sp.shape, dtype=bool)
    fixed[:, ::5] = True
    x[:, :, fixed[0]] = x[:, :1, fixed[0]]
    neb = optimize.NEB(model(), sp, x, cell=cell, pbc=pbc, fixed=fixed, k=np.linspace(0.05, 0.3, 6), climb=climb,
                       method=method)
    got = np64(neb.neb_forces)
    ref = oracle_forces(neb, sp, fixed)
    assert np.abs(got - ref).max() <= 1e-12 * np.abs(ref).max()
    neb.climb = not climb   # the public attribute reaches the device
    got = np64(neb.neb_forces)
    ref = oracle_forces(neb, sp, fixed)
    assert np.abs(got - ref).max() <= 1e-12 * np.abs(ref).max()
    neb.climb = climb
    assert (got[:, :, fixed[0]] == 0).all()
    assert (got[np.broadcast_to((sp < 0)[:, None], got.shape[:3])] == 0).all()
    branches = set()
    E = np64(neb.energies)
    for b in range(len(sp)):
        no.get_forces_dots(np64(neb.positions)[b], E[b], np64(neb.forces)[b], 0.1, method, climb, None, branches)
    if name == "randbatch_ani2x":   # (the one band of small264 rises through every image)
        assert branches & {"up", "down"} and branches & {"max", "min"}, branches


@pytest.mark.parametrize("method", no.METHODS)
@pytest.mark.parametrize("name", ["small264_nopbc_ani2x", "water30_pbc_ani2x", "randbatch_ani2x"])
def test_three_steps_vs_oracle(name, method):
    neb, sp = make(name, n=5, method=method, climb=True, steps_per_replay=1, maxstep=0.05)
    B, m, A = neb.n_bands, 3, sp.shape[1]
    par = fo.params(0.0, maxstep=0.05)
    x, v = np64(neb.positions), np.zeros((B, m, A, 3))
    sc = [fo.init(par) for _ in range(B)]
    k = np64(neb.springs)
    for t in range(3):
        E, F = np64(neb.energies), np64(neb.forces) * mo.HARTREE_EV
        fmax, imax = np.zeros(B), np.zeros(B, dtype=np.int64)
        for b in range(B):
            scale = (sp[b] >= 0).astype(np.float64)
            x[b], v[b], sc[b], fmax[b], _, imax[b] = no.step(x[b], v[b], sc[b], E[b], F[b] * scale[None, :, None], k[b],
                                                             par, t, method, True, scale)
        assert not neb.run(fmax=0.0, steps=1)
        log = neb.log
        assert log.step[-1] == t and np.array_equal(log.imax[-1], imax)
        assert np.abs(log.fmax[-1] - fmax).max() <= 1e-12 * fmax.max()
        assert np.array_equal(log.emax[-1], E[np.arange(B), imax])
        for got, ref, what in ((np64(neb.positions), x, "x"), (np64(neb.v).reshape(v.shape), v, "v")):
            assert np.abs(got - ref).max() <= 1e-12 * max(np.abs(ref).max(), 1e-300), (what, t)
    c32 = np64(neb.ws.coords).reshape(B, m, A, 3)
    cell = neb._cell32.double().cpu().numpy() if neb.pbc else None
    ref = np.stack([[mo.wrap(x[b, i], cell) for i in range(1, m + 1)] for b in range(B)]) if neb.pbc else x[:, 1:-1]
    assert np.abs(c32 - ref.astype(np.float32)).max() <= 4e-6


def test_neb_launches_are_bitwise_reproducible():
    neb, _ = make("randbatch_ani2x", n=6, climb=True, steps_per_replay=4)
    neb.run(0.0, 6)
    saved = neb._buf.clone()
    outs = []
    for _ in range(2):
        neb._buf.copy_(saved)
        neb._integrate()
        torch.cuda.synchronize()
        outs.append((neb._buf.clone().view(torch.int64), neb.ws.coords.clone().view(torch.int32),
                     neb._neb_force.clone().view(torch.int64)))
    for a, b in zip(*outs):
        assert torch.equal(a, b)
    assert not torch.equal(outs[0][0], saved.view(torch.int64))


def lj3_bands(n_bands, n_images, seed=11):
    """Bands of LJ3 in the z = 0 plane: atom 1 crosses the 0-2 axis to its mirror image; every band randomly rotated
    about z and shifted."""
    r0 = 2.0 ** (1.0 / 6.0) * LJ_SIGMA
    a = np.array([[0.0, 0.0, 0.0], [0.5 * r0, 0.8660254 * r0, 0.0], [r0, 0.0, 0.0]])
    b = a.copy()
    b[1, 1] *= -1.0
    x = a[None] + np.linspace(0.0, 1.0, n_images)[:, None, None] * (b - a)[None]
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n_bands):
        th = rng.uniform(0, 2 * np.pi)
        R = np.array([[np.cos(th), -np.sin(th), 0.0], [np.sin(th), np.cos(th), 0.0], [0.0, 0.0, 1.0]])
        out.append(x @ R.T + np.array([rng.uniform(-3, 3), rng.uniform(-3, 3), 0.0]))
    return np.stack(out)


def test_lj3_climbing_images_reach_the_saddle():
    """64 bands of 6 interior images: every climbing image reaches E* within 1e-4 eps, collinear with equal bonds."""
    from torchani_b200 import optimize
    es, rs = no.lj3_saddle(LJ_SIGMA, 1.0)
    x = lj3_bands(64, 8)
    neb = optimize.NEB(lj_model(), np.zeros((64, 3), dtype=np.int64), x, climb=False, steps_per_replay=10)
    assert neb.run(fmax=0.05, steps=2000)
    neb.climb = True
    assert neb.run(fmax=2e-4, steps=20000)
    pos = np64(neb.positions)
    e = np64(neb.energies) * mo.HARTREE_EV / LJ_EPS
    for b in range(64):
        i = neb.imax[b]
        assert abs(e[b, i] - es) <= 1e-4, (b, e[b, i], es)
        p = pos[b, i]
        d01, d12, d02 = (np.linalg.norm(p[1] - p[0]), np.linalg.norm(p[2] - p[1]), np.linalg.norm(p[2] - p[0]))
        assert abs(d01 - d12) <= 1e-3 * LJ_SIGMA and abs(d02 - d01 - d12) <= 1e-4 * LJ_SIGMA
    assert np.abs(neb.barrier - (e[np.arange(64), neb.imax] - e[:, 0]) * LJ_EPS / mo.HARTREE_EV).max() < 1e-12


def test_what_never_moves():
    """Fixed atoms and endpoints stay bitwise constant; a converged band stays bitwise constant while others run.
    Band 0 is the straight LJ3 band, bands 1-3 have their interior images displaced by 0.3 sigma in the plane, so band 0
    converges first (the float64 oracle: step 56 against about 100 at fmax 0.02 eV / A)."""
    from torchani_b200 import optimize
    x = lj3_bands(4, 7)
    rng = np.random.default_rng(1)
    x[1:, 1:-1, 1:, :2] += 0.3 * LJ_SIGMA * rng.standard_normal((3, 5, 2, 2))
    fixed = np.array([True, False, False])
    neb = optimize.NEB(lj_model(), np.zeros((4, 3), dtype=np.int64), x, fixed=fixed, steps_per_replay=2)
    p0 = np64(neb.positions)
    frames = []
    neb.run(fmax=0.02, steps=400, callback=lambda step, pos, log: frames.append((step, np64(pos))))
    p = np64(neb.positions)
    assert np.array_equal(p[:, :, 0], p0[:, :, 0])
    assert np.array_equal(p[:, [0, -1]], p0[:, [0, -1]])
    assert np.abs(p - p0).max() > 1e-3
    conv = neb.converged_step
    assert conv[0] >= 0 and conv[0] + 10 < np.where(conv[1:] >= 0, conv[1:], 1 << 30).min(), conv
    later = [pos for step, pos in frames if step > conv[0] + 1]
    assert len(later) >= 5
    for pos in later:
        assert np.array_equal(pos[0], p[0])


def test_continuation_and_replay_shapes():
    """20 steps as replays of 1, of 7 (+ an eager remainder of 6) and of 20 agree; a second run continues the step
    count and FIRE's state after ``climb`` is switched on."""
    from torchani_b200 import optimize
    x = lj3_bands(3, 6, seed=3)
    runs = []
    for K in (1, 7, 20):
        neb = optimize.NEB(lj_model(), np.zeros((3, 3), dtype=np.int64), x, steps_per_replay=K)
        neb.run(0.0, 20)
        runs.append((np64(neb.positions), neb.log))
    for p, log in runs[1:]:
        assert np.abs(p - runs[0][0]).max() <= 1e-5
        assert np.array_equal(log.step, np.arange(20))
    neb = optimize.NEB(lj_model(), np.zeros((3, 3), dtype=np.int64), x, steps_per_replay=7)
    neb.run(0.0, 10)
    sc = np64(neb._scalars[10 % 2])
    neb.climb = True
    neb.run(0.0, 3)
    assert np.array_equal(neb.log.step, np.arange(13)) and neb.step == 13
    assert np.abs(np64(neb._scalars[13 % 2]) - sc).max() > 0   # the scalars went on from step 10, not from dt0
    assert not np.allclose(np64(neb._scalars[13 % 2])[:, 0], 0.1)


def test_rejections():
    from torchani_b200 import optimize
    sp, x, cell, pbc = band_of("small264_nopbc_ani2x", 5)
    M = model()
    bad = [dict(images=x[:, :2]), dict(method="eb"), dict(method="spline"), dict(method="string"),
           dict(remove_rotation_and_translation=True), dict(precon="Exp"), dict(k=0.0), dict(k=float("nan")),
           dict(k=np.ones(3)), dict(dt=-1.0), dict(fdec=2.0)]
    for kw in bad:
        args = dict(images=x)
        args.update(kw)
        with pytest.raises(ValueError):
            optimize.NEB(M, sp, **args)
    fixed = np.zeros(sp.shape[1], dtype=bool)
    fixed[0] = True
    with pytest.raises(ValueError, match="fixed"):
        optimize.NEB(M, sp, x, fixed=fixed)
    with pytest.raises(ValueError, match="65535"):
        optimize.NEB(M, np.zeros((1, 1), dtype=np.int64), np.zeros((65536, 3, 1, 3)))
    sp2, x2, cell2, _ = band_of("water30_pbc_ani2x", 5)
    with pytest.raises(ValueError, match="partial PBC"):
        optimize.NEB(M, sp2, x2, cell=cell2, pbc=[True, True, False])


def kernel_launches(fn):
    """The kernels ``fn`` launches, counted by torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "emcpy" not in e.name
               and "emset" not in e.name)


def test_launches_and_other_loops_unchanged():
    """A step is the force step's launches + 3; afterwards MD, FIRE, CellFIRE and L-BFGS issue the launches they issued
    before and compute what they computed."""
    from torchani_b200 import md, optimize
    sp, co, cell, pbc = system("water30_pbc_ani2x")
    eng = model().engine(torch.device(DEV))
    m = np.where(sp >= 0, 1.008, 0.0)

    def step_of(loop):
        return kernel_launches(lambda: (loop._integrate(), loop._force_step())), kernel_launches(loop._force_step)

    def others():
        dyn = md.VelocityVerlet(model(), sp, co, m, cell=cell, pbc=True, steps_per_replay=5, record_every=0)
        dyn.run(10)
        f = optimize.FIRE(model(), sp, co, cell=cell, pbc=True, steps_per_replay=5)
        f.run(0.0, 10)
        cf = optimize.CellFIRE(model(), sp, co, cell, steps_per_replay=5)
        cf.run(0.0, 5)
        lb = optimize.LBFGS(model(), sp, co, cell=cell, pbc=True, steps_per_replay=5)
        lb.run(0.0, 5)
        counts = [step_of(o) for o in (dyn, f, cf, lb)]
        return dyn.thermo.potential, np64(f.x), np64(cf.x), np64(lb.x), eng.launches_per_step, counts

    md0, f0, c0, l0, n0, k0 = others()
    neb, _ = make("water30_pbc_ani2x", n=4, steps_per_replay=5)
    neb.run(0.0, 5)
    total, force = step_of(neb)
    assert total == force + 3, (total, force)
    assert kernel_launches(neb._integrate) == 3
    md1, f1, c1, l1, n1, k1 = others()
    assert n1 == n0 and k1 == k0, (k0, k1)
    assert np.abs(md1 - md0).max() <= 1e-5
    assert np.abs(f1 - f0).max() <= 1e-5 and np.abs(c1 - c0).max() <= 1e-5 and np.abs(l1 - l0).max() <= 1e-4


# ------------------------------------------------------------------------------------------------------------------
# the device loop against a host loop; the periodic vacancy hop; the operand-range fallback
# ------------------------------------------------------------------------------------------------------------------
# three device runs of the same band (climbing, aseneb) were measured on an H100 at most 2.8e-8 A (small264_nopbc_ani2x)
# and 2.4e-8 A (water30_pbc_ani2x) apart after TRAJ_STEPS steps (the force step's atomics); TRAJ_BAR leaves a factor of
# 35 over the larger
TRAJ_STEPS = 10
TRAJ_BAR = 1e-6


@pytest.mark.parametrize("name", ["small264_nopbc_ani2x", "water30_pbc_ani2x"])
def test_device_loop_vs_host_loop(name):
    """TRAJ_STEPS steps on the device against Engine.step on the interior images (and the endpoints) plus oracle
    steps on the same float32 coordinates (TRAJ_BAR)."""
    from torchani_b200 import optimize
    sp, x, cell, pbc = band_of(name, 5)
    neb = optimize.NEB(model(), sp, x, cell=cell, pbc=pbc, climb=True, steps_per_replay=TRAJ_STEPS)
    eng = model().engine(torch.device(DEV))
    cell_t = None if cell is None else torch.tensor(cell, dtype=torch.float32, device=DEV)
    scale = (sp[0] >= 0).astype(np.float64)

    def evaluate(imgs):
        xc = np.stack([mo.wrap(y, cell) for y in imgs]) if pbc else imgs
        r = eng.step(torch.as_tensor(np.repeat(sp, len(imgs), 0)).to(DEV),
                     torch.tensor(xc, dtype=torch.float32, device=DEV), cell_t, pbc)
        return np64(r.energies), np64(r.grad).reshape(imgs.shape)

    xs = x[0].copy()
    e_end, _ = evaluate(xs[[0, -1]])
    par = fo.params(0.0)
    v, sc = np.zeros_like(xs[1:-1]), fo.init(par)
    for t in range(TRAJ_STEPS):
        e, g = evaluate(xs[1:-1])
        E = np.concatenate([e_end[:1], e, e_end[1:]])
        xs, v, sc, _, _, _ = no.step(xs, v, sc, E, -g * mo.HARTREE_EV * scale[None, :, None], 0.1, par, t, "aseneb",
                                     True, scale)
    neb.run(0.0, TRAJ_STEPS)
    assert np.abs(np64(neb.end_energies)[0] - e_end).max() <= 1e-5
    err = np.abs(np64(neb.positions)[0] - xs).max()
    assert err <= TRAJ_BAR, err


def vacancy_hop(n):
    """A vacancy hop in test_gpu_cell_optimize's fcc LJ crystal (smooth cutoff, 4 x 4 x 4 cells, site 0 empty, 255
    atoms): endpoint A relaxed with FIRE, endpoint B its mirror image through the plane between site 0 and the hopping
    atom's site (0, a/2, a/2): (x, y, z) -> (x, a/2 - z, a/2 - y), which maps the crystal onto itself.  Returns the
    linear band of n images (atom 0 hops) and the cell."""
    from test_gpu_cell_optimize import fcc, lattice_constant, lj_cut_model
    from torchani_b200 import optimize
    a = lattice_constant(0.0)
    r, h = fcc(a)
    L = h[0, 0]
    sites = r[1:]   # site 1 is (0, a/2, a/2): the hopping atom is atom 0
    opt = optimize.FIRE(lj_cut_model(), np.zeros(255, dtype=np.int64), sites, cell=h, pbc=True, steps_per_replay=20)
    assert opt.run(fmax=1e-4, steps=3000)
    xa = np64(opt.x)[0]

    def mirror(p):
        return np.stack([p[..., 0], 0.5 * a - p[..., 2], 0.5 * a - p[..., 1]], -1)
    ms = mirror(sites)
    xb = np.empty_like(xa)
    xb[0] = mirror(xa[0])
    for i in range(1, 255):
        d = sites - ms[i]
        k = int(np.argmin(np.abs(d - L * np.round(d / L)).sum(1)))
        y = mirror(xa[k])
        xb[i] = y - L * np.round((y - xa[i]) / L)
    return optimize.interpolate(xa, xb, n), h


def lj_oracle_energy_grad(cell):
    """The float64 energy and gradient (eV, eV / A) of the crystal from lj_coulomb_oracle."""
    import oracle.lj_coulomb_oracle as ljo
    from test_gpu_cell_optimize import LJ_RC
    one, zero = torch.ones(1, dtype=torch.float64), torch.zeros(1, dtype=torch.float64)
    spec = ljo.Spec("lj", LJ_RC, "smooth", one * 0.5 / mo.HARTREE_EV, one * 2.5, zero, zero)
    c = torch.as_tensor(cell)

    def eg(y):
        out = ljo.compute(spec, torch.zeros(1, len(y), dtype=torch.long), torch.tensor(y[None], dtype=torch.float64), c,
                          torch.ones(3, dtype=torch.bool), neighborlist="all_pairs")
        return float(out["energy"][0]) * mo.HARTREE_EV, -out["forces"][0].numpy() * mo.HARTREE_EV
    return eg


def test_periodic_vacancy_hop():
    """7 images (odd: the middle one on the mirror plane).  The converged band is symmetric, E_i = E_{n-1-i}; the
    climbing barrier matches the float64 oracle's, converged from the device's band; a batch of two bands with a shared
    cell and one with a cell per band (the second band a translated copy, and a 1 % larger crystal) match single-band
    runs."""
    from test_gpu_cell_optimize import lj_cut_model
    from torchani_b200 import optimize
    band, h = vacancy_hop(7)
    sp = np.zeros(255, dtype=np.int64)
    neb = optimize.NEB(lj_cut_model(), sp, band, cell=h, pbc=True, steps_per_replay=20)
    assert neb.run(fmax=0.01, steps=3000)
    neb.climb = True
    assert neb.run(fmax=1e-3, steps=5000)
    e = np64(neb.energies)[0] * mo.HARTREE_EV
    pos = np64(neb.positions)[0]
    eg = lj_oracle_energy_grad(h)
    e_ref = np.array([eg(p)[0] for p in pos])
    bar = 10 * np.abs(e - e_ref).max() + 1e-6   # the float32 spread of the device's energies
    assert np.abs(e - e[::-1]).max() <= bar, (e, bar)
    assert neb.imax[0] == 3
    xo, Eo, c = no.run(pos, eg, 0.1, fo.params(1e-3), 500, "aseneb", climb=True)
    assert c >= 0
    barrier_ref = Eo[no.imax_of(Eo)] - Eo[0]
    assert abs(neb.barrier[0] * mo.HARTREE_EV - barrier_ref) <= bar, (neb.barrier[0] * mo.HARTREE_EV, barrier_ref)
    # batches against single bands: 30 steps from the linear band
    shift = np.array([0.5, 0.5, 0.0]) * h[0, 0] / 4
    for per_band in (False, True):
        b2 = band * 1.01 if per_band else band + shift
        cells = np.stack([h, h * 1.01]) if per_band else h
        batch = optimize.NEB(lj_cut_model(), sp, np.stack([band, b2]), cell=cells, pbc=True, climb=True,
                             steps_per_replay=10)
        assert batch.per_conf == per_band
        batch.run(0.0, 30)
        for k, (bk, hk) in enumerate(((band, h), (b2, cells[1] if per_band else h))):
            one = optimize.NEB(lj_cut_model(), sp, bk, cell=hk, pbc=True, climb=True, steps_per_replay=10)
            one.run(0.0, 30)
            assert np.abs(np64(batch.end_energies)[k] - np64(one.end_energies)[0]).max() <= 1e-5
            assert np.abs(np64(batch.positions)[k] - np64(one.positions)[0]).max() <= 1e-4
            assert np.array_equal(batch.log.imax[:, k], one.log.imax[:, 0])


def test_operand_range_fallback_matches_a_bf16x3_loop():
    """A band of test_gpu_operand_range's hydrogen with 48 neighbours 0.8 A away (beyond the 2 x fp16 operand range):
    the NEB built on that build switches to 3 x bfloat16 (endpoint energies included) and then runs what a NEB built on
    3 x bfloat16 from the start runs."""
    from test_gpu_operand_range import cap_system
    from test_gpu_optimize import _model, _nothing
    from torchani_b200 import _lib, optimize
    if not _lib.available("bf16x3"):
        pytest.skip("the 3 x bfloat16 build is missing")
    s = cap_system(48)
    sp, co = s.species.numpy(), s.coords.double().numpy()
    rng = np.random.default_rng(4)
    end = co + 0.02 * rng.standard_normal(co.shape) * (sp >= 0)[..., None]
    x = co[:, None] + np.linspace(0.0, 1.0, 4).reshape(1, 4, 1, 1) * (end - co)[:, None]
    runs = []
    for variant in ("", "bf16x3"):
        mdl = _model()
        if variant:
            mdl.neural_networks.use_variant("bf16x3")
        ctx = pytest.warns(UserWarning, match="bfloat16") if not variant else _nothing()
        with ctx:
            neb = optimize.NEB(mdl, sp, x, maxstep=0.01, climb=True, steps_per_replay=5)
            neb.run(0.0, 12)
        assert mdl.neural_networks._variant == "bf16x3"
        runs.append((np64(neb.positions), np64(neb.end_energies), neb.log))
    assert np.abs(runs[0][0] - runs[1][0]).max() <= 1e-5
    assert np.abs(runs[0][1] - runs[1][1]).max() <= 1e-5
    assert np.abs(runs[0][2].emax - runs[1][2].emax).max() <= 1e-5
