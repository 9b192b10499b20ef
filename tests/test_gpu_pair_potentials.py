"""Pair potentials in the fused step (csrc/pair.cu): xTB and ZBL repulsion evaluated over the neighbour list of the AEV
forward -- the kernel on its own against float64 in grid modes 0-3 and on a diatomic scan, whole models (networks +
repulsion) on every MLP launch form and the 3 x bf16 build, additivity, shards, Verlet reuse, the query-by-committee
step, graph replay, launch counts, and the drop-in paths against the staged reference."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import oracle.ani_oracle as orc
import oracle.pair_oracle as porc
from helpers import E_ATOL, E_RTOL, F_ATOL, GOLD, ROOT, assert_close, golden_inputs, load_golden

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PBC = torch.tensor([True, True, True])
RCR = 5.1
SYSTEMS = ["water999_pbc_ani2x", "1c17_chunk_hcnos_ani2x", "randbatch_ani2x", "6w8h_triclinic_ani2x"]
# Forces: the helpers' absolute bar plus a relative term.  The synthetic boxes hold close contacts where one repulsive
# pair pushes with up to ~30 Ha/A and dF/dR ~ 1e2 Ha/A^2, and the float32 positions the kernel is given (|x| up to 30 A)
# carry 2e-6 A each: 1e-5 of the force is what float32 INPUTS allow there; everywhere else the absolute bar rules.
F_RTOL = 1e-5
_cache = {}


def pair_golden(name):
    z = np.load(os.path.join(GOLD, f"pair_{name}.npz"))
    return {k: z[k] for k in z.files}


def xtb_tables():
    z = np.load(os.path.join(GOLD, "pair_params.npz"))
    return tuple(torch.tensor(z[k]) for k in ("y_ab", "sqrt_alpha_ab", "k_rep_ab"))


def spec(kind, fn):
    return porc.PairSpec("xtb", RCR, fn, xtb_tables()) if kind == "xtb" else porc.zbl_spec(orc.SYMBOLS_2X, RCR, fn)


def potential(kind, fn, cutoff=RCR):
    from torchani_b200 import potentials as P
    if kind == "zbl":
        return P.RepulsionZBL(orc.SYMBOLS_2X, cutoff=cutoff, cutoff_fn=fn)
    pot = P.RepulsionXTB(orc.SYMBOLS_2X, alpha=[1.0] * 7, yeff=[1.0] * 7, cutoff=cutoff, cutoff_fn=fn)
    for key, t in zip(("y_ab", "sqrt_alpha_ab", "k_rep_ab"), xtb_tables()):
        getattr(pot, key).copy_(t.float())
    return pot


def oracle_weights():
    if "w" not in _cache:
        _cache["w"] = orc.make_weights(orc.SYMBOLS_2X, orc.DIMS_2X, 1008, 8, 1234, torch.float64)
    return _cache["w"]


def model(kind=None, fn="cosine", variant="", tag=""):
    """The seeded ANI-2x x 8 of the golden files, with one repulsion term (or none), on the GPU (`tag`: another
    instance with an engine of its own)."""
    from torchani_b200 import models
    key = (kind, fn, variant, tag)
    if key not in _cache:
        w32 = [{s: [(w.float(), b.float()) for w, b in layers] for s, layers in wm.items()} for wm in oracle_weights()]
        base = models.from_weight_lists("2x", w32, periodic_table_index=False)
        pots = {} if kind is None else {f"repulsion_{kind}": potential(kind, fn)}
        m = models.ANI(base.symbols, base.aev_computer, base.neural_networks, base.energy_shifter, False, pots).to(DEV)
        if variant:
            m.neural_networks.use_variant(variant)
        _cache[key] = m
    return _cache[key]


def dev(t):
    return None if t is None else t.to(DEV)


def pair_only(eng, sp, co, cell, pbc, want_virial=False, shard=(0, 1)):
    """The pair kernel on its own: preparation and AEV forward of the step (they leave the neighbour words), then the
    pair launch into zeroed outputs -- no network runs.  Returns energies, atomic, grad (, virial) as float64 numpy."""
    from torchani_b200._lib import check, ptr

    def run(name, fn):
        check(fn(), name)
    with torch.cuda.device(eng.device):
        ws, per_conf = eng._stage_inputs(dev(sp), dev(co).float(), None if cell is None else dev(cell).float(),
                                         pbc is not None)
        n = ws.n
        lo, hi = (n * shard[0]) // shard[1], (n * (shard[0] + 1)) // shard[1]
        lat = eng._prepare(ws, pbc is not None, per_conf, lo, hi, False, ws.grad_ptr, 3 * n,
                           ws.virial if want_virial else None, run)
        eng._aev_forward(ws, lo, hi, False, lat, run)
        ws.atomic.zero_(), ws.energies.zero_(), ws.member_atomic.zero_()
        eng._pair_potentials(ws, lo, hi, lat, ws.grad_ptr, ptr(ws.virial) if want_virial else None, None, run)
        torch.cuda.synchronize()
        eng.check_status(ws)
    out = {"energy": ws.energies.cpu().numpy().copy(), "atomic": ws.atomic.view(sp.shape).double().cpu().numpy(),
           "forces": -ws.grad.view(sp.shape + (3,)).double().cpu().numpy(),
           "member_atomic": ws.member_atomic.view((-1,) + sp.shape).double().cpu().numpy()}
    if want_virial:
        out["virial"] = ws.virial.view(sp.shape[0], -1, 9).sum(1).view(-1, 3, 3).cpu().numpy()
    return out


def check_pair(tag, got, ref, e_rtol=E_RTOL, f_rtol=F_RTOL, sum_rtol=1e-6):
    assert_close(f"{tag} atomic", got["atomic"], ref["atomic"], e_rtol, E_ATOL)
    assert_close(f"{tag} forces", got["forces"], ref["forces"], f_rtol, F_ATOL)
    assert_close(f"{tag} energy", got["energy"], ref["energy"], sum_rtol, 1e-5)
    for m in range(got["member_atomic"].shape[0]):      # every member gets the pair term
        assert np.array_equal(got["member_atomic"][m], got["atomic"])


# ------------------------------------------------------------------------------------------------------------------
# 1. the kernel on its own
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fn", ["cosine", "smooth"])
@pytest.mark.parametrize("kind", ["xtb", "zbl"])
@pytest.mark.parametrize("name", SYSTEMS)
def test_kernel_vs_float64_golden(name, kind, fn):
    sp, co, cell, pbc = golden_inputs(load_golden(name))
    ref = {k[len(f"{kind}_{fn}_"):]: v for k, v in pair_golden(name).items() if k.startswith(f"{kind}_{fn}_")}
    eng = model(kind, fn).engine(torch.device(DEV))
    got = pair_only(eng, sp, co, cell, pbc, want_virial=cell is not None)
    if name == "6w8h_triclinic_ani2x":
        # this box holds overlapping atoms (closest pair 0.043 A, |F| up to 1e4 Ha/A, atomic terms of 1e2 Ha) at
        # |x| up to 49 A: the float64 oracle itself moves by 1.8e-5 (atomic, relative) and 2.2e-4 (forces) when it is
        # given the coordinates rounded to float32, which is all the kernel ever sees
        check_pair(f"{name} {kind} {fn}", got, ref, e_rtol=4e-5, f_rtol=5e-4, sum_rtol=1e-5)
    else:
        check_pair(f"{name} {kind} {fn}", got, ref)
    if cell is not None:
        stress = got["virial"][0] / abs(float(torch.det(cell)))
        s_ref, s_rtol = ref["stress"], 1e-5
        frac = co @ torch.inverse(cell)
        if bool((frac.floor() != 0).any()):
            # atoms outside the cell: the "scaling" stress of the fixture wraps them with a cell that is not scaled, the
            # pair-vector virial does not depend on where the atoms sit; take the float64 value at the wrapped positions
            s_ref = porc.compute(spec(kind, fn), sp, (frac - frac.floor()) @ cell, cell, pbc, "cell_list",
                                 stress=True)["stress"].numpy()
            s_rtol = 1e-4
        assert_close(f"{name} stress", stress, s_ref, s_rtol, 1e-5 * float(np.abs(s_ref).max()))


def periodic_batch(per_conformer):
    """Three perturbed copies of the 90-atom periodic water box; with `per_conformer` every copy in a cell of its own
    (scaled, the last one sheared), the last conformer partly padding."""
    sp, co, cell, _ = golden_inputs(load_golden("water30_pbc_ani2x"))
    g = torch.Generator().manual_seed(17)
    co = co.repeat(3, 1, 1)
    co[1:] += 0.03 * torch.randn(co[1:].shape, generator=g, dtype=torch.float64)
    # (inside the cell: the float64 "scaling" stress of the oracle wraps with a detached cell)
    frac = co @ torch.inverse(cell)
    co = (frac - frac.floor()) @ cell
    sp = sp.repeat(3, 1).clone()
    sp[-1, -3:] = -1
    if not per_conformer:
        return sp, co, cell
    cells = cell.repeat(3, 1, 1).clone()
    for c, (s, shear) in enumerate([(1.0, 0.0), (1.04, 0.0), (0.98, 0.08)]):
        t = torch.eye(3, dtype=torch.float64) * s
        t[0, 1] = shear
        cells[c] = cell @ t
        co[c] = co[c] @ t
    return sp, co, cells


@pytest.mark.parametrize("kind,fn", [("xtb", "smooth"), ("zbl", "cosine")])
@pytest.mark.parametrize("per_conformer", [False, True], ids=["mode2", "mode3"])
def test_kernel_periodic_batches(per_conformer, kind, fn):
    sp, co, cell = periodic_batch(per_conformer)
    eng = model(kind, fn).engine(torch.device(DEV))
    got = pair_only(eng, sp, co, cell, PBC, want_virial=True)
    for c in range(sp.shape[0]):
        ck = cell[c] if per_conformer else cell
        ref = porc.compute(spec(kind, fn), sp[c:c + 1], co[c:c + 1], ck, PBC, "cell_list", stress=True)
        one = {k: v[c:c + 1] for k, v in got.items() if k != "member_atomic"}
        one["member_atomic"] = got["member_atomic"][:, c:c + 1]
        check_pair(f"conformer {c}", one, {k: v.numpy() for k, v in ref.items()})
        assert_close(f"conformer {c} stress", got["virial"][c] / abs(float(torch.det(ck))), ref["stress"].numpy(),
                     1e-5, 1e-8)


@pytest.mark.parametrize("fn", ["cosine", "smooth"])
@pytest.mark.parametrize("kind", ["xtb", "zbl"])
def test_diatomic_scan(kind, fn):
    z = pair_golden("scan")
    sp, co = torch.tensor(z["species"]), torch.tensor(z["coords"])
    R = z["coords"][:, 1, 0]
    eng = model(kind, fn).engine(torch.device(DEV))
    got = pair_only(eng, sp, co, None, None)
    e_ref, a_ref, f_ref = (z[f"{kind}_{fn}_{k}"] for k in ("energy", "atomic", "forces"))
    phys = R >= 0.3      # the bars of the helpers at every physical distance, across the cutoff
    assert_close("scan atomic", got["atomic"][phys], a_ref[phys], E_RTOL, E_ATOL)
    assert_close("scan forces", got["forces"][phys], f_ref[phys], 5e-6, F_ATOL)
    assert (got["energy"][R > RCR] == 0).all() and (got["forces"][R > RCR] == 0).all()
    # below that (down to the 1e-7 clamp, where the term reaches 1e7 Ha and more) the energies stay finite and relative
    assert np.isfinite(got["atomic"]).all() and np.isfinite(got["forces"]).all()
    assert_close("scan core energies", got["energy"][~phys], e_ref[~phys], 1e-4, 0.0)


# ------------------------------------------------------------------------------------------------------------------
# 2. whole models, 3. additivity
# ------------------------------------------------------------------------------------------------------------------
def golden_total(name, kind, fn):
    """float64 totals of networks + repulsion from the two fixtures of a system."""
    rec, pg = load_golden(name), pair_golden(name)
    sp = torch.tensor(rec["species"])
    sae = orc.self_energies(orc.SYMBOLS_2X, orc.GSAES_WB97X_631GD, sp, torch.float64).numpy()
    return {"energy": rec["energy_nn"] + sae.sum(-1) + pg[f"{kind}_{fn}_energy"],
            "atomic": rec["member_atomic"].mean(0) + sae + pg[f"{kind}_{fn}_atomic"],
            "forces": rec["forces"] + pg[f"{kind}_{fn}_forces"], "pair_stress": pg.get(f"{kind}_{fn}_stress")}


@pytest.mark.parametrize("launch", ["auto", "1", "0", "bf16x3"], ids=["resident", "dataflow", "chained", "bf16x3"])
@pytest.mark.parametrize("name,kind,fn", [("water999_pbc_ani2x", "xtb", "smooth"), ("randbatch_ani2x", "zbl", "cosine"),
                                          ("1c17_chunk_hcnos_ani2x", "xtb", "cosine")])
def test_whole_model_vs_golden_totals(name, kind, fn, launch):
    m = model(kind, fn, "bf16x3" if launch == "bf16x3" else "")
    eng = m.engine(torch.device(DEV))
    saved = eng.mlp_mode
    eng.mlp_mode = "auto" if launch == "bf16x3" else launch
    try:
        sp, co, cell, pbc = golden_inputs(load_golden(name), torch.float32)
        ref = golden_total(name, kind, fn)
        e, f = m.energies_and_forces(dev(sp), dev(co), dev(cell), dev(pbc))
        n_real = int((sp >= 0).sum(1).max())
        assert_close(f"{name} energies", e.cpu().numpy(), ref["energy"], 2e-7, 2e-7 * max(n_real, 10) + 1e-5)
        assert_close(f"{name} forces", f.cpu().numpy(), ref["forces"], F_RTOL, F_ATOL)
        a = m.atomic_energies((dev(sp), dev(co)), dev(cell), dev(pbc)).energies
        mask = (sp >= 0).numpy()
        assert_close(f"{name} atomic", a.cpu().numpy()[mask], ref["atomic"][mask], 2e-6, 2e-5)
        ev = m((dev(sp), dev(co)), dev(cell), dev(pbc), ensemble_values=True).energies     # (M, C)
        assert ev.shape[0] == 8 and torch.allclose(ev.double().mean(0).cpu(), torch.tensor(ref["energy"]),
                                                   rtol=0, atol=2e-2)
    finally:
        eng.mlp_mode = saved


def test_stress_and_additivity():
    """calculate_with_stress and the per-conformer virial of a periodic batch; (model with repulsion) - (model without)
    = the kernel alone."""
    from torchani_b200.calculator import HostCalculator
    kind, fn = "xtb", "smooth"
    m1, m0 = model(kind, fn), model(None)
    sp, co, cell, pbc = golden_inputs(load_golden("water999_pbc_ani2x"), torch.float32)
    e1, f1, s1 = HostCalculator(m1, sp[0].numpy(), cell.numpy(), pbc=True).calculate_with_stress(co[0].numpy())
    e0, f0, s0 = HostCalculator(m0, sp[0].numpy(), cell.numpy(), pbc=True).calculate_with_stress(co[0].numpy())
    alone = pair_only(m1.engine(torch.device(DEV)), sp, co, cell, pbc, want_virial=True)
    vol = abs(float(torch.det(cell.double())))
    assert abs((e1 - e0) - alone["energy"][0]) < 1e-6
    assert_close("additive forces", f1 - f0, alone["forces"][0], 0.0, 2e-5)     # fp32 rounding of the two sums
    assert_close("additive stress", s1 - s0, alone["virial"][0] / vol, 1e-6, 1e-9)
    assert_close("pair stress", s1 - s0, golden_total("water999_pbc_ani2x", kind, fn)["pair_stress"], 1e-4, 1e-7)
    # a periodic batch with one cell per conformer
    spb, cob, cells = periodic_batch(True)
    _, _, sb1 = m1.energies_forces_stress(dev(spb), dev(cob).float(), dev(cells).float())
    _, _, sb0 = m0.energies_forces_stress(dev(spb), dev(cob).float(), dev(cells).float())
    for c in range(3):
        ref = porc.compute(spec(kind, fn), spb[c:c + 1], cob[c:c + 1], cells[c], PBC, "cell_list", stress=True)
        assert_close(f"batch stress {c}", (sb1 - sb0)[c].cpu().numpy(), ref["stress"].numpy(), 1e-4, 1e-7)


# ------------------------------------------------------------------------------------------------------------------
# 4. shards, 5. Verlet reuse
# ------------------------------------------------------------------------------------------------------------------
def test_shards_add_up():
    m = model("xtb", "smooth")
    sp, co, cell, pbc = golden_inputs(load_golden("water999_pbc_ani2x"), torch.float32)
    eng = m.engine(torch.device(DEV))
    full = eng.step(dev(sp), dev(co), dev(cell), True, check=True)
    e, g, a = full.energies.clone(), full.grad.clone(), full.atomic_energies.clone()
    es, gs, as_ = torch.zeros_like(e), torch.zeros_like(g), torch.zeros_like(a)
    for rank in range(3):
        part = eng.step(dev(sp), dev(co), dev(cell), True, shard=(rank, 3), check=True)
        es += part.energies
        gs += part.grad
        as_ += part.atomic_energies
    assert torch.allclose(es, e, rtol=0, atol=1e-6)
    assert_close("sharded forces", gs.cpu().numpy(), g.cpu().numpy(), 1e-6, 1e-6)
    assert_close("sharded atomic", as_.cpu().numpy(), a.cpu().numpy(), 0.0, 1e-6)
    alone = [pair_only(eng, sp, co, cell, pbc, shard=(r, 3)) for r in range(3)]
    ref = pair_only(eng, sp, co, cell, pbc)
    assert_close("sharded kernel", sum(x["forces"] for x in alone), ref["forces"], 1e-6, 1e-6)
    assert abs(sum(x["energy"][0] for x in alone) - ref["energy"][0]) < 1e-8


def test_verlet_reuse_matches_fresh_grids():
    from torchani_b200.calculator import HostCalculator
    m, fresh_m = model("xtb", "smooth", tag="skin"), model("xtb", "smooth")     # engines of their own
    sp, co, cell, pbc = golden_inputs(load_golden("water999_pbc_ani2x"), torch.float32)
    eng = m.engine(torch.device(DEV))
    calc = HostCalculator(m, sp[0].numpy(), cell.numpy(), pbc=True, skin=0.4)
    try:
        g = torch.Generator().manual_seed(3)
        pos = co.clone()
        for step in range(12):
            pos = pos + 0.002 * torch.randn(pos.shape, generator=g)
            if step == 8:
                pos[0, 11] += 0.3      # beyond skin / 2: rebuilt
            e, f = calc.calculate(pos[0].numpy())
            e_ref, f_ref = fresh_m.energies_and_forces(dev(sp), dev(pos), dev(cell), dev(pbc))
            assert abs(float(e) - float(e_ref[0])) < 1e-6, step
            assert_close(f"step {step} forces", f, f_ref[0].cpu().numpy(), 0.0, 1e-5)
        assert 1 <= calc.rebuilds < 12, calc.rebuilds
    finally:
        eng.skin = 0.0


# ------------------------------------------------------------------------------------------------------------------
# 6. the query-by-committee step
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,active", [("water999_pbc_ani2x", list(range(8))), ("randbatch_ani2x", [1, 4, 6])])
def test_qbc_step_adds_the_pair_term_to_every_member(name, active):
    kind, fn = "xtb", "smooth"
    m1, m0 = model(kind, fn), model(None)
    sp, co, cell, pbc = golden_inputs(load_golden(name), torch.float32)
    rec, pg = load_golden(name), pair_golden(name)
    try:
        for mm in (m1, m0):
            mm.neural_networks.set_active_members(active)
        args = ((dev(sp), dev(co)), dev(cell), dev(pbc))
        _, e_m, f_m = m1.members_forces(*args)
        _, e_m0, f_m0 = m0.members_forces(*args)
        # every member: its own network term plus the same pair term (arch.py:365-378)
        assert_close("member pair forces", (f_m - f_m0).cpu().numpy(),
                     np.broadcast_to(pg[f"{kind}_{fn}_forces"], f_m.shape), F_RTOL, F_ATOL)
        sae = orc.self_energies(orc.SYMBOLS_2X, orc.GSAES_WB97X_631GD, sp, torch.float64).numpy().sum(-1)
        for k, mem in enumerate(active):
            e_ref = rec["member_atomic"][mem].sum(-1) + sae + pg[f"{kind}_{fn}_energy"]
            assert_close(f"member {mem} energy", e_m[k].cpu().numpy(), e_ref, 0.0, 5e-3)
        # the statistics against their restatement on the members' outputs (arch.py:439-485, 543-576)
        eng = m1.engine(torch.device(DEV))
        r = eng.members_result(eng.workspace(*sp.shape))
        mags = r.grad.double().norm(dim=-1)
        mean = mags.mean(0)
        rstd = (mags.std(0, unbiased=True) + 1e-8) / (mean + 1e-8)
        rrange = (mags.max(0).values - mags.min(0).values + 1e-8) / (mean + 1e-8)
        qbc = r.energies.std(0, unbiased=True) / (dev(sp) >= 0).sum(1, dtype=torch.float64).sqrt()
        assert_close("|F| mean", r.force_magnitudes.cpu().numpy(), mean.cpu().numpy(), 1e-5, 1e-9)
        assert_close("relative std", r.force_relative_stdev.cpu().numpy(), rstd.cpu().numpy(), 1e-4, 1e-6)
        assert_close("relative range", r.force_relative_range.cpu().numpy(), rrange.cpu().numpy(), 1e-4, 1e-6)
        assert_close("qbc", r.qbc.cpu().numpy(), qbc.cpu().numpy(), 1e-6, 1e-9)
        assert_close("mean gradient", eng.workspace(*sp.shape).grad.view(f_m.shape[1:]).cpu().numpy(),
                     -f_m.mean(0).cpu().numpy(), 1e-6, 1e-6)
        # a term common to all members leaves the energy QBC factor alone and changes the force statistics
        eng0 = m0.engine(torch.device(DEV))
        q0 = eng0.members_result(eng0.workspace(*sp.shape)).qbc
        assert torch.allclose(r.qbc, q0, rtol=0, atol=1e-6)                      # float64, on the device
        q1 = m1.energies_qbcs(*args).qbcs                                        # float32 energies at |E| ~ 1e4 Ha
        assert torch.allclose(q1.double(), m0.energies_qbcs(*args).qbcs.double(), rtol=0, atol=1e-3)
        assert not torch.allclose(m1.force_qbc(*args).magnitudes, m0.force_qbc(*args).magnitudes, atol=1e-4)
    finally:
        for mm in (m1, m0):
            mm.neural_networks.set_active_members(list(range(8)))


# ------------------------------------------------------------------------------------------------------------------
# 7. graph replay, launch counts, enabling
# ------------------------------------------------------------------------------------------------------------------
def test_graph_replay_after_composition_change_and_launch_counts():
    m1, m0 = model("xtb", "smooth"), model(None)
    sp, co, cell, pbc = golden_inputs(load_golden("water999_pbc_ani2x"), torch.float32)
    eng1, eng0 = m1.engine(torch.device(DEV)), m0.engine(torch.device(DEV))
    for _ in range(6):      # eager steps, capture, replay
        e_a, f_a = m1.energies_and_forces(dev(sp), dev(co), dev(cell), dev(pbc))
    assert any(k[:2] == (1, 999) for k in eng1._graphs), "the step with the pair launch must be captured"
    sp2 = sp.clone()
    sp2[0, :3] = torch.tensor([4, 0, 0])      # a sulfur: another composition under the same captured graph
    e_b, f_b = m1.energies_and_forces(dev(sp2), dev(co), dev(cell), dev(pbc))
    e_0, f_0 = m0.energies_and_forces(dev(sp2), dev(co), dev(cell), dev(pbc))
    ref = porc.compute(spec("xtb", "smooth"), sp2, co.double(), cell.double(), pbc, "cell_list")
    assert_close("replayed pair forces", (f_b - f_0).cpu().numpy(), ref["forces"].numpy(), F_RTOL, F_ATOL)
    assert abs(float(e_b - e_0) - float(ref["energy"])) < 1e-4
    # one launch more per pair potential, none for a model without
    n1, n0 = eng1.launches_per_step, eng0.launches_per_step
    assert n1 == n0 + 1 and not eng0.pairs
    from torchani_b200.engine import Engine
    plain = Engine(eng0.consts, eng0.nets, eng0.sae.tolist(), nbr_cap=eng0.nbr_cap)
    plain.step(dev(sp2), dev(co), dev(cell), True)
    assert plain.launches_per_step == n0
    # a disabled potential is skipped (arch.py:371-372)
    m1.set_enabled("repulsion_xtb", False)
    try:
        e_off, f_off = m1.energies_and_forces(dev(sp2), dev(co), dev(cell), dev(pbc))
        assert torch.equal(e_off, e_0) or abs(float(e_off - e_0)) < 1e-6
        assert m1.engine(torch.device(DEV)).launches_per_step == n0
    finally:
        m1.set_enabled("repulsion_xtb", True)


def test_bad_arguments_return_codes():
    from torchani_b200 import _lib
    L = _lib.lib()
    p = potential("xtb", "cosine").params()
    null = [None] * 3 + [8, 0, 8, 1, 8] + [None, None, 128] + [None] * 7 + [0, None]
    assert L.ani_b200_pair_potential(C.byref(p), *null) == -1
    assert L.ani_b200_pair_potential(None, *null) == -1
    bad = potential("xtb", "cosine").params()
    bad.kind = 7
    x = torch.zeros(64, dtype=torch.int32, device=DEV)
    args = [x.data_ptr()] * 3 + [8, 0, 8, 1, 8, x.data_ptr(), x.data_ptr(), 4] + [None] * 7 + [0, None]
    assert L.ani_b200_pair_potential(C.byref(bad), *args) == -1
    args_hi = list(args)
    args_hi[5] = 9       # hi > n
    assert L.ani_b200_pair_potential(C.byref(p), *args_hi) == -1
    assert L.ani_b200_pair_potential_cells(C.byref(p), *args[:-1], None, None) == -1      # no lattice table
    assert L.ani_b200_pair_potential_pairs(C.byref(p), None, None, None, None, None, None, 5, 1, 8, None, None, None,
                                           None) == -1


# ------------------------------------------------------------------------------------------------------------------
# 8. the half-list entry point and the drop-in paths
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,fn", [("xtb", "smooth"), ("zbl", "cosine")])
def test_pair_list_entry_point_with_ghost_flags(kind, fn):
    from torchani_b200 import neighbors as nbm
    pot = potential(kind, fn).to(DEV)
    sp, co, cell, pbc = golden_inputs(load_golden("1c17_chunk_hcnos_ani2x"))
    ghost = torch.zeros_like(sp, dtype=torch.bool)
    ghost[0, ::5] = True
    x = dev(co).float().requires_grad_(True)
    nb = nbm.all_pairs(RCR + 0.7, dev(sp), x)          # a wider list: pairs beyond the cutoff are ignored
    e = pot.compute_from_neighbors(dev(sp), x, nb, ghost_flags=dev(ghost))
    (g,) = torch.autograd.grad(e.sum(), x)
    a = pot.compute_from_neighbors(dev(sp), x.detach(), nb, atomic=True, ghost_flags=dev(ghost))
    xr = co.clone().requires_grad_(True)
    nbr = orc.all_pairs(RCR, sp, xr)
    a_ref = porc.energies_from_neighbors(spec(kind, fn), sp, nbr, atomic=True, ghost_flags=ghost)
    (g_ref,) = torch.autograd.grad(a_ref.sum(), xr)
    assert_close("ghost atomic", a.cpu().numpy(), a_ref.detach().numpy(), E_RTOL, E_ATOL)
    assert_close("ghost gradient", g.cpu().numpy(), g_ref.numpy(), F_RTOL, F_ATOL)
    assert abs(float(e) - float(a_ref.sum())) < 1e-4
    # the module's own forward: a neighbour list of its own, atomic numbers in
    z = torch.tensor([orc.ATOMIC_NUMBERS[s] for s in orc.SYMBOLS_2X])[sp]
    e2 = pot(dev(z), dev(co).float())
    ref = pair_golden("1c17_chunk_hcnos_ani2x")[f"{kind}_{fn}_energy"]
    assert abs(float(e2) - float(ref[0])) < 1e-4


def test_drop_in_against_the_staged_reference():
    import oracle.ref_torchani as ref
    if not os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "torchani")):
        pytest.skip("the reference is not staged (oracle/_ref)")
    from torchani_b200 import models
    w = orc.make_weights(orc.SYMBOLS_2X, orc.DIMS_2X, 1008, 2, 1234, torch.float32)
    sp, co, cell, pbc = golden_inputs(load_golden("kat2x5_ani2x"), torch.float32)
    z = torch.tensor([orc.ATOMIC_NUMBERS[s] for s in orc.SYMBOLS_2X])[sp]
    rm = ref.build_model(w, device=DEV, neighborlist="all_pairs", repulsion=True)
    e_ref, f_ref = ref.energies_and_forces(rm, dev(z), dev(co))
    conv = models.from_torchani(rm)
    assert list(conv.potentials) == ["repulsion_xtb"]
    e, f = conv.energies_and_forces(dev(z), dev(co))
    e_ref, f_ref = e_ref.detach(), f_ref.detach()
    assert_close("from_torchani energies", e.cpu().numpy(), e_ref.double().cpu().numpy(), 0.0, 2e-3)
    assert_close("from_torchani forces", f.cpu().numpy(), f_ref.cpu().numpy(), 0.0, 2e-4)
    # external neighbour list (compute_from_external_neighbors) through the pair-list entry point
    A = sp.shape[1]
    tri = torch.triu_indices(A, A, 1)
    idx = (tri.unsqueeze(1) + A * torch.arange(sp.shape[0]).view(1, -1, 1)).reshape(2, -1)
    e_ext = conv.compute_from_external_neighbors(dev(z), dev(co), dev(idx), None)
    assert_close("external list", e_ext.detach().cpu().numpy(), e_ref.cpu().numpy(), 0.0, 2e-3)
    acc = models.accelerate_torchani_(ref.build_model(w, device=DEV, neighborlist="all_pairs", repulsion=True))
    assert type(acc.potentials["repulsion_xtb"]).__name__ == "_DropInPairPotential"
    e_acc, f_acc = ref.energies_and_forces(acc, dev(z[:1]), dev(co[:1]))     # (its cell list takes one conformer)
    e_ref, f_ref = e_ref[:1], f_ref[:1]
    assert_close("accelerate energies", e_acc.detach().cpu().numpy(), e_ref.cpu().numpy(), 0.0, 2e-3)
    assert_close("accelerate forces", f_acc.detach().cpu().numpy(), f_ref.cpu().numpy(), 0.0, 2e-4)
