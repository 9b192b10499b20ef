"""The query-by-committee step: every active member's forces from one AEV-backward launch, the disagreement statistics
on the device, in the step's CUDA graph (Engine.run(..., members=True), HostCalculator.calculate_with_qbc, the ASE
calculator's ``qbc`` flag).

Checked here: members_forces against the float64 oracle per member in grid modes 0-3 with all members and an active
subset; ani_b200_aev_backward_members against ani_b200_aev_backward applied slab by slab; the statistics kernel against
a torch restatement of arch.py:439-576 (one member, padding atoms, an atom without neighbours); the host loop against
eager steps (graph capture, Verlet skin, batches, member changes, the 3 x bf16 switch); the ASE result keys.
"""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

import oracle.ani_oracle as orc
from helpers import F_ATOL, ROOT, assert_close, golden_inputs, load_golden
from test_gpu_conformer_cells import batch as cells_batch
from test_gpu_periodic_batch import golden_batch, model_for

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PBC = torch.tensor([True, True, True])
ALL = list(range(8))


def _case(name):
    """(species, coords float32, cell float32 or None, pbc or None) on the host."""
    if name == "open":                     # grid mode 0, no cell
        sp, co, cell, pbc = golden_inputs(load_golden("kat2x5_ani2x"), torch.float32)
    elif name == "water999":               # grid mode 0, periodic
        sp, co, cell, pbc = golden_inputs(load_golden("water999_pbc_ani2x"), torch.float32)
    elif name == "padded_batch":           # grid mode 1
        sp, co, cell, pbc = golden_inputs(load_golden("randbatch_ani2x"), torch.float32)
    elif name == "shared_cell_batch":      # grid mode 2
        sp, co, cell = golden_batch("water30_pbc_ani2x", 3, seed=71)
        co, cell, pbc = co.float(), cell.float(), PBC
    elif name == "cells_batch":            # grid mode 3
        sp, co, cell = cells_batch("cubic")
        co, cell, pbc = co.float(), cell.float(), PBC
    else:
        raise KeyError(name)
    return sp, co, cell, pbc


def _dev(t):
    return None if t is None else t.to(DEV)


def _oracle_member(om, sp, co, cell, pbc, m):
    """float64 oracle energies (C,) and forces (C, A, 3) of member m (the oracle's cell list takes one conformer)."""
    refs = []
    for k in range(sp.shape[0]):
        ck = None if cell is None else (cell[k] if cell.dim() == 3 else cell).double()
        refs.append(orc.compute(om, sp[k:k + 1], co[k:k + 1].double(), ck, pbc, members=[m]))
    return torch.cat([r["energy"] for r in refs]), torch.cat([r["forces"] for r in refs])


@pytest.fixture
def model():
    m, om = model_for("cell_list")
    m.neural_networks.set_active_members(ALL)
    yield m, om
    m.neural_networks.set_active_members(ALL)


# ------------------------------------------------------------------------------------------------------------------
# 1. member forces against the float64 oracle
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["open", "water999", "padded_batch", "shared_cell_batch", "cells_batch"])
def test_member_forces_vs_float64(model, name):
    m, om = model
    sp, co, cell, pbc = _case(name)
    subsets = [ALL, [1, 4, 6]] if name in ("open", "water999", "cells_batch") else [ALL]
    for active in subsets:
        m.neural_networks.set_active_members(active)
        _, e_m, f_m = m.members_forces((_dev(sp), _dev(co)), _dev(cell), _dev(pbc))
        assert f_m.shape == (len(active),) + tuple(co.shape)
        for k, mem in enumerate(active):
            e_ref, f_ref = _oracle_member(om, sp, co, cell, pbc, mem)
            assert_close(f"{name} member {mem} forces", f_m[k].cpu().numpy(), f_ref.numpy(), 0.0, F_ATOL)
            n_real = int((sp >= 0).sum())
            assert_close(f"{name} member {mem} energies", e_m[k].cpu().numpy(), e_ref.numpy(), 0.0,
                         2e-7 * max(n_real, 10) + 5e-3)


# ------------------------------------------------------------------------------------------------------------------
# 2. the members backward against the single-slab backward
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["water999", "cells_batch"])
def test_backward_members_equals_single_slab_backward(model, name):
    """Same arithmetic per member, only the order of the float atomics differs: |difference| <= 1e-5 of the largest
    gradient component (a sum of ~100 neighbour terms reordered: ~100 x 2^-24 relative)."""
    from torchani_b200._lib import check, ptr
    m, _ = model
    m.neural_networks.set_active_members([6, 1, 4])    # not in index order: output k is member active[k]
    sp, co, cell, pbc = _case(name)
    eng = m.engine(torch.device(DEV))
    e_m, g_m = eng.step_members(_dev(sp), _dev(co), _dev(cell), True)
    ws = eng.workspace(*sp.shape)
    L, n = eng.lib, ws.n
    per_conf = cell.dim() == 3
    for k, mem in enumerate([6, 1, 4]):
        out = torch.zeros(n, 3, dtype=torch.float32, device=DEV)
        args = (C.byref(eng.params), ptr(ws.grid), ptr(ws.spos), ptr(ws.sorted_orig),
                ws.aev_blocks.data_ptr() + 4 * (ws.n_blocks + 1), n, 0, n, ptr(ws.row_of), ws.dx_members[mem].data_ptr(),
                eng.nets.ldx, ptr(ws.nbr_cnt), ptr(ws.nbr_list), ws.nbr_cap, ptr(out), ptr(ws.status), 0, None)
        if per_conf:
            check(L.ani_b200_aev_backward_cells(*args, ptr(ws.lattice), None), "aev_backward_cells")
        else:
            check(L.ani_b200_aev_backward(*args, None), "aev_backward")
        torch.cuda.synchronize()
        got = g_m[k].reshape(n, 3)
        bound = 1e-5 * float(out.abs().max())
        assert float((got - out).abs().max()) <= bound, (name, mem)
    eng.check_status()


# ------------------------------------------------------------------------------------------------------------------
# 2b. per-member slabs of the resident MLP launch
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("active", [ALL, [1, 4, 6]], ids=["all", "subset"])
def test_resident_slabs(model, active):
    """ani_b200_mlp_step_resident_members against the data-flow want_backward=2 slabs, and the scaled sum of its slabs
    against the dx of the ordinary resident step.  Both launches compute the same products in another order: slabs
    agree to 1e-5 of their largest element, as the launches' forces do in test_gpu_mlp_resident.py.  Inactive members'
    slabs are not written and their e_member rows are zeroed."""
    from torchani_b200 import _lib, synthetic
    from torchani_b200._lib import check, ptr
    m, _ = model
    m.neural_networks.set_active_members(active)
    _, idx, co, cell, _ = synthetic.water_box(3333, seed=0)
    eng = m.engine(torch.device(DEV))
    if not eng._resident_ok:
        pytest.skip("the resident MLP kernel is not in this build")
    res = eng.step(idx.to(DEV), co.float().to(DEV), cell.float().to(DEV), True, want_grad=True, check=True)
    assert eng.mlp_resident, "water 10 k must take the resident MLP launch"
    g_step = res.grad.clone()
    ws = eng.workspace(*idx.shape)
    nets, L = eng.nets, eng.lib
    rows_cap, ldx, M = ws.rows_cap, nets.ldx, nets.num_members
    dx_sum = ws.dx.clone()
    unit = _lib.MLPModel.from_buffer_copy(nets.model)
    for k in range(_lib.ANI_MAX_MEMBERS):
        unit.member_scale[k] = 1.0 if k in active else 0.0
    res_slabs = torch.full((M, rows_cap, ldx), float("nan"), device=DEV)
    flow_slabs = torch.zeros(M, rows_cap, ldx, device=DEV)
    e_res = torch.full((M, rows_cap), float("nan"), device=DEV)
    e_flow = torch.zeros(M, rows_cap, device=DEV)
    check(L.ani_b200_mlp_step_resident_members(
        C.byref(unit), ptr(ws.x), ptr(res_slabs), rows_cap * ldx, rows_cap, ptr(ws.row_atom), ptr(ws.layout_info),
        ptr(ws.aev_blocks), ptr(ws.act1), ptr(ws.act2), ptr(e_res), ptr(ws.status), None), "resident_members")
    check(L.ani_b200_mlp_step(
        C.byref(unit), ptr(ws.x), ptr(flow_slabs), rows_cap, ptr(ws.row_atom), ptr(ws.layout_info),
        ptr(ws.aev_blocks), ptr(ws.act1), ptr(ws.act2), ptr(ws.act3), ptr(e_flow), 2, ptr(ws.mlp_sync),
        ptr(ws.status), None), "mlp_step")
    torch.cuda.synchronize()
    eng.check_status(ws)
    used = int(ws.layout_info[4 + nets.num_species]) * 128          # rows of the layout's row tiles
    real = (ws.row_atom[:used] >= 0).nonzero().view(-1)
    nblk = int(ws.aev_blocks[0])
    live = (ws.aev_blocks[1:1 + nblk].long().view(-1, 1) * 32 + torch.arange(32, device=DEV)).view(-1)
    total = torch.zeros(real.numel(), live.numel(), dtype=torch.float64, device=DEV)
    for mem in range(M):
        if mem not in active:
            assert bool(torch.isnan(res_slabs[mem]).all()), f"the slab of inactive member {mem} was written"
            assert float(e_res[mem].abs().max()) == 0.0, f"e_member of inactive member {mem} not zeroed"
            continue
        a = res_slabs[mem][real][:, live]
        b = flow_slabs[mem][real][:, live]
        assert not bool(torch.isnan(a).any()), f"member {mem}: a live column of a real row was not written"
        bound = 1e-5 * float(b.abs().max())
        assert float((a - b).abs().max()) <= bound, f"member {mem}: resident vs data-flow slab"
        assert float((e_res[mem][real] - e_flow[mem][real]).abs().max()) <= 1e-5 * float(e_flow[mem].abs().max())
        total += a.double() / len(active)
    ref = dx_sum[real][:, live].double()
    assert float((total - ref).abs().max()) <= 1e-5 * float(ref.abs().max()), "sum of scaled slabs vs resident dx"
    # the QBC step takes this launch here, and its forces agree with the ordinary step's
    _, g_m = eng.step_members(idx.to(DEV), co.float().to(DEV), cell.float().to(DEV), True)
    assert eng.mlp_resident
    g_mean = g_m.double().mean(0)
    assert float((g_mean - g_step.double()).abs().max()) < 1e-5


# ------------------------------------------------------------------------------------------------------------------
# 3. the statistics kernel against a restatement of arch.py:439-576
# ------------------------------------------------------------------------------------------------------------------
def _stats_ref(e_m, g_m, sp):
    """arch.py:439-485 (energies_qbcs) and 543-576 (force_qbc) in float64 on the members' energies and gradients."""
    mags = g_m.double().norm(dim=-1)                                     # (M, C, A)
    eps = 1e-8
    mean = mags.mean(0)
    if mags.shape[0] == 1:
        rstd, rrange = torch.zeros_like(mean), torch.ones_like(mean)
        qbc = torch.zeros_like(e_m[0])
    else:
        rstd = (mags.std(0, unbiased=True) + eps) / (mean + eps)
        rrange = ((mags.max(0).values - mags.min(0).values) + eps) / (mean + eps)
        qbc = e_m.std(0, unbiased=True)
    qbc = qbc / (sp >= 0).sum(dim=1, dtype=torch.float64).sqrt()
    return qbc, mean, rstd, rrange


@pytest.mark.parametrize("active", [ALL, [2, 5], [3]], ids=["eight", "two", "one"])
@pytest.mark.parametrize("name", ["lonely_atom", "padded_batch", "cells_batch"])
def test_statistics_vs_restatement(model, name, active):
    m, _ = model
    m.neural_networks.set_active_members(active)
    if name == "lonely_atom":     # an atom 40 A from the molecule: no neighbours, zero force for every member
        sp, co, cell, pbc = _case("open")
        sp = torch.cat([sp, torch.zeros(sp.shape[0], 1, dtype=sp.dtype)], 1)
        co = torch.cat([co, co[:, :1] + 40.0], 1)
    else:
        sp, co, cell, pbc = _case(name)
    eng = m.engine(torch.device(DEV))
    spd, cod, celld = _dev(sp), _dev(co), _dev(cell)
    per_conf = cell is not None and cell.dim() == 3
    ws = eng.workspace(*sp.shape)
    if pbc is not None:
        ws.make_periodic()
    ws.species_i32.copy_(spd.reshape(-1))
    ws.coords.copy_(cod.reshape(-1, 3))
    if per_conf:
        ws.cells.copy_(celld.reshape(-1, 9))
    elif pbc is not None:
        ws.cell.copy_(celld.reshape(-1))
    res = eng.run(ws, pbc is not None, True, members=True, conformer_cells=per_conf)
    eng.check_status(ws)
    r = eng.members_result(ws)
    qbc, mean, rstd, rrange = _stats_ref(r.energies, r.grad, spd)
    assert_close(f"{name} qbc", r.qbc.cpu().numpy(), qbc.cpu().numpy(), 1e-6, 1e-9)
    assert_close(f"{name} |F| mean", r.force_magnitudes.cpu().numpy(), mean.cpu().numpy(), 1e-5, 1e-9)
    assert_close(f"{name} relative std", r.force_relative_stdev.cpu().numpy(), rstd.cpu().numpy(), 1e-4, 1e-6)
    assert_close(f"{name} relative range", r.force_relative_range.cpu().numpy(), rrange.cpu().numpy(), 1e-4, 1e-6)
    if name == "lonely_atom":
        assert float(r.force_magnitudes[0, -1]) == 0.0
        assert float(r.force_relative_stdev[0, -1]) == pytest.approx(0.0 if len(active) == 1 else 1.0)
        assert float(r.force_relative_range[0, -1]) == pytest.approx(1.0)
    # the mean gradient is the step's gradient; the step's energies are the ensemble mean
    grad = res.grad.clone()
    e_mean = res.energies.clone()
    assert torch.allclose(e_mean, r.energies.mean(0), rtol=1e-9, atol=1e-6)
    e2, f2 = m.energies_and_forces(spd, cod, celld, _dev(pbc))
    assert_close(f"{name} mean gradient", -grad.cpu().numpy(), f2.cpu().numpy(), 0.0, F_ATOL)
    assert_close(f"{name} energies", e_mean.cpu().numpy(), e2.cpu().numpy(), 1e-9, 1e-6)


# ------------------------------------------------------------------------------------------------------------------
# 4. the host loop
# ------------------------------------------------------------------------------------------------------------------
_EAGER = {}


def _eager(m, sp, co, cell):
    """One uncaptured Engine.run(members=True) on an engine without CUDA graphs that shares the model's networks:
    (energies (C,), grad (C, A, 3), MembersResult, step_members output)."""
    from torchani_b200.engine import Engine
    base = m.engine(torch.device(DEV))
    eng = _EAGER.get(id(base))
    if eng is None or eng.nets is not base.nets:
        eng = _EAGER[id(base)] = Engine(base.consts, base.nets, base.sae.tolist(), nbr_cap=base.nbr_cap,
                                        cuda_graph=False)
    res_m = eng.step_members(_dev(sp), _dev(co), _dev(cell), cell is not None)
    ws = eng.workspace(*sp.shape)
    eng.check_status(ws)
    r = eng.members_result(ws)
    return ws.energies.clone(), ws.grad.view(sp.shape + (3,)).clone(), r, res_m


def _check_host(tag, got, ref, batch):
    e, f, q = got
    e_ref, g_ref, r, _ = ref
    c = slice(None) if batch else 0
    assert np.allclose(e, e_ref.cpu().numpy()[c], rtol=1e-12, atol=1e-6), tag
    assert_close(f"{tag} forces", f, -g_ref.cpu().numpy()[c], 0.0, 1e-5)
    assert_close(f"{tag} energy qbc", q.energy_qbc, r.qbc.cpu().numpy()[c], 1e-6, 1e-8)
    for name, val in (("force_magnitudes", r.force_magnitudes), ("force_relative_stdev", r.force_relative_stdev),
                      ("force_relative_range", r.force_relative_range)):
        assert_close(f"{tag} {name}", getattr(q, name), val.cpu().numpy()[c], 1e-4, 1e-6)


def test_host_loop_graph_capture_and_member_changes(model):
    from torchani_b200.calculator import HostCalculator
    m, _ = model
    sp, co, cell, pbc = _case("water999")
    calc = HostCalculator(m, sp[0].numpy(), cell.numpy(), pbc=True)
    g = torch.Generator().manual_seed(5)
    pos = co.clone()
    for step in range(20):
        pos = pos + 0.01 * torch.randn(pos.shape, generator=g)
        if step == 12:
            m.neural_networks.set_active_members([1, 4, 6])
        got = calc.calculate_with_qbc(pos[0].numpy())
        _check_host(f"step {step}", got, _eager(m, sp, pos, cell), batch=False)
    assert calc._graphs, "the QBC step must be captured after a few calls"
    calc.check_status()


def test_host_loop_verlet_skin(model):
    from torchani_b200.calculator import HostCalculator
    m, _ = model
    sp, co, cell, pbc = _case("water999")
    c1 = HostCalculator(m, sp[0].numpy(), cell.numpy(), pbc=True, skin=0.4)
    try:
        g = torch.Generator().manual_seed(6)
        pos = co.clone()
        for step in range(20):
            pos = pos + 0.002 * torch.randn(pos.shape, generator=g)
            if step == 15:
                pos[0, 7] += 0.3        # beyond skin / 2: the reused grid is invalid, the step is redone
            # against a fresh grid (skin 0) on an engine of its own
            _check_host(f"skin step {step}", c1.calculate_with_qbc(pos[0].numpy()), _eager(m, sp, pos, cell),
                        batch=False)
        assert c1.rebuilds < 20 and c1.redone >= 1, (c1.rebuilds, c1.redone)
    finally:
        m.engine(torch.device(DEV)).skin = 0.0


@pytest.mark.parametrize("cells", ["shared", "per_conformer"])
def test_host_batch_equals_single_calls(model, cells):
    from torchani_b200.calculator import HostCalculator
    m, _ = model
    sp, co, cell, pbc = _case("shared_cell_batch" if cells == "shared" else "cells_batch")
    calc = HostCalculator(m, sp.numpy(), cell.numpy(), pbc=True)
    for _ in range(calc.graph_after + 2):
        e, f, q = calc.calculate_with_qbc(co.numpy())
    assert e.shape == (sp.shape[0],) and q.energy_qbc.shape == (sp.shape[0],)
    assert q.force_magnitudes.shape == tuple(sp.shape)
    for k in range(sp.shape[0]):
        ck = cell if cell.dim() == 2 else cell[k]
        single = HostCalculator(m, sp[k].numpy(), ck.numpy(), pbc=True)
        es, fs, qs = single.calculate_with_qbc(co[k].numpy())
        assert abs(es - e[k]) < 1e-6
        real = sp[k].numpy() >= 0
        assert_close(f"conformer {k} forces", f[k][real], fs[real], 0.0, 1e-5)
        assert abs(qs.energy_qbc - q.energy_qbc[k]) <= 1e-6 * abs(qs.energy_qbc) + 1e-9
        for name in ("force_magnitudes", "force_relative_stdev", "force_relative_range"):
            assert_close(f"conformer {k} {name}", getattr(q, name)[k][real], getattr(qs, name)[real], 1e-4, 1e-6)


def test_host_operand_range_switches_to_bf16x3():
    from test_gpu_bf16x3 import VARIANT, ZNUM, check_ef, switch_model, switched, water_and_close_pair
    from torchani_b200.calculator import HostCalculator
    species, coords, moved, cell, pbc = water_and_close_pair()
    model, om = switch_model()
    z = np.array([ZNUM[int(s)] for s in species[0]])
    calc = HostCalculator(model, z, cell.numpy(), pbc=True)
    for _ in range(calc.graph_after + 1):
        (e, f, q), n = switched(lambda: calc.calculate_with_qbc(coords[0].numpy()))
        assert n == 0
    (e, f, q), n = switched(lambda: calc.calculate_with_qbc(moved[0].numpy()))
    assert n == 1 and model.neural_networks._variant == VARIANT
    ref = orc.compute(om, species, moved.double(), cell.double(), pbc)
    check_ef(e, f, ref, "qbc after the switch")
    # the same statistics as the model API on the 3 x bf16 build
    zt = torch.tensor(z, device=DEV).unsqueeze(0)
    idx, e_m, f_m = model.members_forces((zt, moved.float().to(DEV)), cell.float().to(DEV), pbc.to(DEV))
    qbc, mean, rstd, rrange = _stats_ref(e_m.double(), -f_m, idx)
    assert abs(q.energy_qbc - float(qbc[0])) <= 1e-5 * abs(float(qbc[0])) + 1e-8
    assert_close("bf16x3 |F| mean", q.force_magnitudes, mean[0].cpu().numpy(), 1e-4, 1e-6)
    assert_close("bf16x3 relative std", q.force_relative_stdev, rstd[0].cpu().numpy(), 1e-3, 1e-5)
    assert_close("bf16x3 relative range", q.force_relative_range, rrange[0].cpu().numpy(), 1e-3, 1e-5)


def test_host_rejects_sharding(model):
    from torchani_b200.calculator import HostCalculator
    m, _ = model
    sp, co, cell, pbc = _case("water999")
    calc = HostCalculator(m, sp[0].numpy(), cell.numpy(), pbc=True, shard=(0, 2))
    with pytest.raises(ValueError):
        calc.calculate_with_qbc(co[0].numpy())
    eng = m.engine(torch.device(DEV))
    with pytest.raises(ValueError):
        eng.run(eng.workspace(1, sp.shape[1]), True, True, shard=(0, 2), members=True)


# ------------------------------------------------------------------------------------------------------------------
# 5. ASE
# ------------------------------------------------------------------------------------------------------------------
def test_ase_calculator_qbc_keys():
    try:
        import ase  # noqa: F401
    except ImportError:
        sys.path.insert(0, os.path.join(ROOT, "tests", "stubs"))
    from ase import Atoms
    from torchani_b200 import models, synthetic
    from torchani_b200.ase import Calculator
    from torchani_b200.calculator import HostCalculator
    w = synthetic.make_weights(models.SYMBOLS_2X, synthetic.DIMS_2X, 1008, 8, seed=1234)
    model = models.from_weight_lists("2x", w, device=DEV, periodic_table_index=True)
    rec = load_golden("water30_pbc_ani2x")
    species, coords, cell, pbc = golden_inputs(rec, torch.float64)
    zmap = {0: 1, 1: 6, 2: 7, 3: 8, 4: 16, 5: 9, 6: 17}
    numbers = [zmap[int(s)] for s in species[0]]
    atoms = Atoms(numbers, coords[0].numpy(), cell=cell.numpy(), pbc=True)
    atoms.calc = Calculator(model, qbc=True)
    e = atoms.get_potential_energy()
    res = atoms.calc.results
    host = HostCalculator(model, np.array(numbers), cell.numpy(), pbc=True)
    e_h, f_h, q = host.calculate_with_qbc(coords[0].numpy())
    ha = 27.211386024367243
    assert abs(e - e_h * ha) < 1e-6 * abs(e)
    assert abs(res["energy_qbc"] - q.energy_qbc * ha) <= 1e-6 * abs(res["energy_qbc"]) + 1e-9
    assert res["force_magnitudes"].shape == (len(numbers),)
    assert_close("eV/A magnitudes", res["force_magnitudes"], q.force_magnitudes * ha, 1e-4, 1e-6)
    assert_close("relative std", res["force_relative_stdev"], q.force_relative_stdev, 1e-4, 1e-6)
    assert_close("relative range", res["force_relative_range"], q.force_relative_range, 1e-4, 1e-6)
    # a stress request keeps the QBC keys (the stress step, then the QBC step on the same positions)
    atoms.calc = Calculator(model, stress_kind="fdotr", qbc=True)
    atoms.get_stress()
    assert abs(atoms.calc.results["energy_qbc"] - q.energy_qbc * ha) <= 1e-6 * abs(q.energy_qbc * ha) + 1e-9
    assert_close("relative std with stress", atoms.calc.results["force_relative_stdev"], q.force_relative_stdev,
                 1e-4, 1e-6)
    assert atoms.calc.results["stress"].shape == (3, 3)
    # the magnitudes are those of the members' forces in eV/A
    _, _, f_m = model.members_forces((torch.tensor(numbers, device=DEV).unsqueeze(0), coords.float().to(DEV)),
                                     cell.float().to(DEV), pbc.to(DEV))
    assert_close("magnitudes vs members_forces", res["force_magnitudes"],
                 (f_m.double().norm(dim=-1).mean(0)[0] * ha).cpu().numpy(), 1e-4, 1e-6)
