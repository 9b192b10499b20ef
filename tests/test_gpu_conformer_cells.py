"""Periodic batches with one cell per conformer (grid mode 3): a (C, 3, 3) cell, one engine step.

Buckets are numbered conformer-major as in mode 2, with sub-grid dims common to the batch (per axis the minimum over
the conformers of the buckets their own cell admits); every atom is wrapped, and every image shift is taken, in its
own conformer's lattice (the lattice table the preparation writes).  Checked here: C equal cells give bit for bit the
results of the shared (3, 3) cell (mode 2) -- preparation outputs, AEV rows, energies, forces, virial; with distinct
cubic, orthorhombic and triclinic cells the preparation against a float64 restatement per conformer and the model API
against the float64 oracle per conformer; graph replay with changed cells, shards, both MLP launches, the status words,
the 3 x bf16 build, the batched HostCalculator and the rejected inputs.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import oracle.ani_oracle as orc
from helpers import E_ATOL, E_RTOL, F_ATOL, assert_close
from test_gpu_periodic_batch import StepCounter, golden_batch, model_for
from test_gpu_prepare import ROOT, in_cell, layout_ref

DEV = "cuda:0"
PBC = torch.tensor([True, True, True])
RC = 5.1            # ANI-2x radial cutoff
BUCKET = np.float32(RC) + np.float32(1e-5)


def strained(sp, co, cell, strains):
    """Conformer c in cell @ strains[c] with its fractional coordinates kept: (C, 3, 3) cells, (C, A, 3) coords."""
    inv = torch.linalg.inv(cell)
    cells = torch.stack([cell @ torch.as_tensor(s, dtype=torch.float64) for s in strains])
    return sp, torch.stack([co[c] @ inv @ cells[c] for c in range(len(strains))]), cells


def diag(x, y, z):
    return np.diag([x, y, z])


def gas(n_conf: int = 4, n: int = 40, seed: int = 3):
    """Random atoms (H, C, N, O) in cubic cells of about 15.4 A (3 buckets per axis) whose volumes differ by a few per
    cent, and one conformer in a 21 A cell (4 buckets of its own per axis): the common dims are 3 x 3 x 3."""
    rng = np.random.default_rng(seed)
    edges = [15.4 * (1.0 + 0.01 * (c % 3 - 1)) for c in range(n_conf)]
    edges[2] = 21.0
    cells = torch.tensor(np.stack([np.eye(3) * e for e in edges]))
    co = torch.tensor(np.stack([in_cell(cells[c].numpy(), n, seed=seed + c, min_dist=1.1) for c in range(n_conf)]))
    sp = torch.tensor(rng.integers(0, 4, size=(n_conf, n)))
    sp[-1, -4:] = -1                                         # a padded conformer
    return sp, co, cells


def batch(case: str):
    """(species (C, A), coords (C, A, 3), cells (C, 3, 3)) float64 on the host."""
    if case == "cubic":
        sp, co, cell = golden_batch("water30_pbc_ani2x", 4, seed=51)
        return strained(sp, co, cell, [np.eye(3) * s for s in (1.0, 0.97, 1.032, 0.99)])   # volumes -9 % .. +10 %
    if case == "orthorhombic":
        sp, co, cell = golden_batch("water30_pbc_ani2x", 4, seed=52)
        return strained(sp, co, cell, [diag(1.0, 1.0, 1.0), diag(1.05, 0.98, 1.0), diag(0.96, 1.0, 0.98),
                                       diag(1.0, 1.04, 1.05)])
    if case == "triclinic":
        sp, co, cell = golden_batch("6w8h_triclinic_ani2x", 3, seed=53)
        shear = np.eye(3)
        shear[1, 0] = 0.04
        return strained(sp, co, cell, [np.eye(3), 0.97 * shear, np.eye(3) * 1.03])
    if case == "gas":
        return gas()
    raise KeyError(case)


CASES = ["cubic", "orthorhombic", "triclinic", "gas"]


def dev(sp, co, cells):
    return sp.to(DEV), co.float().to(DEV), cells.float().to(DEV)


def wrapped(co, cells):
    """float64 coordinates wrapped into each conformer's own cell (the oracle's stress needs wrapped atoms)."""
    return torch.stack([x - torch.floor(x @ torch.linalg.inv(L)) @ L for x, L in zip(co, cells)])


def eager_engine(base, **kw):
    from torchani_b200.engine import Engine
    return Engine(base.consts, base.nets, base.sae.tolist(), nbr_cap=kw.get("nbr_cap", base.nbr_cap),
                  cuda_graph=kw.get("cuda_graph", False))


# ------------------------------------------------------------------------------------------------------------------
# 1. equal cells: exactly mode 2
# ------------------------------------------------------------------------------------------------------------------
OUTPUTS = ("bin_start", "sorted_orig", "orig_to_sorted", "spos", "sbin", "bucket_ranges", "row_of", "row_atom",
           "tile_species", "layout_info", "nbr_cnt", "nbr_list", "atomic", "member_atomic")


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["water", "triclinic"])
def test_equal_cells_are_mode_2_bit_for_bit(case):
    model, _ = model_for("cell_list")
    eng = eager_engine(model.engine(torch.device(DEV)))
    if case == "water":
        sp, co, cell = golden_batch("water30_pbc_ani2x", 5, seed=61)
    else:
        sp, co, cell = golden_batch("6w8h_triclinic_ani2x", 3, seed=62)
    sp, co, cell = sp.to(DEV), co.float().to(DEV), cell.float().to(DEV)
    cells = cell.expand(sp.shape[0], 3, 3).contiguous()
    got = []
    for c in (cell, cells):
        res = eng.step(sp, co, c, True, want_virial=True, check=True)
        ws = eng.workspace(*sp.shape)
        out = {k: getattr(ws, k).clone() for k in OUTPUTS}
        out.update(energies=res.energies.clone(), grad=res.grad.clone(), virial=res.virial.clone(),
                   grid=ws.grid.clone(), x=ws.x.clone(), blocks=ws.aev_blocks[:-1].clone())   # (not the changed flag)
        got.append(out)
    a, b = got
    assert int(a["grid"][26]) == 2 and int(b["grid"][26]) == 3
    keep = torch.ones_like(a["grid"], dtype=torch.bool)
    keep[26] = False                                     # the mode word
    assert torch.equal(a["grid"][keep], b["grid"][keep]), "grid"
    for k in OUTPUTS + ("x", "blocks"):
        assert torch.equal(a[k].view(torch.uint8), b[k].view(torch.uint8)), k
    # forces, conformer energies and the virial are accumulated with atomics (order-dependent in the last bits; the
    # virial's float32 partial sums follow dE/dAEV, whose member sum is atomic too)
    assert (a["grad"] - b["grad"]).abs().max() < 1e-6
    assert torch.allclose(a["energies"], b["energies"], rtol=1e-12, atol=0)
    assert torch.allclose(a["virial"], b["virial"], rtol=1e-5, atol=1e-6 * float(a["virial"].abs().max()))
    # the AEV rows on every AEV kernel path through the ABI: with the range table, with the per-bucket species offsets,
    # and with the ranges derived on the fly (image shifts from the lattice table)
    from torchani_b200._lib import check, lib
    ws = eng.workspace(*sp.shape)
    comp = model.aev_computer
    out_dim, cap, n = comp.constants.out_dim, comp.nbr_cap, ws.n
    rows = []
    for use_ranges in (True, False):
        aev = torch.zeros(n, out_dim, device=DEV)
        cnt = torch.zeros(n, dtype=torch.int32, device=DEV)
        lst = torch.zeros(n * cap, dtype=torch.int32, device=DEV)
        status = torch.zeros(1, dtype=torch.int32, device=DEV)
        check(lib().ani_b200_aev_forward_cells(
            C.byref(comp._params()), ws.grid.data_ptr(), ws.bin_start.data_ptr(), ws.spos.data_ptr(),
            ws.sbin.data_ptr(), ws.bucket_ranges.data_ptr() if use_ranges else None, None, None, n, 0, n,
            ws.sorted_orig.data_ptr(), aev.data_ptr(), out_dim, 0, cnt.data_ptr(), lst.data_ptr(), cap,
            status.data_ptr(), ws.lattice.data_ptr(), torch.cuda.current_stream().cuda_stream), "aev_forward_cells")
        torch.cuda.synchronize()
        assert int(status.item()) == 0
        rows.append(aev)
    assert torch.equal(rows[0].view(torch.int32), rows[1].view(torch.int32))
    per = comp(sp, co, cell, PBC.to(DEV))                # mode 2 through the AEVComputer
    assert torch.equal(rows[0].view(torch.int32), per.view(n, -1).view(torch.int32))


@pytest.mark.gpu
@pytest.mark.parametrize("var", ["ANI_B200_PREP_FUSED=0", "ANI_B200_AEV_LEGACY=1", "ANI_B200_AEV_TMA=1",
                                 "ANI_B200_AEV_BSS=1"])
def test_process_wide_variants(var):
    """The five-launch preparation and the warp-per-atom / TMA-staged AEV kernels are chosen once per process: re-run
    this file's bit-for-bit and preparation tests in a child process."""
    k, v = var.split("=")
    child_env = dict(os.environ, **{k: v})
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
        "-m", "pytest", os.path.abspath(__file__), "-q", "-m", "gpu", "-p", "no:cacheprovider",
        "-k", "bit_for_bit or preparation_restatement"]
    res = subprocess.run(cmd, cwd=ROOT, env=child_env, capture_output=True, text=True, timeout=1200)
    assert res.returncode == 0, res.stdout[-4000:] + res.stderr[-2000:]
    assert " passed" in res.stdout and " failed" not in res.stdout


# ------------------------------------------------------------------------------------------------------------------
# 2. distinct cells: the preparation against a float64 restatement, conformer by conformer
# ------------------------------------------------------------------------------------------------------------------
def own_dims(cell: np.ndarray) -> np.ndarray:
    widths = 1.0 / np.linalg.norm(np.linalg.inv(cell.astype(np.float64)), axis=0)
    return np.floor(widths / np.float64(BUCKET)).astype(int)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_preparation_restatement(case):
    model, _ = model_for("cell_list")
    eng = eager_engine(model.engine(torch.device(DEV)))
    sp, co, cells = batch(case)
    spd, cod, celld = dev(sp, co, cells)
    eng.step(spd, cod, celld, True, check=True)
    ws = eng.workspace(*sp.shape)
    Cn, A = sp.shape
    n = Cn * A
    cells32 = celld.cpu().numpy().astype(np.float64)
    g = ws.grid.cpu().numpy()
    dims = g[21:24].astype(int)
    assert g[26] == 3 and g[24] == 1 and g[27] == A
    # common dims: the per-axis minimum of what every conformer's own cell admits (the capacity does not bind here)
    own = np.stack([own_dims(c) for c in cells32])
    assert (dims == own.min(0)).all(), (dims, own)
    if case == "gas":
        assert (own[2] > dims).all(), "a conformer whose own cell admits more buckets"
    nb = int(dims.prod())
    assert g[25] == Cn * nb
    # the lattice table: each conformer's cell and its inverse (double, rounded)
    lat = ws.lattice.cpu().numpy()
    for c in range(Cn):
        assert (lat[c, :9] == celld[c].cpu().numpy().reshape(-1)).all(), c
        inv = np.linalg.inv(cells32[c]).astype(np.float32).reshape(-1)
        assert np.allclose(lat[c, 9:], inv, rtol=4e-7, atol=1e-9), c
    # wrapped positions with the conformer's own cell; buckets inside the conformer's sub-grid
    so = ws.sorted_orig.cpu().numpy()
    spos = ws.spos.cpu().numpy()
    sbin = ws.sbin.cpu().numpy()
    bs = ws.bin_start.cpu().numpy()
    real = sp.reshape(-1).numpy() >= 0
    n_real = int(real.sum())
    assert bs[Cn * nb] == n_real
    x = cod.reshape(n, 3).cpu().numpy().astype(np.float64)
    for i in range(n_real):
        a = so[i]
        c = a // A
        L = cells32[c]
        frac = spos[i, :3].astype(np.float64) @ np.linalg.inv(L)
        assert (frac > -1e-5).all() and (frac < 1 + 1e-5).all(), (case, a, frac)
        k = (x[a] - spos[i, :3]) @ np.linalg.inv(L)
        assert np.abs(k - np.round(k)).max() < 1e-4, (case, a, k)
        assert c * nb <= sbin[i] < (c + 1) * nb, (case, a)
        ijk = np.clip(np.floor(np.clip(frac, 0, 1 - 1e-7) * dims), 0, dims - 1).astype(int)
        local = (ijk[0] * dims[1] + ijk[1]) * dims[2] + ijk[2]
        near = np.abs(frac * dims - np.round(frac * dims)).min() < 1e-4
        assert near or sbin[i] == c * nb + local, (case, a)
    # pair completeness over all lattice images: radial neighbour counts of every centre against brute force
    cnt = ws.nbr_cnt.cpu().numpy()
    shifts = np.array([(i, j, k) for i in (-1, 0, 1) for j in (-1, 0, 1) for k in (-1, 0, 1)], dtype=np.float64)
    pos = spos[:, :3].astype(np.float64)
    conf_of = so // A
    for i in range(n_real):
        c = conf_of[i]
        js = np.nonzero((conf_of[:n_real] == c))[0]
        d = pos[js][None, :, :] + (shifts @ cells32[c])[:, None, :] - pos[i]
        r = np.sqrt((d ** 2).sum(-1))
        self_img = (js[None, :] == i) & (np.abs(shifts).sum(1)[:, None] == 0)
        inside = (r <= RC) & ~self_img
        edge = np.abs(r - RC) < 1e-4
        assert abs(int(inside.sum()) - int(cnt[i])) <= int(edge.sum()), (case, i, int(inside.sum()), int(cnt[i]))
    # the row layout of the species-grouped MLP rows
    lay = layout_ref(ws.spos.cpu().numpy().view(np.int32)[:, 3], n_real, 0, n, 7, ws.rows_cap)
    assert (ws.row_of.cpu().numpy()[lay.owned] == lay.row_of).all()
    assert (ws.row_atom.cpu().numpy() == lay.row_atom).all()
    assert (ws.layout_info.cpu().numpy()[:13] == lay.info).all()


# ------------------------------------------------------------------------------------------------------------------
# 3. the model API against the float64 oracle, per conformer with its own cell
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_against_the_oracle(case):
    model, om = model_for("cell_list")
    sp, co, cells = batch(case)
    spd, cod, celld = dev(sp, co, cells)
    pbcd = PBC.to(DEV)
    c32 = celld.double().cpu()                   # the cells the device sees
    co32 = cod.double().cpu()
    refs = [orc.compute(om, sp[c:c + 1], co32[c:c + 1], c32[c], PBC) for c in range(sp.shape[0])]
    eng = model.engine(torch.device(DEV))
    x = cod.clone().requires_grad_(True)
    with StepCounter(eng) as cnt:
        e = model((spd, x), celld, pbcd).energies
    assert cnt.calls == 1, "a batch with one cell per conformer must be one engine step"
    (g,) = torch.autograd.grad(e.sum(), x)
    e64 = model.energies_f64((spd, cod), celld, pbcd)
    at = model((spd, cod), celld, pbcd, atomic=True).energies
    ens = model((spd, cod), celld, pbcd, ensemble_values=True).energies
    e2, f2 = model.energies_and_forces(spd, cod, celld, pbcd)
    assert torch.allclose(e2, e64, rtol=1e-12, atol=0)
    for k, ref in enumerate(refs):
        assert abs(float(e64[k]) - float(ref["energy"][0])) < 5e-3, (case, k)
        assert_close(f"{case}[{k}] forces", -g[k:k + 1].cpu().numpy(), ref["forces"].numpy(), 0.0, F_ATOL)
        assert_close(f"{case}[{k}] forces (energies_and_forces)", f2[k:k + 1].cpu().numpy(), ref["forces"].numpy(),
                     0.0, F_ATOL)
        sae = model.energy_shifter(spd[k:k + 1], atomic=True).cpu().double()
        assert_close(f"{case}[{k}] atomic", at[k:k + 1].cpu().numpy(), (ref["atomic_nn"] + sae).numpy(), E_RTOL, E_ATOL)
    # ensemble members: energies and forces of one pass, against the ensemble values and the oracle per member
    _, e_m, f_m = model.members_forces((spd, cod), celld, pbcd)
    assert torch.allclose(e_m.double(), ens.double(), rtol=1e-6, atol=1e-4)
    for m in (0, 3):
        for k in range(sp.shape[0]):
            ref = orc.compute(om, sp[k:k + 1], co32[k:k + 1], c32[k], PBC, members=[m])
            assert_close(f"{case}[{k}] member {m} forces", f_m[m, k:k + 1].cpu().numpy(), ref["forces"].numpy(), 0.0,
                         F_ATOL)
    # stress: the virial of each conformer over the volume of its own cell
    e3, f3, stress = model.energies_forces_stress(spd, cod, celld, pbcd)
    assert stress.shape == (sp.shape[0], 3, 3)
    w = wrapped(co32, c32)
    for k in range(sp.shape[0]):
        ref = orc.compute(om, sp[k:k + 1], w[k:k + 1], c32[k], PBC, stress=True)
        assert_close(f"{case}[{k}] stress", stress[k].cpu().numpy(), ref["stress"].numpy(), 1e-4, 1e-8)


# ------------------------------------------------------------------------------------------------------------------
# 4. the engine: graph replay with new cells, shards, both MLP launches, status words, the 3 x bf16 build
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n_conf", [3, 70], ids=["chained", "resident"])
def test_graph_replay_shards_and_mlp_launches(n_conf):
    model, _ = model_for("cell_list")
    base = model.engine(torch.device(DEV))
    eager = eager_engine(base)
    graphed = eager_engine(base, cuda_graph=True)
    sp, co, cell = golden_batch("water30_pbc_ani2x", n_conf, seed=71)
    strains = [np.eye(3) * (1.0 + 0.03 * np.sin(c)) for c in range(n_conf)]
    sp, co, cells = dev(*strained(sp, co, cell, strains))
    n = sp.numel()
    assert graphed._use_resident_mlp(n, True) == (n_conf == 70)

    def clone(res):
        return res.energies.clone(), res.grad.clone(), res.atomic_energies.clone(), res.virial.clone()

    ref = clone(eager.step(sp, co, cells, True, want_virial=True, check=True))
    for _ in range(graphed.graph_after + 2):     # eager uses, capture, replay
        got = clone(graphed.step(sp, co, cells, True, want_virial=True, check=True))
    assert len(graphed._graphs) == 1
    assert torch.equal(got[2], ref[2]) and torch.allclose(got[0], ref[0], rtol=1e-12, atol=0)
    assert (got[1] - ref[1]).abs().max() < 1e-6
    # new cells (and the coordinates with them) between replays: the captured graph reads them, no recapture
    cells2 = cells * torch.tensor([1.02, 0.99, 1.01], device=DEV).view(1, 3, 1)
    co2 = torch.stack([co[c] @ torch.linalg.inv(cells[c]) @ cells2[c] for c in range(n_conf)])
    ref2 = clone(eager.step(sp, co2, cells2, True, want_virial=True, check=True))
    got2 = clone(graphed.step(sp, co2, cells2, True, want_virial=True, check=True))
    assert len(graphed._graphs) == 1
    assert not torch.equal(got2[0], got[0])
    assert torch.equal(got2[2], ref2[2]) and torch.allclose(got2[0], ref2[0], rtol=1e-12, atol=0)
    assert (got2[1] - ref2[1]).abs().max() < 1e-6
    assert torch.allclose(got2[3], ref2[3], rtol=1e-5, atol=1e-6 * float(ref2[3].abs().max()))
    # shards (rank, world): partial results summed over the ranks
    for world in (2, 3):
        e_sum = torch.zeros_like(ref[0])
        g_sum = torch.zeros_like(ref[1])
        for rank in range(world):
            res = eager.step(sp, co, cells, True, shard=(rank, world), check=True)
            e_sum += res.energies
            g_sum += res.grad
        assert (g_sum - ref[1]).abs().max() < 1e-6, world
        assert torch.allclose(e_sum, ref[0], rtol=1e-12, atol=1e-9), world


@pytest.mark.gpu
def test_status_words():
    model, _ = model_for("cell_list")
    base = model.engine(torch.device(DEV))
    small = eager_engine(base, nbr_cap=32)
    sp, co, cell = golden_batch("water30_pbc_ani2x", 3, seed=81)
    sp, co, cells = dev(*strained(sp, co, cell, [np.eye(3) * s for s in (1.0, 1.02, 0.98)]))
    sp[0, 6:] = -1            # sparse conformers: few neighbours, within nbr_cap = 32
    sp[2, 6:] = -1
    small.step(sp[[0, 2]], co[[0, 2]], cells[[0, 2]], True, check=True)
    with pytest.raises(RuntimeError, match="nbr_cap"):
        small.step(sp, co, cells, True, check=True)               # conformer 1 overflows inside the batch
    thin = cells.clone()
    thin[1] = torch.tensor([[4.2, 0.0, 0.0], [0.3, 3.9, 0.0], [0.0, 0.2, 9.0]], device=DEV)
    with pytest.raises(RuntimeError, match="Cell is too small"):
        base.step(sp, co, thin, True, check=True)
    with pytest.raises(RuntimeError, match="Cell is too small"):   # the model too: no supercell route per conformer
        model_for("all_pairs")[0]((sp, co), thin, PBC.to(DEV))
    ws = base.workspace(3, sp.shape[1])
    ws.make_periodic()
    with pytest.raises(ValueError, match="reuse"):
        base.run(ws, True, reuse=True, conformer_cells=True)


@pytest.mark.gpu
def test_bf16x3_build():
    """One batch on the 3 x bf16 build, reached through the operand-range fallback of models.ANI."""
    from torchani_b200 import _lib, models
    if not _lib.available("bf16x3"):
        pytest.skip("the 3 x bf16 build is not built")
    om = model_for("cell_list")[1]
    w32 = [{s: [(w.float(), b.float()) for w, b in layers] for s, layers in wm.items()} for wm in om.weights]
    model = models.from_weight_lists("2x", w32, device=DEV, neighborlist="cell_list", periodic_table_index=False)
    sp, co, cells = batch("orthorhombic")
    spd, cod, celld = dev(sp, co, cells)
    calls = []
    orig = model.engine

    def engine(device):   # the first step reports an operand-range overflow, as a too-large value would
        eng = orig(device)
        if not calls:
            calls.append(1)

            def overflow(*a, **k):
                del eng.step
                raise _lib.OperandRangeError("test")
            eng.step = overflow
        return eng
    model.engine = engine
    with pytest.warns(UserWarning, match="bfloat16"):
        e64 = model.energies_f64((spd, cod), celld, PBC.to(DEV))
    assert model.neural_networks._variant == "bf16x3"
    e, f = model.energies_and_forces(spd, cod, celld, PBC.to(DEV))
    c32, co32 = celld.double().cpu(), cod.double().cpu()
    for k in range(sp.shape[0]):
        ref = orc.compute(om, sp[k:k + 1], co32[k:k + 1], c32[k], PBC)
        assert abs(float(e64[k]) - float(ref["energy"][0])) < 5e-3, k
        assert_close(f"bf16x3 [{k}] forces", f[k:k + 1].cpu().numpy(), ref["forces"].numpy(), 0.0, F_ATOL)


# ------------------------------------------------------------------------------------------------------------------
# 5. the batched host calculator
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["per_conformer", "shared"])
def test_host_calculator_batch(kind):
    from torchani_b200.calculator import HostCalculator
    model, _ = model_for("cell_list")
    sp, co, cells = batch("orthorhombic")
    if kind == "shared":
        cells = cells[:1].expand(sp.shape[0], 3, 3).contiguous()
    spd, cod, celld = dev(sp, co, cells)
    cell_arg = celld.cpu().numpy() if kind == "per_conformer" else celld[0].cpu().numpy()
    calc = HostCalculator(model, sp.numpy(), cell=cell_arg, pbc=True)
    e_ref, f_ref, s_ref = model.energies_forces_stress(spd, cod, celld if kind == "per_conformer" else celld[0],
                                                        PBC.to(DEV))
    e, f, s = calc.calculate_with_stress(cod.cpu().numpy())
    assert e.shape == (sp.shape[0],) and e.dtype == np.float64 and f.shape == tuple(co.shape)
    assert np.allclose(e, e_ref.cpu().numpy(), rtol=1e-12, atol=0)
    assert np.abs(f - f_ref.cpu().numpy()).max() < 1e-5
    assert np.allclose(s, s_ref.cpu().numpy(), rtol=1e-6, atol=1e-10)
    # new cells on every call, through the eager steps, the capture and the replays
    for it in range(calc.graph_after + 3):
        scale = torch.tensor([1.0 + 0.01 * it, 1.0, 1.0 - 0.005 * it], device=DEV).view(1, 3, 1)
        cells_i = celld * scale
        co_i = torch.stack([cod[c] @ torch.linalg.inv(celld[c]) @ cells_i[c] for c in range(sp.shape[0])])
        arg = cells_i.cpu().numpy() if kind == "per_conformer" else cells_i[0].cpu().numpy()
        e, f = calc.calculate(co_i.cpu().numpy(), cell=arg)
        e_ref, f_ref = model.energies_and_forces(spd, co_i, cells_i if kind == "per_conformer" else cells_i[0],
                                                 PBC.to(DEV))
        assert np.allclose(e, e_ref.cpu().numpy(), rtol=1e-12, atol=0), it
        assert np.abs(f - f_ref.cpu().numpy()).max() < 1e-5, it
    assert len(calc._graphs) == 1


# ------------------------------------------------------------------------------------------------------------------
# 6. rejected inputs
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_rejections():
    from torchani_b200 import _lib, neighbors
    from torchani_b200.aev import AEVComputer
    from torchani_b200.calculator import HostCalculator
    model, _ = model_for("cell_list")
    sp, co, cells = dev(*batch("cubic"))
    pbcd = PBC.to(DEV)
    with pytest.raises(ValueError, match="one cell per conformer"):
        model((sp, co), cells[:3], pbcd)                                   # C != batch size
    with pytest.raises(ValueError, match="one cell per conformer"):
        model.engine(torch.device(DEV)).step(sp, co, cells[:2], True)
    with pytest.raises(ValueError, match="all three directions"):
        model((sp, co), cells, torch.tensor([True, True, False], device=DEV))
    with pytest.raises(ValueError, match="models.ANI only"):
        AEVComputer.like_2x().to(DEV)(sp, co, cells, pbcd)
    with pytest.raises(ValueError, match="models.ANI only"):
        neighbors.AllPairs()(5.2, sp, co, cells, pbcd)
    with pytest.raises(ValueError, match="models.ANI only"):
        neighbors.cell_list(5.2, sp[:1], co[:1], cells[:1], pbcd)
    with pytest.raises(ValueError, match="no skin"):
        HostCalculator(model, sp.cpu().numpy(), cell=cells.cpu().numpy(), pbc=True, skin=0.5)
    with pytest.raises(ValueError, match="no skin"):
        HostCalculator(model, sp.cpu().numpy(), cell=cells.cpu().numpy(), pbc=True, sharded=object())
    # the C-ABI: mode 3 only through the entry points that take the lattice table
    L = _lib.lib()
    buf = torch.zeros(1 << 16, dtype=torch.int32, device=DEV)
    q = buf.data_ptr()
    st = torch.cuda.current_stream().cuda_stream
    assert L.ani_b200_build_cells(q, q, 4, 10, q, 1, 3, 5.1, 1000, q, q, q, q, q, q, q, q, q, st) == -2
    args = (q, q, 4, 10, q, 1, 3, 5.1, 1000, q, q, q, q, q, q, q, 0, 40, 4, 256, q, q, q, q, 16, 32, 384, 416, 0, q,
            None, 0, None, 0, None, q, q)
    assert L.ani_b200_prepare_step(*args, st) == -2
    assert L.ani_b200_prepare_step_cells(*args, None, st) == -1
    a2 = list(args)
    a2[6] = 2
    assert L.ani_b200_prepare_step_cells(*a2, q, st) == -2
    p = model.aev_computer._params()
    assert L.ani_b200_aev_forward_cells(C.byref(p), q, q, q, q, None, None, None, 40, 0, 40, q, q, 416, 0, q, q, 128,
                                        q, None, st) == -1
    assert L.ani_b200_aev_backward_cells(C.byref(p), q, q, q, None, 40, 0, 40, q, q, 416, q, q, 128, q, q, 0, None,
                                         None, st) == -1
    torch.cuda.synchronize()
    assert int(buf.abs().sum()) == 0
