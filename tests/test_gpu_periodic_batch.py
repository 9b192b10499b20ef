"""Periodic batches (grid mode 2): C conformers in one shared periodic cell, evaluated in ONE step.

Every conformer gets its own sub-grid of the shared cell, numbered conformer-major (bucket c * nb + local), with the
bucket capacity of a single-system workspace of its atoms.  A conformer's sub-grid, wrapped positions and (species,
input index) order are then those of a single-system preparation of that conformer alone, and everything downstream
without atomics is bit-identical per conformer.  Checked here: the preparation outputs in every form against
single-system preparations, the AEVs bit for bit against per-conformer AEVs (every AEV kernel path), the half
neighbour list against the concatenation of per-conformer lists, energies / forces / ensemble statistics against the
float64 oracle and per-conformer steps, one engine step per module call, graph replay, shards, the per-conformer
virial and the status words.  The five-launch preparation and the warp-per-atom / TMA-staged AEV kernels are chosen
once per process, so the file re-runs its own preparation and AEV tests in child processes for them.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import oracle.ani_oracle as orc
from helpers import (AEV_ATOL, AEV_RTOL, E_ATOL, E_RTOL, F_ATOL, assert_close, golden_inputs, load_golden,
                     oracle_model)
from test_gpu_aev import live_blocks, skewed_cell_system
from test_gpu_prepare import (MAX_SPECIES, ROOT, SENT, Problem, Run, env, in_cell, layout_ref, same_outputs, water)

DEV = "cuda:0"
ERR_UNSUPPORTED = -2
PBC = torch.tensor([True, True, True])


# ------------------------------------------------------------------------------------------------------------------
# batches
# ------------------------------------------------------------------------------------------------------------------
class Batch(Problem):
    """A Problem of n_conf conformers in one shared cell (grid mode 2)."""

    @property
    def mode(self) -> int:
        return 2

    @property
    def bins(self) -> int:
        # every conformer gets the bucket capacity of a single-system workspace of its atoms
        return self.max_bins or self.n_conf * (max(64, self.n_per_conf + 2) - 1) + 1


def replicate(xyz: np.ndarray, sp: np.ndarray, n_conf: int, seed: int, noise: float = 0.05):
    """n_conf seeded perturbations of one conformer -> (C, A, 3) float64, (C, A) int32."""
    rng = np.random.default_rng(seed)
    co = np.stack([xyz.astype(np.float64) + (noise * rng.standard_normal(xyz.shape) if c else 0.0)
                   for c in range(n_conf)])
    return co, np.tile(sp.astype(np.int32), (n_conf, 1))


def batch_problem(name: str) -> Batch:
    if name == "water_c2_1x1x1":
        xyz, sp, cell = water(10, seed=1)
        co, spc = replicate(xyz, sp, 2, seed=2)
        return Batch(name, co.reshape(-1, 3).astype(np.float32), spc.reshape(-1), cell, 4, n_conf=2)
    if name == "water_c7_3x3x3":
        xyz, sp, cell = water(150, seed=4)
        co, spc = replicate(xyz, sp, 7, seed=5)
        spc[3] = -1                                          # a conformer that is entirely padding
        c64 = cell.astype(np.float64)
        co[5, 0] = 0.0                                       # on cell faces and corners, and outside the cell
        co[5, 1] = c64[0]
        co[5, 2] = 0.5 * c64[1] + c64[2]
        co[5, 3] += 2 * c64[0] - 3 * c64[2]
        co[5, 4] -= c64[1]
        spc[6, ::9] = -1                                     # padding between real atoms
        spc[6, 1] = 1                                        # an element only this conformer has
        return Batch(name, co.reshape(-1, 3).astype(np.float32), spc.reshape(-1), cell, 4, n_conf=7)
    if name == "skewed_c64":
        s = skewed_cell_system()
        co, spc = replicate(s.coords[0].numpy(), s.species[0].numpy(), 64, seed=6, noise=0.02)
        return Batch(name, co.reshape(-1, 3).astype(np.float32), spc.reshape(-1), s.cell.numpy(), 7, n_conf=64)
    if name == "dilute_c3_capacity":
        cell = np.eye(3) * 60.0                              # 11^3 buckets wanted, 63 per conformer available
        xyz = in_cell(cell, 20, seed=17, min_dist=2.0, faces=[(0, 0, 0), (0.5, 0.5, 1.0)])
        co, spc = replicate(xyz, (np.arange(20) % 3).astype(np.int32), 3, seed=8, noise=0.3)
        return Batch(name, co.reshape(-1, 3).astype(np.float32), spc.reshape(-1), cell.astype(np.float32), 3,
                     n_conf=3)
    raise KeyError(name)


BATCHES = ["water_c2_1x1x1", "water_c7_3x3x3", "skewed_c64", "dilute_c3_capacity"]


def single(p: Batch, c: int) -> Problem:
    """Conformer c of a batch as a single system (mode 0) with the engine's capacity for it."""
    a = p.n_per_conf
    return Problem(f"{p.name}[{c}]", p.coords[c * a:(c + 1) * a], p.species[c * a:(c + 1) * a], p.cell, p.S)


# ------------------------------------------------------------------------------------------------------------------
# 1. preparation
# ------------------------------------------------------------------------------------------------------------------
def check_against_singles(r: Run, singles) -> None:
    """Every conformer's slice of the batch outputs, mapped back by its bases, bit for bit a single-system
    preparation; the batch-wide outputs (padding, row layout, live blocks, zero-fills) against the restatement."""
    p, o = r.p, r.o
    name = f"{p.name} / {r.form}"
    A, n = p.n_per_conf, p.n
    gd = r.grid()
    nb = int(np.prod(gd["dims"]))
    nbins = p.n_conf * nb
    real = p.species >= 0
    n_real = int(real.sum())
    assert (gd["mode"], gd["nbins"], gd["n_per_conf"], gd["n_real"], gd["pbc"]) == (2, nbins, A, n_real, 1), name
    assert nbins <= p.bins - 1, name
    bs, so, sbin = o["bin_start"], o["sorted_orig"], o["sbin"]
    spos = o["spos"].reshape(n, 4)
    rng = o["ranges"].reshape(-1, 27, 8)
    for c, s in enumerate(singles):
        off, end = int(bs[c * nb]), int(bs[(c + 1) * nb])
        if s is None:                                      # an all-padding conformer owns no atom
            assert end == off and not real[c * A:(c + 1) * A].any(), name
            continue
        tag = f"{name}, conformer {c}"
        g0 = s.grid()
        m = g0["n_real"]
        assert g0["dims"] == gd["dims"], (tag, g0["dims"], gd["dims"])
        assert (o["grid"][:21] == s.o["grid"][:21]).all(), f"{tag}: cell / inverse / origin"
        assert end - off == m, tag
        assert (bs[c * nb:(c + 1) * nb + 1] - off == s.o["bin_start"][:nb + 1]).all(), f"{tag}: bin_start"
        assert (so[off:end] - c * A == s.o["sorted_orig"][:m]).all(), f"{tag}: sorted_orig"
        assert (sbin[off:end] - c * nb == s.o["sbin"][:m]).all(), f"{tag}: sbin"
        assert (spos[off:end] == s.o["spos"].reshape(-1, 4)[:m]).all(), f"{tag}: spos"
        t, t0 = rng[c * nb:(c + 1) * nb], s.o["ranges"].reshape(-1, 27, 8)[:nb]
        assert (t[..., 0] - off == t0[..., 0]).all() and (t[..., 1] - off == t0[..., 1]).all(), f"{tag}: ranges"
        assert (t[..., 2] == t0[..., 2]).all() and (t[..., 4:] == t0[..., 4:]).all(), f"{tag}: ranges"
        if r.form == "build_cells":
            assert (t[..., 3] == 0).all(), tag
        else:
            assert (t[..., 3] - c * nb == t0[..., 3]).all(), f"{tag}: neighbour bucket word"
            assert (o["bss"].reshape(-1, MAX_SPECIES)[c * nb:(c + 1) * nb] ==
                    s.o["bss"].reshape(-1, MAX_SPECIES)[:nb]).all(), f"{tag}: bucket_species"
    # documented sizes: nothing written beyond the buckets in use (the guard bands are checked by Run)
    assert (bs[nbins + 2:] == SENT).all() and (rng[nbins:] == SENT).all(), name
    assert bs[nbins] == n_real and bs[nbins + 1] == n, name
    assert set(so[n_real:].tolist()) == set(np.nonzero(~real)[0].tolist()), name
    assert (sbin[n_real:] == nbins).all() and (o["spos"].view(np.float32).reshape(n, 4)[n_real:, :3] == 0).all(), name
    sw = spos[:, 3]
    lo, hi = p.slice
    lay = layout_ref(sw, n_real, lo, hi, p.S, r.rows_cap)
    assert (o["row_of"][lay.owned] == lay.row_of).all() and (o["row_atom"] == lay.row_atom).all(), f"{name}: rows"
    assert (o["tile_species"] == lay.tile_species).all(), name
    assert (o["layout_info"][:13] == lay.info).all(), name
    spec, pad, ldx = r.shape
    mask = int(np.bitwise_or.reduce(1 << p.species[real], initial=0))    # the union over the batch
    ids = live_blocks(spec, pad, mask, ldx)
    blk = o["aev_blocks"]
    assert blk[0] == len(ids) and blk[1:1 + len(ids)].tolist() == ids and blk[ldx // 32 + 1] == mask, name
    if r.form != "build_cells":
        assert (o["bss"].reshape(-1, MAX_SPECIES)[nbins:] == SENT).all(), name
        assert (o["zero_f32"] == 0).all() and (o["zero_f64"] == 0).all(), name


def singles_of(p: Batch, form: str):
    out = []
    for c in range(p.n_conf):
        s = single(p, c)
        out.append(None if (s.species < 0).all() else Run(s, form))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", BATCHES)
def test_prep_contract(name):
    p = batch_problem(name)
    with env(ANI_B200_PREP_CLUSTER=0):      # (mode 0 references through the same kernel as the batch)
        runs = [Run(p, "prepare_step"), Run(p, "build_cells")]
        refs = {"prepare_step": singles_of(p, "prepare_step"), "build_cells": singles_of(p, "build_cells")}
    for r in runs:
        check_against_singles(r, refs[r.form])
    same_outputs(runs[0], runs[1])


@pytest.mark.gpu
def test_prep_argument_checks():
    """mode 2 needs pbc, a cell and n_conf + 1 <= max_bins; refused before any CUDA call."""
    from torchani_b200._lib import lib
    L = lib()
    buf = torch.zeros(1 << 16, dtype=torch.int32, device=DEV)
    q = buf.data_ptr()
    st = torch.cuda.current_stream().cuda_stream
    for pbc, cell, n_conf, max_bins in ((0, q, 4, 1000), (1, None, 4, 1000), (1, q, 4, 4)):
        rc = L.ani_b200_build_cells(q, q, n_conf, 10, cell, pbc, 2, 5.1, max_bins, q, q, q, q, q, q, q, q, q, st)
        assert rc == ERR_UNSUPPORTED, (pbc, cell, max_bins, rc)
        rc = L.ani_b200_prepare_step(q, q, n_conf, 10, cell, pbc, 2, 5.1, max_bins, q, q, q, q, q, q, q, 0, 40, 4, 256,
                                     q, q, q, q, 16, 32, 384, 416, 0, q, None, 0, None, 0, None, q, q, st)
        assert rc == ERR_UNSUPPORTED, (pbc, cell, max_bins, rc)
    torch.cuda.synchronize()
    assert int(buf.abs().sum()) == 0


# ------------------------------------------------------------------------------------------------------------------
# 2. AEVs, 3. half neighbour list
# ------------------------------------------------------------------------------------------------------------------
def tensors(p: Batch):
    sp = torch.tensor(p.species, dtype=torch.long, device=DEV).view(p.n_conf, -1)
    co = torch.tensor(p.coords, device=DEV).view(p.n_conf, -1, 3)
    return sp, co, torch.tensor(p.cell, device=DEV)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["water_c7_3x3x3", "skewed_c64"])
def test_aev_bit_for_bit(name):
    """AEVComputer on the batch == per-conformer AEVs bit for bit; so is the AEV forward fed by the range table and the
    per-bucket species offsets of ani_b200_prepare_step; a few conformers against the float64 oracle."""
    from torchani_b200._lib import check, lib
    from torchani_b200.aev import AEVComputer
    p = batch_problem(name)
    sp, co, cell = tensors(p)
    comp = AEVComputer.like_2x(num_species=p.S).to(DEV)
    pbc = PBC.to(DEV)
    aev = comp(sp, co, cell, pbc)
    per = torch.cat([comp(sp[c:c + 1], co[c:c + 1], cell, pbc) for c in range(p.n_conf)])
    assert torch.equal(aev.view(torch.int32), per.view(torch.int32)), "batch AEVs differ from per-conformer AEVs"
    assert (aev.view(p.n, -1)[torch.tensor(p.species < 0, device=DEV)] == 0).all()
    # the ABI with the preparation's tables
    r = Run(p, "prepare_step", calls=1)
    b = r.b
    consts = comp.constants
    out_dim, cap = consts.out_dim, comp.nbr_cap
    for use_ranges, use_bss in ((True, True), (True, False), (False, False)):
        out = torch.zeros(p.n, out_dim, device=DEV)
        nbr_cnt = torch.zeros(p.n, dtype=torch.int32, device=DEV)
        nbr_list = torch.zeros(p.n * cap, dtype=torch.int32, device=DEV)
        status = torch.zeros(1, dtype=torch.int32, device=DEV)
        check(lib().ani_b200_aev_forward(
            C.byref(comp._params()), b["grid"].ptr, b["bin_start"].ptr, b["spos"].ptr, b["sbin"].ptr,
            b["ranges"].ptr if use_ranges else None, b["bss"].ptr if use_bss else None, None, p.n, 0, p.n,
            b["sorted_orig"].ptr, out.data_ptr(), out_dim, 0, nbr_cnt.data_ptr(), nbr_list.data_ptr(), cap,
            status.data_ptr(), torch.cuda.current_stream().cuda_stream), "aev_forward")
        torch.cuda.synchronize()
        assert int(status.item()) == 0
        assert torch.equal(out.view(torch.int32), aev.view(p.n, -1).view(torch.int32)), (use_ranges, use_bss)
    om = oracle_model("2x", torch.float64, "cell_list")
    c64 = torch.tensor(p.coords, dtype=torch.float64).view(p.n_conf, -1, 3)
    s64 = torch.tensor(p.species, dtype=torch.long).view(p.n_conf, -1)
    for c in (0, 1, p.n_conf - 1):
        if p.S == 7 and not (s64[c] < 0).all():
            ref = orc.compute(om, s64[c:c + 1], c64[c:c + 1], torch.tensor(p.cell, dtype=torch.float64), PBC,
                              forces=False)
            assert_close(f"aev {name}[{c}]", aev[c:c + 1].cpu().numpy(), ref["aev"].numpy(), AEV_RTOL, AEV_ATOL)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["water_c7_3x3x3", "skewed_c64"])
def test_half_list_is_the_concatenation(name):
    from torchani_b200 import neighbors
    p = batch_problem(name)
    sp, co, cell = tensors(p)
    pbc = PBC.to(DEV)
    nb = neighbors.AllPairs()(5.1, sp, co, cell, pbc)
    per = [neighbors.AllPairs()(5.1, sp[c:c + 1], co[c:c + 1], cell, pbc) for c in range(p.n_conf)]
    idx = torch.cat([q.indices + c * p.n_per_conf for c, q in enumerate(per)], 1)
    assert torch.equal(nb.indices, idx)
    assert torch.equal(nb.distances, torch.cat([q.distances for q in per]))
    assert torch.equal(nb.diff_vectors, torch.cat([q.diff_vectors for q in per]))


@pytest.mark.gpu
@pytest.mark.parametrize("var", ["ANI_B200_PREP_FUSED=0", "ANI_B200_AEV_LEGACY=1", "ANI_B200_AEV_TMA=1",
                                 "ANI_B200_AEV_BSS=1"])
def test_process_wide_variants(var):
    """The five-launch preparation, the warp-per-atom and TMA-staged AEV kernels and the engine's per-bucket species
    offsets are chosen once per process: re-run this file's preparation, AEV and engine tests in a child process."""
    k, v = var.split("=")
    child_env = dict(os.environ, **{k: v})
    sel = "prep_contract or aev_bit or graph_replay" if k != "ANI_B200_PREP_FUSED" else "prep_contract or aev_bit"
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
        "-m", "pytest", os.path.abspath(__file__), "-q", "-m", "gpu", "-k", sel, "-p", "no:cacheprovider"]
    res = subprocess.run(cmd, cwd=ROOT, env=child_env, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stdout[-4000:] + res.stderr[-2000:]
    assert " passed" in res.stdout and " failed" not in res.stdout


# ------------------------------------------------------------------------------------------------------------------
# 4.-5. the module API against the oracle, one engine step per call
# ------------------------------------------------------------------------------------------------------------------
_model_cache = {}


def model_for(neighborlist: str = "cell_list"):
    from torchani_b200 import models
    if neighborlist not in _model_cache:
        om = oracle_model("2x", torch.float64, neighborlist)
        w32 = [{s: [(w.float(), b.float()) for w, b in layers] for s, layers in wm.items()} for wm in om.weights]
        _model_cache[neighborlist] = models.from_weight_lists("2x", w32, device=DEV, neighborlist=neighborlist,
                                                              periodic_table_index=False)
    return _model_cache[neighborlist], oracle_model("2x", torch.float64, neighborlist)


def golden_batch(case: str, n_conf: int, seed: int, mixed: bool = True):
    """n_conf seeded perturbations of a golden periodic system; with `mixed`, conformer 1 carries an element no other
    conformer has and the last conformer is partly padding."""
    species, coords, cell, _ = golden_inputs(load_golden(case), torch.float64)
    g = torch.Generator().manual_seed(seed)
    co = coords.repeat(n_conf, 1, 1)
    co[1:] += 0.03 * torch.randn(co[1:].shape, generator=g, dtype=torch.float64)
    sp = species.repeat(n_conf, 1).clone()
    if mixed and n_conf > 2:
        present = set(species[species >= 0].tolist())
        absent = [e for e in range(7) if e not in present]
        if absent:
            sp[1, 0] = absent[0]
        sp[-1, -3:] = -1
    return sp, co, cell


class StepCounter:
    def __init__(self, eng):
        self.eng, self.calls, self._orig = eng, 0, eng.step

    def __enter__(self):
        def counted(*a, **k):
            self.calls += 1
            return self._orig(*a, **k)
        self.eng.step = counted
        return self

    def __exit__(self, *exc):
        del self.eng.step


def oracle_per_conf(om, sp, co, cell, pbc, **kw):
    return [orc.compute(om, sp[c:c + 1], co[c:c + 1], cell, pbc, **kw) for c in range(sp.shape[0])]


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["water30_pbc_ani2x", "benzene_pbc_ani2x", "tightcell_pbc_ani2x",
                                  "6w8h_triclinic_ani2x"])
def test_energies_forces_against_the_oracle(case):
    model, om = model_for("cell_list")
    sp, co, cell = golden_batch(case, 5, seed=11)
    refs = oracle_per_conf(om, sp, co, cell, PBC)
    spd, celld, pbcd = sp.to(DEV), cell.float().to(DEV), PBC.to(DEV)
    c = co.float().to(DEV).requires_grad_(True)
    eng = model.engine(torch.device(DEV))
    with StepCounter(eng) as cnt:
        e = model((spd, c), celld, pbcd).energies
    assert cnt.calls == 1, "a periodic batch must be one engine step"
    (g,) = torch.autograd.grad(e.sum(), c)
    at = model((spd, co.float().to(DEV)), celld, pbcd, atomic=True).energies
    ens = model((spd, co.float().to(DEV)), celld, pbcd, ensemble_values=True).energies
    # (the float32 energies of `forward` round |E| ~ 1.7e5 Ha to 0.016 Ha: the float64 sums of the device are compared)
    with StepCounter(eng) as cnt:
        e64 = model.energies_f64((spd, co.float().to(DEV)), celld, pbcd)
    assert cnt.calls == 1
    assert torch.allclose(e.detach().double(), e64, rtol=1e-7, atol=0)
    for k, ref in enumerate(refs):
        assert abs(float(e64[k]) - float(ref["energy"][0])) < 5e-3, (case, k)
        assert_close(f"{case}[{k}] forces", -g[k:k + 1].cpu().numpy(), ref["forces"].numpy(), 0.0, F_ATOL)
        sae = model.energy_shifter(spd[k:k + 1], atomic=True).cpu().double()
        assert_close(f"{case}[{k}] atomic", at[k:k + 1].cpu().numpy(), (ref["atomic_nn"] + sae).numpy(), E_RTOL,
                     E_ATOL)
    # per-conformer engine steps: the same model, one conformer at a time
    for k in range(sp.shape[0]):
        c1 = co[k:k + 1].float().to(DEV).requires_grad_(True)
        e1 = model((spd[k:k + 1], c1), celld, pbcd).energies
        (g1,) = torch.autograd.grad(e1.sum(), c1)
        at1 = model((spd[k:k + 1], co[k:k + 1].float().to(DEV)), celld, pbcd, atomic=True).energies
        ens1 = model((spd[k:k + 1], co[k:k + 1].float().to(DEV)), celld, pbcd, ensemble_values=True).energies
        assert_close(f"{case}[{k}] atomic vs single", at[k:k + 1].cpu().numpy(), at1.cpu().numpy(), 1e-6, 1e-7)
        assert_close(f"{case}[{k}] forces vs single", g[k:k + 1].cpu().numpy(), g1.cpu().numpy(), 0.0, 1e-5)
        assert_close(f"{case}[{k}] members vs single", ens[:, k].cpu().numpy(), ens1[:, 0].cpu().numpy(), 1e-6, 1e-6)
    # members_forces (one engine pass) against per-conformer calls
    e_m, f_m = model.members_forces((spd, co.float().to(DEV)), celld, pbcd)[1:]
    for k in range(sp.shape[0]):
        e1, f1 = model.members_forces((spd[k:k + 1], co[k:k + 1].float().to(DEV)), celld, pbcd)[1:]
        assert_close(f"{case}[{k}] member energies", e_m[:, k].cpu().numpy(), e1[:, 0].cpu().numpy(), 1e-6, 1e-6)
        assert_close(f"{case}[{k}] member forces", f_m[:, k].cpu().numpy(), f1[:, 0].cpu().numpy(), 0.0, 1e-5)


@pytest.mark.gpu
def test_partial_pbc_and_thin_cell_batches_are_one_pass():
    # PBC in two directions only
    model, om = model_for("all_pairs")
    sp, co, cell = golden_batch("water30_pbc_ani2x", 3, seed=12, mixed=False)
    pbc = torch.tensor([True, True, False])
    refs = oracle_per_conf(om, sp, co, cell, pbc)
    eng = model.engine(torch.device(DEV))
    c = co.float().to(DEV).requires_grad_(True)
    with StepCounter(eng) as cnt:
        e = model((sp.to(DEV), c), cell.float().to(DEV), pbc.to(DEV)).energies
    assert cnt.calls == 1
    (g,) = torch.autograd.grad(e.sum(), c)
    for k, ref in enumerate(refs):
        assert abs(float(e[k].detach()) - float(ref["energy"][0])) < 5e-3
        assert_close(f"slab forces [{k}]", -g[k:k + 1].cpu().numpy(), ref["forces"].numpy(), 0.0, F_ATOL)
    # a cell thinner than the cutoff on an all_pairs model: a supercell of every conformer within its own row
    gen = torch.Generator().manual_seed(4)
    thin = torch.tensor([[4.2, 0.0, 0.0], [0.3, 3.9, 0.0], [0.0, 0.2, 9.0]], dtype=torch.float64)
    sp = torch.tensor([[3, 0, 0, 1, 0, 2], [3, 0, 0, 1, 0, -1], [2, 2, 0, 1, 0, 3]])
    co = torch.rand(3, 6, 3, generator=gen, dtype=torch.float64) @ thin
    refs = oracle_per_conf(om, sp, co, thin, PBC)
    c = co.float().to(DEV).requires_grad_(True)
    with StepCounter(eng) as cnt:
        e = model((sp.to(DEV), c), thin.float().to(DEV), PBC.to(DEV)).energies
    assert cnt.calls == 1
    (g,) = torch.autograd.grad(e.sum(), c)
    for k, ref in enumerate(refs):
        assert abs(float(e[k].detach()) - float(ref["energy"][0])) < 2e-3
        assert_close(f"thin forces [{k}]", -g[k:k + 1].cpu().numpy(), ref["forces"].numpy(), 0.0, F_ATOL)
    at = model((sp.to(DEV), co.float().to(DEV)), thin.float().to(DEV), PBC.to(DEV), atomic=True).energies
    assert at.shape == (3, 6)
    # what raised before still raises: a cell-list model in a thin cell, a batch on the standalone cell list
    from torchani_b200 import neighbors
    strict, _ = model_for("cell_list")
    with pytest.raises(RuntimeError, match="too small"):
        strict((sp.to(DEV), co.float().to(DEV)), thin.float().to(DEV), PBC.to(DEV))
    with pytest.raises(ValueError, match="batches"):
        neighbors.cell_list(5.1, sp.to(DEV), co.float().to(DEV), thin.float().to(DEV), PBC.to(DEV))


# ------------------------------------------------------------------------------------------------------------------
# 6.-8. the engine: graph replay, shards, both MLP launches, virial, status words
# ------------------------------------------------------------------------------------------------------------------
def engine_inputs(n_conf: int, seed: int):
    sp, co, cell = golden_batch("water30_pbc_ani2x", n_conf, seed=seed)
    return sp.to(DEV), co.float().to(DEV), cell.float().to(DEV)


@pytest.mark.gpu
@pytest.mark.parametrize("n_conf", [3, 70], ids=["chained", "resident"])
def test_graph_replay_and_shards(n_conf):
    from torchani_b200.engine import Engine
    model, _ = model_for("cell_list")
    base = model.engine(torch.device(DEV))
    eager = Engine(base.consts, base.nets, base.sae.tolist(), nbr_cap=base.nbr_cap, cuda_graph=False)
    graphed = Engine(base.consts, base.nets, base.sae.tolist(), nbr_cap=base.nbr_cap, cuda_graph=True)
    sp, co, cell = engine_inputs(n_conf, seed=21)
    n = sp.numel()
    assert graphed._use_resident_mlp(n, True) == (n_conf == 70)

    def clone(res):
        return res.energies.clone(), res.grad.clone(), res.atomic_energies.clone()

    ref = clone(eager.step(sp, co, cell, True, check=True))
    for _ in range(graphed.graph_after + 2):     # eager uses, capture, replay
        got = clone(graphed.step(sp, co, cell, True, check=True))
    assert len(graphed._graphs) == 1
    assert torch.equal(got[2], ref[2]) and torch.allclose(got[0], ref[0], rtol=1e-12, atol=0)
    assert (got[1] - ref[1]).abs().max() < 1e-6
    # the composition changes between replays: an element appears in conformer 0
    sp2 = sp.clone()
    sp2[0, 0] = 4
    ref2 = clone(eager.step(sp2, co, cell, True, check=True))
    got2 = clone(graphed.step(sp2, co, cell, True, check=True))
    assert len(graphed._graphs) == 1
    assert torch.equal(got2[2], ref2[2]) and torch.allclose(got2[0], ref2[0], rtol=1e-12, atol=0)
    assert (got2[1] - ref2[1]).abs().max() < 1e-6
    # shards (rank, world): partial results summed over the ranks
    for world in (2, 3):
        e_sum = torch.zeros_like(ref[0])
        g_sum = torch.zeros_like(ref[1])
        for rank in range(world):
            res = eager.step(sp, co, cell, True, shard=(rank, world), check=True)
            e_sum += res.energies
            g_sum += res.grad
        assert (g_sum - ref[1]).abs().max() < 1e-6, world
        assert torch.allclose(e_sum, ref[0], rtol=1e-12, atol=1e-9), world


@pytest.mark.gpu
def test_virial_per_conformer():
    model, _ = model_for("cell_list")
    eng = model.engine(torch.device(DEV))
    sp, co, cell = engine_inputs(4, seed=31)
    res = eng.step(sp, co, cell, True, want_virial=True, check=True)
    vir = res.virial.clone()
    assert vir.shape == (4, 3, 3)
    volume = torch.det(cell.double()).abs()
    om = oracle_model("2x", torch.float64, "cell_list")
    cell64 = cell.double().cpu()
    for k in range(4):
        one = eng.step(sp[k:k + 1], co[k:k + 1], cell, True, want_virial=True, check=True).virial.clone()
        assert one.shape == (3, 3)
        assert_close(f"virial [{k}]", vir[k].cpu().numpy(), one.cpu().numpy(), 1e-6, 1e-6 * float(one.abs().max()))
        c64 = co[k:k + 1].double().cpu()
        wrapped = c64 - torch.floor(c64 @ torch.linalg.inv(cell64)) @ cell64
        ref = orc.compute(om, sp[k:k + 1].cpu(), wrapped, cell64, PBC, stress=True)
        assert_close(f"stress [{k}]", (vir[k] / volume).cpu().numpy(), ref["stress"].numpy(), 1e-4, 1e-8)
    # model level: (C, 3, 3) stress of a batch
    e, f, stress = model.energies_forces_stress(sp, co, cell, PBC.to(DEV))
    assert stress.shape == (4, 3, 3) and torch.allclose(stress, vir / volume, rtol=1e-5, atol=1e-10)


@pytest.mark.gpu
def test_status_words():
    from torchani_b200.engine import Engine
    model, _ = model_for("cell_list")
    base = model.engine(torch.device(DEV))
    small = Engine(base.consts, base.nets, None, nbr_cap=32, cuda_graph=False)
    sp, co, cell = engine_inputs(3, seed=41)
    sp[0, 6:] = -1            # a sparse conformer: few neighbours, within nbr_cap = 32
    sp[2, 6:] = -1
    small.step(sp[0:1], co[0:1], cell, True, check=True)      # fine on its own
    with pytest.raises(RuntimeError, match="nbr_cap"):
        small.step(sp[1:2], co[1:2], cell, True, check=True)  # overflows on its own ...
    with pytest.raises(RuntimeError, match="nbr_cap"):
        small.step(sp, co, cell, True, check=True)            # ... and inside the batch
    small.step(sp[[0, 2]], co[[0, 2]], cell, True, check=True)
    thin = torch.tensor([[4.2, 0.0, 0.0], [0.3, 3.9, 0.0], [0.0, 0.2, 9.0]], device=DEV)
    with pytest.raises(RuntimeError, match="Cell is too small"):
        base.step(sp, co, thin, True, check=True)
    ws = base.workspace(3, sp.shape[1])
    ws.make_periodic()
    with pytest.raises(ValueError, match="reuse"):
        base.run(ws, True, reuse=True)
