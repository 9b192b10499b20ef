"""The Lennard-Jones and fixed-charge Coulomb pair potentials in the fused step (ani_b200_pair_potential_search,
csrc/pair.cu) against float64.

The kernel runs as ``test_gpu_pair_potentials.pair_only`` runs the repulsion kernel: the step's preparation and AEV
forward, then the term into zeroed outputs, on engines with tiny synthetic networks (``test_gpu_aev.tiny_weights``).
The reference is ``oracle/lj_coulomb_oracle.py`` in float64 on the float32-rounded inputs (periodic ones wrapped into
the cell), on every case of the golden fixtures of oracle/make_lj_coulomb_golden.py and on the cases below; the bars are those of ``test_gpu_step_terms``: atomic
1e-5 |e| + 1e-6 Ha, forces 1e-5 |F| + 1e-4 Ha/A, conformer energies 1e-6 |E| + 1e-5 Ha, stress 1e-5 |s| + 1e-5 max
|s|.  Covered: each kind, grid modes 0-3 and the triclinic 6W8H box, 8 / 12 A and no cutoff, both envelopes, the
query-by-committee members, a shard, a Verlet skin across a rebuild, eager runs and graph replay, xTB through the
search against xTB over the AEV's neighbour words, two new terms with xTB and D3 in one model, unchanged launch counts
without the new kinds, and a cell 0.01 A thinner than cutoff + skin.  The module prints the worst error / bar of every
group at its end (pytest -s).

Measured on an H100 80GB HBM3 (700 W power limit), worst error / bar: fixture cases LJ 0.48, RepulsionLJ 0.42,
DispersionLJ 0.23, FixedCoulomb 0.21, FixedMNOK 0.22; periodic batches 0.10-0.45; model (eager, graph replay, members,
stress) 0.45; no cutoff 0.10; shard 0.09; Verlet skin 0.76; xTB search / words 0.17.  About 37 s.
"""
import ctypes
import math
import typing as tp

import numpy as np
import pytest
import torch

import oracle.ani_oracle as orc
import oracle.lj_coulomb_oracle as lorc
import test_gpu_step_terms as tst
from helpers import E_RTOL, F_ATOL, GOLD, golden_inputs, load_golden

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F_RTOL = 1e-5
SYSTEMS = ["water999_pbc_ani2x", "1c17_chunk_hcnos_ani2x", "randbatch_ani2x", "6w8h_triclinic_ani2x"]
SYM = orc.SYMBOLS_2X
_cache: tp.Dict[tp.Any, tp.Any] = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    tst._WORST.clear()   # (tst.close notes the worst error / bar of every group there)
    yield
    if tst._WORST:
        print("\nworst error / bar of test_gpu_long_range_pairs.py:")
        for k in sorted(tst._WORST):
            print(f"  {k:28s} {tst._WORST[k]:.3f}")


def params():
    return dict(np.load(f"{GOLD}/ljc_params.npz"))


def term(kind: str, cutoff: float, fn: str):
    """The CUDA module of a fixture case, with the fixture's parameters."""
    from torchani_b200 import potentials as P
    p = params()
    eps, sigma, q, eta = ([float(v) for v in p[k]] for k in ("eps", "sigma", "charges", "eta"))
    kw = dict(cutoff=cutoff, cutoff_fn="smooth" if fn == "dummy" else fn)
    if kind in ("lj", "rep_lj", "disp_lj"):
        return getattr(P, lorc.CLASSES[kind])(SYM, eps, sigma, **kw)
    if kind == "coulomb":
        return P.FixedCoulomb(SYM, float(p["dielectric"]), q, **kw)
    return P.FixedMNOK(SYM, float(p["dielectric"]), q, eta, **kw)


def engine(key, pots, members: int = 1, skin: float = 0.0):
    from torchani_b200.engine import AEVConstants, Engine, PackedNetworks
    from test_gpu_aev import tiny_weights
    if key not in _cache:
        consts = AEVConstants(*orc.aev_spec_2x(7))
        symbols, w = tiny_weights(7, consts.out_dim)
        nets = PackedNetworks([[wm[s] for s in symbols] for wm in w] * members, consts.out_dim, torch.device(DEV),
                              radial_len=consts.radial_len)
        _cache[key] = Engine(consts, nets, nbr_cap=128, cuda_graph=False, pairs=[p.params() for p in pots])
    eng = _cache[key]
    eng.skin = skin
    return eng


def dev(t):
    return t.to(DEV)


def search_only(eng, sp, co, cell, pbc, want_virial=False, shard=(0, 1)):
    """The search launches of the engine on their own, into zeroed outputs (as tpp.pair_only)."""
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
        eng._search_pairs(ws, lo, hi, lat, ws.grad_ptr, ptr(ws.virial) if want_virial else None, None, run)
        torch.cuda.synchronize()
        eng.check_status(ws)
    out = {"energy": ws.energies.cpu().numpy().copy(), "atomic": ws.atomic.view(sp.shape).double().cpu().numpy(),
           "forces": -ws.grad.view(sp.shape + (3,)).double().cpu().numpy(),
           "member_atomic": ws.member_atomic.view((-1,) + sp.shape).double().cpu().numpy()}
    if want_virial:
        out["virial"] = ws.virial.view(sp.shape[0], -1, 9).sum(1).view(-1, 3, 3).cpu().numpy()
    return out, ws


def check(group, tag, got, ref, cell=None):
    if cell is not None and "virial" in got:
        vol = torch.det(cell.double().view(-1, 3, 3)).abs().numpy().reshape(-1, 1, 1)
        got = dict(got, stress=got["virial"] / vol)
    ref = dict(ref)
    if "stress" in ref and ref["stress"].ndim == 2:
        ref["stress"] = ref["stress"][None]
    tst.check_pair(group, tag, got, ref)


def fixture_cases(name: str):
    z = np.load(f"{GOLD}/ljc_{name}.npz")
    keys = sorted({k.rsplit("_", 1)[0] for k in z.files})
    out = []
    for key in keys:
        kind = next(kd for kd in sorted(lorc.KINDS, key=len, reverse=True) if key.startswith(kd + "_"))
        fn, cut = key[len(kind) + 1:].split("_")
        out.append((kind, math.inf if cut == "inf" else float(cut), fn, key))
    return out


# ------------------------------------------------------------------------------------------------------------------
# 1. every fixture case: each kind, grid modes 0 / 1, the triclinic box, 8 / 12 A / no cutoff, both envelopes
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", SYSTEMS)
def test_kernel_vs_float64_on_fixture_cases(name):
    """Every case of the system's fixture, against the oracle on the float32-rounded inputs (the overlapping atoms of
    the golden boxes turn the rounding of the inputs into 1e-5 relative changes of an x^6 or x^12 term)."""
    s = tst.golden_sys(name)
    cases = fixture_cases(name)
    assert cases
    p = params()
    for kind, cutoff, fn, key in cases:
        pot = term(kind, cutoff, fn)
        eng = engine(("fixture", key), [pot])
        assert len(eng.search_pairs) == 1 and not eng.pairs
        got, _ = search_only(eng, s.species, s.coords, s.cell, s.pbc, want_virial=s.cell is not None)
        ref = tst.oracle([(lorc, lorc.spec_from_params(kind, cutoff, fn, p))], s, stress=s.cell is not None,
                         nl="cell_list" if s.cell is not None else "all_pairs")
        check(f"kernel {kind}", f"{name} {key}", got, ref, s.cell)


# ------------------------------------------------------------------------------------------------------------------
# 2. periodic batches (grid modes 2 and 3), against the oracle on float32 inputs
# ------------------------------------------------------------------------------------------------------------------
def water_batch(per_conformer: bool) -> tst.Sys:
    s = tst.golden_sys("water999_pbc_ani2x")
    g = torch.Generator().manual_seed(5)
    co = s.coords.repeat(2, 1, 1)
    co[1] += 0.05 * torch.randn(co[1].shape, generator=g, dtype=torch.float64)
    sp = s.species.repeat(2, 1).clone()
    sp[1, -4:] = -1
    cell = s.cell
    if per_conformer:
        t = torch.eye(3, dtype=torch.float64) * 1.03
        t[0, 1] = 0.06
        cell = torch.stack([s.cell, s.cell @ t])
        co[1] = co[1] @ t
    frac = co @ torch.inverse(cell if cell.dim() == 2 else cell[0])
    if per_conformer:
        frac[1] = co[1] @ torch.inverse(cell[1])
    cells = cell if cell.dim() == 3 else cell.expand(2, 3, 3)
    co = torch.stack([(frac[c] - frac[c].floor()) @ cells[c] for c in range(2)])
    return tst.Sys(sp, tst.f32(co), tst.f32(cell), tst.PBC3)


@pytest.mark.parametrize("per_conformer", [False, True], ids=["mode2", "mode3"])
@pytest.mark.parametrize("kind,cutoff,fn", [("lj", 8.0, "cosine"), ("coulomb", 12.0, "smooth"),
                                            ("mnok", 8.0, "smooth")])
def test_periodic_batches(per_conformer, kind, cutoff, fn):
    s = water_batch(per_conformer)
    pot = term(kind, cutoff, fn)
    eng = engine(("batch", kind, cutoff, fn), [pot])
    got, _ = search_only(eng, s.species, s.coords, s.cell, s.pbc, want_virial=True)
    spec = lorc.spec_from_params(kind, cutoff, fn, params())
    ref = tst.oracle([(lorc, spec)], s, stress=True, nl="cell_list")
    check(f"batch {kind}", f"{kind} {'mode3' if per_conformer else 'mode2'}", got, ref, s.cell)


# ------------------------------------------------------------------------------------------------------------------
# 3. a shard, xTB through the search, the refusal of a thin cell
# ------------------------------------------------------------------------------------------------------------------
def test_shards_add_up():
    s = tst.golden_sys("water999_pbc_ani2x")
    eng = engine(("shard",), [term("coulomb", 12.0, "smooth")])
    parts = [search_only(eng, s.species, s.coords, s.cell, s.pbc, want_virial=True, shard=(r, 2))[0] for r in range(2)]
    got = {k: parts[0][k] + parts[1][k] for k in parts[0]}
    assert np.count_nonzero(parts[0]["atomic"]) and np.count_nonzero(parts[1]["atomic"])
    ref = tst.oracle([(lorc, lorc.spec_from_params("coulomb", 12.0, "smooth", params()))], s, stress=True,
                     nl="cell_list")
    check("shard", "coulomb 12 A", got, ref, s.cell)


def test_xtb_through_the_search_matches_the_neighbour_words():
    import test_gpu_pair_potentials as tpp
    from torchani_b200._lib import check as ck, ptr
    pot = tst.xtb_custom(7, cutoff=4.6)
    for name in ("water999_pbc_ani2x", "1c17_chunk_hcnos_ani2x", "randbatch_ani2x"):
        sp, co, cell, pbc = golden_inputs(load_golden(name))
        eng = engine(("xtb",), [pot])
        words = tpp.pair_only(eng, sp, co, cell, pbc, want_virial=cell is not None)
        ws = eng.workspace(*sp.shape)
        ws.atomic.zero_(), ws.energies.zero_(), ws.grad.zero_()
        p = pot.params()
        with torch.cuda.device(eng.device):
            ck(eng.lib.ani_b200_pair_potential_search(
                ctypes.byref(p), ptr(ws.grid), ptr(ws.bin_start), ptr(ws.spos), ptr(ws.sorted_orig), ws.n, 0, ws.n,
                ws.n_conf, ws.n_per_conf, 0.0, ptr(ws.atomic), ws.energies_ptr, ws.grad_ptr, None, None, None, None, 0,
                ptr(ws.status), torch.cuda.current_stream().cuda_stream), "pair_potential_search")
            torch.cuda.synchronize()
            eng.check_status(ws)
        srch = {"atomic": ws.atomic.view(sp.shape).double().cpu().numpy(), "energy": ws.energies.cpu().numpy(),
                "forces": -ws.grad.view(sp.shape + (3,)).double().cpu().numpy()}
        for k in srch:   # the same pairs in another order: float32 rounding apart
            scale = float(np.abs(words[k]).max())
            tst.close("xtb search/words", f"{name} {k}", srch[k], words[k], 2e-6, 1e-6 * scale + 1e-9)


def test_cell_thinner_than_cutoff_plus_skin_is_refused():
    pot = term("lj", 8.0, "smooth")
    skin = 0.5
    s = tst.box_sys(40, 8.0 + skin - 0.01, 7, seed=3, min_dist=1.2)
    eng = engine(("thin", skin), [pot], skin=skin)
    with pytest.raises(RuntimeError, match="Cell is too small"):
        search_only(eng, s.species, s.coords, s.cell, s.pbc)
    ws = eng.workspace(*s.species.shape)
    assert not bool(ws.atomic.any()) and not bool(ws.energies.any())   # nothing written
    s2 = tst.box_sys(40, 8.0 + skin + 0.01, 7, seed=3, min_dist=1.2)
    search_only(eng, s2.species, s2.coords, s2.cell, s2.pbc)
    eng.skin = 0.0


# ------------------------------------------------------------------------------------------------------------------
# 4. through the model: members, graph replay, launch counts, xTB + D3 + two new terms, a Verlet skin
# ------------------------------------------------------------------------------------------------------------------
def _model(potentials):
    from torchani_b200 import models
    base = models.ANI2x(seed=0)
    return models.ANI(base.symbols, base.aev_computer, base.neural_networks, base.energy_shifter, False,
                      potentials).to(DEV)


def oracle_terms(specs, s: tst.Sys):
    return tst.oracle([(lorc, sp) if isinstance(sp, lorc.Spec) else sp for sp in specs], s,
                      stress=False, nl="cell_list" if s.cell is not None else "all_pairs")


def test_model_terms_members_graphs_and_launches():
    s = tst.golden_sys("water999_pbc_ani2x")
    p = params()
    lj, cou = term("lj", 8.0, "cosine"), term("coulomb", 12.0, "smooth")
    xtb = tst.xtb_custom(7, cutoff=5.1)
    d3 = tst.d3_term(7, 8.0)
    plain = _model(None)
    full = _model({"xtb": xtb, "lj": lj, "coulomb": cou, "d3": d3})
    only_old = _model({"xtb": xtb, "d3": d3})
    sp, co, cell, pbc = dev(s.species), dev(s.coords).float(), dev(s.cell).float(), dev(s.pbc)
    e0, f0 = plain.energies_and_forces(sp, co, cell, pbc)
    eo, fo = only_old.energies_and_forces(sp, co, cell, pbc)
    eng_plain, eng_old = plain.engine(torch.device(DEV)), only_old.engine(torch.device(DEV))
    runs = []
    for _ in range(5):   # eager, then the captured graph replayed
        e1, f1 = full.energies_and_forces(sp, co, cell, pbc)
        runs.append((e1.clone(), f1.clone()))
    eng = full.engine(torch.device(DEV))
    assert len(eng._graphs) >= 1
    assert eng.launches_per_step == eng_old.launches_per_step + 2
    assert eng_old.launches_per_step == eng_plain.launches_per_step + 1 + 3 and not eng_old.search_pairs
    specs = [lorc.spec_from_params("lj", 8.0, "cosine", p), lorc.spec_from_params("coulomb", 12.0, "smooth", p)]
    ref = oracle_terms(specs, s)
    for tag, (e1, f1) in (("eager", runs[0]), ("graph replay", runs[-1])):
        tst.close("model", f"{tag} energy", (e1 - eo).cpu().numpy(), ref["energy"], 1e-6, 1e-5)
        tst.close("model", f"{tag} forces", (f1 - fo).double().cpu().numpy(), ref["forces"], F_RTOL, F_ATOL)
    # atomic energies and every query-by-committee member carry the terms
    a_full = full.atomic_energies((sp, co), cell, pbc, ensemble_values=True).energies
    a_old = only_old.atomic_energies((sp, co), cell, pbc, ensemble_values=True).energies
    for m in range(a_full.shape[0]):
        tst.close("model", f"member {m} atomic", (a_full[m] - a_old[m]).double().cpu().numpy()[None],
                  ref["atomic"], E_RTOL, 1e-5)
    mf_full = full.members_forces((sp, co), cell, pbc).forces
    mf_old = only_old.members_forces((sp, co), cell, pbc).forces
    for m in range(mf_full.shape[0]):
        tst.close("model", f"member {m} forces", (mf_full[m] - mf_old[m]).double().cpu().numpy(), ref["forces"],
                  F_RTOL, F_ATOL)
    # stress
    _, _, st_full = full.energies_forces_stress(sp, co, cell, pbc)
    _, _, st_old = only_old.energies_forces_stress(sp, co, cell, pbc)
    refs = tst.oracle([(lorc, sp_) for sp_ in specs], s, stress=True, nl="cell_list")
    tst.close("model", "stress", (st_full - st_old).cpu().numpy(), refs["stress"][0], 1e-5,
              1e-5 * float(np.abs(refs["stress"]).max()))


def test_model_no_cutoff_open_and_refused_periodic():
    s = tst.golden_sys("1c17_chunk_hcnos_ani2x")
    p = params()
    m = _model({"mnok": term("mnok", math.inf, "dummy")})
    base = _model(None)
    sp, co = dev(s.species), dev(s.coords).float()
    e1, f1 = m.energies_and_forces(sp, co)
    e0, f0 = base.energies_and_forces(sp, co)
    ref = oracle_terms([lorc.spec_from_params("mnok", math.inf, "dummy", p)], s)
    tst.close("no cutoff", "energy", (e1 - e0).cpu().numpy(), ref["energy"], 1e-6, 1e-5)
    tst.close("no cutoff", "forces", (f1 - f0).double().cpu().numpy(), ref["forces"], F_RTOL, F_ATOL)
    w = tst.golden_sys("water999_pbc_ani2x")
    with pytest.raises(ValueError, match="infinite cutoff"):
        m((dev(w.species), dev(w.coords).float()), dev(w.cell).float(), dev(w.pbc))
    eng = m.engine(torch.device(DEV))
    with pytest.raises(ValueError, match="infinite cutoff"):
        eng.step(dev(w.species), dev(w.coords).float(), dev(w.cell).float(), True)


def test_verlet_skin_across_a_rebuild():
    from torchani_b200.calculator import HostCalculator
    s = tst.golden_sys("water999_pbc_ani2x")
    p = params()
    m = _model({"lj": term("lj", 8.0, "smooth")})
    base = _model(None)
    spec = lorc.spec_from_params("lj", 8.0, "smooth", p)
    numbers = s.species[0].numpy()   # element indices: the models take them (periodic_table_index=False)
    calc = HostCalculator(m, numbers, s.cell.float(), pbc=True, skin=1.0)
    calc0 = HostCalculator(base, numbers, s.cell.float(), pbc=True)
    g = np.random.default_rng(0)
    x = s.coords[0].numpy().copy()
    frac_cell = s.cell.numpy()
    for step, amp in enumerate([0.0, 0.05, 0.05, 0.6, 0.05]):   # the 0.6 A move forces a rebuild
        x = x + g.normal(0.0, amp / 3, x.shape) if amp else x
        xf = np.float32(x).astype(np.float64)
        frac = xf @ np.linalg.inv(frac_cell)
        xw = np.float32((frac - np.floor(frac)) @ frac_cell).astype(np.float64)
        e1, f1 = calc.calculate(np.float32(xw))
        e0, f0 = calc0.calculate(np.float32(xw))
        ss = tst.Sys(s.species, torch.tensor(xw).view(1, -1, 3), s.cell, s.pbc)
        ref = oracle_terms([spec], ss)
        tst.close("skin", f"step {step} energy", np.atleast_1d(float(e1) - float(e0)), ref["energy"], 1e-6, 1e-5)
        tst.close("skin", f"step {step} forces", (np.asarray(f1, np.float64) - np.asarray(f0, np.float64))[None],
                  ref["forces"], F_RTOL, F_ATOL)
    assert calc.redone >= 1   # the large move was recomputed on a rebuilt grid
