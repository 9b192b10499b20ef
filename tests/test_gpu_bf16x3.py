"""The 3 x bfloat16 build (libani_b200_bf16x3.so) end to end against float64, and the switch to it.

The 2 x fp16 operand format has a range limit (DESIGN.md section 3); when a value leaves it, the Python layer switches
the model to the 3 x bf16 build of the same sources and redoes the step.  That build is a second compilation of every
kernel: the AEV writer with three pieces and 24 KB K-blocks, the preparation, the AEV backward, the data-flow and
chained MLP launches (it has no resident launch).  It takes over exactly when inputs are extreme, so it is held to the
golden bars of tests/test_gpu_parity.py on its own:
* the tiled AEV operand the step writes, decoded, against plain AEV rows written with the step's own arguments (the
  same kernel path and order of additions) to 2^-24 relative: three bf16 pieces hold the whole float32 significand.
  With and without ``ang_pad``, on every AEV kernel path;
* AEV, member and atomic energies 1e-5 relative, forces 1e-4 Ha/A against the float64 oracle on every golden system,
  on both MLP launches and the independent-chain launch, a 256-conformer batch, a periodic batch, shards, graph replay
  (including a capture with two elements replayed with seven), the virial, ``step_members``, the smooth cutoff and an
  active-member subset;
* a model whose activations reach ~1e4 and gradients ~1e3, relative to the scale of the float64 result (the 2 x fp16
  build must flag the same model).

The switch: every model path, ``HostCalculator.calculate`` (with and without a Verlet skin, with the overflow
appearing only after the step's graph was captured), ``HostCalculator.calculate_with_stress`` and the ASE calculator
must switch once with a warning, give the oracle's results, and stay on the 3 x bf16 build.  A model whose head seed
is in range for the ensemble mean (member_scale = 1/M) but not for one member (member_scale = 1) switches in
``members_forces`` only.

NaN weights are not tested here: the 3 x bf16 build has no range check, so they give NaN energies without a status.
The module prints the worst error / bar of every group at its end (pytest -s).
"""
import os
import subprocess
import sys
import typing as tp
import warnings

import numpy as np
import pytest
import torch

import oracle.ani_oracle as orc
from helpers import (E_ATOL, E_RTOL, F_ATOL, GOLDEN_CASES, assert_close, golden_inputs, load_golden, oracle_model)

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VARIANT = "bf16x3"
PBC = torch.tensor([True, True, True])
_WORST: tp.Dict[str, float] = {}


def _note(group: str, ratio: float) -> None:
    _WORST[group] = max(_WORST.get(group, 0.0), ratio)


@pytest.fixture(scope="module", autouse=True)
def _needs_the_build():
    from torchani_b200 import _lib
    if not _lib.available(VARIANT):
        pytest.skip(f"{_lib.variant_path(VARIANT)} has not been built")
    yield
    if _WORST:
        print("\nworst error / bar of test_gpu_bf16x3.py:")
        for k in sorted(_WORST):
            print(f"  {k:36s} {_WORST[k]:.3e}")


def make_engine(kind: str = "2x", ang_pad: bool = False, cuda_graph: bool = True, members: int = 8, weights=None,
                variant: str = VARIANT):
    from torchani_b200.engine import Engine, PackedNetworks, constants_1x, constants_2x
    consts = constants_2x() if kind == "2x" else constants_1x()
    m = oracle_model(kind, members=members)
    w = m.weights if weights is None else weights
    nets = PackedNetworks([[wm[s] for s in m.symbols] for wm in w], consts.out_dim, torch.device(DEV),
                          variant=variant, radial_len=consts.num_species * len(consts.shf_r) if ang_pad else 0)
    return Engine(consts, nets, [m.sae[s] for s in m.symbols], cuda_graph=cuda_graph)


@pytest.fixture(scope="module")
def engines():
    return {"2x": make_engine("2x"), "1x": make_engine("1x")}


def compare(eng, species, coords32, cell32, pbc, model=None, tag: str = ""):
    """run_and_compare of test_gpu_parity (it also checks the tiled AEV operand against the plain rows), plus the
    worst ratios for the report."""
    from test_gpu_parity import gpu_aev, run_and_compare
    assert eng.variant == VARIANT
    kind = "2x" if eng.consts.num_species == 7 else "1x"
    if model is None:
        model = oracle_model(kind, torch.float64, "cell_list" if cell32 is not None else "all_pairs")
    ref, res = run_and_compare(eng, model, species, coords32, cell32, pbc)
    aev, _ = gpu_aev(eng, species, coords32, cell32, pbc)
    _note("aev", float(((aev.double() - ref["aev"]).abs() / (1e-5 * ref["aev"].abs() + 1e-5)).max()))
    ma = res.member_atomic.cpu().double()
    _note("member energies", float(((ma - ref["member_atomic"]).abs() / (E_RTOL * ref["member_atomic"].abs()
                                                                        + E_ATOL)).max()))
    _note("forces", float((-res.grad.cpu().double() - ref["forces"]).abs().max()) / F_ATOL)
    return ref, res


@pytest.mark.parametrize("mlp_mode", ["0", "1"], ids=["chained", "dataflow"])
@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_golden_cases(engines, name, mlp_mode):
    rec = load_golden(name)
    species, coords, cell, pbc = golden_inputs(rec, torch.float32)
    eng = engines[rec["kind"]]
    saved = eng.mlp_mode
    try:
        eng.mlp_mode = mlp_mode
        compare(eng, species, coords, cell, pbc, oracle_model(rec["kind"], torch.float64, rec["neighborlist"]))
    finally:
        eng.mlp_mode = saved


@pytest.mark.parametrize("name", ["water30_pbc_ani2x", "sevenel_pbc_ani2x", "1c17_chunk_hcnos_ani2x",
                                  "randbatch_ani2x"])
def test_ang_pad(name):
    """The angular block on a 32-column boundary of the tiled operand (the library's default packing)."""
    rec = load_golden(name)
    species, coords, cell, pbc = golden_inputs(rec, torch.float32)
    eng = make_engine(rec["kind"], ang_pad=True)
    assert eng.nets.col_pad == 16
    compare(eng, species, coords, cell, pbc, oracle_model(rec["kind"], torch.float64, rec["neighborlist"]))


@pytest.mark.parametrize("var", ["ANI_B200_AEV_LEGACY=1", "ANI_B200_AEV_TMA=1", "ANI_B200_AEV_BSS=1"])
def test_aev_kernel_paths(var):
    """The warp-per-atom, TMA-staged and per-bucket species offset AEV paths are chosen once per process: re-run a
    subset of this file in a child process."""
    k, v = var.split("=")
    env = dict(os.environ, **{k: v})
    sel = "(test_golden_cases and dataflow and (water30 or sevenel or randbatch or 6w8h)) or test_ang_pad"
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
        "-m", "pytest", os.path.abspath(__file__), "-q", "-m", "gpu", "-k", sel, "-p", "no:cacheprovider"]
    res = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stdout[-4000:] + res.stderr[-2000:]
    assert "8 passed" in res.stdout and " failed" not in res.stdout


@pytest.mark.parametrize("name", ["water999_pbc_ani2x", "sevenel_pbc_ani2x"])
def test_independent_chain_launch(name, monkeypatch):
    monkeypatch.setenv("ANI_B200_MLP_CHAIN", "1")
    rec = load_golden(name)
    species, coords, cell, pbc = golden_inputs(rec, torch.float32)
    eng = make_engine("2x", cuda_graph=False)
    eng.mlp_mode = "1"
    compare(eng, species, coords, cell, pbc, oracle_model("2x", torch.float64, rec["neighborlist"]))


def test_conformer_batch_256(engines):
    species, coords = orc.conformer_batch(256, seed=1234)
    compare(engines["2x"], species, coords, None, None, oracle_model("2x", torch.float64, "all_pairs"))


def test_periodic_batch(engines):
    from test_gpu_periodic_batch import golden_batch, oracle_per_conf
    eng = engines["2x"]
    sp, co, cell = golden_batch("water30_pbc_ani2x", 5, seed=11)
    co = co.float().double()
    refs = oracle_per_conf(oracle_model("2x", torch.float64, "cell_list"), sp, co, cell.float().double(), PBC)
    res = eng.step(sp.to(DEV), co.float().to(DEV), cell.float().to(DEV), True, check=True)
    for k, ref in enumerate(refs):
        assert_close(f"member atomic [{k}]", res.member_atomic[:, k].cpu().numpy(), ref["member_atomic"][:, 0].numpy(),
                     E_RTOL, E_ATOL)
        assert_close(f"forces [{k}]", -res.grad[k].cpu().numpy(), ref["forces"][0].numpy(), 0.0, F_ATOL)
        _note("periodic batch forces", float((-res.grad[k].cpu().double() - ref["forces"][0]).abs().max()) / F_ATOL)


def test_shards_add_up(engines):
    rec = load_golden("water999_pbc_ani2x")
    species, coords, cell, pbc = golden_inputs(rec, torch.float32)
    eng = engines["2x"]
    sp, co, ce = species.to(DEV), coords.to(DEV), cell.to(DEV)
    whole = eng.step(sp, co, ce, True, check=True)
    e0, g0 = whole.energies.clone(), whole.grad.clone()
    ref = orc.compute(oracle_model("2x", torch.float64, "cell_list"), species, coords.double(), cell.double(), pbc)
    for world in (3, 8):
        e, g = torch.zeros_like(e0), torch.zeros_like(g0)
        for rank in range(world):
            r = eng.step(sp, co, ce, True, shard=(rank, world), check=True)
            e += r.energies
            g += r.grad
        assert float((g - g0).abs().max()) < 2e-6 and abs(float(e[0] - e0[0])) < 1e-6 * abs(float(e0[0]))
        assert_close(f"forces of {world} shards", -g.cpu().numpy(), ref["forces"].numpy(), 0.0, F_ATOL)


def test_graph_replay_with_more_elements():
    """Captured with two elements (H and O), replayed with seven: the AEV backward's table is sized at capture."""
    rec = load_golden("sevenel_pbc_ani2x")
    species, coords, cell, pbc = golden_inputs(rec, torch.float32)
    eng = make_engine("2x", ang_pad=True)
    co, ce = coords.to(DEV), cell.to(DEV)
    water = torch.where(species == 0, 0, 3).to(DEV)
    for _ in range(eng.graph_after + 1):
        eng.step(water, co, ce, True)
    eng.check_status()
    ws = eng.workspace(*species.shape)
    assert len(eng._graphs) == 1 and ws.max_elements == 2
    for _ in range(2):
        res = eng.step(species.to(DEV), co, ce, True, check=True)
    assert len(eng._graphs) == 1 and int(ws.aev_blocks[0]) == 32
    ref = orc.compute(oracle_model("2x", torch.float64, "cell_list"), species, coords.double(), cell.double(), pbc)
    assert_close("member atomic energies", res.member_atomic.cpu().numpy(), ref["member_atomic"].numpy(),
                 E_RTOL, E_ATOL)
    assert_close("forces", -res.grad.cpu().numpy(), ref["forces"].numpy(), 0.0, F_ATOL)


@pytest.mark.parametrize("name", ["water30_pbc_ani2x", "6w8h_triclinic_ani2x", "sevenel_pbc_ani2x"])
def test_virial(engines, name):
    rec = load_golden(name)
    species, coords, cell, pbc = golden_inputs(rec, torch.float32)
    eng = engines["2x"]
    res = eng.step(species.to(DEV), coords.to(DEV), cell.to(DEV), True, want_virial=True, check=True)
    volume = abs(float(torch.det(cell.double())))
    c64, cell64 = coords.double(), cell.double()
    wrapped = c64 - torch.floor(c64 @ torch.linalg.inv(cell64)) @ cell64
    ref = orc.compute(oracle_model("2x", torch.float64, "cell_list"), species, wrapped, cell64, pbc, stress=True)
    got = res.virial.cpu().double() / volume
    r = float((got - ref["stress"]).abs().max()) / (1e-5 * float(ref["stress"].abs().max()))
    _note("virial (1e-5 of max |W|)", r)
    assert r <= 1.0, f"virial {r:.3f} x the bar"


@pytest.mark.parametrize("name", ["water30_pbc_ani2x", "kat2x5_ani2x"])
def test_step_members(engines, name):
    rec = load_golden(name)
    species, coords, cell, pbc = golden_inputs(rec, torch.float32)
    eng = engines["2x"]
    e_m, g_m = eng.step_members(species.to(DEV), coords.to(DEV), None if cell is None else cell.to(DEV),
                                cell is not None)
    eng.check_status()
    om = oracle_model("2x", torch.float64, rec["neighborlist"])
    n_real = int((species >= 0).sum())
    for m in range(8):
        ref = orc.compute(om, species, coords.double(), None if cell is None else cell.double(), pbc, members=[m])
        assert_close(f"member {m} energies", e_m[m].cpu().numpy(), ref["energy"].numpy(), 0.0, 2e-7 * max(n_real, 10))
        assert_close(f"member {m} forces", -g_m[m].cpu().numpy(), ref["forces"].numpy(), 0.0, F_ATOL)
        _note("member forces", float((-g_m[m].cpu().double() - ref["forces"]).abs().max()) / F_ATOL)


def test_smooth_cutoff_and_active_members(engines):
    from torchani_b200.engine import Engine, constants_2x
    eng = engines["2x"]
    rec = load_golden("benzene_pbc_ani2x")
    species, coords, cell, pbc = golden_inputs(rec, torch.float32)
    eng_s = Engine(constants_2x(cutoff_fn="smooth"), eng.nets, None)
    m = oracle_model("2x", torch.float64, "cell_list")
    m = m._replace(spec=m.spec._replace(cutoff_fn="smooth"))
    compare(eng_s, species, coords, cell, pbc, m._replace(sae={s: 0.0 for s in m.symbols}))
    eng.nets.set_active_members([1, 4, 6])
    try:
        res = eng.step(species.to(DEV), coords.to(DEV), cell.to(DEV), True, check=True)
        ref = orc.compute(oracle_model("2x", torch.float64, "cell_list"), species, coords.double(), cell.double(),
                          pbc, members=[1, 4, 6])
        assert_close("atomic", res.atomic_energies.cpu().numpy(), ref["atomic_nn"].numpy(), E_RTOL, E_ATOL)
        assert_close("forces", -res.grad.cpu().numpy(), ref["forces"].numpy(), 0.0, F_ATOL)
    finally:
        eng.nets.set_active_members(list(range(8)))


# ------------------------------------------------------------------------------------------------------------------
# large values
# ------------------------------------------------------------------------------------------------------------------
def large_weights(members: int = 2):
    """Layer 1 x 5e4 (activations ~1e4), the head x 2e4 (head seeds G3 ~1e3); layer 2 takes layer 1's output / 5e4."""
    om = oracle_model("2x", torch.float64, members=members)
    out = []
    for wm in om.weights:
        per = {}
        for s, ((w1, b1), (w2, b2), (w3, b3), (w4, b4)) in wm.items():
            per[s] = [(w1 * 5e4, b1 * 5e4), (w2 / 5e4, b2), (w3, b3), (w4 * 2e4, b4 * 2e4)]
        out.append(per)
    return om._replace(weights=out)


def test_large_values():
    rec = load_golden("water30_pbc_ani2x")
    species, coords, cell, pbc = golden_inputs(rec, torch.float32)
    om = large_weights()
    ref = orc.compute(om, species, coords.double(), cell.double(), pbc)
    w32 = [{s: [(w.float(), b.float()) for w, b in layers] for s, layers in wm.items()} for wm in om.weights]
    sp, co, ce = species.to(DEV), coords.to(DEV), cell.to(DEV)
    fp16 = make_engine("2x", members=2, weights=w32, variant="")
    fp16.step(sp, co, ce, True)
    from torchani_b200 import _lib
    with pytest.raises(_lib.OperandRangeError):
        fp16.check_status()
    eng = make_engine("2x", members=2, weights=w32)
    res = eng.step(sp, co, ce, True, check=True)
    fs = float(ref["forces"].abs().max())
    es = float(ref["member_atomic"].abs().max())
    assert fs > 100.0 and es > 1e3, (fs, es)
    rf = float((-res.grad.cpu().double() - ref["forces"]).abs().max()) / (1e-4 * fs)
    re = float((res.member_atomic.cpu().double() - ref["member_atomic"]).abs().max()) / (1e-5 * es)
    _note("large values forces (1e-4 of max |F|)", rf)
    _note("large values member energies (1e-5 of max |e|)", re)
    assert rf <= 1.0 and re <= 1.0, (rf, re)


# ------------------------------------------------------------------------------------------------------------------
# the switch
# ------------------------------------------------------------------------------------------------------------------
ZNUM = {0: 1, 1: 6, 2: 7, 3: 8, 4: 16, 5: 9, 6: 17}
B1, C1, NEURON = 1000.0, 200.0, 7


def threshold_weights():
    """The H network's layer-1 neuron NEURON reads only AEV column 0 (H neighbours at ShfR = 0.8 A):
    a1 = 1000 + 200 * x0, and layer 2 ignores it, so the energies are those of the unmodified model.  x0 of an H atom
    is ~0 in the water box (H-H distances >= 1.5 A) and ~0.24 with two H atoms 0.8 A apart: a1 crosses 1023.5 only
    then."""
    om = oracle_model("2x", torch.float64)
    out = []
    for wm in om.weights:
        per = {}
        for s, ((w1, b1), (w2, b2), rest3, rest4) in wm.items():
            if s != "H":
                per[s] = wm[s]
                continue
            w1, b1, w2 = w1.clone(), b1.clone(), w2.clone()
            w1[NEURON] = 0.0
            w1[NEURON, 0] = C1
            b1[NEURON] = B1
            w2[:, NEURON] = 0.0
            per[s] = [(w1, b1), (w2, b2), rest3, rest4]
        out.append(per)
    return om._replace(weights=out)


def water_and_close_pair():
    """The water box, and the same box with an H atom moved 0.8 A from another H atom (asserted with the oracle)."""
    rec = load_golden("water30_pbc_ani2x")
    species, coords, cell, pbc = golden_inputs(rec, torch.float64)
    h = (species[0] == 0).nonzero().view(-1).tolist()
    moved = coords.clone()
    moved[0, h[0]] = coords[0, h[-1]] + torch.tensor([0.8, 0.0, 0.0], dtype=torch.float64)
    spec = orc.aev_spec_2x()
    for c, inside in ((coords, True), (moved, False)):
        nb = orc.neighborlist("cell_list", spec.rcr, species, c.float().double(), cell, pbc)
        x0 = float(orc.aev_from_neighbors(spec, species, nb)[0, h, 0].max())
        a1 = B1 + C1 * x0
        assert (a1 < 1023.0) if inside else (a1 > 1024.0), (inside, a1)
    return species, coords.float(), moved.float(), cell.float(), pbc


def switch_model():
    from torchani_b200 import models
    om = threshold_weights()
    w32 = [{s: [(w.float(), b.float()) for w, b in layers] for s, layers in wm.items()} for wm in om.weights]
    model = models.from_weight_lists("2x", w32, device=DEV, periodic_table_index=True)
    assert model.neural_networks._variant == ""
    return model, om._replace(neighborlist="cell_list")


def switched(fn):
    """Run fn, return (result, number of switch warnings)."""
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        out = fn()
    return out, sum("bfloat16" in str(w.message) for w in caught)


def check_ef(e, f, ref, tag):
    """Energy within 1e-5 Ha (plus float32 rounding where the path returns float32), forces at the golden bar."""
    e_ref = float(ref["energy"][0])
    tol = 1e-5 + 1e-7 * abs(e_ref) + (2.0 ** -24 * abs(e_ref) if getattr(e, "dtype", None) == torch.float32 else 0.0)
    assert abs(float(e) - e_ref) < tol, (tag, float(e), e_ref)
    assert_close(f"{tag} forces", np.asarray(f).reshape(-1, 3), ref["forces"][0].numpy(), 0.0, F_ATOL)


PATHS = ["forward", "energies_and_forces", "energies_f64", "energies_forces_stress", "members_forces"]


@pytest.mark.parametrize("path", PATHS)
def test_model_paths_switch(path):
    species, coords, moved, cell, pbc = water_and_close_pair()
    model, om = switch_model()
    z = torch.tensor([[ZNUM[int(s)] for s in species[0]]], device=DEV)
    ce, pb = cell.to(DEV), pbc.to(DEV)

    def call(c):
        c = c.to(DEV)
        if path == "forward":
            c = c.clone().requires_grad_(True)
            e = model((z, c), ce, pb).energies
            (g,) = torch.autograd.grad(e.sum(), c)
            return e.detach(), -g
        if path == "energies_and_forces":
            return model.energies_and_forces(z, c, ce, pb)
        if path == "energies_f64":
            return model.energies_f64((z, c), ce, pb), None
        if path == "energies_forces_stress":
            e, f, s = model.energies_forces_stress(z, c, ce, pb)
            return e, (f, s)
        return model.members_forces((z, c), ce, pb)[1:]

    _, n = switched(lambda: call(coords))
    assert n == 0 and model.neural_networks._variant == "", "an in-range call switched"
    out, n = switched(lambda: call(moved))
    assert n == 1 and model.neural_networks._variant == VARIANT
    assert model.engine(torch.device(DEV)).variant == VARIANT
    for pos, label in ((moved, "moved"), (coords, "in range")):
        if label == "in range":
            out, n = switched(lambda: call(coords))
            assert n == 0 and model.neural_networks._variant == VARIANT
        stress = path == "energies_forces_stress"
        ref = orc.compute(om, species, pos.double(), cell.double(), pbc, stress=stress,
                          members=None if path != "members_forces" else [3])
        if path == "members_forces":
            e_m, f_m = out
            check_ef(e_m[3, 0].cpu(), f_m[3].cpu(), ref, f"{path} {label}")
        elif path == "energies_f64":
            assert abs(float(out[0][0]) - float(ref["energy"][0])) < 1e-5, label
        else:
            e, f = out
            if stress:
                f, s = f
            check_ef(e[0].cpu(), f.detach().cpu(), ref, f"{path} {label}")
            if stress:
                c64, cell64 = pos.double(), cell.double()
                wrapped = c64 - torch.floor(c64 @ torch.linalg.inv(cell64)) @ cell64
                rs = orc.compute(om, species, wrapped, cell64, pbc, stress=True)["stress"]
                assert_close(f"stress {label}", s.cpu().numpy(), rs.numpy(), 1e-4, 1e-8)


def test_members_forces_switches_alone():
    """w4 = 15.994 on one neuron with z3 = 1 > 0 in every network: the ensemble's head seed is 15.994 / 8 (in range),
    one member's is 15.994 (4096 * 15.994 = 65511 > 65504, and below 65520, so both half pieces stay finite and only
    the head's own check can raise the bit).  The unmodified model's members_forces stays on 2 x fp16."""
    from torchani_b200 import models
    om = oracle_model("2x", torch.float64)
    rec = load_golden("water30_pbc_ani2x")
    species, coords, cell, pbc = golden_inputs(rec, torch.float32)
    z = torch.tensor([[ZNUM[int(s)] for s in species[0]]], device=DEV)
    args = (coords.to(DEV), cell.to(DEV), pbc.to(DEV))
    stock = models.from_weight_lists("2x", [{s: [(w.float(), b.float()) for w, b in layers] for s, layers in wm.items()}
                                            for wm in om.weights], device=DEV, periodic_table_index=True)
    _, n = switched(lambda: stock.members_forces((z, args[0]), args[1], args[2]))
    assert n == 0 and stock.neural_networks._variant == "", "the unmodified model's members_forces switched"
    out = []
    for wm in om.weights:
        per = {}
        for s, (l1, l2, (w3, b3), (w4, b4)) in wm.items():
            w3, b3, w4 = w3.clone(), b3.clone(), w4.clone()
            w3[NEURON] = 0.0
            b3[NEURON] = 1.0
            w4[0, NEURON] = 15.994
            per[s] = [l1, l2, (w3, b3), (w4, b4)]
        out.append(per)
    om = om._replace(weights=out, neighborlist="cell_list")
    w32 = [{s: [(w.float(), b.float()) for w, b in layers] for s, layers in wm.items()} for wm in om.weights]
    model = models.from_weight_lists("2x", w32, device=DEV, periodic_table_index=True)
    (e, f), n = switched(lambda: model.energies_and_forces(z, *args))
    assert n == 0 and model.neural_networks._variant == ""
    ref = orc.compute(om, species, coords.double(), cell.double(), pbc)
    check_ef(e[0].cpu(), f.cpu(), ref, "ensemble")
    (e_m, f_m), n = switched(lambda: model.members_forces((z, args[0]), args[1], args[2])[1:])
    assert n == 1 and model.neural_networks._variant == VARIANT
    for m in (0, 5):
        ref = orc.compute(om, species, coords.double(), cell.double(), pbc, members=[m])
        check_ef(e_m[m, 0].cpu(), f_m[m].cpu(), ref, f"member {m}")


@pytest.mark.parametrize("skin", [0.0, 0.4], ids=["fresh_grid", "verlet_skin"])
def test_host_calculator_switches_after_capture(skin):
    from torchani_b200.calculator import HostCalculator
    species, coords, moved, cell, pbc = water_and_close_pair()
    model, om = switch_model()
    z = np.array([ZNUM[int(s)] for s in species[0]])
    calc = HostCalculator(model, z, cell.numpy(), pbc=True, skin=skin)
    try:
        ref = orc.compute(om, species, coords.double(), cell.double(), pbc)
        for _ in range(calc.graph_after + 2):       # eager steps, the capture, a replay: all in range
            (e, f), n = switched(lambda: calc.calculate(coords[0].numpy()))
            assert n == 0
            check_ef(e, f, ref, "in range")
        assert calc._graphs and model.neural_networks._variant == ""
        ref_m = orc.compute(om, species, moved.double(), cell.double(), pbc)
        (e, f), n = switched(lambda: calc.calculate(moved[0].numpy()))
        assert n == 1 and model.neural_networks._variant == VARIANT and calc.engine.variant == VARIANT
        check_ef(e, f, ref_m, "switched")
        for _ in range(calc.graph_after + 2):       # later in-range calls stay on the 3 x bf16 build, graphs included
            (e, f), n = switched(lambda: calc.calculate(coords[0].numpy()))
            assert n == 0 and calc.engine.variant == VARIANT
            check_ef(e, f, ref, "after the switch")
        assert calc._graphs
        calc.check_status()
    finally:
        model.engine(torch.device(DEV)).skin = 0.0


def stress_ref(om, species, pos, cell, pbc):
    c64, cell64 = pos.double(), cell.double()
    wrapped = c64 - torch.floor(c64 @ torch.linalg.inv(cell64)) @ cell64
    return orc.compute(om, species, wrapped, cell64, pbc, stress=True)


def test_host_calculator_with_stress_switches():
    from torchani_b200.calculator import HostCalculator
    species, coords, moved, cell, pbc = water_and_close_pair()
    model, om = switch_model()
    z = np.array([ZNUM[int(s)] for s in species[0]])
    calc = HostCalculator(model, z, cell.numpy(), pbc=True)
    (e, f, s), n = switched(lambda: calc.calculate_with_stress(coords[0].numpy()))
    assert n == 0 and model.neural_networks._variant == ""
    for pos in (moved, coords):
        (e, f, s), n = switched(lambda: calc.calculate_with_stress(pos[0].numpy()))
        assert n == (1 if pos is moved else 0) and model.neural_networks._variant == VARIANT
        ref = stress_ref(om, species, pos, cell, pbc)
        check_ef(e, f, ref, "with stress")
        assert_close("stress", s, ref["stress"].numpy(), 1e-4, 1e-8)


def test_ase_calculator_switches():
    try:
        import ase  # noqa: F401
    except ImportError:
        sys.path.insert(0, os.path.join(ROOT, "tests", "stubs"))
    from ase import Atoms
    species, coords, moved, cell, pbc = water_and_close_pair()
    model, om = switch_model()
    numbers = [ZNUM[int(s)] for s in species[0]]
    atoms = Atoms(numbers, moved[0].double().numpy(), cell=cell.double().numpy(), pbc=True)
    atoms.calc = model.ase(stress_kind="fdotr")
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        atoms.calc.calculate(atoms, ["energy", "forces", "stress"])
    assert sum("bfloat16" in str(w.message) for w in caught) == 1
    assert model.neural_networks._variant == VARIANT
    ha = 27.211386024367243
    res = atoms.calc.results
    ref = stress_ref(om, species, moved.double(), cell, pbc)
    check_ef(res["energy"] / ha, res["forces"] / ha, ref, "ase")
    assert_close("ase stress", res["stress"] / ha, ref["stress"].numpy(), 1e-4, 1e-8)
