"""Analytic Hessians on the GPU (csrc/hessian.cu, Engine.hessian, models.ANI.energies_forces_hessians, the double
backward of the fused step and torchani_b200.grad) against float64 double backward of the oracle models
(oracle/hessian_oracle.py).

Bars.  The kernels work in fp32 from fp32 positions, so every comparison is made on float32-rounded inputs and its bar
is sized from the oracle's OWN float32-vs-float64 spread on those inputs: the largest |H32 - H64| of the oracle's
double backward in float32 against float64, times SPREAD_FACTOR = 8, plus FLOOR = 2e-6 of max |H64| (the spread of a
tiny molecule can come out as small as the float64 rounding itself).  Kernel-level blocks use the same rule on the
blocks.  Symmetry and translational invariance are judged against the same bar.
"""
import os
import typing as tp

import numpy as np
import pytest
import torch

import oracle.ani_oracle as orc
import oracle.gelu_oracle as gor
import oracle.hessian_oracle as hor
import oracle.pair_oracle as porc

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SPREAD_FACTOR = 8.0
FLOOR = 2e-6
_cache: tp.Dict[tp.Any, tp.Any] = {}


def bar(energy, coords32, h64):
    """The bar of this file's header for the oracle energy ``energy`` at float32-rounded ``coords32``."""
    h32 = hor.hessian(energy, coords32.float()).double()
    return SPREAD_FACTOR * float((h32 - h64).abs().max()) + FLOOR * float(h64.abs().max())


def weights(kind):
    key = ("w", kind)
    if key not in _cache:
        symbols, dims, dim = (orc.SYMBOLS_2X, orc.DIMS_2X, 1008) if kind == "2x" else (orc.SYMBOLS_1X, orc.DIMS_1X, 384)
        _cache[key] = orc.make_weights(symbols, dims, dim, 8, 1234, torch.float64)
    return _cache[key]


def xtb_tables():
    z = np.load(os.path.join(GOLD, "pair_params.npz"))
    return tuple(torch.tensor(z[k]) for k in ("y_ab", "sqrt_alpha_ab", "k_rep_ab"))


def model(kind="2x", pot=None, variant="", gelu=False):
    """Seeded ANI-1x / 2x x 8 (CELU) or the GELU bias-free ANI-2xr shape, optionally with xTB or ZBL at Rcr."""
    from torchani_b200 import models, nn
    from torchani_b200 import potentials as P
    key = (kind, pot, variant, gelu)
    if key in _cache:
        return _cache[key]
    if gelu:
        spec = gor.gelu_spec()
        symbols = orc.SYMBOLS_2X
        aev = models.AEVComputer.from_constants(spec.rcr, spec.rca, spec.eta_r, spec.shf_r, spec.eta_a, spec.zeta,
                                                spec.shf_a, spec.shf_z, 7, cutoff_fn="smooth")
        w = gor.make_weights(symbols, orc.DIMS_2X, spec.out_dim, 8, 4321)
        members = [nn.ANINetworks.default(symbols, spec.out_dim) for _ in range(8)]
        with torch.no_grad():
            for net, wm in zip(members, w):
                for s in symbols:
                    for (dst, _), (src, _) in zip(net.atomics[s].linear_pairs(), wm[s]):
                        dst.copy_(src)
        base = models.ANI(symbols, aev, nn.Ensemble(members), models.SelfEnergy.with_gsaes(symbols), False)
        rcr = spec.rcr
    else:
        w32 = [{s: [(a.float(), b.float()) for a, b in layers] for s, layers in wm.items()} for wm in weights(kind)]
        base = models.from_weight_lists(kind, w32, periodic_table_index=False)
        rcr = base.aev_computer.constants.rcr
        symbols = base.symbols
    pots = {}
    fn = "smooth" if gelu else "cosine"
    if pot == "xtb":
        p = P.RepulsionXTB(symbols, alpha=[1.0] * 7, yeff=[1.0] * 7, cutoff=rcr, cutoff_fn=fn)
        for k, t in zip(("y_ab", "sqrt_alpha_ab", "k_rep_ab"), xtb_tables()):
            getattr(p, k).copy_(t.float())
        pots["repulsion_xtb"] = p
    elif pot == "zbl":
        pots["repulsion_zbl"] = P.RepulsionZBL(symbols, cutoff=rcr, cutoff_fn=fn)
    m = models.ANI(symbols, base.aev_computer, base.neural_networks, base.energy_shifter, False, pots).to(DEV)
    m.requires_grad_(False)
    if variant:
        m.neural_networks.use_variant(variant)
    _cache[key] = m
    return m


def oracle_energy(kind, species, pot=None, gelu=False, members=None):
    if gelu:
        spec = gor.gelu_spec()
        om = orc.Model(spec, orc.SYMBOLS_2X, gor.make_weights(orc.SYMBOLS_2X, orc.DIMS_2X, spec.out_dim, 8, 4321,
                                                              torch.float64), {}, "all_pairs")
    else:
        spec = orc.aev_spec_2x() if kind == "2x" else orc.aev_spec_1x()
        om = orc.Model(spec, orc.SYMBOLS_2X if kind == "2x" else orc.SYMBOLS_1X, weights(kind), {}, "all_pairs")
    pairs = []
    fn = "smooth" if gelu else "cosine"
    if pot == "xtb":
        pairs.append(porc.PairSpec("xtb", spec.rcr, fn, xtb_tables()))
    elif pot == "zbl":
        pairs.append(porc.zbl_spec(orc.SYMBOLS_2X, spec.rcr, fn))
    return hor.energy_fn(om, species, "gelu" if gelu else "celu", pairs, members), om


def water():
    sp = torch.tensor([[3, 0, 0]])
    co = torch.tensor([[[0.0, 0.0, 0.1173], [0.0, 0.7572, -0.4692], [0.0, -0.7572, -0.4692]]], dtype=torch.float64)
    return sp, co


def fixture(name):
    z = np.load(os.path.join(GOLD, name + ".npz"))
    return torch.tensor(z["species"]), torch.tensor(z["coords"], dtype=torch.float64)


def seven_element_molecule():
    """About 20 atoms of all seven ANI-2x elements, open (the first atoms of the seven-element fixture's box that lie
    within 4 A of its first atom)."""
    sp, co = fixture("sevenel_pbc_ani2x")
    d = (co[0] - co[0, 0]).norm(dim=-1)
    keep = torch.argsort(d)[:20]
    return sp[:, keep], co[:, keep]


CASES = {   # name: (model kind, inputs, potential, gelu)
    "ch4_1x": ("1x", lambda: fixture("ch4_ani1x"), None, False),
    "water_1x": ("1x", water, None, False),
    "sevenel_2x": ("2x", seven_element_molecule, None, False),
    "randbatch_2x": ("2x", lambda: fixture("randbatch_ani2x"), None, False),
    "gelu_xtb": ("2x", seven_element_molecule, "xtb", True),
    "zbl_2x": ("2x", seven_element_molecule, "zbl", False),
}


def run_case(name, variant=""):
    kind, inputs, pot, gelu = CASES[name]
    sp, co = inputs()
    co32 = co.float().double()
    m = model(kind, pot, variant, gelu)
    e, f, h = m.energies_forces_hessians(sp.to(DEV), co32.float().to(DEV))
    energy, _ = oracle_energy(kind, sp, pot, gelu)
    h64 = hor.hessian(energy, co32)
    return h.double().cpu(), h64, bar(energy, co32, h64), (sp, co32, m, energy)


@pytest.mark.parametrize("name", list(CASES))
def test_end_to_end_hessian_matches_float64(name):
    h, h64, b, (sp, *_), = run_case(name)
    err = float((h - h64).abs().max())
    assert err <= b, f"{name}: max |dH| {err:.3e} > bar {b:.3e} (max |H| {float(h64.abs().max()):.3e})"
    pad = (sp.reshape(sp.shape[0], -1) < 0).repeat_interleave(3, dim=1)   # padding atoms: zero rows and columns
    assert float((h.abs() * pad.unsqueeze(2)).sum()) == 0.0 and float((h.abs() * pad.unsqueeze(1)).sum()) == 0.0


def test_symmetry_and_translation_invariance():
    h, h64, b, _ = run_case("sevenel_2x")
    assert float((h - h.transpose(1, 2)).abs().max()) <= b
    t = torch.zeros(h.shape[1], dtype=torch.float64)
    for c in range(3):
        t.zero_()
        t[c::3] = 1.0
        assert float((h[0] @ t).abs().max()) <= b * 3 ** 0.5


@pytest.mark.parametrize("variant", ["", "bf16x3"])
def test_both_operand_builds(variant):
    h, h64, b, _ = run_case("randbatch_2x", variant)
    assert float((h - h64).abs().max()) <= b


def test_active_member_subset():
    sp, co = seven_element_molecule()
    co32 = co.float().double()
    m = model("2x")
    m.set_active_members([1, 4, 6])
    try:
        _, _, h = m.energies_forces_hessians(sp.to(DEV), co32.float().to(DEV))
    finally:
        m.set_active_members(list(range(8)))
    energy, _ = oracle_energy("2x", sp, members=[1, 4, 6])
    h64 = hor.hessian(energy, co32)
    assert float((h.double().cpu() - h64).abs().max()) <= bar(energy, co32, h64)


def test_chunked_equals_unchunked():
    sp, co = fixture("randbatch_ani2x")
    m = model("2x")
    eng = m.engine(DEV)
    eng.step(sp.to(DEV), co.float().to(DEV), want_grad=True, check=True)
    ws = eng.workspace(*sp.shape)
    whole = eng.hessian(ws).double()
    small = eng.hessian(ws, row_budget=64).double()
    assert float((whole - small).abs().max()) <= 1e-5 * float(whole.abs().max())


def test_1c17_chunk_hessian_vector_products():
    sp, co = fixture("1c17_chunk_hcnos_ani2x")
    co32 = co.float().double()
    m = model("2x")
    _, _, h = m.energies_forces_hessians(sp.to(DEV), co32.float().to(DEV))
    energy, _ = oracle_energy("2x", sp)
    gen = torch.Generator().manual_seed(7)
    v = torch.randn(3, *co.shape, generator=gen, dtype=torch.float64)
    ref = hor.hvp(energy, co32, v)
    got = torch.einsum("cij,kcj->kci", h.double().cpu(), v.reshape(3, 1, -1)).reshape_as(ref)
    # a product sums 936 terms: the bar is the float32 spread of the same product by the oracle
    ref32 = hor.hvp(energy, co32.float(), v.float()).double()
    b = SPREAD_FACTOR * float((ref32 - ref).abs().max()) + FLOOR * float(ref.abs().max())
    assert float((got - ref).abs().max()) <= b


def _neighbours(eng, ws, i_sorted):
    """orig indices of sorted atom i's neighbour words, in word order."""
    cnt = int(ws.nbr_cnt[i_sorted])
    words = ws.nbr_list[i_sorted * ws.nbr_cap:i_sorted * ws.nbr_cap + cnt].cpu()
    so = ws.sorted_orig.cpu()
    return [int(so[int(w) & ((1 << 26) - 1)]) for w in words]


def _stage_blocks(name, stage):
    """Run one case's step and then only the given Hessian stage(s) of one chunk; returns per-atom blocks."""
    from torchani_b200._lib import ptr
    from torchani_b200.engine import _hessian_chunks
    import ctypes as C
    kind, inputs, pot, gelu = CASES[name]
    sp, co = inputs()
    co32 = co.float().double()
    m = model(kind, pot, "", gelu)
    eng = m.engine(DEV)
    eng.step(sp.to(DEV), co32.float().to(DEV), want_grad=True, check=True)
    ws = eng.workspace(*sp.shape)
    n_real = int(eng.grid_info(ws).n_real)
    cnt = ws.nbr_cnt[:n_real].clamp(max=ws.nbr_cap).cpu().numpy()
    species = ws.spos[:n_real, 3].contiguous().view(torch.int32).cpu().numpy()
    (plan,) = list(_hessian_chunks(cnt, species, 10 ** 9))
    ch, keep = eng.hessian_chunk_args(plan)
    L, nets = eng.lib, eng.nets
    jac = torch.empty(plan.rows, nets.ldx, dtype=torch.float32, device=DEV)
    hmax = L.ani_b200_hessian_hidden_max(C.byref(nets.model))
    scratch = torch.empty(4 * plan.rows * hmax + len(plan.atom) * 5 * hmax, device=DEV)
    blocks = torch.zeros(plan.block_floats, device=DEV)
    st = torch.cuda.current_stream(DEV).cuda_stream
    assert L.ani_b200_hessian_jacobian(C.byref(eng.params), ptr(ws.spos), ptr(ws.nbr_cnt), ptr(ws.nbr_list),
                                       ws.nbr_cap, C.byref(ch), ptr(jac), nets.ldx, st) == 0
    if stage == "network":
        assert L.ani_b200_hessian_network(C.byref(nets.model), C.byref(nets.plain_weights), ptr(ws.x), ptr(ws.row_of),
                                          ptr(ws.spos), ptr(ws.nbr_cnt), ws.nbr_cap, C.byref(ch), ptr(jac),
                                          ptr(scratch), ptr(blocks), st) == 0
    elif stage == "geometric":
        assert L.ani_b200_hessian_geometric(C.byref(eng.params), ptr(ws.spos), ptr(ws.nbr_cnt), ptr(ws.nbr_list),
                                            ws.nbr_cap, ptr(ws.row_of), ptr(ws.dx), nets.ldx, None, C.byref(ch),
                                            ptr(blocks), st) == 0
    torch.cuda.synchronize()
    out = []
    so = ws.sorted_orig.cpu()
    for k, a in enumerate(plan.atom):
        m3 = 3 * int(cnt[a])
        rows = jac[int(plan.row_off[k]):int(plan.row_off[k]) + m3].double().cpu()
        b = blocks[int(plan.block_off[k]):int(plan.block_off[k]) + m3 * m3].view(m3, m3).double().cpu()
        out.append((int(so[int(a)]), _neighbours(eng, ws, int(a)), rows, b, int(ws.row_of[int(a)])))
    return out, (sp, co32, eng, ws)


def _internal_columns(eng, out_dim):
    """reference AEV column c -> column of the internal order (radial | ang_pad zeros | angular)."""
    RL = eng.consts.radial_len
    return torch.tensor([c if c < RL else c + eng.params.ang_pad for c in range(out_dim)])


def _aev_of(kind, sp, x, i):
    spec = orc.aev_spec_2x() if kind == "2x" else orc.aev_spec_1x()
    nb = orc.neighborlist("all_pairs", spec.rcr, sp, x)
    return orc.aev_from_neighbors(spec, sp, nb).reshape(-1, spec.out_dim)[i]


@pytest.mark.parametrize("name", ["water_1x", "sevenel_2x"])
def test_jacobian_rows_match_autograd(name):
    kind = CASES[name][0]
    out, (sp, co32, eng, ws) = _stage_blocks(name, "jacobian")
    cols = _internal_columns(eng, eng.consts.out_dim)
    for oi, nbrs, rows, _, _ in out[:6]:
        jac = torch.autograd.functional.jacobian(lambda x: _aev_of(kind, sp, x, oi), co32)   # (D, 1, A, 3)
        ref = torch.stack([jac[:, 0, j, c] for j in nbrs for c in range(3)])                # (3 n, D)
        ref32 = torch.autograd.functional.jacobian(lambda x: _aev_of(kind, sp, x, oi), co32.float())
        ref32 = torch.stack([ref32[:, 0, j, c] for j in nbrs for c in range(3)]).double()
        b = SPREAD_FACTOR * float((ref32 - ref).abs().max()) + FLOOR * float(ref.abs().max())
        assert float((rows[:, cols] - ref).abs().max()) <= b


def _relative(f, co32, oi, nbrs):
    """f(coords) as a function of the displacements y (3 n) of atom oi's neighbours."""
    def g(y):
        x = co32.clone().reshape(-1, 3)
        x = x.index_add(0, torch.tensor(nbrs), y.view(-1, 3))
        return f(x.view_as(co32))
    return g


@pytest.mark.parametrize("name", ["water_1x", "sevenel_2x"])
def test_network_blocks_match_float64(name):
    kind = CASES[name][0]
    out, (sp, co32, eng, ws) = _stage_blocks(name, "network")
    energy, om = oracle_energy(kind, sp)
    for oi, nbrs, _, blk, _ in out[:4]:
        s = int(sp.reshape(-1)[oi])
        a0 = _aev_of(kind, sp, co32, oi)
        J = torch.autograd.functional.jacobian(_relative(lambda x: _aev_of(kind, sp, x, oi), co32, oi, nbrs),
                                               torch.zeros(3 * len(nbrs), dtype=torch.float64))

        def nn_lin(y, dtype=torch.float64):
            a = (a0 + J @ y).to(dtype).view(1, -1)
            tot = 0.0
            for wm in om.weights:
                tot = tot + orc.atomic_network(a, [(w.to(dtype), b.to(dtype)) for w, b in wm[om.symbols[s]]]).sum()
            return tot / len(om.weights)
        y0 = torch.zeros(3 * len(nbrs), dtype=torch.float64)
        ref = torch.autograd.functional.hessian(nn_lin, y0)
        ref32 = torch.autograd.functional.hessian(lambda y: nn_lin(y.double(), torch.float32), y0.float()).double()
        b = SPREAD_FACTOR * float((ref32 - ref).abs().max()) + FLOOR * float(ref.abs().max())
        assert float((blk - ref).abs().max()) <= b


@pytest.mark.parametrize("name", ["water_1x", "sevenel_2x"])
def test_geometric_blocks_match_float64(name):
    kind = CASES[name][0]
    out, (sp, co32, eng, ws) = _stage_blocks(name, "geometric")
    cols = _internal_columns(eng, eng.consts.out_dim)
    for oi, nbrs, _, blk, row in out[:4]:
        g = ws.dx[row].double().cpu()[cols]
        f = _relative(lambda x: (g * _aev_of(kind, sp, x, oi)).sum(), co32, oi, nbrs)
        y0 = torch.zeros(3 * len(nbrs), dtype=torch.float64)
        ref = torch.autograd.functional.hessian(f, y0)
        f32 = _relative(lambda x: (g.float() * _aev_of(kind, sp, x, oi)).sum(), co32.float(), oi, nbrs)
        ref32 = torch.autograd.functional.hessian(f32, y0.float()).double()
        b = SPREAD_FACTOR * float((ref32 - ref).abs().max()) + FLOOR * float(ref.abs().max())
        assert float((blk - ref).abs().max()) <= b


def test_api_paths_agree_with_one_hessian_each():
    from torchani_b200 import grad
    sp, co = seven_element_molecule()
    x = co.float().to(DEV)
    m = model("2x")
    eng = m.engine(DEV)
    n0 = eng.hessian_count
    e1, f1, h1 = m.energies_forces_hessians(sp.to(DEV), x)
    assert eng.hessian_count == n0 + 1
    xr = x.clone()
    e2, f2, h2 = grad.energies_forces_and_hessians(m, sp.to(DEV), xr)
    assert eng.hessian_count == n0 + 2
    assert float((f1 - f2.detach()).abs().max()) < 1e-6
    assert float((h1 - h2).abs().max()) <= 1e-6 * float(h1.abs().max())
    from oracle import ref_torchani
    if os.path.isdir(os.path.join(os.path.dirname(GOLD), "..", "oracle", "_ref", "torchani")):
        torchani = ref_torchani.load()
        xr = x.clone()
        _, f3, h3 = torchani.grad.energies_forces_and_hessians(m, sp.to(DEV), xr)
        assert eng.hessian_count == n0 + 3
        assert float((h1 - h3).abs().max()) <= 1e-6 * float(h1.abs().max())


def test_vibrational_frequencies_on_gpu_hessian():
    from torchani_b200 import grad
    h, h64, b, (sp, co32, m, energy) = run_case("water_1x")
    masses = torch.tensor([[15.999, 1.008, 1.008]], dtype=torch.float64)
    got = grad.vibrational_analysis(masses, h, "mdn")
    ref = hor.vibrational_analysis(masses[0].numpy(), h64[0].numpy(), "mdn")
    # the three vibrations (the six largest |w| minus the rigid motions): 1e-3 relative covers the float32 Hessian
    f_got = np.sort(got.freqs.numpy())[-3:]
    f_ref = np.sort(ref["freqs"])[-3:]
    assert np.allclose(f_got, f_ref, rtol=1e-3), (f_got, f_ref)


def test_rejections():
    from torchani_b200 import models, potentials as P
    m = model("2x")
    sp, co = seven_element_molecule()
    eng = m.engine(DEV)
    cell = torch.eye(3, device=DEV) * 30.0
    eng.step(sp.to(DEV), co.float().to(DEV), cell, True, want_grad=True, check=True)
    with pytest.raises(ValueError, match="periodic"):
        eng.hessian(eng.workspace(*sp.shape))
    ws, _ = eng._stage_inputs(sp.to(DEV), co.float().to(DEV), None, False)
    eng.run(ws, False, True, shard=(0, 2))
    with pytest.raises(ValueError, match="unsharded"):
        eng.hessian(ws)
    eng.run(ws, False, False)
    with pytest.raises(ValueError, match="dE/dAEV"):
        eng.hessian(ws)
    # D3 and LJ / Coulomb terms
    base = model("2x")
    lj = models.ANI(base.symbols, base.aev_computer, base.neural_networks, base.energy_shifter, False,
                    {"lj": P.LennardJones(base.symbols, cutoff=8.0)}).to(DEV)
    with pytest.raises(NotImplementedError, match="Lennard-Jones"):
        lj.energies_forces_hessians(sp.to(DEV), co.float().to(DEV))
    # periodic input through autograd
    x = co.float().to(DEV).requires_grad_(True)
    e = m((sp.to(DEV), x), cell, torch.ones(3, dtype=torch.bool, device=DEV)).energies
    with pytest.raises(ValueError, match="periodic"):
        torch.autograd.grad(e.sum(), x, create_graph=True)


def test_create_graph_guards_on_module_functions():
    m = model("2x")
    sp, co = seven_element_molecule()
    x = co.float().to(DEV).requires_grad_(True)
    aev = m.aev_computer(sp.to(DEV), x)
    e = m.neural_networks(sp.to(DEV), aev)
    with pytest.raises(NotImplementedError, match="second derivatives"):
        torch.autograd.grad(e.sum(), x, create_graph=True)
    from torchani_b200.neighbors import all_pairs
    nb = all_pairs(5.1, sp.to(DEV), x)
    e2 = m.compute_from_neighbors(sp.to(DEV), x, nb)
    with pytest.raises(NotImplementedError, match="second derivatives"):
        torch.autograd.grad(e2.sum(), x, create_graph=True)


def test_d3_and_accelerated_models_are_rejected():
    import test_gpu_gelu_networks as tg
    m = tg.gelu_model(d3=True)
    sp, co = seven_element_molecule()
    with pytest.raises(NotImplementedError, match="D3"):
        m.energies_forces_hessians(sp.to(DEV), co.float().to(DEV))
    from oracle import ref_torchani
    if not ref_torchani.available():
        return
    from torchani_b200 import models
    ref = ref_torchani.build_model(weights("2x"), "2x", device=DEV, periodic_table_index=False)
    models.accelerate_torchani_(ref)
    x = co.float().to(DEV).requires_grad_(True)
    e = ref((sp.to(DEV), x)).energies
    with pytest.raises(NotImplementedError, match="from_torchani"):
        torch.autograd.grad(e.sum(), x, create_graph=True)


@pytest.mark.parametrize("name", ["ch4_1x", "water_1x", "sevenel_2x", "randbatch_2x", "zbl_2x"])
def test_hessian_matches_the_reference_fixtures(name):
    """Against tests/golden/hessian_*.npz (the reference's torchani.grad in float64 at the fixture's float64
    coordinates); the bar also covers rounding the coordinates to float32: the oracle's float32 Hessian at the rounded
    coordinates against the fixture, times SPREAD_FACTOR, plus FLOOR."""
    from torchani_b200 import grad
    z = np.load(os.path.join(GOLD, f"hessian_{name}.npz"))
    kind, _, pot, gelu = CASES[name]
    sp, co = torch.tensor(z["species"]), torch.tensor(z["coords"])
    ref = torch.tensor(z["hessian"])
    _, _, h = model(kind, pot).energies_forces_hessians(sp.to(DEV), co.float().to(DEV))
    energy, _ = oracle_energy(kind, sp, pot)
    h32 = hor.hessian(energy, co.float()).double()
    b = SPREAD_FACTOR * float((h32 - ref).abs().max()) + FLOOR * float(ref.abs().max())
    assert float((h.double().cpu() - ref).abs().max()) <= b
    if name == "water_1x":   # the vibrations on the GPU Hessian (frequency bar: 1e-3 relative)
        va = grad.vibrational_analysis(torch.tensor(z["masses"]), h.double().cpu(), "mdn")
        f_ref = z["vib_0_mdn_cm_freqs"]
        keep = np.abs(f_ref) > 1e-3 * np.abs(f_ref).max()
        np.testing.assert_allclose(va.freqs.numpy()[keep], f_ref[keep], rtol=1e-3)
