"""Atomic charges and dipoles of charge models (ANIq, ANImbis) on the GPU.

* ``ani_b200_charges`` alone against float64 (``charge_oracle.normalize`` / ``dipole`` on the float32 inputs), on one
  10 k-atom conformer and on 300 conformers of 1-40 real atoms padded to 40: padding atoms, both values of the q^2
  flag, ``normalize`` off, a nonzero total charge, all three dipole frames.  Bars: charges within
  1e-5 * max|q| + 1e-6 e, sum q equal to Q within 1e-5 * sum|q|, dipoles within 1e-5 * sum_i |q_i| |r_i - r_ref|, and
  two runs bitwise equal.  The kernel sums in float64 and rounds each charge once to float32, so these bars hold with
  orders of magnitude to spare; they are the ones proposed for it.
* ``models.ANIq`` against the charges_* fixtures of the reference (oracle/make_charge_golden.py), in the 2 x fp16 and
  the 3 x bf16 build, eagerly and on graph replay.  The charges come out of a network pass on float32 AEVs, so their
  bar is that of the atomic energies (E_RTOL relative to max|q| + 1e-6 e); a dipole may carry every charge's error
  along its lever arm: 1e-5 * sum_i |q_i| |r_i - r_ref| + (charge bar) * sum_i |r_i - r_ref|.  Energies and forces
  use the bars of tests/test_gpu_gelu_networks.py.
* Periodic batches with one cell per conformer, partial PBC, the thin-cell supercell route, Verlet-skin reuse
  through ``HostCalculator``, the energy step unchanged, the operand-range fallback of both network sets, the drop-in
  conversion of a seeded reference ANIq (where oracle/_ref exists), the rejected cases and the calculators.
"""
import os
import warnings

import numpy as np
import pytest
import torch

import oracle.ani_oracle as orc
import oracle.charge_oracle as cor
import oracle.gelu_oracle as gor
from helpers import E_RTOL, F_ATOL, GOLD, assert_close

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
SYSTEMS = {"mbis": ["water999_pbc", "1c17_chunk_hcnos", "randbatch", "6w8h_triclinic", "sevenel_pbc", "small264_nopbc"],
           "simple": ["randbatch", "small264_nopbc", "water999_pbc"]}
FIXTURES = [(c, n) for c, ns in SYSTEMS.items() for n in ns]
_cache = {}


def fixture(config, name):
    z = np.load(os.path.join(GOLD, f"charges_{config}_{name}.npz"))
    return {k: z[k] for k in z.files}


def inputs(rec, dtype=torch.float32):
    sp = torch.tensor(rec["species"]).to(DEV)
    co = torch.tensor(rec["coords"]).to(dtype).to(DEV)
    cell = torch.tensor(rec["cell"]).to(dtype).to(DEV) if rec["cell"].size else None
    pbc = torch.tensor(rec["pbc"]).to(DEV) if rec["pbc"].size else None
    return sp, co, cell, pbc


def weights(config, rec):
    symbols = tuple(str(s) for s in rec["symbols"])
    if config == "mbis":
        spec = orc.aev_spec_2x()
        ew = orc.make_weights(symbols, orc.DIMS_2X, spec.out_dim, 8, int(rec["energy_seed"]))
    else:
        spec = gor.gelu_spec()
        ew = gor.make_weights(symbols, orc.DIMS_2X, spec.out_dim, 8, int(rec["energy_seed"]))
    cw = cor.make_charge_weights(symbols, orc.DIMS_2X, spec.out_dim, 2 if config == "mbis" else 1,
                                 int(rec["charge_seed"]))
    return symbols, spec, ew, cw


def oracle_model(config, rec, neighborlist="cell_list", cw=None):
    symbols, spec, ew, cw0 = weights(config, rec)
    sae = dict(zip(symbols, rec["self_energies"].tolist()))
    return cor.ChargeModel(orc.Model(spec, symbols, ew, sae, neighborlist), config == "simple",
                           cw if cw is not None else cw0, int(rec["kept"]), tuple(rec["norm_weights"].tolist()),
                           bool(rec["scale_by_q2"]), tuple(rec["masses"].tolist()))


def build_model(config, variant="", neighborlist="cell_list", fresh=False):
    """The fixtures' model assembled here (element indices as species: periodic_table_index=False)."""
    from torchani_b200 import electro, models, nn
    key = (config, variant, neighborlist)
    if fresh or key not in _cache:
        rec = fixture(config, SYSTEMS[config][0])
        symbols, spec, ew, cw = weights(config, rec)
        aev = models.AEVComputer.from_constants(spec.rcr, spec.rca, spec.eta_r, spec.shf_r, spec.eta_a, spec.zeta,
                                                spec.shf_a, spec.shf_z, 7, cutoff_fn=spec.cutoff_fn,
                                                neighborlist=neighborlist)
        if config == "mbis":
            members = [nn.ANINetworks.like_2x(symbols, spec.out_dim) for _ in range(8)]
        else:
            members = [nn.ANINetworks.default(symbols, spec.out_dim) for _ in range(8)]
        qnets = nn.ChargeNetworks.like_2x(symbols, spec.out_dim, out_dim=2 if config == "mbis" else 1)
        with torch.no_grad():
            for net, wm in zip(members, ew):
                for s in symbols:
                    for (dst, b_dst), (w, b) in zip(net.atomics[s].linear_pairs(), wm[s]):
                        dst.copy_(w)
                        if b_dst is not None:
                            b_dst.copy_(b)
            for s in symbols:
                for (dst, b_dst), w in zip(qnets.atomics[s].linear_pairs(), cw[s]):
                    assert b_dst is None
                    dst.copy_(w)
        norm = electro.ChargeNormalizer(symbols, rec["norm_weights"].tolist(), bool(rec["scale_by_q2"]))
        m = models.ANIq(symbols, aev, nn.Ensemble(members), models.SelfEnergy(symbols, rec["self_energies"].tolist()),
                        None, False, qnets, norm).to(DEV)
        m.requires_grad_(False)
        if variant:
            m.neural_networks.use_variant(variant)
        if fresh:
            return m
        _cache[key] = m
    return _cache[key]


def charge_bar(q_ref):
    return E_RTOL * float(np.abs(q_ref).max()) + 1e-6


def dipole_bar(species, coords, q, frame, masses):
    """1e-5 * sum |q_i| |r_i - r_ref| + (charge bar) * sum |r_i - r_ref| per conformer (float64 numpy inputs)."""
    sp = torch.tensor(species)
    co = torch.tensor(coords, dtype=torch.float64)
    real = (sp >= 0).double()
    if frame == "origin":
        ref = torch.zeros(co.shape[0], 1, 3, dtype=torch.float64)
    else:
        m = (torch.tensor(masses, dtype=torch.float64)[sp.clamp(min=0)] if frame == "center_of_mass"
             else torch.ones_like(real)) * real
        ref = (m.unsqueeze(-1) * co).sum(1, keepdim=True) / m.sum(1).view(-1, 1, 1)
    lever = (co - ref).norm(dim=-1) * real
    qa = torch.tensor(q, dtype=torch.float64).abs()
    return (1e-5 * (qa * lever).sum(1) + charge_bar(q) * lever.sum(1)).numpy().reshape(-1, 1)


def check_dipoles(tag, got, ref, bar):
    err = np.abs(np.asarray(got, dtype=np.float64) - ref)
    assert (err <= bar).all(), f"{tag}: dipole error {err.max():.3e}, bar {bar.min():.3e}"


# -- the kernel alone ---------------------------------------------------------------------------------------------
def random_inputs(kind, seed=7):
    g = torch.Generator().manual_seed(seed)
    if kind == "big":
        C, A = 1, 10000
        sp = torch.randint(0, 7, (C, A), generator=g)
        sp[torch.rand(C, A, generator=g) < 0.05] = -1
    else:
        C, A = 300, 40
        sp = torch.randint(0, 7, (C, A), generator=g)
        real = torch.randint(1, 41, (C,), generator=g)
        sp[torch.arange(A).view(1, -1) >= real.view(-1, 1)] = -1
    q = (0.3 * torch.randn(C, A, generator=g)).float() * (sp >= 0)
    q = torch.where(sp >= 0, q, torch.full_like(q, 123.0))    # garbage under the padding must not matter
    co = (50.0 * torch.rand(C, A, 3, generator=g)).float()
    w = tuple(float(np.float32(v)) for v in (0.5 + torch.rand(7, generator=g)).tolist())
    masses = tuple(float(np.float32(v)) for v in (1.0 + 30.0 * torch.rand(7, generator=g)).tolist())
    return sp, q, co, w, masses


@pytest.mark.parametrize("kind", ["big", "batch"])
@pytest.mark.parametrize("q2,normalize,Q", [(False, True, 0.0), (True, True, 0.0), (True, True, -1.5),
                                            (False, True, 2.0), (False, False, 0.0)])
def test_charges_kernel_matches_float64(kind, q2, normalize, Q):
    from torchani_b200.electro import run_charges
    sp, q, co, w, masses = random_inputs(kind)
    q64 = torch.where(sp >= 0, q, torch.zeros_like(q)).double()
    ref_q = cor.normalize(sp, q64, w, q2, Q) if normalize else q64
    ref_q = torch.where(sp >= 0, ref_q, torch.zeros_like(ref_q))
    for fi, frame in enumerate(cor.FRAMES):
        got_q, dip = run_charges(sp.to(DEV), q.to(DEV), co.to(DEV), w, q2, normalize, Q, masses, fi, True)
        got_q2, dip2 = run_charges(sp.to(DEV), q.to(DEV), co.to(DEV), w, q2, normalize, Q, masses, fi, True)
        assert torch.equal(got_q, got_q2) and torch.equal(dip, dip2), "two runs differ"
        gq = got_q.double().cpu()
        assert float((gq - ref_q).abs().max()) <= 1e-5 * float(ref_q.abs().max()) + 1e-6
        assert bool((gq[sp < 0] == 0).all())
        if normalize:
            tot = gq.sum(1)
            assert float((tot - Q).abs().max()) <= 1e-5 * float(gq.abs().sum(1).max())
        ref_mu = cor.dipole(sp, co.double(), ref_q, frame, masses)
        real = (sp >= 0).double()
        if frame == "origin":
            r0 = torch.zeros(sp.shape[0], 1, 3, dtype=torch.float64)
        else:
            mm = (torch.tensor(masses, dtype=torch.float64)[sp.clamp(min=0)] if frame == "center_of_mass"
                  else torch.ones_like(real)) * real
            r0 = (mm.unsqueeze(-1) * co.double()).sum(1, keepdim=True) / mm.sum(1).view(-1, 1, 1)
        bar = 1e-5 * ((ref_q.abs() * (co.double() - r0).norm(dim=-1)) * real).sum(1)
        assert bool(((dip.cpu() - ref_mu).abs() <= bar.view(-1, 1) + 1e-12).all()), frame


def test_charges_kernel_rejects_bad_arguments():
    from torchani_b200 import _lib
    L = _lib.lib()
    x = torch.zeros(4, device=DEV)
    s = torch.zeros(4, dtype=torch.int32, device=DEV)
    d = torch.zeros(3, dtype=torch.float64, device=DEV)
    P = _lib.ptr
    # NULL raw charges, one of row_of / orig_to_sorted alone, a frame out of range, the centre of mass without masses
    assert L.ani_b200_charges(None, None, None, P(s), P(x), 1, 4, None, 1, 0, 0, 0.0, None, 2, P(x), None, None) != 0
    assert L.ani_b200_charges(P(x), P(s), None, P(s), P(x), 1, 4, None, 1, 0, 0, 0.0, None, 2, P(x), None, None) != 0
    assert L.ani_b200_charges(P(x), None, None, P(s), P(x), 1, 4, None, 1, 0, 0, 0.0, None, 3, P(x), None, None) != 0
    assert L.ani_b200_charges(P(x), None, None, P(s), P(x), 1, 4, None, 1, 0, 0, 0.0, None, 0, P(x), P(d), None) != 0
    assert L.ani_b200_charges(P(x), None, None, P(s), P(x), 1, 4, None, 1, 0, 1, 0.0, None, 2, P(x), None, None) != 0


# -- models.ANIq against the reference fixtures --------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["", "bf16x3"], ids=["fp16x2", "bf16x3"])
@pytest.mark.parametrize("config,name", FIXTURES)
def test_aniq_matches_the_reference_fixtures(config, name, variant):
    rec = fixture(config, name)
    m = build_model(config, variant)
    sp, co, cell, pbc = inputs(rec)
    n_real = int((sp >= 0).sum(1).max())
    eng = m.engine(torch.device(DEV))
    for call in range(eng.graph_after + 2):   # eager calls, the capture, a replay
        x = co.clone().requires_grad_(True)
        out = m((sp, x), cell, pbc)
        (g,) = torch.autograd.grad(out.energies.sum(), x)
        if call not in (0, eng.graph_after + 1):
            continue
        tag = f"{config} {name} {variant or 'fp16x2'} call {call}"
        assert_close(f"{tag} energies", out.energies.detach().double().cpu().numpy(), rec["energy"], 2e-7,
                     2e-7 * max(n_real, 10) + 1e-3)
        assert_close(f"{tag} forces", (-g).cpu().numpy(), rec["forces"], 1e-5, F_ATOL)
        assert_close(f"{tag} charges", out.atomic_charges.detach().cpu().numpy(), rec["charges"], 0.0,
                     charge_bar(rec["charges"]))
    ws = eng.workspace(*sp.shape)
    assert_close(f"{config} {name} raw charges", eng.raw_charges(ws).cpu().numpy(), rec["raw_charges"], 0.0,
                 charge_bar(rec["raw_charges"]))
    for frame in cor.FRAMES:
        dip = m.dipoles((sp, co), cell, pbc, reference=frame, masses=rec["masses"].tolist())
        check_dipoles(f"{config} {name} {frame}", dip.cpu().numpy(), rec["dipole_" + frame],
                      dipole_bar(rec["species"], rec["coords"], rec["charges"], frame, rec["masses"]))


def test_energy_step_is_unchanged():
    """ANIq energies / forces are those of an ANI with the same energy networks, and a step without charges issues the
    launches of the ANI step."""
    from torchani_b200 import models
    rec = fixture("mbis", "water999_pbc")
    m = build_model("mbis")
    ani = models.ANI(m.symbols, m.aev_computer, m.neural_networks, m.energy_shifter, False)
    sp, co, cell, pbc = inputs(rec)
    e_q, f_q = m.energies_and_forces(sp, co, cell, pbc)
    e_a, f_a = ani.energies_and_forces(sp, co, cell, pbc)
    assert torch.equal(e_q, e_a) and float((f_q - f_a).abs().max()) < 1e-6
    x = co.clone().requires_grad_(True)
    out = m((sp, x), cell, pbc)
    (g,) = torch.autograd.grad(out.energies.sum(), x)
    assert float((out.energies.detach().double() - e_a).abs().max()) < 1e-2 and float((-g - f_a).abs().max()) < 1e-6
    eq, ea = m.engine(torch.device(DEV)), ani.engine(torch.device(DEV))
    eq.step(sp, co, cell, True)
    n_plain = eq.launches_per_step
    ea.step(sp, co, cell, True)
    assert n_plain == ea.launches_per_step
    eq.step(sp, co, cell, True, want_charges=True)
    assert eq.launches_per_step == n_plain + eq._charge_launches(eq.workspace(*sp.shape))


def water(n, seed, scale=1.0):
    from torchani_b200 import synthetic
    z, idx, coords, cell, pbc = synthetic.water_box(n, seed=seed)
    sym = fixture("mbis", "water999_pbc")["symbols"].tolist()
    sp = torch.tensor([sym.index({1: "H", 8: "O"}[int(a)]) for a in z.view(-1).tolist()]).view(1, -1)
    return sp, coords.view(1, -1, 3).double() * scale, cell.double() * scale


def oracle_charges(config, sp, co, cell, pbc, nl):
    om = oracle_model(config, fixture(config, SYSTEMS[config][0]), nl)
    return cor.compute(om, sp, co, cell, pbc, forces=False)


def test_periodic_batch_with_one_cell_per_conformer():
    m = build_model("mbis")
    sps, cos, cells = zip(*[water(40, seed=s, scale=f) for s, f in ((1, 1.0), (2, 1.05), (3, 0.97))])
    sp, co, cell = torch.cat(sps).to(DEV), torch.cat(cos).float().to(DEV), torch.stack(cells).float().to(DEV)
    pbc = torch.ones(3, dtype=torch.bool, device=DEV)
    out = m((sp, co), cell, pbc)
    dip = m.dipoles((sp, co), cell, pbc, reference="center_of_geometry")
    for c in range(3):
        one = m((sp[c:c + 1], co[c:c + 1]), cell[c], pbc)
        assert float((out.atomic_charges[c] - one.atomic_charges[0]).abs().max()) < 1e-7
        d1 = m.dipoles((sp[c:c + 1], co[c:c + 1]), cell[c], pbc, reference="center_of_geometry")
        assert float((dip[c] - d1[0]).abs().max()) < 1e-6


@pytest.mark.parametrize("route", ["partial_pbc", "thin_cell"])
def test_partial_pbc_and_thin_cell(route):
    if route == "partial_pbc":
        m = build_model("mbis")
        sp, co, cell = water(60, seed=5)
        pbc = torch.tensor([True, True, False])
        nl = "all_pairs"   # (the oracle's cell list takes full PBC only)
    else:
        m = build_model("mbis", neighborlist="all_pairs")
        sp, co, cell = water(4, seed=6)     # a cell thinner than the cutoff: the supercell route
        pbc = torch.ones(3, dtype=torch.bool)
        nl = "all_pairs"
    ref = oracle_charges("mbis", sp, co, cell, pbc, nl)
    out = m((sp.to(DEV), co.float().to(DEV)), cell.float().to(DEV), pbc.to(DEV))
    assert_close(f"{route} charges", out.atomic_charges.cpu().numpy(), ref["charges"].numpy(), 0.0,
                 charge_bar(ref["charges"].numpy()))
    assert_close(f"{route} energies", out.energies.double().cpu().numpy(), ref["energy"].numpy(), 2e-7, 1e-3)
    dip = m.dipoles((sp.to(DEV), co.float().to(DEV)), cell.float().to(DEV), pbc.to(DEV), reference="origin")
    check_dipoles(route, dip.cpu().numpy(), ref["dipole_origin"].numpy(),
                  dipole_bar(sp.numpy(), co.numpy(), ref["charges"].numpy(), "origin", None))


def test_host_calculator_with_verlet_skin_and_ase():
    from torchani_b200.calculator import HostCalculator
    rec = fixture("mbis", "water999_pbc")
    m = build_model("mbis")
    sp, co, cell, pbc = inputs(rec)
    host = HostCalculator(m, sp.cpu().numpy()[0], cell.cpu().numpy(), pbc=True, skin=1.0)
    masses = rec["masses"].tolist()
    host.set_dipole_reference("center_of_mass", masses)
    d2h = host.d2h_bytes
    g = torch.Generator().manual_seed(3)
    pos = co[0].cpu()
    for step in range(6):   # eager, capture, replays, grid reuse within the skin
        pos = pos + 0.02 * torch.randn(pos.shape, generator=g)
        e, f, q, dip = host.calculate_with_charges(pos.numpy())
        out = m((sp, pos.view(1, -1, 3).to(DEV)), cell, pbc)
        assert abs(e - float(m.energies_f64((sp, pos.view(1, -1, 3).to(DEV)), cell, pbc)[0])) < 1e-6
        assert float(np.abs(q - out.atomic_charges[0].cpu().numpy()).max()) < 1e-7
        ref_dip = m.dipoles((sp, pos.view(1, -1, 3).to(DEV)), cell, pbc, reference="center_of_mass", masses=masses)
        assert float(np.abs(dip - ref_dip[0].cpu().numpy()).max()) < 1e-5
    assert host.rebuilds < 6 and host.d2h_bytes == d2h
    e2, _ = host.calculate(pos.numpy())
    assert host.d2h_bytes == d2h and abs(e2 - e) < 1e-6


def test_ase_charges_and_dipole(monkeypatch):
    """The ASE calculator of an ANIq model: "charges" and "dipole" (about the centre of mass of the Atoms) agree with
    ANIq.forward / ANIq.dipoles; atoms of one element with different masses raise.  Without ase, the shim of
    tests/stubs/ase (as tests/test_gpu_ase.py), whose Atoms gets a get_masses here."""
    import sys
    from helpers import ROOT
    try:
        import ase
    except ImportError:
        sys.path.insert(0, os.path.join(ROOT, "tests", "stubs"))
        import ase
    from ase.calculators.calculator import all_changes
    from torchani_b200 import electro, models
    rec = fixture("mbis", "small264_nopbc")
    base = build_model("mbis")
    m = models.ANIq(base.symbols, base.aev_computer, base.neural_networks, base.energy_shifter, None, True,
                    base.charge_networks, base.charge_normalizer).to(DEV)
    sym = [str(s) for s in rec["symbols"]]
    numbers = rec["atomic_numbers"][0]
    mass_of = {orc.ATOMIC_NUMBERS[s]: float(v) for s, v in zip(sym, rec["masses"])}
    odd = {"first_h": False}

    def get_masses(self):
        z = np.asarray(self.get_atomic_numbers())
        out = np.array([mass_of[int(v)] for v in z])
        if odd["first_h"]:
            out[int(np.nonzero(z == 1)[0][0])] = 2.014
        return out
    monkeypatch.setattr(type(ase.Atoms(numbers=numbers, positions=rec["coords"][0])), "get_masses", get_masses,
                        raising=False)
    atoms = ase.Atoms(numbers=numbers, positions=rec["coords"][0])
    calc = m.ase()
    assert "charges" in calc.implemented_properties and "dipole" in calc.implemented_properties
    calc.calculate(atoms, ["energy", "charges", "dipole"], all_changes)
    q, dip = calc.results["charges"], calc.results["dipole"]
    znum = torch.tensor(numbers).view(1, -1).to(DEV)
    co = torch.tensor(rec["coords"]).float().to(DEV)
    out = m((znum, co))
    assert float(np.abs(q - out.atomic_charges[0].cpu().numpy()).max()) < 1e-7
    per_symbol = [mass_of[orc.ATOMIC_NUMBERS[s]] for s in sym]
    ref = m.dipoles((znum, co), reference="center_of_mass", masses=per_symbol)
    assert float(np.abs(dip - ref[0].cpu().numpy()).max()) < 1e-5
    # the standalone DipoleComputer on the same charges (masses indexed by atomic number)
    table = [0.0] * 18
    for s, mass in zip(sym, per_symbol):
        table[orc.ATOMIC_NUMBERS[s]] = mass
    d2 = electro.DipoleComputer(table, "center_of_mass")(znum, co.double(), out.atomic_charges.double())
    assert float((d2[0].cpu() - ref[0].cpu().double()).abs().max()) < 1e-5
    odd["first_h"] = True
    with pytest.raises(ValueError):
        m.ase().calculate(atoms, ["energy", "dipole"], all_changes)


def test_operand_range_switches_both_network_sets():
    rec = fixture("mbis", "small264_nopbc")
    m = build_model("mbis", fresh=True)
    symbols, spec, ew, cw = weights("mbis", rec)
    # layer-1 weights of the charge networks x 4000: their activations leave the range of the 2 x fp16 pieces
    cw_big = {s: [w * (4000.0 if k == 0 else 1.0) for k, w in enumerate(ws)] for s, ws in cw.items()}
    with torch.no_grad():
        for s in symbols:
            m.charge_networks.atomics[s].layers[0].weight.mul_(4000.0)
    sp, co, cell, pbc = inputs(rec)
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        out = m((sp, co), cell, pbc)
    assert any("3 x bfloat16" in str(w.message) for w in caught)
    assert m.neural_networks._variant == "bf16x3" and m.charge_networks._variant == "bf16x3"
    ref = cor.compute(oracle_model("mbis", rec, "cell_list", cw_big), torch.tensor(rec["species"]),
                      torch.tensor(rec["coords"]).float().double(), None, None, forces=False)
    assert_close("bf16x3 charges", out.atomic_charges.cpu().numpy(), ref["charges"].numpy(), 0.0,
                 2 * charge_bar(ref["charges"].numpy()))
    assert_close("bf16x3 energies", out.energies.double().cpu().numpy(), rec["energy"], 2e-7, 1e-3)


def test_rejections():
    from torchani_b200 import electro, models
    from torchani_b200.calculator import HostCalculator
    m = build_model("mbis")
    rec = fixture("mbis", "randbatch")
    sp, co, cell, pbc = inputs(rec)
    with pytest.raises(AssertionError):
        m((sp, co), charge=1)                      # the model asserts neutrality, as the reference
    with pytest.raises(ValueError):
        m.members_forces((sp, co))                 # no charges in the query-by-committee step
    eng = m.engine(torch.device(DEV))
    ws = eng.workspace(*sp.shape)
    eng._stage_inputs(sp, co, None, False)
    with pytest.raises(ValueError):
        eng.run(ws, False, members=True, charges=True)
    with pytest.raises(ValueError):
        eng.run(ws, False, shard=(0, 2), charges=True)
    with pytest.raises(NotImplementedError):
        m.compute_from_full_neighborlist(sp, co, None, None, None)
    with pytest.raises(ValueError):               # merged charge networks
        models.ANIq(m.symbols, m.aev_computer, m.neural_networks, m.energy_shifter, None, False, None)
    with pytest.raises(ValueError):               # tables are not shipped
        models.ANImbis()
    with pytest.raises(ValueError):
        electro.ChargeNormalizer.from_electronegativity_and_hardness(["H", "C"])
    with pytest.raises(ValueError):
        electro.DipoleComputer()
    with pytest.raises(ValueError):
        m.dipoles((sp, co), reference="center_of_mass")
    x = co.clone().requires_grad_(True)
    out = m((sp, x))
    with pytest.raises(NotImplementedError):       # charges carry no gradient
        torch.autograd.grad(out.atomic_charges.sum(), x)
    ani = models.ANI(m.symbols, m.aev_computer, m.neural_networks, m.energy_shifter, False).to(DEV)
    ani_host = HostCalculator(ani, rec["species"][0])
    with pytest.raises(ValueError):
        ani_host.calculate_with_charges(rec["coords"][0])


def test_animbis_and_compute_from_neighbors():
    """ANImbis with passed tables; compute_from_neighbors gives the forward's charges."""
    from torchani_b200 import models
    en = [2.2, 2.55, 3.04, 3.44, 2.58, 3.98, 3.16]
    hd = [6.4, 5.0, 7.2, 6.1, 4.1, 7.0, 4.7]
    m = models.ANImbis(device=DEV, electronegativity=en, hardness=hd)
    assert m.charge_networks.kept_output == 1 and m.charge_normalizer.scale_weights_by_charges_squared
    rec = fixture("mbis", "small264_nopbc")
    z = torch.tensor(rec["atomic_numbers"]).to(DEV)
    co = torch.tensor(rec["coords"]).float().to(DEV)
    out = m((z, co))
    assert float(out.atomic_charges.sum().abs()) < 1e-5 * float(out.atomic_charges.abs().sum()) + 1e-6
    elem = m.species_converter(z)
    nb = m.neighborlist(m.cutoff, elem, co)
    r = m.compute_from_neighbors(elem, co, nb)
    assert float((r.scalars - out.atomic_charges).abs().max()) < 1e-6
    assert float((r.energies.double() - out.energies.double()).abs().max()) < 1e-2


def _reference_mbis():
    import oracle.ref_torchani as rt
    if not os.path.isdir(os.path.join(rt.STAGED, "torchani")):
        pytest.skip("oracle/_ref (the staged reference) is not built")
    rt.load()
    import oracle.make_charge_golden as mcg
    ref, _ = mcg.reference_model("mbis")
    return ref.float().to(DEV)


@pytest.mark.parametrize("how", ["from_torchani", "accelerate"])
def test_dropin_of_a_reference_aniq(how):
    from torchani_b200 import models
    ref = _reference_mbis()
    rec = fixture("mbis", "small264_nopbc")
    z = torch.tensor(rec["atomic_numbers"]).to(DEV)
    co = torch.tensor(rec["coords"]).float().to(DEV)
    if how == "from_torchani":
        m = models.from_torchani(ref)
        assert isinstance(m, models.ANIq)
        out = m((z, co))
        e, q = out.energies, out.atomic_charges
    else:
        m = models.accelerate_torchani_(ref)
        out = m((z, co))
        e, q = out.energies, out.atomic_charges
    assert_close(f"{how} charges", q.cpu().numpy(), rec["charges"], 0.0, charge_bar(rec["charges"]))
    assert_close(f"{how} energies", e.double().cpu().numpy(), rec["energy"], 2e-7, 1e-3)
