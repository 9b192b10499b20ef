"""GPU parity of the fused engine (through the C-ABI) against the CPU oracle / golden vectors.

Bars (north_star): AEV and atomic energies 1e-5 relative, forces 1e-4 Ha/A, vs the float64
oracle evaluated on the same float32-rounded inputs (helpers.py spells out the tolerances)."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle.ani_oracle as orc
from helpers import (AEV_ATOL, AEV_RTOL, E_ATOL, E_RTOL, F_ATOL, GOLDEN_CASES, assert_close, golden_inputs,
                     load_golden, oracle_model)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engines():
    from torchani_b200.engine import Engine, PackedNetworks, constants_1x, constants_2x
    dev = torch.device("cuda:0")
    out = {}
    for kind, consts in (("2x", constants_2x()), ("1x", constants_1x())):
        m = oracle_model(kind)
        nets = PackedNetworks([[wm[s] for s in m.symbols] for wm in m.weights], consts.out_dim, dev)
        out[kind] = Engine(consts, nets, [m.sae[s] for s in m.symbols])
    return out


def gpu_aev(eng, species, coords, cell, pbc):
    """AEV forward only, returned in input order (C, A, D)."""
    from torchani_b200._lib import check, ptr
    dev = eng.device
    res = eng.step(species.to(dev), coords.to(dev), None if cell is None else cell.to(dev), pbc is not None,
                   want_grad=False)
    ws = eng.workspace(*species.shape)
    n = species.numel()
    st = torch.cuda.current_stream().cuda_stream
    plain = torch.zeros(ws.rows_cap, eng.nets.ldx, device=dev)
    check(eng.lib.ani_b200_aev_forward(C.byref(eng.params), ptr(ws.grid), ptr(ws.bin_start), ptr(ws.spos),
                                     ptr(ws.sbin), None, None, None, n, 0, n, ptr(ws.row_of), ptr(plain), eng.nets.ldx, 0,
                                     ptr(ws.nbr_cnt), ptr(ws.nbr_list), ws.nbr_cap, ptr(ws.status), st))
    # the plain rows once more with the step's own arguments (range table, bucket species, element mask): the same
    # kernel path and order of additions as the tiled operand the step wrote
    same = torch.zeros(ws.rows_cap, eng.nets.ldx, device=dev)
    check(eng.lib.ani_b200_aev_forward(C.byref(eng.params), ptr(ws.grid), ptr(ws.bin_start), ptr(ws.spos),
                                       ptr(ws.sbin), ptr(ws.bucket_ranges), ptr(ws.bucket_species),
                                       ws.aev_blocks.data_ptr() + 4 * (ws.n_blocks + 1), n, 0, n, ptr(ws.row_of),
                                       ptr(same), eng.nets.ldx, 0, ptr(ws.nbr_cnt), ptr(ws.nbr_list), ws.nbr_cap,
                                       ptr(ws.status), st))
    torch.cuda.synchronize()
    eng.check_status(ws)
    D = eng.consts.out_dim
    n_real = int((species >= 0).sum())
    so = ws.sorted_orig[:n_real].long()
    rows = ws.row_of[:n_real].long()
    # the engine's own AEV buffer holds the same numbers as 16-bit pieces: 2 x fp16 of 64*x, 22 bits and an absolute
    # floor of 2^-31; 3 x bf16, 24 bits (the whole float32 significand: exact but for the bfloat16 subnormal range)
    from torchani_b200.engine import untile_a_operand
    tiled = untile_a_operand(ws.x.reshape(-1), ws.rows_cap, eng.nets.ldx, variant=eng.variant)
    cols = torch.arange(D, device=dev)   # the tiled operand's internal column order: ang_pad zeros after the radial block
    cols = torch.where(cols < eng.nets.radial_len, cols, cols + eng.nets.col_pad) if eng.nets.col_pad else cols
    rel, floor = (2.0 ** -24, 2.0 ** -120) if eng.variant == "bf16x3" else (2.0 ** -21, 2.0 ** -30)
    err = (tiled[rows][:, cols] - same[rows, :D]).abs()
    assert bool((err <= same[rows, :D].abs() * rel + floor).all()), \
        f"tiled and plain AEV outputs differ by up to {float((err / same[rows, :D].abs().clamp(min=1e-30)).max()):.3e}"
    assert bool(((same[rows, :D] - plain[rows, :D]).abs() <= plain[rows, :D].abs() * 2.0 ** -21 + 2.0 ** -30).all())
    aev = torch.zeros(n, D, device=dev)
    aev[so] = plain[rows, :D]
    return aev.view(*species.shape, D).cpu(), res


def run_and_compare(eng, model, species, coords32, cell32, pbc):
    ref = orc.compute(model, species, coords32.double(), None if cell32 is None else cell32.double(), pbc)
    aev, _ = gpu_aev(eng, species, coords32, cell32, pbc)
    dev = eng.device
    res = eng.step(species.to(dev), coords32.to(dev), None if cell32 is None else cell32.to(dev),
                   pbc is not None, want_grad=True)
    torch.cuda.synchronize()
    eng.check_status()
    assert_close("aev", aev.numpy(), ref["aev"].numpy(), AEV_RTOL, AEV_ATOL)
    assert_close("member atomic energies", res.member_atomic.cpu().numpy(), ref["member_atomic"].numpy(),
                 E_RTOL, E_ATOL)
    assert_close("atomic energies", res.atomic_energies.cpu().numpy(), ref["atomic_nn"].numpy(), E_RTOL, E_ATOL)
    n_real = int((species >= 0).sum())
    assert_close("total energies", res.energies.cpu().numpy(), ref["energy"].numpy(), 0.0, 2e-7 * max(n_real, 10))
    assert_close("forces", -res.grad.cpu().numpy(), ref["forces"].numpy(), 0.0, F_ATOL)
    return ref, res


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_golden_cases(engines, name):
    rec = load_golden(name)
    species, coords, cell, pbc = golden_inputs(rec, torch.float32)
    eng = engines[rec["kind"]]
    model = oracle_model(rec["kind"], torch.float64, rec["neighborlist"])
    ref, res = run_and_compare(eng, model, species, coords, cell, pbc)
    # and against the reference-generated fixture itself (float64 inputs there, float32 here)
    assert np.abs(-res.grad.cpu().numpy() - rec["forces"]).max() < F_ATOL
    assert np.abs(res.member_atomic.cpu().numpy() - rec["member_atomic"]).max() < 2e-5
    ws = eng.workspace(*species.shape)
    n_real = int((species >= 0).sum())
    assert int(ws.nbr_cnt[:n_real].sum().item()) == 2 * int(rec["num_pairs"])
    if name == "sevenel_pbc_ani2x":   # every element pair present: every 32-column block of layer 1 is live
        assert int(ws.aev_blocks[0]) == 32


def test_composition_change_under_a_captured_graph():
    """A problem shape captured into a CUDA graph with two elements (water: H and O) and replayed with all seven.
    At capture time Engine.note_composition sizes the shared-memory gradient table of the AEV backward for two
    elements; on the replay the other element pairs are read from global memory.  The replay must still match the
    float64 oracle at the golden bars."""
    from torchani_b200.engine import Engine, PackedNetworks, constants_2x
    dev = torch.device("cuda:0")
    rec = load_golden("sevenel_pbc_ani2x")
    species, coords, cell, pbc = golden_inputs(rec, torch.float32)
    consts = constants_2x()
    m = oracle_model("2x")
    nets = PackedNetworks([[wm[s] for s in m.symbols] for wm in m.weights], consts.out_dim, dev)
    eng = Engine(consts, nets, [m.sae[s] for s in m.symbols])
    co, ce = coords.to(dev), cell.to(dev)
    water = torch.where(species == 0, 0, 3).to(dev)     # the same atoms as H and O only
    for _ in range(eng.graph_after + 1):                 # eager uses, then the capture
        eng.step(water, co, ce, True)
    eng.check_status()
    ws = eng.workspace(*species.shape)
    assert len(eng._graphs) == 1 and ws.max_elements == 2
    res = eng.step(species.to(dev), co, ce, True)       # a replay of that graph, now with seven elements
    torch.cuda.synchronize()
    eng.check_status()
    assert len(eng._graphs) == 1 and int(ws.aev_blocks[0]) == 32
    ref = orc.compute(oracle_model("2x", torch.float64, "cell_list"), species, coords.double(), cell.double(), pbc)
    assert_close("member atomic energies", res.member_atomic.cpu().numpy(), ref["member_atomic"].numpy(),
                 E_RTOL, E_ATOL)
    assert_close("total energies", res.energies.cpu().numpy(), ref["energy"].numpy(), 0.0, 2e-7 * species.numel())
    assert_close("forces", -res.grad.cpu().numpy(), ref["forces"].numpy(), 0.0, F_ATOL)
    assert np.abs(-res.grad.cpu().numpy() - rec["forces"]).max() < F_ATOL


def test_conformer_batch_256(engines):
    """BASELINE config 3: 256 GDB-like conformers, -1 padding, no PBC."""
    species, coords = orc.conformer_batch(256, seed=1234)
    model = oracle_model("2x", torch.float64, "all_pairs")
    run_and_compare(engines["2x"], model, species, coords, None, None)


def test_water_1k_box(engines):
    """BASELINE config 2: 999-atom periodic water box."""
    _, idx, coords, cell, pbc = orc.water_box(333, seed=5)
    run_and_compare(engines["2x"], oracle_model("2x", torch.float64, "cell_list"), idx, coords, cell, pbc)


def test_uniform_random_box_close_contacts(engines):
    """_testing.make_molecs-style uniform random HCNO box (worst-case close contacts)."""
    g = torch.Generator().manual_seed(11)
    n, L = 600, (600 / 0.1) ** (1 / 3)
    coords = (torch.rand(1, n, 3, generator=g) * L + 1e-3)
    idx = torch.randint(0, 4, (1, n), generator=g)
    cell = torch.eye(3) * (L + 2e-3)
    pbc = torch.tensor([True, True, True])
    model = oracle_model("2x", torch.float64, "cell_list")
    ref = orc.compute(model, idx, coords.double(), cell.double(), pbc)
    eng = engines["2x"]
    aev, res = gpu_aev(eng, idx, coords, cell, pbc)
    assert_close("aev", aev.numpy(), ref["aev"].numpy(), 2e-5, 2e-5)
    res = eng.step(idx.cuda(), coords.cuda(), cell.cuda(), True)
    # random overlaps give forces of O(10) Ha/A: judge them relative to that scale
    f_ref = ref["forces"].numpy()
    assert np.abs(-res.grad.cpu().numpy() - f_ref).max() <= 1e-5 * np.abs(f_ref).max() + F_ATOL


def test_water_10k_box_properties(engines):
    """BASELINE config 4 size: checked through size-independent properties + the oracle."""
    eng = engines["2x"]
    _, idx, coords, cell, pbc = orc.water_box(3333, seed=0)
    d = eng.device
    sp, co, ce = idx.to(d), coords.to(d), cell.to(d)
    r0 = eng.step(sp, co, ce, True)
    e0, g0, at0 = r0.energies.clone(), r0.grad.clone(), r0.atomic_energies.clone()
    eng.check_status()
    # Newton's third law: the net force vanishes
    assert float(g0.sum(1).abs().max()) < 5e-5
    # energy is the sum of atomic energies + self energies
    sae = torch.tensor([orc.GSAES_WB97X_631GD[s] for s in orc.SYMBOLS_2X], dtype=torch.float64, device=d)
    assert abs(float(at0.double().sum() + sae[sp].sum() - e0[0])) < 1e-6 * 9999
    # translation by an arbitrary vector (atoms leave the cell and are wrapped back)
    shift = torch.tensor([3.21, -47.5, 101.3], device=d)
    r1 = eng.step(sp, co + shift, ce, True)
    assert abs(float(r1.energies[0] - e0[0])) < 2e-4
    assert float((r1.grad - g0).abs().max()) < 2e-5
    # permutation of the atom order
    perm = torch.randperm(9999, generator=torch.Generator().manual_seed(1)).to(d)
    r2 = eng.step(sp[:, perm], co[:, perm], ce, True)
    assert abs(float(r2.energies[0] - e0[0])) < 1e-5
    assert float((r2.grad - g0[:, perm]).abs().max()) < 2e-5
    # sharded evaluation (what every rank of a multi-GPU run computes) adds up to the whole
    parts_e, parts_g = 0.0, torch.zeros_like(g0)
    for r in range(4):
        rr = eng.step(sp, co, ce, True, shard=(r, 4))
        parts_e += float(rr.energies[0])
        parts_g += rr.grad
    assert abs(parts_e - float(e0[0])) < 1e-5
    assert float((parts_g - g0).abs().max()) < 2e-5
    # finally the oracle itself at full size (float64, a few seconds)
    ref = orc.compute(oracle_model("2x", torch.float64, "cell_list"), idx, coords.double(), cell.double(), pbc)
    assert_close("forces", -g0.cpu().numpy(), ref["forces"].numpy(), 0.0, F_ATOL)
    assert_close("atomic energies", at0.cpu().numpy(), ref["atomic_nn"].numpy(), E_RTOL, E_ATOL)
    assert abs(float(e0[0]) - float(ref["energy"][0])) < 5e-3


def test_forces_are_the_gradient_of_the_energy(engines):
    """Central finite differences of the float64-accumulated energy vs the analytic forces."""
    eng = engines["2x"]
    rec = load_golden("water30_pbc_ani2x")
    species, coords, cell, pbc = golden_inputs(rec, torch.float32)
    d = eng.device
    sp, ce = species.to(d), cell.to(d)
    res = eng.step(sp, coords.to(d), ce, True)
    grad = res.grad.clone().cpu()
    h = 2e-3
    for (a, k) in [(0, 0), (7, 2), (13, 1), (29, 0)]:
        cp, cm = coords.clone(), coords.clone()
        cp[0, a, k] += h
        cm[0, a, k] -= h
        ep = float(eng.step(sp, cp.to(d), ce, True, want_grad=False).energies[0])
        em = float(eng.step(sp, cm.to(d), ce, True, want_grad=False).energies[0])
        assert abs((ep - em) / (2 * h) - float(grad[0, a, k])) < 2e-4


def test_edge_cases(engines):
    eng = engines["1x"]
    d = eng.device
    rca, rcr = 3.5, 5.2
    # tests/test_aev.py:61-131: atoms exactly at / just beyond the cutoffs, lone atom
    for dist in [1.0, rca, rca + 1e-4, rcr, rcr + 1e-4, 2 * rcr]:
        coords = torch.tensor([[[-dist, 0.0, 0.0], [0.0, 0.0, 0.0], [0.0, 0.0, dist]]])
        species = torch.tensor([[3, 1, 3]])
        ref = orc.compute(oracle_model("1x", torch.float64, "all_pairs"), species, coords.double())
        aev, res = gpu_aev(eng, species, coords, None, None)
        assert_close(f"aev d={dist}", aev.numpy(), ref["aev"].numpy(), AEV_RTOL, AEV_ATOL)
    aev, res = gpu_aev(eng, torch.tensor([[0]]), torch.zeros(1, 1, 3), None, None)
    assert float(aev.abs().max()) == 0.0
    # coincident atoms: no NaN (tests/test_aev.py:184-189)
    coords = torch.tensor([[[0.0, 0.0, 0.0], [0.0, 0.0, 0.0], [1.0, 0.0, 0.0]]])
    res = eng.step(torch.tensor([[0, 0, 1]], device=d), coords.to(d), None, False)
    assert bool(torch.isfinite(res.grad).all()) and bool(torch.isfinite(res.energies).all())
    # a fully padded conformer in a batch gives zero energy and zero AEV
    species = torch.tensor([[1, 0, 0, 0, 0], [-1, -1, -1, -1, -1]])
    coords = torch.randn(2, 5, 3, generator=torch.Generator().manual_seed(0))
    res = eng.step(species.to(d), coords.to(d), None, False)
    assert float(res.energies[1]) == 0.0 and float(res.grad[1].abs().max()) == 0.0
    # periodic cell thinner than the cutoff is an error (neighbors.py:402-403)
    eng2 = engines["2x"]
    res = eng2.step(torch.zeros(1, 4, dtype=torch.long, device=d), torch.rand(1, 4, 3, device=d),
                    torch.eye(3, device=d) * 4.0, True)
    with pytest.raises(RuntimeError, match="too small"):
        eng2.check_status()


def test_smooth_cutoff_and_active_members(engines):
    from torchani_b200.engine import Engine, constants_2x
    eng = engines["2x"]
    rec = load_golden("benzene_pbc_ani2x")
    species, coords, cell, pbc = golden_inputs(rec, torch.float32)
    # smooth cutoff (cutoffs.py:84-101)
    eng_s = Engine(constants_2x(cutoff_fn="smooth"), eng.nets, None)
    m = oracle_model("2x", torch.float64, "cell_list")
    m = m._replace(spec=m.spec._replace(cutoff_fn="smooth"))
    run_and_compare(eng_s, m._replace(sae={s: 0.0 for s in m.symbols}), species, coords, cell, pbc)
    # subset of active ensemble members (nn/_core.py:99-110)
    eng.nets.set_active_members([1, 4, 6])
    try:
        d = eng.device
        res = eng.step(species.to(d), coords.to(d), cell.to(d), True)
        ref = orc.compute(oracle_model("2x", torch.float64, "cell_list"), species, coords.double(), cell.double(),
                          pbc, members=[1, 4, 6])
        assert_close("atomic", res.atomic_energies.cpu().numpy(), ref["atomic_nn"].numpy(), E_RTOL, E_ATOL)
        assert_close("forces", -res.grad.cpu().numpy(), ref["forces"].numpy(), 0.0, F_ATOL)
    finally:
        eng.nets.set_active_members(list(range(8)))


def test_protein_in_water_50k_properties(engines):
    """BASELINE config 5 size (1C17 protein, H C N O S, in lattice water, ~50k atoms): five elements live, so the
    block-sparse layer 1 runs 20 of its 32 AEV column blocks (water: 5).  Size-independent properties at full size;
    value parity of an all-five-element system is the golden case 1c17_chunk_hcnos_ani2x (real reference)."""
    from torchani_b200 import synthetic
    eng = engines["2x"]
    d = eng.device
    _, idx, coords, cell, _ = synthetic.protein_in_water(50001, seed=0)
    n = idx.shape[1]
    assert 49000 < n <= 50001 and set(idx.unique().tolist()) == {0, 1, 2, 3, 4}
    sp, co, ce = idx.to(d), coords.to(d), cell.to(d)
    r0 = eng.step(sp, co, ce, True)
    e0, g0, at0 = r0.energies.clone(), r0.grad.clone(), r0.atomic_energies.clone()
    eng.check_status()
    assert bool(torch.isfinite(g0).all()) and bool(torch.isfinite(at0).all())
    scale = float(g0.abs().max())
    assert float(g0.double().sum(1).abs().max()) < 1e-6 * n * max(1.0, scale)          # Newton's third law
    sae = torch.tensor([orc.GSAES_WB97X_631GD[s] for s in orc.SYMBOLS_2X], dtype=torch.float64, device=d)
    assert abs(float(at0.double().sum() + sae[sp].sum() - e0[0])) < 1e-6 * n
    shift = torch.tensor([13.7, -80.2, 5.5], device=d)                                   # translation, re-wrapping
    r1 = eng.step(sp, co + shift, ce, True)
    assert abs(float(r1.energies[0] - e0[0])) < 2e-3
    assert float((r1.grad - g0).abs().max()) < 1e-4 * max(1.0, scale)
    parts_e, parts_g = 0.0, torch.zeros_like(g0)                                         # what 8 ranks would compute
    for r in range(8):
        rr = eng.step(sp, co, ce, True, shard=(r, 8))
        parts_e += float(rr.energies[0])
        parts_g += rr.grad
    assert abs(parts_e - float(e0[0])) < 1e-4
    assert float((parts_g - g0).abs().max()) < 1e-4 * max(1.0, scale)


@pytest.mark.parametrize("n_mol", [20, 333, 800, 3333])
def test_dataflow_mlp_launch_matches_the_chained_launches(engines, n_mol):
    """The two ways the MLP of a step is launched -- one persistent data-flow launch (csrc/gemm_tc.cuh) and the
    six chained launches (csrc/gemm_tc.cuh) -- run the same tile code and must agree to rounding (the split-K
    accumulation order of the layer-1 backward is not fixed), on lists much shorter than, comparable to and much
    longer than the number of SMs; both agree with the oracle through the golden cases."""
    from torchani_b200 import synthetic
    eng = engines["2x"]
    d = eng.device
    _, idx, coords, cell, _ = synthetic.water_box(n_mol, seed=11)
    sp, co, ce = idx.to(d), coords.to(d), cell.to(d)
    saved = eng.mlp_mode
    try:
        out = {}
        for mode in ("0", "1"):
            eng.mlp_mode = mode
            for _ in range(5):          # eager uses, then the captured graph (replays must agree too)
                r = eng.step(sp, co, ce, True)
            out[mode] = (r.energies.clone(), r.grad.clone(), r.member_atomic.clone())
            eng.check_status()
        assert abs(float(out["0"][0][0] - out["1"][0][0])) < 1e-6 * max(1, 3 * n_mol)
        assert float((out["0"][1] - out["1"][1]).abs().max()) < 2e-6
        assert float((out["0"][2] - out["1"][2]).abs().max()) < 1e-6
    finally:
        eng.mlp_mode = saved


@pytest.mark.parametrize("n_mol,shard,dilate", [(10, (0, 1), 1.0), (333, (0, 1), 1.0), (3333, (0, 1), 1.0),
                                                (3333, (1, 4), 1.0), (5000, (3, 8), 1.0), (20, (0, 1), 4.0)])
def test_cluster_preparation_matches_the_persistent_grid_kernel(n_mol, shard, dilate, monkeypatch):
    """ani_b200_prepare_step has two single-launch forms: a persistent grid with device-wide barriers
    (k_prep_fused) and, for periodic single systems of MD size, one thread-block cluster (k_prep_cluster).
    Everything they hand to the rest of the step must be bit-identical: the bucket grid, the deterministic
    (bucket, species, input index) order, the neighbour-range table, the row layout and the live AEV blocks --
    for the whole system and for the owned slice of a rank."""
    from torchani_b200 import synthetic
    from torchani_b200.engine import Engine, PackedNetworks, constants_2x
    dev = torch.device("cuda:0")
    consts = constants_2x()
    m = oracle_model("2x")
    nets = PackedNetworks([[wm[s] for s in m.symbols] for wm in m.weights], consts.out_dim, dev)
    _, idx, coords, cell, _ = synthetic.water_box(n_mol, seed=3)
    coords, cell = coords * dilate, cell * dilate   # dilate > 1: a dilute system with more buckets than atoms
    idx = idx.clone()
    idx[0, 5] = -1      # one padding atom: the trash bucket is exercised too
    sp, co, ce = idx.to(dev), coords.to(dev), cell.to(dev)
    out = {}
    for flag in ("0", "1"):
        monkeypatch.setenv("ANI_B200_PREP_CLUSTER", flag)
        eng = Engine(consts, nets, [m.sae[s] for s in m.symbols], cuda_graph=False)
        for _ in range(2):   # the second call starts from the first one's leftovers in the scratch area
            r = eng.step(sp, co, ce, True, shard=shard)
        eng.check_status()
        ws = eng.workspace(*idx.shape)
        grid = ws.grid.clone()
        nbins = int(grid.cpu()[25])   # ani_grid: 21 floats, dims[3], pbc, nbins, ...
        rec = dict(grid=grid, bin_start=ws.bin_start[:nbins + 2].clone(), sorted_orig=ws.sorted_orig.clone(),
                   orig_to_sorted=ws.orig_to_sorted.clone(), spos=ws.spos.clone(), sbin=ws.sbin.clone(),
                   ranges=ws.bucket_ranges[:nbins * 27 * 8].clone().view(torch.int32),
                   row_atom=ws.row_atom.clone(), tile_species=ws.tile_species.clone(),
                   layout_info=ws.layout_info.clone(), aev_blocks=ws.aev_blocks[:ws.n_blocks + 2].clone(),
                   energies=r.energies.clone(), grad=r.grad.clone())
        lo = int(ws.n * shard[0] // shard[1])
        hi = int(ws.n * (shard[0] + 1) // shard[1])
        n_real = int(rec["bin_start"][nbins])
        rec["row_of"] = ws.row_of[lo:min(hi, n_real)].clone()
        out[flag] = rec
        assert nbins > 0
    for k in out["0"]:
        a, b = out["0"][k], out["1"][k]
        if k in ("energies", "grad"):
            assert torch.allclose(a, b, rtol=0, atol=2e-6), k    # (split-K order of the layer-1 backward)
        elif k == "spos":
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), k
        else:
            assert torch.equal(a, b), k


def test_aligned_angular_block_and_row_tile_windows(monkeypatch):
    """Two internal re-arrangements that must not change any result: (i) the angular block of the tiled AEV operand
    starts on a 32-column boundary (ani_aev_params::ang_pad; water then has 5 live GEMM blocks instead of 8) --
    compared with networks packed in the reference's column order; (ii) the data-flow MLP launch cut into windows of
    the row tiles (ANI_B200_MLP_CHUNKS) -- compared with one launch over all row tiles."""
    from torchani_b200 import synthetic
    from torchani_b200.engine import Engine, PackedNetworks, constants_2x
    dev = torch.device("cuda:0")
    consts = constants_2x()
    m = oracle_model("2x")
    w = [[wm[s] for s in m.symbols] for wm in m.weights]
    sae = [m.sae[s] for s in m.symbols]
    _, idx, coords, cell, _ = synthetic.water_box(1000, seed=5)
    sp, co, ce = idx.to(dev), coords.to(dev), cell.to(dev)
    out = {}
    for name, rl, chunks in (("ref_order", 0, "1"), ("aligned", consts.num_species * len(consts.shf_r), "1"),
                             ("aligned_windows", consts.num_species * len(consts.shf_r), "3")):
        monkeypatch.setenv("ANI_B200_MLP_CHUNKS", chunks)
        nets = PackedNetworks(w, consts.out_dim, dev, radial_len=rl)
        eng = Engine(consts, nets, sae, cuda_graph=False)
        eng.mlp_mode = "1"
        r = eng.step(sp, co, ce, True)
        eng.check_status()
        ws = eng.workspace(*idx.shape)
        out[name] = (r.energies.clone(), r.grad.clone(), r.member_atomic.clone(), int(ws.aev_blocks[0]), nets.col_pad)
    assert out["ref_order"][4] == 0 and out["aligned"][4] == 16
    assert out["ref_order"][3] == 8 and out["aligned"][3] == 5      # live 32-column blocks of a water box
    for name in ("aligned", "aligned_windows"):
        assert abs(float(out[name][0][0] - out["ref_order"][0][0])) < 3e-3, name
        assert float((out[name][1] - out["ref_order"][1]).abs().max()) < 2e-6, name
        assert float((out[name][2] - out["ref_order"][2]).abs().max()) < 1e-6, name


@pytest.mark.parametrize("n_mol,depth", [(20, "0"), (333, "2"), (3333, "0"), (3333, "3")])
def test_independent_chain_mlp_launch_matches_the_chained_launches(engines, n_mol, depth, monkeypatch):
    """The opt-in third schedule of the MLP (csrc/gemm_tc.cuh, ANI_B200_MLP_CHAIN=1): a CTA owns whole (row tile,
    member) chains and interleaves them, no synchronisation between CTAs.  Same tile code, so it must agree with the six
    chained launches to rounding -- with fewer chains than SMs, a handful per CTA, and a fixed interleave depth."""
    from torchani_b200 import synthetic
    eng = engines["2x"]
    d = eng.device
    _, idx, coords, cell, _ = synthetic.water_box(n_mol, seed=13)
    sp, co, ce = idx.to(d), coords.to(d), cell.to(d)
    saved, saved_graph = eng.mlp_mode, eng.cuda_graph
    try:
        eng.cuda_graph = False
        out = {}
        for mode, chain in (("0", "0"), ("1", "1")):
            monkeypatch.setenv("ANI_B200_MLP_CHAIN", chain)
            monkeypatch.setenv("ANI_B200_CHAIN_DEPTH", depth)
            eng.mlp_mode = mode
            for _ in range(2):
                r = eng.step(sp, co, ce, True)
            out[mode] = (r.energies.clone(), r.grad.clone(), r.member_atomic.clone())
            eng.check_status()
        assert abs(float(out["0"][0][0] - out["1"][0][0])) < 1e-6 * max(1, 3 * n_mol)
        assert float((out["0"][1] - out["1"][1]).abs().max()) < 2e-6
        assert float((out["0"][2] - out["1"][2]).abs().max()) < 1e-6
    finally:
        eng.mlp_mode, eng.cuda_graph = saved, saved_graph
