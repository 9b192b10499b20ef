"""The resident-chain MLP launch (ani_b200_mlp_step_resident, csrc/mlp_resident.cuh) against float64, and against the
data-flow launch inside the engine.

Kernel level: the same synthetic weights, species-grouped rows, AEV-like and wide-range inputs, float64 reference and
bars as tests/test_gpu_mlp.py.  The launch keeps the gradient pieces G3, G2, G1 in shared memory, so what is compared is
what leaves it: the activations a1, a2 in act1 / act2, the per-member energies and dE/dAEV.  The contracts beyond the
values are checked too: padding rows get e_member = 0, dead dE/dAEV blocks, rows past the layout and the guard bands
around dx keep their sentinel, an operand out of the fp16 pieces' range raises the status bit, and a model the kernel
cannot hold (a hidden width above 256, or the 3 x bf16 build) is refused with ANI_ERR_UNSUPPORTED.

Engine level: on the 10k-atom water box and the 50k-atom protein in water, the engine's default launch (resident
chains) and the data-flow launch (mlp_mode "1") must agree to the order of the members' dE/dAEV additions."""
import ctypes as C
import typing as tp

import pytest
import torch

from helpers import E_ATOL, E_RTOL
from test_gpu_mlp import (BLOCKS, DEV, EPS, GUARD, MODEL_BARS, R2X, ROW_BARS, SENTINEL, TILE, WIDTHS, Case,
                          compare_rows, make_layout, make_x, packed, reference, reference_weights)

pytestmark = pytest.mark.gpu

ERR_UNSUPPORTED = -2


CASES = [
    # 2x widths, rows 0 / 1 / 127 / 128 / 129 per species in one launch; every block list with and without b1_compact
    Case("dense"),
    Case("water5", blocks="water5"),
    Case("water5_nocompact", blocks="water5", compact=False),
    Case("all32", blocks="all32"),
    Case("all32_nocompact", blocks="all32", compact=False),
    Case("scattered", blocks="scattered"),
    Case("scattered_nocompact", blocks="scattered", compact=False),
    Case("one_block", blocks="one"),
    Case("one_block_nocompact", blocks="one", compact=False),
    # member counts (M = 1: plain stores into dx, no zero-fill) and an active subset of M = 16
    Case("M1", M=1, blocks="water5"),
    Case("M3", M=3, blocks="scattered"),
    Case("M16_active_subset", M=16, blocks="all32", active=(0, 3, 4, 9, 15)),
    Case("G_rows_8k", rows=(3000, 1500, 400, 700, 100, 60, 40), rows_cap=8192, blocks="water5"),
    # widths
    Case("ani1x_padded_widths", widths="1x", rows=(200, 130, 60, 1)),
    Case("h32", widths="h32", M=3, rows=(128, 129, 5), blocks="scattered"),
    Case("h3_256", widths="h3_256", rows=(300, 129), blocks="all32"),
]
CASES += [c._replace(name=c.name + "-wide_range", values="wide") for c in CASES]


def _setup(case: Case):
    from torchani_b200 import _lib
    L = _lib.lib(case.variant)
    symbols, dims, in_dim = WIDTHS[case.widths]
    S, M = len(symbols), case.M
    nets = packed(case.widths, M, case.variant)
    seed = sum(map(ord, case.name)) + 17
    n = sum(case.rows) + 2
    rows_cap = max((n + S * (TILE - 1) + TILE - 1) // TILE * TILE, case.rows_cap)
    row_atom, layout_info, first = make_layout(L, case.rows, S, rows_cap, seed)
    active = list(case.active) if case.active is not None else list(range(M))
    model = _lib.MLPModel.from_buffer_copy(nets.model)
    for m in range(_lib.ANI_MAX_MEMBERS):
        model.member_scale[m] = (1.0 / len(active)) if m in active else 0.0
    if not case.compact:
        model.b1_compact = None
    return L, nets, model, rows_cap, row_atom, layout_info, first, seed


def _call(L, model, case: Case, nets, rows_cap, row_atom, layout_info, x_t, blk, act, e_member, dx, status) -> int:
    from torchani_b200._lib import ptr
    st = torch.cuda.current_stream(DEV).cuda_stream
    return L.ani_b200_mlp_step_resident(C.byref(model), ptr(x_t), ptr(dx), rows_cap, ptr(row_atom), ptr(layout_info),
                                        ptr(blk), ptr(act[0]), ptr(act[1]), ptr(e_member), ptr(status), st)


def _buffers(case: Case, nets, rows_cap: int, ldx: int, blocks):
    from torchani_b200.engine import operand_buffer
    blk = None
    if blocks is not None:
        blk = torch.zeros(ldx // 32 + 3, dtype=torch.int32, device=DEV)
        blk[0] = len(blocks)
        blk[1:1 + len(blocks)] = torch.tensor(blocks, dtype=torch.int32)
    act = [operand_buffer(rows_cap, w, DEV, case.variant) for w in nets.ld[:2]]
    e_member = torch.full((case.M, rows_cap), SENTINEL, dtype=torch.float32, device=DEV)
    dx_all = torch.full((2 * GUARD + rows_cap * ldx,), SENTINEL, dtype=torch.float32, device=DEV)
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    return blk, act, e_member, dx_all, status


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_resident_mlp_matches_float64(case: Case):
    from torchani_b200 import _lib
    from torchani_b200._lib import check
    from torchani_b200.engine import tile_a_operand, untile_a_operand
    fmt = _lib.operand_format(case.variant)
    model_bar = 0.0 if case.values == "aev" else MODEL_BARS[case.variant]
    row_bar = ROW_BARS[case.variant]
    symbols, dims, in_dim = WIDTHS[case.widths]
    S, M = len(symbols), case.M
    L, nets, model, rows_cap, row_atom, layout_info, first, seed = _setup(case)
    ldx = nets.ldx
    blocks = BLOCKS[case.blocks]
    live_blocks = blocks if blocks is not None else list(range(ldx // 32))
    live_cols = (torch.tensor(live_blocks, device=DEV).view(-1, 1) * 32 + torch.arange(32, device=DEV)).view(-1)
    x_t = tile_a_operand(make_x(case, rows_cap, ldx, in_dim, live_cols, seed), variant=case.variant)
    blk, act, e_member, dx_all, status = _buffers(case, nets, rows_cap, ldx, blocks)
    dx = dx_all[GUARD:GUARD + rows_cap * ldx]
    check(_call(L, model, case, nets, rows_cap, row_atom, layout_info, x_t, blk, act, e_member, dx, status),
          "mlp_step_resident")
    torch.cuda.synchronize()
    assert int(status.item()) == 0, f"status word {int(status.item())}"

    x64 = untile_a_operand(x_t, rows_cap, ldx, variant=case.variant).double()
    x64[:, ~torch.isin(torch.arange(ldx, device=DEV), live_cols)] = 0.0
    rws = reference_weights(case.widths, M, ldx)
    scale = torch.tensor([model.member_scale[m] for m in range(M)], dtype=torch.float64, device=DEV)
    ld = nets.ld
    got = {"a1": untile_a_operand(act[0], rows_cap, ld[0], fmt.value_scale, variant=case.variant),
           "a2": untile_a_operand(act[1], rows_cap, ld[1], fmt.value_scale, variant=case.variant)}
    tag = "resident " + ("aev" if case.values == "aev" else "wide")
    ra = row_atom.cpu()
    fails: tp.List[str] = []
    dxv = dx.view(rows_cap, ldx)
    for s in range(S):
        r0, r1 = first[s] * TILE, first[s + 1] * TILE
        if r1 == r0:
            continue
        valid = (ra[r0:r1] >= 0).to(DEV)
        ref = reference(rws[s], x64[r0:r1], valid, scale, False, model_bar)
        p = rws[s]["p"]
        where = f"{case.name} species {symbols[s]}"
        for k, v in got.items():
            w = p[0 if k == "a1" else 1]
            mine = v[r0:r1].view(r1 - r0, -1)[:, :M * w].view(r1 - r0, M, w).permute(1, 0, 2)
            compare_rows(f"{tag} activations", mine, ref[k], ref["d" + k], row_bar, model_bar, f"{where}: {k}", fails)
        em = e_member[:, r0:r1].double()
        bound = E_ATOL + E_RTOL * ref["e"].abs() + model_bar * EPS * ref["de"]
        real = valid.view(1, -1).expand_as(em)
        if not bool(((em - ref["e"]).abs() <= bound)[real].all()):
            fails.append(f"{where}: e_member off by {float((em - ref['e']).abs()[real].max()):.3e}")
        if bool((~real).any()):
            assert float(em[~real].abs().max()) == 0.0, f"{where}: padding rows must get e_member = 0"
        compare_rows(f"{tag} dE/dAEV", dxv[r0:r1][:, live_cols].double(), ref["dx"][:, live_cols],
                     ref["ddx"][:, live_cols], row_bar, model_bar, f"{where}: dE/dAEV", fails)
    assert not fails, "\n".join(fails)
    used = first[S] * TILE
    dead = ~torch.isin(torch.arange(ldx, device=DEV), live_cols)
    if bool(dead.any()):
        assert bool((dxv[:, dead] == SENTINEL).all()), "a dead column block of dE/dAEV was written"
    assert bool((dxv[used:] == SENTINEL).all()), "rows beyond the layout's row tiles were written"
    assert bool((e_member[:, used:] == SENTINEL).all()), "e_member rows beyond the layout were written"
    assert bool((dx_all[:GUARD] == SENTINEL).all()) and bool((dx_all[-GUARD:] == SENTINEL).all()), \
        "dE/dAEV written outside [rows_cap][ldx]"


def test_resident_mlp_reports_operand_range_overflow():
    from torchani_b200._lib import STATUS_OPERAND_RANGE, check
    from torchani_b200.engine import tile_a_operand
    case = Case("over_operand_limit", values="over_limit")
    L, nets, model, rows_cap, row_atom, layout_info, first, seed = _setup(case)
    ldx = nets.ldx
    live_cols = torch.arange(ldx, device=DEV)
    x_t = tile_a_operand(make_x(case, rows_cap, ldx, WIDTHS["2x"][2], live_cols, seed))
    blk, act, e_member, dx_all, status = _buffers(case, nets, rows_cap, ldx, None)
    check(_call(L, model, case, nets, rows_cap, row_atom, layout_info, x_t, blk, act, e_member,
                dx_all[GUARD:GUARD + rows_cap * ldx], status), "mlp_step_resident")
    torch.cuda.synchronize()
    assert int(status.item()) & STATUS_OPERAND_RANGE, "the operand range overflow was not reported"


@pytest.mark.parametrize("case", [Case("h1_288", widths="h1_wide", M=4, rows=(300, 129, 1)),
                                  Case("bf16x3", variant="bf16x3")], ids=["h1_288", "bf16x3"])
def test_resident_mlp_refuses_what_it_cannot_hold(case: Case):
    from torchani_b200 import _lib
    if case.variant and not _lib.available(case.variant):
        pytest.skip(f"{_lib.variant_path(case.variant)} has not been built")
    L, nets, model, rows_cap, row_atom, layout_info, first, seed = _setup(case)
    ldx = nets.ldx
    x_t = torch.zeros(rows_cap * ldx * 4, dtype=torch.uint8, device=DEV)
    blk, act, e_member, dx_all, status = _buffers(case, nets, rows_cap, ldx, None)
    rc = _call(L, model, case, nets, rows_cap, row_atom, layout_info, x_t, blk, act, e_member, dx_all, status)
    torch.cuda.synchronize()
    assert rc == ERR_UNSUPPORTED
    assert bool((dx_all == SENTINEL).all()) and bool((e_member == SENTINEL).all())


@pytest.fixture(scope="module")
def engine_2x():
    from helpers import oracle_model
    from torchani_b200.engine import Engine, PackedNetworks, constants_2x
    consts = constants_2x()
    m = oracle_model("2x")
    nets = PackedNetworks([[wm[s] for s in m.symbols] for wm in m.weights], consts.out_dim, DEV)
    return Engine(consts, nets, [m.sae[s] for s in m.symbols])


@pytest.mark.parametrize("system", ["water10k", "protein50k"])
def test_resident_launch_matches_the_dataflow_launch(engine_2x, system):
    """Same step, two MLP launches: energies to 1e-6 relative, forces to 1e-5 Ha/A.  The resident chains add the
    members' dE/dAEV contributions in another order than the data-flow launch (which contracts member pairs or
    quadruples in one accumulator); that is the only difference left."""
    from torchani_b200 import synthetic
    eng = engine_2x
    if system == "water10k":
        _, idx, coords, cell, _ = synthetic.water_box(3333, seed=0)
    else:
        _, idx, coords, cell, _ = synthetic.protein_in_water(50001, seed=0)
    sp, co, ce = idx.to(DEV), coords.to(DEV), cell.to(DEV)
    saved = eng.mlp_mode
    out = {}
    try:
        for mode in ("auto", "1"):
            eng.mlp_mode = mode
            for _ in range(5):          # eager uses, then the captured graph (replays must agree too)
                r = eng.step(sp, co, ce, True)
            eng.check_status()
            assert eng.mlp_resident == (mode == "auto") and eng.mlp_fused
            out[mode] = (r.energies.clone(), r.grad.clone(), r.member_atomic.clone())
    finally:
        eng.mlp_mode = saved
    (e_r, g_r, m_r), (e_d, g_d, m_d) = out["auto"], out["1"]
    assert abs(float(e_r[0] - e_d[0])) <= 1e-6 * abs(float(e_d[0]))
    assert float((g_r - g_d).abs().max()) < 1e-5
    assert float((m_r - m_d).abs().max()) < 1e-5
