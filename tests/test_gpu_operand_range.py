"""The operand-range checks of the 2 x fp16 build, at every site, on both sides of the limit.

Every GEMM operand of the default build is stored as two IEEE half pieces of s * x (s = 64 for AEVs and activations,
s = 4096 for the gradients dE/d(activation); DESIGN.md section 3).  A producer raises ANI_STATUS_OPERAND_RANGE when a
value it stores has |s * x| > 65504 (the largest half) or is NaN: |x| > 1023.5 for values, |g| > 65504 / 4096 =
15.9921875 for gradients.  The sites are the tiled-AEV writer of the AEV forward kernels, the k_gemm_wg epilogues
(a1, a2, the head's seed G3, G2, G1) and the epilogues of the resident-chain launch.

MLP sites.  Synthetic weights (three species of hidden widths 32, four members) where one neuron puts exactly the
target value on the site a case names and nothing else near a limit:
* a1 / a2: a zero weight row and bias T give CELU(z) = T; the next layer ignores that neuron (zero column);
* G3 = member_scale * w4 * CELU'(z3): a neuron with z3 = 1 > 0 and w4 = T / member_scale;
* G2 = W3^T G3 * CELU'(z2) and G1 = W2^T G2 * CELU'(z1): a chain of neurons with z > 0 and one weight T.
Each case asserts on the host, with the float64 reference, that the named site reaches T and every other site stays
well inside the range.  Below the limit (T = 1023.0 / 15.98) the status word must stay 0 and every output must meet
the plain bars of tests/test_gpu_mlp.py (ROW_BARS, e_member 1e-5 relative + 1e-6) against float64: accuracy holds up to
the edge.  Above it (T = 1023.6 / 15.994, so 65504 < s * T < 65520) the bit must be set, the call must succeed and
nothing may be written outside dE/dAEV's live blocks of the layout's rows.  In that band a half rounds to 65504, not to
inf, so both pieces stay finite and only the site's own check can raise the bit: a value of 1024 would give inf pieces,
the next GEMM would multiply them by the zero weights that isolate the site, and the NaN would be flagged one layer
later even with the site's check removed.  A NaN bias is flagged in both kinds of epilogue (max_abs_nan), and the
exact rule is pinned at 1023.49 / 1023.51.

AEV writer.  A central atom with a tight cap of k neighbours 0.8 A away (ShfA[0]): the angular features grow like k^2.
The float64 oracle puts the largest feature at 1015.4 for k = 40 and above 1123.5 for k = 48 (asserted on the host).
The default CTA kernel and the explicit-rows entry point (ani_b200_aev_forward_rows, on the oracle's pair list) run
here; the warp-per-atom, TMA-staged and per-bucket species offset paths are chosen once per process and run in child
processes.

The module prints the worst error / bar of every group of below-limit cases at its end (pytest -s).
"""
import ctypes as C
import math
import os
import subprocess
import sys
import typing as tp

import numpy as np
import pytest
import torch

import oracle.ani_oracle as orc
from helpers import E_ATOL, E_RTOL
from test_gpu_mlp import (DEV, GUARD, ROW_BARS, SENTINEL, TILE, WIDTHS, BLOCKS, Case, compare_rows, make_layout,
                          make_x, reference, reference_weights)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HALF_MAX = 65504.0
VALUE_LIMIT = HALF_MAX / 64.0       # 1023.5
GRAD_LIMIT = HALF_MAX / 4096.0      # 15.9921875
# target values below / above the limit, far enough from it that fp32 rounding of the produced value cannot cross it.
# Above it, s * T stays below 65520, where a half rounds to 65504 rather than to inf: both pieces of the stored value
# are finite, so no inf * 0 = NaN downstream can raise the bit in the next GEMM's epilogue in place of the site's own
# check.
TARGETS = {"value": (1023.0, 1023.6), "grad": (15.98, 15.994)}
HALF_INF_FROM = 65520.0
SITES = {"a1": "value", "a2": "value", "G3": "grad", "G2": "grad", "G1": "grad"}
I1, K2, J3 = 3, 5, 0                # the neurons of layers 1, 2, 3 that carry the target
WIDTH, M = "h32", 4
ROWS = (129, 1, 40)
ENTRIES = {   # name -> want_backward
    "chained": 1, "chained_forward": 0, "dataflow": 1, "dataflow_forward": 0, "split": 1, "chain": 1,
    "resident": 1, "slabs": 2,
}

_WORST: tp.Dict[str, float] = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if _WORST:
        print("\nworst error / bar of the below-limit cases (test_gpu_operand_range):")
        for k in sorted(_WORST):
            print(f"  {k:36s} {_WORST[k]:.3e}")


def site_weights(site: str, T: float, member_scale: float):
    """The seeded weights of WIDTHS[WIDTH] with the target T placed on `site` (see the module docstring)."""
    symbols, dims, in_dim = WIDTHS[WIDTH]
    base = orc.make_weights(symbols, dims, in_dim, M, seed=97, dtype=torch.float32)
    out = []
    for wm in base:
        per = {}
        for s in symbols:
            (W1, b1), (W2, b2), (W3, b3), (W4, b4) = [(w.clone(), b.clone()) for w, b in wm[s]]
            if site in ("a1", "nan_a1", "exact"):
                W1[I1] = 0.0
                b1[I1] = T
                W2[:, I1] = 0.0
            elif site == "a2":
                W2[K2] = 0.0
                b2[K2] = T
                W3[:, K2] = 0.0
            elif site in ("G3", "nan_G3"):
                W3[J3] = 0.0
                b3[J3] = 1.0 if site == "G3" else T
                W4[0, J3] = (T if site == "G3" else 1.0) / member_scale
            elif site == "G2":
                W2[K2] = 0.0
                b2[K2] = 1.0
                W3[J3] = 0.0
                W3[:, K2] = 0.0
                W3[J3, K2] = T
                b3[J3] = 0.0
                W4[0, J3] = 1.0 / member_scale
            elif site == "G1":
                W1[I1] = 0.0
                b1[I1] = 1.0
                W2[K2] = 0.0
                W2[:, I1] = 0.0
                W2[K2, I1] = T
                b2[K2] = 0.0
                W3[J3] = 0.0
                W3[:, K2] = 0.0
                W3[J3, K2] = 1.0
                b3[J3] = 0.0
                W4[0, J3] = 1.0 / member_scale
            per[s] = [(W1, b1), (W2, b2), (W3, b3), (W4, b4)]
        out.append(per)
    return out


class Run(tp.NamedTuple):
    status: int
    got: tp.Dict[str, torch.Tensor]     # decoded operand buffers, [rows_cap, M * p]
    e_member: torch.Tensor
    dx_all: torch.Tensor                # dE/dAEV with its guard bands
    dx: torch.Tensor                    # [slabs, rows_cap, ldx]
    first: tp.List[int]
    row_atom: torch.Tensor
    scale: torch.Tensor
    live_cols: torch.Tensor


def run_site(site: str, T: float, entry: str, monkeypatch) -> tp.Tuple[Run, tp.Any, tp.Any]:
    from torchani_b200 import _lib
    from torchani_b200._lib import check, ptr
    from torchani_b200.engine import PackedNetworks, operand_buffer, tile_a_operand, untile_a_operand
    for k in ("ANI_B200_MLP_CHAIN", "ANI_B200_CHAIN_DEPTH", "ANI_B200_MLP_CHUNKS"):
        monkeypatch.delenv(k, raising=False)
    if entry == "chain":
        monkeypatch.setenv("ANI_B200_MLP_CHAIN", "1")   # read per call
    wb = ENTRIES[entry]
    member_scale = 1.0 if wb == 2 else 1.0 / M
    symbols, dims, in_dim = WIDTHS[WIDTH]
    S = len(symbols)
    w = site_weights(site, T, member_scale)
    nets = PackedNetworks([[wm[s] for s in symbols] for wm in w], in_dim, torch.device(DEV))
    L = _lib.lib()
    ldx, ld = nets.ldx, nets.ld
    n = sum(ROWS) + 2
    rows_cap = (n + S * (TILE - 1) + TILE - 1) // TILE * TILE
    seed = sum(map(ord, site + entry))
    row_atom, layout_info, first = make_layout(L, ROWS, S, rows_cap, seed)
    model = _lib.MLPModel.from_buffer_copy(nets.model)
    for m in range(_lib.ANI_MAX_MEMBERS):
        model.member_scale[m] = member_scale if m < M else 0.0
    scale = torch.full((M,), member_scale, dtype=torch.float64, device=DEV)
    blocks = BLOCKS["water5"]
    live_cols = (torch.tensor(blocks, device=DEV).view(-1, 1) * 32 + torch.arange(32, device=DEV)).view(-1)
    x_t = tile_a_operand(make_x(Case(site, widths=WIDTH, M=M, rows=ROWS), rows_cap, ldx, in_dim, live_cols, seed))
    blk = torch.zeros(ldx // 32 + 3, dtype=torch.int32, device=DEV)
    blk[0] = len(blocks)
    blk[1:1 + len(blocks)] = torch.tensor(blocks, dtype=torch.int32)
    act = [operand_buffer(rows_cap, v, DEV) for v in ld]
    e_member = torch.full((M, rows_cap), SENTINEL, dtype=torch.float32, device=DEV)
    slabs = M if wb == 2 else 1
    dx_all = torch.full((2 * GUARD + slabs * rows_cap * ldx,), SENTINEL, dtype=torch.float32, device=DEV)
    dx = dx_all[GUARD:GUARD + slabs * rows_cap * ldx]
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    sync = torch.zeros(6 * (rows_cap // TILE) * _lib.ANI_MAX_MEMBERS + 8, dtype=torch.int32, device=DEV)
    st = torch.cuda.current_stream(DEV).cuda_stream
    M_ = C.byref(model)
    common = (rows_cap, ptr(row_atom), ptr(layout_info), ptr(blk))
    snap = None
    if entry in ("chained", "chained_forward"):
        check(L.ani_b200_mlp_forward_backward(M_, ptr(x_t), ptr(dx) if wb else None, *common, ptr(act[0]),
                                              ptr(act[1]), ptr(act[2]), ptr(e_member), wb, ptr(status), st), entry)
    elif entry == "split":
        check(L.ani_b200_mlp_forward(M_, ptr(x_t), *common, ptr(act[0]), ptr(act[1]), ptr(act[2]), ptr(e_member), 1,
                                     ptr(status), st), "mlp_forward")
        snap = [a.clone() for a in act]
        check(L.ani_b200_zero_live_blocks(M_, ptr(dx), ptr(layout_info), ptr(blk), st), "zero_live_blocks")
        check(L.ani_b200_mlp_backward(M_, ptr(dx), *common, ptr(act[0]), ptr(act[1]), ptr(act[2]), 1, ptr(status),
                                      st), "mlp_backward")
    elif entry == "resident":
        check(L.ani_b200_mlp_step_resident(M_, ptr(x_t), ptr(dx), *common, ptr(act[0]), ptr(act[1]), ptr(e_member),
                                           ptr(status), st), "mlp_step_resident")
        snap = act
    else:
        check(L.ani_b200_mlp_step(M_, ptr(x_t), ptr(dx), *common, ptr(act[0]), ptr(act[1]), ptr(act[2]),
                                  ptr(e_member), wb, ptr(sync), ptr(status), st), "mlp_step")
    torch.cuda.synchronize()
    fmt = _lib.operand_format()
    dec = lambda t, width, sc: untile_a_operand(t, rows_cap, width, sc)   # noqa: E731
    if wb == 0:
        got = {"a1": dec(act[0], ld[0], fmt.value_scale), "a2": dec(act[1], ld[1], fmt.value_scale)}
    elif entry == "resident":
        got = {"a1": dec(act[0], ld[0], fmt.value_scale), "a2": dec(act[1], ld[1], fmt.value_scale)}
    else:
        got = {"G1": dec(act[0], ld[0], fmt.grad_scale), "G2": dec(act[1], ld[1], fmt.grad_scale),
               "G3": dec(act[2], ld[2], fmt.grad_scale)}
        if snap is not None:
            got.update({"a1": dec(snap[0], ld[0], fmt.value_scale), "a2": dec(snap[1], ld[1], fmt.value_scale)})
    x64 = untile_a_operand(x_t, rows_cap, ldx).double()
    x64[:, ~torch.isin(torch.arange(ldx, device=DEV), live_cols)] = 0.0
    run = Run(int(status.item()), got, e_member, dx_all, dx.view(slabs, rows_cap, ldx), first, row_atom, scale,
              live_cols)
    return run, reference_weights(WIDTH, M, ldx, w), x64


def references(run: Run, rws, x64, per_member: bool):
    ra = run.row_atom.cpu()
    out = []
    for s in range(len(rws)):
        r0, r1 = run.first[s] * TILE, run.first[s + 1] * TILE
        if r1 == r0:
            continue
        valid = (ra[r0:r1] >= 0).to(DEV)
        out.append((s, r0, r1, valid, reference(rws[s], x64[r0:r1], valid, run.scale, per_member, 0.0)))
    return out


def assert_reaches(site: str, T: float, refs) -> None:
    """The float64 reference puts T on the named site and keeps every other site well inside the range."""
    peak = {k: max(float(ref[k].abs().max()) for *_, ref in refs) for k in SITES}
    assert abs(peak[site] - T) <= 1e-6 * T, (site, peak)
    for k, kind in SITES.items():
        if k != site:
            assert peak[k] < 0.5 * (VALUE_LIMIT if kind == "value" else GRAD_LIMIT), (site, k, peak)


def assert_nothing_outside(run: Run, wb: int, ldx: int) -> None:
    if not wb:
        return
    used = run.first[-1] * TILE
    dead = ~torch.isin(torch.arange(ldx, device=DEV), run.live_cols)
    assert bool((run.dx[:, :, dead] == SENTINEL).all()), "a dead column block of dE/dAEV was written"
    assert bool((run.dx[:, used:] == SENTINEL).all()), "rows beyond the layout's row tiles were written"
    assert bool((run.dx_all[:GUARD] == SENTINEL).all()) and bool((run.dx_all[-GUARD:] == SENTINEL).all()), \
        "dE/dAEV written outside [rows_cap][ldx]"


CASES = [(site, side, entry) for site, kind in SITES.items() for side in ("below", "above") for entry in ENTRIES
         if kind == "value" or ENTRIES[entry] > 0]


@pytest.mark.parametrize("site,side,entry", CASES, ids=[f"{a}-{b}-{c}" for a, b, c in CASES])
def test_mlp_site(site, side, entry, monkeypatch):
    from torchani_b200 import _lib
    T = TARGETS[SITES[site]][side == "above"]
    wb = ENTRIES[entry]
    run, rws, x64 = run_site(site, T, entry, monkeypatch)
    refs = references(run, rws, x64, wb == 2)
    assert_reaches(site, T, refs)
    ldx = x64.shape[1]
    if side == "above":
        s = 64.0 if SITES[site] == "value" else 4096.0
        assert HALF_MAX < s * float(np.float32(T)) < HALF_INF_FROM
        assert run.status & _lib.STATUS_OPERAND_RANGE, f"status {run.status}: {site} = {T} was not flagged"
        assert_nothing_outside(run, wb, ldx)
        return
    assert run.status == 0, f"status word {run.status} with {site} = {T}"
    bar = ROW_BARS[""]
    fails: tp.List[str] = []
    group = f"{SITES[site]} sites {'resident' if entry == 'resident' else 'k_gemm_wg'}"
    M_ = len(run.scale)
    worst = [0.0]
    for s, r0, r1, valid, ref in refs:
        p = rws[s]["p"]
        for k, v in run.got.items():
            width = p[{"a1": 0, "a2": 1, "G3": 2, "G2": 1, "G1": 0}[k]]
            mine = v[r0:r1].view(r1 - r0, -1)[:, :M_ * width].view(r1 - r0, M_, width).permute(1, 0, 2)
            d = (mine.double() - ref[k]).abs().amax(-1) / (bar * ref[k].abs().amax(-1)).clamp(min=1e-12)
            worst[0] = max(worst[0], float(d.max()))
            compare_rows("operand range " + group, mine, ref[k], ref["d" + k], bar, 0.0, f"species {s}: {k}", fails)
        em = run.e_member[:, r0:r1].double()
        real = valid.view(1, -1).expand_as(em)
        r = ((em - ref["e"]).abs() / (E_ATOL + E_RTOL * ref["e"].abs()))[real]
        worst[0] = max(worst[0], float(r.max()))
        if float(r.max()) > 1.0:
            fails.append(f"species {s}: e_member {float(r.max()):.3g} x the bar")
        if wb:
            live = run.dx[:, r0:r1][..., run.live_cols].double()
            if wb == 1:
                live = live[0]
            dref = ref["dx"][..., run.live_cols]
            d = (live - dref).abs().amax(-1) / (bar * dref.abs().amax(-1)).clamp(min=1e-12)
            worst[0] = max(worst[0], float(d.max()))
            compare_rows("operand range " + group, live, dref, ref["ddx"][..., run.live_cols], bar, 0.0,
                         f"species {s}: dE/dAEV", fails)
    _WORST[group] = max(_WORST.get(group, 0.0), worst[0])
    assert not fails, "\n".join(fails)
    assert_nothing_outside(run, wb, ldx)


NAN_CASES = [("nan_a1", "chained"), ("nan_a1", "dataflow_forward"), ("nan_a1", "resident"),
             ("nan_G3", "chained"), ("nan_G3", "split"), ("nan_G3", "slabs")]


@pytest.mark.parametrize("site,entry", NAN_CASES, ids=[f"{a}-{b}" for a, b in NAN_CASES])
def test_nan_is_flagged(site, entry, monkeypatch):
    """A NaN bias: layer 1's (a1) or the head's (z3, so G3 = w4 * CELU'(z3) is NaN).  A NaN compares false with
    everything, so only a NaN-propagating max flags it."""
    from torchani_b200 import _lib
    run, _, x64 = run_site(site, float("nan"), entry, monkeypatch)
    assert run.status & _lib.STATUS_OPERAND_RANGE, f"status {run.status}: a NaN was not flagged"
    assert_nothing_outside(run, ENTRIES[entry], x64.shape[1])


@pytest.mark.parametrize("entry", ["chained_forward", "resident"])
def test_exact_limit(entry, monkeypatch):
    """Flag iff |64 * a| > 65504: a1 = 1023.49 (64 a = 65503.36) passes, a1 = 1023.51 (65504.64) is flagged, although
    both round to a finite half."""
    from torchani_b200 import _lib
    for T, flagged in ((1023.49, False), (1023.51, True)):
        assert (64.0 * float(np.float32(T)) > HALF_MAX) == flagged
        run, rws, x64 = run_site("exact", T, entry, monkeypatch)
        assert_reaches("a1", float(np.float32(T)), references(run, rws, x64, False))
        assert bool(run.status & _lib.STATUS_OPERAND_RANGE) == flagged, (T, run.status)
        stored = float(run.got["a1"].abs().max())            # both pieces of the stored value are finite
        assert abs(stored - float(np.float32(T))) <= 2.0 ** -21 * T, stored


# ------------------------------------------------------------------------------------------------------------------
# the tiled-AEV writer
# ------------------------------------------------------------------------------------------------------------------
CAP_K = {"below": 40, "above": 48}


def cap_system(k: int):
    """A centre (H) with k H neighbours on a spherical cap of half-angle 0.5 rad, 0.8 A away."""
    from test_gpu_aev import System
    i = np.arange(k) + 0.5
    z = 1.0 - (1.0 - math.cos(0.5)) * i / k
    phi = i * math.pi * (3.0 - math.sqrt(5.0))
    r = np.sqrt(1.0 - z * z)
    xyz = np.concatenate([np.zeros((1, 3)), 0.8 * np.stack([r * np.cos(phi), r * np.sin(phi), z], 1)])
    xyz += np.array([5.0, 5.0, 5.0])
    return System(torch.zeros(1, k + 1, dtype=torch.long), torch.tensor(xyz, dtype=torch.float32).view(1, -1, 3), None)


def rows_forward(eng, sysm, spec) -> tp.Tuple[torch.Tensor, int]:
    """ani_b200_aev_forward_rows (the explicit-rows entry point of AEVComputer.compute_from_neighbors) in the tiled
    layout, on rows built from the oracle's pair list by ani_b200_pairs_to_rows: (decoded operand [n, ldx], status)."""
    from torchani_b200 import _lib
    from torchani_b200._lib import check, ptr
    from torchani_b200.engine import operand_buffer, untile_a_operand
    n = sysm.species.shape[1]
    nb = orc.neighborlist("all_pairs", spec.rcr, sysm.species, sysm.coords.double())
    idx = nb.indices.to(DEV, torch.int64).contiguous()
    dv = nb.diff_vectors.detach().to(DEV, torch.float32).contiguous()
    P = int(idx.shape[1])
    i32 = dict(dtype=torch.int32, device=DEV)
    spos = torch.zeros(n, 4, dtype=torch.float32, device=DEV)
    spos[:, 3] = sysm.species.reshape(-1).to(torch.int32).to(DEV).view(torch.float32)
    grid = torch.zeros(C.sizeof(_lib.Grid) // 4, **i32)
    grid[_lib.Grid.n_real.offset // 4] = n
    row_start, row_j = torch.zeros(n + 1, **i32), torch.zeros(2 * P, **i32)
    row_d = torch.zeros(2 * P, 4, dtype=torch.float32, device=DEV)
    scratch, status = torch.zeros(2 * n, **i32), torch.zeros(1, **i32)
    L, st = _lib.lib(), torch.cuda.current_stream(DEV).cuda_stream
    check(L.ani_b200_pairs_to_rows(idx[0].data_ptr(), idx[1].data_ptr(), ptr(dv), P, n, eng.nbr_cap, ptr(row_start),
                                   ptr(row_j), ptr(row_d), ptr(scratch), ptr(status), st), "pairs_to_rows")
    rows_cap = (n + TILE - 1) // TILE * TILE
    out = operand_buffer(rows_cap, eng.nets.ldx, DEV)
    check(L.ani_b200_aev_forward_rows(C.byref(eng.params), ptr(grid), ptr(spos), ptr(row_start), ptr(row_j),
                                      ptr(row_d), n, ptr(torch.arange(n, **i32)), ptr(out), eng.nets.ldx, 1,
                                      eng.nbr_cap, ptr(status), st), "aev_forward_rows")
    torch.cuda.synchronize()
    return untile_a_operand(out.reshape(-1), rows_cap, eng.nets.ldx)[:n], int(status.item())


@pytest.mark.parametrize("side", ["below", "above"])
def test_aev_writer(side):
    from torchani_b200 import _lib
    from torchani_b200.engine import untile_a_operand
    from test_gpu_aev import AEV_ATOL, AEV_RTOL, Gpu, Ref, internal_cols, make_engine
    spec = orc.aev_spec_2x()
    sysm = cap_system(CAP_K[side])
    ref = Ref(spec, sysm)
    peak = float(ref.values.max())
    assert int(ref.ang_counts.max()) <= 96 and int(ref.counts.max()) <= 128
    if side == "below":
        assert 1000.0 < peak < VALUE_LIMIT - 5.0, peak
    else:
        assert peak > VALUE_LIMIT + 100.0, peak
    eng, _, _ = make_engine(spec)
    gpu = Gpu(eng, sysm)
    x, status = gpu.forward(1)
    _, status_plain = gpu.forward(0)
    assert status_plain == 0, "plain rows have no range limit"
    t_rows, status_rows = rows_forward(eng, sysm, spec)
    if side == "above":
        assert status & _lib.STATUS_OPERAND_RANGE, f"status {status}: an AEV of {peak:.1f} was not flagged"
        assert status_rows & _lib.STATUS_OPERAND_RANGE, f"explicit rows: status {status_rows}, AEV {peak:.1f}"
        return
    assert status == 0 and status_rows == 0, f"status words {status} (bucket grid), {status_rows} (explicit rows)"
    t = untile_a_operand(x.reshape(-1), gpu.ws.rows_cap, gpu.ldx)
    cols = internal_cols(spec, gpu.pad).to(DEV)
    got = torch.zeros(gpu.n, spec.out_dim, dtype=torch.float64)
    got[gpu.so.cpu()] = t[gpu.rows][:, cols].double().cpu()
    for name, g in (("aev writer (tiled, decoded)", got), ("aev writer, explicit rows", t_rows[:, cols].double().cpu())):
        r = float(((g - ref.values).abs() / (AEV_RTOL * ref.values.abs() + AEV_ATOL)).max())
        _WORST[name] = max(_WORST.get(name, 0.0), r)
        assert r <= 1.0, f"{name}: AEV error {r:.3f} x the bar"


@pytest.mark.parametrize("var", ["ANI_B200_AEV_LEGACY=1", "ANI_B200_AEV_TMA=1", "ANI_B200_AEV_BSS=1"])
def test_aev_writer_process_wide_variants(var):
    """The warp-per-atom, TMA-staged and per-bucket species offset paths are chosen once per process: re-run the
    AEV writer cases in a child process."""
    k, v = var.split("=")
    env = dict(os.environ, **{k: v})
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
        "-m", "pytest", os.path.abspath(__file__), "-q", "-m", "gpu", "-k", "test_aev_writer and not variants",
        "-p", "no:cacheprovider"]
    res = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stdout[-4000:] + res.stderr[-2000:]
    assert "2 passed" in res.stdout and " failed" not in res.stdout
