"""Kernel-level parity of the ensemble-MLP GEMMs (k_gemm_wg, csrc/gemm_tc.cuh) against float64.

The C-ABI is called directly on synthetic inputs whose values the test controls: seeded float32 weights packed by
the library's own packing kernel (engine.PackedNetworks), species-grouped rows from ani_b200_species_layout, and an
AEV matrix with per-column magnitudes spread over 1e-6 .. 1e3, stored with engine.tile_a_operand.  The reference is
plain float64 torch (cuBLAS DGEMM on the GPU, not this library) on the float32 weights and on the operand DECODED
back with engine.untile_a_operand -- exactly what the kernel reads -- so the only differences left are the GEMM's
own: the 16-bit weight pieces, the dropped cross products, fp32 accumulation and the rounding of the stored outputs.

Every layer is compared on its own: the activations a1, a2 (forward), the gradient seed G3 = member_scale * w4 *
CELU'(z3) that the fused head stores in act3, the backward pieces G2 and G1 that overwrite act2 and act1, dE/dAEV
and the per-member energies.  Each case names the branch of the kernel it is meant to reach and asserts it where
the host can compute it: narrow (half-accumulator) or wide (256-column) tiles of the layer-1 forward from the SM
count, and the member group G of the grouped layer-1 backward from rows_cap and M.

Bars.  Two input sets run every configuration.  AEV-like inputs (per-column magnitudes 1e-6 .. 1, values >= 0) are
held to the plain bars: per row, normwise, max_j |d_ij| <= 1e-5 * max_j |ref_ij| (floor 1e-12) for the activations,
gradient pieces and dE/dAEV, and e_member within 1e-5 relative + 1e-6 absolute.  Wide-range inputs (1e-6 .. 1e3, the
"-wide_range" ids) cannot meet them: AEV entries up to 1e3 give activations of O(100), whose absolute fp32 error
CELU'(z) = exp(z / alpha) turns into a relative gradient error of ~4e-4.  Only those cases add MODEL_BARS * EPS times
the rounding-error scale that reference() propagates along with every value (EPS = 2^-22, DESIGN.md section 3).

Measured on an H100 80GB HBM3 (700 W), worst error / 1e-5 plain bar, AEV-like inputs: 2 x fp16 pieces 0.75
(activations), 0.60 (gradient pieces), 0.64 (dE/dAEV), 0.12 (e_member); 3 x bf16 pieces 1.09, 0.90, 0.55, 0.15.  The
bf16x3 build issues six products per K-step instead of three, and its plain bar is 2e-5.  None is small enough to
tighten a bar.  Wide-range inputs against the plain bar: 0.83, 284, 24, 23 (fp16x2) and 1.25, 367, 32, 29 (bf16x3);
against the bar they are held to, at most 0.66.  The 94 cases take ~15 s.  The module prints both ratios for every
group of cases at its end (pytest -s).
"""
import ctypes as C
import os
import typing as tp

import pytest
import torch

import oracle.ani_oracle as orc
from helpers import E_ATOL, E_RTOL

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
ALPHA = 0.1
ROW_BAR = 1e-5          # the plain per-row bar every ratio is also reported against
# applied plain bar per build: 3 x bf16 pieces issue six products per K-step into the fp32 accumulator instead of three,
# and its layer-1 activations were measured at up to 1.09e-5 of the row's max on AEV-like inputs
ROW_BARS = {"": 1e-5, "bf16x3": 2e-5}
EPS = 2.0 ** -22         # operand precision of the 2 x fp16 pieces (3 x bf16: 2^-24)
# wide-range inputs only: allowed multiple of the rounding-error scale (reference(): d<name>)
MODEL_BARS = {"": 8.0, "bf16x3": 16.0}
TILE = 128
TN_MAX = 256
SENTINEL = 7.25          # dE/dAEV entries nobody may write keep this value
GUARD = 4096             # floats of sentinel before and after dE/dAEV

# read ONCE per process by the library (static initialisers): a test cannot change them, and with one of them set
# the host-side predictions of the launch configuration below would be wrong
_PINNED = ("ANI_B200_L1B_GROUP", "ANI_B200_NARROW_TILES", "ANI_B200_B1_COMPACT")

WIDTHS = {   # name -> (species names, hidden widths per species, AEV length)
    "2x": (orc.SYMBOLS_2X, orc.DIMS_2X, 1008),                                     # seven species of different widths
    "1x": (orc.SYMBOLS_1X, orc.DIMS_1X, 384),                                      # 144 and 112: zero-padded to 160, 128
    "h32": (("A", "B", "C"), {"A": (32, 32, 32), "B": (32, 32, 32), "C": (32, 32, 32)}, 1008),
    "h3_256": (("A", "B"), {"A": (256, 256, 256), "B": (64, 96, 256)}, 1008),       # h3 = TN_MAX in one accumulator
    "h1_wide": (("A", "B", "C"), {"A": (288, 192, 160), "B": (320, 128, 96), "C": (160, 128, 96)}, 1008),  # 2 N tiles
}
BLOCKS = {   # live 32-column AEV blocks (aev_blocks); None = every block live
    None: None,
    "water5": [0, 1, 4, 7, 22],          # the five blocks of a water box (H, O) in the aligned column order
    "one": [9],
    "all32": list(range(32)),            # every element pair present (seven-element systems)
    "scattered": [0, 3, 9, 10, 17, 30, 31],
}
R2X = [129, 0, 1, 127, 128, 300, 3]      # rows per species: 0, 1, 127, 128, 129 in one call (9 row tiles)


class Case(tp.NamedTuple):
    name: str
    widths: str = "2x"
    M: int = 8
    rows: tp.Tuple[int, ...] = tuple(R2X)
    entry: str = "chained"        # chained | dataflow | chain0 | chain3 | chunks3 | split | forward
    blocks: tp.Optional[str] = None
    compact: bool = True          # b1_compact scratch given (used only with a block list)
    variant: str = ""
    rows_cap: int = 0             # 0: just enough row tiles
    active: tp.Optional[tp.Tuple[int, ...]] = None
    wb: int = 1                   # want_backward
    values: str = "aev"           # aev (O(1), plain bars) | wide (1e-6 .. 1e3, model term) | near_limit | over_limit
    boundary: int = 0             # -1 / +1: rows chosen from the SM count just below / above the narrow-tile boundary
    tiles: tp.Optional[str] = None   # expected layer-1 forward tiles: "narrow" | "wide" (None: not asserted)
    group: tp.Optional[int] = None   # expected member group G of the layer-1 backward


CASES = [
    # entry points, on the 2x widths with rows 0 / 1 / 127 / 128 / 129 per species in one launch
    Case("chained", tiles="wide", group=1),
    Case("chained_water5", blocks="water5", group=1),
    Case("chained_water5_nocompact", blocks="water5", compact=False, group=1),
    Case("dataflow_all32", entry="dataflow", blocks="all32", tiles="wide", group=1),
    Case("dataflow_all32_nocompact", entry="dataflow", blocks="all32", compact=False, group=1),
    Case("dataflow_one_block", entry="dataflow", blocks="one"),
    Case("dataflow_one_block_nocompact", entry="dataflow", blocks="one", compact=False),
    Case("chained_scattered", blocks="scattered"),
    Case("chained_scattered_nocompact", blocks="scattered", compact=False),
    Case("chain_depth0", entry="chain0", rows=(600, 300, 0, 200, 50, 20, 7), blocks="water5", tiles="wide", group=1),
    Case("chain_depth3", entry="chain3", rows=(600, 300, 0, 200, 50, 20, 7), tiles="wide", group=1),
    Case("chunks3", entry="chunks3", rows=(1500, 800, 300, 600, 100, 50, 20), blocks="scattered", group=2),
    Case("split", entry="split", blocks="water5", group=1),
    Case("split_nocompact", entry="split", blocks="all32", compact=False),
    Case("forward_only", entry="forward", wb=0),
    Case("forward_only_dataflow", entry="dataflow", wb=0),
    # narrow (half-accumulator) and wide column tiles on both sides of the boundary 2 x units <= SMs
    Case("narrow_boundary", boundary=-1, tiles="narrow", group=1),
    Case("narrow_boundary_dataflow", boundary=-1, entry="dataflow", blocks="scattered", tiles="narrow"),
    Case("wide_boundary", boundary=+1, tiles="wide", group=1),
    Case("wide_boundary_dataflow", boundary=+1, entry="dataflow", blocks="water5", tiles="wide"),
    Case("members_slabs", entry="dataflow", blocks="water5", wb=2, active=(1, 4, 6), group=1),
    Case("members_slabs_dense", entry="dataflow", wb=2, M=3, group=1),
    # member counts and active subsets (M = 16 = ANI_MAX_MEMBERS)
    Case("M1", M=1, tiles="narrow", group=1),
    Case("M3", M=3, entry="dataflow", blocks="scattered", tiles="narrow", group=1),
    Case("M16_active_subset", M=16, entry="dataflow", blocks="all32", active=(0, 3, 4, 9, 15), group=1),
    Case("M16_chained", M=16, rows=(300, 200, 100, 50, 20, 10, 5), group=1),
    # member group G of the layer-1 backward: 2 for rows_cap in [4096, 32768), 4 from 32768, 3 for M = 6 there
    Case("G2_dataflow", entry="dataflow", rows=(3000, 1500, 400, 700, 100, 60, 40), rows_cap=8192,
         blocks="scattered", tiles="wide", group=2),
    Case("G2_chained", rows=(3000, 1500, 400, 700, 100, 60, 40), rows_cap=8192, blocks="water5", compact=False,
         group=2),
    Case("G4_dataflow_32k", entry="dataflow", rows=(16000, 8000, 2500, 4000, 800, 500, 400), rows_cap=32768,
         blocks="water5", tiles="wide", group=4),
    Case("G4_chained_32k", rows=(16000, 8000, 2500, 4000, 800, 500, 400), rows_cap=32768, group=4),
    Case("G3_M6", M=6, entry="dataflow", rows=(2000, 1000, 0, 500, 129, 1, 64), rows_cap=32768, blocks="all32",
         group=3),
    Case("G3_M6_chained", M=6, rows=(2000, 1000, 0, 500, 129, 1, 64), rows_cap=32768, group=3),
    # widths
    Case("ani1x_padded_widths", widths="1x", entry="dataflow", rows=(200, 130, 60, 1), tiles="narrow", group=1),
    Case("ani1x_chained", widths="1x", rows=(200, 130, 60, 1), group=1),
    Case("h32", widths="h32", M=3, rows=(128, 129, 5), blocks="scattered", tiles="narrow", group=1),
    Case("h32_dataflow", widths="h32", M=3, entry="dataflow", rows=(128, 129, 5), group=1),
    Case("h3_256", widths="h3_256", entry="dataflow", rows=(300, 129), blocks="all32", group=1),
    Case("h3_256_chained", widths="h3_256", rows=(300, 129), group=1),
    Case("h1_288_320_chained", widths="h1_wide", M=4, rows=(300, 129, 1), tiles="narrow", group=1),
    Case("h1_288_320_dataflow", widths="h1_wide", M=4, entry="dataflow", rows=(300, 129, 1), blocks="water5",
         group=1),
    # ANI_B200_MLP_CHAIN=1 with h1 > 256: use_chain_launch falls back to the phase-major list
    Case("h1_288_320_chain_fallback", widths="h1_wide", M=4, entry="chain0", rows=(300, 129, 1), tiles="narrow",
         group=1),
    # values at the edge of the operand range of the 2 x fp16 pieces
    Case("near_operand_limit", values="near_limit", blocks="water5"),
    Case("over_operand_limit", values="over_limit"),
    # the 3 x bf16 build
    Case("bf16x3_chained", variant="bf16x3", group=1),
    Case("bf16x3_dataflow_all32", variant="bf16x3", entry="dataflow", blocks="all32", group=1),
    Case("bf16x3_G2_scattered", variant="bf16x3", entry="dataflow", rows=(3000, 1500, 400, 700, 100, 60, 40),
         rows_cap=8192, blocks="scattered", group=2),
    Case("bf16x3_split_h1_wide", variant="bf16x3", widths="h1_wide", M=4, entry="split", rows=(300, 129, 1)),
    Case("bf16x3_members_slabs", variant="bf16x3", entry="dataflow", wb=2, active=(0, 2), M=3),
]
# every configuration once more on the wide-range values
CASES += [c._replace(name=c.name + "-wide_range", values="wide") for c in CASES if c.values == "aev"]

WORST: tp.Dict[str, tp.List[float]] = {}   # group -> [worst error / applied bar, worst error / plain bar]


@pytest.fixture(scope="module", autouse=True)
def _report():
    pinned = [k for k in _PINNED if k in os.environ]
    if pinned:
        pytest.skip(f"{pinned} pin a launch configuration for the whole process")
    yield
    print("\nworst error / bar per group of cases (test_gpu_mlp): applied bar, plain bar (1e-5 of the row's max "
          "|ref|; e_member: 1e-5 relative + 1e-6)")
    for k in sorted(WORST):
        print(f"  {k:40s} {WORST[k][0]:.3e}  {WORST[k][1]:.3e}")


def _note(group: str, ratio: float, plain: float) -> None:
    w = WORST.setdefault(group, [0.0, 0.0])
    w[0], w[1] = max(w[0], ratio), max(w[1], plain)


_weights: tp.Dict[tp.Any, tp.Any] = {}
_nets: tp.Dict[tp.Any, tp.Any] = {}


def weights(widths: str, M: int):
    key = (widths, M)
    if key not in _weights:
        symbols, dims, in_dim = WIDTHS[widths]
        _weights[key] = orc.make_weights(symbols, dims, in_dim, M, seed=4321 + M, dtype=torch.float32)
    return _weights[key]


def packed(widths: str, M: int, variant: str):
    from torchani_b200.engine import PackedNetworks
    key = (widths, M, variant)
    if key not in _nets:
        symbols, _, in_dim = WIDTHS[widths]
        w = weights(widths, M)
        _nets[key] = PackedNetworks([[w[m][s] for s in symbols] for m in range(M)], in_dim, DEV, variant=variant)
    return _nets[key]


def _pad32(v: int) -> int:
    return (v + 31) // 32 * 32


def reference_weights(widths: str, M: int, ldx: int, w=None):
    """float64 copies of the float32 weights (``w``, default the seeded weights of these widths), zero-padded to the
    kernel's widths (multiples of 32, ldx columns)."""
    symbols, dims, in_dim = WIDTHS[widths]
    w = weights(widths, M) if w is None else w
    out = []
    for s in symbols:
        h = dims[s]
        p = [_pad32(v) for v in h]
        W1 = torch.zeros(M, p[0], ldx, dtype=torch.float64)
        W2 = torch.zeros(M, p[1], p[0], dtype=torch.float64)
        W3 = torch.zeros(M, p[2], p[1], dtype=torch.float64)
        b1, b2, b3 = (torch.zeros(M, p[k], dtype=torch.float64) for k in range(3))
        w4 = torch.zeros(M, p[2], dtype=torch.float64)
        b4 = torch.zeros(M, dtype=torch.float64)
        for m in range(M):
            (a, ab), (bw, bb), (cw, cb), (dw, db) = w[m][s]
            W1[m, :h[0], :in_dim] = a.double()
            W2[m, :h[1], :h[0]] = bw.double()
            W3[m, :h[2], :h[1]] = cw.double()
            b1[m, :h[0]], b2[m, :h[1]], b3[m, :h[2]] = ab.double(), bb.double(), cb.double()
            w4[m, :h[2]] = dw.double().view(-1)
            b4[m] = db.double().view(())
        out.append(dict(p=p, W1=W1.to(DEV), W2=W2.to(DEV), W3=W3.to(DEV), b1=b1.to(DEV), b2=b2.to(DEV),
                        b3=b3.to(DEV), w4=w4.to(DEV), b4=b4.to(DEV)))
    return out


def _celu(z):
    return torch.where(z > 0, z, ALPHA * torch.expm1(z / ALPHA))


def _dcelu(z):
    return torch.where(z > 0, torch.ones_like(z), torch.exp(z / ALPHA))


def reference(rw, x64, valid, scale, per_member: bool, model_bar: float):
    """float64 forward + backward-to-input of one species' rows: a1, a2, G3, G2, G1 [M, R, p], e [M, R],
    dx [R, ldx] (sum over the members) or [M, R, ldx] (per_member).

    With every value, ``d<name>`` holds the scale of its rounding error in units of the operand precision EPS,
    propagated to first order: a GEMM output z carries |A| @ |B| + |bias| of its own (operand pieces and the tensor
    cores' fp32 accumulation, which grows with K rather than sqrt(K)) plus the errors of its inputs carried through the
    weights (in quadrature: independent signs); a stored value |value|; and CELU'(z) = exp(z / alpha) for z < 0 --
    recovered from the stored activation y as y / alpha + 1 -- carries d(y) / alpha: an absolute pre-activation error
    dz becomes a RELATIVE gradient error dz / alpha (10 dz)."""
    M = rw["W1"].shape[0]
    X = x64.unsqueeze(0).expand(M, -1, -1)
    W1, W2, W3 = rw["W1"], rw["W2"], rw["W3"]
    sq = lambda t: t * t    # noqa: E731
    rss = lambda *t: torch.sqrt(sum(sq(v) for v in t))   # noqa: E731

    def gemm(a, da, w, b):   # z = a @ w^T + b; its own error (linear in K) plus the inputs' (in quadrature)
        z = torch.baddbmm(b.unsqueeze(1), a, w.transpose(1, 2))
        own = torch.baddbmm(b.abs().unsqueeze(1), a.abs(), w.abs().transpose(1, 2))
        return z, own + torch.sqrt(torch.bmm(sq(da), sq(w).transpose(1, 2)))

    z1, dz1 = gemm(X, torch.zeros_like(X), W1, rw["b1"])
    a1 = _celu(z1)
    da1 = rss(_dcelu(z1) * dz1, a1)
    z2, dz2 = gemm(a1, da1, W2, rw["b2"])
    a2 = _celu(z2)
    da2 = rss(_dcelu(z2) * dz2, a2)
    z3, dz3 = gemm(a2, da2, W3, rw["b3"])
    a3 = _celu(z3)
    da3 = rss(_dcelu(z3) * dz3, a3)
    w4 = rw["w4"].unsqueeze(1)
    e = (a3 * w4).sum(-1) + rw["b4"].view(M, 1)
    de = (a3 * w4).abs().sum(-1) + rw["b4"].abs().view(M, 1) + torch.sqrt((sq(da3) * sq(w4)).sum(-1))
    seed = scale.view(M, 1, 1) * valid.view(1, -1, 1).to(torch.float64)
    # d CELU' / dy for the stored y, wherever z may be negative within its own error (CELU' has a kink at 0)
    neg = lambda z, dz: (z <= model_bar * EPS * dz).to(torch.float64) / ALPHA   # noqa: E731
    G3 = seed * w4 * _dcelu(z3)
    dG3 = rss(seed * w4 * da3 * neg(z3, dz3), G3)
    P2, dP2 = gemm(G3, dG3, W3.transpose(1, 2), torch.zeros_like(rw["b2"]))
    G2 = P2 * _dcelu(z2)
    dG2 = rss(dP2 * _dcelu(z2), P2 * da2 * neg(z2, dz2), G2)
    P1, dP1 = gemm(G2, dG2, W2.transpose(1, 2), torch.zeros_like(rw["b1"]))
    G1 = P1 * _dcelu(z1)
    dG1 = rss(dP1 * _dcelu(z1), P1 * da1 * neg(z1, dz1), G1)
    if per_member:
        dx = torch.bmm(G1, W1)
        ddx = torch.bmm(G1.abs(), W1.abs()) + torch.sqrt(torch.bmm(sq(dG1), sq(W1)))
    else:
        R = x64.shape[0]
        flat = lambda t: t.permute(1, 0, 2).reshape(R, -1)   # noqa: E731
        W1f = W1.reshape(-1, W1.shape[-1])
        dx = flat(G1) @ W1f
        ddx = flat(G1.abs()) @ W1f.abs() + torch.sqrt(flat(sq(dG1)) @ sq(W1f))
    return dict(a1=a1, a2=a2, G3=G3, G2=G2, G1=G1, e=e, dx=dx,
                da1=da1, da2=da2, dG3=dG3, dG2=dG2, dG1=dG1, de=de, ddx=ddx)


def compare_rows(group: str, got: torch.Tensor, ref: torch.Tensor, dref: torch.Tensor, row_bar: float, model_bar: float,
                 what: str, fails: tp.List[str]) -> None:
    """Per row (the second-to-last dim), normwise: max_j |got - ref| <= row_bar * max_j |ref| + model_bar * EPS *
    max_j dref (the rounding-error scale of reference(); model_bar = 0 for the O(1) inputs), floor 1e-12.  The worst
    ratio to that bar and to ROW_BAR * max_j |ref| alone are recorded for the report."""
    if not bool(torch.isfinite(got).all()):
        fails.append(f"{what}: non-finite values")
        return
    d = (got.double() - ref).abs()
    err = d.amax(-1)
    plain = (ROW_BAR * ref.abs().amax(-1)).clamp(min=1e-12)
    bound = (row_bar * ref.abs().amax(-1) + model_bar * EPS * dref.amax(-1)).clamp(min=1e-12)
    r = err / bound
    ratio = float(r.max()) if r.numel() else 0.0
    _note(group, ratio, float((err / plain).max()) if r.numel() else 0.0)
    if ratio > 1.0:
        i = int(r.argmax())
        row = d.reshape(-1, d.shape[-1])[i]
        j = int(row.argmax())
        rg, rr = got.reshape(-1, got.shape[-1])[i], ref.reshape(-1, ref.shape[-1])[i]
        fails.append(f"{what}: worst row error {ratio:.3g} x the bar at (slab, row) {divmod(i, r.shape[-1])} column "
                     f"{j}: got {float(rg[j]):.6e} ref {float(rr[j]):.6e}, row max |ref| {float(rr.abs().max()):.3e}, "
                     f"row error scale {float(EPS * dref.reshape(-1, d.shape[-1])[i].max()):.3e}")


def l1b_group(M: int, rows_cap: int) -> int:
    """mlp.cu l1b_group: members contracted by one unit of the grouped layer-1 backward."""
    g = 1 if rows_cap < 4096 else 2 if rows_cap < 32768 else 4
    while g > 1 and M % g:
        g -= 1
    return g


def layer1_forward_tiles(tiles_per_species, p1, M: int, sms: int) -> str:
    """gemm_tc.cuh build_tile_map for the layer-1 forward: narrow when twice the 256-column units fit in one wave."""
    units = sum(t * M * ((p + TN_MAX - 1) // TN_MAX) for t, p in zip(tiles_per_species, p1))
    return "narrow" if units > 0 and 2 * units <= sms else "wide"


def make_layout(L, rows, S: int, rows_cap: int, seed: int):
    """Species-grouped rows as nn._MLPFunction.forward builds them: real atoms first (shuffled species), two padding
    atoms, species bits in spos, ani_b200_species_layout."""
    from torchani_b200._lib import Grid, check, ptr
    sp = torch.cat([torch.full((r,), s, dtype=torch.int32) for s, r in enumerate(rows)])
    sp = sp[torch.randperm(sp.numel(), generator=torch.Generator().manual_seed(seed))]
    n_real = sp.numel()
    sp = torch.cat([sp, torch.full((2,), -1, dtype=torch.int32)]).to(DEV)
    n = sp.numel()
    spos = torch.zeros(n, 4, dtype=torch.float32, device=DEV)
    spos[:, 3] = sp.view(torch.float32)
    grid = torch.zeros(C.sizeof(Grid) // 4, dtype=torch.int32, device=DEV)
    grid[Grid.n_real.offset // 4] = n_real
    i32 = dict(dtype=torch.int32, device=DEV)
    row_of, row_atom = torch.zeros(n, **i32), torch.zeros(rows_cap, **i32)
    tile_species, layout_info = torch.zeros(rows_cap // TILE, **i32), torch.zeros(16, **i32)
    scratch = torch.zeros((n // 256 + 3) * 8 + 64, **i32)
    st = torch.cuda.current_stream(DEV).cuda_stream
    check(L.ani_b200_species_layout(ptr(spos), ptr(grid), n, 0, n, S, rows_cap, ptr(row_of), ptr(row_atom),
                                    ptr(tile_species), ptr(layout_info), ptr(scratch), st), "species_layout")
    info = layout_info.cpu().tolist()
    first = info[4:4 + S + 1]
    for s in range(S):   # the layout itself: one block of ceil(rows / 128) row tiles per species
        assert first[s + 1] - first[s] == (rows[s] + TILE - 1) // TILE, (s, first)
    return row_atom, layout_info, first


def make_x(case: Case, rows_cap: int, ldx: int, in_dim: int, live_cols: torch.Tensor, seed: int):
    """Plain AEV rows with per-column magnitudes log-uniform over 1e-6 .. 1 and values in [0, magnitude] like an AEV
    ("aev"), or over 1e-6 .. 1e3 with random signs ("wide" and the operand-limit cases: the x64 value scale puts the
    smallest values in the subnormal range of the second half piece, the largest near the range limit); dead blocks
    hold junk of |x| <= 800."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    if case.values == "aev":
        mag = 10.0 ** (-6.0 + 6.0 * torch.rand(ldx, generator=g, device=DEV))
        x = torch.rand(rows_cap, ldx, generator=g, device=DEV) * mag
    else:
        mag = 10.0 ** (-6.0 + 9.0 * torch.rand(ldx, generator=g, device=DEV))
        x = (torch.rand(rows_cap, ldx, generator=g, device=DEV) * 2 - 1) * mag
    if case.values == "near_limit":        # a few entries per row just inside |x| < 1023
        cols = live_cols[torch.randint(0, live_cols.numel(), (rows_cap, 3), generator=g, device=DEV)]
        sign = torch.where(torch.rand(rows_cap, 3, generator=g, device=DEV) < 0.5, -1.0, 1.0)
        x.scatter_(1, cols, 1022.9 * sign)
    elif case.values == "over_limit":      # one entry of one row outside the range of the fp16 pieces
        x[5, int(live_cols[0])] = 1030.0
    dead = torch.ones(ldx, dtype=torch.bool, device=DEV)
    dead[live_cols] = False
    junk = (torch.rand(rows_cap, ldx, generator=g, device=DEV) * 2 - 1) * 800.0
    return torch.where(dead.view(1, -1), junk, x)


def _set_env(monkeypatch, entry: str) -> None:
    for k in ("ANI_B200_MLP_CHAIN", "ANI_B200_CHAIN_DEPTH", "ANI_B200_MLP_CHUNKS"):
        monkeypatch.delenv(k, raising=False)
    if entry in ("chain0", "chain3"):
        monkeypatch.setenv("ANI_B200_MLP_CHAIN", "1")
        monkeypatch.setenv("ANI_B200_CHAIN_DEPTH", entry[-1])
    elif entry == "chunks3":
        monkeypatch.setenv("ANI_B200_MLP_CHUNKS", "3")


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_mlp_gemm_matches_float64(case: Case, monkeypatch):
    from torchani_b200 import _lib
    from torchani_b200._lib import check, ptr
    from torchani_b200.engine import operand_buffer, tile_a_operand, untile_a_operand
    if case.variant and not _lib.available(case.variant):
        pytest.skip(f"{_lib.variant_path(case.variant)} has not been built")
    fmt = _lib.operand_format(case.variant)
    if case.values in ("near_limit", "over_limit") and fmt.parts != 2:
        pytest.skip("the operand range limit exists only for the 2 x fp16 pieces")
    _set_env(monkeypatch, case.entry)
    model_bar = 0.0 if case.values == "aev" else MODEL_BARS[case.variant]   # O(1) inputs: the plain bars
    row_bar = ROW_BARS[case.variant]
    L = _lib.lib(case.variant)
    symbols, dims, in_dim = WIDTHS[case.widths]
    S, M = len(symbols), case.M
    nets = packed(case.widths, M, case.variant)
    ldx = nets.ldx
    st = torch.cuda.current_stream(DEV).cuda_stream
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    seed = sum(map(ord, case.name))

    if case.boundary:
        # T row tiles of 8 members are the most that still run narrow: T - 1 (+1 on the wide side) for species 0,
        # one for species 2
        T = sms // (2 * M)
        case = case._replace(rows=((T - 2 + (case.boundary > 0)) * TILE + 1, 0, 5) + (0,) * (S - 3))
    n = sum(case.rows) + 2    # (make_layout adds two padding atoms)
    rows_cap = max((n + S * (TILE - 1) + TILE - 1) // TILE * TILE, case.rows_cap)   # what species_layout accepts
    row_atom, layout_info, first = make_layout(L, case.rows, S, rows_cap, seed)

    # the model: member scales of the active subset, compaction on or off (a copy of PackedNetworks.model)
    active = list(case.active) if case.active is not None else list(range(M))
    model = _lib.MLPModel.from_buffer_copy(nets.model)
    for m in range(_lib.ANI_MAX_MEMBERS):
        model.member_scale[m] = (1.0 / len(active)) if m in active else 0.0
    if not case.compact:
        model.b1_compact = None
    scale = torch.tensor([model.member_scale[m] for m in range(M)], dtype=torch.float64, device=DEV)

    # the branches this case is meant to reach
    p1 = [_pad32(dims[s][0]) for s in symbols]
    chain = case.entry in ("chain0", "chain3") and max(p1) <= TN_MAX and \
        max(_pad32(dims[s][k]) for s in symbols for k in (1, 2)) <= TN_MAX
    tiles = [first[s + 1] - first[s] for s in range(S)]
    windows = L.ani_b200_mlp_step_windows(C.byref(model), rows_cap) if case.entry not in ("chained", "split",
                                                                                             "forward") else 1
    if case.entry == "chunks3":
        assert windows == 3 and rows_cap // TILE >= 24
    elif case.entry == "chain0" and not chain:
        assert windows == 1      # h1 > 256: no independent chains, the phase-major list
    if case.tiles is not None:
        win0 = [t // windows for t in tiles]   # window 0 of the row tiles of every species (build_tile_map)
        assert ("wide" if chain else layer1_forward_tiles(win0, p1, M, sms)) == case.tiles
    if case.group is not None:
        assert (1 if (chain or case.wb == 2) else l1b_group(M, rows_cap)) == case.group

    # inputs
    blocks = BLOCKS[case.blocks]
    live_blocks = blocks if blocks is not None else list(range(ldx // 32))
    live_cols = (torch.tensor(live_blocks, device=DEV).view(-1, 1) * 32 + torch.arange(32, device=DEV)).view(-1)
    x_plain = make_x(case, rows_cap, ldx, in_dim, live_cols, seed)
    x_t = tile_a_operand(x_plain, variant=case.variant)
    blk = None
    if blocks is not None:
        blk = torch.zeros(ldx // 32 + 3, dtype=torch.int32, device=DEV)
        blk[0] = len(blocks)
        blk[1:1 + len(blocks)] = torch.tensor(blocks, dtype=torch.int32)
    ld = nets.ld
    act = [operand_buffer(rows_cap, w, DEV, case.variant) for w in ld]
    e_member = torch.full((M, rows_cap), SENTINEL, dtype=torch.float32, device=DEV)
    slabs = M if case.wb == 2 else 1
    dx_all = torch.full((2 * GUARD + slabs * rows_cap * ldx,), SENTINEL, dtype=torch.float32, device=DEV)
    dx = dx_all[GUARD:GUARD + slabs * rows_cap * ldx]
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    sync = torch.zeros(6 * (rows_cap // TILE) * _lib.ANI_MAX_MEMBERS + 8, dtype=torch.int32, device=DEV)
    M_ = C.byref(model)
    wb = case.wb
    fwd_snap = None

    if case.entry == "chained" or case.entry == "forward":
        check(L.ani_b200_mlp_forward_backward(M_, ptr(x_t), ptr(dx) if wb else None, rows_cap, ptr(row_atom),
                                              ptr(layout_info), ptr(blk), ptr(act[0]), ptr(act[1]), ptr(act[2]),
                                              ptr(e_member), wb, ptr(status), st), "mlp_forward_backward")
    elif case.entry == "split":
        check(L.ani_b200_mlp_forward(M_, ptr(x_t), rows_cap, ptr(row_atom), ptr(layout_info), ptr(blk), ptr(act[0]),
                                     ptr(act[1]), ptr(act[2]), ptr(e_member), 1, ptr(status), st), "mlp_forward")
        fwd_snap = [a.clone() for a in act]
        check(L.ani_b200_zero_live_blocks(M_, ptr(dx), ptr(layout_info), ptr(blk), st), "zero_live_blocks")
        check(L.ani_b200_mlp_backward(M_, ptr(dx), rows_cap, ptr(row_atom), ptr(layout_info), ptr(blk), ptr(act[0]),
                                      ptr(act[1]), ptr(act[2]), 1, ptr(status), st), "mlp_backward")
    else:
        check(L.ani_b200_mlp_step(M_, ptr(x_t), ptr(dx), rows_cap, ptr(row_atom), ptr(layout_info), ptr(blk),
                                  ptr(act[0]), ptr(act[1]), ptr(act[2]), ptr(e_member), wb, ptr(sync), ptr(status),
                                  st), "mlp_step")
    torch.cuda.synchronize()
    code = int(status.item())
    if case.values == "over_limit":
        assert code & _lib.STATUS_OPERAND_RANGE, f"status {code}: the operand range overflow was not reported"
        return
    assert code == 0, f"status word {code}"

    # what the kernel reads, and the reference on it
    x64 = untile_a_operand(x_t, rows_cap, ldx, variant=case.variant).double()
    x64[:, ~torch.isin(torch.arange(ldx, device=DEV), live_cols)] = 0.0
    rws = reference_weights(case.widths, M, ldx)
    sv, sg = fmt.value_scale, fmt.grad_scale
    dec = lambda t, w, sc: untile_a_operand(t, rows_cap, w, sc, variant=case.variant)  # noqa: E731
    if wb == 0:
        got = {"a1": dec(act[0], ld[0], sv), "a2": dec(act[1], ld[1], sv)}
    else:
        got = {"G1": dec(act[0], ld[0], sg), "G2": dec(act[1], ld[1], sg), "G3": dec(act[2], ld[2], sg)}
    if fwd_snap is not None:
        got.update({"a1": dec(fwd_snap[0], ld[0], sv), "a2": dec(fwd_snap[1], ld[1], sv),
                    "G3_forward": dec(fwd_snap[2], ld[2], sg)})
    tag = ("bf16x3 " if case.variant else "fp16x2 ") + ("aev" if case.values == "aev" else "wide")
    ra = row_atom.cpu()
    fails: tp.List[str] = []
    dxv = dx.view(slabs, rows_cap, ldx)
    for s in range(S):
        if tiles[s] == 0:
            continue
        r0, r1 = first[s] * TILE, first[s + 1] * TILE
        valid = (ra[r0:r1] >= 0).to(DEV)
        ref = reference(rws[s], x64[r0:r1], valid, scale, (wb == 2), model_bar)
        p = rws[s]["p"]
        where = f"{case.name} species {symbols[s]}"
        for k, v in got.items():
            name = k.split("_")[0]
            w = p[{"a1": 0, "a2": 1, "G3": 2, "G2": 1, "G1": 0}[name]]
            mine = v[r0:r1].view(r1 - r0, -1)[:, :M * w].view(r1 - r0, M, w).permute(1, 0, 2)
            compare_rows(f"{tag} {'activations' if name[0] == 'a' else 'gradient pieces'}", mine, ref[name],
                         ref["d" + name], row_bar, model_bar, f"{where}: {k}", fails)
        # per-member energies: real rows against the reference, padding rows exactly 0
        em = e_member[:, r0:r1].double()
        plain = E_ATOL + E_RTOL * ref["e"].abs()
        bound = plain + model_bar * EPS * ref["de"]
        err = (em - ref["e"]).abs()
        real = valid.view(1, -1).expand_as(em)
        _note(f"{tag} e_member", float((err / bound)[real].max()), float((err / plain)[real].max()))
        if not bool((err <= bound)[real].all()):
            fails.append(f"{where}: e_member off by {float(err[real].max()):.3e}")
        if bool((~real).any()):
            assert float(em[~real].abs().max()) == 0.0, f"{where}: padding rows must get e_member = 0"
        if wb:
            live = dxv[:, r0:r1][..., live_cols].double()
            if wb == 1:
                live = live[0]
            compare_rows(f"{tag} dE/dAEV", live, ref["dx"][..., live_cols], ref["ddx"][..., live_cols], row_bar,
                         model_bar, f"{where}: dE/dAEV", fails)
    assert not fails, "\n".join(fails)
    # contracts beyond the values
    if wb:
        used = first[S] * TILE
        dead = ~torch.isin(torch.arange(ldx, device=DEV), live_cols)
        if bool(dead.any()):
            assert bool((dxv[:, :, dead] == SENTINEL).all()), "a dead column block of dE/dAEV was written"
        assert bool((dxv[:, used:] == SENTINEL).all()), "rows beyond the layout's row tiles were written"
        assert bool((dx_all[:GUARD] == SENTINEL).all()) and bool((dx_all[-GUARD:] == SENTINEL).all()), \
            "dE/dAEV written outside [rows_cap][ldx]"
