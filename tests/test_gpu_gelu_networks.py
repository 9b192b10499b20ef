"""GELU bias-free networks (ANI-2xr style) on the GPU: the ensemble-MLP kernels (csrc/gemm_tc.cuh,
csrc/mlp_resident.cuh) against float64, whole models against the gelu_* golden fixtures of the reference's
``simple_ani`` (oracle/make_gelu_golden.py), and the drop-in conversion of real reference models.

Every MLP entry point of the C-ABI runs a GELU model (ani_mlp_model::activation = ANI_ACT_GELU) on species-grouped
rows whose weights are rescaled layer by layer so that the pre-activations of all three layers spread over about
[-8, 8] (standard deviation 2.5), through the minimum of GELU near -0.75.  The reference is plain float64 torch on the
float32 weights and on the operand decoded back from its tiled form, as in tests/test_gpu_mlp.py, whose bars apply:
per row, normwise, 1e-5 of the row's max |ref| (2e-5 for the 3 x bf16 build) for the stored operands and dE/dAEV,
e_member within E_RTOL relative + E_ATOL.  Widths that are not multiples of 32 (100 / 72 / 40 ...) leave zero-padded
columns, where z = 0 gives GELU = 0 but GELU' = 1/2: the results stay exact only through the zero rows of the
transposed weights, which these cases check rather than assume.

Also: a CELU and a GELU model packed and run alternately in one process, each against its own reference, the operand
range check at the GELU sites a1, a2, G3, G2, G1 on the resident and chained launches, and rejected activation codes.
"""
import ctypes as C
import math
import os
import sys
import typing as tp

import numpy as np

import pytest
import torch

import oracle.ani_oracle as orc
import oracle.gelu_oracle as gor
import test_gpu_mlp as base
from helpers import E_ATOL, E_RTOL, F_ATOL, GOLD, ROOT, assert_close

F_RTOL = 1e-5    # forces: the repulsion's reach 160 Ha/A in the random batch (float32 positions), as in the pair tests
# 6w8h's shortest contacts give repulsion forces up to 5e3 Ha/A, which the float32 rounding of the positions alone moves
# by up to 2e-4 relative: its forces are compared with the float64 oracle on the float32-rounded positions instead
F32_ORACLE = ("6w8h_triclinic",)

pytestmark = pytest.mark.gpu

DEV = base.DEV
TILE = 128
ROW_BARS = base.ROW_BARS
# pre-activations up to |z| ~ 8 (not O(1) as in the plain cases of tests/test_gpu_mlp.py): the bars add this multiple of
# the propagated rounding-error scale, as test_gpu_mlp's wide-range cases do
MODEL_BAR = 8.0
Z_STD = 2.5
WIDTHS = {
    "w256": (("A", "B", "C"), {"A": (256, 192, 160), "B": (224, 192, 160), "C": (160, 128, 96)}, 1008),
    "odd": (("A", "B", "C"), {"A": (100, 72, 40), "B": (130, 100, 70), "C": (40, 33, 35)}, 1008),
}
ROWS = (300, 129, 1)
ROWS_BIG = (2000, 1000, 129)     # 25 row tiles: three windows of the data-flow list (ANI_B200_MLP_CHUNKS=3)


class Case(tp.NamedTuple):
    entry: str          # chained | split | split_dirty | forward | dataflow | chunks3 | slabs | resident | resident_members
    widths: str
    variant: str = ""


ENTRIES = ["chained", "split", "split_dirty", "forward", "dataflow", "chunks3", "slabs", "resident", "resident_members"]
CASES = [Case(e, w, v) for v in ("", "bf16x3") for w in WIDTHS for e in ENTRIES
         if not (v and e.startswith("resident"))]


def gelu(z):
    return 0.5 * z * (1.0 + torch.erf(z / math.sqrt(2.0)))


def dgelu(z):
    return 0.5 * (1.0 + torch.erf(z / math.sqrt(2.0))) + z * torch.exp(-0.5 * z * z) / math.sqrt(2.0 * math.pi)


def gelu_weights(widths: str, M: int, x64_rows: tp.List[torch.Tensor], in_dim: int, scale=(1.0, 1.0, 1.0, 1.0)):
    """Seeded bias-free float32 weights, each hidden layer rescaled so that its pre-activations on the rows of its
    species have standard deviation Z_STD (times ``scale``, per layer and w4)."""
    symbols, dims, _ = WIDTHS[widths]
    w = gor.make_weights(symbols, dims, in_dim, M, seed=777 + M)
    for s, sym in enumerate(symbols):
        x = x64_rows[s][:, :in_dim]
        for m in range(M):
            a = x
            layers = w[m][sym]
            for k in range(3):
                z = a @ layers[k][0].double().to(DEV).t()
                f = Z_STD / max(float(z.std()), 1e-30) * scale[k]
                layers[k] = ((layers[k][0] * f).float(), None)
                a = gelu(z * f)
            layers[3] = ((layers[3][0] * scale[3]).float(), None)
    return w


def d2gelu(z):
    return torch.exp(-0.5 * z * z) / math.sqrt(2.0 * math.pi) * (2.0 - z * z)


def reference(w, symbols, dims, s, M, ldx, x64, valid, scale):
    """float64 forward + backward of species s: z1..z3, a1, a2, d1, d2, G3, G2, G1 [M, R, padded width], e [M, R],
    dx [R, ldx] (member sum) and dxm [M, R, ldx].  With every value, ``d<name>`` holds the scale of its rounding error
    in units of the operand precision, propagated to first order as in tests/test_gpu_mlp.py reference(): a GEMM output
    carries |A| @ |B| of its own plus its inputs' errors through the weights (in quadrature), a stored value |value|,
    GELU(z) and GELU'(z) the pre-activation's error times GELU'(z) and GELU''(z)."""
    sym = symbols[s]
    h = dims[sym]
    p = [base._pad32(v) for v in h]
    W1 = torch.zeros(M, p[0], ldx, dtype=torch.float64)
    W2 = torch.zeros(M, p[1], p[0], dtype=torch.float64)
    W3 = torch.zeros(M, p[2], p[1], dtype=torch.float64)
    w4 = torch.zeros(M, p[2], dtype=torch.float64)
    for m in range(M):
        (a, _), (b, _), (c, _), (d, _) = w[m][sym]
        W1[m, :h[0], :a.shape[1]] = a.double()
        W2[m, :h[1], :h[0]] = b.double()
        W3[m, :h[2], :h[1]] = c.double()
        w4[m, :h[2]] = d.double().view(-1)
    W1, W2, W3, w4 = W1.to(DEV), W2.to(DEV), W3.to(DEV), w4.to(DEV).unsqueeze(1)
    X = x64.unsqueeze(0).expand(M, -1, -1)
    sq = lambda t: t * t    # noqa: E731
    rss = lambda *t: torch.sqrt(sum(sq(v) for v in t))   # noqa: E731

    def gemm(a, da, wt):   # z = a @ wt, its own error plus the inputs'
        return torch.bmm(a, wt), torch.bmm(a.abs(), wt.abs()) + torch.sqrt(torch.bmm(sq(da), sq(wt)))

    def act(z, dz):
        return gelu(z), rss(dgelu(z) * dz, gelu(z)), dgelu(z), rss(d2gelu(z) * dz, dgelu(z))

    z1, dz1 = gemm(X, torch.zeros_like(X), W1.transpose(1, 2))
    a1, da1, d1, dd1 = act(z1, dz1)
    z2, dz2 = gemm(a1, da1, W2.transpose(1, 2))
    a2, da2, d2, dd2 = act(z2, dz2)
    z3, dz3 = gemm(a2, da2, W3.transpose(1, 2))
    a3, da3, d3, dd3 = act(z3, dz3)
    e = (a3 * w4).sum(-1)
    de = (a3 * w4).abs().sum(-1) + torch.sqrt((sq(da3) * sq(w4)).sum(-1))
    seed = scale.view(M, 1, 1) * valid.view(1, -1, 1).to(torch.float64)
    G3, dG3 = seed * w4 * d3, (seed * w4).abs() * dd3
    P2, dP2 = gemm(G3, dG3, W3)
    G2, dG2 = P2 * d2, rss(dP2 * d2, P2 * dd2, P2 * d2)
    P1, dP1 = gemm(G2, dG2, W2)
    G1, dG1 = P1 * d1, rss(dP1 * d1, P1 * dd1, P1 * d1)
    dxm, ddxm = gemm(G1, dG1, W1)
    return dict(p=p, z=(z1, z2, z3), a1=a1, a2=a2, d1=d1, d2=d2, G3=G3, G2=G2, G1=G1, e=e, dx=dxm.sum(0), dxm=dxm,
                da1=da1, da2=da2, dd1=dd1, dd2=dd2, dG3=dG3, dG2=dG2, dG1=dG1, de=de,
                ddx=torch.sqrt(sq(ddxm).sum(0)), ddxm=ddxm)


def run_case(entry: str, widths: str, variant: str, monkeypatch, scale=(1.0, 1.0, 1.0, 1.0), M: int = 8,
             active=None, check: bool = True):
    """Runs one GELU case; returns (status word, fails, pre-activation range)."""
    from torchani_b200 import _lib
    from torchani_b200._lib import check as ok, ptr
    from torchani_b200.engine import PackedNetworks, operand_buffer, tile_a_operand, untile_a_operand
    if variant and not _lib.available(variant):
        pytest.skip(f"{_lib.variant_path(variant)} has not been built")
    base._set_env(monkeypatch, "chunks3" if entry == "chunks3" else "chained")
    fmt = _lib.operand_format(variant)
    L = _lib.lib(variant)
    symbols, dims, in_dim = WIDTHS[widths]
    S = len(symbols)
    rows = ROWS_BIG if entry == "chunks3" else ROWS
    n = sum(rows) + 2
    rows_cap = (n + S * (TILE - 1) + TILE - 1) // TILE * TILE
    seed = sum(map(ord, entry + widths + variant))
    row_atom, layout_info, first = base.make_layout(L, rows, S, rows_cap, seed)
    ldx = (in_dim + 31) // 32 * 32
    g = torch.Generator(device=DEV).manual_seed(seed)
    x_plain = (torch.rand(rows_cap, ldx, generator=g, device=DEV) * 2 - 1) * 3.0
    x_plain[:, in_dim:] = 0.0
    x_t = tile_a_operand(x_plain, variant=variant)
    x64 = untile_a_operand(x_t, rows_cap, ldx, variant=variant).double()
    w = gelu_weights(widths, M, [x64[first[s] * TILE:first[s + 1] * TILE] for s in range(S)], in_dim, scale)
    nets = PackedNetworks([[w[m][s] for s in symbols] for m in range(M)], in_dim, DEV, variant=variant,
                          activation=_lib.ACT_GELU)
    assert nets.model.activation == _lib.ACT_GELU
    active = list(range(M)) if active is None else list(active)
    model = _lib.MLPModel.from_buffer_copy(nets.model)
    for m in range(_lib.ANI_MAX_MEMBERS):
        model.member_scale[m] = (1.0 / len(active)) if m in active else 0.0
    scl = torch.tensor([model.member_scale[m] for m in range(M)], dtype=torch.float64, device=DEV)
    ld, cols = nets.ld, nets.act_cols
    assert cols == (2 * ld[0], 2 * ld[1], ld[2])
    act = [operand_buffer(rows_cap, c, DEV, variant) for c in cols]
    e_member = torch.full((M, rows_cap), base.SENTINEL, dtype=torch.float32, device=DEV)
    slabs = M if entry in ("slabs", "resident_members") else 1
    dx = torch.full((slabs * rows_cap * ldx,), base.SENTINEL, dtype=torch.float32, device=DEV)
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    sync = torch.zeros(6 * (rows_cap // TILE) * _lib.ANI_MAX_MEMBERS + 8, dtype=torch.int32, device=DEV)
    st = torch.cuda.current_stream(DEV).cuda_stream
    M_ = C.byref(model)
    A = [ptr(a) for a in act]
    fwd = None
    if entry in ("chained", "forward"):
        wb = int(entry == "chained")
        ok(L.ani_b200_mlp_forward_backward(M_, ptr(x_t), ptr(dx) if wb else None, rows_cap, ptr(row_atom),
                                           ptr(layout_info), None, *A, ptr(e_member), wb, ptr(status), st), entry)
    elif entry in ("split", "split_dirty"):
        ok(L.ani_b200_mlp_forward(M_, ptr(x_t), rows_cap, ptr(row_atom), ptr(layout_info), None, *A, ptr(e_member), 1,
                                  ptr(status), st), "mlp_forward")
        fwd = [a.clone() for a in act]
        zeroed = entry == "split"
        if zeroed:
            ok(L.ani_b200_zero_live_blocks(M_, ptr(dx), ptr(layout_info), None, st), "zero_live_blocks")
        ok(L.ani_b200_mlp_backward(M_, ptr(dx), rows_cap, ptr(row_atom), ptr(layout_info), None, *A, int(zeroed),
                                   ptr(status), st), "mlp_backward")
    elif entry in ("dataflow", "chunks3", "slabs"):
        if entry == "chunks3":
            assert L.ani_b200_mlp_step_windows(M_, rows_cap) == 3
        ok(L.ani_b200_mlp_step(M_, ptr(x_t), ptr(dx), rows_cap, ptr(row_atom), ptr(layout_info), None, *A,
                               ptr(e_member), 2 if entry == "slabs" else 1, ptr(sync), ptr(status), st), "mlp_step")
    elif entry == "resident":
        ok(L.ani_b200_mlp_step_resident(M_, ptr(x_t), ptr(dx), rows_cap, ptr(row_atom), ptr(layout_info), None, A[0],
                                        A[1], ptr(e_member), ptr(status), st), "mlp_step_resident")
    else:
        ok(L.ani_b200_mlp_step_resident_members(M_, ptr(x_t), ptr(dx), rows_cap * ldx, rows_cap, ptr(row_atom),
                                                ptr(layout_info), None, A[0], A[1], ptr(e_member), ptr(status), st),
           "mlp_step_resident_members")
    torch.cuda.synchronize()
    code = int(status.item())
    if not check:
        return code, [], None
    assert code == 0, f"status word {code}"

    sv, sg = fmt.value_scale, fmt.grad_scale
    dec = lambda t, c, sc: untile_a_operand(t, rows_cap, c, sc, variant=variant)  # noqa: E731
    got = {}

    def operand(t, i, second):   # act1 / act2 of a GELU model: [activation operand | derivative operand]
        n_el = rows_cap * fmt.parts * ld[i]
        return t.reshape(-1)[n_el if second else 0:][:n_el].view(rows_cap, fmt.parts * ld[i])
    half = lambda t, i, sc: dec(operand(t, i, False) if i < 2 else t, ld[i], sc)     # noqa: E731
    back = lambda t, i, sc: dec(operand(t, i, True), ld[i], sc)                      # noqa: E731
    if entry == "forward":
        got.update(a1=half(act[0], 0, sv), a2=half(act[1], 1, sv))
    elif entry.startswith("resident"):     # act1 / act2 hold d1 / d2 (no derivative operand behind them)
        got.update(d1=half(act[0], 0, sv), d2=half(act[1], 1, sv))
    else:
        got.update(G1=half(act[0], 0, sg), G2=half(act[1], 1, sg), G3=half(act[2], 2, sg),
                   d1=back(act[0], 0, sv), d2=back(act[1], 1, sv))
    if fwd is not None:
        got.update(a1=half(fwd[0], 0, sv), a2=half(fwd[1], 1, sv), G3_forward=half(fwd[2], 2, sg))
    row_bar = ROW_BARS[variant]
    tag = f"gelu {'bf16x3' if variant else 'fp16x2'}"
    fails: tp.List[str] = []
    ra = row_atom.cpu()
    dxv = dx.view(slabs, rows_cap, ldx)
    zmin, zmax = [], []
    for s in range(S):
        r0, r1 = first[s] * TILE, first[s + 1] * TILE
        valid = (ra[r0:r1] >= 0).to(DEV)
        ref = reference(w, symbols, dims, s, M, ldx, x64[r0:r1], valid, scl)
        for z in ref["z"]:
            zv = z[:, valid]
            zmin.append(float(zv.min()))
            zmax.append(float(zv.max()))
        p = ref["p"]
        where = f"{entry}/{widths}/{variant or 'fp16x2'} species {s}"
        for k, v in got.items():
            name = k.split("_")[0]
            wd = p[{"a1": 0, "a2": 1, "d1": 0, "d2": 1, "G3": 2, "G2": 1, "G1": 0}[name]]
            mine = v[r0:r1].reshape(r1 - r0, -1)[:, :M * wd].view(r1 - r0, M, wd).permute(1, 0, 2)
            refv, dref = ref[name], ref["d" + name]
            if name[0] in "ad":   # forward values of padding rows are not defined by the contract
                mine, refv, dref = mine[:, valid], refv[:, valid], dref[:, valid]
            if entry == "resident_members" and name[0] == "d":
                mine, refv, dref = mine[active], refv[active], dref[active]
            base.compare_rows(f"{tag} {name[0]}", mine, refv, dref, row_bar, MODEL_BAR, f"{where}: {k}", fails)
        em = e_member[:, r0:r1].double()
        live_m = torch.tensor([m in active for m in range(M)], device=DEV)
        real = valid.view(1, -1) & live_m.view(-1, 1)
        err = (em - ref["e"]).abs()
        if not bool((err <= E_ATOL + E_RTOL * ref["e"].abs() + MODEL_BAR * base.EPS * ref["de"])[real].all()):
            fails.append(f"{where}: e_member off by {float(err[real].max()):.3e}")
        if entry != "forward":
            if slabs > 1:
                mine, refv, dref = dxv[:, r0:r1].double()[active], ref["dxm"][active], ref["ddxm"][active]
            else:
                mine, refv, dref = dxv[0, r0:r1].double(), ref["dx"], ref["ddx"]
            base.compare_rows(f"{tag} dE/dAEV", mine[..., :in_dim], refv[..., :in_dim], dref[..., :in_dim], row_bar,
                              MODEL_BAR, f"{where}: dE/dAEV", fails)
    return code, fails, (min(zmin), max(zmax))


@pytest.mark.parametrize("case", CASES, ids=[f"{c.entry}-{c.widths}-{c.variant or 'fp16x2'}" for c in CASES])
def test_gelu_entry_points_match_float64(case: Case, monkeypatch):
    active = (1, 4, 6) if case.entry == "resident_members" else None
    _, fails, (zlo, zhi) = run_case(case.entry, case.widths, case.variant, monkeypatch, active=active)
    assert not fails, "\n".join(fails)
    assert zlo < -6.0 and zhi > 6.0, f"pre-activations cover only [{zlo:.2f}, {zhi:.2f}]"


def test_celu_and_gelu_models_alternate_in_one_process(monkeypatch):
    """A CELU model (test_gpu_mlp's seeded 1x widths) and a GELU model, packed side by side and run alternately through
    the chained and the resident launch: each keeps matching its own float64 reference."""
    for rnd in range(2):
        for entry in ("chained", "resident"):
            _, fails, _ = run_case(entry, "odd", "", monkeypatch)
            assert not fails, f"GELU after CELU, round {rnd}:\n" + "\n".join(fails)
            celu = base.Case(f"alternate_celu_{entry}_{rnd}", widths="1x", rows=(200, 130, 60, 1),
                             entry="chained" if entry == "chained" else "dataflow")
            base.test_mlp_gemm_matches_float64(celu, monkeypatch)


# Values over the range of the 2 x fp16 pieces at each GELU site, reached by rescaling one layer (the pre-activation
# std of layer k times the factor, and w4): a1 ~ |z1| > 1023.5, a2 likewise; G3 = scale * w4 * GELU'(z3) over 16; G2 over
# 16 with a2 small (layer 2 scaled down); G1 over 16 with a1 small.
OVER = {"a1": (600.0, 1.0, 1.0, 1.0), "a2": (1.0, 600.0, 1.0, 1.0), "G3": (1.0, 1.0, 1.0, 3000.0),
        "G2": (1.0, 1e-3, 1.0, 400.0), "G1": (1e-3, 1.0, 1.0, 400.0)}


@pytest.mark.parametrize("entry", ["resident", "chained"])
@pytest.mark.parametrize("site", list(OVER))
def test_gelu_operand_range_sites(site, entry, monkeypatch):
    code, _, _ = run_case(entry, "w256", "", monkeypatch, scale=OVER[site], check=False)
    from torchani_b200 import _lib
    assert code & _lib.STATUS_OPERAND_RANGE, f"{site} over the limit on the {entry} launch: status {code}"


def test_unknown_activation_code_is_rejected():
    from torchani_b200 import _lib
    from torchani_b200.engine import PackedNetworks
    symbols, dims, in_dim = WIDTHS["odd"]
    w = gor.make_weights(symbols, dims, in_dim, 2, seed=5)
    nets = PackedNetworks([[w[m][s] for s in symbols] for m in range(2)], in_dim, DEV, activation=_lib.ACT_GELU)
    model = _lib.MLPModel.from_buffer_copy(nets.model)
    model.activation = 2
    L = _lib.lib()
    n = 256
    dummy = torch.zeros(1 << 20, dtype=torch.int32, device=DEV)
    p = dummy.data_ptr()
    rc = L.ani_b200_mlp_forward_backward(C.byref(model), p, p, n, p, p, None, p, p, p, p, 1, p, 0)
    assert rc == -1                                            # ANI_ERR_BAD_ARG, before anything is launched
    rc = L.ani_b200_mlp_step_resident(C.byref(model), p, p, n, p, p, None, p, p, p, p, 0)
    assert rc == -1


# ---- whole models against the gelu_* fixtures ------------------------------------------------------------------------
SYMBOLS = gor.SYMBOLS      # the fixtures' (the reference's) element order
SYSTEMS = ["water999_pbc", "1c17_chunk_hcnos", "randbatch", "6w8h_triclinic", "sevenel_pbc", "small264_nopbc"]
RCR = gor.RCR
_cache: tp.Dict[tp.Any, tp.Any] = {}


def fixture(name):
    z = np.load(os.path.join(GOLD, f"gelu_{name}.npz"))
    return {k: z[k] for k in z.files}


def ref_forces(name):
    """The fixture's forces, or (F32_ORACLE) the float64 oracle's on the float32-rounded positions."""
    rec = fixture(name)
    if name not in F32_ORACLE:
        return rec["forces"]
    if ("f32", name) not in _cache:
        import oracle.pair_oracle as porc
        sp = torch.tensor(rec["species"])
        co = torch.tensor(rec["coords"]).float().double()
        cell = torch.tensor(rec["cell"]).float().double()
        pbc = torch.tensor(rec["pbc"])
        spec = gor.gelu_spec()
        w = gor.make_weights(SYMBOLS, orc.DIMS_2X, spec.out_dim, 8, int(rec["weight_seed"]))
        om = orc.Model(spec, SYMBOLS, w, dict(zip(SYMBOLS, rec["self_energies"].tolist())), "cell_list")
        zp = np.load(os.path.join(GOLD, "pair_params.npz"))
        tab = tuple(torch.tensor(_reorder(zp[k])).double() for k in ("y_ab", "sqrt_alpha_ab", "k_rep_ab"))
        f = gor.compute(om, sp, co, cell, pbc)["forces"] + porc.compute(porc.PairSpec("xtb", RCR, "smooth", tab), sp, co,
                                                                        cell, pbc, "cell_list")["forces"]
        _cache[("f32", name)] = f.numpy()
    return _cache[("f32", name)]


def e32_tol(rec, n_real):
    """Member energies come back in float32: two ulps of the largest total energy, plus 2e-6 Ha per atom."""
    return 2.0 * 2.0 ** -23 * float(np.abs(rec["energy"]).max()) * 2 + 2e-6 * max(n_real, 10)


def inputs(rec, dtype=torch.float32):
    sp = torch.tensor(rec["species"]).to(DEV)
    co = torch.tensor(rec["coords"]).to(dtype).to(DEV)
    cell = torch.tensor(rec["cell"]).to(dtype).to(DEV) if rec["cell"].size else None
    pbc = torch.tensor(rec["pbc"]).to(DEV) if rec["pbc"].size else None
    return sp, co, cell, pbc


def gelu_model(d3: bool = False, variant: str = ""):
    """The fixtures' model assembled here: simple_ani's AEV constants, ANINetworks.default (GELU, no biases) x 8 with
    the seeded weights, xTB repulsion at 5.2 A (the parameter tables of pair_params.npz in this element order) and
    optionally the D3 term of tests/test_gpu_dispersion.py (an ANI-2dr-shaped model)."""
    from torchani_b200 import models, nn
    key = (d3, variant)
    if key not in _cache:
        rec = fixture("water999_pbc")
        spec = gor.gelu_spec()
        aev = models.AEVComputer.from_constants(spec.rcr, spec.rca, spec.eta_r, spec.shf_r, spec.eta_a, spec.zeta,
                                                spec.shf_a, spec.shf_z, 7, cutoff_fn="smooth")
        w = gor.make_weights(SYMBOLS, orc.DIMS_2X, spec.out_dim, 8, int(rec["weight_seed"]))
        members = [nn.ANINetworks.default(SYMBOLS, spec.out_dim) for _ in range(8)]
        with torch.no_grad():
            for net, wm in zip(members, w):
                for s in SYMBOLS:
                    for (dst, b), (src, _) in zip(net.atomics[s].linear_pairs(), wm[s]):
                        assert b is None
                        dst.copy_(src)
        sae = models.SelfEnergy(SYMBOLS, rec["self_energies"].tolist())
        pots = {"repulsion_xtb": xtb_module()}
        if d3:
            pots["dispersion_d3"] = d3_module()
        m = models.ANI(SYMBOLS, aev, nn.Ensemble(members), sae, False, pots).to(DEV)
        m.requires_grad_(False)
        if variant:
            m.neural_networks.use_variant(variant)
        _cache[key] = m
    return _cache[key]


PERM = [orc.SYMBOLS_2X.index(s) for s in SYMBOLS]


def _reorder(a):
    """A per-element table of the SYMBOLS_2X order (element axes first) in the fixtures' order."""
    a = np.asarray(a)
    for ax in range(min(a.ndim, 2)):
        if a.shape[ax] == len(PERM):
            a = np.take(a, PERM, axis=ax)
    return a


def xtb_module():
    from torchani_b200 import potentials as P
    zp = np.load(os.path.join(GOLD, "pair_params.npz"))
    pot = P.RepulsionXTB(SYMBOLS, alpha=[1.0] * 7, yeff=[1.0] * 7, cutoff=RCR, cutoff_fn="smooth")
    for key in ("y_ab", "sqrt_alpha_ab", "k_rep_ab"):
        getattr(pot, key).copy_(torch.tensor(_reorder(zp[key])).float())
    return pot


def d3_module():
    """tests/test_gpu_dispersion.py's D3 module (the buffers of the d3_ fixtures), in the fixtures' element order."""
    import test_gpu_dispersion as disp
    from torchani_b200 import potentials as P
    z = {k: _reorder(v) for k, v in disp.params_npz().items()}
    sq = np.sqrt(np.diag(z["sqrt_charge_ab"]))
    pot = P.TwoBodyDispersionD3(SYMBOLS, float(z["s6"]), float(z["s8"]), float(z["a1"]), float(z["a2"]),
                                sq.tolist(), (z["covalent_radii"] / P.ANGSTROM_TO_BOHR).tolist(),
                                coeff6=z["precalc_coeff6"], coordnums_a=z["precalc_coordnums_a"],
                                coordnums_b=z["precalc_coordnums_b"], cutoff=disp.CUTOFF, cutoff_fn="smooth")
    for key in ("sqrt_charge_ab", "covalent_radii"):
        getattr(pot, key).copy_(torch.tensor(z[key]).float())
    pot._damp_fn.cutoff_radii.copy_(torch.tensor(z["cutoff_radii"]).float())
    return pot


@pytest.mark.parametrize("launch", ["auto", "1", "0", "bf16x3"], ids=["resident", "dataflow", "chained", "bf16x3"])
@pytest.mark.parametrize("name", SYSTEMS)
def test_gelu_model_matches_the_reference_fixtures(name, launch):
    rec = fixture(name)
    m = gelu_model(variant="bf16x3" if launch == "bf16x3" else "")
    eng = m.engine(torch.device(DEV))
    saved = eng.mlp_mode
    eng.mlp_mode = "auto" if launch == "bf16x3" else launch
    try:
        sp, co, cell, pbc = inputs(rec)
        n_real = int((sp >= 0).sum(1).max())
        e, f = m.energies_and_forces(sp, co, cell, pbc)
        assert_close(f"{name} energies", e.cpu().numpy(), rec["energy"], 2e-7, 2e-7 * max(n_real, 10) + 1e-5)
        assert_close(f"{name} forces", f.cpu().numpy(), ref_forces(name), F_RTOL, F_ATOL)
        ev = m((sp, co), cell, pbc, ensemble_values=True).energies.double().cpu()      # (M, C): NN + sae + xTB
        nn_m = rec["member_atomic"].sum(-1)                                           # (M, C) NN only
        assert_close(f"{name} member spread", (ev - ev.mean(0)).numpy(), nn_m - nn_m.mean(0), 0.0,
                     e32_tol(rec, n_real))
        if cell is not None and launch == "auto":
            _, _, stress = m.energies_forces_stress(sp, co, cell, pbc)
            assert_close(f"{name} stress", stress.cpu().numpy()[0] if stress.dim() == 3 else stress.cpu().numpy(),
                         rec["stress"], 1e-4, 2e-7)
    finally:
        eng.mlp_mode = saved


@pytest.mark.parametrize("name", ["water999_pbc", "randbatch"])
def test_gelu_members_forces_and_qbc(name):
    rec = fixture(name)
    m = gelu_model()
    sp, co, cell, pbc = inputs(rec)
    n_real = (sp >= 0).sum(1).double().cpu()
    _, e_m, f_m = m.members_forces((sp, co), cell, pbc)
    nn_m = rec["member_atomic"].sum(-1)
    tol = e32_tol(rec, int(n_real.max()))
    assert_close(f"{name} member energies", (e_m.double().cpu() - e_m.double().cpu().mean(0)).numpy(),
                 nn_m - nn_m.mean(0), 0.0, tol)
    assert_close(f"{name} mean member forces", f_m.double().mean(0).cpu().numpy(), rec["forces"], F_RTOL, F_ATOL)
    _, e, qbc = m.energies_qbcs((sp, co), cell, pbc)
    ref_qbc = torch.tensor(nn_m).std(0, unbiased=True) / n_real.sqrt()
    assert_close(f"{name} qbc", qbc.double().cpu().numpy(), ref_qbc.numpy(), 1e-4, tol / float(n_real.min().sqrt()))


@pytest.mark.parametrize("per_conformer", [False, True], ids=["shared_cell", "cell_per_conformer"])
def test_gelu_periodic_batch(per_conformer):
    rec = fixture("water999_pbc")
    m = gelu_model()
    sp, co, cell, pbc = inputs(rec)
    shift = torch.tensor([0.3, -0.2, 0.5], device=DEV)      # the second conformer: the same system translated
    spb, cob = torch.cat([sp, sp]), torch.cat([co, co + shift])
    cellb = torch.stack([cell, cell]) if per_conformer else cell
    e, f = m.energies_and_forces(spb, cob, cellb, pbc)
    n = int((sp >= 0).sum())
    for c in range(2):
        assert_close(f"conformer {c} energy", e[c:c + 1].cpu().numpy(), rec["energy"], 2e-7, 2e-7 * n + 1e-5)
        assert_close(f"conformer {c} forces", f[c:c + 1].cpu().numpy(), rec["forces"], F_RTOL, F_ATOL)


def test_gelu_graph_replay_matches_fresh_evaluation():
    rec = fixture("1c17_chunk_hcnos")
    m = gelu_model()
    sp, co, cell, pbc = inputs(rec)
    outs = [m.energies_and_forces(sp, co, cell, pbc) for _ in range(5)]    # the later calls replay a captured graph
    for e, f in outs[1:]:
        assert torch.equal(e, outs[0][0]) or float((e - outs[0][0]).abs().max()) < 1e-6 * float(e.abs().max())
        assert float((f - outs[0][1]).abs().max()) < 1e-5
    assert_close("replayed energy", outs[-1][0].cpu().numpy(), rec["energy"], 2e-7, 2e-7 * sp.shape[1] + 1e-5)
    assert_close("replayed forces", outs[-1][1].cpu().numpy(), rec["forces"], F_RTOL, F_ATOL)


def test_gelu_ase_calculator():
    try:
        import ase  # noqa: F401
    except ImportError:
        sys.path.insert(0, os.path.join(ROOT, "tests", "stubs"))
    from ase import Atoms
    from torchani_b200 import models
    HA = 27.211386024367243
    rec = fixture("water999_pbc")
    base_m = gelu_model()
    m = models.ANI(SYMBOLS, base_m.aev_computer, base_m.neural_networks, base_m.energy_shifter, True,
                   dict(base_m.potentials.items()) if hasattr(base_m, "potentials") else {}).to(DEV)
    atoms = Atoms(rec["atomic_numbers"][0].tolist(), rec["coords"][0], cell=rec["cell"], pbc=True)
    atoms.calc = m.ase()
    n = len(atoms.get_positions())
    assert abs(atoms.get_potential_energy() / HA - float(rec["energy"][0])) < 2e-7 * n + 1e-4
    assert np.abs(atoms.get_forces() / HA - rec["forces"][0]).max() < F_ATOL
    assert np.abs(atoms.get_stress() / HA - rec["stress"]).max() < 1e-6 + 1e-3 * np.abs(rec["stress"]).max()


@pytest.mark.parametrize("name", ["water999_pbc", "6w8h_triclinic", "1c17_chunk_hcnos"])
def test_gelu_with_d3_like_ani2dr(name):
    """Networks + xTB + D3: the gelu fixture plus the D3 term of the d3_ fixture of the same system."""
    import test_gpu_dispersion as disp
    rec = fixture(name)
    d3 = disp.d3_golden(name + "_ani2x")
    m = gelu_model(d3=True)
    sp, co, cell, pbc = inputs(rec)
    e, f = m.energies_and_forces(sp, co, cell, pbc)
    n = int((sp >= 0).sum(1).max())
    ref_e = rec["energy"] + d3["smooth_energy"]
    ref_f = ref_forces(name) + d3["smooth_forces"]
    assert_close(f"{name} energies", e.cpu().numpy(), ref_e, 2e-7, 2e-7 * n + 1e-5)
    assert_close(f"{name} forces", f.cpu().numpy(), ref_f, F_RTOL, F_ATOL)


# ---- drop-in against the real reference (oracle/_ref) ---------------------------------------------------------------
def _reference_simple_ani():
    import oracle.ref_torchani as rt
    if not rt.available():
        pytest.skip("the reference is not staged (oracle/_ref)")
    torchani = rt.load()
    rec = fixture("water999_pbc")
    ref = torchani.arch.simple_ani(list(SYMBOLS), "wb97x-631gd", ensemble_size=8, strategy="pyaev", repulsion=True,
                                   dispersion=False)
    w = gor.make_weights(SYMBOLS, orc.DIMS_2X, gor.gelu_spec().out_dim, 8, int(rec["weight_seed"]))
    with torch.no_grad():
        for member, wm in zip(ref.potentials["nnp"].neural_networks.members, w):
            for s in SYMBOLS:
                an = member.atomics[s]
                for layer, (src, _) in zip(list(an.layers) + [an.final_layer], wm[s]):
                    layer.weight.copy_(src)
    return ref.to(DEV)


def _check_fixture(m, name, tag):
    rec = fixture(name)
    sp = torch.tensor(rec["atomic_numbers"]).to(DEV)
    co = torch.tensor(rec["coords"]).float().to(DEV).requires_grad_(True)
    cell = torch.tensor(rec["cell"]).float().to(DEV) if rec["cell"].size else None
    pbc = torch.tensor(rec["pbc"]).to(DEV) if rec["pbc"].size else None
    e = m((sp, co), cell, pbc).energies
    (g,) = torch.autograd.grad(e.sum(), co)
    n = int((sp >= 0).sum(1).max())
    assert_close(f"{tag} {name} energies", e.detach().double().cpu().numpy(), rec["energy"], 2e-7, 2e-7 * n + 1e-4)
    assert_close(f"{tag} {name} forces", (-g).double().cpu().numpy(), rec["forces"], F_RTOL, F_ATOL)


def test_from_torchani_of_a_reference_simple_ani_model():
    from torchani_b200 import models, nn
    ref = _reference_simple_ani()
    ours = models.from_torchani(ref)
    assert isinstance(ours.neural_networks, nn.Ensemble)
    assert ours.neural_networks[0].activation_kind == 1 and not ours.neural_networks[0].atomics["H"].has_biases
    for name in ("water999_pbc", "randbatch"):
        _check_fixture(ours, name, "from_torchani")
    bmm = models.from_torchani(ref.to_infer_model())      # BmmEnsemble: _beta == 0, no biases
    _check_fixture(bmm, "randbatch", "from_torchani(to_infer_model())")


def test_accelerate_torchani_of_a_reference_simple_ani_model():
    from torchani_b200 import models
    ref = _reference_simple_ani()
    models.accelerate_torchani_(ref)
    _check_fixture(ref, "water999_pbc", "accelerate_torchani_")


def test_reference_state_dict_loads_into_a_model_assembled_here():
    from torchani_b200 import models
    ref = _reference_simple_ani()
    mine = gelu_model()
    target = models.ANI(SYMBOLS, mine.aev_computer, mine.neural_networks, mine.energy_shifter, True,
                        dict(mine.potentials.items())).to(DEV)
    with torch.no_grad():
        for p in target.neural_networks.parameters():
            p.zero_()
    # (the species converters' tables differ in length: this package's covers the elements it supports)
    sd = {k: v for k, v in ref.state_dict().items() if not k.startswith("species_converter.")}
    missing, unexpected = target.load_state_dict(sd, strict=False)
    assert not [k for k in missing if "neural_networks" in k], missing
    _check_fixture(target, "water999_pbc", "load_state_dict")
