"""The step terms (csrc/pair.cu, csrc/disp.cu) against float64 where the golden fixtures never take them: pair cutoffs
below Rcr, the xTB ``powf`` branch and non-default ZBL constants, two pair terms in one step, D3 stencil reaches 1, 2,
3, reach = dims and its refusal, open-system clipping (planar and linear molecules too), the hit queue of grid mode 1
beyond 32 hits per atom, element counts 1, 4 and 8 (an element pair without a C6 reference, C6 exponents at the e^80
cap), a Verlet skin, partial PBC, and the half-list entry points on padded batches, periodic lists, without an envelope
and on an empty list.

The kernels run as ``test_gpu_pair_potentials.pair_only`` / ``test_gpu_dispersion.d3_only`` run them (the step's
preparation and AEV forward, then the term into zeroed outputs) on engines with tiny synthetic networks
(``test_gpu_aev.tiny_weights``), or through the public model API where the case is about the model.  The reference is
``oracle/pair_oracle.py`` / ``oracle/d3_oracle.py`` in float64 on the float32-rounded inputs (periodic ones wrapped
into the cell), with the bars of the two existing modules: pair atomic 1e-5 |e| + 1e-6 Ha, forces 1e-5 |F| + 1e-4
Ha/A, conformer energies 1e-6 |E| + 1e-5 Ha; D3 conformer energies 1e-5 |E|, atomic 1e-5 |e| + 1e-9 Ha, forces 1e-4
max |F| + 1e-8 Ha/A, stress 1e-4 max |s|.  The 6W8H box keeps the wider pair bars of ``test_gpu_pair_potentials``
(overlapping atoms at |x| up to 49 A, measured there).

The host-only tests (no GPU) assert that every case reaches the branch it names: the reach
``ceil((cutoff + skin) dims_d / perp_d)`` of each D3 system restated from the bucket-grid rule of csrc/cells.cu (the
GPU tests compare it with the step's own ``ani_grid``), clipping, hits per atom, pairs in (cutoff, Rcr], ``k_rep``
values, element counts, and the no-reference and capped-exponent pairs from the oracle's float64 coordination numbers.
The module prints the worst error / bar of every group at its end (pytest -s).

Measured on an H100 80GB HBM3 (700 W power limit), worst error / bar: pair below Rcr 0.22, custom pair parameters
0.07, two pair terms 0.08; D3 reach 1 / 2 / 3 0.09 / 0.08 / 0.14 (reach 0, the flat molecules, 0.02), hit queue 0.17;
S = 1 / 4 / 8 0.57 / 0.19 / 0.16; Verlet skin 0.02, partial PBC 0.02; half lists xTB 0.08, ZBL 0.09, D3 0.40, without
envelope 0.03.  The GPU part of the module takes about 17 s.
"""
import math
import os
import typing as tp

import numpy as np
import pytest
import torch

import oracle.ani_oracle as orc
import oracle.d3_oracle as d3o
import oracle.pair_oracle as porc
import test_gpu_dispersion as td3
import test_gpu_pair_potentials as tpp
from helpers import E_ATOL, E_RTOL, F_ATOL, GOLD, golden_inputs, load_golden
from test_gpu_aev import tiny_weights

DEV = "cuda:0"
RCR = 5.1
F_RTOL = tpp.F_RTOL
PBC3 = torch.tensor([True, True, True])
LN_EPS = math.log(1e-35)          # D3_LN_EPS of csrc/disp.cu
SYMS = {1: ("C",), 4: ("H", "C", "S", "F"), 7: orc.SYMBOLS_2X, 8: orc.SYMBOLS_2X + ("Br",)}

_WORST: tp.Dict[str, float] = {}
_cache: tp.Dict[tp.Any, tp.Any] = {}


def _note(group: str, ratio: float) -> None:
    _WORST[group] = max(_WORST.get(group, 0.0), ratio)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if _WORST:
        print("\nworst error / bar of test_gpu_step_terms.py:")
        for k in sorted(_WORST):
            print(f"  {k:28s} {_WORST[k]:.3f}")


def close(group: str, tag: str, got, ref, rtol: float, atol: float) -> None:
    got = np.asarray(got, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    err = np.abs(got - ref)
    bound = atol + rtol * np.abs(ref)
    ratio = float(np.where(bound > 0, err / np.where(bound > 0, bound, 1.0), np.where(err > 0, np.inf, 0.0)).max()) \
        if err.size else 0.0
    _note(group, ratio)
    assert ratio <= 1.0, f"{tag}: max-abs err {err.max():.3e} (|ref| max {np.abs(ref).max():.3e}), {ratio:.3f} of the bar"


# ------------------------------------------------------------------------------------------------------------------
# systems: (species (C, A), coords (C, A, 3) float64 holding float32 values, cell None / (3, 3) / (C, 3, 3), pbc)
# ------------------------------------------------------------------------------------------------------------------
class Sys(tp.NamedTuple):
    species: torch.Tensor
    coords: torch.Tensor
    cell: tp.Optional[torch.Tensor]
    pbc: tp.Optional[torch.Tensor]


def f32(t):
    return None if t is None else t.float().double()


def golden_sys(name: str) -> Sys:
    sp, co, cell, pbc = golden_inputs(load_golden(name))
    co, cell = f32(co), f32(cell)
    if cell is not None:
        co = f32(td3.wrapped(co, cell))
    return Sys(sp, co, cell, pbc)


def placed(n: int, seed: int, min_dist: float, cell: tp.Optional[np.ndarray] = None, radius: float = 0.0) -> np.ndarray:
    """n points a minimum (image) distance apart: in a periodic cell, or in a ball of `radius` about the origin."""
    rng = np.random.default_rng(seed)
    pts = np.zeros((0, 3))
    while len(pts) < n:
        if cell is not None:
            p = rng.uniform(0.0, 1.0, 3) @ cell
            d = (pts - p) @ np.linalg.inv(cell)
            d = (d - np.round(d)) @ cell
        else:
            p = rng.uniform(-radius, radius, 3)
            if p @ p > radius * radius:
                continue
            d = pts - p
        if len(pts) == 0 or float((d * d).sum(1).min()) >= min_dist ** 2:
            pts = np.vstack([pts, p])
    return pts


def box_sys(n: int, width: float, S: int, seed: int, min_dist: float = 1.0) -> Sys:
    cell = np.eye(3) * width
    x = placed(n, seed, min_dist, cell)
    sp = torch.tensor([k % S for k in range(n)]).view(1, -1)
    return Sys(sp, f32(torch.tensor(x)).view(1, -1, 3), f32(torch.tensor(cell)), PBC3)


def molecule_sys(kind: str) -> Sys:
    """Benzene in the plane z = 0 (bounding box 2e-3 A thick in z) or H-C#C-C#C-H on the x axis (thick in y and z)."""
    if kind == "planar":
        ang = np.arange(6) * np.pi / 3
        ring = np.stack([np.cos(ang), np.sin(ang), np.zeros(6)], 1)
        x = np.concatenate([1.39 * ring, 2.47 * ring])
        sp = [1] * 6 + [0] * 6
    else:
        x = np.zeros((6, 3))
        x[:, 0] = np.cumsum([0.0, 1.06, 1.20, 1.38, 1.20, 1.06])
        sp = [0, 1, 1, 1, 1, 0]
    return Sys(torch.tensor(sp).view(1, -1), f32(torch.tensor(x)).view(1, -1, 3), None, None)


QUEUE_REAL = [31, 32, 33, 64, 65, 97]
QUEUE_CUTOFF = 15.0


def queue_batch() -> Sys:
    """An open batch (grid mode 1) of conformers with 31 .. 97 real atoms in a ball of radius 7.3 A (every pair within
    the 15 A cutoff), padding scattered between them."""
    A = 100
    g = np.random.default_rng(11)
    sp = -torch.ones(len(QUEUE_REAL), A, dtype=torch.long)
    co = torch.zeros(len(QUEUE_REAL), A, 3, dtype=torch.float64)
    for c, n in enumerate(QUEUE_REAL):
        slots = np.sort(g.permutation(A)[:n])
        sp[c, slots] = torch.tensor(g.integers(0, 7, n))
        co[c, slots] = torch.tensor(placed(n, 100 + c, 1.4, radius=7.3))
    return Sys(sp, f32(co), None, None)


def pair_sys(name: str) -> Sys:
    if name in ("mode2", "mode3"):
        sp, co, cell = tpp.periodic_batch(name == "mode3")
        return Sys(sp, f32(co), f32(cell), PBC3)
    return golden_sys(name)


def d3_sys(name: str) -> Sys:
    """The systems of the D3 reach / refusal / clipping cases."""
    if name not in _cache:
        if name.startswith("cube"):      # cube<width>: 30 atoms in a cubic cell of that width
            s = box_sys(30, float(name[4:]), 7, seed=5, min_dist=1.2)
        elif name == "dilute":           # 60 atoms in 30 A: the bucket capacity narrows the grid to 3 x 4 x 4
            s = box_sys(60, 30.0, 7, seed=6, min_dist=1.5)
        elif name in ("planar", "linear"):
            s = molecule_sys(name)
        elif name.startswith("box_s"):   # the element-count boxes
            S = int(name[5:])
            s = box_sys(300, 18.2, S, seed=S, min_dist=1.3)
        else:
            s = golden_sys(name)
        _cache[name] = s
    return _cache[name]


# ------------------------------------------------------------------------------------------------------------------
# the bucket grid and the D3 stencil, restated (csrc/cells.cu compute_grid, csrc/disp.cu d3_neighbours)
# ------------------------------------------------------------------------------------------------------------------
def grid_dims(s: Sys, grid_cutoff: float = RCR) -> tp.Tuple[tp.List[int], np.ndarray]:
    """dims and the float32 inverse (column norms = 1 / perpendicular widths) of a single system's grid."""
    b = np.float32(np.float32(grid_cutoff) + np.float32(1e-5))
    n = s.species.numel()
    if s.cell is not None:
        inv64 = np.linalg.inv(s.cell.numpy())
        widths = 1.0 / np.linalg.norm(inv64, axis=0)
        dims = [max(1, int(math.floor(w / float(b)))) for w in widths]
        inv = inv64.astype(np.float32)
    else:
        x = s.coords[0][s.species[0] >= 0].numpy().astype(np.float32)
        ext = (x.max(0) - x.min(0)) + np.float32(2e-3)
        dims = [max(1, int(math.floor(np.float32(e) / b))) for e in ext]
        inv = np.diag(np.float32(1.0) / ext).astype(np.float32)
    cap = max(64, n + 2) - 1
    while dims[0] * dims[1] * dims[2] > cap:
        big = int(np.argmax(dims))
        dims[big] = max(1, dims[big] - max(1, dims[big] // 8))
    return dims, inv


def reach(dims: tp.Sequence[int], inv: np.ndarray, cutoff: float, skin: float, pbc: bool
          ) -> tp.Tuple[tp.Optional[tp.List[int]], tp.List[int]]:
    """(the stencil reach per lattice direction, or None where a periodic width is below cutoff + skin; the reach
    before clipping) in the float32 arithmetic of the kernel."""
    L = np.float32(np.float32(cutoff) + np.float32(skin))
    raw = []
    for d in range(3):
        col = inv[:, d].astype(np.float32)
        perp = np.float32(1.0) / np.sqrt(np.float32((col * col).sum(dtype=np.float32)))
        raw.append(int(math.ceil(np.float32(L * np.float32(dims[d])) / perp)))
    if pbc:
        return (None if any(r > n for r, n in zip(raw, dims)) else list(raw)), raw
    return [min(r, n - 1) for r, n in zip(raw, dims)], raw


# D3 cases of the fused step: (system, cutoff) -> the reach they must reach
D3_REACH = [("water999_pbc_ani2x", 4.0), ("water999_pbc_ani2x", 8.0), ("water999_pbc_ani2x", 12.0), ("dilute", 8.0),
            ("tightcell_pbc_ani2x", 11.0), ("cube11.01", 11.0), ("1c17_chunk_hcnos_ani2x", 12.0), ("planar", 8.0),
            ("linear", 8.0)]
D3_REFUSED = ("cube10.99", 11.0)


# ------------------------------------------------------------------------------------------------------------------
# terms and their oracles
# ------------------------------------------------------------------------------------------------------------------
def xtb_custom(S: int, cutoff: float = RCR, fn: str = "smooth", krep: float = 1.3, krep_h: float = 0.8):
    from torchani_b200 import potentials as P
    g = np.random.default_rng(40 + S)
    return P.RepulsionXTB(SYMS[S], krep_hydrogen=krep_h, krep=krep, alpha=g.uniform(0.8, 1.6, S).tolist(),
                          yeff=g.uniform(0.5, 4.0, S).tolist(), cutoff=cutoff, cutoff_fn=fn)


def zbl_custom(S: int, cutoff: float = RCR, fn: str = "cosine"):
    from torchani_b200 import potentials as P
    from torchani_b200.nn import ATOMIC_NUMBER
    return P.RepulsionZBL(SYMS[S], k=0.91, screen_coeffs=(0.2, 0.45, 0.3, 0.05),
                          screen_exponents=(3.0, 1.05, 0.45, 0.25), eff_exponent=0.3,
                          eff_atomic_nums=[0.9 * ATOMIC_NUMBER[s] + 0.1 for s in SYMS[S]], cutoff=cutoff, cutoff_fn=fn)


def pair_spec(pot) -> porc.PairSpec:
    """The float64 oracle's spec of a module, from its (float32) buffers."""
    fn = pot.cutoff_fn
    if pot.kind == 0:
        return porc.PairSpec("xtb", pot.cutoff, fn, tuple(getattr(pot, k).double().cpu() for k in
                                                          ("y_ab", "sqrt_alpha_ab", "k_rep_ab")))
    return porc.PairSpec("zbl", pot.cutoff, fn, (pot._eff_atomic_nums.double().cpu(),), k=pot._k,
                         eff_exponent=pot._kz, coeffs=tuple(pot._coeffs.view(-1).tolist()),
                         exponents=tuple(pot._exponents.view(-1).tolist()))


def d3_tables(S: int) -> tp.Dict[str, tp.Any]:
    """The fixture's D3 tables for the elements SYMS[S] (S <= 7), or (S = 8) the seven fixture elements and a Br whose
    reference coordination numbers (14 .. 16) lie far beyond any an atom reaches: every C6 exponent of its pairs is
    at the e^80 cap.  The fixture has no C6 reference for S-F."""
    z = {k: np.asarray(v) for k, v in np.load(os.path.join(GOLD, "d3_params.npz")).items()}
    if S <= 7:
        ix = [orc.SYMBOLS_2X.index(s) for s in SYMS[S]]
        out = {k: z[k] for k in ("s6", "s8", "a1", "a2")}
        out["covalent_radii"] = z["covalent_radii"][ix]
        for k in ("cutoff_radii", "sqrt_charge_ab", "precalc_coeff6", "precalc_coordnums_a", "precalc_coordnums_b"):
            out[k] = z[k][np.ix_(ix, ix)]
        return out
    out = {k: z[k] for k in ("s6", "s8", "a1", "a2")}
    out["covalent_radii"] = np.append(z["covalent_radii"], 1.12 * z["covalent_radii"][6])
    sq = np.append(np.sqrt(np.diag(z["sqrt_charge_ab"])), 1.1 * np.sqrt(z["sqrt_charge_ab"][6, 6]))
    out["sqrt_charge_ab"] = np.outer(sq, sq)
    cr = np.zeros((8, 8))
    cr[:7, :7] = z["cutoff_radii"]
    cr[7, :7] = cr[:7, 7] = 1.05 * z["cutoff_radii"][6]
    cr[7, 7] = 1.1 * z["cutoff_radii"][6, 6]
    out["cutoff_radii"] = cr
    c6, cna, cnb = (-np.ones((8, 8, 5, 5)) for _ in range(3))
    c6[:7, :7], cna[:7, :7], cnb[:7, :7] = (z[k] for k in ("precalc_coeff6", "precalc_coordnums_a",
                                                          "precalc_coordnums_b"))
    own = 14.0 + np.arange(5)          # Br's reference CNs: row p of the Cl tables
    for b in range(7):
        ok = z["precalc_coeff6"][6, b] > 0
        c6[7, b] = np.where(ok, 1.3 * z["precalc_coeff6"][6, b], -1.0)
        cna[7, b] = np.where(ok, own.reshape(5, 1), -1.0)
        cnb[7, b] = np.where(ok, z["precalc_coordnums_b"][6, b], -1.0)
        c6[b, 7], cna[b, 7], cnb[b, 7] = c6[7, b].T, cnb[7, b].T, cna[7, b].T
    ok = z["precalc_coeff6"][6, 6] > 0
    c6[7, 7] = np.where(ok, 1.69 * z["precalc_coeff6"][6, 6], -1.0)
    cna[7, 7] = np.where(ok, own.reshape(5, 1), -1.0)
    cnb[7, 7] = np.where(ok, own.reshape(1, 5), -1.0)
    out.update(precalc_coeff6=c6, precalc_coordnums_a=cna, precalc_coordnums_b=cnb)
    return out


def d3_term(S: int, cutoff: float, fn: str = "smooth"):
    from torchani_b200 import potentials as P
    z = d3_tables(S)
    pot = P.TwoBodyDispersionD3(SYMS[S], float(z["s6"]), float(z["s8"]), float(z["a1"]), float(z["a2"]),
                                np.sqrt(np.diag(z["sqrt_charge_ab"])).tolist(),
                                (z["covalent_radii"] / P.ANGSTROM_TO_BOHR).tolist(), coeff6=z["precalc_coeff6"],
                                coordnums_a=z["precalc_coordnums_a"], coordnums_b=z["precalc_coordnums_b"],
                                cutoff=cutoff, cutoff_fn=fn)
    for key in ("sqrt_charge_ab", "covalent_radii"):
        getattr(pot, key).copy_(torch.tensor(z[key]).float())
    pot._damp_fn.cutoff_radii.copy_(torch.tensor(z["cutoff_radii"]).float())
    return pot


def d3_spec(pot) -> d3o.D3Spec:
    return d3o.D3Spec(pot.cutoff, pot.cutoff_fn, pot._s6, pot._s8, pot._damp_fn._a1, pot._damp_fn._a2,
                      pot._damp_fn.cutoff_radii.double().cpu(), pot.sqrt_charge_ab.double().cpu(),
                      pot.covalent_radii.double().cpu(), pot.precalc_coeff6.double().cpu(),
                      pot.precalc_coordnums_a.double().cpu(), pot.precalc_coordnums_b.double().cpu())


def oracle(terms: tp.Sequence[tp.Tuple[tp.Any, tp.Any]], s: Sys, stress: bool = False,
           nl: tp.Optional[str] = None) -> tp.Dict[str, np.ndarray]:
    """Sum of float64 oracles ((module, spec) pairs: pair_oracle / d3_oracle) conformer by conformer; "stress" (C, 3, 3)
    with `stress`.  Small systems take the all-pairs list, large ones the cell list."""
    out: tp.Dict[str, tp.List[torch.Tensor]] = {}
    for c in range(s.species.shape[0]):
        ck = None if s.cell is None else (s.cell[c] if s.cell.dim() == 3 else s.cell)
        kind = nl or ("all_pairs" if s.species.shape[1] <= 400 else "cell_list")
        acc: tp.Dict[str, torch.Tensor] = {}
        for mod, spec in terms:
            r = mod.compute(spec, s.species[c:c + 1], s.coords[c:c + 1], ck, s.pbc if ck is not None else None, kind,
                            stress=stress)
            acc = r if not acc else {k: acc[k] + r[k] for k in acc}
        for k, v in acc.items():
            out.setdefault(k, []).append(v if k != "stress" else v.unsqueeze(0))
    return {k: torch.cat(v).numpy() for k, v in out.items()}


# ------------------------------------------------------------------------------------------------------------------
# engines with tiny networks (the networks play no part in pair_only / d3_only)
# ------------------------------------------------------------------------------------------------------------------
def engine(key: str, S: int, pairs=(), d3=None):
    from torchani_b200.engine import AEVConstants, Engine, PackedNetworks
    if ("engine", key) not in _cache:
        consts = AEVConstants(*orc.aev_spec_2x(S))
        symbols, w = tiny_weights(S, consts.out_dim)
        nets = PackedNetworks([[wm[s] for s in symbols] for wm in w], consts.out_dim, torch.device(DEV),
                              radial_len=consts.radial_len)
        kw = {} if d3 is None else {"dispersion": (d3.params(), d3.tables(torch.device(DEV)))}
        _cache[("engine", key)] = Engine(consts, nets, nbr_cap=128, cuda_graph=False, pairs=[p.params() for p in pairs],
                                         **kw)
    return _cache[("engine", key)]


def volumes(s: Sys) -> np.ndarray:
    cells = s.cell.view(-1, 3, 3)
    return np.array([abs(float(torch.det(cells[min(c, cells.shape[0] - 1)]))) for c in range(s.species.shape[0])])


def check_pair(group: str, tag: str, got, ref, e_rtol=E_RTOL, f_rtol=F_RTOL, sum_rtol=1e-6, s_rtol=1e-5) -> None:
    close(group, f"{tag} atomic", got["atomic"], ref["atomic"], e_rtol, E_ATOL)
    close(group, f"{tag} forces", got["forces"], ref["forces"], f_rtol, F_ATOL)
    close(group, f"{tag} energy", got["energy"], ref["energy"], sum_rtol, 1e-5)
    for m in range(got["member_atomic"].shape[0]):      # every member gets the pair term
        assert np.array_equal(got["member_atomic"][m], got["atomic"]), tag
    if "stress" in ref:
        close(group, f"{tag} stress", got["stress"], ref["stress"], s_rtol, 1e-5 * float(np.abs(ref["stress"]).max()))


def check_d3(group: str, tag: str, got, ref, atomic_rtol: float = 1e-5) -> None:
    """td3.check_bars / td3.check_stress, with the worst ratio noted."""
    close(group, f"{tag} energy", got["energy"], ref["energy"], 1e-5, 0.0)
    close(group, f"{tag} atomic", got["atomic"], ref["atomic"], atomic_rtol, 1e-9)
    close(group, f"{tag} forces", got["forces"], ref["forces"], 0.0, 1e-4 * float(np.abs(ref["forces"]).max()) + 1e-8)
    for m in range(got["member_atomic"].shape[0]):
        assert np.array_equal(got["member_atomic"][m], got["atomic"]), tag
    if "stress" in ref:
        for c in range(ref["stress"].shape[0]):
            close(group, f"{tag} stress", got["stress"][c], ref["stress"][c], 0.0,
                  1e-4 * float(np.abs(ref["stress"][c]).max()))


def run_term(kind: str, eng, s: Sys) -> tp.Dict[str, np.ndarray]:
    want_virial = s.cell is not None
    fn = tpp.pair_only if kind == "pair" else td3.d3_only
    got = fn(eng, s.species, s.coords, s.cell, s.pbc, want_virial=want_virial)
    if want_virial:
        got["stress"] = got["virial"] / volumes(s).reshape(-1, 1, 1)
    return got


# ------------------------------------------------------------------------------------------------------------------
# host-only: every case reaches its branch
# ------------------------------------------------------------------------------------------------------------------
PAIR_SYSTEMS = ["water999_pbc_ani2x", "1c17_chunk_hcnos_ani2x", "randbatch_ani2x", "6w8h_triclinic_ani2x", "mode2",
                "mode3"]
BELOW_RCR = [("xtb", 3.2, "smooth"), ("zbl", 2.0, "cosine")]


def test_pair_systems_hold_pairs_between_the_cutoff_and_rcr():
    for name in PAIR_SYSTEMS:
        s = pair_sys(name)
        for c in range(s.species.shape[0]):
            ck = None if s.cell is None else (s.cell[c] if s.cell.dim() == 3 else s.cell)
            nb = orc.neighborlist("cell_list", RCR, s.species[c:c + 1], s.coords[c:c + 1], ck,
                                  None if ck is None else s.pbc)
            d = nb.distances
            for _, cutoff, _ in BELOW_RCR:
                assert bool(((d > cutoff) & (d <= RCR)).any()), (name, c, cutoff)
                assert bool((d <= cutoff).any()) or s.species.shape[0] > 1, (name, cutoff)


def test_custom_pair_parameters_reach_their_branches():
    for S in (1, 4, 7, 8):
        k = xtb_custom(S).k_rep_ab
        assert not bool(((k == 1.0) | (k == 1.5)).any()), S           # every pair on the powf path
        assert {round(float(v), 6) for v in k.unique()} == ({1.3, 0.8} if "H" in SYMS[S] else {1.3})
        z = zbl_custom(S)
        assert abs(sum(z._coeffs.view(-1).tolist()) - 1.0) < 1e-6 and z._k != 0.8853 and z._kz != 0.23
    assert xtb_custom(4).params().num_species == 4 and d3_term(8, 8.0).params().num_species == 8


def test_d3_reaches():
    seen, unequal = set(), False
    for name, cutoff in D3_REACH:
        s = d3_sys(name)
        dims, inv = grid_dims(s)
        r, raw = reach(dims, inv, cutoff, 0.0, s.cell is not None)
        assert r is not None, name
        seen |= set(r)
        unequal |= len(set(r)) > 1
        if name in ("tightcell_pbc_ani2x", "cube11.01"):       # the largest stencil the image codes allow
            assert r == dims, (name, r, dims)
        if s.cell is None:                                      # open systems: clipped to dims - 1
            assert any(a > b for a, b in zip(raw, r)), (name, raw, r)
    assert {1, 2, 3} <= seen and unequal
    assert grid_dims(d3_sys("water999_pbc_ani2x"))[0] == [4, 4, 4]
    assert grid_dims(d3_sys("dilute"))[0] == [3, 4, 4]          # narrowed by the bucket capacity
    assert [reach(*grid_dims(d3_sys("water999_pbc_ani2x")), c, 0.0, True)[0][0] for c in (4.0, 8.0, 12.0)] == [1, 2, 3]
    s = d3_sys(D3_REFUSED[0])
    assert reach(*grid_dims(s), D3_REFUSED[1], 0.0, True)[0] is None
    for name in ("planar", "linear"):                           # a bounding box 2e-3 A thick
        x = d3_sys(name).coords[0]
        assert int((x.max(0).values - x.min(0).values == 0).sum()) == (1 if name == "planar" else 2)


def test_d3_reach_equal_to_dims_holds_pairs_at_two_images():
    for name, cutoff in (("tightcell_pbc_ani2x", 11.0), ("cube11.01", 11.0)):
        s = d3_sys(name)
        nb = orc.all_pairs(cutoff, s.species, s.coords, s.cell, s.pbc)
        i0, i1 = nb.indices
        key = torch.minimum(i0, i1) * s.species.shape[1] + torch.maximum(i0, i1)
        assert int(key.unique(return_counts=True)[1].max()) >= 2, name


def test_hit_queue_counts():
    s = queue_batch()
    for c, n in enumerate(QUEUE_REAL):
        real = s.species[c] >= 0
        assert int(real.sum()) == n and bool((~real).any())
        x = s.coords[c][real]
        d = (x.unsqueeze(0) - x.unsqueeze(1)).norm(dim=-1)
        hits = (d <= QUEUE_CUTOFF).sum(1) - 1
        assert bool((hits == n - 1).all())                      # 30 .. 96 hits per atom: 0 .. 3 full queues
    assert {n - 1 for n in QUEUE_REAL} >= {30, 31, 32, 63, 64, 96}


def element_pairs(s: Sys, pot) -> tp.Tuple[bool, bool]:
    """(an element pair without a positive C6 reference is listed, a listed pair's C6 exponent is capped at e^80) from
    the oracle's float64 coordination numbers."""
    spec = d3_spec(pot)
    nb = orc.cell_list(pot.cutoff, s.species, s.coords, s.cell, s.pbc)
    cn = d3o.coordnums(spec, s.species, nb)
    s12 = s.species.reshape(-1)[nb.indices]
    c6 = spec.coeff6[s12[0], s12[1]].flatten(1, 2)
    g = (cn[nb.indices[0]].view(-1, 1) - spec.coordnums_a[s12[0], s12[1]].flatten(1, 2)) ** 2 + \
        (cn[nb.indices[1]].view(-1, 1) - spec.coordnums_b[s12[0], s12[1]].flatten(1, 2)) ** 2
    gmin = torch.where(c6 > 0, g, torch.full_like(g, math.inf)).min(1).values
    none = ~(c6 > 0).any(1)
    capped = (d3o.K3 * gmin + LN_EPS > 80) & ~none
    return bool(none.any()), bool(capped.any())


def test_element_count_cases():
    for S in (1, 4, 8):
        s = d3_sys(f"box_s{S}")
        assert set(s.species.unique().tolist()) == set(range(S))
        dims, inv = grid_dims(s)
        assert reach(dims, inv, 8.0, 0.0, True)[0] is not None
        pot = d3_term(S, 8.0)
        assert pot.tables(torch.device("cpu")).shape == (S, S, 25, 4)
        none, capped = element_pairs(s, pot)
        assert none == (S in (4, 8)), S          # S-F
        assert capped == (S == 8), S


# ------------------------------------------------------------------------------------------------------------------
# GPU: the pair kernel in the fused step
# ------------------------------------------------------------------------------------------------------------------
def pair_bars(name: str) -> tp.Dict[str, float]:
    # 6W8H: the bars of test_gpu_pair_potentials.test_kernel_vs_float64_golden (overlapping atoms, measured there)
    return dict(e_rtol=4e-5, f_rtol=5e-4, sum_rtol=1e-5) if name.startswith("6w8h") else {}


@pytest.mark.gpu
@pytest.mark.parametrize("kind,cutoff,fn", BELOW_RCR, ids=[f"{k}{c}" for k, c, _ in BELOW_RCR])
@pytest.mark.parametrize("name", PAIR_SYSTEMS)
def test_pair_cutoff_below_rcr(name, kind, cutoff, fn):
    pot = tpp.potential(kind, fn, cutoff)
    s = pair_sys(name)
    got = run_term("pair", engine(f"7-{kind}-{cutoff}", 7, [pot]), s)
    ref = oracle([(porc, pair_spec(pot))], s, stress=s.cell is not None)
    check_pair("pair below Rcr", f"{name} {kind} {cutoff}", got, ref, **pair_bars(name))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["water999_pbc_ani2x", "randbatch_ani2x"])
def test_pair_custom_parameters(name):
    """xTB with k_rep 1.3 / 0.8 (powf), ZBL with its own k, exponent, screening constants and effective charges, as
    two terms of one step."""
    pots = [xtb_custom(7), zbl_custom(7, cutoff=4.0)]
    s = golden_sys(name)
    eng = engine("7-custom", 7, pots)
    got = run_term("pair", eng, s)
    ref = oracle([(porc, pair_spec(p)) for p in pots], s, stress=s.cell is not None)
    check_pair("pair custom", name, got, ref)
    for p in pots:       # and each alone
        one = run_term("pair", engine(f"7-custom-{p.kind}", 7, [p]), s)
        check_pair("pair custom", f"{name} kind {p.kind}", one, oracle([(porc, pair_spec(p))], s, stress=s.cell is not None))


def two_term_model():
    from torchani_b200 import models
    if "two" not in _cache:
        w32 = [{k: [(w.float(), b.float()) for w, b in layers] for k, layers in wm.items()} for wm in tpp.oracle_weights()]
        base = models.from_weight_lists("2x", w32, periodic_table_index=False)
        pots = {"repulsion_xtb": tpp.potential("xtb", "smooth"), "repulsion_zbl": tpp.potential("zbl", "cosine", 3.0)}
        _cache["two"] = models.ANI(base.symbols, base.aev_computer, base.neural_networks, base.energy_shifter, False,
                                   pots).to(DEV)
    return _cache["two"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["water999_pbc_ani2x", "randbatch_ani2x"])
def test_two_pair_terms_in_one_model(name):
    m2, m0 = two_term_model(), tpp.model(None)
    pots = list(m2.potentials.values())
    s = golden_sys(name)
    ref = oracle([(porc, pair_spec(p)) for p in pots], s, stress=s.cell is not None)
    eng2, eng0 = m2.engine(torch.device(DEV)), m0.engine(torch.device(DEV))
    check_pair("two pair terms", name, run_term("pair", eng2, s), ref)
    # one launch per term
    args = (s.species.to(DEV), s.coords.float().to(DEV), None if s.cell is None else s.cell.float().to(DEV),
            s.cell is not None)
    eng2.step(*args, check=True)
    eng0.step(*args, check=True)
    assert len(eng2.pairs) == 2 and eng2.launches_per_step == eng0.launches_per_step + 2
    # every member of the query-by-committee step gets both terms
    x = ((s.species.to(DEV), s.coords.float().to(DEV)), None if s.cell is None else s.cell.float().to(DEV),
         None if s.pbc is None else s.pbc.to(DEV))
    _, _, f2 = m2.members_forces(*x)
    _, _, f0 = m0.members_forces(*x)
    assert f2.shape[0] == 8
    close("two pair terms", f"{name} member forces", (f2 - f0).cpu().numpy(),
          np.broadcast_to(ref["forces"], f2.shape), F_RTOL, F_ATOL)


# ------------------------------------------------------------------------------------------------------------------
# GPU: D3 in the fused step
# ------------------------------------------------------------------------------------------------------------------
def device_reach(eng, s: Sys, cutoff: float) -> tp.List[int]:
    g = eng.grid_info(eng.workspace(*s.species.shape))
    dims = list(g.dims)
    inv = np.array(list(g.inv), dtype=np.float32).reshape(3, 3)
    assert dims == grid_dims(s, RCR + eng.skin)[0], dims
    return reach(dims, inv, cutoff, eng.skin, bool(g.pbc))[0]


@pytest.mark.gpu
@pytest.mark.parametrize("name,cutoff", D3_REACH, ids=[f"{n.split('_')[0]}-{c}" for n, c in D3_REACH])
def test_d3_reach(name, cutoff):
    pot = d3_term(7, cutoff)
    s = d3_sys(name)
    eng = engine(f"7-d3-{cutoff}", 7, d3=pot)
    got = run_term("d3", eng, s)
    r = device_reach(eng, s, cutoff)
    dims, inv = grid_dims(s)
    assert r == reach(dims, inv, cutoff, 0.0, s.cell is not None)[0]
    ref = oracle([(d3o, d3_spec(pot))], s, stress=s.cell is not None)
    check_d3(f"d3 reach {max(r)}", f"{name} {cutoff}", got, ref)


@pytest.mark.gpu
def test_d3_cell_thinner_than_the_cutoff_is_refused():
    name, cutoff = D3_REFUSED
    s = d3_sys(name)
    eng = engine(f"7-d3-{cutoff}", 7, d3=d3_term(7, cutoff))
    with pytest.raises(RuntimeError, match="Cell is too small"):
        td3.d3_only(eng, s.species, s.coords, s.cell, s.pbc, want_virial=True)
    ws = eng.workspace(*s.species.shape)
    assert not bool(ws.atomic.any()) and not bool(ws.energies.any()) and not bool(ws.grad.any())
    assert not bool(ws.member_atomic.any()) and not bool(ws.virial.any())
    assert int(ws.status.item()) == 0      # raised once, then cleared


@pytest.mark.gpu
def test_d3_hit_queue_beyond_32_hits():
    pot = d3_term(7, QUEUE_CUTOFF)
    s = queue_batch()
    got = run_term("d3", engine(f"7-d3-{QUEUE_CUTOFF}", 7, d3=pot), s)
    check_d3("d3 hit queue", "queue", got, oracle([(d3o, d3_spec(pot))], s))
    assert not bool(got["atomic"][s.species.numpy() < 0].any())


@pytest.mark.gpu
@pytest.mark.parametrize("S", [1, 4, 8])
def test_element_counts(S):
    """D3 and both pair terms on engines of S elements; the D3 tables of S = 4 and 8 hold the S-F pair without a C6
    reference, those of S = 8 a Br whose C6 exponents all reach the cap."""
    s = d3_sys(f"box_s{S}")
    d3 = d3_term(S, 8.0)
    got = run_term("d3", engine(f"{S}-d3", S, d3=d3), s)
    check_d3(f"elements S={S}", f"S={S} d3", got, oracle([(d3o, d3_spec(d3))], s, stress=True))
    pots = [xtb_custom(S), zbl_custom(S, cutoff=3.0)]
    got = run_term("pair", engine(f"{S}-pairs", S, pots), s)
    check_pair(f"elements S={S}", f"S={S} pairs", got, oracle([(porc, pair_spec(p)) for p in pots], s, stress=True))


# ------------------------------------------------------------------------------------------------------------------
# GPU: a Verlet skin, partial PBC (the public model API)
# ------------------------------------------------------------------------------------------------------------------
def terms_oracle(co: torch.Tensor, sp: torch.Tensor, cell: torch.Tensor, pbc: torch.Tensor, nl: str):
    xtb = tpp.spec("xtb", "smooth")
    d3 = td3.spec()
    s = Sys(sp, co, cell, pbc)
    return oracle([(porc, xtb), (d3o, d3)], s, nl=nl), oracle([(d3o, d3)], s, nl=nl)


@pytest.mark.gpu
def test_verlet_skin_against_float64():
    from torchani_b200.calculator import HostCalculator
    m1, m0 = td3.model(xtb="smooth", tag="skin-terms"), td3.model(d3=False)
    s = golden_sys("water999_pbc_ani2x")
    eng = m1.engine(torch.device(DEV))
    calc = HostCalculator(m1, s.species[0].numpy(), s.cell.float().numpy(), pbc=True, skin=0.4)
    try:
        g = torch.Generator().manual_seed(8)
        pos = s.coords.float()
        for step in range(6):
            pos = pos + 0.002 * torch.randn(pos.shape, generator=g)
            if step == 3:
                pos[0, 11] += 0.3      # beyond skin / 2: rebuilt
            e1, f1 = calc.calculate(pos[0].numpy())
            if step == 0:
                assert eng.skin == 0.4
                r = device_reach(eng, s, 8.0)
                assert r == [2, 2, 2], r
            e0, f0 = m0.energies_and_forces(s.species.to(DEV), pos.to(DEV), s.cell.float().to(DEV), PBC3.to(DEV))
            ref, ref_d3 = terms_oracle(f32(td3.wrapped(pos.double(), s.cell)), s.species, s.cell, PBC3, "cell_list")
            close("verlet skin", f"step {step} energy", e1 - float(e0[0]), ref["energy"][0], 1e-5,
                  1e-5 * abs(float(ref_d3["energy"][0])) + 1e-5)
            close("verlet skin", f"step {step} forces", f1 - f0[0].cpu().numpy(), ref["forces"][0], F_RTOL,
                  F_ATOL + 1e-4 * float(np.abs(ref_d3["forces"]).max()))
        assert 1 <= calc.rebuilds < 6, calc.rebuilds
    finally:
        eng.skin = 0.0


@pytest.mark.gpu
@pytest.mark.parametrize("flags", [(True, True, False), (False, True, False)], ids=["TTF", "FTF"])
def test_partial_pbc(flags):
    m1, m0 = td3.model(xtb="smooth"), td3.model(d3=False)
    sp, co, cell, _ = golden_inputs(load_golden("tightcell_pbc_ani2x"))
    co, cell = f32(co), f32(cell)
    pbc = torch.tensor(flags)
    args = (sp.to(DEV), co.float().to(DEV), cell.float().to(DEV), pbc.to(DEV))
    e1, f1 = m1.energies_and_forces(*args)
    e0, f0 = m0.energies_and_forces(*args)
    ref, ref_d3 = terms_oracle(co, sp, cell, pbc, "all_pairs")
    close("partial pbc", f"{flags} energy", float(e1[0]) - float(e0[0]), ref["energy"][0], 1e-5,
          1e-5 * abs(float(ref_d3["energy"][0])) + 1e-5)
    close("partial pbc", f"{flags} forces", (f1 - f0)[0].cpu().numpy(), ref["forces"][0], F_RTOL,
          F_ATOL + 1e-4 * float(np.abs(ref_d3["forces"]).max()))
    # the same geometry fully periodic gives other energies: the flags matter
    full, _ = terms_oracle(co, sp, cell, PBC3, "all_pairs")
    assert abs(float(full["energy"][0]) - float(ref["energy"][0])) > 1e-6


# ------------------------------------------------------------------------------------------------------------------
# GPU: the half-list entry points (compute_from_neighbors)
# ------------------------------------------------------------------------------------------------------------------
def listed(s: Sys, cutoff: float):
    """The oracle's half list (float64, coordinates requiring grad) and the same list as float32 device tensors."""
    from torchani_b200.neighbors import Neighbors
    x = s.coords.clone().requires_grad_(True)
    nl = "all_pairs" if s.cell is None else "cell_list"
    nb = orc.neighborlist(nl, cutoff, s.species, x, s.cell, s.pbc)
    dev_nb = Neighbors(nb.indices.to(DEV), nb.distances.detach().float().to(DEV),
                       nb.diff_vectors.detach().float().to(DEV))
    return x, nb, dev_nb


HALF_TERMS = ["xtb", "zbl", "d3"]


def half_term(kind: str, cutoff: float = RCR):
    if kind == "d3":
        return td3.d3_module("smooth", cutoff).to(DEV), d3o, td3.spec("smooth", cutoff)
    pot = tpp.potential(kind, "smooth" if kind == "xtb" else "cosine", cutoff).to(DEV)
    return pot, porc, pair_spec(pot)


@pytest.mark.gpu
@pytest.mark.parametrize("ghost", [False, True], ids=["plain", "ghost"])
@pytest.mark.parametrize("kind", HALF_TERMS)
@pytest.mark.parametrize("name", ["randbatch_ani2x", "water999_pbc_ani2x"])
def test_half_list_batches_and_images(name, kind, ghost):
    cutoff = 8.0 if kind == "d3" else RCR
    pot, mod, spec = half_term(kind, cutoff)
    s = golden_sys(name)
    x_ref, nb, nb_dev = listed(s, cutoff)
    if s.cell is not None:     # the list holds pairs across images
        assert bool((nb.diff_vectors - (x_ref[0][nb.indices[0]] - x_ref[0][nb.indices[1]])).abs().max() > 1.0)
    gflags = None
    if ghost:
        gflags = torch.zeros_like(s.species, dtype=torch.bool)
        gflags[:, ::4] = True
    C = s.species.shape[0]
    w = torch.linspace(0.5, 2.0, C, dtype=torch.float64)          # upstream weights that differ per conformer
    u = torch.linspace(-1.0, 1.5, C, dtype=torch.float64)
    sp = s.species.to(DEV)
    gd = None if gflags is None else gflags.to(DEV)
    x = s.coords.float().to(DEV).requires_grad_(True)
    e = pot.compute_from_neighbors(sp, x, nb_dev, ghost_flags=gd)
    (g_e,) = torch.autograd.grad((w.float().to(DEV) * e).sum(), x)
    a = pot.compute_from_neighbors(sp, x, nb_dev, atomic=True, ghost_flags=gd)
    (g_a,) = torch.autograd.grad((u.float().to(DEV).view(-1, 1) * a).sum(), x)
    e_ref = mod.energies_from_neighbors(spec, s.species, nb, ghost_flags=gflags)
    (ge_ref,) = torch.autograd.grad((w * e_ref).sum(), x_ref, retain_graph=True)
    a_ref = mod.energies_from_neighbors(spec, s.species, nb, atomic=True, ghost_flags=gflags)
    (ga_ref,) = torch.autograd.grad((u.view(-1, 1) * a_ref).sum(), x_ref)
    tag = f"{name} {kind} {'ghost' if ghost else 'plain'}"
    group = f"half list {kind}"
    if kind == "d3":
        close(group, f"{tag} atomic", a.detach().cpu().numpy(), a_ref.detach().numpy(), 1e-5, 1e-9)
        close(group, f"{tag} energies", e.detach().cpu().numpy(), e_ref.detach().numpy(), 1e-5, 0.0)
        for t, g, r in (("weighted", g_e, ge_ref), ("atomic upstream", g_a, ga_ref)):
            close(group, f"{tag} {t} gradient", g.cpu().numpy(), r.numpy(), 0.0, 1e-4 * float(r.abs().max()) + 1e-8)
    else:
        close(group, f"{tag} atomic", a.detach().cpu().numpy(), a_ref.detach().numpy(), E_RTOL, E_ATOL)
        close(group, f"{tag} energies", e.detach().cpu().numpy(), e_ref.detach().numpy(), 1e-6, 1e-5)
        for t, g, r in (("weighted", g_e, ge_ref), ("atomic upstream", g_a, ga_ref)):
            close(group, f"{tag} {t} gradient", g.cpu().numpy(), r.numpy(), F_RTOL, F_ATOL)
    # an upstream that varies inside a conformer is refused
    a = pot.compute_from_neighbors(sp, x, nb_dev, atomic=True, ghost_flags=gd)
    with pytest.raises(NotImplementedError):
        torch.autograd.grad((a * torch.rand_like(a)).sum(), x)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["xtb", "zbl"])
def test_half_list_without_envelope(kind):
    """cutoff = inf: no envelope, every listed pair counts (pairs out to 7 A here)."""
    pot = tpp.potential(kind, "smooth", math.inf).to(DEV)
    assert pot.cutoff_fn == "dummy" and pot.params().cutoff_fn == 2
    spec = pair_spec(pot)
    s = golden_sys("randbatch_ani2x")
    x_ref, nb, nb_dev = listed(s, 7.0)
    assert bool((nb.distances > RCR).any())
    x = s.coords.float().to(DEV).requires_grad_(True)
    a = pot.compute_from_neighbors(s.species.to(DEV), x, nb_dev, atomic=True)
    (g,) = torch.autograd.grad(a.sum(), x)
    a_ref = porc.energies_from_neighbors(spec, s.species, nb, atomic=True)
    (g_ref,) = torch.autograd.grad(a_ref.sum(), x_ref)
    close("half list no envelope", f"{kind} atomic", a.detach().cpu().numpy(), a_ref.detach().numpy(), E_RTOL, E_ATOL)
    close("half list no envelope", f"{kind} gradient", g.cpu().numpy(), g_ref.numpy(), F_RTOL, F_ATOL)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", HALF_TERMS)
def test_half_list_empty(kind):
    from torchani_b200.neighbors import Neighbors
    pot, _, _ = half_term(kind, 8.0 if kind == "d3" else RCR)
    s = golden_sys("randbatch_ani2x")
    nb = Neighbors(torch.zeros(2, 0, dtype=torch.long, device=DEV), torch.zeros(0, device=DEV),
                   torch.zeros(0, 3, device=DEV))
    x = s.coords.float().to(DEV).requires_grad_(True)
    e = pot.compute_from_neighbors(s.species.to(DEV), x, nb)
    (g,) = torch.autograd.grad(e.sum(), x)
    a = pot.compute_from_neighbors(s.species.to(DEV), x.detach(), nb, atomic=True)
    assert e.shape == (s.species.shape[0],) and not bool(e.any()) and not bool(a.any()) and not bool(g.any())
