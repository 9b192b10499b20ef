"""Kernel-level parity of the analytic Hessian stages (csrc/hessian.cu) against float64.

The four C-ABI entry points are called directly on inputs this file crafts inside their contract (include/ani_b200.h
section 9): sorted positions with the element in the fourth word, neighbour words that point at real atoms only,
``nbr_cnt <= cap``, and chunks laid out by ``engine._hessian_chunks``.  Every slot of every chunk is compared.

References.  ``hessian_oracle.center_aev`` / ``center_pair_energy`` give one atom's AEV and pair energy in float64 as
functions of its neighbour vectors; ``torch.func.jacrev`` of them is the reference of the Jacobian rows, of the
geometric blocks (the Hessian of g . A with g held fixed) and of the xTB / ZBL blocks.  The network blocks are
sum_m scale_m R H_m R^T with H_m the double-backward Hessian of member m's network at the kernel's own AEV row (read back
with ``untile_a_operand``), in float64.  The assembly is restated in numpy float64 as H += T^T B T with T the map from
the atom coordinates to the neighbour vectors r_n - r_i.  The references use the kernel's float32 cutoffs.

Bars.  As in test_gpu_hessians.py: 8 x the float32-vs-float64 spread of the same reference (the network stage: of the
float32 reference network on the same rows), plus 2e-6 x max |ref|.  The assembly sums float32 blocks in float64: 1e-12
relative.  Exact: the Jacobian's padding columns, the column blocks a neighbour cannot touch and the padding rows are
zero; block storage past the chunk's ``block_floats`` keeps its sentinel; the network and geometric stages add to what
``blocks`` holds.  The module prints the worst error / bar of each group at its end (pytest -s).

Measured on an H100 80GB HBM3 (power limit not recorded), worst error / bar: Jacobian rows 0.38, network 0.71,
geometric 0.24, pair terms 0.15, cutoff edges 0.19, dense neighbourhood 0.12, end to end 0.20; the assembly's error is
below 1e-3 of its bar.
"""
import ctypes as C
import math
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
ASSEMBLY_BAR = 1e-12
SENTINEL = 7.25
MAX_ANG = 96   # ANI_MAX_ANG

_WORST: tp.Dict[str, float] = {}


def _note(group: str, ratio: float) -> None:
    _WORST[group] = max(_WORST.get(group, 0.0), ratio)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if _WORST:
        print("\nworst error / bar of test_gpu_hessian_kernels.py:")
        for k in sorted(_WORST):
            print(f"  {k:28s} {_WORST[k]:.3f}")


def check_bar(group: str, got: torch.Tensor, ref: torch.Tensor, ref32: torch.Tensor, what: str = "") -> None:
    """got within SPREAD_FACTOR x |ref32 - ref| + FLOOR x max |ref| of ref (all finite)."""
    assert bool(torch.isfinite(got).all()), f"{group} {what}: non-finite values"
    b = SPREAD_FACTOR * float((ref32.double() - ref).abs().max()) + FLOOR * float(ref.abs().max())
    err = float((got.double() - ref).abs().max())
    _note(group, err / b if b > 0 else (0.0 if err == 0 else math.inf))
    assert err <= b, f"{group} {what}: max |d| {err:.3e} > bar {b:.3e} (max |ref| {float(ref.abs().max()):.3e})"


def f32(v: float) -> float:
    return float(np.float32(v))


def lib(variant: str = ""):
    from torchani_b200 import _lib
    return _lib.lib(variant)


def ptr(t):
    from torchani_b200._lib import ptr as p
    return p(t)


def stream() -> int:
    return torch.cuda.current_stream(DEV).cuda_stream


# ------------------------------------------------------------------------------------------------------------------
# AEV constants
# ------------------------------------------------------------------------------------------------------------------
def _specs() -> tp.Dict[str, orc.AEVSpec]:
    from test_gpu_aev import CONFIGS, spec_of
    out = {"1x": orc.aev_spec_1x(), "2x": orc.aev_spec_2x(), "gelu": gor.gelu_spec()}
    out.update({c.name: spec_of(c) for c in CONFIGS if len(spec_of(c).shf_a) * len(spec_of(c).shf_z) == 32})
    return out


SPECS = _specs()


def kernel_spec(spec: orc.AEVSpec) -> orc.AEVSpec:
    """The oracle spec with the kernel's float32 cutoffs (the other constants are float32-rounded by the oracle)."""
    return spec._replace(rcr=f32(spec.rcr), rca=f32(spec.rca))


def aev_params(spec: orc.AEVSpec):
    """(ani_aev_params, ang_pad, ldx) with PackedNetworks' rule for the angular block's alignment."""
    from torchani_b200.engine import AEVConstants
    p = AEVConstants(*spec).to_struct()
    ldx = (spec.out_dim + 31) // 32 * 32
    pad = (-spec.radial_len) % 32 if 0 < spec.radial_len < spec.out_dim else 0
    if spec.out_dim + pad > ldx:
        pad = 0
    p.ang_pad = pad
    return p, pad, ldx


def internal_cols(spec: orc.AEVSpec, pad: int) -> torch.Tensor:
    c = torch.arange(spec.out_dim)
    return torch.where(c < spec.radial_len, c, c + pad)


# ------------------------------------------------------------------------------------------------------------------
# crafted systems and chunks
# ------------------------------------------------------------------------------------------------------------------
class System(tp.NamedTuple):
    coords: np.ndarray            # (N, 3) float32
    species: np.ndarray           # (N,) element index
    words: tp.List[tp.List[int]]  # neighbour words (atom indices) of every atom; only the slots' are read
    slots: tp.List[int]           # the central atoms of the chunks


def ball(n: int, lo: float, hi: float, rng, min_dist: float, existing: np.ndarray) -> np.ndarray:
    """n points with lo <= |p| <= hi, at least min_dist from each other and from ``existing``."""
    pts = existing
    while len(pts) < len(existing) + n:
        p = rng.uniform(-hi, hi, 3)
        r = np.linalg.norm(p)
        if lo <= r <= hi and (len(pts) == 0 or np.linalg.norm(pts - p, axis=1).min() >= min_dist):
            pts = np.vstack([pts, p])
    return pts[len(existing):]


def words_within(coords: np.ndarray, rcr: float, rng, slots=None) -> tp.List[tp.List[int]]:
    """Every atom's neighbours within rcr (float64 distances of the float32 coordinates), in a shuffled order."""
    x = coords.astype(np.float64)
    out = []
    for i in range(len(x)):
        if slots is not None and i not in slots:
            out.append([])
            continue
        d = np.linalg.norm(x - x[i], axis=1)
        out.append([int(j) for j in rng.permutation(len(x)) if j != i and d[j] <= rcr])
    return out


def random_system(spec: orc.AEVSpec, n: int, seed: int, radius: float = 3.4) -> System:
    """A cluster of n atoms plus an isolated atom and a pair (0 and 1 neighbours, no angular pairs)."""
    rng = np.random.default_rng(seed)
    pts = ball(n, 0.0, radius, rng, 0.95, np.zeros((0, 3)))
    far = np.array([[40.0, 0.0, 0.0], [0.0, 40.0, 0.0], [0.0, 41.1, 0.0]])
    x = np.vstack([pts, far]).astype(np.float32)
    sp = rng.integers(0, spec.num_species, len(x))
    rcr = f32(spec.rcr)
    words = words_within(x, rcr, rng)
    # no pair within 1e-5 A of Rca: float32 and float64 distances then agree on the angular rule
    d = np.linalg.norm(x[:, None].astype(np.float64) - x[None].astype(np.float64), axis=-1)
    assert not np.any(np.abs(d - f32(spec.rca)) < 1e-5) and not np.any(np.abs(d - rcr) < 1e-5)
    return System(x, sp, words, list(range(len(x))))


class Device(tp.NamedTuple):
    spos: torch.Tensor
    cnt: torch.Tensor
    nbr: torch.Tensor
    cap: int


def to_device(sysm: System, cap: int) -> Device:
    N = len(sysm.species)
    spos = torch.zeros(N, 4, dtype=torch.float32)
    spos[:, :3] = torch.from_numpy(sysm.coords.astype(np.float32))
    spos[:, 3] = torch.from_numpy(sysm.species.astype(np.int32)).view(torch.float32)
    cnt = np.array([len(w) for w in sysm.words], dtype=np.int32)
    assert cnt.max() <= cap
    nbr = np.zeros((N, cap), dtype=np.int32)
    for i, w in enumerate(sysm.words):
        nbr[i, :len(w)] = w
    return Device(spos.to(DEV), torch.from_numpy(cnt).to(DEV), torch.from_numpy(nbr).view(-1).to(DEV), cap)


def plans(sysm: System, budget: int):
    """The chunks of the slots (engine._hessian_chunks over the slots' counts and elements)."""
    from torchani_b200.engine import _hessian_chunks
    slots = np.asarray(sysm.slots)
    cnt = np.array([len(sysm.words[i]) for i in slots], dtype=np.int64)
    out = [p._replace(atom=slots[p.atom].astype(np.int32)) for p in _hessian_chunks(cnt, sysm.species[slots], budget)]
    assert sorted(int(a) for p in out for a in p.atom) == sorted(sysm.slots)
    return out


def chunk_args(plan):
    from torchani_b200 import _lib
    i32 = torch.from_numpy(np.concatenate([plan.atom, plan.row_off, plan.row_slot, plan.tile_species])).to(DEV)
    b_off = torch.from_numpy(plan.block_off).to(DEV)
    ns, rows = len(plan.atom), plan.rows
    ch = _lib.HessianChunk()
    ch.atom, ch.row_off = i32.data_ptr(), i32.data_ptr() + 4 * ns
    ch.row_slot, ch.tile_species = i32.data_ptr() + 8 * ns, i32.data_ptr() + 4 * (2 * ns + rows)
    ch.block_off = b_off.data_ptr()
    ch.n_slots, ch.rows, ch.max_count = ns, rows, plan.max_count
    return ch, (i32, b_off)


def prefilled_blocks(plan, seed: int, tail: int = 64) -> tp.Tuple[torch.Tensor, torch.Tensor]:
    """Random block storage of the chunk and SENTINEL past block_floats: (device buffer, host copy of the start)."""
    g = torch.Generator().manual_seed(seed)
    host = torch.cat([torch.randn(plan.block_floats, generator=g) * 1e-3, torch.full((tail,), SENTINEL)])
    return host.to(DEV), host


def block_of(buf: torch.Tensor, plan, k: int, n: int) -> torch.Tensor:
    o = int(plan.block_off[k])
    return buf[o:o + 9 * n * n].view(3 * n, 3 * n).double().cpu()


def check_tail(buf: torch.Tensor, plan) -> None:
    assert bool((buf[plan.block_floats:].cpu() == SENTINEL).all()), "block storage past block_floats was written"


def vectors(sysm: System, i: int, dtype=torch.float64) -> torch.Tensor:
    x = torch.from_numpy(sysm.coords.astype(np.float32)).to(dtype)
    return x[sysm.words[i]] - x[i]


# ------------------------------------------------------------------------------------------------------------------
# A. Jacobian rows
# ------------------------------------------------------------------------------------------------------------------
def jacobian_ref(spec: orc.AEVSpec, sysm: System, i: int, dtype=torch.float64) -> torch.Tensor:
    """(3 n, out_dim) dA_i / d(r_n)_c in the reference column order."""
    sn = [int(sysm.species[j]) for j in sysm.words[i]]
    v = vectors(sysm, i, dtype)
    jac = torch.func.jacrev(lambda y: hor.center_aev(spec, int(sysm.species[i]), sn, y), chunk_size=128)(v)   # (D, n, 3)
    return jac.reshape(jac.shape[0], -1).t()


def reachable(spec: orc.AEVSpec, pad: int, ldx: int, sysm: System, i: int) -> torch.Tensor:
    """(3 n, ldx) bool: the internal columns row 3 n + c may hold (the radial block of s_n; the pair blocks (s_n, s_k)
    of n's angular partners k if n itself is within Rca)."""
    nr, S, RL = len(spec.shf_r), spec.num_species, spec.radial_len
    tri = orc.triu_index(S)
    d = np.linalg.norm(vectors(sysm, i).numpy(), axis=1)
    ang = d <= f32(spec.rca)
    sn = [int(sysm.species[j]) for j in sysm.words[i]]
    out = torch.zeros(3 * len(sn), ldx, dtype=torch.bool)
    for n, s in enumerate(sn):
        out[3 * n:3 * n + 3, s * nr:(s + 1) * nr] = True
        if ang[n]:
            for k in range(len(sn)):
                if k != n and ang[k]:
                    c0 = RL + pad + int(tri[s, sn[k]]) * 32
                    out[3 * n:3 * n + 3, c0:c0 + 32] = True
    return out


def run_jacobian(spec: orc.AEVSpec, sysm: System, cap: int, budget: int) -> None:
    p, pad, ldx = aev_params(spec)
    ks = kernel_spec(spec)
    cols = internal_cols(spec, pad)
    dv = to_device(sysm, cap)
    L = lib()
    for plan in plans(sysm, budget):
        ch, _keep = chunk_args(plan)
        jac = torch.full((plan.rows, ldx), float("nan"), device=DEV)   # the stage zeroes the chunk's rows first
        assert L.ani_b200_hessian_jacobian(C.byref(p), ptr(dv.spos), ptr(dv.cnt), ptr(dv.nbr), cap, C.byref(ch),
                                           ptr(jac), ldx, stream()) == 0
        torch.cuda.synchronize()
        jac = jac.cpu()
        assert float(jac[torch.from_numpy(plan.row_slot) < 0].abs().sum()) == 0.0, "padding rows"
        for k, i in enumerate(plan.atom.tolist()):
            n = len(sysm.words[i])
            if n == 0:
                continue
            rows = jac[int(plan.row_off[k]):int(plan.row_off[k]) + 3 * n].double()
            assert float(rows[~reachable(spec, pad, ldx, sysm, i)].abs().sum()) == 0.0, f"atom {i}: unreachable column"
            ref = jacobian_ref(ks, sysm, i)
            ref32 = jacobian_ref(ks, sysm, i, torch.float32)
            check_bar("jacobian", rows[:, cols], ref, ref32, f"atom {i}")


@pytest.mark.parametrize("name", list(SPECS))
def test_jacobian_rows(name):
    spec = SPECS[name]
    sysm = random_system(spec, 16, 100 + len(name), 3.0)
    run_jacobian(spec, sysm, 64, 128)   # several chunks


# ------------------------------------------------------------------------------------------------------------------
# C. geometric term: dE/dAEV rows and the xTB / ZBL pair terms
# ------------------------------------------------------------------------------------------------------------------
def geometric_ref(spec: orc.AEVSpec, sysm: System, i: int, g: torch.Tensor, dtype=torch.float64) -> torch.Tensor:
    sn = [int(sysm.species[j]) for j in sysm.words[i]]
    v = vectors(sysm, i, dtype)
    gg = g.to(dtype)
    h = torch.func.jacrev(torch.func.jacrev(lambda y: (gg * hor.center_aev(spec, int(sysm.species[i]), sn, y)).sum()),
                          chunk_size=96)(v)
    return h.reshape(3 * len(sn), 3 * len(sn))


def pair_ref(pair: porc.PairSpec, sysm: System, i: int, dtype=torch.float64) -> torch.Tensor:
    sn = [int(sysm.species[j]) for j in sysm.words[i]]
    v = vectors(sysm, i, dtype)
    h = torch.func.jacrev(torch.func.jacrev(lambda y: hor.center_pair_energy(pair, int(sysm.species[i]), sn, y)))(v)
    return h.reshape(3 * len(sn), 3 * len(sn))


def xtb_tables():
    z = np.load(os.path.join(GOLD, "pair_params.npz"))
    return tuple(torch.tensor(z[k]) for k in ("y_ab", "sqrt_alpha_ab", "k_rep_ab"))


def pair_terms(kind: str, cutoff: float, fn: str):
    """(device ani_pair_params, oracle PairSpec at the kernel's float32 cutoff) of xTB / ZBL over the 7 ANI-2x
    elements."""
    from torchani_b200 import potentials as P
    if kind == "xtb":
        p = P.RepulsionXTB(orc.SYMBOLS_2X, alpha=[1.0] * 7, yeff=[1.0] * 7, cutoff=cutoff, cutoff_fn=fn)
        for k, t in zip(("y_ab", "sqrt_alpha_ab", "k_rep_ab"), xtb_tables()):
            getattr(p, k).copy_(t.float())
        spec = porc.PairSpec("xtb", f32(cutoff), fn, tuple(t.float().double() for t in xtb_tables()))
    else:
        p = P.RepulsionZBL(orc.SYMBOLS_2X, cutoff=cutoff, cutoff_fn=fn)
        spec = porc.zbl_spec(orc.SYMBOLS_2X, f32(cutoff), fn)
    dev = torch.frombuffer(bytearray(bytes(p.params())), dtype=torch.uint8).to(DEV)
    return dev, spec


def run_geometric(spec: orc.AEVSpec, sysm: System, cap: int, budget: int, pair=None, seed: int = 0,
                  group: str = "geometric") -> None:
    """The g branch (pair None: random dE/dAEV rows of both signs, NaN in the columns it must not read) or one pair
    term, on pre-filled blocks."""
    p, pad, ldx = aev_params(spec)
    ks = kernel_spec(spec)
    cols = internal_cols(spec, pad)
    dv = to_device(sysm, cap)
    N = len(sysm.species)
    gen = torch.Generator().manual_seed(seed)
    g = torch.full((N, ldx), float("nan"))
    g[:, cols] = torch.randn(N, spec.out_dim, generator=gen) * 0.05
    row_of = torch.from_numpy(np.random.default_rng(seed).permutation(N).astype(np.int32))   # any row per atom
    gd, rd = g.to(DEV), row_of.to(DEV)
    L = lib()
    for c, plan in enumerate(plans(sysm, budget)):
        ch, _keep = chunk_args(plan)
        blocks, before = prefilled_blocks(plan, seed + c)
        if pair is None:
            rc = L.ani_b200_hessian_geometric(C.byref(p), ptr(dv.spos), ptr(dv.cnt), ptr(dv.nbr), cap, ptr(rd), ptr(gd),
                                              ldx, None, C.byref(ch), ptr(blocks), stream())
        else:
            rc = L.ani_b200_hessian_geometric(C.byref(p), ptr(dv.spos), ptr(dv.cnt), ptr(dv.nbr), cap, None, None, 0,
                                              ptr(pair[0]), C.byref(ch), ptr(blocks), stream())
        assert rc == 0
        torch.cuda.synchronize()
        check_tail(blocks, plan)
        for k, i in enumerate(plan.atom.tolist()):
            n = len(sysm.words[i])
            if n == 0:
                continue
            got = block_of(blocks, plan, k, n) - block_of(before, plan, k, n)
            if pair is None:
                gi = g[int(row_of[i])][cols].double()
                ref, ref32 = geometric_ref(ks, sysm, i, gi), geometric_ref(ks, sysm, i, gi, torch.float32)
            else:
                ref, ref32 = pair_ref(pair[1], sysm, i), pair_ref(pair[1], sysm, i, torch.float32)
            check_bar(group, got, ref, ref32, f"atom {i}")


@pytest.mark.parametrize("name", list(SPECS))
def test_geometric_blocks(name):
    spec = SPECS[name]
    run_geometric(spec, random_system(spec, 16, 200 + len(name), 3.0), 64, 128, seed=len(name))


@pytest.mark.parametrize("kind", ["xtb", "zbl"])
@pytest.mark.parametrize("fn", ["cosine", "smooth"])
@pytest.mark.parametrize("cutoff", [3.0, 4.6, 5.1])
def test_pair_blocks(kind, fn, cutoff):
    spec = orc.aev_spec_2x()
    run_geometric(spec, random_system(spec, 14, 300, 3.0), 64, 128, pair_terms(kind, cutoff, fn), group="pair")


def edge_system(spec: orc.AEVSpec, cut: float) -> System:
    """A centre at the origin with neighbours on the axes at exactly Rca, Rcr and ``cut`` and one float32 ulp beyond
    Rca and ``cut`` (on an axis the float32 distance is exact), plus two angular partners."""
    up = lambda v: float(np.nextafter(np.float32(v), np.float32(np.inf)))  # noqa: E731
    rca, rcr, cut = f32(spec.rca), f32(spec.rcr), f32(cut)
    assert up(cut) <= rcr
    pts = [(0, 0, 0), (rca, 0, 0), (0, 0, -up(rca)), (0, rcr, 0), (-cut, 0, 0), (0, -up(cut), 0), (1.1, 0.9, 0.4),
           (-0.3, 1.2, 0.8)]
    x = np.array(pts, dtype=np.float32)
    sp = np.arange(len(x)) % min(spec.num_species, 7)   # (the pair tables hold the 7 ANI-2x elements)
    words = [[j for j in (5, 1, 3, 6, 2, 7, 4) if j < len(x)]] + [[] for _ in range(len(x) - 1)]
    return System(x, sp, words, [0])


@pytest.mark.parametrize("name", ["2x", "gelu", "s8_r17", "s3_r7"])
def test_cutoff_edges(name):
    spec = SPECS[name]
    cut = 4.6 if spec.rcr > 4.6 else 3.0   # a pair cutoff below Rcr (the words hold nothing beyond it)
    sysm = edge_system(spec, cut)
    d = np.linalg.norm(sysm.coords[sysm.words[0]].astype(np.float64), axis=1)
    up = float(np.nextafter(np.float32(spec.rca), np.float32(np.inf)))
    assert (d <= f32(spec.rcr)).all() and (d == f32(spec.rca)).sum() == 1 and (d == up).sum() == 1
    assert (d == f32(spec.rcr)).sum() == 1 and (d == f32(cut)).sum() == 1
    run_geometric(spec, sysm, 16, 64, seed=1, group="edges")
    run_jacobian(spec, sysm, 16, 64)
    for kind in ("xtb", "zbl"):
        run_geometric(spec, sysm, 16, 64, pair_terms(kind, cut, spec.cutoff_fn), group="edges")


def dense_system(spec: orc.AEVSpec, n_ang: int, n_rad: int, seed: int = 4) -> System:
    """One centre (slot) with n_ang neighbours within 3.4 A and n_rad - n_ang in the 3.6 - 5.0 A shell, plus two more
    slots of the cluster."""
    rng = np.random.default_rng(seed)
    inner = ball(n_ang, 0.7, 3.4, rng, 0.75, np.zeros((1, 3)))
    outer = ball(n_rad - n_ang, 3.6, 5.0, rng, 0.75, np.vstack([np.zeros((1, 3)), inner]))
    x = np.vstack([np.zeros((1, 3)), inner, outer]).astype(np.float32)
    sp = rng.integers(0, spec.num_species, len(x))
    # besides the centre, the two shell atoms with the fewest angular neighbours (the crowded inner atoms would
    # exceed ANI_MAX_ANG, which a step reports as an overflow)
    d = np.linalg.norm(x[:, None].astype(np.float64) - x[None].astype(np.float64), axis=-1)
    n_in = (d <= f32(spec.rca)).sum(1) - 1
    slots = [0] + [int(j) for j in n_ang + 1 + np.argsort(n_in[n_ang + 1:], kind="stable")[:2]]
    return System(x, sp, words_within(x, f32(spec.rcr), rng, slots), slots)


def test_dense_neighbourhood():
    spec = SPECS["2x"]
    sysm = dense_system(spec, 94, 256)
    d = np.linalg.norm(vectors(sysm, 0).numpy(), axis=1)
    assert len(sysm.words[0]) == 256 and 90 <= int((d <= f32(spec.rca)).sum()) <= MAX_ANG
    for i in sysm.slots:
        di = np.linalg.norm(vectors(sysm, i).numpy(), axis=1)
        assert int((di <= f32(spec.rca)).sum()) <= MAX_ANG
    run_geometric(spec, sysm, 256, 32768, seed=3, group="dense")
    run_jacobian(spec, sysm, 256, 32768)


# ------------------------------------------------------------------------------------------------------------------
# B. network stage
# ------------------------------------------------------------------------------------------------------------------
class Nets(tp.NamedTuple):
    spec: orc.AEVSpec
    symbols: tp.Tuple[str, ...]
    weights: tp.List[tp.Dict[str, tp.List[tp.Tuple[torch.Tensor, tp.Optional[torch.Tensor]]]]]   # float32
    gelu: bool


def network_set(kind: str, zero_bias: bool = False) -> Nets:
    if kind == "gelu":
        spec = gor.gelu_spec()
        return Nets(spec, orc.SYMBOLS_2X, gor.make_weights(orc.SYMBOLS_2X, orc.DIMS_2X, spec.out_dim, 8, 4321), True)
    spec, symbols, dims = ((orc.aev_spec_2x(), orc.SYMBOLS_2X, orc.DIMS_2X) if kind == "2x"
                           else (orc.aev_spec_1x(), orc.SYMBOLS_1X, orc.DIMS_1X))
    w = orc.make_weights(symbols, dims, spec.out_dim, 8, 1234 if kind == "2x" else 99)
    if zero_bias:
        w = [{s: [(W, torch.zeros_like(b) if k < 3 else b) for k, (W, b) in enumerate(layers)]
              for s, layers in wm.items()} for wm in w]
    return Nets(spec, symbols, w, False)


def packed(nets: Nets, variant: str):
    from torchani_b200 import _lib
    from torchani_b200.engine import PackedNetworks
    return PackedNetworks([[wm[s] for s in nets.symbols] for wm in nets.weights], nets.spec.out_dim, DEV,
                          variant=variant, radial_len=nets.spec.radial_len,
                          activation=_lib.ACT_GELU if nets.gelu else _lib.ACT_CELU)


def network_hessian(nets: Nets, s: int, members: tp.Sequence[int], scale: float, pad: int, ldx: int, a: torch.Tensor,
                    R: torch.Tensor, dtype) -> torch.Tensor:
    """sum_m scale R H_m(a) R^T, H_m by double backward of member m's network in the internal column order."""
    cols = internal_cols(nets.spec, pad).to(DEV)
    act = ((lambda z: torch.nn.functional.gelu(z)) if nets.gelu
           else (lambda z: torch.nn.functional.celu(z, alpha=orc.CELU_ALPHA)))
    a, R = a.to(DEV, dtype), R.to(DEV, dtype)
    out = torch.zeros(R.shape[0], R.shape[0], dtype=dtype, device=DEV)
    for m in members:
        layers = nets.weights[m][nets.symbols[s]]
        W1 = torch.zeros(layers[0][0].shape[0], ldx, dtype=dtype, device=DEV)
        W1[:, cols] = layers[0][0].to(DEV, dtype)
        Ws = [W1] + [W.to(DEV, dtype) for W, _ in layers[1:]]
        bs = [torch.zeros(W.shape[0], dtype=dtype, device=DEV) if b is None else b.to(DEV, dtype)
              for (W, b), W in zip(layers, Ws)]

        def f(v):
            h = v
            for k in range(3):
                h = act(Ws[k] @ h + bs[k])
            return (Ws[3] @ h + bs[3]).sum()
        H = torch.func.jacrev(torch.func.jacrev(f))(a)
        out += scale * (R @ H @ R.t())
    return out.cpu()


def network_case(nets: Nets, counts: tp.Sequence[tp.Tuple[int, int]], members: tp.Sequence[int], variant: str = "",
                 zero_rows: tp.Sequence[int] = (), budget: int = 32768, seed: int = 0) -> None:
    """Slots (element, neighbour count) on random Jacobian rows and AEV rows (``zero_rows``: slots whose AEV row is
    zero); NaN scratch, NaN Jacobian padding rows, random finite Jacobian padding columns, pre-filled blocks."""
    from torchani_b200.engine import tile_a_operand, untile_a_operand
    spec = nets.spec
    _, pad, ldx = aev_params(spec)
    pn = packed(nets, variant)
    assert pn.ldx == ldx and pn.col_pad == pad
    pn.set_active_members(list(members))
    scale = 1.0 / len(members)
    L = lib(variant)
    N, Np = len(counts), 257   # slots 0 .. N - 1 among Np atoms, so that 256 distinct words exist
    sp = np.array([s for s, _ in counts])
    rng = np.random.default_rng(seed)
    # the network stage reads the counts, the elements and the rows only: any positions, words at real atoms
    words = [[int(j) for j in rng.choice(np.delete(np.arange(Np), i), c, replace=False)]
             for i, (_, c) in enumerate(counts)]
    sysm = System(np.zeros((Np, 3), np.float32), np.concatenate([sp, np.zeros(Np - N, int)]),
                  words + [[] for _ in range(Np - N)], list(range(N)))
    dv = to_device(sysm, 256)
    cols = internal_cols(spec, pad)
    rows128 = (Np + 127) // 128 * 128
    aev = torch.zeros(rows128, ldx)
    aev[:, cols] = torch.from_numpy(rng.uniform(0.0, 0.6, (rows128, spec.out_dim))).float()
    row_of = torch.from_numpy(rng.permutation(rows128)[:Np].astype(np.int32))
    for i in zero_rows:
        aev[int(row_of[i])] = 0.0
    x = tile_a_operand(aev.to(DEV), variant=variant or None)
    a_kernel = untile_a_operand(x, rows128, ldx, variant=variant or None).cpu()
    hmax = L.ani_b200_hessian_hidden_max(C.byref(pn.model))
    assert hmax > 64
    for c, plan in enumerate(plans(sysm, budget)):
        ch, _keep = chunk_args(plan)
        slot_rows = torch.from_numpy(plan.row_slot) >= 0
        jac = torch.from_numpy(rng.normal(0.0, 0.1, (plan.rows, ldx))).float()
        jac[~slot_rows] = float("nan")
        scratch = torch.full((4 * plan.rows * hmax + len(plan.atom) * 5 * hmax,), float("nan"), device=DEV)
        blocks, before = prefilled_blocks(plan, seed + c)
        jd = jac.to(DEV)
        assert L.ani_b200_hessian_network(C.byref(pn.model), C.byref(pn.plain_weights), ptr(x), ptr(row_of.to(DEV)),
                                          ptr(dv.spos), ptr(dv.cnt), 256, C.byref(ch), ptr(jd), ptr(scratch),
                                          ptr(blocks), stream()) == 0
        torch.cuda.synchronize()
        check_tail(blocks, plan)
        for k, i in enumerate(plan.atom.tolist()):
            n = len(sysm.words[i])
            if n == 0:
                continue
            got = block_of(blocks, plan, k, n) - block_of(before, plan, k, n)
            R = jac[int(plan.row_off[k]):int(plan.row_off[k]) + 3 * n].double()
            a = a_kernel[int(row_of[i])].double()
            ref = network_hessian(nets, int(sp[i]), members, scale, pad, ldx, a, R, torch.float64)
            ref32 = network_hessian(nets, int(sp[i]), members, scale, pad, ldx, a, R, torch.float32)
            check_bar("network", got, ref, ref32, f"slot of atom {i} (element {sp[i]}, {n} neighbours)")


# (element, neighbour count): every element in one chunk, slots that straddle 64-row tiles, 1 .. 256 neighbours
# (1 .. 24 tiles of the 32 x 32 block contraction)
COUNTS_2X = [(0, 21), (0, 22), (1, 1), (2, 256), (3, 43), (4, 171), (5, 2), (6, 11), (6, 85)]
COUNTS_1X = [(0, 21), (0, 22), (1, 1), (2, 128), (3, 5)]


@pytest.mark.parametrize("kind,members,variant", [
    ("1x", list(range(8)), ""), ("2x", [1, 4, 6], ""), ("2x", [3], ""), ("2x", [2, 7], "bf16x3"), ("gelu", [0, 5], "")])
def test_network_blocks(kind, members, variant):
    from torchani_b200 import _lib
    if variant and not _lib.available(variant):
        pytest.fail(f"the {variant} build is missing (build() compiles it)")
    counts = COUNTS_1X if kind == "1x" else COUNTS_2X
    network_case(network_set(kind), counts, members, variant, seed=len(members))


def test_network_blocks_in_several_chunks():
    network_case(network_set("1x"), COUNTS_1X, [0, 7], budget=320, seed=5)


def test_celu_at_exactly_zero():
    """Zero biases and a zero AEV row: every unit of the slot's network sits at z = 0, where the kernel must take the
    second derivative torch's double backward takes (the other slots keep z != 0)."""
    network_case(network_set("1x", zero_bias=True), COUNTS_1X, [0, 2], zero_rows=[0, 4], seed=9)


# ------------------------------------------------------------------------------------------------------------------
# D. assembly
# ------------------------------------------------------------------------------------------------------------------
def assembly_ref(hess: np.ndarray, sysm: System, plan, blocks: np.ndarray, sorted_orig: np.ndarray, A: int) -> None:
    """hess[conf] += T^T B T, T (3 n x 3 A) the map from the conformer's coordinates to the vectors r_n - r_i."""
    for k, i in enumerate(plan.atom.tolist()):
        n = len(sysm.words[i])
        if n == 0:
            continue
        o = int(plan.block_off[k])
        B = blocks[o:o + 9 * n * n].astype(np.float64).reshape(3 * n, 3 * n)
        conf, ai = divmod(int(sorted_orig[i]), A)
        T = np.zeros((3 * n, 3 * A))
        for m, j in enumerate(sysm.words[i]):
            aj = int(sorted_orig[j]) - conf * A
            for c in range(3):
                T[3 * m + c, 3 * aj + c] = 1.0
                T[3 * m + c, 3 * ai + c] = -1.0
        hess[conf] += T.T @ B @ T


def test_assembly():
    """Three conformers of 300 atoms (the last atoms of conformers 1 and 2 are padding), sorted order a random
    permutation of the real atoms, one atom with 256 neighbour words, isolated atoms; random non-symmetric blocks into
    a pre-filled hess, in several chunks."""
    rng = np.random.default_rng(21)
    n_conf, A = 3, 300
    real = [A, A - 7, A - 40]
    orig = np.concatenate([c * A + np.arange(r) for c, r in enumerate(real)])
    perm = rng.permutation(len(orig))
    sorted_orig = orig[perm].astype(np.int32)                    # sorted index -> flat input index
    conf_of = sorted_orig // A
    isolated = np.arange(len(orig)) % 17 == 0                    # no words and in no atom's words
    big = int(np.nonzero((conf_of == 0) & ~isolated)[0][0])      # the atom with 256 words
    words = []
    for i in range(len(sorted_orig)):
        same = np.nonzero((conf_of == conf_of[i]) & ~isolated)[0]
        same = same[same != i]
        c = 256 if i == big else (0 if isolated[i] else int(rng.integers(1, 40)))
        words.append([int(j) for j in rng.choice(same, c, replace=False)])
    N = len(sorted_orig)
    sysm = System(np.zeros((N, 3), np.float32), rng.integers(0, 7, N), words, list(range(N)))
    dv = to_device(sysm, 256)
    so = torch.from_numpy(sorted_orig).to(DEV)
    hess0 = rng.normal(0.0, 1.0, (n_conf, 3 * A, 3 * A))
    hess = torch.from_numpy(hess0).to(DEV)
    ref = hess0.copy()
    L = lib()
    for c, plan in enumerate(plans(sysm, 4096)):
        ch, _keep = chunk_args(plan)
        blocks = rng.normal(0.0, 1.0, plan.block_floats).astype(np.float32)
        bd = torch.from_numpy(blocks).to(DEV)
        assert L.ani_b200_hessian_assemble(ptr(dv.cnt), ptr(dv.nbr), 256, ptr(so), C.byref(ch), ptr(bd), A, ptr(hess),
                                           stream()) == 0
        assembly_ref(ref, sysm, plan, blocks, sorted_orig, A)
    torch.cuda.synchronize()
    got = hess.cpu().numpy()
    err = float(np.abs((got - hess0) - (ref - hess0)).max())
    scale = float(np.abs(ref - hess0).max())
    _note("assembly", err / (ASSEMBLY_BAR * scale))
    assert err <= ASSEMBLY_BAR * scale, (err, scale)
    # padding atoms and atoms without neighbours in any word list: rows and columns untouched
    touched = {int(sorted_orig[i]) for i in range(N) if words[i]} | {int(sorted_orig[j]) for w in words for j in w}
    for flat in range(n_conf * A):
        if flat in touched:
            continue
        c, a = divmod(flat, A)
        assert np.array_equal(got[c, 3 * a:3 * a + 3], hess0[c, 3 * a:3 * a + 3])
        assert np.array_equal(got[c, :, 3 * a:3 * a + 3], hess0[c, :, 3 * a:3 * a + 3])
    assert len(touched) == len(orig) - int(isolated.sum())


# ------------------------------------------------------------------------------------------------------------------
# E. end to end, new edges
# ------------------------------------------------------------------------------------------------------------------
def test_single_atoms_have_zero_hessians():
    """A chunk whose atoms have no neighbour has no contraction tiles: a single atom and a batch of one-atom
    conformers get zero Hessians."""
    import test_gpu_hessians as th
    m = th.model("2x")
    sp = torch.tensor([[1]], device=DEV)
    e, f, h = m.energies_forces_hessians(sp, torch.zeros(1, 1, 3, device=DEV))
    assert h.shape == (1, 3, 3) and float(h.abs().max()) == 0.0
    sp = torch.tensor([[0], [3], [6], [0]], device=DEV)
    co = torch.randn(4, 1, 3, device=DEV)
    e, f, h = m.energies_forces_hessians(sp, co)
    assert h.shape == (4, 3, 3) and float(h.abs().max()) == 0.0


def test_isolated_atoms_beside_molecules():
    """Water and a far chlorine atom in one conformer, a lone hydrogen in the other: with a 64-row budget the isolated
    atoms form chunks of their own."""
    import test_gpu_hessians as th
    sp0, co0 = th.water()
    sp = torch.tensor([[3, 0, 0, 6], [0, -1, -1, -1]])
    co = torch.zeros(2, 4, 3, dtype=torch.float64)
    co[0, :3] = co0[0]
    co[0, 3] = torch.tensor([30.0, 0.0, 0.0])
    co[1, 0] = torch.tensor([1.0, 2.0, 3.0])
    co32 = co.float().double()
    m = th.model("2x")
    eng = m.engine(DEV)
    eng.step(sp.to(DEV), co32.float().to(DEV), want_grad=True, check=True)
    ws = eng.workspace(*sp.shape)
    h = eng.hessian(ws, row_budget=64).double().cpu()
    energy, _ = th.oracle_energy("2x", sp)
    h64 = hor.hessian(energy, co32)
    b = th.bar(energy, co32, h64)
    err = float((h - h64).abs().max())
    _note("end to end", err / b)
    assert err <= b
    assert float(h[0, 9:].abs().max()) == 0.0 and float(h[0, :, 9:].abs().max()) == 0.0 and float(h[1].abs().max()) == 0.0


def test_dense_cluster_end_to_end():
    """28 atoms of the seven ANI-2x elements in a 2.9 A ball: every atom has all 27 others as angular
    neighbours."""
    import test_gpu_hessians as th
    rng = np.random.default_rng(12)
    x = ball(28, 0.0, 2.9, rng, 1.0, np.zeros((0, 3)))
    sp = torch.tensor(rng.integers(0, 7, 28)).view(1, -1)
    co32 = torch.tensor(x, dtype=torch.float32).double().view(1, -1, 3)
    m = th.model("2x")
    _, _, h = m.energies_forces_hessians(sp.to(DEV), co32.float().to(DEV))
    energy, _ = th.oracle_energy("2x", sp)
    h64 = hor.hessian(energy, co32)
    b = th.bar(energy, co32, h64)
    err = float((h.double().cpu() - h64).abs().max())
    _note("end to end", err / b)
    assert err <= b
