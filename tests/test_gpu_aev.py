"""Kernel-level parity of the AEV kernels (csrc/aev.cu) against float64.

The C-ABI entry points are called directly: ``ani_b200_aev_forward`` in plain (layout 0) and tiled (layout 1) form,
``ani_b200_aev_backward`` with a cotangent the test controls, and the explicit-row entry points through the
``AEVComputer`` module.  The bucket grid, the range table and the row layout come from an ``Engine`` step (tiny
synthetic networks; the MLP plays no part in the checks except in the end-to-end cases).  The reference is
``orc.neighborlist`` + ``orc.aev_from_neighbors`` in float64 on the float32-rounded coordinates, with
``torch.autograd`` for the vector-Jacobian products (VJPs).  ``orc.AEVSpec`` and ``engine.AEVConstants`` have the
same fields, so one tuple drives both sides.

Configurations.  A covering set of AEV constants (``CONFIGS``), not the full product: radial shifts 1, 7, 15, 16, 17,
32; 1, 3, 7 and 8 elements; ShfA x ShfZ = 8x4 and 4x8; cosine and smooth cutoffs; (Rcr, Rca) = (5.1, 3.5),
(6.5, 2.0), (4.0, 3.9); zeta = 1.5, 14.1, 32.  Each case asserts on the host that it reaches the branch it targets:
angular neighbour counts 0 .. 96 (every lanes-per-row split of the rotation and the ordered-pair path), 97 (angular
overflow), radial counts at nbr_cap and nbr_cap + 1, more than 1024 staged candidates in one CTA, a skewed
triclinic cell with 1, 2 and 3 buckets across its directions.

Checks.
* AEVs element-wise at the golden bars (1e-5 relative + 1e-5 absolute).  The tiled operand equals the plain rows
  to the precision of its 16-bit pieces, in the internal column order (``ang_pad`` zero columns between the radial
  and the angular block).
* VJPs dL/dcoords normwise: max |g - g_ref| <= bar * max |g_ref|, 1e-5 for a dense random cotangent, 2e-5 for a
  cotangent on one radial element block or one element-pair block (each term judged at its own scale); the virial
  sum_pairs (dL/dDelta)_a Delta_b against the oracle's strain derivative at 1e-5 of max |W_ref|.
* Exact: neighbour counts against the oracle's (atoms with a pair within 1e-5 A of Rcr excepted), the status word,
  untouched rows and columns (sentinel), dead element blocks not written when the element mask is given, the live
  32-column block list.

Measured on an H100 80GB HBM3 (400 W power limit), worst error / bar: AEVs 0.28 (skewed cell; 0.23 over the
configurations); dense VJPs 0.25, per-block VJPs 0.80 of 1e-5 (0.40 of the 2e-5 bar they are held to), virials
0.39, explicit rows 0.22 (AEV) and 0.16 (VJP), the AEVComputer module 0.10 and 0.14; end-to-end member energies
0.07 of the golden bar.  The module prints the worst ratio of every group at its end (pytest -s).
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
from helpers import E_ATOL, E_RTOL, F_ATOL

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
AEV_RTOL, AEV_ATOL = 1e-5, 1e-5   # element-wise AEV bar (helpers.AEV_RTOL / AEV_ATOL)
VJP_BAR = 1e-5                    # normwise VJP bar, relative to max |g_ref| of the same cotangent
VJP_BLOCK_BAR = 2e-5              # the same for a cotangent on one radial element block or one element-pair block
F_REL_BAR = 1e-4                  # end-to-end forces, normwise relative to max |F_ref| (besides F_ATOL)
VIR_BAR = 1e-5                    # normwise virial bar, relative to max |W_ref|
EDGE = 1e-5                       # pairs this close to Rcr may fall on either side in float32
SENTINEL = 7.25
MAX_ANG = 96                      # ANI_MAX_ANG
STATUS_NBR_OVERFLOW, STATUS_ANG_OVERFLOW = 1, 2

_WORST: tp.Dict[str, float] = {}


def _note(group: str, ratio: float) -> None:
    _WORST[group] = max(_WORST.get(group, 0.0), ratio)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if _WORST:
        print("\nworst error / bar of test_gpu_aev.py:")
        for k in sorted(_WORST):
            print(f"  {k:28s} {_WORST[k]:.3f}")


# ------------------------------------------------------------------------------------------------------------------
# configurations
# ------------------------------------------------------------------------------------------------------------------
class Cfg(tp.NamedTuple):
    name: str
    S: int
    nR: int
    ang: str         # "8x4" | "4x8"  (ShfA x ShfZ)
    cutoff: str
    rcr: float
    rca: float
    zeta: float
    density: float  # of the random box of the config test
    n_atoms: int = 240


CONFIGS = [
    Cfg("s1_r1", 1, 1, "8x4", "cosine", 5.1, 3.5, 14.1, 0.05),
    Cfg("s3_r7", 3, 7, "4x8", "smooth", 6.5, 2.0, 1.5, 0.1),
    Cfg("s7_r16", 7, 16, "8x4", "cosine", 5.1, 3.5, 14.1, 0.1),
    Cfg("s8_r17", 8, 17, "8x4", "smooth", 4.0, 3.9, 32.0, 0.2),
    Cfg("s3_r32", 3, 32, "4x8", "cosine", 5.1, 3.5, 32.0, 0.1),
    # 7 x 15 radial columns: the angular block is not 16-byte aligned in the rows without ang_pad
    Cfg("s7_r15", 7, 15, "4x8", "cosine", 4.0, 3.9, 1.5, 0.2),
    Cfg("s8_r32", 8, 32, "8x4", "smooth", 6.5, 2.0, 14.1, 0.15),
]
CFG = {c.name: c for c in CONFIGS}


def spec_of(c: Cfg) -> orc.AEVSpec:
    na, nz = (8, 4) if c.ang == "8x4" else (4, 8)
    # Gaussian widths that keep neighbouring radial shifts overlapping as in ANI-2x (eta = 19.7 at 16 shifts on 4.3 A)
    step = (c.rcr - 0.8) / c.nR
    eta_r = min(19.7 * (0.26875 / step) ** 2, 100.0)
    a0 = math.pi / nz / 2
    return orc.AEVSpec(c.S, c.rcr, c.rca, eta_r, orc._linspace(0.8, c.rcr, c.nR), 12.5, c.zeta,
                       orc._linspace(0.8, c.rca, na), orc._linspace(a0, math.pi + a0, nz), c.cutoff)


def pair_list(S: int) -> tp.List[tp.Tuple[int, int]]:
    return [(a, b) for a in range(S) for b in range(a, S)]


def internal_cols(spec: orc.AEVSpec, pad: int) -> torch.Tensor:
    """Reference column c -> column of the internal order (radial | pad zero columns | angular)."""
    c = torch.arange(spec.out_dim)
    return torch.where(c < spec.radial_len, c, c + pad)


def live_blocks(spec: orc.AEVSpec, pad: int, mask: int, ldx: int) -> tp.List[int]:
    """32-column blocks of the internal order with at least one live column for the element mask."""
    RL, S, nR = spec.radial_len, spec.num_species, len(spec.shf_r)
    pairs = pair_list(S)

    def live(c: int) -> bool:
        if c < RL:
            return bool((mask >> (c // nR)) & 1)
        c -= pad
        if c < RL or c >= spec.out_dim:
            return False
        a, b = pairs[(c - RL) // spec.angular_sub]
        return bool((mask >> a) & 1 and (mask >> b) & 1)

    return [b for b in range(ldx // 32) if any(live(c) for c in range(32 * b, 32 * b + 32))]


# ------------------------------------------------------------------------------------------------------------------
# geometries (numpy float64, returned float32-rounded)
# ------------------------------------------------------------------------------------------------------------------
class System(tp.NamedTuple):
    species: torch.Tensor            # (1, N) int64
    coords: torch.Tensor             # (1, N, 3) float32
    cell: tp.Optional[torch.Tensor]  # (3, 3) float32 or None
    groups: tp.Optional[np.ndarray] = None   # cluster id of every atom (constructed clusters)


def random_box(n: int, density: float, elements: tp.Sequence[int], seed: int, min_dist: float = 0.8) -> System:
    """Periodic cubic box of n atoms at `density` atoms/A^3, random sequential placement with a minimum distance."""
    rng = np.random.default_rng(seed)
    L = (n / density) ** (1.0 / 3.0)
    pts = np.zeros((0, 3))
    while len(pts) < n:
        p = rng.uniform(0.0, L, 3)
        d = pts - p
        d -= L * np.round(d / L)
        if len(pts) == 0 or float((d * d).sum(1).min()) >= min_dist ** 2:
            pts = np.vstack([pts, p])
    sp = np.array([elements[k % len(elements)] for k in range(n)])
    rng.shuffle(sp)
    return System(torch.tensor(sp).view(1, -1), torch.tensor(pts, dtype=torch.float32).view(1, -1, 3),
                  torch.eye(3, dtype=torch.float32) * L)


def fib_dirs(k: int) -> np.ndarray:
    i = np.arange(k) + 0.5
    z = 1.0 - 2.0 * i / max(k, 1)
    phi = i * math.pi * (3.0 - math.sqrt(5.0))
    r = np.sqrt(np.maximum(1.0 - z * z, 0.0))
    return np.stack([r * np.cos(phi), r * np.sin(phi), z], 1)


def cluster(k_in: int, k_out: int, S: int, rng, r_in=(2.6, 3.3), r_out=(4.0, 5.0)) -> tp.Tuple[np.ndarray, np.ndarray]:
    """A centre (element 0) with k_in neighbours on a shell inside Rca and k_out on a shell beyond it."""
    pts = [np.zeros((1, 3))]
    for k, (lo, hi) in ((k_in, r_in), (k_out, r_out)):
        if k:
            pts.append(fib_dirs(k) * rng.uniform(lo, hi, (k, 1)))
    sp = np.concatenate([[0], np.arange(k_in + k_out) % S])
    return np.concatenate(pts), sp


def clusters_system(specs: tp.Sequence[tp.Tuple[int, int]], S: int, seed: int = 0, spacing: float = 16.0) -> System:
    """Non-periodic system of well separated clusters ((k_in, k_out) each), laid out along x."""
    rng = np.random.default_rng(seed)
    xyz, sp, grp = [], [], []
    for g, (ki, ko) in enumerate(specs):
        p, s = cluster(ki, ko, S, rng)
        xyz.append(p + np.array([g * spacing, 0.0, 0.0]))
        sp.append(s)
        grp.append(np.full(len(s), g))
    return System(torch.tensor(np.concatenate(sp)).view(1, -1),
                  torch.tensor(np.concatenate(xyz), dtype=torch.float32).view(1, -1, 3), None, np.concatenate(grp))


ANG_KS = [0, 1, 2, 3, 4, 5, 8, 9, 16, 17, 31, 32, 33, 48, 64, 95, 96]


def radial_cluster(cap: int, extra: int) -> tp.Tuple[int, int]:
    """(k_in, k_out) of a centre with cap + extra neighbours within Rcr, at most 30 of them within Rca."""
    k_in = min(cap // 4, 30)
    return k_in, cap + extra - k_in


def skewed_cell_system(seed: int = 5) -> System:
    """Triclinic cell 1 x 2 x 3 buckets wide at Rcr = 5.1 A; some atoms on bucket and cell faces, some several lattice
    vectors outside the cell."""
    cell = np.array([[6.2, 0.0, 0.0], [-3.1, 11.4, 0.0], [2.0, -4.0, 16.8]])
    images = np.array([(a, b, c) for a in (-1, 0, 1) for b in (-1, 0, 1) for c in (-1, 0, 1)]) @ cell

    def min_d2(frac: np.ndarray, f: np.ndarray) -> float:
        d = ((frac - f) - np.round(frac - f)) @ cell
        return float(((d[:, None, :] + images[None]) ** 2).sum(-1).min()) if len(frac) else 1e9

    # on faces: fractional 0, 1/2, 1/3, 2/3 and 1 in some directions (bucket and cell faces)
    frac = np.array([[0.0, 0.5, 1.0 / 3.0], [0.5, 0.0, 2.0 / 3.0], [1.0, 0.25, 0.0], [0.75, 1.0, 1.0 / 3.0]])
    rng = np.random.default_rng(seed)
    while len(frac) < 110:
        f = rng.uniform(0.0, 1.0, 3)
        if min_d2(frac, f) >= 0.9 ** 2:
            frac = np.vstack([frac, f])
    xyz = frac @ cell
    shifts = np.array([[2, 0, -3], [-1, 4, 1], [0, -2, 5], [3, 3, 3]])   # several lattice vectors outside
    for j, s in enumerate(shifts):
        xyz[4 + j] += s @ cell
    sp = np.arange(len(xyz)) % 7
    return System(torch.tensor(sp).view(1, -1), torch.tensor(xyz, dtype=torch.float32).view(1, -1, 3),
                  torch.tensor(cell, dtype=torch.float32))


# ------------------------------------------------------------------------------------------------------------------
# float64 oracle
# ------------------------------------------------------------------------------------------------------------------
class Ref:
    def __init__(self, spec: orc.AEVSpec, sysm: System, kind: tp.Optional[str] = None):
        self.spec = spec
        N = sysm.species.shape[1]
        self.c64 = sysm.coords.double().clone().requires_grad_(True)
        self.strain = torch.eye(3, dtype=torch.float64, requires_grad=True)
        cc = self.c64 @ self.strain
        cell, pbc = None, None
        if sysm.cell is not None:
            cell, pbc = sysm.cell.double() @ self.strain, torch.tensor([True, True, True])
        kind = kind or ("cell_list" if sysm.cell is not None else "all_pairs")
        nb = orc.neighborlist(kind, spec.rcr, sysm.species, cc, cell, pbc)
        self.aev = orc.aev_from_neighbors(spec, sysm.species, nb).view(N, spec.out_dim)
        d = nb.distances.detach()
        i0, i1 = nb.indices
        self.counts = torch.bincount(i0, minlength=N) + torch.bincount(i1, minlength=N)
        a = d <= spec.rca
        self.ang_counts = torch.bincount(i0[a], minlength=N) + torch.bincount(i1[a], minlength=N)
        e = (d - spec.rcr).abs() < EDGE
        self.near_edge = torch.zeros(N, dtype=torch.bool)
        self.near_edge[i0[e]] = True
        self.near_edge[i1[e]] = True
        self.values = self.aev.detach()

    def vjp(self, w: torch.Tensor) -> tp.Tuple[torch.Tensor, torch.Tensor]:
        """(dL/dcoords (N, 3), virial W_ab = sum_pairs (dL/dDelta)_a Delta_b) of L = sum(w * aev)."""
        g, gs = torch.autograd.grad((self.aev * w).sum(), [self.c64, self.strain], retain_graph=True)
        return g.view(-1, 3), gs.t()


# ------------------------------------------------------------------------------------------------------------------
# GPU side
# ------------------------------------------------------------------------------------------------------------------
def tiny_weights(S: int, in_dim: int, dims=(32, 32, 32), members: int = 1, seed: int = 7):
    symbols = tuple(f"E{k}" for k in range(S))
    w = orc.make_weights(symbols, {s: dims for s in symbols}, in_dim, members, seed, torch.float32)
    return symbols, w


def make_engine(spec: orc.AEVSpec, nbr_cap: int = 128, col_pad: bool = True, dims=(32, 32, 32), members: int = 1,
                cuda_graph: bool = False):
    from torchani_b200.engine import AEVConstants, Engine, PackedNetworks
    consts = AEVConstants(*spec)
    symbols, w = tiny_weights(spec.num_species, spec.out_dim, dims, members)
    nets = PackedNetworks([[wm[s] for s in symbols] for wm in w], consts.out_dim, torch.device(DEV),
                          radial_len=consts.radial_len if col_pad else 0)
    return Engine(consts, nets, nbr_cap=nbr_cap, cuda_graph=cuda_graph), symbols, w


class Gpu:
    """One system on an engine: the step's preparation, then direct calls of the AEV entry points."""

    def __init__(self, eng, sysm: System):
        from torchani_b200._lib import lib
        self.eng, self.L = eng, lib()
        sp, co = sysm.species.to(DEV), sysm.coords.to(DEV)
        ce = None if sysm.cell is None else sysm.cell.to(DEV)
        self.periodic = sysm.cell is not None
        for _ in range(2):   # the second step sees an unchanged composition: dead element blocks are skipped
            eng.step(sp, co, ce, self.periodic, want_grad=False)
        torch.cuda.synchronize()
        self.ws = ws = eng.workspace(*sysm.species.shape)
        self.n = ws.n
        self.so = ws.sorted_orig[:self.n].long()
        self.rows = ws.row_of[:self.n].long()
        self.ldx = eng.nets.ldx
        self.pad = eng.nets.col_pad
        self.D = eng.consts.out_dim
        self.mask_ptr = ws.aev_blocks.data_ptr() + 4 * (ws.n_blocks + 1)
        self.mask = int(ws.aev_blocks[ws.n_blocks + 1].item())
        self.st = torch.cuda.current_stream().cuda_stream

    def forward(self, layout: int, masked: bool = False) -> tp.Tuple[torch.Tensor, int]:
        from torchani_b200._lib import check, ptr
        from torchani_b200.engine import operand_buffer
        ws, eng = self.ws, self.eng
        out = (torch.full((ws.rows_cap, self.ldx), SENTINEL, device=DEV) if layout == 0
               else operand_buffer(ws.rows_cap, self.ldx, DEV))
        status = torch.zeros(1, dtype=torch.int32, device=DEV)
        check(self.L.ani_b200_aev_forward(
            C.byref(eng.params), ptr(ws.grid), ptr(ws.bin_start), ptr(ws.spos), ptr(ws.sbin), ptr(ws.bucket_ranges),
            ptr(ws.bucket_species), self.mask_ptr if masked else None, self.n, 0, self.n, ptr(ws.row_of), ptr(out),
            self.ldx, layout, ptr(ws.nbr_cnt), ptr(ws.nbr_list), ws.nbr_cap, ptr(status), self.st), "aev_forward")
        torch.cuda.synchronize()
        return out, int(status.item())

    def counts(self) -> torch.Tensor:
        c = torch.zeros(self.n, dtype=torch.long)
        c[self.so.cpu()] = self.ws.nbr_cnt[:self.n].long().cpu()
        return c

    def to_orig(self, plain: torch.Tensor) -> torch.Tensor:
        out = torch.zeros(self.n, self.D, dtype=torch.float64)
        out[self.so.cpu()] = plain[self.rows, :self.D].double().cpu()
        return out

    def backward(self, w: torch.Tensor, lo: int = 0, hi: tp.Optional[int] = None, masked: bool = False,
                 max_elements: int = 0, virial: bool = False) -> tp.Tuple[torch.Tensor, tp.Optional[torch.Tensor], int]:
        from torchani_b200._lib import ANI_VIRIAL_SLOTS, check, ptr
        ws, eng = self.ws, self.eng
        hi = self.n if hi is None else hi
        gaev = torch.zeros(ws.rows_cap, self.ldx, device=DEV)
        cols = internal_cols(eng.consts, self.pad).to(DEV)
        wd = w.to(DEV, torch.float32)
        gaev[self.rows.view(-1, 1), cols.view(1, -1)] = wd[self.so]
        grad = torch.zeros(self.n, 3, device=DEV)
        vir = torch.zeros(ANI_VIRIAL_SLOTS, 9, dtype=torch.float64, device=DEV) if virial else None
        status = torch.zeros(1, dtype=torch.int32, device=DEV)
        check(self.L.ani_b200_aev_backward(
            C.byref(eng.params), ptr(ws.grid), ptr(ws.spos), ptr(ws.sorted_orig), self.mask_ptr if masked else None,
            self.n, lo, hi, ptr(ws.row_of), ptr(gaev), self.ldx, ptr(ws.nbr_cnt), ptr(ws.nbr_list), ws.nbr_cap,
            ptr(grad), ptr(status), max_elements, ptr(vir), self.st), "aev_backward")
        torch.cuda.synchronize()
        return grad.double().cpu(), (vir.sum(0).view(3, 3).cpu() if virial else None), int(status.item())


def aev_ratio(got: torch.Tensor, ref: torch.Tensor) -> float:
    return float(((got - ref).abs() / (AEV_RTOL * ref.abs() + AEV_ATOL)).max()) if got.numel() else 0.0


def norm_ratio(got: torch.Tensor, ref: torch.Tensor, bar: float) -> float:
    scale = max(float(ref.abs().max()), 1e-12)
    return float((got - ref).abs().max()) / (bar * scale)


def block_cotangents(spec: orc.AEVSpec, present: tp.Sequence[int], N: int, seed: int):
    """(name, w) with w random on one radial element block or one element-pair block of the present elements."""
    g = torch.Generator().manual_seed(seed)
    nR, RL = len(spec.shf_r), spec.radial_len
    out = []
    for e in present:
        w = torch.zeros(N, spec.out_dim, dtype=torch.float64)
        w[:, e * nR:(e + 1) * nR] = torch.rand(N, nR, generator=g, dtype=torch.float64) * 2 - 1
        out.append((f"radial{e}", w))
    for p, (a, b) in enumerate(pair_list(spec.num_species)):
        if a in present and b in present:
            w = torch.zeros(N, spec.out_dim, dtype=torch.float64)
            c0 = RL + p * spec.angular_sub
            w[:, c0:c0 + spec.angular_sub] = torch.rand(N, spec.angular_sub, generator=g, dtype=torch.float64) * 2 - 1
            out.append((f"pair{a}{b}", w))
    return out


def dense_cotangent(spec: orc.AEVSpec, N: int, seed: int) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    return torch.rand(N, spec.out_dim, generator=g, dtype=torch.float64) * 2 - 1


def check_forward(gpu: Gpu, ref: Ref, group: str, rows: tp.Optional[torch.Tensor] = None,
                  expect_status: int = 0, check_counts: bool = True) -> None:
    """Plain and tiled AEVs, status, neighbour counts, sentinel and dead-block contracts of one system."""
    from torchani_b200.engine import untile_a_operand
    spec, n, D, ldx, pad = ref.spec, gpu.n, gpu.D, gpu.ldx, gpu.pad
    plain, status = gpu.forward(0)
    assert status == expect_status, f"status {status} != {expect_status}"
    got = gpu.to_orig(plain)
    sel = torch.arange(n) if rows is None else rows
    r = aev_ratio(got[sel], ref.values[sel])
    _note(f"aev {group}", r)
    assert r <= 1.0, f"AEV error {r:.3f} x the bar"
    # rows of no atom and columns past the AEV are never written
    mapped = torch.zeros(plain.shape[0], dtype=torch.bool, device=DEV)
    mapped[gpu.rows] = True
    assert bool((plain[~mapped] == SENTINEL).all()) and bool((plain[:, D:] == SENTINEL).all())
    if check_counts:
        cnt = gpu.counts()
        ok = ~ref.near_edge[sel]
        assert torch.equal(cnt[sel][ok], ref.counts[sel][ok]), "neighbour counts differ from the oracle"
    # tiled operand: the same numbers in the internal column order, zeros in the ang_pad columns and past the AEV
    x, status_t = gpu.forward(1)
    assert status_t == expect_status
    t = untile_a_operand(x.reshape(-1), gpu.ws.rows_cap, ldx)
    cols = internal_cols(spec, pad).to(DEV)
    tv, pv = t[gpu.rows][:, cols], plain[gpu.rows, :D]
    assert bool(((tv - pv).abs() <= pv.abs() * 2.0 ** -21 + 2.0 ** -30).all()), "tiled and plain AEVs differ"
    dead = torch.ones(ldx, dtype=torch.bool, device=DEV)
    dead[cols] = False
    assert bool((t[:, dead] == 0).all()) and bool((t[~mapped] == 0).all())
    # element mask of the step: live columns bit for bit, dead element blocks untouched
    pm, status_m = gpu.forward(0, masked=True)
    assert status_m == expect_status
    present = [e for e in range(spec.num_species) if (gpu.mask >> e) & 1]
    live = torch.zeros(D, dtype=torch.bool)
    nR = len(spec.shf_r)
    for e in present:
        live[e * nR:(e + 1) * nR] = True
    for p, (a, b) in enumerate(pair_list(spec.num_species)):
        if a in present and b in present:
            live[spec.radial_len + p * spec.angular_sub:spec.radial_len + (p + 1) * spec.angular_sub] = True
    lv = live.to(DEV)
    pr = pm[gpu.rows][:, :D]
    assert torch.equal(pr[:, lv], plain[gpu.rows][:, :D][:, lv])
    # dead element blocks, radial and element-pair, are never written (both forward kernels share the feature code)
    dead_ang = ~lv & (torch.arange(D, device=DEV) >= spec.radial_len)
    dead_rad = ~lv & (torch.arange(D, device=DEV) < spec.radial_len)
    assert bool((pr[:, dead_ang] == SENTINEL).all())
    assert bool((pr[:, dead_rad] == SENTINEL).all())
    # live 32-column blocks of the internal order (aev_column_live)
    ws = gpu.ws
    blocks = ws.aev_blocks[1:1 + int(ws.aev_blocks[0])].tolist()
    assert blocks == live_blocks(spec, pad, gpu.mask, ldx)


def check_vjps(gpu: Gpu, ref: Ref, group: str, seed: int, per_block: bool = True, variants: bool = True) -> None:
    spec, N = ref.spec, gpu.n
    present = [e for e in range(spec.num_species) if (gpu.mask >> e) & 1]
    w = dense_cotangent(spec, N, seed)
    g_ref, vir_ref = ref.vjp(w)
    g, vir, st = gpu.backward(w, virial=True)
    assert st == 0
    r = norm_ratio(g, g_ref, VJP_BAR)
    _note(f"vjp dense {group}", r)
    assert r <= 1.0, f"dense VJP error {r:.3f} x the bar"
    rv = norm_ratio(vir, vir_ref, VIR_BAR)
    _note(f"virial {group}", rv)
    assert rv <= 1.0, f"virial error {rv:.3f} x the bar"
    if variants:
        # the compact gradient table sized for the element mask, and for fewer elements than present (the pairs
        # beyond it come from global memory); shards (r, 4) that add up to the whole
        runs = [("masked", dict(masked=True))]
        if len(present) >= 2:
            runs.append(("max_elements1", dict(masked=True, max_elements=1)))
        for name, kw in runs:
            gm, _, st = gpu.backward(w, **kw)
            assert st == 0
            r = norm_ratio(gm, g_ref, VJP_BAR)
            _note(f"vjp {name}", r)
            assert r <= 1.0, f"{name}: VJP error {r:.3f} x the bar"
        gs = torch.zeros_like(g)
        vs = torch.zeros(3, 3, dtype=torch.float64)
        for rank in range(4):
            gr, vr, _ = gpu.backward(w, lo=(N * rank) // 4, hi=(N * (rank + 1)) // 4, virial=True)
            gs += gr
            vs += vr
        r = norm_ratio(gs, g_ref, VJP_BAR)
        _note("vjp shards", r)
        assert r <= 1.0
        assert norm_ratio(vs, vir_ref, VIR_BAR) <= 1.0
    if per_block:
        for name, wb in block_cotangents(spec, present, N, seed + 1):
            gb_ref, _ = ref.vjp(wb)
            gb, _, st = gpu.backward(wb, masked=True)
            assert st == 0
            r = norm_ratio(gb, gb_ref, VJP_BLOCK_BAR)
            _note(f"vjp {'radial' if name.startswith('radial') else 'pair'} block", r)
            assert r <= 1.0, f"{name}: VJP error {r:.3f} x the bar"


# ------------------------------------------------------------------------------------------------------------------
# host-only checks of the constructions
# ------------------------------------------------------------------------------------------------------------------
def test_configs_cover_every_value():
    from torchani_b200.engine import AEVConstants
    assert {c.nR for c in CONFIGS} >= {1, 7, 16, 17, 32}
    assert {c.S for c in CONFIGS} >= {1, 3, 7, 8}
    assert {c.ang for c in CONFIGS} == {"8x4", "4x8"}
    assert {c.cutoff for c in CONFIGS} == {"cosine", "smooth"}
    assert {(c.rcr, c.rca) for c in CONFIGS} == {(5.1, 3.5), (6.5, 2.0), (4.0, 3.9)}
    assert {c.zeta for c in CONFIGS} == {1.5, 14.1, 32.0}
    for c in CONFIGS:
        spec = spec_of(c)
        AEVConstants(*spec).to_struct()
    # radial lengths that are not a multiple of 32 (ang_pad 1 .. 31) and one whose angular block is misaligned
    assert {(-spec_of(c).radial_len) % 32 for c in CONFIGS} - {0}
    assert any(spec_of(c).radial_len % 4 for c in CONFIGS)


def test_live_blocks_host_rule():
    spec = spec_of(CFG["s3_r7"])     # RL = 21, pad 11: angular pair blocks start at column 32
    assert live_blocks(spec, 11, 0b111, 224) == list(range(7))
    assert live_blocks(spec, 11, 0b001, 224) == [0, 1]
    assert live_blocks(spec, 11, 0b100, 224) == [0, 6]
    assert live_blocks(spec, 0, 0b001, 224) == [0, 1]   # without pad the (0, 0) block straddles 21 .. 52


def test_cluster_constructions_reach_their_counts():
    spec = spec_of(CFG["s3_r32"])
    sysm = clusters_system([(k, 0) for k in ANG_KS], 3)
    ref = Ref(spec, sysm)
    centres = [int(np.flatnonzero(sysm.groups == g)[0]) for g in range(len(ANG_KS))]
    assert ref.ang_counts[centres].tolist() == ANG_KS
    assert int(ref.ang_counts.max()) <= MAX_ANG
    over = clusters_system([(97, 0), (40, 0), (7, 0)], 3)
    ro = Ref(spec, over)
    assert int(ro.ang_counts[0]) == 97 and int(ro.ang_counts[over.groups != 0].max()) <= MAX_ANG
    for cap in (32, 128, 256):
        s = clusters_system([radial_cluster(cap, 0)], 3)
        r = Ref(spec, s)
        assert int(r.counts[0]) == cap and int(r.counts.max()) == cap and int(r.ang_counts.max()) <= MAX_ANG
        s = clusters_system([radial_cluster(cap, 1), (10, 0)], 3)
        r = Ref(spec, s)
        assert int(r.counts[0]) == cap + 1 and int(r.counts[s.groups == 1].max()) <= cap
        assert int(r.ang_counts.max()) <= MAX_ANG


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cfg", CONFIGS, ids=[c.name for c in CONFIGS])
def test_config(cfg):
    """Random box of each configuration; every element but the last present (S >= 3), so that dead element blocks
    exist and max_elements = 1 reads most element pairs from global memory."""
    spec = spec_of(cfg)
    elements = list(range(cfg.S - 1)) if cfg.S >= 3 else list(range(cfg.S))
    sysm = random_box(cfg.n_atoms, cfg.density, elements, seed=cfg.nR)
    ref = Ref(spec, sysm)
    cap = 256 if int(ref.counts.max()) > 128 else 128
    assert int(ref.counts.max()) <= cap and int(ref.ang_counts.max()) <= MAX_ANG
    eng, _, _ = make_engine(spec, nbr_cap=cap)
    gpu = Gpu(eng, sysm)
    check_forward(gpu, ref, "config")
    check_vjps(gpu, ref, "config", seed=cfg.nR)


@pytest.mark.gpu
def test_config_without_ang_pad():
    """7 elements x 15 shifts with plain column order: RL = 105, the angular block of every dE/dAEV row is not
    16-byte aligned; the backward with fewer table rows than element pairs keeps every pair in shared memory."""
    cfg = CFG["s7_r15"]
    spec = spec_of(cfg)
    sysm = random_box(cfg.n_atoms, cfg.density, list(range(6)), seed=3)
    ref = Ref(spec, sysm)
    eng, _, _ = make_engine(spec, col_pad=False)
    gpu = Gpu(eng, sysm)
    assert gpu.pad == 0 and spec.radial_len % 4 == 1
    check_forward(gpu, ref, "config")
    check_vjps(gpu, ref, "config", seed=5, per_block=False)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["s3_r32", "s8_r17"])
def test_angular_clusters(name):
    """A centre with k angular neighbours for every k of ANG_KS, one system of separated clusters: every
    lanes-per-row split of the rotation (k <= 32) and the ordered-pair path (33 .. 96)."""
    cfg = CFG[name]
    spec = spec_of(cfg)
    sysm = clusters_system([(k, 0) for k in ANG_KS], cfg.S)
    ref = Ref(spec, sysm)
    centres = [int(np.flatnonzero(sysm.groups == g)[0]) for g in range(len(ANG_KS))]
    assert ref.ang_counts[centres].tolist() == ANG_KS and int(ref.ang_counts.max()) <= MAX_ANG
    eng, _, _ = make_engine(spec)
    gpu = Gpu(eng, sysm)
    check_forward(gpu, ref, "clusters")
    check_vjps(gpu, ref, "clusters", seed=11)


@pytest.mark.gpu
def test_angular_overflow():
    """97 angular neighbours set exactly ANG_OVERFLOW; the atoms of the other clusters keep exact values and VJPs."""
    spec = spec_of(CFG["s3_r32"])
    sysm = clusters_system([(97, 0), (40, 0), (7, 0)], 3)
    ref = Ref(spec, sysm)
    assert int(ref.ang_counts[0]) == 97
    eng, _, _ = make_engine(spec)
    gpu = Gpu(eng, sysm)
    others = torch.from_numpy(np.flatnonzero(sysm.groups != 0))
    check_forward(gpu, ref, "overflow others", rows=others, expect_status=STATUS_ANG_OVERFLOW)
    w = dense_cotangent(spec, gpu.n, 2)
    w[torch.from_numpy(sysm.groups == 0)] = 0.0
    g_ref, _ = ref.vjp(w)
    g, _, st = gpu.backward(w)
    assert st == STATUS_ANG_OVERFLOW
    r = norm_ratio(g[others], g_ref[others], VJP_BAR)
    _note("vjp overflow others", r)
    assert r <= 1.0


@pytest.mark.gpu
@pytest.mark.parametrize("cap", [32, 128, 256])
def test_radial_cap(cap):
    """A centre with exactly nbr_cap radial neighbours (no overflow, exact values), and one with nbr_cap + 1 (exactly
    NBR_OVERFLOW) beside a cluster that does not overflow (exact values there)."""
    spec = spec_of(CFG["s3_r32"])
    sysm = clusters_system([radial_cluster(cap, 0)], 3)
    ref = Ref(spec, sysm)
    assert int(ref.counts[0]) == cap and int(ref.counts.max()) == cap
    eng, _, _ = make_engine(spec, nbr_cap=cap)
    gpu = Gpu(eng, sysm)
    check_forward(gpu, ref, "cap")
    check_vjps(gpu, ref, "cap", seed=cap, per_block=False, variants=False)
    sysm = clusters_system([radial_cluster(cap, 1), (10, 0)], 3)
    ref = Ref(spec, sysm)
    assert int(ref.counts[0]) == cap + 1
    gpu = Gpu(eng, sysm)
    others = torch.from_numpy(np.flatnonzero(sysm.groups == 1))
    check_forward(gpu, ref, "cap+1 others", rows=others, expect_status=STATUS_NBR_OVERFLOW)
    assert int(gpu.counts()[0]) == cap


@pytest.mark.gpu
def test_dense_window():
    """1100 atoms at 0.3 atoms/A^3 in a 3 x 3 x 3 bucket grid: every CTA stages all 1100 candidates (more than one
    768-candidate window and more than the 1024-entry range table of the staging pass); up to ~80 angular
    neighbours (ordered-pair backward)."""
    cfg = CFG["s7_r16"]
    spec = spec_of(cfg)
    sysm = random_box(1100, 0.3, list(range(7)), seed=17)
    ref = Ref(spec, sysm)
    assert int(ref.counts.max()) <= 256 and 32 < int(ref.ang_counts.max()) <= MAX_ANG
    eng, _, _ = make_engine(spec, nbr_cap=256)
    gpu = Gpu(eng, sysm)
    g = eng.grid_info(gpu.ws)
    assert min(g.dims) >= 3
    rng = gpu.ws.bucket_ranges.view(-1, 27, 2, 4)[:, :, 0, :2].contiguous().view(torch.int32).cpu()
    T = (rng[..., 1] - rng[..., 0]).clamp(min=0).sum(1)
    occupied = torch.unique(gpu.ws.sbin[:gpu.n].long().cpu())
    assert int(T[occupied].max()) > 1024
    check_forward(gpu, ref, "dense window")
    check_vjps(gpu, ref, "dense window", seed=17, per_block=False)


@pytest.mark.gpu
def test_skewed_cell_edges():
    """Triclinic cell 1 x 2 x 3 buckets wide, atoms on bucket and cell faces and several lattice vectors outside."""
    spec = spec_of(CFG["s7_r16"])
    sysm = skewed_cell_system()
    ref = Ref(spec, sysm, kind="all_pairs")
    eng, _, _ = make_engine(spec)
    gpu = Gpu(eng, sysm)
    assert sorted(eng.grid_info(gpu.ws).dims) == [1, 2, 3]
    check_forward(gpu, ref, "skewed cell")
    check_vjps(gpu, ref, "skewed cell", seed=23)


@pytest.mark.gpu
def test_bucket_species_offsets(monkeypatch):
    """ANI_B200_AEV_BSS=1 (per-bucket species offsets instead of the counting pass): a fresh engine and workspace."""
    monkeypatch.setenv("ANI_B200_AEV_BSS", "1")
    cfg = CFG["s8_r17"]
    spec = spec_of(cfg)
    sysm = random_box(cfg.n_atoms, cfg.density, list(range(8)), seed=29)
    ref = Ref(spec, sysm)
    eng, _, _ = make_engine(spec)
    gpu = Gpu(eng, sysm)
    assert gpu.ws.bucket_species is not None
    check_forward(gpu, ref, "bss")
    check_vjps(gpu, ref, "bss", seed=29, per_block=False, variants=False)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["s3_r7", "s1_r1"])
def test_module_path(name):
    """AEVComputer (no range table, plain layout, no element mask, ldx = out_dim) with non-stock constants."""
    from torchani_b200.aev import AEVComputer
    cfg = CFG[name]
    spec = spec_of(cfg)
    sysm = random_box(cfg.n_atoms, cfg.density, list(range(cfg.S)), seed=31)
    ref = Ref(spec, sysm)
    m = AEVComputer.from_constants(spec.rcr, spec.rca, spec.eta_r, spec.shf_r, spec.eta_a, spec.zeta, spec.shf_a,
                                   spec.shf_z, spec.num_species, cutoff_fn=spec.cutoff_fn).to(DEV)
    m.nbr_cap = 256          # Rcr = 6.5 A at 0.1 atoms / A^3: up to ~130 radial neighbours
    c = sysm.coords.to(DEV).requires_grad_(True)
    aev = m(sysm.species.to(DEV), c, sysm.cell.to(DEV), torch.tensor([True, True, True], device=DEV))
    r = aev_ratio(aev.detach().double().cpu()[0], ref.values)
    _note("aev module", r)
    assert r <= 1.0
    N = sysm.species.shape[1]
    w = dense_cotangent(spec, N, 37)
    (g,) = torch.autograd.grad((aev[0] * w.float().to(DEV)).sum(), c)
    g_ref, _ = ref.vjp(w)
    r = norm_ratio(g.double().cpu().view(N, 3), g_ref, VJP_BAR)
    _note("vjp module", r)
    assert r <= 1.0


@pytest.mark.gpu
def test_explicit_rows_from_pairs_and_full_list():
    """ani_b200_aev_forward_rows / _backward_rows: from a half pair list (compute_from_neighbors) and from a full
    list with ghost atoms (compute_from_full_neighborlist)."""
    from torchani_b200.aev import AEVComputer
    from torchani_b200.neighbors import Neighbors
    spec = spec_of(CFG["s8_r17"])
    m = AEVComputer.from_constants(spec.rcr, spec.rca, spec.eta_r, spec.shf_r, spec.eta_a, spec.zeta, spec.shf_a,
                                   spec.shf_z, spec.num_species, cutoff_fn=spec.cutoff_fn).to(DEV)
    # (a) half pair list of a periodic box, taken from the oracle (float32 diff vectors)
    sysm = random_box(200, 0.2, list(range(8)), seed=41)
    ref = Ref(spec, sysm)
    N = sysm.species.shape[1]
    nb = orc.neighborlist("cell_list", spec.rcr, sysm.species, sysm.coords.double(), sysm.cell.double(),
                          torch.tensor([True, True, True]))
    c = sysm.coords.to(DEV).requires_grad_(True)
    diff = nb.diff_vectors.float().to(DEV)    # x[i0] - x[i1] + image shift, rounded once
    aev = m.compute_from_neighbors(sysm.species.to(DEV), c,
                                   Neighbors(nb.indices.to(DEV), nb.distances.float().to(DEV), diff))
    r = aev_ratio(aev.detach().double().cpu()[0], ref.values)
    _note("aev rows pairs", r)
    assert r <= 1.0
    w = dense_cotangent(spec, N, 43)
    (g,) = torch.autograd.grad((aev[0] * w.float().to(DEV)).sum(), c)
    g_ref, _ = ref.vjp(w)
    r = norm_ratio(g.double().cpu().view(N, 3), g_ref, VJP_BAR)
    _note("vjp rows pairs", r)
    assert r <= 1.0
    # (b) full list over local + ghost atoms of a cluster system: the AEV rows of the local atoms only
    sysm = clusters_system([(40, 0), (12, 0)], 8)
    ref = Ref(spec, sysm)
    N = sysm.species.shape[1]
    local = torch.arange(0, N, 2)          # every other atom is a ghost
    jl = [torch.tensor([j for j in range(N) if j != int(i)]) for i in local]
    c = sysm.coords.to(DEV).requires_grad_(True)
    aev = m.compute_from_full_neighborlist(sysm.species.to(DEV), c, local.to(DEV), torch.cat(jl).to(DEV),
                                           torch.tensor([len(x) for x in jl]).to(DEV))
    got = aev.detach().double().cpu()[0]
    r = aev_ratio(got[local], ref.values[local])
    _note("aev rows full list", r)
    assert r <= 1.0
    ghosts = torch.ones(N, dtype=torch.bool)
    ghosts[local] = False
    assert float(got[ghosts].abs().max()) == 0.0
    w = dense_cotangent(spec, N, 47)
    w[ghosts] = 0.0
    (g,) = torch.autograd.grad((aev[0] * w.float().to(DEV)).sum(), c)
    g_ref, _ = ref.vjp(w)
    r = norm_ratio(g.double().cpu().view(N, 3), g_ref, VJP_BAR)
    _note("vjp rows full list", r)
    assert r <= 1.0


@pytest.mark.gpu
@pytest.mark.parametrize("col_pad", [True, False], ids=["ang_pad", "no_pad"])
@pytest.mark.parametrize("name", ["s8_r17", "s3_r7"])
def test_engine_end_to_end(name, col_pad):
    """Synthetic two-member networks through the whole step against orc.compute at the golden bars, then a graph
    captured with two elements and replayed with all of them (the AEV backward's table is sized for two elements at
    capture).  8 x 17: 36 element pairs, ldx = 1312 (41 K-blocks); 3 x 7: RL = 21 (ang_pad 11, or a misaligned
    angular block without it)."""
    cfg = CFG[name]
    spec = spec_of(cfg)
    sysm = random_box(cfg.n_atoms, 0.1, list(range(cfg.S)), seed=53)
    eng, symbols, w = make_engine(spec, nbr_cap=256, dims=(96, 64, 32), members=2, col_pad=col_pad, cuda_graph=True)
    assert (eng.nets.col_pad > 0) == col_pad
    sae = {s: 0.0 for s in symbols}
    model = orc.Model(spec, symbols, [{s: [(a.double(), b.double()) for a, b in wm[s]] for s in symbols} for wm in w],
                      sae, "cell_list")
    pbc = torch.tensor([True, True, True])
    ref = orc.compute(model, sysm.species, sysm.coords.double(), sysm.cell.double(), pbc)
    sp, co, ce = sysm.species.to(DEV), sysm.coords.to(DEV), sysm.cell.to(DEV)
    two = torch.where(sp % 2 == 0, 0, 1)
    for _ in range(eng.graph_after + 1):   # eager uses, then the capture, all with two elements
        eng.step(two, co, ce, True)
    ws = eng.workspace(*sysm.species.shape)
    assert len(eng._graphs) == 1 and ws.max_elements == 2
    res = eng.step(sp, co, ce, True)       # replay with every element
    torch.cuda.synchronize()
    eng.check_status()
    assert len(eng._graphs) == 1
    assert ws.aev_blocks[1:1 + int(ws.aev_blocks[0])].tolist() == live_blocks(spec, eng.nets.col_pad,
                                                                               (1 << cfg.S) - 1, eng.nets.ldx)
    ma = res.member_atomic.cpu().double()
    ratio_e = float(((ma - ref["member_atomic"]).abs() / (E_RTOL * ref["member_atomic"].abs() + E_ATOL)).max())
    _note("engine member energies", ratio_e)
    assert ratio_e <= 1.0
    ratio_f = float((-res.grad.cpu().double() - ref["forces"]).abs().max()) / F_ATOL
    _note("engine forces", ratio_f)
    assert ratio_f <= 1.0
    r = norm_ratio(-res.grad.cpu().double().view(-1, 3), ref["forces"].view(-1, 3), F_REL_BAR)
    _note("engine forces relative", r)
    assert r <= 1.0


@pytest.mark.gpu
@pytest.mark.parametrize("var", ["ANI_B200_AEV_TMA", "ANI_B200_AEV_LEGACY"])
def test_forward_variants(var):
    """The bulk-copy staging and the warp-per-atom forward are chosen once per process (function statics): re-run a
    subset of this file in a child process with the switch set, under a timeout."""
    env = dict(os.environ, **{var: "1"})
    sel = "test_config and (s3_r7 or s8_r17) or test_angular_clusters and s3_r32 or test_dense_window"
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
        "-m", "pytest", os.path.abspath(__file__), "-q", "-m", "gpu", "-k", sel, "-p", "no:cacheprovider"]
    res = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stdout[-4000:] + res.stderr[-2000:]
    assert " passed" in res.stdout and " failed" not in res.stdout
