"""The step preparation kernels (csrc/cells.cu) against a plain restatement of their contract.

The preparation turns (coords, species, cell) into the bucket grid, the deterministic (bucket, species, input index)
order, wrapped positions, the 27-bucket range table, the species-grouped row layout, the live AEV column blocks, the
per-bucket species offsets and the zero-fills that every later kernel reads.  It exists in four forms that must agree:
``k_prep_cluster`` (one thread-block cluster: periodic single systems up to 16,384 atoms), ``k_prep_fused`` (a
persistent grid with device-wide barriers), five launches (``ANI_B200_PREP_FUSED=0``) and the module API
``ani_b200_build_cells`` + ``ani_b200_species_layout`` + ``ani_b200_active_aev_blocks``.

The entry points are called directly, with every output and scratch area exactly as large as ``include/ani_b200.h``
documents it and a guard band of sentinels on both sides; every form runs twice on the same buffers.  The
restatement below (numpy, float64) gives the grid dimensions, the admissible bucket of every atom (an atom within
4 ulp of a bucket or cell face may sit on either side), the order, the wrapped positions, the range table, the row
layout and the block list; a float64 brute force over all lattice images gives the pairs every central atom must be
able to reach through its 27 ranges.  The cluster form proves that it ran by the ``%globaltimer`` stamps it writes
with ``ANI_B200_PREP_TRACE=1``.  The five-launch form and the 8-CTA cluster are chosen once per process, so the file
re-runs itself in child processes for them.

Also here: the Verlet refresh (``ani_b200_verlet_positions``), the energy reduction (``ani_b200_reduce_energies``)
and the reference-format half neighbour lists of ``neighbors.cell_list`` / ``all_pairs`` on the same edge geometries.
With ``pytest -s`` every case prints the form that ran, how many atoms used the face allowance and how many pairs
within 1e-5 A of the cutoff were excused.
"""
import ctypes as C
import math
import os
import subprocess
import sys
import typing as tp
from contextlib import contextmanager

import numpy as np
import pytest
import torch
from scipy.spatial.distance import cdist

import oracle.ani_oracle as orc
from test_gpu_aev import live_blocks, skewed_cell_system

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUTOFF = 5.1
EDGE = 1e-5                # pairs this close to the cutoff may fall on either side in float32
TILE = 128                 # ANI_TILE_ROWS
MAX_SPECIES = 8            # ANI_MAX_SPECIES
CHUNK = 256                # rows of one layout chunk (LAYOUT_CHUNK)
CLUSTER_MAX_ATOMS = 16384  # PREP_CLUSTER_MAX_ATOMS
BRUTE_MAX = 2500           # the float64 all-images brute force runs up to this many atoms
GUARD = 16                 # sentinel words on each side of every buffer (64 B keep float4 / int4 alignment)
SENT = 0x5A5A5A5A
GRID_WORDS = 29            # sizeof(ani_grid) / 4
STATUS_CELL_TOO_SMALL = 4
U = 2.0 ** -24             # unit roundoff of float32


# ------------------------------------------------------------------------------------------------------------------
# problems
# ------------------------------------------------------------------------------------------------------------------
class Problem(tp.NamedTuple):
    name: str
    coords: np.ndarray            # (n, 3) float32, flat over the conformers
    species: np.ndarray           # (n,) int32, -1 = padding
    cell: tp.Optional[np.ndarray]  # (3, 3) float32, rows are lattice vectors
    S: int                        # num_species
    n_conf: int = 1
    max_bins: int = 0             # 0: what the engine uses
    lo: int = 0
    hi: int = -1                  # -1: n
    cutoff: float = CUTOFF
    ang_pad: bool = True

    @property
    def n(self) -> int:
        return len(self.species)

    @property
    def pbc(self) -> int:
        return int(self.cell is not None)

    @property
    def mode(self) -> int:
        return 0 if self.n_conf == 1 else 1

    @property
    def n_per_conf(self) -> int:
        return self.n // self.n_conf

    @property
    def bins(self) -> int:
        if self.max_bins:
            return self.max_bins
        return max(64, self.n + 2) if self.n_conf == 1 else self.n_conf + 2

    @property
    def slice(self) -> tp.Tuple[int, int]:
        return self.lo, (self.n if self.hi < 0 else self.hi)


class AEVShape(tp.NamedTuple):
    spec: orc.AEVSpec
    pad: int
    ldx: int

    @staticmethod
    def of(S: int, ang_pad: bool) -> "AEVShape":
        spec = orc.aev_spec_2x(S)
        pad = (-spec.radial_len) % 32 if ang_pad else 0
        return AEVShape(spec, pad, -(-(spec.out_dim + pad) // 32) * 32)


def water(n_mol: int, seed: int = 0) -> tp.Tuple[np.ndarray, np.ndarray, np.ndarray]:
    _, idx, xyz, cell, _ = orc.water_box(n_mol, seed=seed)
    return xyz[0].numpy(), idx[0].numpy().astype(np.int32), cell.numpy()


def uniform_box(n: int, density: float, S: int, seed: int) -> tp.Tuple[np.ndarray, np.ndarray, np.ndarray]:
    rng = np.random.default_rng(seed)
    L = (n / density) ** (1.0 / 3.0)
    return (rng.uniform(0.0, L, (n, 3)).astype(np.float32), rng.integers(0, S, n).astype(np.int32),
            (np.eye(3) * L).astype(np.float32))


def in_cell(cell: np.ndarray, n: int, seed: int, min_dist: float = 0.9, faces=()) -> np.ndarray:
    """n points of a periodic cell (float64), some at given fractional positions, a minimum image distance apart."""
    rng = np.random.default_rng(seed)
    frac = np.array(faces, dtype=np.float64).reshape(-1, 3)
    while len(frac) < n:
        f = rng.uniform(0.0, 1.0, 3)
        d = (frac - f) - np.round(frac - f)
        if len(frac) == 0 or float(((d @ cell) ** 2).sum(1).min()) >= min_dist ** 2:
            frac = np.vstack([frac, f])
    return frac @ cell


def with_padding(xyz: np.ndarray, sp: np.ndarray, every: int, far: float = 0.0) -> tp.Tuple[np.ndarray, np.ndarray]:
    """Insert a padding atom (species -1, coordinates `far`) after every `every` atoms."""
    out_x, out_s = [], []
    for k in range(len(sp)):
        out_x.append(xyz[k])
        out_s.append(sp[k])
        if k % every == every - 1:
            out_x.append(np.full(3, far))
            out_s.append(-1)
    return np.array(out_x, dtype=np.float32), np.array(out_s, dtype=np.int32)


def bucket_len(cutoff: float) -> float:
    return float(np.float32(cutoff) + np.float32(1e-5))   # compute_grid: cutoff + 1e-5f in float32


def sheared_cell() -> np.ndarray:
    """Directions 0 and 1 have EDGE lengths of 2+ buckets but perpendicular WIDTHS of 1 bucket."""
    return np.array([[12.0, 0.0, 0.0], [9.0, 6.5, 0.0], [0.0, 0.0, 11.0]])


def build_problem(name: str) -> Problem:
    if name == "water999":
        xyz, sp, cell = water(333)
        return Problem(name, xyz, sp, cell, 4)
    if name == "water40k":
        xyz, sp, cell = water(13334, seed=3)
        return Problem(name, xyz, sp, cell, 4)
    if name in ("box16384", "box16385"):
        xyz, sp, cell = uniform_box(int(name[3:]), 0.1, 4, seed=int(name[3:]))
        return Problem(name, xyz, sp, cell, 4)
    if name == "skewed":
        s = skewed_cell_system()
        return Problem(name, s.coords[0].numpy(), s.species[0].numpy().astype(np.int32), s.cell.numpy(), 7)
    if name == "sheared":
        cell = sheared_cell()
        xyz = in_cell(cell, 90, seed=7, faces=[(0, 0, 0), (0.5, 0.5, 0.5), (1.0, 0.0, 0.5), (0.0, 1.0, 0.0)])
        xyz[5] += np.array([2, -1, 1]) @ cell
        return Problem(name, xyz.astype(np.float32), (np.arange(90) % 5).astype(np.int32),
                       cell.astype(np.float32), 5)
    if name == "one_bucket_s8":
        cell = np.eye(3) * 8.0
        xyz = in_cell(cell, 150, seed=11, min_dist=0.8, faces=[(0, 0, 0), (0.5, 0, 1)])
        rng = np.random.default_rng(11)
        sp = rng.choice(8, 150, p=[0.4, 0.3, 0.1, 0.05, 0.05, 0.04, 0.03, 0.03])
        sp[:8] = np.arange(8)
        return Problem(name, xyz.astype(np.float32), sp.astype(np.int32), cell.astype(np.float32), 8)
    if name == "width_edges":
        # widths 3 b (1 + 1e-6), 3 b (1 - 1e-6), 4 b (1 + 1e-6) for the bucket length b: dims 3, 2, 4
        b = bucket_len(CUTOFF)
        cell = np.diag([3 * b * (1 + 1e-6), 3 * b * (1 - 1e-6), 4 * b * (1 + 1e-6)]).astype(np.float32)
        c64 = cell.astype(np.float64)
        faces = [(k / 3, 0.5, j / 4) for k in range(4) for j in range(5)] + [(0.5, 0.5, 0.5), (0, 0, 0)]
        xyz = in_cell(c64, 1300, seed=13, min_dist=0.95, faces=faces)
        sp = (np.arange(1300) * 7 % 6).astype(np.int32)
        return Problem(name, xyz.astype(np.float32), sp, cell, 6)
    if name.startswith("dilute"):
        cell = np.eye(3) * 60.0
        xyz = in_cell(cell, 20, seed=17, min_dist=2.0, faces=[(0, 0, 0), (0.5, 0.5, 1.0)])
        bins = {"dilute_n+2": 22, "dilute_64": 64, "dilute_1400": 1400}[name]
        return Problem(name, xyz.astype(np.float32), (np.arange(20) % 3).astype(np.int32), cell.astype(np.float32),
                       3, max_bins=bins)
    if name == "thin_cell":
        cell = np.diag([14.0, 4.0, 12.0])
        xyz = in_cell(cell, 40, seed=19)
        return Problem(name, xyz.astype(np.float32), (np.arange(40) % 4).astype(np.int32),
                       cell.astype(np.float32), 4)
    if name == "open_far":
        rng = np.random.default_rng(23)
        xyz = rng.uniform(0.0, 22.0, (600, 3)) + np.array([1000.0, -600.0, 500.0])
        xyz, sp = with_padding(xyz, (np.arange(600) % 4).astype(np.int32), 7, far=1e6)
        return Problem(name, xyz, sp, None, 4)
    if name == "batch":
        sp, xyz = orc.conformer_batch(40, 9, 26, seed=29)
        sp = torch.cat([sp, torch.full((1, sp.shape[1]), -1)])          # one fully padded conformer
        xyz = torch.cat([xyz, torch.zeros(1, sp.shape[1], 3)])
        sp, xyz = sp[[0, 1, 2, 40, 3] + list(range(4, 40))], xyz[[0, 1, 2, 40, 3] + list(range(4, 40))]
        return Problem(name, xyz.reshape(-1, 3).numpy(), sp.reshape(-1).numpy().astype(np.int32), None, 4,
                       n_conf=sp.shape[0])
    if name == "padded_periodic":
        xyz, sp, cell = water(333, seed=5)
        xyz, sp = with_padding(xyz, sp, 30)
        return Problem(name, xyz, sp, cell, 4)
    raise KeyError(name)


SYSTEMS = ["water999", "water40k", "box16384", "box16385", "skewed", "sheared", "one_bucket_s8", "width_edges",
           "dilute_n+2", "dilute_64", "dilute_1400", "thin_cell", "open_far", "batch", "padded_periodic"]


# ------------------------------------------------------------------------------------------------------------------
# the restatement (host, float64)
# ------------------------------------------------------------------------------------------------------------------
class GridRef(tp.NamedTuple):
    cell: np.ndarray    # float64 values of the float32 cell the kernels use
    inv: np.ndarray     # its float64 inverse
    origin: np.ndarray
    dims: tp.Tuple[int, int, int]
    pbc: int
    nbins: int
    mode: int
    n_per_conf: int
    n_real: int
    too_small: bool


def grid_ref(p: Problem) -> GridRef:
    """Bucket grid of compute_grid: perpendicular widths of the cell (bounding box + 2e-3 without PBC) over
    cutoff + 1e-5, then the capacity rule (shrink the largest dimension by max(1, d // 8) while the product exceeds
    max_bins - 1); one bucket per conformer in mode 1."""
    real = p.species >= 0
    n_real = int(real.sum())
    b = bucket_len(p.cutoff)
    too_small = False
    if p.mode == 1:
        return GridRef(np.eye(3), np.eye(3), np.zeros(3), (1, 1, 1), 0, p.n_conf, 1, p.n_per_conf, n_real, False)
    if p.pbc:
        cell = p.cell.astype(np.float64)
        inv = np.linalg.inv(cell)
        widths = 1.0 / np.linalg.norm(inv, axis=0)
        dims = [int(math.floor(w / b)) for w in widths]
        too_small = min(dims) < 1
        dims = [max(1, d) for d in dims]
        origin = np.zeros(3)
    else:
        x = p.coords[real] if n_real else np.zeros((1, 3), np.float32)
        mn, mx = x.min(0), x.max(0)
        ext = (mx - mn) + np.float32(2e-3)                     # float32, as the kernel
        origin = (mn - np.float32(1e-3)).astype(np.float64)
        cell = np.diag(ext.astype(np.float64))
        inv = np.diag(1.0 / ext.astype(np.float64))
        dims = [max(1, int(math.floor(float(np.float32(e) / np.float32(b))))) for e in ext]
    while dims[0] * dims[1] * dims[2] > p.bins - 1:
        big = int(np.argmax(dims))
        dims[big] = max(1, dims[big] - max(1, dims[big] // 8))
    return GridRef(cell, inv, origin, tuple(dims), p.pbc, dims[0] * dims[1] * dims[2], 0, p.n_per_conf, n_real,
                   too_small)


def ulp(m: float) -> float:
    return 2.0 ** (math.floor(math.log2(max(m, 1e-30))) - 23)


def bucket_check(g: GridRef, p: Problem, k_dev: np.ndarray, idx_dev: np.ndarray) -> tp.Tuple[np.ndarray, int]:
    """Is the device's (lattice vector k, bucket index) of every real atom admissible?  Returns (ok per real atom,
    atoms that used the face allowance).  k_dev, idx_dev: (n_real, 3) ints of the real atoms in input order."""
    x = p.coords[p.species >= 0].astype(np.float64)
    frac = (x - g.origin) @ g.inv
    M = max(float(np.abs(p.coords[p.species >= 0]).max(initial=0.0)), float(np.abs(g.cell).max()),
            float(np.abs(g.origin).max()))
    tol = 4 * ulp(M) * np.abs(g.inv).sum(0) + 2 * U          # fractional units, per direction
    dims = np.array(g.dims)
    k0 = np.floor(frac) if g.pbc else np.zeros_like(frac)
    u = (frac - k0) * dims
    i0 = np.clip(np.floor(u), 0, dims - 1)
    main = (k_dev == k0) & (idx_dev == i0)
    j = np.round(u)
    near = np.abs(u - j) <= tol * dims
    alt = near & (j > 0) & (j < dims) & (k_dev == k0) & ((idx_dev == j - 1) | (idx_dev == j))
    low = near & (j == 0) & (((k_dev == k0) & (idx_dev == 0)) | (bool(g.pbc) & (k_dev == k0 - 1) & (idx_dev == dims - 1)))
    high = near & (j == dims) & (((k_dev == k0) & (idx_dev == dims - 1)) | (bool(g.pbc) & (k_dev == k0 + 1) & (idx_dev == 0)))
    ok = main | alt | low | high
    return ok.all(1), int((ok.all(1) & ~main.all(1)).sum())


def decode_bucket(b: np.ndarray, dims) -> np.ndarray:
    return np.stack([b // (dims[1] * dims[2]), (b // dims[2]) % dims[1], b % dims[2]], -1)


def ranges_ref(g: GridRef, bin_start: np.ndarray):
    """Range table of every bucket: (lo, hi, code, neighbour bucket, image word w (3), exists), each (nbins, 27[, 3])."""
    dims = np.array(g.dims)
    b3 = decode_bucket(np.arange(g.nbins), g.dims)[:, None, :]
    off = np.array([(o // 9 - 1, (o // 3) % 3 - 1, o % 3 - 1) for o in range(27)])[None]
    j = b3 + off
    w = np.floor_divide(j, dims)
    jm = j - w * dims
    nb = (jm[..., 0] * dims[1] + jm[..., 1]) * dims[2] + jm[..., 2]
    exists = np.full(nb.shape, True) if g.pbc else (w == 0).all(-1)
    lo = np.where(exists, bin_start[nb], 0)
    hi = np.where(exists, bin_start[nb + 1], 0)
    code = 9 * (w[..., 0] + 1) + 3 * (w[..., 1] + 1) + (w[..., 2] + 1)
    return lo, hi, code, np.where(exists, nb, 0), w, exists


def image_shifts(cell: np.ndarray, cutoff: float) -> np.ndarray:
    reps = np.ceil(cutoff * np.linalg.norm(np.linalg.inv(cell), axis=0)).astype(int)
    return np.array([(a, b, c) for a in range(-reps[0], reps[0] + 1) for b in range(-reps[1], reps[1] + 1)
                     for c in range(-reps[2], reps[2] + 1)])


def brute_pairs(x: np.ndarray, cell: tp.Optional[np.ndarray], cutoff: float, atoms: np.ndarray,
                groups: tp.Optional[np.ndarray] = None):
    """Every ORDERED pair (a, c, n), a != c or n != 0, with |x_c + n @ cell - x_a| <= cutoff + EDGE, over all lattice
    images, in float64.  x: (n, 3) input coordinates; atoms: indices that take part; groups: conformer of each atom
    (pairs only inside one).  Returns (a, c, n (P, 3), d)."""
    x = x.astype(np.float64)
    xa = x[atoms]
    if cell is None:
        kw = np.zeros_like(xa)
        shifts = np.zeros((1, 3), dtype=int)
        cell = np.eye(3)
    else:
        kw = np.floor(xa @ np.linalg.inv(cell))
        shifts = image_shifts(cell, cutoff + EDGE)
    xw = xa - kw @ cell
    A, Cc, Nn, D = [], [], [], []
    for s in shifts:
        d = cdist(xw, xw + s @ cell)
        ok = d <= cutoff + EDGE
        if not s.any():
            np.fill_diagonal(ok, False)
        if groups is not None:
            ga = groups[atoms]
            ok &= ga[:, None] == ga[None, :]
        a, c = np.nonzero(ok)
        A.append(atoms[a])
        Cc.append(atoms[c])
        # x_c + n cell - x_a = xw_c + s cell - xw_a  ->  n = s - kw_c + kw_a
        Nn.append((s[None] - kw[c] + kw[a]).astype(np.int64))
        D.append(d[a, c])
    return np.concatenate(A), np.concatenate(Cc), np.concatenate(Nn), np.concatenate(D)


def completeness(g: GridRef, pairs, k_atom: np.ndarray, bucket_atom: np.ndarray, sorted_of: np.ndarray, table,
                 cutoff: float) -> tp.Tuple[int, int]:
    """Every pair within the cutoff must be reachable: the central atom's bucket has a range that holds the
    neighbour's sorted position and whose image word w gives the pair's lattice shift (w = n + k_c - k_a, with k the
    lattice vector that wrapped each atom).  Returns (missing pairs beyond the edge allowance, excused pairs)."""
    a, c, n, d = pairs
    lo, hi, code = table
    w = n + k_atom[c] - k_atom[a]
    valid = (np.abs(w) <= 1).all(1)
    wc = 9 * (w[:, 0] + 1) + 3 * (w[:, 1] + 1) + (w[:, 2] + 1)
    ba, ic = bucket_atom[a], sorted_of[c]
    hit = ((lo[ba] <= ic[:, None]) & (ic[:, None] < hi[ba]) & (code[ba] == wc[:, None])).any(1) & valid
    inside = d <= cutoff
    edge = np.abs(d - cutoff) < EDGE
    missing = inside & ~hit & ~edge
    return int(missing.sum()), int((inside & ~hit & edge).sum())


class LayoutRef(tp.NamedTuple):
    row_of: np.ndarray        # rows of the owned atoms (sorted positions `owned`)
    owned: np.ndarray
    row_atom: np.ndarray
    tile_species: np.ndarray
    info: np.ndarray          # layout_info[0..12]


def layout_ref(sp_sorted: np.ndarray, n_real: int, lo: int, hi: int, S: int, rows_cap: int) -> LayoutRef:
    """row_of[i] = base[s] + #{owned i' < i of species s}, base = 128-row padded prefix of the species counts."""
    owned = np.arange(lo, max(lo, min(hi, n_real)))
    sp = sp_sorted[owned]
    tot = np.array([(sp == s).sum() for s in range(S)], dtype=np.int64)
    padded = -(-tot // TILE) * TILE
    base = np.concatenate([[0], np.cumsum(padded)])
    row_of = np.zeros(len(owned), dtype=np.int64)
    for s in range(S):
        m = sp == s
        row_of[m] = base[s] + np.arange(int(m.sum()))
    row_atom = np.full(rows_cap, -1, dtype=np.int64)
    row_atom[row_of] = owned
    r = np.arange(rows_cap // TILE) * TILE
    tile = np.full(len(r), -1, dtype=np.int64)
    for s in range(S):
        tile[(r >= base[s]) & (r < base[s] + tot[s])] = s
    total = int(base[S])
    info = [total // TILE, total, len(owned), 0] + [int(base[s]) // TILE for s in range(S + 1)]
    info += [total // TILE] * (MAX_SPECIES - S)
    return LayoutRef(row_of, owned, row_atom, tile, np.array(info))


def bss_ref(sbin: np.ndarray, sp_sorted: np.ndarray, nbins: int) -> np.ndarray:
    out = np.zeros((nbins, MAX_SPECIES), dtype=np.int64)
    real = sbin < nbins
    for s in range(1, MAX_SPECIES):
        np.add.at(out[:, s], sbin[real & (sp_sorted < s)], 1)
    return out


def canon(i0: np.ndarray, i1: np.ndarray, m: np.ndarray) -> tp.Set[tp.Tuple[int, ...]]:
    """Unordered pairs (i0, i1, m) ~ (i1, i0, -m) as a set of (low, high, m) with m lexicographically positive for
    self-image pairs."""
    flip = (i0 > i1) | ((i0 == i1) & ~lex_pos(m))
    a, b = np.where(flip, i1, i0), np.where(flip, i0, i1)
    mm = np.where(flip[:, None], -m, m)
    return set(map(tuple, np.concatenate([a[:, None], b[:, None], mm], 1).tolist()))


def lex_pos(m: np.ndarray) -> np.ndarray:
    return (m[:, 0] > 0) | ((m[:, 0] == 0) & ((m[:, 1] > 0) | ((m[:, 1] == 0) & (m[:, 2] > 0))))


# ------------------------------------------------------------------------------------------------------------------
# device side: buffers of exactly the documented sizes between sentinel guard bands
# ------------------------------------------------------------------------------------------------------------------
class Guarded:
    def __init__(self, words: int, zero: bool = False):
        self.words = words
        self.full = torch.full((words + 2 * GUARD,), SENT, dtype=torch.int32, device=DEV)
        if zero:
            self.full[GUARD:GUARD + words] = 0

    @property
    def ptr(self) -> int:
        return self.full.data_ptr() + 4 * GUARD

    def inner(self) -> np.ndarray:
        return self.full[GUARD:GUARD + self.words].cpu().numpy()

    def guards_ok(self) -> bool:
        f = self.full.cpu().numpy()
        return bool((f[:GUARD] == SENT).all() and (f[GUARD + self.words:] == SENT).all())


@contextmanager
def env(**kv):
    old = {k: os.environ.get(k) for k in kv}
    os.environ.update({k: str(v) for k, v in kv.items()})
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def expected_form(p: Problem, ldx: int) -> str:
    """The host-side rule of ani_b200_prepare_step (cluster_ok)."""
    fe, ce = os.environ.get("ANI_B200_PREP_FUSED"), os.environ.get("ANI_B200_PREP_CLUSTER")
    if fe is not None and int(fe) == 0:
        return "five launches"
    if ((ce is None or int(ce) != 0) and p.pbc and p.mode == 0 and p.n <= CLUSTER_MAX_ATOMS
            and p.bins - 1 <= CLUSTER_MAX_ATOMS + 1 and ldx // 32 <= 64):
        return "cluster"
    return "persistent grid"


def rows_cap_of(p: Problem) -> int:
    lo, hi = p.slice
    return -(-((hi - lo) + p.S * (TILE - 1)) // TILE) * TILE     # the smallest legal capacity


class Run:
    """One form of the preparation on one problem, twice on the same buffers."""

    def __init__(self, p: Problem, form: str, calls: int = 2, species_seq: tp.Optional[tp.List[np.ndarray]] = None):
        from torchani_b200._lib import check, lib
        self.p, self.form = p, form
        self.shape = AEVShape.of(p.S, p.ang_pad)
        n, mb = p.n, p.bins
        lo, hi = p.slice
        self.rows_cap = rows_cap_of(p)
        nchunk = max(1, -(-(hi - lo) // CHUNK))     # an empty slice still takes one layout chunk
        self.b = b = {
            "grid": Guarded(GRID_WORDS), "bin_start": Guarded(mb + 2), "sorted_orig": Guarded(n),
            "orig_to_sorted": Guarded(n), "spos": Guarded(4 * n), "sbin": Guarded(n),
            "ranges": Guarded((mb - 1) * 27 * 8), "row_of": Guarded(n), "row_atom": Guarded(self.rows_cap),
            "tile_species": Guarded(self.rows_cap // TILE), "layout_info": Guarded(16),
            "aev_blocks": Guarded(self.shape.ldx // 32 + 3), "status": Guarded(1, zero=True),
        }
        if form == "build_cells":
            b["scratch"] = Guarded(3 * n + mb + 2, zero=True)
            b["scratch_layout"] = Guarded((-(-n // 256) + 2) * MAX_SPECIES + 64, zero=True)
            b["scratch_blocks"] = Guarded(1, zero=True)
        else:
            b["scratch"] = Guarded(3 * n + mb + 4 + (nchunk + 2) * MAX_SPECIES + 32, zero=True)
            b["bss"] = Guarded(mb * MAX_SPECIES)
            b["zero_f32"] = Guarded(3 * n)
            b["zero_f64"] = Guarded(2 * p.n_conf)
        L = lib()
        st = torch.cuda.current_stream().cuda_stream
        coords = torch.tensor(p.coords, device=DEV).contiguous()
        cell = None if p.cell is None else torch.tensor(p.cell, device=DEV).reshape(-1).contiguous()
        cp = None if cell is None else cell.data_ptr()
        spec, pad, ldx = self.shape
        asub = len(spec.shf_a) * len(spec.shf_z)
        self.blocks_after: tp.List[np.ndarray] = []
        for k in range(calls):
            sp_np = p.species if species_seq is None else species_seq[k]
            species = torch.tensor(sp_np, dtype=torch.int32, device=DEV)
            if form == "build_cells":
                check(L.ani_b200_build_cells(
                    coords.data_ptr(), species.data_ptr(), p.n_conf, p.n_per_conf, cp, p.pbc, p.mode, p.cutoff, mb,
                    b["grid"].ptr, b["bin_start"].ptr, b["sorted_orig"].ptr, b["orig_to_sorted"].ptr, b["spos"].ptr,
                    b["sbin"].ptr, b["ranges"].ptr, b["scratch"].ptr, b["status"].ptr, st), "build_cells")
                check(L.ani_b200_species_layout(
                    b["spos"].ptr, b["grid"].ptr, n, lo, hi, p.S, self.rows_cap, b["row_of"].ptr, b["row_atom"].ptr,
                    b["tile_species"].ptr, b["layout_info"].ptr, b["scratch_layout"].ptr, st), "species_layout")
                check(L.ani_b200_active_aev_blocks(
                    b["spos"].ptr, b["grid"].ptr, n, p.S, len(spec.shf_r), asub, spec.out_dim, ldx, pad,
                    b["aev_blocks"].ptr, b["scratch_blocks"].ptr, st), "active_aev_blocks")
            else:
                b["zero_f32"].full.fill_(SENT)
                b["zero_f64"].full.fill_(SENT)
                with env(ANI_B200_PREP_TRACE=1):
                    check(L.ani_b200_prepare_step(
                        coords.data_ptr(), species.data_ptr(), p.n_conf, p.n_per_conf, cp, p.pbc, p.mode, p.cutoff, mb,
                        b["grid"].ptr, b["bin_start"].ptr, b["sorted_orig"].ptr, b["orig_to_sorted"].ptr,
                        b["spos"].ptr, b["sbin"].ptr, b["ranges"].ptr, lo, hi, p.S, self.rows_cap, b["row_of"].ptr,
                        b["row_atom"].ptr, b["tile_species"].ptr, b["layout_info"].ptr, len(spec.shf_r), asub,
                        spec.out_dim, ldx, pad, b["aev_blocks"].ptr, b["zero_f32"].ptr, 3 * n, b["zero_f64"].ptr,
                        p.n_conf, b["bss"].ptr, b["scratch"].ptr, b["status"].ptr, st), "prepare_step")
            torch.cuda.synchronize()
            self.blocks_after.append(b["aev_blocks"].inner())
        self.species = p.species if species_seq is None else species_seq[-1]
        for key, buf in b.items():
            assert buf.guards_ok(), f"{p.name} / {form}: a guard word of `{key}` was overwritten"
        self.o = {k: v.inner() for k, v in b.items()}
        self.nchunk = nchunk

    def trace_stamps(self) -> np.ndarray:
        """The 12 %globaltimer words k_prep_cluster writes behind species_base (ANI_B200_PREP_TRACE=1)."""
        n, mb = self.p.n, self.p.bins
        sb = 3 * n + 2 + (mb + 1) + 2 + (self.nchunk + 1) * MAX_SPECIES
        addr = self.b["scratch"].ptr + 4 * (sb + MAX_SPECIES)
        first = (((addr + 7) & ~7) - self.b["scratch"].ptr) // 4
        return self.o["scratch"][first:first + 24].view(np.int64)

    # -- decoded outputs
    def grid(self) -> tp.Dict[str, tp.Any]:
        w = self.o["grid"]
        f = w.view(np.float32)
        return dict(cell=f[0:9].reshape(3, 3), inv=f[9:18].reshape(3, 3), origin=f[18:21], dims=tuple(w[21:24]),
                    pbc=int(w[24]), nbins=int(w[25]), mode=int(w[26]), n_per_conf=int(w[27]), n_real=int(w[28]))


def check_run(r: Run, stats: tp.Dict[str, int]) -> None:
    """Every output of one form against the restatement."""
    p, o = r.p, r.o
    name = f"{p.name} / {r.form}"
    species = r.species
    pp = p._replace(species=species)
    g = grid_ref(pp)
    gd = r.grid()
    n, n_real = p.n, g.n_real
    # ---- grid
    assert gd["dims"] == g.dims, (name, gd["dims"], g.dims)
    assert (gd["pbc"], gd["nbins"], gd["mode"], gd["n_per_conf"], gd["n_real"]) == (g.pbc, g.nbins, g.mode,
                                                                                    g.n_per_conf, n_real), name
    assert np.allclose(gd["cell"], g.cell, rtol=U, atol=U * np.abs(g.cell).max()), name
    assert np.allclose(gd["inv"], g.inv, rtol=2 * U, atol=2 * U * np.abs(g.inv).max()), name
    assert np.allclose(gd["origin"], g.origin, rtol=U, atol=0), name
    status = int(o["status"][0])
    assert bool(status & STATUS_CELL_TOO_SMALL) == g.too_small, (name, status)
    assert status & ~STATUS_CELL_TOO_SMALL == 0, (name, status)
    # ---- order
    so, o2s, sbin = o["sorted_orig"], o["orig_to_sorted"], o["sbin"]
    assert sorted(so.tolist()) == list(range(n)), name
    assert (o2s[so] == np.arange(n)).all(), name
    bs = o["bin_start"]
    pop = np.bincount(sbin, minlength=g.nbins + 1)
    assert len(pop) == g.nbins + 1, name
    assert (bs[:g.nbins + 2] == np.concatenate([[0], np.cumsum(pop)])).all(), name
    assert (bs[g.nbins + 2:] == SENT).all(), name        # bin_start[nbins + 2 ..] is never written
    assert (np.diff(sbin) >= 0).all(), name
    real_sorted = so[:n_real]
    assert (species[real_sorted] >= 0).all() and (species[so[n_real:]] < 0).all(), name
    assert (sbin[n_real:] == g.nbins).all(), name
    same = sbin[1:n_real] == sbin[:n_real - 1]
    s0, s1 = species[real_sorted[:-1]], species[real_sorted[1:]]
    i0, i1 = real_sorted[:-1], real_sorted[1:]
    assert ((s0 < s1) | ((s0 == s1) & (i0 < i1)))[same].all(), f"{name}: (species, index) order inside a bucket"
    if r.form == "build_cells":     # k_bin_finalize ranks the padding atoms by index too
        assert (np.diff(so[n_real:]) > 0).all(), name
    # ---- wrapped positions, bucket of every real atom
    spos = o["spos"].view(np.float32).reshape(n, 4)
    sw = o["spos"].reshape(n, 4)[:, 3]
    assert (sw == species[so]).all(), f"{name}: spos.w is not the species"
    assert (spos[n_real:, :3] == 0).all(), name
    real = np.nonzero(species >= 0)[0]
    pos = spos[o2s[real], :3].astype(np.float64)
    x = p.coords[real].astype(np.float64)
    if g.mode == 1:
        k = np.zeros((len(real), 3))
        assert (sbin[o2s[real]] == real // p.n_per_conf).all(), name
    else:
        kf = (x - pos) @ g.inv
        k = np.round(kf)
        assert np.abs(kf - k).max(initial=0) < 1e-3, name
        kmax = max(1.0, float(np.abs(k).max(initial=0)))
        M = max(float(np.abs(x).max(initial=0)), kmax * float(np.abs(g.cell).max()))
        assert np.abs(pos - (x - k @ g.cell)).max(initial=0) <= 4 * ulp(M), f"{name}: wrapped position"
        ok, allowance = bucket_check(g, pp, k, decode_bucket(sbin[o2s[real]], g.dims))
        assert ok.all(), f"{name}: {int((~ok).sum())} atoms in an inadmissible bucket, e.g. {real[~ok][:5]}"
        stats["face allowance"] = stats.get("face allowance", 0) + allowance
    home = (k == 0).all(1)
    assert (spos[o2s[real[home]], :3].view(np.int32) == p.coords[real[home]].view(np.int32)).all(), \
        f"{name}: an atom inside the cell did not keep its float32 coordinates bit for bit"
    if not g.pbc:
        assert home.all(), name
    # ---- range table
    rng = o["ranges"].reshape(-1, 27, 8)
    if g.mode == 0:
        lo_r, hi_r, code, nb, w, exists = ranges_ref(g, bs)
        t = rng[:g.nbins]
        assert (t[..., 0] == lo_r).all() and (t[..., 1] == hi_r).all(), f"{name}: range bounds"
        assert (t[..., 2] == code).all(), f"{name}: image codes"
        assert (t[..., 3] == (0 if r.form == "build_cells" else nb)).all(), f"{name}: neighbour bucket word"
        shift = w @ g.cell
        tf = t.view(np.float32)
        scale = np.abs(w[..., :, None] * g.cell[None, None]).sum(-2)
        assert (np.abs(tf[..., 4:7] - shift) <= np.maximum(scale, 1e-30) * 2 * U).all(), f"{name}: image shifts"
        assert (t[..., 7] == 0).all(), name
        assert (rng[g.nbins:] == SENT).all(), name
        if n <= BRUTE_MAX and not g.too_small:   # (a cell thinner than the cutoff needs more than 27 buckets)
            pairs = brute_pairs(p.coords, g.cell if g.pbc else None, p.cutoff, real)
            k_all = np.zeros((n, 3), dtype=np.int64)
            k_all[real] = k.astype(np.int64)
            missing, excused = completeness(g, pairs, k_all, sbin[o2s], o2s, (lo_r, hi_r, code), p.cutoff)
            assert missing == 0, f"{name}: {missing} pairs within the cutoff are unreachable"
            stats["excused pairs"] = stats.get("excused pairs", 0) + excused
            stats["pairs checked"] = stats.get("pairs checked", 0) + int((pairs[3] <= p.cutoff).sum())
    else:
        assert (rng == SENT).all(), name
    # ---- layout
    lo, hi = p.slice
    lay = layout_ref(sw, n_real, lo, hi, p.S, r.rows_cap)
    assert (o["row_of"][lay.owned] == lay.row_of).all(), f"{name}: row_of"
    assert (o["row_atom"] == lay.row_atom).all(), f"{name}: row_atom"
    assert (o["tile_species"] == lay.tile_species).all(), f"{name}: tile_species"
    assert (o["layout_info"][:13] == lay.info).all(), (name, o["layout_info"][:13], lay.info)
    # ---- live AEV blocks
    spec, pad, ldx = r.shape
    mask = int(np.bitwise_or.reduce(1 << species[species >= 0], initial=0))
    ids = live_blocks(spec, pad, mask, ldx)
    blk = o["aev_blocks"]
    assert blk[0] == len(ids) and blk[1:1 + len(ids)].tolist() == ids, f"{name}: live blocks"
    assert blk[ldx // 32 + 1] == mask, name
    assert blk[ldx // 32 + 2] == 0, f"{name}: the changed flag after a repeated call"
    assert r.blocks_after[0][ldx // 32 + 2] == 1, f"{name}: the changed flag after the first call"
    if r.form == "build_cells":
        return
    # ---- per-bucket species offsets, zero-fills, cluster stamps
    bss = o["bss"].reshape(-1, MAX_SPECIES)
    assert (bss[:g.nbins] == bss_ref(sbin, sw, g.nbins)).all(), f"{name}: bucket_species"
    assert (bss[g.nbins:] == SENT).all(), name
    assert (o["zero_f32"] == 0).all() and (o["zero_f64"] == 0).all(), f"{name}: zero-fill"
    stamps = r.trace_stamps()
    assert (stamps != 0).all() if r.form == "cluster" else (stamps == 0).all(), \
        f"{name}: the cluster kernel's trace stamps do not match the expected form"


def same_outputs(a: Run, b: Run) -> None:
    """Two forms bit for bit, except the order of the padding atoms and the range word .w of build_cells."""
    n_real = a.grid()["n_real"]
    name = f"{a.p.name}: {a.form} vs {b.form}"
    for k in ("grid", "bin_start", "sbin", "spos", "row_atom", "tile_species", "layout_info", "aev_blocks"):
        assert (a.o[k] == b.o[k]).all(), f"{name}: {k}"
    assert (a.o["sorted_orig"][:n_real] == b.o["sorted_orig"][:n_real]).all(), name
    assert set(a.o["sorted_orig"][n_real:].tolist()) == set(b.o["sorted_orig"][n_real:].tolist()), name
    real = np.nonzero(a.species >= 0)[0]
    assert (a.o["orig_to_sorted"][real] == b.o["orig_to_sorted"][real]).all(), name
    lo, hi = a.p.slice
    own = np.arange(lo, min(hi, n_real))
    assert (a.o["row_of"][own] == b.o["row_of"][own]).all(), name
    ra, rb = a.o["ranges"].reshape(-1, 8), b.o["ranges"].reshape(-1, 8)
    cols = [0, 1, 2, 4, 5, 6, 7] if "build_cells" in (a.form, b.form) else list(range(8))
    assert (ra[:, cols] == rb[:, cols]).all(), f"{name}: ranges"
    if "build_cells" not in (a.form, b.form):
        for k in ("bss", "zero_f32", "zero_f64"):
            assert (a.o[k] == b.o[k]).all(), f"{name}: {k}"


def report(name: str, forms: tp.Sequence[str], stats: tp.Dict[str, int]) -> None:
    extra = ", ".join(f"{k} {v}" for k, v in stats.items())
    print(f"\n  {name}: {' + '.join(forms)}" + (f"; {extra}" if extra else ""))


def run_forms(p: Problem, **kw) -> tp.List[Run]:
    """prepare_step as the environment selects it, prepare_step without the cluster, build_cells + layout + blocks:
    each against the restatement, then against each other."""
    ldx = AEVShape.of(p.S, p.ang_pad).ldx
    runs, stats = [], {}
    seen = set()
    for cl in ("1", "0"):
        with env(ANI_B200_PREP_CLUSTER=cl):
            form = expected_form(p, ldx)
            if form in seen:
                continue
            seen.add(form)
            runs.append(Run(p, form, **kw))
    runs.append(Run(p, "build_cells", **kw))
    for r in runs:
        check_run(r, stats)
    for r in runs[1:]:
        same_outputs(runs[0], r)
    report(p.name, [r.form for r in runs], stats)
    return runs


# ------------------------------------------------------------------------------------------------------------------
# CPU: the restatement itself against the oracle
# ------------------------------------------------------------------------------------------------------------------
def emulate(p: Problem) -> tp.Tuple[GridRef, np.ndarray, np.ndarray, np.ndarray]:
    """What the preparation must produce, from the restatement alone: (grid, sorted_orig, sbin, lattice vector k of
    every atom), binning in float64."""
    g = grid_ref(p)
    x = p.coords.astype(np.float64)
    frac = (x - g.origin) @ g.inv
    k = np.floor(frac) if g.pbc else np.zeros_like(frac)
    dims = np.array(g.dims)
    idx = np.clip(np.floor((frac - k) * dims), 0, dims - 1).astype(np.int64)
    b = np.where(p.species >= 0, (idx[:, 0] * dims[1] + idx[:, 1]) * dims[2] + idx[:, 2], g.nbins)
    order = np.lexsort((np.arange(p.n), p.species, b))
    return g, order, b[order], k.astype(np.int64)


@pytest.mark.parametrize("name", ["skewed", "sheared", "one_bucket_s8", "dilute_64", "open_far"])
def test_restatement_against_the_oracle(name):
    """No device: the restated grid, bucket order and range table of a system reach every pair of
    orc.neighborlist('all_pairs'); the brute force used by the GPU tests finds exactly the oracle's pairs; an
    edge-length grid (what the restatement must NOT be) misses pairs in the sheared cell; the layout rule equals a
    plain loop."""
    p = build_problem(name)
    g, order, sbin, k = emulate(p)
    real = np.nonzero(p.species >= 0)[0]
    # dims: perpendicular widths; equal to the oracle's edge-length rule for an orthorhombic cell
    if p.pbc and np.count_nonzero(p.cell - np.diag(np.diag(p.cell))) == 0 and p.max_bins == 0:
        edge = np.floor(np.linalg.norm(p.cell.astype(np.float64), axis=1) / bucket_len(p.cutoff)).astype(int)
        assert g.dims == tuple(edge)
    # the brute force == the oracle
    pairs = brute_pairs(p.coords, g.cell if g.pbc else None, p.cutoff, real)
    keep = pairs[3] <= p.cutoff
    mine = canon(pairs[0][keep], pairs[1][keep], -pairs[2][keep])
    sp_t = torch.tensor(p.species, dtype=torch.long).view(1, -1)
    x_t = torch.tensor(p.coords, dtype=torch.float64).view(1, -1, 3)
    if p.pbc:
        nb = orc.neighborlist("all_pairs", p.cutoff, sp_t, x_t, torch.tensor(p.cell, dtype=torch.float64),
                              torch.tensor([True, True, True]))
    else:
        nb = orc.neighborlist("all_pairs", p.cutoff, sp_t, x_t)
    i0, i1 = nb.indices.numpy()
    raw = p.coords[i0].astype(np.float64) - p.coords[i1].astype(np.float64)
    m = np.round((nb.diff_vectors.numpy() - raw) @ g.inv).astype(np.int64) if p.pbc else np.zeros((len(i0), 3), int)
    theirs = canon(i0, i1, m)
    assert len(theirs) == len(i0) > 0
    sym = mine ^ theirs
    assert not sym, f"{len(sym)} pairs differ between the brute force and the oracle"
    # completeness of the emulated preparation
    pos = np.empty(p.n, dtype=np.int64)
    pos[order] = np.arange(p.n)
    bs = np.concatenate([[0], np.cumsum(np.bincount(sbin, minlength=g.nbins + 1))])
    if g.mode == 0:
        lo_r, hi_r, code, _, _, _ = ranges_ref(g, bs)
        missing, _ = completeness(g, pairs, k, sbin[pos], pos, (lo_r, hi_r, code), p.cutoff)
        assert missing == 0
        if name == "sheared":
            # a grid from edge lengths has buckets thinner than the cutoff here: pairs two buckets apart are lost
            edge = tuple(int(v) for v in np.floor(np.linalg.norm(g.cell, axis=1) / bucket_len(p.cutoff)))
            assert edge != g.dims
            ge = g._replace(dims=edge, nbins=int(np.prod(edge)))
            frac = p.coords.astype(np.float64) @ g.inv
            kk = np.floor(frac)
            idx = np.clip(np.floor((frac - kk) * np.array(edge)), 0, np.array(edge) - 1).astype(np.int64)
            be = (idx[:, 0] * edge[1] + idx[:, 1]) * edge[2] + idx[:, 2]
            oe = np.lexsort((np.arange(p.n), p.species, be))
            pe = np.empty(p.n, dtype=np.int64)
            pe[oe] = np.arange(p.n)
            bse = np.concatenate([[0], np.cumsum(np.bincount(be, minlength=ge.nbins + 1))])
            lo_e, hi_e, code_e, _, _, _ = ranges_ref(ge, bse)
            missing, _ = completeness(ge, pairs, kk.astype(np.int64), be, pe, (lo_e, hi_e, code_e), p.cutoff)
            assert missing > 0
    # layout rule against a plain loop
    sp_sorted = p.species[order]
    lo, hi = p.n // 5, p.n - 3
    lay = layout_ref(sp_sorted, g.n_real, lo, hi, p.S, 4096)
    base, row_of = 0, {}
    for s in range(p.S):
        mine_s = [i for i in range(lo, min(hi, g.n_real)) if sp_sorted[i] == s]
        for j, i in enumerate(mine_s):
            row_of[i] = base + j
        base += -(-len(mine_s) // TILE) * TILE
    assert dict(zip(lay.owned.tolist(), lay.row_of.tolist())) == row_of
    assert lay.info[1] == base and lay.info[4 + p.S] == base // TILE


# ------------------------------------------------------------------------------------------------------------------
# GPU: every system, every form
# ------------------------------------------------------------------------------------------------------------------
def system_branch(p: Problem) -> None:
    """What each system is there for, asserted on the host."""
    g = grid_ref(p)
    lo, hi = p.slice
    ldx = AEVShape.of(p.S, p.ang_pad).ldx
    form = expected_form(p, ldx)
    if p.name == "water999":
        assert form in ("cluster", "five launches") and min(g.dims) >= 3
    if p.name == "water40k":
        assert form != "cluster" and -(-(hi - lo) // CHUNK) > 128
    if p.name == "box16384":
        assert p.n == CLUSTER_MAX_ATOMS and form in ("cluster", "five launches")
    if p.name == "box16385":
        assert p.n == CLUSTER_MAX_ATOMS + 1 and form != "cluster"
    if p.name == "skewed":
        assert sorted(g.dims) == [1, 2, 3]
    if p.name == "sheared":
        edge = np.floor(np.linalg.norm(g.cell, axis=1) / bucket_len(p.cutoff)).astype(int)
        assert g.dims[0] == 1 and g.dims[1] == 1 and edge[0] >= 2 and edge[1] >= 2
    if p.name == "one_bucket_s8":
        assert g.dims == (1, 1, 1) and p.n > 100 and set(p.species.tolist()) == set(range(8))
    if p.name == "width_edges":
        assert g.dims == (3, 2, 4) and p.n > 1024
    if p.name.startswith("dilute"):
        full = int(math.floor(60.0 / bucket_len(p.cutoff))) ** 3
        assert (g.nbins == full > p.n) if p.bins > full else g.nbins < full
    if p.name == "thin_cell":
        assert g.too_small
    if p.name == "open_far":
        assert not p.pbc and (p.species < 0).any() and np.abs(p.coords[p.species >= 0]).min() > 400
    if p.name == "batch":
        assert p.mode == 1 and (p.species.reshape(p.n_conf, -1) < 0).all(1).any()


@pytest.mark.gpu
@pytest.mark.parametrize("name", SYSTEMS)
def test_preparation_forms(name):
    p = build_problem(name)
    system_branch(p)
    run_forms(p)


@pytest.mark.gpu
@pytest.mark.parametrize("shard", [(0, 1), (1, 4), (3, 8), (7, 8), (0, 16)], ids=lambda s: f"{s[0]}of{s[1]}")
def test_shards(shard):
    """Owned slices of the sorted atoms: a 10-atom periodic system (16 ranks: an empty slice) and a periodic water
    box with padding atoms (the last slices end beyond n_real)."""
    rank, world = shard
    cell = np.eye(3) * 11.0
    xyz = in_cell(cell, 10, seed=31, min_dist=1.5)
    small = Problem("ten atoms", xyz.astype(np.float32), np.array([0, 1, 0, 2, 3, 0, 1, 1, 0, 3], np.int32),
                    cell.astype(np.float32), 4)
    big = build_problem("padded_periodic")
    for p in (small, big):
        lo, hi = p.n * rank // world, p.n * (rank + 1) // world
        q = p._replace(name=f"{p.name} shard {rank}/{world}", lo=lo, hi=hi)
        if (rank, world) == (0, 16) and p is small:
            assert lo == hi
        if p is big and rank == world - 1:
            assert hi > int((p.species >= 0).sum())
        run_forms(q)


@pytest.mark.gpu
@pytest.mark.parametrize("ang_pad", [True, False], ids=["ang_pad", "no_pad"])
def test_element_subsets(ang_pad):
    """{H, O}, {C, S}, a single element on the same buffers: the live blocks follow the composition and the changed
    flag is raised exactly by the calls that change it."""
    xyz, _, cell = water(100, seed=37)
    n = len(xyz)
    rng = np.random.default_rng(37)
    seq = [rng.choice([0, 3], n), None, rng.choice([1, 4], n), None, np.full(n, 5), None]
    for k in range(len(seq)):
        if seq[k] is None:
            seq[k] = seq[k - 1]
    seq = [s.astype(np.int32) for s in seq]
    p = Problem(f"elements ({'ang_pad' if ang_pad else 'no pad'})", xyz, seq[-1], cell, 7, ang_pad=ang_pad)
    ldx = AEVShape.of(7, ang_pad).ldx
    for form in (expected_form(p, ldx), "build_cells"):
        r = Run(p, form, calls=len(seq), species_seq=seq)
        flags = [int(b[ldx // 32 + 2]) for b in r.blocks_after]
        assert flags == [1, 0, 1, 0, 1, 0], (form, flags)
        for b, s in zip(r.blocks_after, seq):
            mask = int(np.bitwise_or.reduce(1 << s))
            ids = live_blocks(r.shape.spec, r.shape.pad, mask, ldx)
            assert b[ldx // 32 + 1] == mask and b[0] == len(ids) and b[1:1 + len(ids)].tolist() == ids
        stats: tp.Dict[str, int] = {}
        r.blocks_after = r.blocks_after[-2:]      # the last composition, set by the call before the repeat
        check_run(r, stats)
        report(p.name, [form], stats)


@pytest.mark.gpu
def test_permuted_input():
    """The same system with its input order permuted: the same atoms in every bucket, ordered by the new indices."""
    p = build_problem("skewed")
    perm = np.random.default_rng(41).permutation(p.n)
    q = p._replace(name="skewed permuted", coords=p.coords[perm], species=p.species[perm])
    a, b = run_forms(p)[0], run_forms(q)[0]
    assert (a.o["sbin"] == b.o["sbin"]).all() and (a.o["bin_start"] == b.o["bin_start"]).all()
    nb = a.grid()["nbins"]
    bs = a.o["bin_start"]
    for k in range(nb):
        ia = set(a.o["sorted_orig"][bs[k]:bs[k + 1]].tolist())
        ib = set(perm[b.o["sorted_orig"][bs[k]:bs[k + 1]]].tolist())
        assert ia == ib, k


# ------------------------------------------------------------------------------------------------------------------
# Verlet refresh
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_verlet_refresh():
    from torchani_b200._lib import check, lib
    L = lib()
    st = torch.cuda.current_stream().cuda_stream
    skin = 1.0
    xyz, sp, cell = water(333, seed=43)
    xyz, sp = with_padding(xyz, sp, 40)
    p = Problem("verlet", xyz, sp, cell, 4, cutoff=CUTOFF + skin)
    r = Run(p, expected_form(p, AEVShape.of(4, True).ldx))
    check_run(r, {})
    n, n_real = p.n, r.grid()["n_real"]
    ldx = r.shape.ldx
    so = r.o["sorted_orig"]
    ref_pos, ref_shift, moved = Guarded(4 * n), Guarded(4 * n), Guarded(1, zero=True)
    coords = torch.tensor(xyz, device=DEV)
    b = r.b
    check(L.ani_b200_verlet_positions(0, coords.data_ptr(), b["grid"].ptr, b["sorted_orig"].ptr, n, skin,
                                      b["spos"].ptr, ref_pos.ptr, ref_shift.ptr, moved.ptr, None, 0, None, ldx, st),
          "verlet_positions")
    torch.cuda.synchronize()
    spos0 = b["spos"].inner().reshape(n, 4)
    rp, rs = ref_pos.inner().reshape(n, 4), ref_shift.inner().reshape(n, 4)
    assert (rp[:n_real] == spos0[:n_real]).all() and (rp[n_real:] == SENT).all() and (rs[n_real:] == SENT).all()
    x_sorted = xyz[so[:n_real]]
    assert (rs[:n_real, :3].view(np.float32) == spos0[:n_real, :3].view(np.float32) - x_sorted).all()
    assert (rs[:n_real, 3] == 0).all()
    sh = rs[:n_real, :3].view(np.float32)
    rng = np.random.default_rng(43)
    real = np.nonzero(sp >= 0)[0]
    half = skin / 2
    for f, want in ((0.5, 0), (0.69, 0), (0.71, 2), (1.02, 3), (math.nan, 3)):
        d = rng.normal(size=(n, 3))
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        disp = d * rng.uniform(0.0, 0.6 * half, (n, 1))
        one = real[rng.integers(len(real))]
        disp[one] = d[one] * (half * f if not math.isnan(f) else 1.0)
        x2 = (xyz.astype(np.float64) + disp).astype(np.float32)
        if math.isnan(f):
            x2[one, 1] = np.nan
        if f == 0.69:
            x2 = (xyz.astype(np.float64) + d * 0.69 * half).astype(np.float32)   # every atom near the limit
        c2 = torch.tensor(x2, device=DEV)
        moved.full[GUARD] = 0
        b["spos"].full[GUARD + 4 * n_real:GUARD + 4 * n] = SENT
        zero = Guarded(3 * n)
        b["aev_blocks"].full[GUARD + ldx // 32 + 2] = 1
        check(L.ani_b200_verlet_positions(1, c2.data_ptr(), b["grid"].ptr, b["sorted_orig"].ptr, n, skin,
                                          b["spos"].ptr, ref_pos.ptr, ref_shift.ptr, moved.ptr, zero.ptr, 3 * n,
                                          b["aev_blocks"].ptr, ldx, st), "verlet_positions")
        torch.cuda.synchronize()
        assert int(moved.inner()[0]) == want, (f, int(moved.inner()[0]))
        for buf in (ref_pos, ref_shift, moved, zero, b["spos"], b["aev_blocks"]):
            assert buf.guards_ok()
        assert (zero.inner() == 0).all()
        assert b["aev_blocks"].inner()[ldx // 32 + 2] == 0
        sp1 = b["spos"].inner().reshape(n, 4)
        assert (sp1[n_real:] == SENT).all(), "rows at or beyond n_real were written"
        expect = x2[so[:n_real]] + sh
        got = sp1[:n_real, :3].view(np.float32)
        assert ((got == expect) | (np.isnan(got) & np.isnan(expect))).all()
        assert (sp1[:n_real, 3] == rp[:n_real, 3]).all()
        if want == 0:
            # the grid built with cutoff + skin still reaches every pair within the true cutoff
            g = grid_ref(p)
            k_all = np.zeros((n, 3), dtype=np.int64)
            k_all[so[:n_real]] = np.round(-sh.astype(np.float64) @ g.inv).astype(np.int64)
            lo_r, hi_r, code, _, _, _ = ranges_ref(g, r.o["bin_start"])
            pairs = brute_pairs(x2, g.cell, CUTOFF, real)
            o2s = r.o["orig_to_sorted"]
            missing, excused = completeness(g, pairs, k_all, r.o["sbin"][o2s], o2s, (lo_r, hi_r, code), CUTOFF)
            assert missing == 0, (f, missing)
            report(f"verlet displacement {f} x skin/2", [r.form], {"excused pairs": excused})


# ------------------------------------------------------------------------------------------------------------------
# energy reduction
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("npc", [1, 17, 32, 33])
def test_reduce_energies(npc):
    from torchani_b200._lib import MLPModel, check, lib
    L = lib()
    st = torch.cuda.current_stream().cuda_stream
    rng = np.random.default_rng(npc)
    n_conf = max(3, 600 // npc)
    sp = rng.integers(0, 4, (n_conf, npc))
    sp[rng.random((n_conf, npc)) < 0.15] = -1
    sp[1] = -1                                            # a fully padded conformer
    xyz = np.zeros((n_conf, npc, 3), np.float32)
    for c in range(n_conf):
        xyz[c] = in_cell(np.eye(3) * 9.0, npc, seed=c, min_dist=1.0) if npc > 1 else 0.0
    M = 5
    sae = torch.tensor([-0.5, -38.1, -54.7, -75.2], dtype=torch.float64, device=DEV)
    for (rank, world) in ((0, 1), (1, 3), (2, 3)):
        n = n_conf * npc
        lo, hi = n * rank // world, n * (rank + 1) // world
        p = Problem(f"reduce {npc}", xyz.reshape(-1, 3), sp.reshape(-1).astype(np.int32), None, 4, n_conf=n_conf,
                    lo=lo, hi=hi)
        r = Run(p, expected_form(p, AEVShape.of(4, True).ldx), calls=1)
        rows_cap = r.rows_cap
        e_member = torch.tensor(rng.normal(0.0, 0.3, (M, rows_cap)) + rng.choice([-1.0, 1.0], (M, rows_cap)) * 2.0,
                                dtype=torch.float32, device=DEV)
        for scales in ([1.0 / M] * M, [0.5, 0.0, 0.5, 0.0, 0.0]):
            model = MLPModel()
            model.num_members = M
            for m in range(M):
                model.member_scale[m] = scales[m]
            for with_sae, with_atomic in ((True, True), (False, False)):
                atomic = Guarded(n) if with_atomic else None
                member = Guarded(M * n) if with_atomic else None
                energies = Guarded(2 * n_conf)
                species = torch.tensor(p.species, device=DEV)
                check(L.ani_b200_reduce_energies(
                    C.byref(model), e_member.data_ptr(), rows_cap, r.b["row_of"].ptr, r.b["orig_to_sorted"].ptr,
                    species.data_ptr(), n, lo, hi, n_conf, npc, sae.data_ptr() if with_sae else None,
                    atomic.ptr if atomic else None, member.ptr if member else None, energies.ptr, st),
                    "reduce_energies")
                torch.cuda.synchronize()
                for buf in (atomic, member, energies):
                    if buf is not None:
                        assert buf.guards_ok()
                em = e_member.double().cpu().numpy()
                o2s, row_of = r.o["orig_to_sorted"], r.o["row_of"]
                spf = p.species
                i = o2s
                owned = (spf >= 0) & (i >= lo) & (i < hi)
                rows = np.where(owned, row_of[np.clip(i, 0, n - 1)], 0)
                terms = np.array(scales)[:, None] * em[:, rows]                # (M, n)
                e = np.where(owned, terms.sum(0), 0.0)
                bar_atom = np.where(owned, M * U * np.abs(terms).sum(0), 0.0)
                s64 = sae.cpu().numpy()
                contrib = e + (np.where(owned, s64[np.clip(spf, 0, 3)], 0.0) if with_sae else 0.0)
                want = contrib.reshape(n_conf, npc).sum(1)
                bar = bar_atom.reshape(n_conf, npc).sum(1) + 1e-12 * np.abs(contrib).reshape(n_conf, npc).sum(1)
                got = energies.inner().view(np.float64)
                assert (np.abs(got - want) <= bar).all(), (npc, rank, world, scales, np.abs(got - want).max())
                if with_atomic:
                    at = atomic.inner().view(np.float32).astype(np.float64)
                    assert (np.abs(at - e) <= bar_atom).all()
                    assert (at[~owned] == 0).all()
                    mem = member.inner().view(np.float32).reshape(M, n)
                    assert (mem[:, owned] == e_member.cpu().numpy()[:, rows[owned]]).all()
                    assert (mem[:, ~owned] == 0).all()
        # 1, 17 and 33 atoms per conformer: warps that straddle conformers (the non-uniform branch of the kernel)
        straddle = any(len(set((np.arange(32 * w, min(32 * w + 32, n)) // npc).tolist())) > 1
                       for w in range(-(-n // 32)))
        assert straddle == (npc != 32)


# ------------------------------------------------------------------------------------------------------------------
# half neighbour lists (build_cells + k_half_list)
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["skewed", "sheared", "one_bucket_s8", "width_edges", "dilute_64", "open_far",
                                  "batch"])
def test_half_neighbor_lists(name):
    from torchani_b200 import neighbors
    p = build_problem(name)
    sp = torch.tensor(p.species, dtype=torch.long, device=DEV).view(p.n_conf, -1)
    co = torch.tensor(p.coords, device=DEV).view(p.n_conf, -1, 3)
    if p.mode == 1:
        nb = neighbors.all_pairs(p.cutoff, sp, co)
    elif p.pbc:
        nb = neighbors.cell_list(p.cutoff, sp, co, torch.tensor(p.cell, device=DEV),
                                 torch.tensor([True, True, True], device=DEV))
    else:
        nb = neighbors.cell_list(p.cutoff, sp, co)
    torch.cuda.synchronize()
    i0, i1 = (t.cpu().numpy() for t in nb.indices)
    diff = nb.diff_vectors.cpu().numpy().astype(np.float64)
    dist = nb.distances.cpu().numpy().astype(np.float64)
    x = p.coords.astype(np.float64)
    cell = p.cell.astype(np.float64) if p.pbc else np.eye(3)
    raw = x[i0] - x[i1]
    mf = (diff - raw) @ np.linalg.inv(cell)
    m = np.round(mf).astype(np.int64)
    if p.pbc:
        assert np.abs(mf - m).max(initial=0) < 1e-3
    else:
        assert (m == 0).all()
    # each unordered pair once, at the lower input index (self-image pairs: the upper half of the image codes, i.e. a
    # lexicographically negative lattice shift on the difference vector)
    assert ((i0 < i1) | ((i0 == i1) & ~lex_pos(m) & m.any(1))).all()
    got = canon(i0, i1, m)
    assert len(got) == len(i0)
    real = np.nonzero(p.species >= 0)[0]
    groups = np.arange(p.n) // p.n_per_conf if p.mode == 1 else None
    a, c, n_, d = brute_pairs(p.coords, cell if p.pbc else None, p.cutoff, real, groups)
    inside = d <= p.cutoff
    want = canon(a[inside], c[inside], -n_[inside])
    edge = canon(a[np.abs(d - p.cutoff) < EDGE], c[np.abs(d - p.cutoff) < EDGE], -n_[np.abs(d - p.cutoff) < EDGE])
    bad = (got ^ want) - edge
    assert not bad, f"{len(bad)} pairs differ, e.g. {sorted(bad)[:4]}"
    ref = raw + m @ cell
    M = max(float(np.abs(x[real]).max()), float(np.abs(cell).max()) * max(1, int(np.abs(m).max(initial=0)) + 1))
    tol = 8 * ulp(M)
    assert np.abs(diff - ref).max(initial=0) <= tol
    assert np.abs(dist - np.linalg.norm(ref, axis=1)).max(initial=0) <= tol
    report(f"half list {name}", ["build_cells"], {"pairs": len(got), "excused pairs": len((got ^ want) & edge)})


# ------------------------------------------------------------------------------------------------------------------
# the forms chosen once per process
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("var", ["ANI_B200_PREP_FUSED=0", "ANI_B200_PREP_CLUSTER_CTAS=8"])
def test_process_wide_forms(var):
    """The five-launch preparation and the 8-CTA cluster are function statics: re-run this file's GPU tests in a
    child process with the switch set, under a timeout."""
    k, v = var.split("=")
    child_env = dict(os.environ, **{k: v})
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
        "-m", "pytest", os.path.abspath(__file__), "-q", "-m", "gpu", "-k", "not process_wide and not water40k",
        "-p", "no:cacheprovider"]
    res = subprocess.run(cmd, cwd=ROOT, env=child_env, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stdout[-4000:] + res.stderr[-2000:]
    assert " passed" in res.stdout and " failed" not in res.stdout
