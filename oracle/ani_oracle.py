"""CPU oracle for the ANI energy+force hot path.

TEST INFRASTRUCTURE ONLY.  This file is the checker, never the product: only
``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import it.  Nothing under ``torchani_b200/`` does.

It is a from-scratch restatement (plain torch on the CPU, any float dtype, forces
through ``torch.autograd`` exactly like the reference takes them) of the
algorithm in aiqm/torchani @ 800dcdd.  Each function cites the reference
file:line it follows (paths relative to /root/reference/torchani/).

Parity pin: ``oracle/make_golden.py`` imports the real reference in the build
container and checks this restatement against it (fp64, max-abs ~1e-13) before
writing ``tests/golden/*.npz``; ``tests/test_oracle_golden.py`` re-checks the
oracle against those committed vectors everywhere (no reference needed).
"""
from __future__ import annotations

import math
import typing as tp

import numpy as np
import torch
from torch import Tensor

# --------------------------------------------------------------------------------------
# Constants (aev/_computer.py:499-600, aev/_terms.py:188-207,345-366, utils.py:101-107)
# --------------------------------------------------------------------------------------


def _linspace(start: float, stop: float, steps: int) -> tp.Tuple[float, ...]:
    # utils.py:101-107 -- endpoint excluded, pure python floats
    return tuple(start + ((stop - start) / steps) * j for j in range(steps))


class AEVSpec(tp.NamedTuple):
    """The constants that define an ANI-style AEV (radial + angular)."""

    num_species: int
    rcr: float
    rca: float
    eta_r: float
    shf_r: tp.Tuple[float, ...]
    eta_a: float
    zeta: float
    shf_a: tp.Tuple[float, ...]
    shf_z: tp.Tuple[float, ...]
    cutoff_fn: str = "cosine"  # or "smooth"

    @property
    def radial_len(self) -> int:
        return self.num_species * len(self.shf_r)

    @property
    def angular_sub(self) -> int:
        return len(self.shf_a) * len(self.shf_z)

    @property
    def angular_len(self) -> int:
        return self.num_species * (self.num_species + 1) // 2 * self.angular_sub

    @property
    def out_dim(self) -> int:
        return self.radial_len + self.angular_len


def aev_spec_2x(num_species: int = 7, cutoff_fn: str = "cosine") -> AEVSpec:
    # aev/_computer.py:551-600
    n_sec = 4
    a0 = math.pi / n_sec / 2
    return AEVSpec(
        num_species, 5.1, 3.5, 19.7, _linspace(0.8, 5.1, 16), 12.5, 14.1,
        _linspace(0.8, 3.5, 8), _linspace(a0, math.pi + a0, n_sec), cutoff_fn,
    )


def aev_spec_1x(num_species: int = 4, cutoff_fn: str = "cosine") -> AEVSpec:
    # aev/_computer.py:499-548
    n_sec = 8
    a0 = math.pi / n_sec / 2
    return AEVSpec(
        num_species, 5.2, 3.5, 16.0, _linspace(0.9, 5.2, 16), 8.0, 32.0,
        _linspace(0.9, 3.5, 4), _linspace(a0, math.pi + a0, n_sec), cutoff_fn,
    )


SYMBOLS_2X = ("H", "C", "N", "O", "S", "F", "Cl")
SYMBOLS_1X = ("H", "C", "N", "O")
ATOMIC_NUMBERS = {"H": 1, "C": 6, "N": 7, "O": 8, "F": 9, "S": 16, "Cl": 17}

# nn/_containers.py:507-570 -- hidden layer widths per element
DIMS_2X = {
    "H": (256, 192, 160), "C": (224, 192, 160), "N": (192, 160, 128), "O": (192, 160, 128),
    "S": (160, 128, 96), "F": (160, 128, 96), "Cl": (160, 128, 96),
}
DIMS_1X = {"H": (160, 128, 96), "C": (144, 112, 96), "N": (128, 112, 96), "O": (128, 112, 96)}

# constants.py:88-96 (wb97x-631gd GSAEs, Hartree), used as self energies by models.ANI2x
GSAES_WB97X_631GD = {
    "H": -0.4993212, "C": -37.8338334, "N": -54.5732825, "O": -75.0424519,
    "S": -398.0814169, "F": -99.6949007, "Cl": -460.1167008,
}

CELU_ALPHA = 0.1  # nn/_core.py:163-167 (TightCELU)


# --------------------------------------------------------------------------------------
# Deterministic synthetic weights (pretrained ANI weights are not available offline).
# numpy's PCG64 stream is stable across numpy versions, so the same (seed, dims) gives
# the same weights in the golden-vector generator, in the tests and on the GPU box.
# --------------------------------------------------------------------------------------


def make_weights(
    symbols: tp.Sequence[str],
    dims: tp.Dict[str, tp.Tuple[int, ...]],
    in_dim: int,
    members: int,
    seed: int = 1234,
    dtype: torch.dtype = torch.float32,
) -> tp.List[tp.Dict[str, tp.List[tp.Tuple[Tensor, Tensor]]]]:
    """weights[member][symbol] = [(W [out,in], b [out]) for each of the 4 Linear layers].

    Layout follows ``torch.nn.Linear`` (nn/_core.py:117-149).  Values are uniform in
    +-1/sqrt(fan_in) (the torch default init range); biases get a small offset so that
    CELU sees both signs.
    """
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(members):
        per_sym = {}
        for s in symbols:
            layer_dims = (in_dim,) + tuple(dims[s]) + (1,)
            layers = []
            for fan_in, fan_out in zip(layer_dims[:-1], layer_dims[1:]):
                bound = 1.0 / math.sqrt(fan_in)
                w = rng.uniform(-bound, bound, size=(fan_out, fan_in))
                b = rng.uniform(-bound, bound, size=(fan_out,))
                layers.append((torch.tensor(w, dtype=dtype), torch.tensor(b, dtype=dtype)))
            per_sym[s] = layers
        out.append(per_sym)
    return out


# --------------------------------------------------------------------------------------
# Cutoff functions (cutoffs.py:70-101)
# --------------------------------------------------------------------------------------


def cutoff_cosine(d: Tensor, rc: float) -> Tensor:
    # cutoffs.py:80-81
    return 0.5 * torch.cos(d * (math.pi / rc)) + 0.5


def cutoff_smooth(d: Tensor, rc: float, order: int = 2, eps: float = 1e-10) -> Tensor:
    # cutoffs.py:99-101
    return torch.exp(1 - 1 / (1 - (d / rc) ** order).clamp(min=eps))


def _cutoff(name: str):
    return {"cosine": cutoff_cosine, "smooth": cutoff_smooth}[name]


# --------------------------------------------------------------------------------------
# Neighbour lists (neighbors.py)
# --------------------------------------------------------------------------------------


class Neighbors(tp.NamedTuple):
    # neighbors.py:13-18
    indices: Tensor  # (2, P) int64, index the flattened (C*A) atoms
    distances: Tensor  # (P,)
    diff_vectors: Tensor  # (P, 3) = x[idx0] - x[idx1] + shift


def map_to_central(coords: Tensor, cell: Tensor, pbc: Tensor) -> Tensor:
    # utils.py:237-255
    frac = coords @ torch.inverse(cell)
    frac = frac - frac.floor() * pbc.to(frac.dtype)
    return frac @ cell


def _screen(
    cutoff: float, species: Tensor, coords: Tensor, idx: Tensor, shifts: tp.Optional[Tensor]
) -> Neighbors:
    """neighbors.py:64-113 (narrow_down): drop dummy pairs, keep d <= cutoff (inclusive,
    screened on detached coords), then recompute diff/dist with autograd."""
    flat_sp = species.reshape(-1)
    keep = (flat_sp[idx[0]] != -1) & (flat_sp[idx[1]] != -1)
    idx = idx[:, keep]
    if shifts is not None:
        shifts = shifts[keep]
    x = coords.reshape(-1, 3)
    with torch.no_grad():
        d = x[idx[0]] - x[idx[1]]
        if shifts is not None:
            d = d + shifts
        inside = d.norm(2, -1) <= cutoff
    idx = idx[:, inside]
    diff = x[idx[0]] - x[idx[1]]
    if shifts is not None:
        diff = diff + shifts[inside]
    return Neighbors(idx, diff.norm(2, -1), diff)


def _image_shifts(cutoff: float, cell: Tensor, pbc: Tensor) -> Tensor:
    """neighbors.py:250-275: integer lattice shifts of the half-space (the centre image
    and the mirrored half are excluded) that can hold a neighbour within ``cutoff``."""
    inv_d = torch.inverse(cell).t().norm(2, -1)
    reps = torch.ceil(cutoff * inv_d).long()
    reps = torch.where(pbc, reps, torch.zeros_like(reps)).tolist()
    out = []
    for a in range(0, reps[0] + 1):
        for b in range(-reps[1], reps[1] + 1):
            for c in range(-reps[2], reps[2] + 1):
                if a > 0 or (a == 0 and (b > 0 or (b == 0 and c > 0))):
                    out.append((a, b, c))
    return torch.tensor(out, dtype=torch.long).reshape(-1, 3)


def all_pairs(
    cutoff: float, species: Tensor, coords: Tensor,
    cell: tp.Optional[Tensor] = None, pbc: tp.Optional[Tensor] = None,
) -> Neighbors:
    """neighbors.py:187-242.  O(A^2) per molecule; with PBC every half-space image shift is
    paired with every ordered (i, j) (including i == j)."""
    C, A = species.shape
    tri = torch.triu_indices(A, A, 1)
    if pbc is not None:
        assert cell is not None and C == 1
        sh = _image_shifts(cutoff, cell.detach(), pbc)
        ar = torch.arange(A)
        full = torch.cartesian_prod(torch.arange(sh.shape[0]), ar, ar)
        idx = torch.cat([tri, full[:, 1:].t()], dim=1)
        shift_idx = torch.cat([torch.zeros(tri.shape[1], 3, dtype=torch.long), sh[full[:, 0]]])
        shifts = shift_idx.to(cell.dtype) @ cell
        return _screen(cutoff, species, map_to_central(coords, cell, pbc), idx, shifts)
    idx = (tri.unsqueeze(1) + A * torch.arange(C).view(1, -1, 1)).reshape(2, -1)
    return _screen(cutoff, species, coords, idx, None)


# half-surround bucket offsets (self bucket handled separately); any half of the 26
# neighbours that is closed under "exactly one of +o/-o" works (neighbors.py:510-550).
_HALF_OFFSETS = [
    (a, b, c) for a in (-1, 0, 1) for b in (-1, 0, 1) for c in (-1, 0, 1)
    if a > 0 or (a == 0 and (b > 0 or (b == 0 and c > 0)))
]


def cell_list(
    cutoff: float, species: Tensor, coords: Tensor,
    cell: tp.Optional[Tensor] = None, pbc: tp.Optional[Tensor] = None,
) -> Neighbors:
    """neighbors.py:366-507: bucket the (single) conformer into a grid with >= 1 bucket per
    cutoff (neighbors.py:618-662), pair every bucket with itself and with 13 half-surround
    buckets (periodic wrap gives the image shift), then screen by distance."""
    assert species.shape[0] == 1
    A = species.shape[1]
    x = coords.detach().reshape(-1, 3)
    if pbc is not None:
        assert cell is not None and bool(pbc.all())
        cellm = cell.detach()
    else:
        # neighbors.py:116-137,391-394: bounding cell with 2*cutoff padding -> no images
        eps = 2 * cutoff + 1e-3
        lo = x.min(0).values - eps
        x = x - lo
        cellm = torch.diag(x.max(0).values + eps)
    lengths = torch.linalg.norm(cellm, dim=0)
    grid = torch.div(lengths, cutoff + 1e-5, rounding_mode="floor").long()
    if pbc is not None and bool((grid == 0).any()):
        raise RuntimeError("Cell is too small to perform pbc calculations")
    grid = grid.clamp(min=1)
    frac = torch.remainder(x @ torch.inverse(cellm), 1.0)
    g3 = (frac * grid).floor().long()
    g3 = torch.minimum(g3, grid - 1)
    flat = (g3[:, 0] * grid[1] + g3[:, 1]) * grid[2] + g3[:, 2]
    ncell = int(grid.prod())
    order = torch.argsort(flat, stable=True)
    counts = torch.bincount(flat, minlength=ncell)
    start = torch.cumsum(counts, 0) - counts
    m = int(counts.max())
    slot = torch.arange(m)
    # padded occupancy table: occ[c, k] = atom index or -1
    occ = torch.full((ncell, m), -1, dtype=torch.long)
    valid = slot.view(1, -1) < counts.view(-1, 1)
    occ[valid] = order
    c3 = torch.stack(torch.meshgrid(*[torch.arange(int(g)) for g in grid], indexing="ij"), -1).view(-1, 3)
    pair_i, pair_j, pair_s = [], [], []
    # within-bucket pairs
    a = occ.unsqueeze(2).expand(-1, -1, m)
    b = occ.unsqueeze(1).expand(-1, m, -1)
    keep = (a >= 0) & (b >= 0) & (slot.view(1, -1, 1) < slot.view(1, 1, -1))
    pair_i.append(a[keep]); pair_j.append(b[keep])
    pair_s.append(torch.zeros(int(keep.sum()), 3, dtype=torch.long))
    for off in _HALF_OFFSETS:
        n3 = c3 + torch.tensor(off)
        wrap = torch.div(n3, grid, rounding_mode="floor")  # -1, 0, +1 images
        if pbc is None:
            inside = (wrap == 0).all(-1)
        else:
            inside = torch.ones(ncell, dtype=torch.bool)
        n3m = n3 - wrap * grid
        nflat = (n3m[:, 0] * grid[1] + n3m[:, 1]) * grid[2] + n3m[:, 2]
        b = occ[nflat].unsqueeze(1).expand(-1, m, -1)
        keep = (a >= 0) & (b >= 0) & inside.view(-1, 1, 1)
        pair_i.append(a[keep]); pair_j.append(b[keep])
        # x_i - (x_j + wrap*cell)  ->  shift on the difference vector is -wrap
        pair_s.append((-wrap).view(-1, 1, 1, 3).expand(-1, m, m, -1)[keep])
    idx = torch.stack([torch.cat(pair_i), torch.cat(pair_j)])
    if pbc is not None:
        shifts = torch.cat(pair_s).to(cell.dtype) @ cell
        return _screen(cutoff, species, map_to_central(coords, cell.detach(), pbc), idx, shifts)
    return _screen(cutoff, species, coords, idx, None)


def neighborlist(kind: str, cutoff, species, coords, cell=None, pbc=None) -> Neighbors:
    if kind == "all_pairs":
        return all_pairs(cutoff, species, coords, cell, pbc)
    if kind == "cell_list":
        return cell_list(cutoff, species, coords, cell, pbc)
    raise ValueError(kind)


# --------------------------------------------------------------------------------------
# AEV (aev/_terms.py, aev/_computer.py:274-350)
# --------------------------------------------------------------------------------------


def triu_index(num_species: int) -> Tensor:
    # aev/_computer.py:184-191: row-major upper triangle, symmetric lookup
    s1, s2 = torch.triu_indices(num_species, num_species).unbind(0)
    ret = torch.zeros(num_species, num_species, dtype=torch.long)
    ret[s1, s2] = torch.arange(s1.shape[0])
    ret[s2, s1] = torch.arange(s1.shape[0])
    return ret


def _f32const(values, dtype) -> Tensor:
    """The reference registers eta/zeta/shifts as float32 buffers (aev/_terms.py:153-156,
    288-292); ``.double()`` keeps the float32-rounded values.  Those are the canonical
    constants, so every dtype goes through float32 first."""
    return torch.tensor(values, dtype=torch.float32).to(dtype)


def f32(v: float) -> float:
    """float32-rounded python float (canonical value of an AEV constant)."""
    return float(np.float32(v))


def radial_terms(spec: AEVSpec, d: Tensor) -> Tensor:
    # aev/_terms.py:99-104,186: 0.25*exp(-eta (d-ShfR)^2) * fc(d)
    shf = _f32const(spec.shf_r, d.dtype)
    eta = _f32const([spec.eta_r], d.dtype)
    g = 0.25 * torch.exp(-eta * (d.view(-1, 1) - shf.view(1, -1)) ** 2)
    return g * _cutoff(spec.cutoff_fn)(d, spec.rcr).view(-1, 1)


def angular_terms(spec: AEVSpec, d1: Tensor, d2: Tensor, v1: Tensor, v2: Tensor) -> Tensor:
    # aev/_terms.py:34-55 (cos of the angle, clamp 1e-10), :324-325 (radial factor),
    # :341-343 (0.95 inside acos, 2*((1+cos)/2)^zeta); feature order ShfA major, ShfZ minor.
    fc = _cutoff(spec.cutoff_fn)
    shf_a = _f32const(spec.shf_a, d1.dtype)
    shf_z = _f32const(spec.shf_z, d1.dtype)
    eta_a = _f32const([spec.eta_a], d1.dtype)
    zeta = _f32const([spec.zeta], d1.dtype)
    cos = (v1 * v2).sum(-1) / torch.clamp(d1 * d2, min=1e-10)
    ang = torch.acos(0.95 * cos)
    f1 = 2 * ((1 + torch.cos(ang.view(-1, 1) - shf_z.view(1, -1))) / 2) ** zeta
    f2 = torch.exp(-eta_a * (((d1 + d2) / 2).view(-1, 1) - shf_a.view(1, -1)) ** 2)
    terms = (f2.unsqueeze(2) * f1.unsqueeze(1)).reshape(d1.shape[0], -1)
    return terms * (fc(d1, spec.rca) * fc(d2, spec.rca)).view(-1, 1)


def aev_from_neighbors(
    spec: AEVSpec, species: Tensor, nb: Neighbors, triple_chunk: int = 2_000_000
) -> Tensor:
    """aev/_computer.py:274-350 + neighbors.py:968-1002, restated with a padded per-atom
    neighbour table instead of sort/unique/tril_indices.  Returns (C, A, out_dim)."""
    C, A = species.shape
    S = spec.num_species
    flat_sp = species.reshape(-1)
    dtype = nb.distances.dtype
    n_at = C * A
    # ---- radial: each half pair feeds both ends (aev/_computer.py:337-350)
    rt = radial_terms(spec, nb.distances)
    nr = len(spec.shf_r)
    radial = torch.zeros(n_at * S, nr, dtype=dtype)
    i0, i1 = nb.indices[0], nb.indices[1]
    radial = radial.index_add(0, i0 * S + flat_sp[i1], rt)
    radial = radial.index_add(0, i1 * S + flat_sp[i0], rt)
    radial = radial.view(n_at, S * nr)
    # ---- angular: neighbours within Rca (neighbors.py:46-55), directed table
    close = nb.distances <= spec.rca
    i0, i1 = i0[close], i1[close]
    d = nb.distances[close]
    v = nb.diff_vectors[close]
    cen = torch.cat([i0, i1])
    oth = torch.cat([i1, i0])
    dd = torch.cat([d, d])
    vv = torch.cat([v, -v])  # same orientation convention on both sides of a triple
    order = torch.argsort(cen, stable=True)
    cen, oth, dd, vv = cen[order], oth[order], dd[order], vv[order]
    counts = torch.bincount(cen, minlength=n_at)
    start = torch.cumsum(counts, 0) - counts
    nsub = spec.angular_sub
    npairs = S * (S + 1) // 2
    angular = torch.zeros(n_at * npairs, nsub, dtype=dtype)
    tri = triu_index(S)
    m = int(counts.max()) if counts.numel() > 0 else 0
    if m >= 2:
        ja, jb = torch.triu_indices(m, m, 1).unbind(0)
        per_atom = ja.shape[0]
        step = max(1, triple_chunk // per_atom)
        atoms = torch.nonzero(counts >= 2).view(-1)
        for lo in range(0, atoms.shape[0], step):
            at = atoms[lo:lo + step]
            ok = (jb.view(1, -1) < counts[at].view(-1, 1))
            ea = (start[at].view(-1, 1) + ja.view(1, -1))[ok]
            eb = (start[at].view(-1, 1) + jb.view(1, -1))[ok]
            central = at.view(-1, 1).expand(-1, per_atom)[ok]
            terms = angular_terms(spec, dd[ea], dd[eb], vv[ea], vv[eb])
            index = central * npairs + tri[flat_sp[oth[ea]], flat_sp[oth[eb]]]
            angular = angular.index_add(0, index, terms)
    angular = angular.view(n_at, npairs * nsub)
    return torch.cat([radial, angular], dim=-1).view(C, A, spec.out_dim)


# --------------------------------------------------------------------------------------
# Networks (nn/_core.py:117-167, nn/_containers.py:377-421,608-651), SAE (sae.py:54-64)
# --------------------------------------------------------------------------------------


def atomic_network(x: Tensor, layers) -> Tensor:
    # nn/_core.py:146-149: celu(alpha=0.1) after every layer but the last
    for w, b in layers[:-1]:
        x = torch.nn.functional.celu(torch.addmm(b, x, w.t()), alpha=CELU_ALPHA)
    w, b = layers[-1]
    return torch.addmm(b, x, w.t())


def member_atomic_energies(symbols, weights_m, species: Tensor, aev: Tensor) -> Tensor:
    """nn/_containers.py:407-421 for one ensemble member -> (C, A) atomic scalars."""
    C, A = species.shape
    flat = species.reshape(-1)
    x = aev.reshape(C * A, -1)
    out = torch.zeros(C * A, dtype=aev.dtype)
    for i, s in enumerate(symbols):
        sel = torch.nonzero(flat == i).view(-1)
        if sel.numel():
            layers = [(w.to(aev.dtype), b.to(aev.dtype)) for w, b in weights_m[s]]
            out = out.index_add(0, sel, atomic_network(x[sel], layers).view(-1))
    return out.view(C, A)


def ensemble_atomic_energies(symbols, weights, species, aev, members=None) -> Tensor:
    """(M_active, C, A) per-member atomic energies (nn/_containers.py:638-651)."""
    members = list(range(len(weights))) if members is None else members
    return torch.stack([member_atomic_energies(symbols, weights[j], species, aev) for j in members])


def self_energies(symbols, sae: tp.Dict[str, float], species: Tensor, dtype) -> Tensor:
    # sae.py:54-64 -> (C, A) with 0 for padding
    table = torch.tensor([sae[s] for s in symbols], dtype=dtype)
    e = table[species.clamp(min=0)]
    return e.masked_fill(species == -1, 0.0)


class Model(tp.NamedTuple):
    spec: AEVSpec
    symbols: tp.Tuple[str, ...]
    weights: list  # make_weights(...)
    sae: tp.Dict[str, float]
    neighborlist: str = "cell_list"


def ani2x_model(seed: int = 1234, members: int = 8, neighborlist: str = "cell_list") -> Model:
    spec = aev_spec_2x()
    return Model(spec, SYMBOLS_2X, make_weights(SYMBOLS_2X, DIMS_2X, spec.out_dim, members, seed),
                 GSAES_WB97X_631GD, neighborlist)


def ani1x_model(seed: int = 1234, members: int = 8, neighborlist: str = "all_pairs") -> Model:
    spec = aev_spec_1x()
    sae = {s: GSAES_WB97X_631GD[s] for s in SYMBOLS_1X}
    return Model(spec, SYMBOLS_1X, make_weights(SYMBOLS_1X, DIMS_1X, spec.out_dim, members, seed),
                 sae, neighborlist)


def compute(
    model: Model, species: Tensor, coords: Tensor,
    cell: tp.Optional[Tensor] = None, pbc: tp.Optional[Tensor] = None,
    forces: bool = True, members: tp.Optional[tp.List[int]] = None, stress: bool = False,
) -> tp.Dict[str, Tensor]:
    """arch.py:302-381 (+ grad.py:42-64 for forces).  ``species`` are element indices
    (0..S-1, -1 padding).  Returns aev, per-member atomic NN energies, NN energies (C,),
    total energies (C,) and forces (C, A, 3)."""
    coords = coords.detach().clone().requires_grad_(forces)
    scaling = None
    coords_in = coords
    if stress:
        # ase.py:110-121 ("scaling" stress): coordinates and cell are multiplied by a 3x3 matrix that
        # starts as the identity; stress = dE/d(scaling) / volume (ase.py:170-173)
        assert cell is not None and pbc is not None, "stress needs a periodic cell"
        scaling = torch.eye(3, dtype=coords.dtype, requires_grad=True)
        coords = coords @ scaling
        cell = cell @ scaling
    nb = neighborlist(model.neighborlist, model.spec.rcr, species, coords, cell, pbc)
    aev = aev_from_neighbors(model.spec, species, nb)
    e_m = ensemble_atomic_energies(model.symbols, model.weights, species, aev, members)
    atomic_nn = e_m.mean(0)
    e_nn = atomic_nn.sum(-1)
    e_sae = self_energies(model.symbols, model.sae, species, coords.dtype).sum(-1)
    out = {
        "aev": aev.detach(), "member_atomic": e_m.detach(), "atomic_nn": atomic_nn.detach(),
        "energy_nn": e_nn.detach(), "energy": (e_nn + e_sae).detach(),
        "num_pairs": torch.tensor(nb.indices.shape[1]),
    }
    if forces:
        out["forces"] = -torch.autograd.grad(e_nn.sum(), coords_in, retain_graph=stress)[0]
    if stress:
        volume = torch.det(cell.detach()).abs()
        out["stress"] = (torch.autograd.grad(e_nn.sum(), scaling)[0] / volume).detach()   # Hartree / A^3
    return out


# --------------------------------------------------------------------------------------
# A second, loop-level restatement for tiny systems (pure python over atoms/triples) that
# follows the per-term formulas directly (SURVEY appendix A; aev.cu:427-461,817-828).
# Used only to cross-check the vectorised oracle above on a handful of atoms.
# --------------------------------------------------------------------------------------


def aev_loops(spec: AEVSpec, species: tp.Sequence[int], coords: np.ndarray,
              cell: tp.Optional[np.ndarray] = None) -> np.ndarray:
    n = len(species)
    S = spec.num_species
    nr, na, nz = len(spec.shf_r), len(spec.shf_a), len(spec.shf_z)
    out = np.zeros((n, spec.out_dim))
    spec = spec._replace(eta_r=f32(spec.eta_r), eta_a=f32(spec.eta_a), zeta=f32(spec.zeta),
                         shf_r=tuple(map(f32, spec.shf_r)), shf_a=tuple(map(f32, spec.shf_a)),
                         shf_z=tuple(map(f32, spec.shf_z)))
    images = [np.zeros(3)]
    if cell is not None:
        reps = [int(math.ceil(spec.rcr * np.linalg.norm(np.linalg.inv(cell).T[k]))) for k in range(3)]
        images = [a * cell[0] + b * cell[1] + c * cell[2]
                  for a in range(-reps[0], reps[0] + 1) for b in range(-reps[1], reps[1] + 1)
                  for c in range(-reps[2], reps[2] + 1)]
        coords = (coords @ np.linalg.inv(cell) % 1.0) @ cell

    def fc(r, rc):
        if spec.cutoff_fn == "cosine":
            return 0.5 * math.cos(math.pi * r / rc) + 0.5
        return math.exp(1 - 1 / max(1e-10, 1 - (r / rc) ** 2))

    def pair_index(a, b):
        lo, hi = min(a, b), max(a, b)
        return lo * (2 * S - lo + 1) // 2 + (hi - lo)

    for i in range(n):
        if species[i] < 0:
            continue
        nbrs = []
        for j in range(n):
            if species[j] < 0:
                continue
            for sh in images:
                if j == i and not sh.any():
                    continue
                v = coords[j] + sh - coords[i]
                r = float(np.linalg.norm(v))
                if r <= spec.rcr:
                    nbrs.append((species[j], v, r))
        for sj, v, r in nbrs:
            for m, shf in enumerate(spec.shf_r):
                out[i, sj * nr + m] += 0.25 * math.exp(-spec.eta_r * (r - shf) ** 2) * fc(r, spec.rcr)
        close = [t for t in nbrs if t[2] <= spec.rca]
        for a in range(len(close)):
            for b in range(a + 1, len(close)):
                sj, vj, rj = close[a]
                sk, vk, rk = close[b]
                cos = float(vj @ vk) / max(rj * rk, 1e-10)
                th = math.acos(0.95 * cos)
                base = spec.radial_len + pair_index(sj, sk) * na * nz
                for ia, sa in enumerate(spec.shf_a):
                    f2 = math.exp(-spec.eta_a * ((rj + rk) / 2 - sa) ** 2)
                    for iz, sz in enumerate(spec.shf_z):
                        f1 = 2 * ((1 + math.cos(th - sz)) / 2) ** spec.zeta
                        out[i, base + ia * nz + iz] += f1 * f2 * fc(rj, spec.rca) * fc(rk, spec.rca)
    return out


# --------------------------------------------------------------------------------------
# Synthetic inputs (SURVEY.md section 8d)
# --------------------------------------------------------------------------------------


def water_box(n_molecules: int, seed: int = 0, density: float = 0.1,
              dtype: torch.dtype = torch.float32):
    """Seeded synthetic periodic water box: O on a jittered cubic lattice, two H at 0.9572 A
    in random directions.  Returns (Z (1,N), elem_idx (1,N), coords (1,N,3), cell, pbc)."""
    g = torch.Generator().manual_seed(seed)
    n_atoms = 3 * n_molecules
    L = (n_atoms / density) ** (1.0 / 3.0)
    k = int(math.ceil(n_molecules ** (1.0 / 3.0)))
    grid = torch.stack(torch.meshgrid(*[torch.arange(k)] * 3, indexing="ij"), -1).view(-1, 3)
    grid = grid[:n_molecules].to(torch.float64)
    o = (grid + 0.5) * (L / k) + (torch.rand(n_molecules, 3, generator=g, dtype=torch.float64) - 0.5) * 0.3
    dirs = torch.randn(n_molecules, 2, 3, generator=g, dtype=torch.float64)
    dirs = dirs / dirs.norm(dim=-1, keepdim=True)
    h = o.unsqueeze(1) + 0.9572 * dirs
    coords = torch.cat([o.unsqueeze(1), h], 1).view(1, n_atoms, 3).to(dtype)
    z = torch.tensor([8, 1, 1]).repeat(n_molecules).view(1, -1)
    idx = torch.tensor([3, 0, 0]).repeat(n_molecules).view(1, -1)
    cell = torch.eye(3, dtype=dtype) * L
    pbc = torch.tensor([True, True, True])
    return z, idx, coords, cell, pbc


def seven_element_box(n_atoms: int = 1200, seed: int = 11, density: float = 0.1,
                      dtype: torch.dtype = torch.float64):
    """Periodic box with all seven ANI-2x elements (H C N O S F Cl): random-walk chains of 4-12 atoms in the style
    of ``conformer_batch`` (bonds 1.1-1.5 A), every contact >= 0.9 A under the minimum image, ~0.1 atoms / A^3.
    Every element pair is present, so every 32-column block of the AEV is live.
    Returns (elem_idx (1,N), coords (1,N,3), cell, pbc)."""
    rng = np.random.default_rng(seed)
    L = (n_atoms / density) ** (1.0 / 3.0)
    pts = np.zeros((0, 3))

    def free(p):
        d = pts - p
        d -= L * np.round(d / L)
        return len(pts) == 0 or float((d * d).sum(1).min()) >= 0.81

    while len(pts) < n_atoms:
        start = rng.uniform(0.0, L, 3)
        if not free(start):
            continue
        chain = [start]
        pts = np.vstack([pts, start])
        n = int(rng.integers(4, 13))
        for _ in range(50):
            if len(chain) >= n or len(pts) >= n_atoms:
                break
            d = rng.normal(size=3)
            p = (chain[int(rng.integers(0, len(chain)))] + d / np.linalg.norm(d) * rng.uniform(1.1, 1.5)) % L
            if free(p):
                chain.append(p)
                pts = np.vstack([pts, p])
    species = rng.choice(7, size=n_atoms, p=[0.45, 0.25, 0.08, 0.1, 0.04, 0.04, 0.04])
    species[rng.permutation(n_atoms)[:7]] = np.arange(7)    # every element at least once
    return (torch.tensor(species).view(1, -1), torch.tensor(pts, dtype=dtype).view(1, -1, 3),
            torch.eye(3, dtype=dtype) * L, torch.tensor([True, True, True]))


def conformer_batch(n_conf: int = 256, a_min: int = 9, a_max: int = 26, seed: int = 1234,
                    dtype: torch.dtype = torch.float32):
    """GDB-11-like padded batch (SURVEY.md 8d config 3): random-walk chains of H/C/N/O,
    bond 1.1-1.5 A, no contact below 0.8 A, -1 padding.  Returns (elem_idx (C,A), coords)."""
    rng = np.random.default_rng(seed)
    species = -np.ones((n_conf, a_max), dtype=np.int64)
    coords = np.zeros((n_conf, a_max, 3))
    for c in range(n_conf):
        n = int(rng.integers(a_min, a_max + 1))
        pts = [np.zeros(3)]
        while len(pts) < n:
            anchor = pts[int(rng.integers(0, len(pts)))]
            d = rng.normal(size=3)
            p = anchor + d / np.linalg.norm(d) * rng.uniform(1.1, 1.5)
            if min(np.linalg.norm(p - q) for q in pts) >= 0.8:
                pts.append(p)
        coords[c, :n] = np.array(pts)
        species[c, :n] = rng.choice(4, size=n, p=[0.5, 0.3, 0.1, 0.1])
    return torch.tensor(species), torch.tensor(coords, dtype=dtype)
