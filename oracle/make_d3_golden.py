"""Generate tests/golden/d3_*.npz from the REAL reference's D3 dispersion (aiqm/torchani under /root/reference).

TEST INFRASTRUCTURE ONLY; runs on the CPU where the reference sources are present.  The reference reads its C6 tables
from c6.h5 through h5py, which is not installed here, and the tables are not shipped with this project: the reference's
``_load_c6_constants`` is patched to return SEEDED SYNTHETIC tables of the real shape and structure (five references
per element, -1 where one is missing, reference coordination numbers between 0 and about 4, C6 that grows strongly
with the coordination numbers so that the chain term of the forces is large, one element pair without any valid
reference).  The covalent radii and empirical charges are the reference's own (its atomic_constants.json).

For the systems of existing golden fixtures (their inputs are reused, not stored again) it evaluates the reference's
``TwoBodyDispersionD3`` (float64; the cell list for the large single systems, all_pairs for batches and for cells
thinner than the cutoff -- the same pairs) at a cutoff of 8 A with the smooth envelope, plus one cosine case:
energies, atomic energies, autograd forces and, for periodic systems, the "scaling" stress of ase.py:110-121,170-173.
``d3_oracle`` must agree with the reference to < 1e-11 before anything is written.

  tests/golden/d3_params.npz    the module's buffers (tables, radii, charges) and its scalars
  tests/golden/d3_<system>.npz  <fn>_{energy,atomic,forces[,stress]}, cutoff
  tests/golden/d3_scan.npz      diatomic scan 1.0 - 8.4 A across the cutoff over all element pairs

Usage:  python oracle/make_d3_golden.py
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

import oracle.ani_oracle as orc          # noqa: E402
import oracle.d3_oracle as d3o           # noqa: E402
from oracle.make_golden import import_reference   # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
CUTOFF = 8.0
# B97-3c D3(BJ) constants (the functional of the reference's dispersion-corrected ANI models)
S6, S8, A1, A2 = 1.0, 1.5, 0.37, 4.1
# (system, cutoff, envelopes): water30_pbc is exactly 8.0 A wide, evaluated at 8.5 A so that it is clearly thinner
SYSTEMS = [("water999_pbc_ani2x", CUTOFF, ("smooth", "cosine")), ("sevenel_pbc_ani2x", CUTOFF, ("smooth",)),
           ("tightcell_pbc_ani2x", CUTOFF, ("smooth",)), ("6w8h_triclinic_ani2x", CUTOFF, ("smooth",)),
           ("1c17_chunk_hcnos_ani2x", CUTOFF, ("smooth",)), ("randbatch_ani2x", CUTOFF, ("smooth",)),
           ("benzene_pbc_ani2x", CUTOFF, ("smooth",)), ("water30_pbc_ani2x", 8.5, ("smooth",))]
NO_REFERENCE = ("S", "F")   # the element pair without a valid C6 reference
TOL = 1e-11


def synthetic_c6_tables(seed: int = 20261017):
    """Tables indexed by atomic number, (Z, Z, 5, 5) each, like those of c6.h5: C6ref, CN of the first and of the
    second atom per reference pair.  Symmetric as the real ones: C6ref[a, b, p, q] = C6ref[b, a, q, p] and
    CNa[a, b, p, q] = CNb[b, a, q, p]."""
    g = np.random.default_rng(seed)
    zmax = 18
    c6 = -np.ones((zmax, zmax, 5, 5))
    cna = -np.ones((zmax, zmax, 5, 5))
    cnb = -np.ones((zmax, zmax, 5, 5))
    scale = {"H": 3.0, "C": 20.0, "N": 15.0, "O": 12.0, "S": 80.0, "F": 8.0, "Cl": 90.0}
    nref = {"H": 2, "C": 5, "N": 4, "O": 3, "S": 4, "F": 2, "Cl": 3}
    cnref = {}
    for s in orc.SYMBOLS_2X:
        v = -np.ones(5)
        v[:nref[s]] = np.sort(np.concatenate([[0.0], g.uniform(0.3, 4.2, nref[s] - 1)]))
        cnref[s] = v
    for a in orc.SYMBOLS_2X:
        for b in orc.SYMBOLS_2X:
            za, zb = orc.ATOMIC_NUMBERS[a], orc.ATOMIC_NUMBERS[b]
            if za > zb or {a, b} == set(NO_REFERENCE):
                continue
            base = np.sqrt(scale[a] * scale[b])
            noise = g.uniform(0.9, 1.1, (5, 5))
            for p in range(nref[a]):
                for q in range(nref[b]):
                    val = base * (1 + 0.8 * cnref[a][p]) * (1 + 0.8 * cnref[b][q]) * noise[p, q]
                    for (x, y, i, j, ci, cj) in ((za, zb, p, q, cnref[a][p], cnref[b][q]),
                                                 (zb, za, q, p, cnref[b][q], cnref[a][p])):
                        c6[x, y, i, j], cna[x, y, i, j], cnb[x, y, i, j] = val, ci, cj
    return tuple(torch.tensor(t, dtype=torch.float32) for t in (c6, cna, cnb))


def reference_module(cutoff: float, fn: str):
    import torchani.potentials.dftd3 as dftd3
    tables = synthetic_c6_tables()
    dftd3._load_c6_constants = lambda: tables
    return dftd3.TwoBodyDispersionD3(orc.SYMBOLS_2X, S6, S8, A1, A2, cutoff=cutoff, cutoff_fn=fn).double()


def spec_of(mod, cutoff: float, fn: str) -> d3o.D3Spec:
    return d3o.D3Spec(cutoff, fn, mod._s6, mod._s8, mod._damp_fn._a1, mod._damp_fn._a2,
                      mod._damp_fn.cutoff_radii.detach(), mod.sqrt_charge_ab.detach(), mod.covalent_radii.detach(),
                      mod.precalc_coeff6.detach(), mod.precalc_coordnums_a.detach(), mod.precalc_coordnums_b.detach())


def _thin(cell, cutoff) -> bool:
    return cell is not None and bool((1 / torch.linalg.norm(torch.inverse(cell), dim=0) < cutoff).any())


def reference_results(pot, species, coords, cell, pbc, stress):
    from torchani.neighbors import all_pairs, cell_list
    x0 = coords.clone().requires_grad_(True)
    x, c, scaling = x0, cell, None
    if stress:
        scaling = torch.eye(3, dtype=torch.float64, requires_grad=True)
        x, c = x0 @ scaling, cell @ scaling
    mk = cell_list if (species.shape[0] == 1 and not _thin(cell, pot.cutoff)) else all_pairs
    atomic = pot.compute_from_neighbors(species, x, mk(pot.cutoff, species, x, c, pbc), atomic=True).energies
    energy = atomic.sum(-1)
    out = {"energy": energy.detach(), "atomic": atomic.detach(),
           "forces": -torch.autograd.grad(energy.sum(), x0, retain_graph=stress)[0]}
    if stress:
        out["stress"] = torch.autograd.grad(energy.sum(), scaling)[0] / torch.det(cell).abs()
    return out, ("cell_list" if mk is cell_list else "all_pairs")


def scan_distances() -> np.ndarray:
    return np.concatenate([np.linspace(1.0, 8.4, 38), [7.999, 8.0, 8.001]])


def main() -> None:
    import_reference()
    mod = reference_module(CUTOFF, "smooth")
    np.savez_compressed(
        os.path.join(GOLD, "d3_params.npz"), symbols=np.array(orc.SYMBOLS_2X), s6=S6, s8=S8, a1=A1, a2=A2,
        cutoff_radii=mod._damp_fn.cutoff_radii.numpy(), sqrt_charge_ab=mod.sqrt_charge_ab.numpy(),
        covalent_radii=mod.covalent_radii.numpy(), precalc_coeff6=mod.precalc_coeff6.numpy(),
        precalc_coordnums_a=mod.precalc_coordnums_a.numpy(), precalc_coordnums_b=mod.precalc_coordnums_b.numpy())

    for name, cutoff, fns in SYSTEMS:
        z = np.load(os.path.join(GOLD, name + ".npz"))
        species = torch.tensor(z["species"])
        coords = torch.tensor(z["coords"], dtype=torch.float64)
        cell = torch.tensor(z["cell"], dtype=torch.float64) if z["cell"].size else None
        pbc = torch.tensor(z["pbc"]) if z["pbc"].size else None
        rec = {"cutoff": cutoff}
        for fn in fns:
            pot = reference_module(cutoff, fn)
            ref, nl = reference_results(pot, species, coords, cell, pbc, cell is not None)
            got = d3o.compute(spec_of(pot, cutoff, fn), species, coords, cell, pbc, nl, stress=cell is not None)
            for k, v in ref.items():
                err = float((got[k] - v).abs().max())
                assert err < TOL, (name, fn, k, err)
                rec[f"{fn}_{k}"] = v.detach().numpy()
            print(f"{name} {fn} ({nl}): E = {ref['energy'].tolist()[:2]}")
        np.savez_compressed(os.path.join(GOLD, f"d3_{name}.npz"), **rec)

    # diatomic scan: every element pair (a <= b) at every distance, one two-atom conformer each
    S = len(orc.SYMBOLS_2X)
    dist = scan_distances()
    pairs = [(a, b) for a in range(S) for b in range(a, S)]
    species = torch.tensor([[a, b] for (a, b) in pairs for _ in dist])
    coords = torch.zeros(len(species), 2, 3, dtype=torch.float64)
    coords[:, 1, 0] = torch.tensor(np.tile(dist, len(pairs)))
    rec = {"species": species.numpy(), "coords": coords.numpy(), "cutoff": CUTOFF}
    for fn in ("smooth", "cosine"):
        pot = reference_module(CUTOFF, fn)
        ref, _ = reference_results(pot, species, coords, None, None, False)
        got = d3o.compute(spec_of(pot, CUTOFF, fn), species, coords, None, None, "all_pairs")
        for k, v in ref.items():
            err = float((got[k] - v).abs().max())
            assert err < TOL, ("scan", fn, k, err)
            rec[f"{fn}_{k}"] = v.detach().numpy()
    np.savez_compressed(os.path.join(GOLD, "d3_scan.npz"), **rec)
    print("wrote", sorted(f for f in os.listdir(GOLD) if f.startswith("d3_")))


if __name__ == "__main__":
    main()
