"""Generate tests/golden/ljc_*.npz from the REAL reference's Lennard-Jones and fixed-charge Coulomb potentials
(aiqm/torchani under /root/reference).

TEST INFRASTRUCTURE ONLY; runs on the CPU where the reference sources are present.  For the systems of existing golden
fixtures (their inputs are reused, not stored again) it evaluates the reference's ``LennardJones``, ``RepulsionLJ``,
``DispersionLJ``, ``FixedCoulomb`` and ``FixedMNOK`` in float64 with seeded per-element parameters: at 8 A under the
cosine envelope, at 12 A under the smooth one, and on the open systems without a cutoff (the reference's default, no
envelope).  Energies, atomic energies, autograd forces and, for periodic systems, the "scaling" stress of
ase.py:110-121,170-173.  ``lj_coulomb_oracle`` must agree with the reference to < 1e-11 before anything is written.
The 3410-atom 6W8H box keeps LennardJones and FixedCoulomb only, to keep the fixtures small.

  tests/golden/ljc_params.npz    the per-element parameters (float32 values, as the reference's buffers hold them)
  tests/golden/ljc_<system>.npz  <kind>_<fn>_<cutoff>_{energy,atomic,forces[,stress]}, cutoff "8" / "12" / "inf"

Usage:  python oracle/make_lj_coulomb_golden.py
"""
from __future__ import annotations

import math
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

import oracle.ani_oracle as orc              # noqa: E402
import oracle.lj_coulomb_oracle as lorc      # noqa: E402
from oracle.make_golden import import_reference   # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
SYSTEMS = ["water999_pbc_ani2x", "1c17_chunk_hcnos_ani2x", "randbatch_ani2x", "6w8h_triclinic_ani2x"]
CASES = [(8.0, "cosine"), (12.0, "smooth")]
TOL = 1e-11
HARTREE_TO_KCALPERMOL = 627.5094738898777


def cutoff_name(cutoff: float) -> str:
    return "inf" if cutoff == math.inf else f"{cutoff:g}"


def make_params(seed: int = 2024) -> dict:
    """Seeded per-element parameters, rounded to float32 (the reference's buffers are float32)."""
    g = np.random.default_rng(seed)
    S = len(orc.SYMBOLS_2X)
    f32 = lambda v: np.asarray(v, dtype=np.float32)   # noqa: E731
    return {"symbols": np.array(orc.SYMBOLS_2X),
            "eps": f32(g.uniform(0.05, 0.3, S) / HARTREE_TO_KCALPERMOL),
            "sigma": f32(g.uniform(1.0, 2.0, S)),
            "charges": f32(g.uniform(-0.8, 0.8, S)),
            "eta": f32(g.uniform(0.3, 0.8, S)),
            "dielectric": np.float64(2.0)}


def reference_potential(kind: str, cutoff: float, fn: str, params: dict):
    import torchani.potentials as rp
    cls = getattr(rp, lorc.CLASSES[kind])
    sym = orc.SYMBOLS_2X
    kw = dict(cutoff=cutoff, cutoff_fn=fn)
    vals = {k: [float(v) for v in params[k]] for k in ("eps", "sigma", "charges", "eta")}
    if kind in ("lj", "rep_lj", "disp_lj"):
        pot = cls(sym, vals["eps"], vals["sigma"], **kw)
    elif kind == "coulomb":
        pot = cls(sym, float(params["dielectric"]), vals["charges"], **kw)
    else:
        pot = cls(sym, float(params["dielectric"]), vals["charges"], vals["eta"], **kw)
    return pot.double()


def reference_results(pot, species, coords, cell, pbc, stress):
    x0 = coords.clone().requires_grad_(True)
    x, c, scaling = x0, cell, None
    if stress:
        scaling = torch.eye(3, dtype=torch.float64, requires_grad=True)
        x, c = x0 @ scaling, cell @ scaling
    # (by keyword: Potential.forward hands `atomic` on positionally into the `charge` slot, core.py:65-67)
    from torchani.neighbors import adaptive_list, all_pairs
    mk = adaptive_list if (species.shape[0] == 1 and pot.cutoff != math.inf) else all_pairs
    atomic = pot.compute_from_neighbors(species, x, mk(pot.cutoff, species, x, c, pbc), atomic=True).energies
    energy = atomic.sum(-1)
    out = {"energy": energy.detach(), "atomic": atomic.detach(),
           "forces": -torch.autograd.grad(energy.sum(), x0, retain_graph=stress)[0]}
    if stress:
        out["stress"] = torch.autograd.grad(energy.sum(), scaling)[0] / torch.det(cell).abs()
    return out


def main() -> None:
    import_reference()
    params = make_params()
    np.savez_compressed(os.path.join(GOLD, "ljc_params.npz"), **params)
    for name in SYSTEMS:
        z = np.load(os.path.join(GOLD, name + ".npz"))
        species = torch.tensor(z["species"])
        coords = torch.tensor(z["coords"], dtype=torch.float64)
        cell = torch.tensor(z["cell"], dtype=torch.float64) if z["cell"].size else None
        pbc = torch.tensor(z["pbc"]) if z["pbc"].size else None
        cases = CASES + ([(math.inf, "dummy")] if pbc is None else [])
        kinds = ("lj", "coulomb") if name.startswith("6w8h") else lorc.KINDS
        rec = {}
        for kind in kinds:
            for cutoff, fn in cases:
                ref_fn = "smooth" if fn == "dummy" else fn     # (the reference ignores it without a cutoff)
                ref = reference_results(reference_potential(kind, cutoff, ref_fn, params), species, coords, cell, pbc,
                                        cell is not None)
                nl = "cell_list" if species.shape[0] == 1 else "all_pairs"
                spec = lorc.spec_from_params(kind, cutoff, fn, params)
                got = lorc.compute(spec, species, coords, cell, pbc, nl, stress=cell is not None)
                key = f"{kind}_{fn}_{cutoff_name(cutoff)}"
                for k, v in ref.items():
                    err = float(((got[k] - v).abs() / (1.0 + v.abs())).max())
                    assert err < TOL, (name, key, k, err)
                    rec[f"{key}_{k}"] = v.detach().numpy()
                print(f"{name} {key}: E = {ref['energy'].tolist()[:2]}")
        np.savez_compressed(os.path.join(GOLD, f"ljc_{name}.npz"), **rec)
    print("wrote", sorted(f for f in os.listdir(GOLD) if f.startswith("ljc_")))


if __name__ == "__main__":
    main()
