"""Generate tests/golden/pair_*.npz from the REAL reference's pair potentials (aiqm/torchani under /root/reference).

TEST INFRASTRUCTURE ONLY; runs on the CPU where the reference sources are present.  For the systems of existing golden
fixtures (their inputs are reused, not stored again) it evaluates the reference's ``RepulsionXTB`` and ``RepulsionZBL``
(float64, cutoff = the ANI-2x radial cutoff, cosine and smooth envelopes): energies, atomic energies, autograd forces
and, for periodic systems, the "scaling" stress of ase.py:110-121,170-173.  ``pair_oracle`` must agree with the
reference to < 1e-11 before anything is written.  The fixtures hold the pair terms alone; the totals of a model with
networks are these plus the network results of the system's own golden file.

  tests/golden/pair_params.npz   the xTB parameter tensors of the reference module (y_ab, sqrt_alpha_ab, k_rep_ab)
  tests/golden/pair_<system>.npz <kind>_<fn>_{energy,atomic,forces[,stress]}
  tests/golden/pair_scan.npz     diatomic scan 0.3 - 5.2 A over all element pairs of ANI-2x (+ the 1e-7 clamp)

Usage:  python oracle/make_pair_golden.py
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
import oracle.pair_oracle as porc        # noqa: E402
from oracle.make_golden import import_reference   # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
SYSTEMS = ["water999_pbc_ani2x", "1c17_chunk_hcnos_ani2x", "randbatch_ani2x", "6w8h_triclinic_ani2x"]
RCR = 5.1
FNS = ("cosine", "smooth")
TOL = 1e-11


def scan_distances() -> np.ndarray:
    """0.3 .. 5.2 A, across the cutoff, plus points at and below the 1e-7 clamp."""
    return np.concatenate([[1e-9, 1e-7, 1e-3, 0.05], np.linspace(0.3, 5.2, 50), [5.0999, 5.1, 5.1001]])


def reference_potential(kind: str, fn: str):
    from torchani.potentials import RepulsionXTB, RepulsionZBL
    cls = RepulsionXTB if kind == "xtb" else RepulsionZBL
    return cls(orc.SYMBOLS_2X, cutoff=RCR, cutoff_fn=fn).double()


def reference_results(pot, species, coords, cell, pbc, stress):
    x0 = coords.clone().requires_grad_(True)
    x, c, scaling = x0, cell, None
    if stress:
        scaling = torch.eye(3, dtype=torch.float64, requires_grad=True)
        x, c = x0 @ scaling, cell @ scaling
    # (Potential.forward hands `atomic` on positionally into the `charge` slot, core.py:65-67: call the reference's
    # neighbour list and compute_from_neighbors themselves, by keyword)
    from torchani.neighbors import adaptive_list, all_pairs
    mk = adaptive_list if species.shape[0] == 1 else all_pairs
    atomic = pot.compute_from_neighbors(species, x, mk(pot.cutoff, species, x, c, pbc), atomic=True).energies
    energy = atomic.sum(-1)
    out = {"energy": energy.detach(), "atomic": atomic.detach(),
           "forces": -torch.autograd.grad(energy.sum(), x0, retain_graph=stress)[0]}
    if stress:
        out["stress"] = torch.autograd.grad(energy.sum(), scaling)[0] / torch.det(cell).abs()
    # the non-atomic path of the reference (core.py:201-206) must be the sum of the split
    e2 = pot(species, coords, cell, pbc, atomic_nums_input=False)
    assert float((e2 - out["energy"]).abs().max()) < 1e-9
    return out


def main() -> None:
    import_reference()
    xtb = reference_potential("xtb", "cosine")
    tables = tuple(getattr(xtb, k).detach().clone() for k in ("y_ab", "sqrt_alpha_ab", "k_rep_ab"))
    np.savez_compressed(os.path.join(GOLD, "pair_params.npz"), symbols=np.array(orc.SYMBOLS_2X), cutoff=RCR,
                        y_ab=tables[0].numpy(), sqrt_alpha_ab=tables[1].numpy(), k_rep_ab=tables[2].numpy())

    def spec(kind, fn):
        return porc.PairSpec("xtb", RCR, fn, tables) if kind == "xtb" else porc.zbl_spec(orc.SYMBOLS_2X, RCR, fn)

    for name in SYSTEMS:
        z = np.load(os.path.join(GOLD, name + ".npz"))
        species = torch.tensor(z["species"])
        coords = torch.tensor(z["coords"], dtype=torch.float64)
        cell = torch.tensor(z["cell"], dtype=torch.float64) if z["cell"].size else None
        pbc = torch.tensor(z["pbc"]) if z["pbc"].size else None
        rec = {}
        for kind in ("xtb", "zbl"):
            for fn in FNS:
                ref = reference_results(reference_potential(kind, fn), species, coords, cell, pbc, cell is not None)
                nl = "cell_list" if species.shape[0] == 1 else "all_pairs"
                got = porc.compute(spec(kind, fn), species, coords, cell, pbc, nl, stress=cell is not None)
                for k, v in ref.items():
                    err = float((got[k] - v).abs().max())
                    assert err < TOL, (name, kind, fn, k, err)
                    rec[f"{kind}_{fn}_{k}"] = v.detach().numpy()
                print(f"{name} {kind} {fn}: E = {ref['energy'].tolist()[:2]}")
        np.savez_compressed(os.path.join(GOLD, f"pair_{name}.npz"), **rec)

    # diatomic scan: every element pair (a <= b) of ANI-2x at every distance, one two-atom conformer each
    S = len(orc.SYMBOLS_2X)
    dist = scan_distances()
    pairs = [(a, b) for a in range(S) for b in range(a, S)]
    species = torch.tensor([[a, b] for (a, b) in pairs for _ in dist])
    coords = torch.zeros(len(species), 2, 3, dtype=torch.float64)
    coords[:, 1, 0] = torch.tensor(np.tile(dist, len(pairs)))
    rec = {"species": species.numpy(), "coords": coords.numpy()}
    for kind in ("xtb", "zbl"):
        for fn in FNS:
            ref = reference_results(reference_potential(kind, fn), species, coords, None, None, False)
            got = porc.compute(spec(kind, fn), species, coords, None, None, "all_pairs")
            for k, v in ref.items():
                err = float(((got[k] - v).abs() / (1.0 + v.abs())).max())     # the clamp region reaches 1e9 Ha: relative
                assert err < TOL, (kind, fn, k, err)
                rec[f"{kind}_{fn}_{k}"] = v.detach().numpy()
    np.savez_compressed(os.path.join(GOLD, "pair_scan.npz"), **rec)
    print("wrote", sorted(f for f in os.listdir(GOLD) if f.startswith("pair_")))


if __name__ == "__main__":
    main()
