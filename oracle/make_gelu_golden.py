"""Generate tests/golden/gelu_*.npz from the REAL reference's ``simple_ani`` models (aiqm/torchani under /root/reference).

TEST INFRASTRUCTURE ONLY; runs on the CPU where the reference sources are present.  The model is what
``torchani.arch.simple_ani`` assembles for ANI-2xr-style networks (arch.py:992-1069): the seven ANI-2x elements in
the reference's atomic-number order (``SYMBOLS_2X_ZNUM_ORDER``: H C N O F S Cl), ``cover_linearly`` AEV constants with
the smooth cutoff, ``ANINetworks.default`` = ANI-2x widths with GELU and NO biases, xTB repulsion at the radial cutoff
(5.2 A), no dispersion, 8 members, lot wb97x-631gd, AEV strategy "pyaev".  Its network weights are replaced by seeded
bias-free weights (``gelu_oracle.make_weights``).  For the systems of existing golden fixtures (their
inputs are reused; the species are re-indexed to the model's element order, periodic systems wrapped into the cell)
the reference is evaluated in float64, and ``gelu_oracle`` plus ``pair_oracle`` (xTB) must agree with it to < 1e-11 before anything is
written.

  tests/golden/gelu_<system>.npz  symbols, self_energies, species (model order), atomic_numbers, coords, cell, pbc,
                                  weight_seed, member_atomic (M, C, A) NN atomic energies, energy_nn, energy
                                  (NN + repulsion + self energies), forces, stress (periodic systems: the "scaling" stress of
                                  ase.py:110-121,170-173), state_dict_keys (the reference model's)

Usage:  python oracle/make_gelu_golden.py
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
import oracle.gelu_oracle as gor         # noqa: E402
import oracle.pair_oracle as porc        # noqa: E402
from oracle.make_golden import import_reference   # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
SYSTEMS = ["water999_pbc", "1c17_chunk_hcnos", "randbatch", "6w8h_triclinic", "sevenel_pbc", "small264_nopbc"]
SYMBOLS = gor.SYMBOLS     # the reference's SYMBOLS_2X_ZNUM_ORDER
MEMBERS = 8
SEED = 4321
RCR = gor.RCR
TOL = 1e-11


def oracle_model() -> orc.Model:
    spec = gor.gelu_spec()
    weights = gor.make_weights(SYMBOLS, orc.DIMS_2X, spec.out_dim, MEMBERS, SEED)
    return orc.Model(spec, SYMBOLS, weights, orc.GSAES_WB97X_631GD, "cell_list")   # (sae: main())


def reference_model(model: orc.Model):
    torchani = import_reference()
    ref = torchani.arch.simple_ani(list(SYMBOLS), "wb97x-631gd", ensemble_size=MEMBERS, strategy="pyaev",
                                   repulsion=True, dispersion=False)
    nets = ref.potentials["nnp"].neural_networks
    with torch.no_grad():
        for m, member in enumerate(nets.members):
            for s in SYMBOLS:
                an = member.atomics[s]
                for layer, (w, b) in zip(list(an.layers) + [an.final_layer], model.weights[m][s]):
                    assert layer.bias is None and b is None
                    layer.weight.copy_(w)
    return ref.double()


def reference_results(ref, znums, coords, cell, pbc):
    stress = cell is not None
    x0 = coords.clone().requires_grad_(True)
    x, c, scaling = x0, cell, None
    if stress:
        scaling = torch.eye(3, dtype=torch.float64, requires_grad=True)
        x, c = x0 @ scaling, cell @ scaling
    energy = ref((znums, x), cell=c, pbc=pbc).energies
    out = {"energy": energy.detach(), "forces": -torch.autograd.grad(energy.sum(), x0, retain_graph=stress)[0]}
    if stress:
        out["stress"] = torch.autograd.grad(energy.sum(), scaling)[0] / torch.det(cell).abs()
    nnp = ref.potentials["nnp"]
    elem = ref.species_converter(znums)
    with torch.no_grad():
        aev = nnp.aev_computer(elem, coords, cell=cell, pbc=pbc)
        out["member_atomic"] = nnp.neural_networks(elem, aev, atomic=True, ensemble_values=True)
    return out


def main() -> None:
    model = oracle_model()
    ref = reference_model(model)
    # the reference's ground-state atomic energies of the lot (set_gsaes_as_self_energies), not those of ANI-2x
    sae = dict(zip(SYMBOLS, ref.energy_shifter.self_energies.tolist()))
    model = model._replace(sae=sae)
    rep = ref.potentials["repulsion_xtb"]
    assert float(rep.cutoff) == RCR
    pair = porc.PairSpec("xtb", RCR, "smooth", tuple(getattr(rep, k).detach().clone().double()
                                                     for k in ("y_ab", "sqrt_alpha_ab", "k_rep_ab")))
    keys = np.array(sorted(ref.state_dict().keys()))
    for name in SYSTEMS:
        z = np.load(os.path.join(GOLD, name + "_ani2x.npz"))
        sp2x = torch.tensor(z["species"])
        znums = torch.tensor([orc.ATOMIC_NUMBERS[s] for s in orc.SYMBOLS_2X])[sp2x.clamp(min=0)].masked_fill(sp2x < 0, -1)
        species = torch.tensor([SYMBOLS.index(s) for s in orc.SYMBOLS_2X])[sp2x.clamp(min=0)].masked_fill(sp2x < 0, -1)
        coords = torch.tensor(z["coords"], dtype=torch.float64)
        cell = torch.tensor(z["cell"], dtype=torch.float64) if z["cell"].size else None
        pbc = torch.tensor(z["pbc"]) if z["pbc"].size else None
        periodic = cell is not None
        if periodic:   # wrapped into the cell: there the reference's "scaling" stress is the pair-vector virial
            frac = coords @ torch.inverse(cell)
            coords = (frac - frac.floor()) @ cell
        r = reference_results(ref, znums, coords, cell, pbc)
        nl = "cell_list" if species.shape[0] == 1 else "all_pairs"
        got = gor.compute(model._replace(neighborlist=nl), species, coords, cell, pbc, stress=periodic)
        gp = porc.compute(pair, species, coords, cell, pbc, nl, stress=periodic)
        mine = {"energy": got["energy"] + gp["energy"], "forces": got["forces"] + gp["forces"],
                "member_atomic": got["member_atomic"]}
        if periodic:
            mine["stress"] = got["stress"] + gp["stress"]
        for k, v in r.items():   # (total energies reach 1e5 Ha: relative to them, the sum order of float64 shows)
            err = float((mine[k] - v).abs().max()) / (1.0 + float(v.abs().max()) if k == "energy" else 1.0)
            assert err < TOL, (name, k, err)
        np.savez_compressed(
            os.path.join(GOLD, f"gelu_{name}.npz"), symbols=np.array(SYMBOLS),
            self_energies=np.array([sae[s] for s in SYMBOLS]), species=species.numpy(), atomic_numbers=znums.numpy(),
            coords=coords.numpy(), cell=z["cell"], pbc=z["pbc"], weight_seed=SEED,
            member_atomic=r["member_atomic"].numpy(), energy_nn=got["energy_nn"].numpy(), energy=r["energy"].numpy(),
            forces=r["forces"].numpy(), **({"stress": r["stress"].numpy()} if periodic else {}),
            state_dict_keys=keys)
        print(f"{name}: E = {r['energy'].tolist()[:2]}")


if __name__ == "__main__":
    main()
