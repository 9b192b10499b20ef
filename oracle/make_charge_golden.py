"""Generate tests/golden/charges_<config>_<system>.npz from the REAL reference's ANIq models (aiqm/torchani under
/root/reference).

TEST INFRASTRUCTURE ONLY; runs on the CPU where the reference sources are present and never reaches the network:
the models are assembled, not downloaded, and their weights are seeded.

  mbis    ``Assembler(cls=ANIq)`` exactly as ``torchani.models.ANImbis`` assembles it (models.py:201-252): ANI-2x AEV
          (cosine cutoff) and 8-member CELU ensemble with seeded weights (``ani_oracle.make_weights``), one
          ``_ANINetworksDiscardFirstScalar`` charge container (ANI-2x widths, GELU, no biases, ``out_dim = 2``) with
          seeded weights, ``ChargeNormalizer.from_electronegativity_and_hardness(..., scale_weights_by_charges_squared=
          True)``, wb97x-631gd self energies.
  simple  ``torchani.arch.simple_aniq`` (arch.py:1071-1182): smooth cutoff, GELU bias-free energy networks
          (``gelu_oracle.make_weights``), a plain ``ANINetworks`` charge container (``out_dim = 1``), no q^2 scaling,
          no repulsion.

For the systems of the existing golden fixtures (species re-indexed to the model's element order, periodic systems
wrapped into the cell) the reference is evaluated in float64; ``charge_oracle`` must agree with it to < 1e-11 before
anything is written.  The normaliser weights (the module's non-persistent ``weights`` buffer) and the masses of the
reference's table (``torchani.constants.MASS``) are stored as data.

  charges_<config>_<system>.npz  config, symbols, kept (charge network output column), scale_by_q2, norm_weights,
                                 masses (per element), energy_seed, charge_seed, self_energies, species (model order),
                                 atomic_numbers, coords, cell, pbc, raw_charges, charges, dipole_<frame> for the three
                                 frames, energy, forces, state_dict_keys

Usage:  python oracle/make_charge_golden.py
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
import oracle.charge_oracle as cor       # noqa: E402
import oracle.gelu_oracle as gor         # noqa: E402
from oracle.make_golden import import_reference   # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
SYSTEMS = {"mbis": ["water999_pbc", "1c17_chunk_hcnos", "randbatch", "6w8h_triclinic", "sevenel_pbc", "small264_nopbc"],
           "simple": ["randbatch", "small264_nopbc", "water999_pbc"]}
MEMBERS = 8
ENERGY_SEED = 2468
CHARGE_SEED = 1357
TOL = 1e-11


def reference_model(config: str):
    """(reference model in float64, oracle ChargeModel with the same weights)."""
    torchani = import_reference()
    from torchani.arch import ANIq, Assembler
    from torchani.constants import MASS
    from torchani.electro import ChargeNormalizer
    from torchani.nn._internal import _ANINetworksDiscardFirstScalar
    if config == "mbis":
        symbols = orc.SYMBOLS_2X
        asm = Assembler(cls=ANIq, periodic_table_index=True)
        asm.set_symbols(symbols)
        asm.set_global_cutoff_fn("cosine")
        asm.set_aev_computer(radial="ani2x", angular="ani2x", strategy="pyaev")
        asm.set_atomic_networks(ctor="ani2x")
        asm.set_charge_networks(
            cls=_ANINetworksDiscardFirstScalar, ctor="ani2x",
            kwargs={"out_dim": 2, "bias": False, "activation": "gelu"},
            normalizer=ChargeNormalizer.from_electronegativity_and_hardness(
                asm.symbols, scale_weights_by_charges_squared=True))
        asm.set_neighborlist("all_pairs")
        asm.set_gsaes_as_self_energies("wb97x-631gd")
        ref = asm.assemble(MEMBERS)
        spec = orc.aev_spec_2x()
        ew = orc.make_weights(symbols, orc.DIMS_2X, spec.out_dim, MEMBERS, ENERGY_SEED)
        kept, out_dim, gelu = 1, 2, False
    else:
        symbols = gor.SYMBOLS
        ref = torchani.arch.simple_aniq(list(symbols), "wb97x-631gd", ensemble_size=MEMBERS, repulsion=False,
                                        scale_charge_normalizer_weights=False, strategy="pyaev")
        spec = gor.gelu_spec()
        ew = gor.make_weights(symbols, orc.DIMS_2X, spec.out_dim, MEMBERS, ENERGY_SEED)
        kept, out_dim, gelu = 0, 1, True
    cw = cor.make_charge_weights(symbols, orc.DIMS_2X, spec.out_dim, out_dim, CHARGE_SEED)
    nnp = ref.potentials["nnp"]
    with torch.no_grad():
        for m, member in enumerate(nnp.neural_networks.members):
            for s in symbols:
                an = member.atomics[s]
                for layer, (w, b) in zip(list(an.layers) + [an.final_layer], ew[m][s]):
                    layer.weight.copy_(w)
                    if b is not None:
                        layer.bias.copy_(b)
        for s in symbols:
            an = nnp.charge_networks.atomics[s]
            for layer, w in zip(list(an.layers) + [an.final_layer], cw[s]):
                assert layer.bias is None
                layer.weight.copy_(w)
    norm = nnp.charge_normalizer
    norm_w = tuple(float(v) for v in norm.weights.tolist())
    q2 = bool(norm.scale_weights_by_charges_squared)
    masses = tuple(float(MASS[orc.ATOMIC_NUMBERS[s]]) for s in symbols)
    sae = dict(zip(symbols, ref.energy_shifter.self_energies.tolist()))
    model = cor.ChargeModel(orc.Model(spec, tuple(symbols), ew, sae, "cell_list"), gelu, cw, kept, norm_w, q2, masses)
    return ref.double(), model


def reference_results(ref, znums, coords, cell, pbc):
    from torchani.electro import DipoleComputer
    x0 = coords.clone().requires_grad_(True)
    out = ref((znums, x0), cell=cell, pbc=pbc)
    res = {"energy": out.energies.detach(), "forces": -torch.autograd.grad(out.energies.sum(), x0)[0],
           "charges": out.atomic_charges.detach()}
    nnp = ref.potentials["nnp"]
    elem = ref.species_converter(znums)
    with torch.no_grad():
        aev = nnp.aev_computer(elem, coords, cell=cell, pbc=pbc)
        res["raw_charges"] = nnp.charge_networks(elem, aev, atomic=True)
        for f in cor.FRAMES:
            res["dipole_" + f] = DipoleComputer(reference=f, dtype=torch.float64)(znums, coords, res["charges"])
    return res


def main() -> None:
    for config, systems in SYSTEMS.items():
        ref, model = reference_model(config)
        symbols = model.energy.symbols
        keys = np.array(sorted(ref.state_dict().keys()))
        for name in systems:
            z = np.load(os.path.join(GOLD, name + "_ani2x.npz"))
            sp2x = torch.tensor(z["species"])
            znums = torch.tensor([orc.ATOMIC_NUMBERS[s] for s in orc.SYMBOLS_2X])[sp2x.clamp(min=0)].masked_fill(
                sp2x < 0, -1)
            species = torch.tensor([symbols.index(s) for s in orc.SYMBOLS_2X])[sp2x.clamp(min=0)].masked_fill(
                sp2x < 0, -1)
            coords = torch.tensor(z["coords"], dtype=torch.float64)
            cell = torch.tensor(z["cell"], dtype=torch.float64) if z["cell"].size else None
            pbc = torch.tensor(z["pbc"]) if z["pbc"].size else None
            if cell is not None:
                frac = coords @ torch.inverse(cell)
                coords = (frac - frac.floor()) @ cell
            r = reference_results(ref, znums, coords, cell, pbc)
            nl = "cell_list" if species.shape[0] == 1 else "all_pairs"
            got = cor.compute(model._replace(energy=model.energy._replace(neighborlist=nl)), species, coords, cell, pbc)
            for k, v in r.items():
                err = float((got[k] - v).abs().max()) / (1.0 + float(v.abs().max()) if k == "energy" else 1.0)
                assert err < TOL, (config, name, k, err)
            np.savez_compressed(
                os.path.join(GOLD, f"charges_{config}_{name}.npz"), config=config, symbols=np.array(symbols),
                kept=model.kept, scale_by_q2=model.scale_by_q2, norm_weights=np.array(model.norm_weights),
                masses=np.array(model.masses), energy_seed=ENERGY_SEED, charge_seed=CHARGE_SEED,
                self_energies=np.array([model.energy.sae[s] for s in symbols]), species=species.numpy(),
                atomic_numbers=znums.numpy(), coords=coords.numpy(), cell=z["cell"], pbc=z["pbc"],
                state_dict_keys=keys, **{k: v.numpy() for k, v in r.items()})
            print(f"{config} {name}: E = {r['energy'].tolist()[:2]}, |q| max = {float(r['charges'].abs().max()):.3f}")


if __name__ == "__main__":
    main()
