"""Generate tests/golden/hessian_*.npz from the REAL reference's ``torchani.grad`` (aiqm/torchani under
/root/reference), in float64 on the CPU with this repository's seeded weights.

TEST INFRASTRUCTURE ONLY.  For every case the reference model is evaluated through
``torchani.grad.energies_forces_and_hessians`` and ``torchani.grad.vibrational_analysis`` (every mode kind, both units,
per conformer), and ``hessian_oracle`` must reproduce its Hessians to < 1e-10 (relative to max |H|) before anything is
written.  Cases (open systems, all-pairs neighbour lists):

  ch4_1x, water_1x      ANI-1x shape, CELU x 8 (ani_oracle.make_weights seed 1234)
  sevenel_2x            ANI-2x shape, the 20 atoms of the seven-element fixture nearest its first atom
  randbatch_2x          ANI-2x shape, the 8 x 12 padded conformers of randbatch_ani2x.npz
  gelu_xtb              simple_ani (ANI-2xr shape): GELU bias-free x 8 (gelu_oracle seed 4321), smooth cutoff, xTB at Rcr
  zbl_2x                ANI-2x shape with ZBL repulsion at Rcr (cosine envelope)

  tests/golden/hessian_<case>.npz  kind, symbols, species (model order, -1 padding), coords, energy (C,),
                                   forces (C, A, 3), hessian (C, 3A, 3A), masses (C, A) AMU (the reference's table),
                                   gelu_xtb: the reference's xTB tables xtb_{y_ab, sqrt_alpha_ab, k_rep_ab},
                                   and per real conformer c, mode kind k in mdu / mdn / mwn and unit u in cm / mev:
                                   vib_<c>_<k>_<u>_{freqs, modes, fconstants, rmasses}

Usage:  python oracle/make_hessian_golden.py
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
import oracle.hessian_oracle as hor      # noqa: E402
import oracle.pair_oracle as porc        # noqa: E402
from oracle.make_golden import import_reference   # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
TOL = 1e-10
UNITS = {"cm": "cm^-1", "mev": "meV"}


def water():
    sp = torch.tensor([[3, 0, 0]])
    co = torch.tensor([[[0.0, 0.0, 0.1173], [0.0, 0.7572, -0.4692], [0.0, -0.7572, -0.4692]]], dtype=torch.float64)
    return sp, co


def fixture(name):
    z = np.load(os.path.join(GOLD, name + ".npz"))
    return torch.tensor(z["species"]), torch.tensor(z["coords"], dtype=torch.float64)


def seven_element_molecule():
    sp, co = fixture("sevenel_pbc_ani2x")
    keep = torch.argsort((co[0] - co[0, 0]).norm(dim=-1))[:20]
    return sp[:, keep], co[:, keep]


def xtb_tables():
    z = np.load(os.path.join(GOLD, "pair_params.npz"))
    return tuple(torch.tensor(z[k]) for k in ("y_ab", "sqrt_alpha_ab", "k_rep_ab"))


def celu_case(kind, inputs, pot=None):
    torchani = import_reference()
    from oracle import ref_torchani
    symbols = orc.SYMBOLS_2X if kind == "2x" else orc.SYMBOLS_1X
    spec = orc.aev_spec_2x() if kind == "2x" else orc.aev_spec_1x()
    w = orc.make_weights(symbols, orc.DIMS_2X if kind == "2x" else orc.DIMS_1X, spec.out_dim, 8, 1234, torch.float64)
    ref = ref_torchani.build_model(w, kind, dtype=torch.float64, neighborlist="all_pairs", periodic_table_index=False)
    pairs = []
    if pot == "zbl":   # (a model takes its potentials at construction)
        from torchani.arch import ANI
        from torchani.potentials import RepulsionZBL
        nnp = ref.potentials["nnp"]
        default = torch.get_default_dtype()
        torch.set_default_dtype(torch.float32)
        zbl = RepulsionZBL(symbols, cutoff=spec.rcr, cutoff_fn="cosine")
        torch.set_default_dtype(default)
        ref = ANI(symbols, nnp.aev_computer, nnp.neural_networks, ref.energy_shifter,
                  potentials={"repulsion_zbl": zbl}, periodic_table_index=False).double()
        pairs.append(porc.zbl_spec(symbols, spec.rcr, "cosine"))
    sp, co = inputs()
    om = orc.Model(spec, symbols, w, {}, "all_pairs")
    return torchani, ref, symbols, sp, co, hor.energy_fn(om, sp, "celu", pairs)


def gelu_case():
    from oracle import make_gelu_golden as mg
    torchani = import_reference()
    model = mg.oracle_model()
    ref = mg.reference_model(model)
    ref.neighborlist = torchani.neighbors.AllPairs() if hasattr(torchani.neighbors, "AllPairs") else ref.neighborlist
    rep = ref.potentials["repulsion_xtb"]
    pair = porc.PairSpec("xtb", gor.RCR, "smooth", tuple(getattr(rep, k).detach().clone().double()
                                                         for k in ("y_ab", "sqrt_alpha_ab", "k_rep_ab")))
    sp2x, co = seven_element_molecule()
    species = torch.tensor([gor.SYMBOLS.index(s) for s in orc.SYMBOLS_2X])[sp2x]
    om = model._replace(neighborlist="all_pairs")
    return torchani, ref, gor.SYMBOLS, species, co, hor.energy_fn(om, species, "gelu", [pair]), {
        k: t.numpy() for k, t in zip(("xtb_y_ab", "xtb_sqrt_alpha_ab", "xtb_k_rep_ab"), pair.tables)}


def write(name, torchani, ref, symbols, species, coords, energy, extra=None):
    znums = torch.tensor([orc.ATOMIC_NUMBERS[s] for s in symbols])
    sp_ref = species if not ref.periodic_table_index else znums[species.clamp(min=0)].masked_fill(species < 0, -1)
    x = coords.clone()
    out = torchani.grad.energies_forces_and_hessians(ref, sp_ref, x)
    h_ref = out.hessians.detach()
    h = hor.hessian(energy, coords)
    err = float((h - h_ref).abs().max()) / float(h_ref.abs().max())
    assert err < TOL, (name, err)
    from torchani.constants import ATOMIC_MASS
    masses = torch.tensor([[ATOMIC_MASS[symbols[int(e)]] if e >= 0 else 0.0 for e in row] for row in species],
                          dtype=torch.float64)
    rec = dict(kind=name, symbols=np.array(symbols), species=species.numpy(), coords=coords.numpy(),
               energy=out.energies.detach().numpy(), forces=out.forces.detach().numpy(), hessian=h_ref.numpy(),
               masses=masses.numpy(), **(extra or {}))
    for c in range(species.shape[0]):
        real = species[c] >= 0
        idx = torch.nonzero(real).view(-1)
        cols = torch.stack([3 * idx + k for k in range(3)], 1).reshape(-1)
        hc = h_ref[c][cols][:, cols].unsqueeze(0)
        for kind in ("mdu", "mdn", "mwn"):
            for u, unit in UNITS.items():
                va = torchani.grad.vibrational_analysis(masses[c, idx].unsqueeze(0), hc, kind, unit)
                for field in ("freqs", "modes", "fconstants", "rmasses"):
                    rec[f"vib_{c}_{kind}_{u}_{field}"] = getattr(va, field).detach().numpy()
    np.savez_compressed(os.path.join(GOLD, f"hessian_{name}.npz"), **rec)
    print(f"{name}: max |H| {float(h_ref.abs().max()):.3e}, oracle rel err {err:.1e}")


def main() -> None:
    # the reference then builds its AEV constants as the oracle does (to 1e-10); its ZBL screening constants are
    # float32 buffers all the same (celu_case)
    torch.set_default_dtype(torch.float64)
    cases = {
        "ch4_1x": lambda: celu_case("1x", lambda: fixture("ch4_ani1x")),
        "water_1x": lambda: celu_case("1x", water),
        "sevenel_2x": lambda: celu_case("2x", seven_element_molecule),
        "randbatch_2x": lambda: celu_case("2x", lambda: fixture("randbatch_ani2x")),
        "gelu_xtb": gelu_case,
        "zbl_2x": lambda: celu_case("2x", seven_element_molecule, "zbl"),
    }
    only = sys.argv[1:]
    for name, make in cases.items():
        if only and name not in only:
            continue
        write(name, *make())


if __name__ == "__main__":
    main()
