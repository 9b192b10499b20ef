"""Charge models without a GPU: the float64 charge oracle (oracle/charge_oracle.py) against every charges_* fixture of
the reference's ANIq models (oracle/make_charge_golden.py), the charge container's module tree and packing, the
normaliser / dipole modules' table rule, and the new C-ABI prototype."""
import glob
import os

import numpy as np
import pytest
import torch

import oracle.ani_oracle as orc
import oracle.charge_oracle as cor
import oracle.gelu_oracle as gor
from helpers import GOLD, ROOT

FILES = sorted(os.path.basename(f)[len("charges_"):-len(".npz")] for f in glob.glob(os.path.join(GOLD, "charges_*.npz")))


def fixture(tag):
    z = np.load(os.path.join(GOLD, f"charges_{tag}.npz"))
    return {k: z[k] for k in z.files}


def test_every_configuration_has_fixtures():
    assert {t.split("_", 1)[0] for t in FILES} == {"mbis", "simple"} and len(FILES) == 9


@pytest.mark.parametrize("tag", FILES)
def test_oracle_reproduces_the_reference_fixture(tag):
    rec = fixture(tag)
    config = str(rec["config"])
    symbols = tuple(str(s) for s in rec["symbols"])
    if config == "mbis":
        spec = orc.aev_spec_2x()
        ew = orc.make_weights(symbols, orc.DIMS_2X, spec.out_dim, 8, int(rec["energy_seed"]))
    else:
        spec = gor.gelu_spec()
        ew = gor.make_weights(symbols, orc.DIMS_2X, spec.out_dim, 8, int(rec["energy_seed"]))
    cw = cor.make_charge_weights(symbols, orc.DIMS_2X, spec.out_dim, int(rec["kept"]) + 1, int(rec["charge_seed"]))
    sp = torch.tensor(rec["species"])
    co = torch.tensor(rec["coords"], dtype=torch.float64)
    cell = torch.tensor(rec["cell"], dtype=torch.float64) if rec["cell"].size else None
    pbc = torch.tensor(rec["pbc"]) if rec["pbc"].size else None
    nl = "cell_list" if sp.shape[0] == 1 else "all_pairs"
    model = cor.ChargeModel(orc.Model(spec, symbols, ew, dict(zip(symbols, rec["self_energies"].tolist())), nl),
                            config == "simple", cw, int(rec["kept"]), tuple(rec["norm_weights"].tolist()),
                            bool(rec["scale_by_q2"]), tuple(rec["masses"].tolist()))
    got = cor.compute(model, sp, co, cell, pbc)
    scale = 1.0 + float(np.abs(rec["energy"]).max())
    assert float((got["energy"] - torch.tensor(rec["energy"])).abs().max()) < 1e-11 * scale
    assert float((got["forces"] - torch.tensor(rec["forces"])).abs().max()) < 1e-10
    for k in ["raw_charges", "charges"] + ["dipole_" + f for f in cor.FRAMES]:
        assert float((got[k] - torch.tensor(rec[k])).abs().max()) < 1e-11, k
    # the normalised charges add up to the (zero) total charge
    assert float(np.abs(rec["charges"].sum(-1)).max()) < 1e-12
    # the origin dipole is the plain sum q r; the frames agree when the charges sum to zero
    real = rec["species"] >= 0
    mu0 = (rec["charges"][..., None] * rec["coords"] * real[..., None]).sum(1)
    assert np.allclose(mu0, rec["dipole_origin"], rtol=0, atol=1e-12)
    assert np.allclose(rec["dipole_center_of_mass"], rec["dipole_origin"], rtol=0, atol=1e-9)


def test_charge_container_tree_and_packing():
    from torchani_b200 import nn
    q = nn.ChargeNetworks.like_2x(("H", "C"), 64)
    assert q.out_dim == 2 and q.kept_output == 1
    keys = set(q.state_dict().keys())
    assert "atomics.H.layers.0.weight" in keys and "atomics.C.final_layer.weight" in keys
    assert not any(k.endswith("bias") for k in keys)
    pairs = q._packing_pairs(q.atomics["H"])
    w_full = q.atomics["H"].final_layer.weight
    assert pairs[-1][0].shape == (1, w_full.shape[1]) and torch.equal(pairs[-1][0][0], w_full[1])
    one = nn.ChargeNetworks.like_2x(("H",), 64, out_dim=1)
    assert one.kept_output == 0
    with pytest.raises(ValueError):
        nn.ChargeNetworks.like_2x(("H",), 64, out_dim=3)
    with pytest.raises(ValueError):
        nn.ChargeNetworks({"H": nn.AtomicNetwork((64, 32, 32, 32, 2), "gelu", bias=False)}, kept_output=0)


def test_normalizer_and_dipole_tables_are_not_shipped():
    from torchani_b200 import electro
    with pytest.raises(ValueError, match="from_torchani"):
        electro.ChargeNormalizer.from_electronegativity_and_hardness(["H", "O"])
    n = electro.ChargeNormalizer.from_electronegativity_and_hardness(["H", "O"], [2.0, 4.0], [4.0, 2.0], True)
    assert np.allclose(n.weights.numpy(), [0.25, 4.0]) and n.scale_weights_by_charges_squared
    assert np.allclose(electro.ChargeNormalizer(["H", "O"]).weights.numpy(), [1.0, 1.0])
    with pytest.raises(ValueError):
        electro.DipoleComputer(reference="center_of_mass")
    electro.DipoleComputer(reference="center_of_geometry")
    electro.DipoleComputer([0.0, 1.008], reference="center_of_mass")
    with pytest.raises(ValueError):
        electro.DipoleComputer(reference="nowhere")
    from torchani_b200 import models
    with pytest.raises(ValueError, match="not shipped"):
        models.ANImbis()


def test_charges_prototype_is_declared():
    from torchani_b200 import _lib
    assert "ani_b200_charges" in _lib.EXPORTED_SYMBOLS
    with open(os.path.join(ROOT, "include", "ani_b200.h")) as fh:
        assert "int ani_b200_charges(" in fh.read()
