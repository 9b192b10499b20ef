"""GELU bias-free networks (ANI-2xr style) without a GPU: the float64 oracle against the gelu_* fixtures of the
reference's ``simple_ani`` (oracle/make_gelu_golden.py), module construction and the network kinds the kernels
reject, state-dict keys against the reference model's, and the activation field of ``ani_mlp_model``."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

import oracle.ani_oracle as orc
import oracle.gelu_oracle as gor
import oracle.pair_oracle as porc
from helpers import GOLD, ROOT

SYMBOLS = gor.SYMBOLS
RCR = gor.RCR


def fixture(name):
    z = np.load(os.path.join(GOLD, f"gelu_{name}.npz"))
    return {k: z[k] for k in z.files}


def oracle_model(rec):
    spec = gor.gelu_spec()
    w = gor.make_weights(SYMBOLS, orc.DIMS_2X, spec.out_dim, 8, int(rec["weight_seed"]))
    return orc.Model(spec, SYMBOLS, w, dict(zip(SYMBOLS, rec["self_energies"].tolist())), "cell_list")


def xtb_spec():
    zp = np.load(os.path.join(GOLD, "pair_params.npz"))
    perm = [orc.SYMBOLS_2X.index(s) for s in SYMBOLS]
    tab = tuple(torch.tensor(zp[k])[perm][:, perm].double() for k in ("y_ab", "sqrt_alpha_ab", "k_rep_ab"))
    return porc.PairSpec("xtb", RCR, "smooth", tab)


@pytest.mark.parametrize("name", ["randbatch", "small264_nopbc", "1c17_chunk_hcnos", "water999_pbc"])
def test_oracle_matches_the_reference_fixture(name):
    rec = fixture(name)
    assert tuple(rec["symbols"]) == SYMBOLS
    sp = torch.tensor(rec["species"])
    co = torch.tensor(rec["coords"], dtype=torch.float64)
    cell = torch.tensor(rec["cell"], dtype=torch.float64) if rec["cell"].size else None
    pbc = torch.tensor(rec["pbc"]) if rec["pbc"].size else None
    nl = "cell_list" if sp.shape[0] == 1 else "all_pairs"
    got = gor.compute(oracle_model(rec)._replace(neighborlist=nl), sp, co, cell, pbc, stress=cell is not None)
    pair = porc.compute(xtb_spec(), sp, co, cell, pbc, nl, stress=cell is not None)
    scale = 1.0 + float(np.abs(rec["energy"]).max())
    assert float((got["member_atomic"] - torch.tensor(rec["member_atomic"])).abs().max()) < 1e-11
    assert float((got["energy"] + pair["energy"] - torch.tensor(rec["energy"])).abs().max()) < 1e-11 * scale
    assert float((got["forces"] + pair["forces"] - torch.tensor(rec["forces"])).abs().max()) < 1e-10
    if cell is not None:
        assert float((got["stress"] + pair["stress"] - torch.tensor(rec["stress"])).abs().max()) < 1e-12
    # the NN energy is the mean over the members of their atomic sums
    assert np.allclose(rec["member_atomic"].sum(-1).mean(0), rec["energy_nn"], rtol=0, atol=1e-10)


def test_network_kinds():
    from torchani_b200 import _lib, nn
    g = nn.AtomicNetwork((1008, 100, 72, 40, 1), "gelu", bias=False)
    assert g.activation_kind == _lib.ACT_GELU and isinstance(g.activation, torch.nn.GELU)
    assert not g.has_biases and all(b is None for _, b in g.linear_pairs())
    g2 = nn.AtomicNetwork((8, 4, 4, 4, 1), torch.nn.GELU(approximate="none"), bias=False)
    assert g2.activation_kind == _lib.ACT_GELU
    c = nn.AtomicNetwork((8, 4, 4, 4, 1))
    assert c.activation_kind == _lib.ACT_CELU and c.has_biases
    assert nn.AtomicNetwork((8, 4, 4, 4, 1), nn.TightCELU(), bias=True).activation_kind == _lib.ACT_CELU
    rejected = [
        dict(activation="gelu"),                                        # GELU with biases (bias defaults to True)
        dict(activation="gelu", bias=True),
        dict(activation="celu", bias=False),                            # CELU without biases
        dict(activation=torch.nn.GELU(approximate="tanh"), bias=False),
        dict(activation=torch.nn.ReLU(), bias=False),
        dict(activation="relu", bias=True),
        dict(activation=torch.nn.CELU(0.1), bias=True),
    ]
    for kw in rejected:
        with pytest.raises(ValueError):
            nn.AtomicNetwork((8, 4, 4, 4, 1), **kw)
    # one activation per container
    mixed = {"H": nn.AtomicNetwork((8, 4, 4, 4, 1)), "C": nn.AtomicNetwork((8, 4, 4, 4, 1), "gelu", bias=False)}
    with pytest.raises(ValueError):
        nn.ANINetworks(mixed)
    a = nn.ANINetworks({"H": nn.AtomicNetwork((8, 4, 4, 4, 1))})
    b = nn.ANINetworks({"H": nn.AtomicNetwork((8, 4, 4, 4, 1), "gelu", bias=False)})
    with pytest.raises(ValueError):
        nn.Ensemble([a, b])


def test_constructors_match_the_reference_defaults():
    from torchani_b200 import _lib, nn
    d = nn.ANINetworks.default(SYMBOLS, 1008)
    assert d.activation_kind == _lib.ACT_GELU and not d.atomics["C"].has_biases
    assert d.atomics["C"].layers[0].out_features == 224          # like_2x widths
    dr = nn.ANINetworks.like_dr()
    assert dr.activation_kind == _lib.ACT_GELU and dr.atomics["C"].layers[0].out_features == 256
    assert nn.ANINetworks.like_2x().activation_kind == _lib.ACT_CELU
    assert nn.ANINetworks.like_1x().activation_kind == _lib.ACT_CELU
    b = nn.ANINetworks.build(("H",), 16, {"H": (8, 8, 8)})
    assert b.activation_kind == _lib.ACT_GELU and not b.atomics["H"].has_biases
    assert nn.ANINetworks.build(("H",), 16, {"H": (8, 8, 8)}, activation="celu", bias=True).atomics["H"].has_biases


def test_state_dict_keys_match_the_reference_model():
    from torchani_b200 import nn
    rec = fixture("water999_pbc")
    ref_keys = {str(k) for k in rec["state_dict_keys"]}
    prefix = "potentials.nnp.neural_networks."
    ref_nn = {k[len(prefix):] for k in ref_keys if k.startswith(prefix)}
    ours = nn.Ensemble([nn.ANINetworks.default(SYMBOLS, 1008) for _ in range(8)])
    assert set(ours.state_dict().keys()) == ref_nn
    assert not [k for k in ref_nn if k.endswith(".bias")]


def test_mlp_model_activation_field(tmp_path):
    from torchani_b200 import _lib
    assert _lib.MLPModel.activation.offset == 28 and _lib.MLPModel.celu_alpha.offset == 32
    assert "pad_" not in [f[0] for f in _lib.MLPModel._fields_]
    prog = tmp_path / "off.c"
    prog.write_text(
        '#include <stdio.h>\n#include <stddef.h>\n#include "ani_b200.h"\n'
        'int main(){printf("%zu %zu %d %d\\n", offsetof(ani_mlp_model, activation), offsetof(ani_mlp_model, celu_alpha),'
        ' ANI_ACT_CELU, ANI_ACT_GELU);return 0;}\n')
    exe = tmp_path / "off"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    out = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert out == [_lib.MLPModel.activation.offset, _lib.MLPModel.celu_alpha.offset, _lib.ACT_CELU, _lib.ACT_GELU]
    assert C.sizeof(_lib.MLPModel) > 0
