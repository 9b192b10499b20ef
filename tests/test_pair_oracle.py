"""Pair potentials without a GPU: the float64 restatement (oracle/pair_oracle.py) against the reference-generated
fixtures tests/golden/pair_*.npz, and the host-side rules of torchani_b200.potentials / models (constructor errors, the
cutoff rule, the missing xTB parameter table, state-dict keys, refusing a reference potential that cannot be
converted)."""
import math
import os

import numpy as np
import pytest
import torch

import oracle.ani_oracle as orc
import oracle.pair_oracle as porc
from helpers import GOLD, golden_inputs, load_golden

SYSTEMS = ["water999_pbc_ani2x", "1c17_chunk_hcnos_ani2x", "randbatch_ani2x", "6w8h_triclinic_ani2x"]


def pair_golden(name):
    z = np.load(os.path.join(GOLD, f"pair_{name}.npz"))
    return {k: z[k] for k in z.files}


def xtb_tables():
    z = np.load(os.path.join(GOLD, "pair_params.npz"))
    return tuple(torch.tensor(z[k]) for k in ("y_ab", "sqrt_alpha_ab", "k_rep_ab"))


def spec(kind, fn, cutoff=5.1):
    return porc.PairSpec("xtb", cutoff, fn, xtb_tables()) if kind == "xtb" else porc.zbl_spec(orc.SYMBOLS_2X, cutoff, fn)


@pytest.mark.parametrize("fn", ["cosine", "smooth"])
@pytest.mark.parametrize("kind", ["xtb", "zbl"])
@pytest.mark.parametrize("name", SYSTEMS[:3])
def test_oracle_matches_the_reference_fixture(name, kind, fn):
    sp, co, cell, pbc = golden_inputs(load_golden(name))
    ref = pair_golden(name)
    got = porc.compute(spec(kind, fn), sp, co, cell, pbc, "cell_list" if sp.shape[0] == 1 else "all_pairs",
                       stress=cell is not None)
    for key in ("energy", "atomic", "forces") + (("stress",) if cell is not None else ()):
        assert np.abs(got[key].numpy() - ref[f"{kind}_{fn}_{key}"]).max() < 1e-10, key


def test_oracle_scan_and_ghost_weight():
    z = pair_golden("scan")
    sp, co = torch.tensor(z["species"]), torch.tensor(z["coords"])
    for kind in ("xtb", "zbl"):
        got = porc.compute(spec(kind, "smooth"), sp, co)
        ref = z[f"{kind}_smooth_energy"]
        assert (np.abs(got["energy"].numpy() - ref) / (1.0 + np.abs(ref))).max() < 1e-11
        beyond = co[:, 1, 0].numpy() > 5.1
        assert beyond.any() and (ref[beyond] == 0).all()
    # a pair that touches a ghost atom counts half (potentials/core.py:170-177)
    sp2 = torch.tensor([[0, 3, 0]])
    co2 = torch.tensor([[[0.0, 0, 0], [0.96, 0, 0], [0.3, 0.9, 0]]], dtype=torch.float64)
    nb = orc.all_pairs(5.1, sp2, co2)
    full = porc.pair_energies(spec("xtb", "cosine"), sp2, nb)
    ghost = porc.pair_energies(spec("xtb", "cosine"), sp2, nb, torch.tensor([[False, False, True]]))
    touches = (nb.indices == 2).any(0)
    assert torch.equal(ghost[touches], full[touches] * 0.5) and torch.equal(ghost[~touches], full[~touches])


def test_constructor_rules():
    from torchani_b200 import potentials as P
    sym = orc.SYMBOLS_2X
    with pytest.raises(ValueError, match="not shipped"):
        P.RepulsionXTB(sym, cutoff=5.1)
    with pytest.raises(ValueError, match="one value per symbol"):
        P.RepulsionXTB(sym, alpha=[1.0] * 3, yeff=[1.0] * 7, cutoff=5.1)
    with pytest.raises(ValueError, match="cutoff function"):
        P.RepulsionZBL(sym, cutoff=5.1, cutoff_fn="biweight")
    with pytest.raises(ValueError, match="sum to 1"):
        P.RepulsionZBL(sym, screen_coeffs=(0.5, 0.5, 0.5, 0.5), cutoff=5.1)
    with pytest.raises(ValueError, match="same len"):
        P.RepulsionZBL(sym, screen_coeffs=(0.5, 0.5), cutoff=5.1)
    pot = P.RepulsionXTB(sym, alpha=[2.0] * 7, yeff=[1.5] * 7, krep_hydrogen=1.0, cutoff=5.1, cutoff_fn="cosine")
    assert float(pot.k_rep_ab[0, 0]) == 1.0 and float(pot.k_rep_ab[0, 1]) == 1.5 and float(pot.k_rep_ab[1, 1]) == 1.5
    assert float(pot.y_ab[2, 3]) == 2.25 and float(pot.sqrt_alpha_ab[2, 3]) == 2.0
    p = pot.params()
    assert (p.kind, p.cutoff_fn, p.num_species) == (0, 0, 7) and p.cutoff == np.float32(5.1)
    assert p.a[2][3] == 2.25 and p.c[0][0] == 1.0
    assert P.RepulsionZBL(sym).cutoff_fn == "dummy" and P.RepulsionZBL(sym).params().cutoff_fn == 2
    z = P.RepulsionZBL(sym, cutoff=4.0).params()
    assert z.a[1][3] == 48.0 and z.b[0][0] == pytest.approx(2.0 / 0.8853)


def _model(potentials):
    from torchani_b200 import models
    base = models.ANI2x(seed=0)
    return models.ANI(base.symbols, base.aev_computer, base.neural_networks, base.energy_shifter, True, potentials)


def test_cutoff_rule_and_state_dict_keys():
    from torchani_b200 import potentials as P
    sym = orc.SYMBOLS_2X
    tabs = dict(alpha=[2.0] * 7, yeff=[1.5] * 7)
    with pytest.raises(ValueError, match="radial AEV cutoff"):
        _model({"repulsion_xtb": P.RepulsionXTB(sym, **tabs)})                    # cutoff = inf
    with pytest.raises(ValueError, match="radial AEV cutoff"):
        _model({"repulsion_zbl": P.RepulsionZBL(sym, cutoff=5.2)})
    with pytest.raises(ValueError, match="other symbols"):
        _model({"repulsion_zbl": P.RepulsionZBL(("H", "C"), cutoff=5.1)})
    m = _model({"repulsion_xtb": P.RepulsionXTB(sym, cutoff=5.1, **tabs), "zbl": P.RepulsionZBL(sym, cutoff=3.0)})
    assert list(m.potentials) == ["repulsion_xtb", "zbl"]
    keys = set(m.state_dict())
    assert {"potentials.repulsion_xtb.y_ab", "potentials.repulsion_xtb.sqrt_alpha_ab",
            "potentials.repulsion_xtb.k_rep_ab"} <= keys
    assert not any(k.startswith("potentials.zbl") for k in keys)       # its buffers are not persistent (zbl.py:56-64)
    # round trip, and the legacy numbered keys of arch.py:278-290
    sd = m.state_dict()
    sd["potentials.repulsion_xtb.y_ab"] = sd["potentials.repulsion_xtb.y_ab"] * 2
    m.load_state_dict(sd)
    assert float(m.potentials["repulsion_xtb"].y_ab[0, 0]) == 4.5
    legacy = {k.replace("potentials.repulsion_xtb.", "potentials.1."): v for k, v in m.state_dict().items()}
    m2 = _model({"repulsion_xtb": P.RepulsionXTB(sym, cutoff=5.1, **tabs)})
    m2.load_state_dict(legacy)
    assert float(m2.potentials["repulsion_xtb"].y_ab[0, 0]) == 4.5
    m.set_enabled("zbl", False)
    assert [type(p).__name__ for p in m._enabled_potentials()] == ["RepulsionXTB"]
    assert len(_model(None).state_dict()) == len(m.state_dict()) - 3


def test_from_torchani_refuses_what_it_cannot_convert():
    import oracle.ref_torchani as ref
    if not ref.available():
        pytest.skip("the reference is not staged")
    ref.load()
    from torchani.potentials import PairPotential, RepulsionXTB
    from torchani_b200 import models, potentials as P
    w = orc.make_weights(orc.SYMBOLS_2X, orc.DIMS_2X, 1008, 1, 1234, torch.float32)

    class Square(PairPotential):
        tensors = ["bias"]

        def pair_energies(self, elem_idxs, neighbors):
            return self.bias + neighbors.distances ** 2

    rm = ref.build_model(w, repulsion=True)
    conv = models.from_torchani(rm, device="cpu")
    pot = conv.potentials["repulsion_xtb"]
    assert isinstance(pot, P.RepulsionXTB) and pot.cutoff == 5.1 and pot.cutoff_fn == "smooth"
    assert torch.equal(pot.y_ab, rm.potentials["repulsion_xtb"].y_ab)
    rm.potentials["square"] = Square(orc.SYMBOLS_2X, bias=0.1, cutoff=5.1)
    with pytest.raises(ValueError, match="square"):
        models.from_torchani(rm, device="cpu")
    with pytest.raises(ValueError, match="no CUDA counterpart"):
        P.from_torchani(rm.potentials["square"])
    assert isinstance(P.from_torchani(RepulsionXTB(orc.SYMBOLS_2X, cutoff=math.inf)), P.RepulsionXTB)
