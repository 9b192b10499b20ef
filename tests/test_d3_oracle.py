"""D3 dispersion without a GPU: the float64 restatement (oracle/d3_oracle.py) against the reference-generated fixtures
tests/golden/d3_*.npz, the host-side rules of torchani_b200.potentials.TwoBodyDispersionD3 / models (missing tables,
state-dict keys including the reference's legacy ones, the model cutoff), the converter on a staged reference module,
and the ani_d3_params layout against the header."""
import os
import subprocess

import numpy as np
import pytest
import torch

import oracle.ani_oracle as orc
import oracle.d3_oracle as d3o
from helpers import GOLD, ROOT, golden_inputs, load_golden

SYSTEMS = ["water999_pbc_ani2x", "sevenel_pbc_ani2x", "tightcell_pbc_ani2x", "1c17_chunk_hcnos_ani2x",
           "randbatch_ani2x", "benzene_pbc_ani2x", "water30_pbc_ani2x"]


def params_npz():
    return np.load(os.path.join(GOLD, "d3_params.npz"))


def d3_golden(name):
    z = np.load(os.path.join(GOLD, f"d3_{name}.npz"))
    return {k: z[k] for k in z.files}


def _thin(cell, cutoff):
    return cell is not None and bool((1 / torch.linalg.norm(torch.inverse(cell), dim=0) < cutoff).any())


@pytest.mark.parametrize("name", SYSTEMS)
def test_oracle_matches_the_reference_fixture(name):
    sp, co, cell, pbc = golden_inputs(load_golden(name))
    ref = d3_golden(name)
    cutoff = float(ref["cutoff"])
    nl = "cell_list" if sp.shape[0] == 1 and not _thin(cell, cutoff) else "all_pairs"
    got = d3o.compute(d3o.spec_from_npz(params_npz(), cutoff, "smooth"), sp, co, cell, pbc, nl,
                      stress=cell is not None)
    for key in ("energy", "atomic", "forces") + (("stress",) if cell is not None else ()):
        assert np.abs(got[key].numpy() - ref[f"smooth_{key}"]).max() < 1e-10, key


def test_scan_chain_and_tables():
    z = d3_golden("scan")
    got = d3o.compute(d3o.spec_from_npz(params_npz(), 8.0, "cosine"), torch.tensor(z["species"]),
                      torch.tensor(z["coords"]))
    assert np.abs(got["energy"].numpy() - z["cosine_energy"]).max() < 1e-11
    beyond = z["coords"][:, 1, 0] > 8.0
    assert beyond.any() and (z["smooth_energy"][beyond] == 0).all()
    # the chain term is not small, and one element pair has no valid reference (C6 = eps / eps = 1)
    sp, co, cell, pbc = golden_inputs(load_golden("sevenel_pbc_ani2x"))
    spec = d3o.spec_from_npz(params_npz(), 8.0, "smooth")
    full = d3o.compute(spec, sp, co, cell, pbc, "cell_list")
    direct = d3o.compute(spec, sp, co, cell, pbc, "cell_list", chain=False)
    assert float((full["forces"] - direct["forces"]).abs().max()) > 1e-2 * float(full["forces"].abs().max())
    c6 = torch.tensor(params_npz()["precalc_coeff6"])
    s, f = orc.SYMBOLS_2X.index("S"), orc.SYMBOLS_2X.index("F")
    assert (c6[s, f] <= 0).all() and (c6[f, s] <= 0).all() and (c6[s, s] > 0).any()


def test_module_rules_and_state_dict():
    from torchani_b200 import potentials as P
    z = params_npz()
    S = 7
    with pytest.raises(ValueError, match="from_torchani"):
        P.TwoBodyDispersionD3(orc.SYMBOLS_2X, 1.0, 1.5, 0.37, 4.1, [1.0] * S, [0.5] * S)
    pot = P.TwoBodyDispersionD3(orc.SYMBOLS_2X, 1.0, 1.5, 0.37, 4.1, [1.0] * S, [0.5] * S,
                                coeff6=z["precalc_coeff6"], coordnums_a=z["precalc_coordnums_a"],
                                coordnums_b=z["precalc_coordnums_b"], cutoff=8.0)
    keys = set(pot.state_dict())
    assert keys == {"precalc_coeff6", "precalc_coordnums_a", "precalc_coordnums_b", "sqrt_charge_ab", "covalent_radii",
                    "_damp_fn.cutoff_radii"}
    legacy = {k.replace("_damp_fn.", "_damp_fn_8."): torch.tensor(z[k.split(".")[-1]]).float() for k in keys}
    legacy["_damp_fn_6.cutoff_radii"] = torch.zeros(S, S)
    pot.load_state_dict(legacy)
    assert torch.equal(pot._damp_fn.cutoff_radii, torch.tensor(z["cutoff_radii"]).float())
    p = pot.params()
    r0 = float(z["cutoff_radii"][1, 3]) * 0.37 + 4.1
    assert abs(p.damp6[1][3] - r0 ** 6) < 1e-6 * r0 ** 6
    assert abs(p.c8_scale[0][0] - 3 * float(z["sqrt_charge_ab"][0, 0])) < 1e-5
    t = pot.tables(torch.device("cpu"))
    assert t.shape == (S, S, 25, 4) and torch.equal(t[..., 0], pot.precalc_coeff6.reshape(S, S, 25))


def test_model_cutoff_and_legacy_keys():
    from torchani_b200 import models, potentials as P
    z = params_npz()
    base = models.ANI2x(seed=0)
    pot = P.TwoBodyDispersionD3(base.symbols, 1.0, 1.5, 0.37, 4.1, [1.0] * 7, [0.5] * 7,
                                coeff6=z["precalc_coeff6"], coordnums_a=z["precalc_coordnums_a"],
                                coordnums_b=z["precalc_coordnums_b"], cutoff=8.0)
    m = models.ANI(base.symbols, base.aev_computer, base.neural_networks, base.energy_shifter, True,
                   {"disp": pot})
    assert m.cutoff == 8.0 and base.cutoff == base.aev_computer.radial.cutoff
    inf = P.TwoBodyDispersionD3(base.symbols, 1.0, 1.5, 0.37, 4.1, [1.0] * 7, [0.5] * 7,
                                coeff6=z["precalc_coeff6"], coordnums_a=z["precalc_coordnums_a"],
                                coordnums_b=z["precalc_coordnums_b"])
    with pytest.raises(ValueError, match="finite cutoff"):
        models.ANI(base.symbols, base.aev_computer, base.neural_networks, base.energy_shifter, True, {"d": inf})
    m2 = models.ANI(base.symbols, base.aev_computer, base.neural_networks, base.energy_shifter, True,
                    {"dispersion_d3": pot})
    old = {}
    for k, v in m2.state_dict().items():
        if k.startswith("potentials.dispersion_d3."):
            k = k.replace("potentials.dispersion_d3.", "potentials.0.").replace("_damp_fn.", "_damp_fn_8.")
        old[k] = v.clone()
    m2.potentials["dispersion_d3"].precalc_coeff6.zero_()
    m2.load_state_dict(old)
    assert torch.equal(m2.potentials["dispersion_d3"].precalc_coeff6, torch.tensor(z["precalc_coeff6"]).float())


def test_from_torchani_of_the_reference_module():
    from oracle import ref_torchani
    if not ref_torchani.available():
        pytest.skip("the reference is not staged")
    ref_torchani.load()
    import torchani.potentials.dftd3 as dftd3
    from oracle.make_d3_golden import synthetic_c6_tables
    from torchani_b200 import potentials as P
    saved = dftd3._load_c6_constants
    dftd3._load_c6_constants = synthetic_c6_tables
    try:
        ref = dftd3.TwoBodyDispersionD3(orc.SYMBOLS_2X, 1.0, 1.5, 0.37, 4.1, cutoff=8.0, cutoff_fn="cosine")
    finally:
        dftd3._load_c6_constants = saved
    conv = P.from_torchani(ref)
    assert isinstance(conv, P.TwoBodyDispersionD3) and conv.cutoff == 8.0 and conv.cutoff_fn == "cosine"
    for k, v in ref.state_dict().items():
        assert torch.allclose(conv.state_dict()[k], v.float(), rtol=1e-6, atol=0), k
    assert (conv._s6, conv._s8, conv._damp_fn._a1, conv._damp_fn._a2) == (1.0, 1.5, 0.37, 4.1)


def test_d3_params_layout_matches_header(tmp_path):
    from torchani_b200 import _lib
    import ctypes as C
    prog = tmp_path / "d3.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "ani_b200.h"\n'
                    'int main(){printf("%zu %zu %zu %zu %zu\\n", sizeof(ani_d3_params), offsetof(ani_d3_params, k3),'
                    ' offsetof(ani_d3_params, rcov), offsetof(ani_d3_params, damp8), offsetof(ani_d3_params, c8_scale));'
                    'return 0;}\n')
    exe = tmp_path / "d3"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    D = _lib.D3Params
    assert got == [C.sizeof(D), D.k3.offset, D.rcov.offset, D.damp8.offset, D.c8_scale.offset]
