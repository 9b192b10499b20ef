"""The Lennard-Jones and fixed-charge Coulomb pair potentials on the CPU: the float64 oracle
(oracle/lj_coulomb_oracle.py) against every fixture of oracle/make_lj_coulomb_golden.py, the tables each constructor
builds, the conversions of reference modules (skipped where the reference is not staged), and the rejections:
trainable parameters, missing charges, an infinite cutoff on a periodic model."""
import math

import numpy as np
import pytest
import torch

import oracle.ani_oracle as orc
import oracle.lj_coulomb_oracle as lorc
from helpers import GOLD, golden_inputs, load_golden

SYSTEMS = ["water999_pbc_ani2x", "1c17_chunk_hcnos_ani2x", "randbatch_ani2x", "6w8h_triclinic_ani2x"]


def params():
    return dict(np.load(f"{GOLD}/ljc_params.npz"))


def cases(name):
    """(kind, cutoff, fn, key prefix) of every entry of a system's fixture."""
    z = np.load(f"{GOLD}/ljc_{name}.npz")
    out = set()
    for k in z.files:
        kind, rest = next((kd, k[len(kd) + 1:]) for kd in sorted(lorc.KINDS, key=len, reverse=True)
                          if k.startswith(kd + "_"))
        fn, cut = rest.split("_")[:2]
        out.add((kind, math.inf if cut == "inf" else float(cut), fn, f"{kind}_{fn}_{cut}"))
    return sorted(out, key=lambda c: c[3]), z


@pytest.mark.parametrize("name", SYSTEMS)
def test_oracle_reproduces_fixtures(name):
    rec = load_golden(name)
    species, coords, cell, pbc = golden_inputs(rec)
    p = params()
    cs, z = cases(name)
    assert {c[3].split("_")[-1] for c in cs} == ({"8", "12"} if cell is not None else {"8", "12", "inf"})
    assert {c[2] for c in cs} >= {"cosine", "smooth"}
    for kind, cutoff, fn, key in cs:
        spec = lorc.spec_from_params(kind, cutoff, fn, p)
        nl = "cell_list" if species.shape[0] == 1 else "all_pairs"
        got = lorc.compute(spec, species, coords, cell, pbc, nl, stress=cell is not None)
        for k, v in got.items():
            ref = torch.as_tensor(z[f"{key}_{k}"])
            err = float(((v - ref).abs() / (1.0 + ref.abs())).max())
            assert err < 1e-10, (name, key, k, err)


def test_constructor_tables():
    from torchani_b200 import potentials as P
    sym = orc.SYMBOLS_2X
    lj = P.LennardJones(sym, cutoff=8.0, cutoff_fn="cosine")
    p = lj.params()
    assert (p.kind, p.cutoff_fn, p.num_species, p.to_bohr) == (2, 0, 7, 1.0) and p.cutoff == np.float32(8.0)
    assert p.a[0][3] == pytest.approx(0.1 / 627.5094738898777, rel=1e-6) and p.b[2][5] == pytest.approx(1.5)
    eps, sigma = [1e-4 * (k + 1) for k in range(7)], [1.0 + 0.1 * k for k in range(7)]
    for cls, kind in ((P.LennardJones, 2), (P.RepulsionLJ, 3), (P.DispersionLJ, 4)):
        q = cls(sym, eps, sigma).params()
        assert q.kind == kind and q.cutoff_fn == 2 and q.cutoff == 0.0
        assert q.a[1][4] == pytest.approx(math.sqrt(eps[1] * eps[4]), rel=1e-6)
        assert q.b[1][4] == pytest.approx((sigma[1] + sigma[4]) / 2, rel=1e-6)
    qs = [0.4, -0.8, 0.1, 0.3, -0.2, 0.5, -0.6]
    c = P.FixedCoulomb(sym, 2.0, qs, cutoff=12.0).params()
    assert (c.kind, c.cutoff_fn) == (5, 1) and c.to_bohr == np.float32(P.ANGSTROM_TO_BOHR)
    assert c.a[0][1] == pytest.approx(0.4 * -0.8 / 2.0, rel=1e-6)
    eta = [0.5 + 0.05 * k for k in range(7)]
    m = P.FixedMNOK(sym, 2.0, qs, eta).params()
    assert m.kind == 6 and m.a[0][1] == pytest.approx(0.4 * -0.8, rel=1e-6)   # no dielectric, as the reference
    assert m.b[2][6] == pytest.approx(2 / (eta[2] + eta[6]), rel=1e-6)
    # non-persistent buffers: no state-dict keys
    for pot in (lj, P.FixedCoulomb(sym, 1.0, qs), P.FixedMNOK(sym, 1.0, qs, eta)):
        assert not pot.state_dict()


def _model(potentials):
    from torchani_b200 import models
    base = models.ANI2x(seed=0)
    return models.ANI(base.symbols, base.aev_computer, base.neural_networks, base.energy_shifter, True, potentials)


def test_rejections_and_model_cutoffs():
    from torchani_b200 import potentials as P
    sym = orc.SYMBOLS_2X
    with pytest.raises(ValueError, match="trainable"):
        P.LennardJones(sym, trainable=("eps",))
    with pytest.raises(ValueError, match="charges"):
        P.FixedCoulomb(sym)
    with pytest.raises(ValueError, match="eta"):
        P.FixedMNOK(sym, 1.0, [0.1] * 7)
    with pytest.raises(ValueError, match="one value per symbol"):
        P.FixedCoulomb(sym, 1.0, [0.1] * 3)
    # any cutoff in a model, an infinite one included; the model's cutoff is the largest
    m = _model({"lj": P.LennardJones(sym, cutoff=12.0), "coulomb": P.FixedCoulomb(sym, 1.0, [0.1] * 7)})
    assert m.cutoff == math.inf and len(_model(None).state_dict()) == len(m.state_dict())
    assert _model({"lj": P.DispersionLJ(sym, cutoff=10.0)}).cutoff == 10.0
    from torchani_b200.neighbors import effective_periodic_cell, supercell_for_thin_cell
    cell, pbc = torch.eye(3) * 20.0, torch.tensor([True, True, True])
    x = torch.zeros(1, 3, 3)
    with pytest.raises(ValueError, match="infinite cutoff"):
        effective_periodic_cell(x, cell, pbc, m.cutoff)
    with pytest.raises(ValueError, match="infinite cutoff"):
        supercell_for_thin_cell(torch.zeros(1, 3, dtype=torch.long), x, cell, pbc, m.cutoff)


def test_from_torchani_round_trips():
    import oracle.ref_torchani as ref
    if not ref.available():
        pytest.skip("the reference is not staged")
    ref.load()
    import torchani.potentials as rp
    from torchani_b200 import potentials as P
    sym = orc.SYMBOLS_2X
    p = params()
    eps, sigma, q, eta = ([float(v) for v in p[k]] for k in ("eps", "sigma", "charges", "eta"))
    for name in ("LennardJones", "RepulsionLJ", "DispersionLJ"):
        r = getattr(rp, name)(sym, eps, sigma, cutoff=8.0, cutoff_fn="cosine")
        c = P.from_torchani(r)
        assert type(c).__name__ == name and c.cutoff == 8.0 and c.cutoff_fn == "cosine"
        assert torch.equal(c._eps, r._eps.float()) and torch.equal(c._sigma, r._sigma.float())
        with pytest.raises(ValueError, match="trainable"):
            P.from_torchani(getattr(rp, name)(sym, eps, sigma, trainable=("sigma",)))
    r = rp.FixedCoulomb(sym, 2.0, q)
    c = P.from_torchani(r)
    assert isinstance(c, P.FixedCoulomb) and c.cutoff == math.inf and c.cutoff_fn == "dummy" and c._dielectric == 2.0
    assert torch.equal(c._charges, r._charges.float())
    r = rp.FixedMNOK(sym, 2.0, q, eta, cutoff=12.0)
    c = P.from_torchani(r)
    assert isinstance(c, P.FixedMNOK) and c.cutoff_fn == "smooth" and torch.equal(c._eta, r._eta.float())
    # a reference model that carries them converts
    from torchani_b200 import models
    w = orc.make_weights(orc.SYMBOLS_2X, orc.DIMS_2X, 1008, 1, 1234, torch.float32)
    rm = ref.build_model(w)
    rm.potentials["lj"] = rp.LennardJones(sym, eps, sigma, cutoff=8.0)
    rm.potentials["coulomb"] = rp.FixedCoulomb(sym, 1.0, q)
    conv = models.from_torchani(rm, device="cpu")
    assert isinstance(conv.potentials["lj"], P.LennardJones) and isinstance(conv.potentials["coulomb"],
                                                                            P.FixedCoulomb)
    assert conv.cutoff == math.inf
