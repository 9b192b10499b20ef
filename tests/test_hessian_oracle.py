"""Hessian infrastructure without a GPU: the float64 oracle's Hessians against finite differences of its forces,
``torchani_b200.grad.vibrational_analysis`` against the oracle's float64 restatement in every mode kind and unit,
the chunk planner of Engine.hessian, the rejections that need no device, and the per-atom restatements
``center_aev`` / ``center_pair_energy`` that the kernel-level GPU tests differentiate."""
import numpy as np
import pytest
import torch

import oracle.ani_oracle as orc
import oracle.hessian_oracle as hor


def _water():
    sp = torch.tensor([[3, 0, 0]])
    co = torch.tensor([[[0.0, 0.0, 0.1173], [0.0, 0.7572, -0.4692], [0.0, -0.7572, -0.4692]]], dtype=torch.float64)
    return sp, co


def _energy():
    spec = orc.aev_spec_1x()
    model = orc.Model(spec, orc.SYMBOLS_1X, orc.make_weights(orc.SYMBOLS_1X, orc.DIMS_1X, spec.out_dim, 2, 1234,
                                                             torch.float64), {}, "all_pairs")
    sp, co = _water()
    return hor.energy_fn(model, sp), co


def test_oracle_hessian_matches_central_differences_of_forces():
    energy, co = _energy()
    h = hor.hessian(energy, co)[0]
    eps = 1e-5
    for k in range(9):
        d = torch.zeros_like(co).view(-1)
        d[k] = eps
        xp = (co.view(-1) + d).view_as(co).requires_grad_(True)
        xm = (co.view(-1) - d).view_as(co).requires_grad_(True)
        (gp,) = torch.autograd.grad(energy(xp).sum(), xp)
        (gm,) = torch.autograd.grad(energy(xm).sum(), xm)
        fd = ((gp - gm) / (2 * eps)).view(-1)
        assert float((h[k] - fd).abs().max()) < 1e-6 * (1.0 + float(h.abs().max()))
    assert float((h - h.t()).abs().max()) < 1e-12 * float(h.abs().max())
    hv = hor.hvp(energy, co, torch.eye(9, dtype=torch.float64).view(9, 1, 3, 3))
    assert float((hv.view(9, 9) - h).abs().max()) < 1e-12 * float(h.abs().max())


@pytest.mark.parametrize("kind", ["mdu", "mdn", "mwn"])
@pytest.mark.parametrize("unit", ["cm^-1", "meV"])
def test_vibrational_analysis_matches_the_float64_restatement(kind, unit):
    from torchani_b200 import grad
    energy, co = _energy()
    h = hor.hessian(energy, co)
    masses = torch.tensor([[15.999, 1.008, 1.008]], dtype=torch.float64)
    got = grad.vibrational_analysis(masses, h, kind, unit)
    ref = hor.vibrational_analysis(masses[0].numpy(), h[0].numpy(), kind, unit)
    # the three translations have eigenvalues at the rounding level of H: nearly degenerate, their modes are not
    # determined and their frequencies are sqrt(rounding); the other modes are compared (away from a minimum the
    # rotations have a curvature of their own)
    vib = np.abs(ref["freqs"]) > 1e-3 * np.abs(ref["freqs"]).max()
    assert vib.sum() >= 3
    for k in ("freqs", "fconstants", "rmasses"):
        np.testing.assert_allclose(getattr(got, k).numpy()[vib], ref[k][vib], rtol=1e-10)
    g, r = got.modes.numpy()[vib].reshape(int(vib.sum()), -1), ref["modes"][vib].reshape(int(vib.sum()), -1)
    sign = np.sign(np.sum(g * r, axis=1, keepdims=True))
    np.testing.assert_allclose(g * sign, r, atol=1e-10 * np.abs(r).max())


def test_unit_constants_follow_codata_2014():
    from torchani_b200 import grad
    assert abs(grad.HARTREE_TO_EV / 27.211386024367243 - 1) < 1e-15
    assert abs(grad.INVCM_TO_EV / 0.0001239841973964072 - 1) < 1e-15
    assert abs(grad.SQRT_MHESSIAN_TO_INVCM / hor.SQRT_MHESSIAN_TO_INVCM - 1) < 1e-14
    assert abs(grad.MHESSIAN_TO_FCONST / hor.MHESSIAN_TO_FCONST - 1) < 1e-14


def test_vibrational_analysis_rejections():
    from torchani_b200 import grad
    h = torch.eye(6, dtype=torch.float64).unsqueeze(0)
    m = torch.ones(1, 2, dtype=torch.float64)
    with pytest.raises(ValueError, match="unit"):
        grad.vibrational_analysis(m, h, "mdu", "eV")
    with pytest.raises(ValueError, match="mode kind"):
        grad.vibrational_analysis(m, h, "xyz")
    with pytest.raises(ValueError, match="one molecule"):
        grad.vibrational_analysis(m.repeat(2, 1), h.repeat(2, 1, 1))
    x = torch.zeros(1, 2, 3)
    with pytest.raises(ValueError, match="require grad"):
        grad.forces(x.sum(), x)


def test_hessian_chunks_fit_the_row_budget():
    from torchani_b200.engine import _hessian_chunks
    rng = np.random.default_rng(3)
    cnt = rng.integers(0, 60, size=300)
    species = rng.integers(0, 7, size=300).astype(np.int32)
    plans = list(_hessian_chunks(cnt, species, 4096))
    assert sorted(int(a) for p in plans for a in p.atom) == list(range(300))
    for p in plans:
        assert p.rows % 64 == 0 and (p.rows <= 4096 or len(p.atom) == 1)
        for k, a in enumerate(p.atom):
            r0 = int(p.row_off[k])
            assert (p.row_slot[r0:r0 + 3 * cnt[a]] == k).all()
            assert p.tile_species[r0 // 64] == species[a] and p.tile_species[(r0 + max(3 * cnt[a], 1) - 1) // 64] == species[a]
        assert int((p.row_slot >= 0).sum()) == 3 * int(cnt[p.atom].sum())
        assert p.block_floats >= int((9 * cnt[p.atom] ** 2).sum())
    with pytest.raises(ValueError, match="row_budget"):
        list(_hessian_chunks(cnt, species, 32))


def test_create_graph_guard():
    from torchani_b200 import _lib
    with torch.enable_grad():
        with pytest.raises(NotImplementedError, match="second derivatives"):
            _lib.forbid_create_graph("x")
    with torch.no_grad():
        _lib.forbid_create_graph("x")


FIXTURES = ["ch4_1x", "water_1x", "sevenel_2x", "randbatch_2x", "gelu_xtb", "zbl_2x"]


def _fixture(name):
    import os
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", f"hessian_{name}.npz"))
    return {k: z[k] for k in z.files}


def _fixture_energy(name, species, rec):
    import oracle.gelu_oracle as gor
    import oracle.pair_oracle as porc
    if name == "gelu_xtb":
        spec = gor.gelu_spec()
        model = orc.Model(spec, gor.SYMBOLS, gor.make_weights(gor.SYMBOLS, orc.DIMS_2X, spec.out_dim, 8, 4321), {},
                          "all_pairs")   # (float32 weights, as the fixture's model holds them)
        tables = tuple(torch.tensor(rec["xtb_" + k]) for k in ("y_ab", "sqrt_alpha_ab", "k_rep_ab"))
        return hor.energy_fn(model, species, "gelu", [porc.PairSpec("xtb", spec.rcr, "smooth", tables)])
    kind = name.split("_")[-1]
    symbols, dims, spec = ((orc.SYMBOLS_2X, orc.DIMS_2X, orc.aev_spec_2x()) if kind == "2x"
                           else (orc.SYMBOLS_1X, orc.DIMS_1X, orc.aev_spec_1x()))
    model = orc.Model(spec, symbols, orc.make_weights(symbols, dims, spec.out_dim, 8, 1234, torch.float64), {},
                      "all_pairs")
    pairs = [porc.zbl_spec(symbols, spec.rcr, "cosine")] if name == "zbl_2x" else []
    return hor.energy_fn(model, species, "celu", pairs)


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_reproduces_the_reference_hessians(name):
    rec = _fixture(name)
    species = torch.tensor(rec["species"])
    h = hor.hessian(_fixture_energy(name, species, rec), torch.tensor(rec["coords"]))
    ref = rec["hessian"]
    assert float(np.abs(h.numpy() - ref).max()) < 1e-10 * float(np.abs(ref).max())


@pytest.mark.parametrize("name", FIXTURES)
def test_vibrational_analysis_reproduces_the_reference(name):
    from torchani_b200 import grad
    rec = _fixture(name)
    species, masses, hess = rec["species"], rec["masses"], torch.tensor(rec["hessian"])
    for c in range(species.shape[0]):
        idx = np.nonzero(species[c] >= 0)[0]
        cols = np.stack([3 * idx + k for k in range(3)], 1).reshape(-1)
        hc = hess[c][cols][:, cols].unsqueeze(0)
        m = torch.tensor(masses[c, idx]).unsqueeze(0)
        for kind in ("mdu", "mdn", "mwn"):
            for u, unit in (("cm", "cm^-1"), ("mev", "meV")):
                got = grad.vibrational_analysis(m, hc, kind, unit)
                ref = {f: rec[f"vib_{c}_{kind}_{u}_{f}"] for f in ("freqs", "modes", "fconstants", "rmasses")}
                # the translations sit at the rounding level of H (nearly degenerate, modes undetermined)
                keep = np.abs(ref["freqs"]) > 1e-3 * np.abs(ref["freqs"]).max()
                for f in ("freqs", "fconstants", "rmasses"):
                    np.testing.assert_allclose(getattr(got, f).numpy()[keep], ref[f][keep], rtol=1e-10,
                                               err_msg=f"{name} {c} {kind} {unit} {f}")
                g, r = got.modes.numpy()[keep].reshape(int(keep.sum()), -1), ref["modes"][keep].reshape(int(keep.sum()), -1)
                sign = np.sign(np.sum(g * r, axis=1, keepdims=True))
                np.testing.assert_allclose(g * sign, r, atol=1e-10 * np.abs(r).max(), err_msg=f"{name} {c} {kind}")


# ---- per-atom restatements: center_aev and center_pair_energy ------------------------------------------------------
def _aev_specs():
    """ANI-1x, ANI-2x, the smooth-cutoff GELU spec and test_gpu_aev's covering configurations (ShfA x ShfZ = 32)."""
    import oracle.gelu_oracle as gor
    from test_gpu_aev import CONFIGS, spec_of
    specs = {"1x": orc.aev_spec_1x(), "2x": orc.aev_spec_2x(), "gelu": gor.gelu_spec()}
    specs.update({c.name: spec_of(c) for c in CONFIGS})
    return specs


AEV_SPECS = _aev_specs()


def _cluster(n, S, radius, seed, min_dist=0.9):
    """n float64 points in a ball (random sequential placement), random elements 0..S-1."""
    rng = np.random.default_rng(seed)
    pts = np.zeros((0, 3))
    while len(pts) < n:
        p = rng.uniform(-radius, radius, 3)
        if np.linalg.norm(p) <= radius and (len(pts) == 0 or np.linalg.norm(pts - p, axis=1).min() >= min_dist):
            pts = np.vstack([pts, p])
    return torch.tensor(rng.integers(0, S, n)).view(1, -1), torch.tensor(pts).view(1, -1, 3)


@pytest.mark.parametrize("name", list(AEV_SPECS))
def test_center_aev_matches_aev_from_neighbors(name):
    spec = AEV_SPECS[name]
    sp, co = _cluster(18, spec.num_species, 3.2, 11)
    ref = orc.aev_from_neighbors(spec, sp, orc.neighborlist("all_pairs", spec.rcr, sp, co))[0]
    x = co[0]
    rng = np.random.default_rng(5)
    for i in range(x.shape[0]):
        d = (x - x[i]).norm(dim=-1)
        nbrs = [j for j in rng.permutation(x.shape[0]).tolist() if j != i and float(d[j]) <= spec.rcr]
        got = hor.center_aev(spec, int(sp[0, i]), sp[0, nbrs].tolist(), x[nbrs] - x[i])
        assert float((got - ref[i]).abs().max()) <= 1e-12 * (1.0 + float(ref[i].abs().max())), (name, i)


def test_center_aev_derivatives_through_torch_func():
    """jacrev of center_aev (the per-stage references of the GPU kernels) equals the full-system Jacobian with respect
    to the neighbours' positions, and is zero in every column block a neighbour cannot touch."""
    spec = orc.aev_spec_2x()
    sp, co = _cluster(10, 7, 2.6, 3)
    x, i = co[0], 4
    nbrs = [j for j in range(10) if j != i]
    jac = torch.func.jacrev(lambda v: hor.center_aev(spec, int(sp[0, i]), sp[0, nbrs].tolist(), v))(x[nbrs] - x[i])

    def row(xx):
        return orc.aev_from_neighbors(spec, sp, orc.neighborlist("all_pairs", spec.rcr, sp, xx.view(1, -1, 3)))[0, i]
    full = torch.autograd.functional.jacobian(row, x)
    assert float((jac - full[:, nbrs]).abs().max()) <= 1e-12 * float(full.abs().max())
    nr = len(spec.shf_r)
    for n, j in enumerate(nbrs):
        other = torch.ones(spec.radial_len, dtype=torch.bool)
        other[int(sp[0, j]) * nr:(int(sp[0, j]) + 1) * nr] = False
        assert float(jac[:spec.radial_len][other, n].abs().sum()) == 0.0


@pytest.mark.parametrize("kind", ["xtb", "zbl"])
@pytest.mark.parametrize("fn", ["cosine", "smooth"])
@pytest.mark.parametrize("cutoff", [3.0, 4.6, 5.1])
def test_center_pair_energy_sums_to_energies_from_neighbors(kind, fn, cutoff):
    import os
    import oracle.pair_oracle as porc
    if kind == "xtb":
        z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pair_params.npz"))
        pair = porc.PairSpec("xtb", cutoff, fn, tuple(torch.tensor(z[k]) for k in ("y_ab", "sqrt_alpha_ab", "k_rep_ab")))
    else:
        pair = porc.zbl_spec(orc.SYMBOLS_2X, cutoff, fn)
    sp, co = _cluster(16, 7, 3.4, 8)
    ref = porc.energies_from_neighbors(pair, sp, orc.neighborlist("all_pairs", cutoff, sp, co))[0]
    x = co[0]
    tot = 0.0
    for i in range(x.shape[0]):
        nbrs = [j for j in range(x.shape[0]) if j != i]
        tot = tot + hor.center_pair_energy(pair, int(sp[0, i]), sp[0, nbrs].tolist(), x[nbrs] - x[i])
    assert abs(float(tot - ref)) <= 1e-12 * abs(float(ref))
