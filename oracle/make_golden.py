"""Generate tests/golden/*.npz from the REAL reference (aiqm/torchani under /root/reference).

TEST INFRASTRUCTURE ONLY; runs only in the build container (the GPU box has no
/root/reference).  For every case it
  1. builds the reference modules (AEVComputer / ANINetworks / Ensemble, fp64) and loads
     the deterministic synthetic weights of ``ani_oracle.make_weights`` into them,
  2. runs the reference pure-PyTorch path (strategy="pyaev") for AEVs, per-member atomic
     energies and autograd forces,
  3. checks the oracle restatement against it (this is the "pin" of the oracle), and
  4. stores inputs + reference outputs as a small fixture.

Usage:  python oracle/make_golden.py            (writes tests/golden/)
        python oracle/make_golden.py --case sevenel_pbc_ani2x   (only the named cases, comma-separated)
"""
from __future__ import annotations

import os
import sys
import types
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
REF = "/root/reference"
RES = os.path.join(REF, "tests", "resources")


def import_reference():
    """The reference only fails to import because h5py is absent; a 3-attribute stub is
    enough for the hot path (SURVEY.md 8c)."""
    if "h5py" not in sys.modules:
        try:
            import h5py  # noqa: F401
        except ImportError:
            stub = types.ModuleType("h5py")
            stub.Group = stub.File = stub.Dataset = type("_Stub", (), {})
            sys.modules["h5py"] = stub
    os.environ.setdefault("TORCHANI_NO_WARN_EXTENSIONS", "1")
    if REF not in sys.path:
        sys.path.insert(0, REF)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        import torchani  # noqa: F401
    return torchani


def read_xyz(path, frame=0):
    """Minimal (ext)xyz reader: returns symbols, coords (n,3), cell (3,3) or None."""
    with open(path) as f:
        lines = f.read().splitlines()
    pos = 0
    for _ in range(frame + 1):
        n = int(lines[pos].split()[0])
        comment = lines[pos + 1]
        body = lines[pos + 2: pos + 2 + n]
        pos += 2 + n
    cell = None
    if 'Lattice="' in comment:
        vals = comment.split('Lattice="')[1].split('"')[0].split()
        cell = np.array([float(v) for v in vals]).reshape(3, 3)
    sym = [ln.split()[0] for ln in body]
    xyz = np.array([[float(v) for v in ln.split()[1:4]] for ln in body])
    return sym, xyz, cell


def build_reference(torchani, kind, weights, neighborlist, symbols, dims):
    from torchani.aev import AEVComputer
    from torchani.nn import ANINetworks, Ensemble

    mk = AEVComputer.like_2x if kind == "2x" else AEVComputer.like_1x
    aevc = mk(neighborlist=neighborlist, strategy="pyaev").double()
    members = []
    for w_m in weights:
        net = (ANINetworks.like_2x() if kind == "2x" else ANINetworks.like_1x()).double()
        with torch.no_grad():
            for s in symbols:
                an = net.atomics[s]
                lins = list(an.layers) + [an.final_layer]
                for lin, (w, b) in zip(lins, w_m[s]):
                    assert lin.weight.shape == w.shape, (s, lin.weight.shape, w.shape)
                    lin.weight.copy_(w.double())
                    lin.bias.copy_(b.double())
        members.append(net)
    return aevc, Ensemble(members)


def run_reference(aevc, ens, idx, coords, cell, pbc):
    coords = coords.double().clone().requires_grad_(True)
    cell_d = None if cell is None else cell.double()
    nb = aevc.neighborlist(aevc.radial.cutoff, idx, coords, cell_d, pbc)
    aev = aevc.compute_from_neighbors(idx, coords, nb)
    e_m = ens(idx, aev, atomic=True, ensemble_values=True)  # (M, C, A)
    e_nn = e_m.mean(0).sum(-1)
    forces = -torch.autograd.grad(e_nn.sum(), coords)[0]
    return {
        "aev": aev.detach(), "member_atomic": e_m.detach(), "energy_nn": e_nn.detach(),
        "forces": forces, "num_pairs": nb.indices.shape[1],
        "pairs": nb.indices.detach(), "distances": nb.distances.detach(),
    }


def main(only=None):
    """``only``: names of the cases to (re)write; all of them by default."""
    torchani = import_reference()
    import oracle.ani_oracle as orc

    out_dir = os.path.join(ROOT, "tests", "golden")
    os.makedirs(out_dir, exist_ok=True)
    sym2 = {s: i for i, s in enumerate(orc.SYMBOLS_2X)}
    sym1 = {s: i for i, s in enumerate(orc.SYMBOLS_1X)}
    T = torch.tensor
    pbc3 = T([True, True, True])
    cases = []

    # 1. ANI-1x single CH4 (tests/resources/CH4-5.xyz frame 0; BASELINE config 1)
    s, x, _ = read_xyz(os.path.join(RES, "CH4-5.xyz"))
    cases.append(dict(name="ch4_ani1x", kind="1x", nl="all_pairs",
                      idx=T([[sym1[a] for a in s]]), coords=T(x).unsqueeze(0), cell=None, pbc=None))
    # 2. the hard-coded 2x5 KAT of tests/test_cuaev.py:38-63 (one padded atom)
    kat = T([[[0.03192167, 0.00638559, 0.01301679], [-0.83140486, 0.39370209, -0.26395324],
              [-0.66518241, -0.84461308, 0.20759389], [0.45554739, 0.54289633, 0.81170881],
              [0.66091919, -0.16799635, -0.91037834]],
             [[-4.1862600, 0.0575700, -0.0381200], [-3.1689400, 0.0523700, 0.0200000],
              [-4.4978600, 0.8211300, 0.5604100], [-4.4978700, -0.8000100, 0.4155600],
              [0.0, 0.0, 0.0]]], dtype=torch.float64)
    cases.append(dict(name="kat2x5_ani2x", kind="2x", nl="all_pairs",
                      idx=T([[1, 0, 0, 0, 0], [2, 0, 0, 0, -1]]), coords=kat, cell=None, pbc=None))
    # 3-5. periodic fixtures shipped with the reference tests
    for fname, name in [("water-0.8nm.xyz", "water30_pbc_ani2x"), ("benzene.xyz", "benzene_pbc_ani2x"),
                        ("tight_cell.xyz", "tightcell_pbc_ani2x")]:
        s, x, cell = read_xyz(os.path.join(RES, fname))
        cases.append(dict(name=name, kind="2x", nl="cell_list", idx=T([[sym2[a] for a in s]]),
                          coords=T(x).unsqueeze(0), cell=T(cell), pbc=pbc3))
    # 6. random padded batch in the style of torchani/_testing.py:115-155 (no PBC)
    g = torch.Generator().manual_seed(7)
    rb_coords = torch.rand(8, 12, 3, generator=g, dtype=torch.float64) * 5.0 + 1e-3
    rb_idx = torch.randint(0, 4, (8, 12), generator=g)
    rb_idx[1, 9:] = -1
    rb_idx[5, 4:] = -1
    rb_idx[7, 11:] = -1
    cases.append(dict(name="randbatch_ani2x", kind="2x", nl="all_pairs", idx=rb_idx, coords=rb_coords,
                      cell=None, pbc=None))
    # 7. synthetic periodic water box, 999 atoms (BASELINE config 2) -- compact fixture
    _, widx, wcoords, wcell, wpbc = orc.water_box(333, seed=0, dtype=torch.float64)
    cases.append(dict(name="water999_pbc_ani2x", kind="2x", nl="cell_list", idx=widx, coords=wcoords,
                      cell=wcell, pbc=wpbc, compact=True))
    # 8. triclinic periodic protein 6W8H (3410 atoms) -- compact fixture
    s, x, cell = read_xyz(os.path.join(RES, "6W8H.xyz"))
    cases.append(dict(name="6w8h_triclinic_ani2x", kind="2x", nl="cell_list", idx=T([[sym2[a] for a in s]]),
                      coords=T(x).unsqueeze(0), cell=T(cell), pbc=pbc3, compact=True))
    # 9. non-periodic protein fragment small.xyz (264 atoms), cell_list without PBC
    s, x, _ = read_xyz(os.path.join(RES, "small.xyz"))
    cases.append(dict(name="small264_nopbc_ani2x", kind="2x", nl="cell_list", idx=T([[sym2[a] for a in s]]),
                      coords=T(x).unsqueeze(0), cell=None, pbc=None, compact=True))
    # 11. periodic box with all seven ANI-2x elements (H C N O S F Cl): every element pair, every AEV block live
    sidx, scoords, scell, spbc = orc.seven_element_box(1200, seed=11)
    cases.append(dict(name="sevenel_pbc_ani2x", kind="2x", nl="cell_list", idx=sidx, coords=scoords, cell=scell,
                      pbc=spbc, compact=True))
    if only:
        cases = [c for c in cases if c["name"] in only]

    seed = 1234
    w2 = orc.make_weights(orc.SYMBOLS_2X, orc.DIMS_2X, 1008, 8, seed, torch.float64)
    w1 = orc.make_weights(orc.SYMBOLS_1X, orc.DIMS_1X, 384, 8, seed, torch.float64)
    proj_rng = np.random.default_rng(99)
    for c in cases:
        kind = c["kind"]
        symbols, dims, w = (orc.SYMBOLS_2X, orc.DIMS_2X, w2) if kind == "2x" else (orc.SYMBOLS_1X, orc.DIMS_1X, w1)
        aevc, ens = build_reference(torchani, kind, w, c["nl"], symbols, dims)
        ref = run_reference(aevc, ens, c["idx"], c["coords"], c["cell"], c["pbc"])
        # ---- pin the oracle against the reference on this case
        spec = orc.aev_spec_2x() if kind == "2x" else orc.aev_spec_1x()
        sae = {s_: orc.GSAES_WB97X_631GD[s_] for s_ in symbols}
        model = orc.Model(spec, symbols, w, sae, c["nl"])
        cell_d = None if c["cell"] is None else c["cell"].double()
        mine = orc.compute(model, c["idx"], c["coords"].double(), cell_d, c["pbc"])
        errs = {
            "aev": (mine["aev"] - ref["aev"]).abs().max().item(),
            "member_atomic": (mine["member_atomic"] - ref["member_atomic"]).abs().max().item(),
            "forces": (mine["forces"] - ref["forces"]).abs().max().item(),
        }
        assert int(mine["num_pairs"]) == ref["num_pairs"], (c["name"], mine["num_pairs"], ref["num_pairs"])
        assert errs["aev"] < 1e-11 and errs["member_atomic"] < 1e-11 and errs["forces"] < 1e-11, (c["name"], errs)
        print(f"{c['name']:28s} pairs={ref['num_pairs']:7d} oracle-vs-reference max-abs {errs}")
        # ---- write fixture
        n_feat = ref["aev"].shape[-1]
        proj = proj_rng.standard_normal((n_feat, 4))
        rec = dict(
            kind=kind, neighborlist=c["nl"], weight_seed=seed,
            species=c["idx"].numpy(), coords=c["coords"].double().numpy(),
            cell=np.zeros((0, 3)) if c["cell"] is None else c["cell"].double().numpy(),
            pbc=np.zeros(0, dtype=bool) if c["pbc"] is None else c["pbc"].numpy(),
            num_pairs=ref["num_pairs"], member_atomic=ref["member_atomic"].numpy(),
            energy_nn=ref["energy_nn"].numpy(), forces=ref["forces"].numpy(),
            aev_proj_matrix=proj, aev_proj=ref["aev"].numpy() @ proj,
            aev_rowsum=ref["aev"].numpy().sum(-1),
        )
        if not c.get("compact"):
            rec["aev"] = ref["aev"].numpy()
            order = np.lexsort((ref["pairs"][1].numpy(), ref["pairs"][0].numpy()))
            rec["pairs"] = ref["pairs"].numpy()[:, order]
            rec["distances"] = ref["distances"].numpy()[order]
        np.savez_compressed(os.path.join(out_dir, c["name"] + ".npz"), **rec)

    if only:
        return
    # ---- loop-level oracle vs vectorised oracle on tiny systems (independent restatement)
    spec = orc.aev_spec_2x()
    s, x, cell = read_xyz(os.path.join(RES, "water-0.8nm.xyz"))
    idx = [sym2[a] for a in s]
    loop = orc.aev_loops(spec, idx, x, cell)
    nb = orc.cell_list(spec.rcr, T([idx]), T(x).unsqueeze(0), T(cell), pbc3)
    vec = orc.aev_from_neighbors(spec, T([idx]), nb)[0].numpy()
    print("loop-vs-vector oracle (water30 pbc) max-abs", np.abs(loop - vec).max())
    assert np.abs(loop - vec).max() < 1e-12


def main_stress():
    """Stress fixture: the reference's "f dot r" stress (ase.py:118-131,164-168) computed with the real
    reference modules on its periodic test structures, and the pin of the oracle's strain-derivative
    stress (ani_oracle.compute(..., stress=True), ase.py:110-121,170-173) against it.
    Usage:  python oracle/make_golden.py --stress   (writes tests/golden/stress_pbc_ani2x.npz)"""
    torchani = import_reference()
    from torchani.neighbors import Neighbors
    import oracle.ani_oracle as orc

    sym2 = {s: i for i, s in enumerate(orc.SYMBOLS_2X)}
    pbc3 = torch.tensor([True, True, True])
    w2 = orc.make_weights(orc.SYMBOLS_2X, orc.DIMS_2X, 1008, 8, 1234, torch.float64)
    aevc, ens = build_reference(torchani, "2x", w2, "cell_list", orc.SYMBOLS_2X, orc.DIMS_2X)
    sae = {s_: orc.GSAES_WB97X_631GD[s_] for s_ in orc.SYMBOLS_2X}
    model = orc.Model(orc.aev_spec_2x(), orc.SYMBOLS_2X, w2, sae, "cell_list")
    rec = {}
    for fname, name in [("water-0.8nm.xyz", "water30_pbc_ani2x"), ("benzene.xyz", "benzene_pbc_ani2x"),
                        ("tight_cell.xyz", "tightcell_pbc_ani2x")]:
        s, x, cell = read_xyz(os.path.join(RES, fname))
        idx = torch.tensor([[sym2[a] for a in s]])
        coords = torch.tensor(x).unsqueeze(0).double()
        cell_t = torch.tensor(cell).double()
        nb = aevc.neighborlist(aevc.radial.cutoff, idx, coords, cell_t, pbc3)
        diff = nb.diff_vectors.detach().clone().requires_grad_(True)
        nb2 = Neighbors(nb.indices, diff.norm(2, -1), diff)
        aev = aevc.compute_from_neighbors(idx, coords, nb2)
        energy = ens(idx, aev).sum()
        (dEdR,) = torch.autograd.grad(energy, diff)
        volume = torch.det(cell_t).abs()
        stress_ref = (dEdR.transpose(0, 1) @ diff.detach() / volume).detach()     # ase.py:164-168
        # oracle: strain derivative on the atoms wrapped into the cell (map_to_central detaches the cell)
        wrapped = coords - torch.floor(coords @ torch.linalg.inv(cell_t)) @ cell_t
        mine = orc.compute(model, idx, wrapped, cell_t, pbc3, stress=True)["stress"]
        err = float((mine - stress_ref).abs().max())
        print(f"{name:24s} |stress|max {float(stress_ref.abs().max()):.3e}  oracle-vs-reference max-abs {err:.2e}")
        assert err < 1e-12, (name, err)
        rec[name] = stress_ref.numpy()
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "stress_pbc_ani2x.npz"), **rec)


if __name__ == "__main__":
    if "--stress" in sys.argv:
        main_stress()
    elif "--case" in sys.argv:
        main(only=sys.argv[sys.argv.index("--case") + 1].split(","))
    else:
        main()
