"""Shared helpers for the test-suite (oracle models, golden loading, tolerances)."""
import os

import numpy as np
import torch

import oracle.ani_oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
GOLDEN_CASES = ["ch4_ani1x", "kat2x5_ani2x", "water30_pbc_ani2x", "benzene_pbc_ani2x", "tightcell_pbc_ani2x",
                "randbatch_ani2x", "small264_nopbc_ani2x", "water999_pbc_ani2x", "6w8h_triclinic_ani2x", "1c17_chunk_hcnos_ani2x",
                "sevenel_pbc_ani2x"]

# Parity bars (BASELINE.json north_star): AEV and atomic energies within 1e-5 relative, forces within
# 1e-4 Ha/A, judged against the float64 oracle.  "Relative" is applied element-wise with an absolute
# floor at 1e-5 of the tensor's scale (|AEV| ~ O(1), |e_atomic| ~ O(0.1)).
AEV_RTOL, AEV_ATOL = 1e-5, 1e-5
E_RTOL, E_ATOL = 1e-5, 1e-6
F_ATOL = 1e-4

_models = {}


def oracle_model(kind, dtype=torch.float32, neighborlist="cell_list", members=8):
    key = (kind, dtype, members)
    if key not in _models:
        if kind == "2x":
            spec, symbols, dims = orc.aev_spec_2x(), orc.SYMBOLS_2X, orc.DIMS_2X
        else:
            spec, symbols, dims = orc.aev_spec_1x(), orc.SYMBOLS_1X, orc.DIMS_1X
        w = orc.make_weights(symbols, dims, spec.out_dim, members, 1234, dtype)
        sae = {s: orc.GSAES_WB97X_631GD[s] for s in symbols}
        _models[key] = orc.Model(spec, symbols, w, sae, neighborlist)
    return _models[key]._replace(neighborlist=neighborlist)


def load_golden(name):
    z = np.load(os.path.join(GOLD, name + ".npz"))
    rec = {k: z[k] for k in z.files}
    rec["kind"] = str(rec["kind"])
    rec["neighborlist"] = str(rec["neighborlist"])
    return rec


def golden_inputs(rec, dtype=torch.float64):
    species = torch.tensor(rec["species"])
    coords = torch.tensor(rec["coords"]).to(dtype)
    cell = torch.tensor(rec["cell"]).to(dtype) if rec["cell"].size else None
    pbc = torch.tensor(rec["pbc"]) if rec["pbc"].size else None
    return species, coords, cell, pbc


def assert_close(name, got, ref, rtol, atol):
    got = np.asarray(got, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    err = np.abs(got - ref)
    bound = atol + rtol * np.abs(ref)
    worst = float((err - bound).max()) if err.size else -1.0
    assert worst <= 0, f"{name}: max-abs err {err.max():.3e} (|ref| max {np.abs(ref).max():.3e}), over the bound by {worst:.3e}"
