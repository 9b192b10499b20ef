#!/usr/bin/env python
"""Time the fused step of a GELU bias-free model (ANI-2xr-shaped) beside ANI-2x (CELU with biases).

Three arms, run in the same process and alternated, on the same seeded inputs (energy + forces, 8-member ensembles,
Engine.step graph-replayed, default launch selection):

    celu       ANI-2x: the AEV constants, widths and CELU networks of models.ANI2x, seeded synthetic weights
    gelu       ANI-2xr-shaped, networks only: simple_ani's AEV (cover_linearly 0.9-5.2 A, smooth cutoff) and
               ANINetworks.default (ANI-2x widths, GELU, no biases), seeded bias-free weights
    gelu_xtb   the same with xTB repulsion at 5.2 A (the parameter tensors of tests/golden/pair_params.npz)

Workloads: the 9 999-atom periodic water box and the GDB-like padded batch of 256 conformers.  Before anything is
timed every arm's energies and forces are compared with the float64 oracle (oracle/ani_oracle.py, gelu_oracle.py,
pair_oracle.py)
on the float32-rounded inputs: 2e-7 |E| + 2e-7 Ha per atom, forces 1e-4 + 1e-5 |F| Ha/A; arms that disagree are not
timed and the script exits non-zero.  A 256 MiB buffer is overwritten before every timed arm (L2 flush, untimed); CUDA events bracket
each arm.  Afterwards a profiled pass of 10 steps per arm gives Engine.stage_times_ms, the per-stage device times.
Output: median and spread per arm, the stage times, the device name and power limit, as JSON in --out.

    python tools/gelu_network_timing.py --out <dir> [--reps 30]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from pair_potential_timing import device_info   # noqa: E402

def build_arms(dev):
    """name -> (model, oracle model, oracle compute function, xTB pair spec of the oracle or None)"""
    import oracle.ani_oracle as orc
    import oracle.gelu_oracle as gor
    import oracle.pair_oracle as porc
    GELU_SYMBOLS, RCR = gor.SYMBOLS, gor.RCR
    from torchani_b200 import models, nn, potentials, synthetic
    w2x = synthetic.make_weights(models.SYMBOLS_2X, synthetic.DIMS_2X, 1008, 8, seed=1234)
    celu = models.from_weight_lists("2x", w2x, periodic_table_index=False).to(dev)
    spec = gor.gelu_spec()
    wg = gor.make_weights(GELU_SYMBOLS, orc.DIMS_2X, spec.out_dim, 8, 4321)
    members = [nn.ANINetworks.default(GELU_SYMBOLS, spec.out_dim) for _ in range(8)]
    with torch.no_grad():
        for net, wm in zip(members, wg):
            for s in GELU_SYMBOLS:
                for (dst, _), (src, _) in zip(net.atomics[s].linear_pairs(), wm[s]):
                    dst.copy_(src)
    aev = models.AEVComputer.from_constants(spec.rcr, spec.rca, spec.eta_r, spec.shf_r, spec.eta_a, spec.zeta,
                                            spec.shf_a, spec.shf_z, 7, cutoff_fn="smooth")
    sae = models.SelfEnergy(GELU_SYMBOLS, [orc.GSAES_WB97X_631GD[s] for s in GELU_SYMBOLS])
    gelu = models.ANI(GELU_SYMBOLS, aev, nn.Ensemble(members), sae, False).to(dev)
    z = np.load(os.path.join(ROOT, "tests", "golden", "pair_params.npz"))
    perm = [orc.SYMBOLS_2X.index(s) for s in GELU_SYMBOLS]
    pot = potentials.RepulsionXTB(GELU_SYMBOLS, alpha=[1.0] * 7, yeff=[1.0] * 7, cutoff=RCR, cutoff_fn="smooth")
    tables = {k: torch.tensor(z[k])[perm][:, perm] for k in ("y_ab", "sqrt_alpha_ab", "k_rep_ab")}
    for key, t in tables.items():
        getattr(pot, key).copy_(t.float())
    gelu_xtb = models.ANI(GELU_SYMBOLS, gelu.aev_computer, gelu.neural_networks, gelu.energy_shifter, False,
                          {"repulsion_xtb": pot}).to(dev)
    celu_o = orc.Model(orc.aev_spec_2x(), orc.SYMBOLS_2X, orc.make_weights(orc.SYMBOLS_2X, orc.DIMS_2X, 1008, 8, 1234),
                       orc.GSAES_WB97X_631GD)
    gelu_o = orc.Model(spec, GELU_SYMBOLS, wg, orc.GSAES_WB97X_631GD, "cell_list")
    xtb_o = porc.PairSpec("xtb", RCR, "smooth", tuple(t.double() for t in tables.values()))
    return {"celu": (celu, celu_o, orc.compute, None), "gelu": (gelu, gelu_o, gor.compute, None),
            "gelu_xtb": (gelu_xtb, gelu_o, gor.compute, xtb_o)}


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=30, help="timed repetitions of each arm")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        print("gelu_network_timing: no CUDA device", file=sys.stderr)
        return 2
    import oracle.pair_oracle as porc
    from torchani_b200 import synthetic
    dev = torch.device("cuda:0")
    arms = build_arms(dev)
    _, idx, coords, cell, pbc = synthetic.water_box(3333, seed=0)
    sp_b, co_b = synthetic.conformer_batch(256)
    workloads = {"water_10k": (idx, coords, cell, pbc), "gdb_batch_256": (sp_b, co_b, None, None)}
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    rows, ok = [], True
    for name, (sp, co, cl, pb) in workloads.items():
        # (species indices: O and H are 3 and 0 in both element orders; the GDB batch holds H C N O only)
        assert int(sp.max()) <= 3
        spd, cod = sp.to(dev), co.float().to(dev)
        cld, pbd = (None if cl is None else cl.float().to(dev)), (None if pb is None else pb.to(dev))
        engines = {a: m.engine(dev) for a, (m, _, _, _) in arms.items()}
        out = {}

        def step(arm):
            r = engines[arm].step(spd, cod, cld, pbd is not None)
            out[arm] = (r.energies, r.grad)
        for _ in range(max(e.graph_after for e in engines.values()) + 3):
            for arm in arms:
                step(arm)
        torch.cuda.synchronize(dev)
        row = {"workload": name, "atoms": int((sp >= 0).sum())}
        n_real = int((sp >= 0).sum(1).max())
        nl = "cell_list" if sp.shape[0] == 1 else "all_pairs"
        co64, cl64 = co.float().double(), (None if cl is None else cl.float().double())
        for arm, (_, om, oracle_compute, pair) in arms.items():
            engines[arm].check_status()
            ref = oracle_compute(om._replace(neighborlist=nl), sp, co64, cl64, pb)
            e_ref, f_ref = ref["energy"], ref["forces"]
            if pair is not None:
                pr = porc.compute(pair, sp, co64, cl64, pb, nl)
                e_ref, f_ref = e_ref + pr["energy"], f_ref + pr["forces"]
            e, g = out[arm]
            de = float(((e.double().cpu() - e_ref).abs() - (2e-7 * e_ref.abs() + 2e-7 * n_real)).max())
            df = float(((-g.double().cpu().view_as(f_ref) - f_ref).abs() - (1e-4 + 1e-5 * f_ref.abs())).max())
            row[f"{arm}_energy_excess"], row[f"{arm}_force_excess"] = de, df
            ok = ok and de <= 0 and df <= 0
        if not ok:
            row["error"] = "an arm disagrees with the oracle: not timed"
            rows.append(row)
            print(json.dumps(row), flush=True)
            break
        times = {arm: [] for arm in arms}
        order = list(arms)
        for rep in range(args.reps):
            for arm in order[rep % 3:] + order[:rep % 3]:      # rotate: no arm always follows the same one
                flush.fill_(1)
                ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                ev0.record()
                step(arm)
                ev1.record()
                ev1.synchronize()
                times[arm].append(ev0.elapsed_time(ev1))
        for arm, t in times.items():
            row[arm] = {"median_ms": statistics.median(t), "min_ms": min(t), "max_ms": max(t)}
            # per-stage device times in a separate, profiled pass (events around every stage: not graph-replayed)
            eng = engines[arm]
            eng.profile, eng.stage_events = True, {}
            for _ in range(10):
                step(arm)
            row[arm]["stages_ms"] = eng.stage_times_ms()
            eng.profile = False
        row["gelu_over_celu"] = row["gelu"]["median_ms"] / row["celu"]["median_ms"]
        row["gelu_xtb_over_gelu"] = row["gelu_xtb"]["median_ms"] / row["gelu"]["median_ms"]
        rows.append(row)
        print(json.dumps(row), flush=True)
    record = {"tool": "gelu_network_timing", **device_info(dev), "reps": args.reps,
              "method": "CUDA events around each arm, arms alternated, 256 MiB L2 flush before each (untimed), "
                        "graph-replayed steps, energy + forces", "rows": rows}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "gelu_network_timing.json"), "w") as fh:
        json.dump(record, fh, indent=1)
    print(json.dumps({k: v for k, v in record.items() if k != "rows"}))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
