#!/usr/bin/env python
"""Time the fused step with and without D3 dispersion, and the D3 launches alone.

Arms, run in the same process and alternated, on the same seeded inputs (energy + forces, ANI-2x-shaped x8 ensemble
with the seeded synthetic weights of bench.py, D3(BJ) with the tables of tests/golden/d3_params.npz, smooth envelope,
cutoff 8 A):

    plain  Engine.step of the model without D3, graph-replayed
    d3     Engine.step of the model with D3: the same graph plus the three ani_b200_dispersion_d3 launches

and, separately, the three D3 launches by themselves (100 calls back to back on the workspace the step left, grid and
positions L2-warm, events around all of them).

Workloads: the 9 999-atom periodic water box and the GDB-like padded batch of 256 conformers.  Every shape is warmed
up (eager uses and the CUDA-graph capture happen before timing).  A 256 MiB buffer is overwritten before every timed
arm (L2 flush, untimed); CUDA events bracket each arm.  Before any time is taken the arms must agree: (d3 - plain)
energies and forces against the D3 launches run alone into zeroed outputs (1e-5 |E| + 1e-5 Ha, 1e-4 max|F| + 1e-5
Ha/A); arms that disagree are not timed and the script exits non-zero.  Output: median and spread per arm, the launch
time, the device name and power limit, as JSON in --out.

    python tools/dispersion_timing.py --out <dir> [--reps 30]
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

CUTOFF = 8.0


def d3_module(symbols):
    from torchani_b200 import potentials as P
    z = np.load(os.path.join(ROOT, "tests", "golden", "d3_params.npz"))
    sq = np.sqrt(np.diag(z["sqrt_charge_ab"]))
    pot = P.TwoBodyDispersionD3(symbols, float(z["s6"]), float(z["s8"]), float(z["a1"]), float(z["a2"]), sq.tolist(),
                                (z["covalent_radii"] / P.ANGSTROM_TO_BOHR).tolist(), coeff6=z["precalc_coeff6"],
                                coordnums_a=z["precalc_coordnums_a"], coordnums_b=z["precalc_coordnums_b"],
                                cutoff=CUTOFF, cutoff_fn="smooth")
    pot._damp_fn.cutoff_radii.copy_(torch.tensor(z["cutoff_radii"]).float())
    pot.covalent_radii.copy_(torch.tensor(z["covalent_radii"]).float())
    return pot


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=30, help="timed repetitions of each arm")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        print("dispersion_timing: no CUDA device", file=sys.stderr)
        return 2
    from torchani_b200 import _lib, models, synthetic
    dev = torch.device("cuda:0")
    weights = synthetic.make_weights(models.SYMBOLS_2X, synthetic.DIMS_2X, 1008, 8, seed=1234)
    base = models.from_weight_lists("2x", weights, periodic_table_index=False)
    plain_m = base.to(dev)
    d3_m = models.ANI(base.symbols, base.aev_computer, base.neural_networks, base.energy_shifter, False,
                      {"dispersion_d3": d3_module(base.symbols)}).to(dev)
    eng_plain, eng_d3 = plain_m.engine(dev), d3_m.engine(dev)
    assert eng_plain is not eng_d3 and eng_plain.dispersion is None and eng_d3.dispersion is not None

    _, idx, coords, cell, pbc = synthetic.water_box(3333, seed=0)
    sp_b, co_b = synthetic.conformer_batch(256)
    workloads = {"water_10k": (idx.to(dev), coords.to(dev), cell.to(dev), pbc.to(dev)),
                 "gdb_batch_256": (sp_b.to(dev), co_b.to(dev), None, None)}
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    rows, ok = [], True

    def run(_name, call):
        _lib.check(call(), "dispersion_d3")

    for name, (sp, co, cl, pb) in workloads.items():
        out = {}

        def plain():
            r = eng_plain.step(sp, co, cl, pb is not None)
            out["plain"] = (r.energies.clone(), r.grad.clone())

        def d3():
            r = eng_d3.step(sp, co, cl, pb is not None)
            out["d3"] = (r.energies.clone(), r.grad.clone())

        for _ in range(eng_plain.graph_after + 3):      # eager uses, capture, replays
            plain(), d3()
        eng_plain.check_status(), eng_d3.check_status()
        # the D3 launches alone into zeroed outputs, on the grid the last step built
        ws = eng_d3.workspace(*sp.shape)
        lat = (ws.lattice.data_ptr(),) if (cl is not None and cl.dim() == 3) else ()
        with torch.cuda.device(dev):
            ws.grad.zero_(), ws.energies.zero_(), ws.atomic.zero_()
            eng_d3._dispersion(ws, 0, ws.n, lat, ws.grad_ptr, None, None, run)
            torch.cuda.synchronize(dev)
        e_alone, g_alone = ws.energies.clone(), ws.grad.clone().view(sp.shape + (3,))
        eng_d3.check_status()
        (e_p, g_p), (e_d, g_d) = out["plain"], out["d3"]
        de = float(((e_d - e_p - e_alone).abs() - (1e-5 * e_alone.abs() + 1e-5)).max())
        dg = float(((g_d - g_p - g_alone).abs() - (1e-4 * float(g_alone.abs().max()) + 1e-5)).max())
        row = {"workload": name, "atoms": int((sp >= 0).sum()), "energy_excess": de, "force_excess": dg,
               "d3_energy_ha": e_alone.sum().item(), "launches_plain": eng_plain.launches_per_step,
               "launches_d3": eng_d3.launches_per_step}
        if de > 0 or dg > 0:
            row["error"] = "the step with D3 and the D3 launches alone disagree: not timed"
            ok = False
            rows.append(row)
            print(json.dumps(row), flush=True)
            continue
        times = {"plain": [], "d3": []}
        arms = [("plain", plain), ("d3", d3)]
        for rep in range(args.reps):
            for arm, fn in arms[rep % 2:] + arms[:rep % 2]:      # alternate: no arm always follows the same one
                flush.fill_(1)
                ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                ev0.record()
                fn()
                ev1.record()
                ev1.synchronize()
                times[arm].append(ev0.elapsed_time(ev1))
        for arm, t in times.items():
            row[arm] = {"median_ms": statistics.median(t), "min_ms": min(t), "max_ms": max(t)}
        row["d3_minus_plain_ms"] = row["d3"]["median_ms"] - row["plain"]["median_ms"]
        with torch.cuda.device(dev):
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            for _timed in (False, True):
                ev0.record()
                for _ in range(100):
                    eng_d3._dispersion(ws, 0, ws.n, lat, ws.grad_ptr, None, None, run)
                ev1.record()
                ev1.synchronize()
        row["d3_launches_us"] = ev0.elapsed_time(ev1) * 1e3 / 100
        row["d3_over_plain"] = row["d3"]["median_ms"] / row["plain"]["median_ms"]
        rows.append(row)
        print(json.dumps(row), flush=True)
    record = {"tool": "dispersion_timing", **device_info(dev), "reps": args.reps,
              "method": "CUDA events around each arm, arms alternated, 256 MiB L2 flush before each (untimed), "
                        "graph-replayed steps, energy + forces; D3 launches alone: 100 back to back, L2-warm",
              "rows": rows}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "dispersion_timing.json"), "w") as fh:
        json.dump(record, fh, indent=1)
    print(json.dumps({k: v for k, v in record.items() if k != "rows"}))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
