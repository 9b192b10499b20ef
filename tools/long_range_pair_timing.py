#!/usr/bin/env python
"""Time the fused step with and without a Lennard-Jones or a FixedCoulomb term at 8, 10 and 12 A.

Arms, run in the same process and alternated, on the same seeded inputs (energy + forces, ANI-2x-shaped x8 ensemble
with the seeded synthetic weights of bench.py, the per-element parameters of tests/golden/ljc_params.npz, smooth
envelope):

    plain          Engine.step of the model without the term, graph-replayed
    lj_<c>         the same model with LennardJones at cutoff c: the same graph plus ONE
                   ani_b200_pair_potential_search launch
    coulomb_<c>    the same with FixedCoulomb at cutoff c

Workloads: the 9 999-atom periodic water box and the GDB-like padded batch of 256 conformers.  Every shape is warmed up
(eager uses and the CUDA-graph capture happen before timing).  A 256 MiB buffer is overwritten before every timed arm
(L2 flush, untimed); CUDA events bracket each arm.  The search launch is also timed by itself (100 launches back to
back on the workspace the step left).  Output: median and spread per arm, the launch time, the device name and power
limit, as JSON in --out.

    python tools/long_range_pair_timing.py --out <dir> [--reps 20]
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
CUTOFFS = (8.0, 10.0, 12.0)


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=20, help="timed repetitions of each arm")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        print("long_range_pair_timing: no CUDA device", file=sys.stderr)
        return 2
    from pair_potential_timing import device_info
    from torchani_b200 import _lib, models, potentials, synthetic
    dev = torch.device("cuda:0")
    weights = synthetic.make_weights(models.SYMBOLS_2X, synthetic.DIMS_2X, 1008, 8, seed=1234)
    base = models.from_weight_lists("2x", weights, periodic_table_index=False)
    z = np.load(os.path.join(ROOT, "tests", "golden", "ljc_params.npz"))
    eps, sigma, q = ([float(v) for v in z[k]] for k in ("eps", "sigma", "charges"))
    sym = models.SYMBOLS_2X
    engines = {"plain": base.to(dev).engine(dev)}
    for c in CUTOFFS:
        for name, pot in ((f"lj_{c:g}", potentials.LennardJones(sym, eps, sigma, cutoff=c)),
                          (f"coulomb_{c:g}", potentials.FixedCoulomb(sym, float(z["dielectric"]), q, cutoff=c))):
            m = models.ANI(base.symbols, base.aev_computer, base.neural_networks, base.energy_shifter, False,
                           {"term": pot}).to(dev)
            engines[name] = m.engine(dev)
            assert len(engines[name].search_pairs) == 1
    _, idx, coords, cell, pbc = synthetic.water_box(3333, seed=0)
    sp_b, co_b = synthetic.conformer_batch(256)
    workloads = {"water_10k": (idx.to(dev), coords.to(dev), cell.to(dev), pbc.to(dev)),
                 "gdb_batch_256": (sp_b.to(dev), co_b.to(dev), None, None)}
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    rows = []
    for wl, (sp, co, cl, pb) in workloads.items():
        arms = list(engines.items())
        for _ in range(engines["plain"].graph_after + 3):      # eager uses, capture, replays
            for _, eng in arms:
                eng.step(sp, co, cl, pb is not None)
        for _, eng in arms:
            eng.check_status()
        times = {name: [] for name, _ in arms}
        for rep in range(args.reps):
            k = rep % len(arms)
            for name, eng in arms[k:] + arms[:k]:      # rotate: no arm always follows the same one
                flush.fill_(1)
                ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                ev0.record()
                eng.step(sp, co, cl, pb is not None)
                ev1.record()
                ev1.synchronize()
                times[name].append(ev0.elapsed_time(ev1))
        row = {"workload": wl, "atoms": int((sp >= 0).sum())}
        for name, t in times.items():
            row[name] = {"median_ms": statistics.median(t), "min_ms": min(t), "max_ms": max(t)}
        plain = row["plain"]["median_ms"]
        for name, eng in arms[1:]:
            row[name]["minus_plain_ms"] = row[name]["median_ms"] - plain
            # the search launch by itself, on the workspace the step left (positions and grid L2-warm)
            ws = eng.workspace(*sp.shape)
            lat = (ws.lattice.data_ptr(),) if (cl is not None and cl.dim() == 3) else ()

            def run(_name, call):
                _lib.check(call(), "pair_potential_search")
            with torch.cuda.device(dev):
                ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                for _ in (False, True):
                    ev0.record()
                    for _ in range(100):
                        eng._search_pairs(ws, 0, ws.n, lat, ws.grad_ptr, None, None, run)
                    ev1.record()
                    ev1.synchronize()
            row[name]["search_launch_us"] = ev0.elapsed_time(ev1) * 1e3 / 100
        rows.append(row)
        print(json.dumps(row), flush=True)
    record = {"tool": "long_range_pair_timing", **device_info(dev), "reps": args.reps,
              "method": "CUDA events around each arm, arms rotated, 256 MiB L2 flush before each (untimed), "
                        "graph-replayed steps, energy + forces", "rows": rows}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "long_range_pair_timing.json"), "w") as fh:
        json.dump(record, fh, indent=1)
    print(json.dumps({k: v for k, v in record.items() if k != "rows"}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
