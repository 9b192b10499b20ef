#!/usr/bin/env python
"""Time a periodic batch (C copies of one water box in a shared cell) as ONE fused step against C single steps.
With ``--cells per_conformer`` every copy has a cell of its own (volumes a few per cent apart, grid mode 3).

Two arms, run in the same process and alternated, on the same seeded inputs (energy + forces, ANI-2x-shaped x8
ensemble with the seeded synthetic weights of bench.py):

    fused  Engine.step on the (C, A) batch (grid mode 2: one sub-grid per conformer; with --cells per_conformer a
           (C, 3, 3) cell, grid mode 3), graph-replayed
    loop   C Engine.step calls on the (1, A) slices (each with its own cell), each graph-replayed -- what the module
           layer did for a periodic batch before it had a kernel path of its own

Every shape is warmed up (eager uses and the CUDA-graph capture happen before timing).  A 256 MiB buffer is
overwritten before every timed arm (L2 flush, untimed); CUDA events bracket each arm.  Before any time is taken the
two arms' atomic energies (1e-6 |ref| + 1e-7 Ha) and forces (1e-5 Ha/A) are compared; arms that disagree are not
timed and the script exits non-zero.  Output: median and spread per arm, atom-steps/s, the device name and power
limit, as JSON in the directory given by --out.

    python tools/periodic_batch_timing.py --out <dir> [--reps 15] [--cells shared|per_conformer]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = {96: (8, 64, 256), 648: (8, 64, 256), 3000: (8, 64)}   # atoms per box -> conformers (3000 x 64 = 192 k atoms)


def device_info(dev) -> dict:
    info = {"device": torch.cuda.get_device_name(dev), "power_limit_w": None, "sm_max_mhz": None}
    try:
        out = subprocess.run(["nvidia-smi", f"--id={dev.index or 0}", "--query-gpu=power.limit,clocks.max.sm",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        pl, mhz = (v.strip() for v in out.strip().split(","))
        info["power_limit_w"], info["sm_max_mhz"] = float(pl), float(mhz)
    except Exception as e:  # noqa: BLE001 -- the reading is reported as missing, the timing stands
        info["power_limit_error"] = repr(e)
    return info


def batch_inputs(a: int, n_conf: int, dev, per_conformer: bool = False):
    """(species (C, A), coords (C, A, 3), cell): one (3, 3) cell, or with `per_conformer` (C, 3, 3) cells whose volumes
    are 0.98 .. 1.02 of the box's (coordinates scaled with them)."""
    from torchani_b200 import synthetic
    _, idx, coords, cell, _ = synthetic.water_box(a // 3, seed=0)
    g = torch.Generator().manual_seed(a * 1000 + n_conf)
    co = coords.repeat(n_conf, 1, 1)
    co[1:] += 0.05 * torch.randn(co[1:].shape, generator=g)
    if per_conformer:
        scale = (1.0 + 0.01 * (torch.arange(n_conf, dtype=torch.float64) % 5 - 2)) ** (1.0 / 3.0)
        co = (co.double() * scale.view(-1, 1, 1)).float()
        cell = (cell.double().unsqueeze(0) * scale.view(-1, 1, 1)).float()
    return idx.repeat(n_conf, 1).to(dev), co.to(dev).contiguous(), cell.to(dev).contiguous()


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=15, help="timed repetitions of each arm")
    ap.add_argument("--cells", choices=("shared", "per_conformer"), default="shared",
                    help="one cell for the batch (grid mode 2) or one per conformer (grid mode 3)")
    args = ap.parse_args()
    per = args.cells == "per_conformer"
    if not torch.cuda.is_available():
        print("periodic_batch_timing: no CUDA device", file=sys.stderr)
        return 2
    from torchani_b200 import models
    from torchani_b200.engine import Engine
    from torchani_b200.synthetic import DIMS_2X, make_weights
    dev = torch.device("cuda:0")
    weights = make_weights(models.SYMBOLS_2X, DIMS_2X, 1008, 8, seed=1234)
    model = models.from_weight_lists("2x", weights, device=dev, periodic_table_index=True)
    base = model.engine(dev)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    rows, ok = [], True
    for a, confs in SIZES.items():
        for n_conf in confs:
            eng = Engine(base.consts, base.nets, base.sae.tolist(), nbr_cap=base.nbr_cap)
            sp, co, cell = batch_inputs(a, n_conf, dev, per)
            slices = [(sp[c:c + 1].contiguous(), co[c:c + 1].contiguous(), cell[c] if per else cell)
                      for c in range(n_conf)]
            e_f = torch.zeros(n_conf, a, device=dev)
            g_f = torch.zeros(n_conf, a, 3, device=dev)
            e_l, g_l = torch.zeros_like(e_f), torch.zeros_like(g_f)

            def fused():
                r = eng.step(sp, co, cell, True)
                e_f.copy_(r.atomic_energies)
                g_f.copy_(r.grad)

            def loop():
                for c, (s1, c1, l1) in enumerate(slices):
                    r = eng.step(s1, c1, l1, True)
                    e_l[c].copy_(r.atomic_energies[0])
                    g_l[c].copy_(r.grad[0])

            for _ in range(eng.graph_after + 3):      # eager uses, capture, replays of both shapes
                fused()
                loop()
            eng.check_status()
            torch.cuda.synchronize(dev)
            de = float(((e_f - e_l).abs() - (1e-6 * e_l.abs() + 1e-7)).max())
            dg = float((g_f - g_l).abs().max())
            row = {"atoms_per_conf": a, "n_conf": n_conf, "atoms": a * n_conf,
                   "max_atomic_energy_excess": de, "max_force_diff": dg}
            if de > 0 or dg > 1e-5:
                row["error"] = "the arms disagree: not timed"
                ok = False
                rows.append(row)
                print(json.dumps(row), flush=True)
                continue
            times = {"fused": [], "loop": []}
            for _ in range(args.reps):
                for arm, fn in (("fused", fused), ("loop", loop)):
                    flush.fill_(1)
                    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    ev0.record()
                    fn()
                    ev1.record()
                    ev1.synchronize()
                    times[arm].append(ev0.elapsed_time(ev1))
            eng.check_status()
            for arm, t in times.items():
                med = statistics.median(t)
                row[arm] = {"median_ms": med, "min_ms": min(t), "max_ms": max(t),
                            "atom_steps_per_s": a * n_conf / (med * 1e-3)}
            row["loop_over_fused"] = row["loop"]["median_ms"] / row["fused"]["median_ms"]
            rows.append(row)
            print(json.dumps(row), flush=True)
            del eng
            torch.cuda.empty_cache()
    record = {"tool": "periodic_batch_timing", "cells": args.cells, **device_info(dev), "reps": args.reps,
              "method": "CUDA events around each arm, arms alternated, 256 MiB L2 flush before each (untimed), "
                        "graph-replayed steps, energy + forces", "rows": rows}
    os.makedirs(args.out, exist_ok=True)
    name = "periodic_batch_timing" + ("_per_conformer" if per else "") + ".json"
    with open(os.path.join(args.out, name), "w") as fh:
        json.dump(record, fh, indent=1)
    print(json.dumps({k: v for k, v in record.items() if k != "rows"}))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
