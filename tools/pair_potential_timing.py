#!/usr/bin/env python
"""Time the fused step with and without a pair potential, and against what there was before the pair kernel.

Three arms, run in the same process and alternated, on the same seeded inputs (energy + forces, ANI-2x-shaped x8
ensemble with the seeded synthetic weights of bench.py, xTB repulsion with the parameter tensors of
tests/golden/pair_params.npz, smooth envelope, cutoff = Rcr):

    plain  Engine.step of the model without repulsion, graph-replayed
    fused  Engine.step of the model with repulsion: the same graph plus ONE ani_b200_pair_potential launch over the
           neighbour words of the AEV forward
    eager  the plain step, then the reference-style evaluation users had before: a materialised half pair list
           (neighbors.all_pairs: bucket grid + count + fill, one host synchronisation), the xTB formula in eager
           PyTorch on its distances, autograd for the forces

Workloads: the 9 999-atom periodic water box and the GDB-like padded batch of 256 conformers.  Every shape is warmed
up (eager uses and the CUDA-graph capture happen before timing).  A 256 MiB buffer is overwritten before every timed
arm (L2 flush, untimed); CUDA events bracket each arm.  Before any time is taken the fused and the eager arm's energies
(1e-6 |E| + 1e-4 Ha) and forces (1e-4 + 1e-5 |F| Ha/A) are compared; arms that disagree are not timed and the script
exits non-zero.  The arms include the staging copies of Engine.step and run from Python, so their spread is tens of
microseconds; the pair launch is therefore also timed by itself (200 launches back to back, L2-warm).  Output: median
and spread per arm, the launch time, the device name and power limit, as JSON in --out.

    python tools/pair_potential_timing.py --out <dir> [--reps 30]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
RCR = 5.1


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


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=30, help="timed repetitions of each arm")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        print("pair_potential_timing: no CUDA device", file=sys.stderr)
        return 2
    from torchani_b200 import _lib, models, neighbors, potentials, synthetic
    dev = torch.device("cuda:0")
    weights = synthetic.make_weights(models.SYMBOLS_2X, synthetic.DIMS_2X, 1008, 8, seed=1234)
    base = models.from_weight_lists("2x", weights, periodic_table_index=False)
    z = np.load(os.path.join(ROOT, "tests", "golden", "pair_params.npz"))
    pot = potentials.RepulsionXTB(models.SYMBOLS_2X, alpha=[1.0] * 7, yeff=[1.0] * 7, cutoff=RCR, cutoff_fn="smooth")
    for key in ("y_ab", "sqrt_alpha_ab", "k_rep_ab"):
        getattr(pot, key).copy_(torch.tensor(z[key]).float())
    plain_m = base.to(dev)
    fused_m = models.ANI(base.symbols, base.aev_computer, base.neural_networks, base.energy_shifter, False,
                         {"repulsion_xtb": pot}).to(dev)
    y_ab, sa_ab, k_ab = (getattr(fused_m.potentials["repulsion_xtb"], k) for k in ("y_ab", "sqrt_alpha_ab", "k_rep_ab"))
    eng_plain, eng_fused = plain_m.engine(dev), fused_m.engine(dev)
    assert eng_plain is not eng_fused and not eng_plain.pairs and len(eng_fused.pairs) == 1

    _, idx, coords, cell, pbc = synthetic.water_box(3333, seed=0)
    sp_b, co_b = synthetic.conformer_batch(256)
    workloads = {"water_10k": (idx.to(dev), coords.to(dev), cell.to(dev), pbc.to(dev)),
                 "gdb_batch_256": (sp_b.to(dev), co_b.to(dev), None, None)}
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    rows, ok = [], True
    for name, (sp, co, cl, pb) in workloads.items():
        out = {}

        def plain():
            r = eng_plain.step(sp, co, cl, pb is not None)
            out["plain"] = (r.energies, r.grad)

        def fused():
            r = eng_fused.step(sp, co, cl, pb is not None)
            out["fused"] = (r.energies, r.grad)

        def eager():
            r = eng_plain.step(sp, co, cl, pb is not None)
            x = co.detach().clone().requires_grad_(True)
            nb = neighbors.all_pairs(RCR, sp, x, cl, pb)
            d = nb.distances.clamp(min=1e-7) * potentials.ANGSTROM_TO_BOHR
            s12 = sp.reshape(-1)[nb.indices]
            e = y_ab[s12[0], s12[1]] / d * torch.exp(-sa_ab[s12[0], s12[1]] * d ** k_ab[s12[0], s12[1]])
            e = e * torch.exp(1 - 1 / (1 - (nb.distances / RCR) ** 2).clamp(min=1e-10))
            conf = torch.div(nb.indices[0], sp.shape[1], rounding_mode="floor")
            e_c = torch.zeros(sp.shape[0], dtype=torch.float64, device=dev).index_add(0, conf, e.double())
            (g,) = torch.autograd.grad(e_c.sum(), x)
            out["eager"] = (r.energies + e_c, r.grad + g)

        for _ in range(eng_plain.graph_after + 3):      # eager uses, capture, replays
            plain(), fused(), eager()
        eng_plain.check_status(), eng_fused.check_status()
        torch.cuda.synchronize(dev)
        (e_f, g_f), (e_e, g_e) = out["fused"], out["eager"]
        de = float(((e_f - e_e).abs() - (1e-6 * e_e.abs() + 1e-4)).max())
        dg = float(((g_f - g_e).abs() - (1e-4 + 1e-5 * g_e.abs())).max())
        row = {"workload": name, "atoms": int((sp >= 0).sum()), "energy_excess": de, "force_excess": dg,
               "launches_plain": eng_plain.launches_per_step, "launches_fused": eng_fused.launches_per_step}
        if de > 0 or dg > 0:
            row["error"] = "the fused and the eager arm disagree: not timed"
            ok = False
            rows.append(row)
            print(json.dumps(row), flush=True)
            continue
        times = {"plain": [], "fused": [], "eager": []}
        arms = [("plain", plain), ("fused", fused), ("eager", eager)]
        for rep in range(args.reps):
            for arm, fn in arms[rep % 3:] + arms[:rep % 3]:      # rotate: no arm always follows the same one
                flush.fill_(1)
                ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                ev0.record()
                fn()
                ev1.record()
                ev1.synchronize()
                times[arm].append(ev0.elapsed_time(ev1))
        for arm, t in times.items():
            row[arm] = {"median_ms": statistics.median(t), "min_ms": min(t), "max_ms": max(t)}
        row["fused_minus_plain_ms"] = row["fused"]["median_ms"] - row["plain"]["median_ms"]
        # the pair launch by itself: 200 launches back to back on the workspace the fused step left (neighbour words
        # and positions L2-warm, as they are right after the AEV backward of a step), events around all of them
        ws = eng_fused.workspace(*sp.shape)
        lat = (ws.lattice.data_ptr(),) if (cl is not None and cl.dim() == 3) else ()

        def run(_name, call):
            _lib.check(call(), "pair_potential")
        with torch.cuda.device(dev):
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            for timed in (False, True):
                ev0.record()
                for _ in range(200):
                    eng_fused._pair_potentials(ws, 0, ws.n, lat, ws.grad_ptr, None, None, run)
                ev1.record()
                ev1.synchronize()
        row["pair_launch_us"] = ev0.elapsed_time(ev1) * 1e3 / 200
        row["fused_over_plain"] = row["fused"]["median_ms"] / row["plain"]["median_ms"]
        row["eager_over_fused"] = row["eager"]["median_ms"] / row["fused"]["median_ms"]
        rows.append(row)
        print(json.dumps(row), flush=True)
    record = {"tool": "pair_potential_timing", **device_info(dev), "reps": args.reps,
              "method": "CUDA events around each arm, arms alternated, 256 MiB L2 flush before each (untimed), "
                        "graph-replayed steps, energy + forces", "rows": rows}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "pair_potential_timing.json"), "w") as fh:
        json.dump(record, fh, indent=1)
    print(json.dumps({k: v for k, v in record.items() if k != "rows"}))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
