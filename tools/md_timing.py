#!/usr/bin/env python
"""Time per MD step and ns/day of the device MD loop (torchani_b200.md) against a host-driven loop, on the workloads of
bench.py (water 1 k, water 10 k, the GDB batch of 256; ANI-2x-shaped x8 ensemble with seeded synthetic weights).

Arms, per workload, velocity Verlet at dt = 0.5 fs:

    device K=1 / 10 / 50   md.VelocityVerlet with steps_per_replay K: one graph replay, one D2H copy and one
                           synchronisation per K steps
    host                   HostCalculator.calculate (one H2D, graph replay, one D2H, synchronise per step) driven by the
                           oracle's float64 velocity Verlet in numpy -- the reference's ASE pattern without ASE

With --npt the arms are instead, on water 1 k and 10 k at K = 10 and 50, Langevin (BAOAB, NVT) against LangevinNPT
(the same with stochastic cell rescaling at 1.01325 bar: the force step also accumulates the virial), timed the same
way, with the integrator launches of both.

Every arm is warmed up (captures happen before timing).  The device arms are timed with a host clock around run()
(which ends in a synchronisation) and with CUDA events around the same call; the host arm with a host clock.  The
integrator's own launches (ani_b200_md_step, two kernels) are timed separately with CUDA events over 200 eager calls.
The arms alternate over --reps rounds; medians are reported with the device name and power limit, as JSON in --out.

    python tools/md_timing.py --out <dir> [--reps 5] [--steps 500] [--npt]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MASSES_2X = np.array([1.008, 12.011, 14.007, 15.999, 32.06, 18.998, 35.45])
DT = 0.5


def workload(name):
    from torchani_b200 import synthetic
    if name == "gdb256":
        sp, co = synthetic.conformer_batch(256)
        return sp.numpy(), co.double().numpy(), None, False
    n = {"water1k": 333, "water10k": 3333}[name]
    _, idx, co, cell, _ = synthetic.water_box(n, seed=1)
    return idx.numpy(), co.double().numpy(), cell.double().numpy(), True


def device_arm(model, name, K, steps, kind="verlet"):
    from torchani_b200 import md
    sp, co, cell, pbc = workload(name)
    m = MASSES_2X[np.maximum(sp, 0)] * (sp >= 0)
    kw = dict(dt=DT, velocities=md.maxwell_boltzmann(m, 300.0, 1), steps_per_replay=K, record_every=0)
    if kind == "verlet":
        dyn = md.VelocityVerlet(model, sp, co, m, cell=cell, pbc=pbc, **kw)
    elif kind == "nvt":
        dyn = md.Langevin(model, sp, co, m, cell=cell, pbc=pbc, **kw)
    else:
        dyn = md.LangevinNPT(model, sp, co, m, cell, **kw)
    steps = steps // K * K
    dyn.run(2 * K)   # capture + warm-up

    def timed():
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        a.record()
        dyn.run(steps)
        b.record()
        b.synchronize()
        return (time.perf_counter() - t0) * 1e3 / steps, a.elapsed_time(b) / steps
    return dyn, timed


def integrator_ms(dyn, reps=200):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    state = dyn._head.clone()
    a.record()
    for _ in range(reps):
        dyn._integrate()
    b.record()
    b.synchronize()
    dyn._head.copy_(state)
    return a.elapsed_time(b) / reps


def host_arm(model, name, steps):
    import oracle.md_oracle as mo
    from torchani_b200.calculator import HostCalculator
    sp, co, cell, pbc = workload(name)
    m = MASSES_2X[np.maximum(sp, 0)] * (sp >= 0)
    inv = np.where(m > 0, 1.0 / np.where(m > 0, m, 1.0), 0.0)
    calc = HostCalculator(model, sp if sp.shape[0] > 1 else sp[0], cell=cell, pbc=pbc)
    batch = sp.shape[0] > 1
    state = {"x": co.copy(), "v": np.zeros_like(co)}

    def grad(x):
        xc = mo.wrap(x, cell) if pbc else x
        _, f = calc.calculate(xc if batch else xc[0])
        return -np.asarray(f, dtype=np.float64).reshape(x.shape)

    state["g"] = grad(state["x"])

    def run(k):
        x, v, g = state["x"], state["v"], state["g"]
        for _ in range(k):
            v = mo.kick(v, g, inv, DT)
            x = x + DT * v
            g = grad(x)
            v = mo.kick(v, g, inv, DT)
        state.update(x=x, v=v, g=g)

    run(10)

    def timed():
        t0 = time.perf_counter()
        run(steps)
        return (time.perf_counter() - t0) * 1e3 / steps, None
    return timed


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=500)
    ap.add_argument("--workloads", default=None)
    ap.add_argument("--npt", action="store_true", help="Langevin against LangevinNPT at K = 10 and 50")
    args = ap.parse_args()
    workloads = args.workloads or ("water1k,water10k" if args.npt else "water1k,water10k,gdb256")
    if not torch.cuda.is_available():
        raise SystemExit("md_timing needs a GPU")
    from torchani_b200 import models
    model = models.ANI2x(seed=0)
    model = models.ANI(model.symbols, model.aev_computer, model.neural_networks, model.energy_shifter, False).cuda()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    result = {"device": torch.cuda.get_device_name(0), "nvidia_smi": smi, "dt_fs": DT, "steps": args.steps,
              "workloads": {}}
    for name in workloads.split(","):
        arms = {}
        dyns = {}
        if args.npt:
            for kind in ("nvt", "npt"):
                for K in (10, 50):
                    dyns[(kind, K)], arms[f"{kind} K={K}"] = device_arm(model, name, K, args.steps, kind)
        else:
            for K in (1, 10, 50):
                dyns[K], arms[f"device K={K}"] = device_arm(model, name, K, args.steps)
            arms["host"] = host_arm(model, name, max(50, args.steps // 5))
        times = {k: ([], []) for k in arms}
        for _ in range(args.reps):
            for k, fn in arms.items():
                wall, dev = fn()
                times[k][0].append(wall)
                if dev is not None:
                    times[k][1].append(dev)
        rec = {}
        for k, (wall, dev) in times.items():
            ms = statistics.median(wall)
            rec[k] = {"ms_per_step": ms, "spread_ms": [min(wall), max(wall)],
                      "device_ms_per_step": statistics.median(dev) if dev else None,
                      "ns_per_day": DT * 1e-6 * 86400e3 / ms}
        if args.npt:
            for kind in ("nvt", "npt"):
                rec[f"{kind} integrator_ms_per_step"] = integrator_ms(dyns[(kind, 50)])
        else:
            rec["integrator_ms_per_step"] = integrator_ms(dyns[50])
        result["workloads"][name] = rec
        print(name, json.dumps(rec, indent=1), flush=True)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "md_timing_npt.json" if args.npt else "md_timing.json"), "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
