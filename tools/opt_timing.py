#!/usr/bin/env python
"""Time per step and time to convergence of the device FIRE loop (torchani_b200.optimize) against a host-driven loop,
on the GDB batch of 256 and water 1 k (ANI-2x-shaped x8 ensemble with seeded synthetic weights, as bench.py), and the
smallest fmax the float32 forces let FIRE reach on a small molecule.

Arms, per workload:

    device K=1 / 10 / 50   optimize.FIRE with steps_per_replay K: one graph replay, one D2H copy and one
                           synchronisation per K steps
    host                   HostCalculator.calculate (one H2D, graph replay, one D2H, synchronise per step) driven by
                           FIRE in numpy: the oracle's step (oracle/fire_oracle.py) vectorised over the conformers

Per step: fmax = 0 (no conformer converges), arms alternated over --reps rounds, medians.  The device arms are timed
with a host clock around run() (which ends in a synchronisation); the host arm with a host clock.  The FIRE launches
alone (ani_b200_opt_step, two kernels) are timed with CUDA events over 200 eager calls.  To fmax 0.05 eV / A: from the
input geometry, once per arm, the wall time and the steps until every conformer converged (or --max-steps).

Floor: one GDB molecule optimised with fmax = 0 for --floor-steps steps; the smallest fmax(t) reached, and the median
of the last 500 steps (where float32 noise of the forces, not the geometry, sets fmax).

Results go to --out as JSON, with the device name and power limit read in the same run.

With --cell: variable-cell FIRE (optimize.CellFIRE) against fixed-cell FIRE per step at K = 1, 10 and 50 on water 1 k
and on a 256-atom fcc Lennard-Jones crystal (a pure-LJ model: zero networks, sigma 2.5 A, eps 0.5 eV, smooth cutoff
6.25 A), arms alternated over --reps rounds, medians; and the two launches of each step form alone under CUDA events
(ani_b200_opt_cell_step against ani_b200_opt_step, 200 eager calls each).  Results go to opt_cell_timing.json.

With --lbfgs: L-BFGS (optimize.LBFGS, ASE's defaults, memory 100) against FIRE per step at K = 1, 10 and 50 on the GDB
batch and water 1 k, the arms alternated over --reps rounds, medians; the four L-BFGS launches alone with a full
history (after 110 steps; ani_b200_lbfgs_step under CUDA events, 200 eager calls) against the two FIRE launches; and
the steps and wall time (K = 50) of both optimisers to fmax 0.05 eV / A on the GDB batch and to 1e-4 and 1e-6 eV / A
on the 26-atom molecule of the floor run.  Results go to opt_lbfgs_timing.json.

    python tools/opt_timing.py --out <dir> [--reps 5] [--steps 500] [--cell | --lbfgs]
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


def workload(name):
    from torchani_b200 import synthetic
    if name == "ljfcc":   # 4 x 4 x 4 conventional cells, strained and sheared, atoms displaced by 0.02 A
        a, shear = 1.56 * 2.5, np.array([[1.03, 0.04, 0.0], [-0.02, 0.98, 0.03], [0.01, 0.0, 1.02]])
        base = np.array([[0, 0, 0], [0, 0.5, 0.5], [0.5, 0, 0.5], [0.5, 0.5, 0]])
        cells = np.array([(i, j, k) for i in range(4) for j in range(4) for k in range(4)])
        r = a * (cells[:, None] + base[None]).reshape(-1, 3) @ shear
        r += 0.02 * np.random.default_rng(0).standard_normal(r.shape)
        return np.zeros((1, len(r)), dtype=np.int64), r[None], 4 * a * np.eye(3) @ shear, True
    if name == "gdb256":
        sp, co = synthetic.conformer_batch(256)
        return sp.numpy(), co.double().numpy(), None, False
    _, idx, co, cell, _ = synthetic.water_box({"water1k": 333}[name], seed=1)
    return idx.numpy(), co.double().numpy(), cell.double().numpy(), True


def device_arm(model, name, K, steps, variable_cell=False, lbfgs=False):
    from torchani_b200 import optimize
    sp, co, cell, pbc = workload(name)
    if lbfgs:
        opt = optimize.LBFGS(model, sp, co, cell=cell, pbc=pbc, steps_per_replay=K)
    elif variable_cell:
        opt = optimize.CellFIRE(model, sp, co, cell, steps_per_replay=K)
    else:
        opt = optimize.FIRE(model, sp, co, cell=cell, pbc=pbc, steps_per_replay=K)
    steps = steps // K * K
    opt.run(0.0, 2 * K)   # capture + warm-up

    def timed():
        t0 = time.perf_counter()
        opt.run(0.0, steps)
        return (time.perf_counter() - t0) * 1e3 / steps
    return opt, timed


def fire_launch_ms(opt, reps=200):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    state = opt._head.clone()
    a.record()
    for _ in range(reps):
        opt._integrate()
    b.record()
    b.synchronize()
    opt._head.copy_(state)
    return a.elapsed_time(b) / reps


class HostFIRE:
    """FIRE over (C, A, 3) numpy arrays: oracle/fire_oracle.step for every conformer at once."""

    def __init__(self, model, name, fmax):
        import oracle.fire_oracle as fo
        import oracle.md_oracle as mo
        from torchani_b200.calculator import HostCalculator
        sp, co, cell, pbc = workload(name)
        self.calc = HostCalculator(model, sp, cell=cell, pbc=pbc)
        self.wrap = (lambda x: np.stack([mo.wrap(c, cell) for c in x])) if pbc else (lambda x: x)
        self.scale = np.where(sp >= 0, fo.HARTREE_EV, 0.0)[..., None]
        self.par = fo.params(fmax)
        C_ = sp.shape[0]
        self.x, self.v = co.copy(), np.zeros_like(co)
        self.dt, self.a, self.n = np.full(C_, self.par[0]), np.full(C_, self.par[6]), np.zeros(C_)
        self.conv = np.zeros(C_, dtype=bool)
        self.t = 0

    def step(self):
        p = self.par
        _, f = self.calc.calculate(self.wrap(self.x))
        f = np.asarray(f, dtype=np.float64).reshape(self.x.shape) * self.scale
        self.conv |= np.sqrt((f * f).sum(-1).max(-1)) < p[8]
        run = ~self.conv
        P, F2, V2 = (f * self.v).sum((1, 2)), (f * f).sum((1, 2)), (self.v * self.v).sum((1, 2))
        c1, c2 = np.ones_like(P), np.zeros_like(P)
        if self.t > 0:
            up = P > 0
            c1 = np.where(up, 1.0 - self.a, 0.0)
            c2 = np.where(up, self.a * np.sqrt(V2 / np.where(F2 > 0, F2, 1.0)), 0.0)
            grow = up & (self.n > p[3])
            dt = np.where(grow, np.minimum(self.dt * p[4], p[2]), np.where(up, self.dt, self.dt * p[5]))
            a = np.where(grow, self.a * p[7], np.where(up, self.a, p[6]))
            n = np.where(up, self.n + 1.0, 0.0)
            self.dt, self.a, self.n = (np.where(run, new, old) for new, old in ((dt, self.dt), (a, self.a), (n, self.n)))
        cf = (c2 + self.dt)[:, None, None]
        v1 = c1[:, None, None] * self.v + cf * f
        dr = self.dt * np.sqrt((v1 * v1).sum((1, 2)))
        st = (self.dt * np.where(dr > p[1], p[1] / np.where(dr > 0, dr, 1.0), 1.0))[:, None, None]
        r = run[:, None, None]
        self.v = np.where(r, v1, self.v)
        self.x = np.where(r, self.x + st * v1, self.x)
        self.t += 1


def host_arm(model, name, steps):
    h = HostFIRE(model, name, 0.0)
    for _ in range(10):
        h.step()

    def timed():
        t0 = time.perf_counter()
        for _ in range(steps):
            h.step()
        return (time.perf_counter() - t0) * 1e3 / steps
    return timed


def to_fmax(model, name, fmax, max_steps):
    from torchani_b200 import optimize
    sp, co, cell, pbc = workload(name)
    out = {}
    for K in (10, 50):
        optimize.FIRE(model, sp, co, cell=cell, pbc=pbc, steps_per_replay=K).run(0.0, K)   # this shape's warm-up
        opt = optimize.FIRE(model, sp, co, cell=cell, pbc=pbc, steps_per_replay=K)
        t0 = time.perf_counter()
        done = opt.run(fmax, max_steps)
        ms = (time.perf_counter() - t0) * 1e3
        out[f"device K={K}"] = {"ms": ms, "steps": opt.step, "last_converged_step": int(opt.converged_step.max()),
                                "converged": float(opt.converged.mean()), "all": done}
    h = HostFIRE(model, name, fmax)
    t0 = time.perf_counter()
    while h.t < max_steps and not h.conv.all():
        h.step()
    out["host"] = {"ms": (time.perf_counter() - t0) * 1e3, "steps": h.t, "converged": float(h.conv.mean())}
    return out


def floor(model, steps):
    from torchani_b200 import optimize
    sp, co, _, _ = workload("gdb256")
    n = int((sp[0] >= 0).sum())
    opt = optimize.FIRE(model, sp[0, :n], co[0, :n], steps_per_replay=50)
    opt.run(0.0, steps)
    f = opt.log.fmax[:, 0]
    return {"atoms": n, "steps": steps, "min_fmax_eV_A": float(f.min()), "step_of_min": int(f.argmin()),
            "median_fmax_last500_eV_A": float(np.median(f[-500:])),
            "fmax_at": {str(s): float(f[s]) for s in (100, 300, 1000, 3000) if s < len(f)}}


def lj_model():
    """Zero networks, no self energies and one Lennard-Jones term (sigma 2.5 A, eps 0.5 eV, smooth cutoff 6.25 A)."""
    from torchani_b200 import models, potentials
    from torchani_b200.grad import HARTREE_TO_EV
    base = models.ANI2x(seed=0)
    with torch.no_grad():
        for p in base.neural_networks.parameters():
            p.zero_()
    S = len(base.symbols)
    lj = potentials.LennardJones(base.symbols, eps=[0.5 / HARTREE_TO_EV] * S, sigma=[2.5] * S, cutoff=6.25,
                                 cutoff_fn="smooth")
    return models.ANI(base.symbols, base.aev_computer, base.neural_networks, models.SelfEnergy(base.symbols, [0.0] * S),
                      False, {"lj": lj}).cuda()


def cell_main(args, model, result) -> None:
    for name in ("water1k", "ljfcc"):
        mdl = lj_model() if name == "ljfcc" else model
        arms, opts = {}, {}
        for K in (1, 10, 50):
            for cell in (False, True):
                key = f"{'CellFIRE' if cell else 'FIRE'} K={K}"
                opts[key], arms[key] = device_arm(mdl, name, K, args.steps, cell)
        times = {k: [] for k in arms}
        for _ in range(args.reps):
            for k, fn in arms.items():
                times[k].append(fn())
        rec = {k: {"ms_per_step": statistics.median(v), "spread_ms": [min(v), max(v)]} for k, v in times.items()}
        rec["launches_ms_per_step"] = {"FIRE": fire_launch_ms(opts["FIRE K=50"]),
                                       "CellFIRE": fire_launch_ms(opts["CellFIRE K=50"])}
        result["workloads"][name] = rec
        print(name, json.dumps(rec, indent=1), flush=True)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "opt_cell_timing.json"), "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps(result))


def lbfgs_to_fmax(model, sp, co, cell, pbc, fmax, max_steps):
    from torchani_b200 import optimize
    out = {}
    for cls in (optimize.FIRE, optimize.LBFGS):
        cls(model, sp, co, cell=cell, pbc=pbc, steps_per_replay=50).run(0.0, 50)   # this shape's warm-up
        opt = cls(model, sp, co, cell=cell, pbc=pbc, steps_per_replay=50)
        t0 = time.perf_counter()
        done = opt.run(fmax, max_steps)
        ms = (time.perf_counter() - t0) * 1e3
        out[cls.__name__] = {"ms": ms, "steps": opt.step, "last_converged_step": int(opt.converged_step.max()),
                             "converged": float(opt.converged.mean()), "all": done,
                             "energy_Ha": float(opt.energies.max())}
    return out


def lbfgs_main(args, model, result) -> None:
    for name in ("gdb256", "water1k"):
        arms, opts = {}, {}
        for K in (1, 10, 50):
            for lb in (False, True):
                key = f"{'LBFGS' if lb else 'FIRE'} K={K}"
                opts[key], arms[key] = device_arm(model, name, K, args.steps, lbfgs=lb)
        times = {k: [] for k in arms}
        for _ in range(args.reps):
            for k, fn in arms.items():
                times[k].append(fn())
        rec = {k: {"ms_per_step": statistics.median(v), "spread_ms": [min(v), max(v)]} for k, v in times.items()}
        lb = opts["LBFGS K=50"]
        if lb.step < 110:
            lb.run(0.0, 110 // 50 * 50 + 50)
        pairs = int(lb._iter[:, 1].min())
        rec["launches_ms_per_step"] = {"FIRE": fire_launch_ms(opts["FIRE K=50"]), "LBFGS": fire_launch_ms(lb),
                                       "LBFGS pairs stored": pairs}
        del opts, arms
        sp, co, cell, pbc = workload(name)
        if name == "gdb256":
            rec["to_fmax_0.05"] = lbfgs_to_fmax(model, sp, co, cell, pbc, 0.05, args.max_steps)
        result["workloads"][name] = rec
        print(name, json.dumps(rec, indent=1), flush=True)
    sp, co, _, _ = workload("gdb256")
    n = int((sp[0] >= 0).sum())
    result["molecule"] = {"atoms": n}
    for fmax in (1e-4, 1e-6):
        result["molecule"][f"to_fmax_{fmax:g}"] = lbfgs_to_fmax(model, sp[0, :n], co[0, :n], None, False, fmax,
                                                                args.floor_steps)
    print("molecule", json.dumps(result["molecule"]), flush=True)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "opt_lbfgs_timing.json"), "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps(result))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=500)
    ap.add_argument("--max-steps", type=int, default=3000)
    ap.add_argument("--floor-steps", type=int, default=5000)
    ap.add_argument("--workloads", default="gdb256,water1k")
    ap.add_argument("--cell", action="store_true", help="variable-cell FIRE against FIRE (see the docstring)")
    ap.add_argument("--lbfgs", action="store_true", help="L-BFGS against FIRE (see the docstring)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("opt_timing needs a GPU")
    from torchani_b200 import models
    model = models.ANI2x(seed=0)
    model = models.ANI(model.symbols, model.aev_computer, model.neural_networks, model.energy_shifter, False).cuda()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    result = {"device": torch.cuda.get_device_name(0), "nvidia_smi": smi, "steps": args.steps, "workloads": {}}
    if args.cell:
        cell_main(args, model, result)
        return
    if args.lbfgs:
        lbfgs_main(args, model, result)
        return
    for name in args.workloads.split(","):
        arms, opts = {}, {}
        for K in (1, 10, 50):
            opts[K], arms[f"device K={K}"] = device_arm(model, name, K, args.steps)
        arms["host"] = host_arm(model, name, max(50, args.steps // 5))
        times = {k: [] for k in arms}
        for _ in range(args.reps):
            for k, fn in arms.items():
                times[k].append(fn())
        rec = {k: {"ms_per_step": statistics.median(v), "spread_ms": [min(v), max(v)]} for k, v in times.items()}
        rec["fire_launches_ms_per_step"] = fire_launch_ms(opts[50])
        rec["to_fmax_0.05"] = to_fmax(model, name, 0.05, args.max_steps)
        result["workloads"][name] = rec
        print(name, json.dumps(rec, indent=1), flush=True)
    result["floor"] = floor(model, args.floor_steps)
    print("floor", json.dumps(result["floor"]), flush=True)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "opt_timing.json"), "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
