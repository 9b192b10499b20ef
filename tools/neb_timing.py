#!/usr/bin/env python
"""Time per step of the device NEB (torchani_b200.optimize.NEB) against host-driven NEB loops, with the ANI-2x-shaped
x8 ensemble and seeded synthetic weights (as bench.py and tools/opt_timing.py).

Workloads (a band: the system, a copy with every real atom displaced by 0.3 A, linear images between them with 0.05 A
of noise on the interior ones; aseneb, climbing image, k = 0.1):

    mol26      one band of 7 interior images of the first 26-atom molecule of synthetic.conformer_batch
    mol26x32   32 such bands (32 x 7 x 26 = 5824 atoms per force step)
    water1k    one band of 5 interior images of the periodic water box of 999 atoms

Arms, per workload (per NEB step; fmax = 0, so no band converges):

    device K=1 / 10 / 50   optimize.NEB with steps_per_replay K: one graph replay, one D2H copy and one
                           synchronisation per K steps; host clock around run(), which ends in a synchronisation
    host batched           HostCalculator.calculate on all interior images of all bands at once (one H2D, graph
                           replay, one D2H, synchronise), then the oracle's NEB projection and FIRE step in numpy
                           (oracle/neb_oracle.py), band by band
    host serial            ASE's NEB pattern: one HostCalculator.calculate per interior image, then the same numpy step
    launches               the three NEB launches alone (ani_b200_neb_step), 200 eager calls under CUDA events

The arms alternate over --reps rounds; medians and the spread are reported.  Results go to --out/neb_timing.json with
the device name and power limit read in the same run.

    python tools/neb_timing.py --out <dir> [--reps 5] [--steps 200]
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
    """(species (B, A), images (B, n, A, 3), cell, pbc)."""
    from torchani_b200 import synthetic
    if name.startswith("mol26"):
        sp, co = synthetic.conformer_batch(256)
        sp, co = sp.numpy(), co.double().numpy()
        c = int(np.argmax((sp >= 0).sum(1) == 26))
        sp, co, n, B = sp[c:c + 1, :26], co[c:c + 1, :26], 9, (32 if name == "mol26x32" else 1)
        cell, pbc = None, False
    else:
        _, idx, co, cell, _ = synthetic.water_box(333, seed=1)
        sp, co, n, B = idx.numpy(), co.double().numpy(), 7, 1
        cell, pbc = cell.double().numpy(), True
    rng = np.random.default_rng(0)
    bands = []
    for _ in range(B):
        end = co[0] + 0.3 * rng.standard_normal(co[0].shape)
        x = co[0][None] + np.linspace(0.0, 1.0, n)[:, None, None] * (end - co[0])[None]
        x[1:-1] += 0.05 * rng.standard_normal(x[1:-1].shape)
        bands.append(x)
    return np.repeat(sp, B, 0), np.stack(bands), cell, pbc


def device_arm(model, name, K, steps):
    from torchani_b200 import optimize
    sp, x, cell, pbc = workload(name)
    neb = optimize.NEB(model, sp, x, cell=cell, pbc=pbc, climb=True, steps_per_replay=K)
    steps = max(steps // K, 1) * K
    neb.run(0.0, 2 * K)   # capture + warm-up

    def timed():
        t0 = time.perf_counter()
        neb.run(0.0, steps)
        return (time.perf_counter() - t0) * 1e3 / steps
    return neb, timed


def launch_ms(neb, reps=200):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    state = neb._head.clone()
    a.record()
    for _ in range(reps):
        neb._integrate()
    b.record()
    b.synchronize()
    neb._head.copy_(state)
    return a.elapsed_time(b) / reps


class HostNEB:
    """NEB + FIRE in numpy (oracle/neb_oracle.step per band) on HostCalculator forces: all interior images in one
    call (batched) or one call per image (serial, ASE's pattern)."""

    def __init__(self, model, name, serial):
        import oracle.fire_oracle as fo
        import oracle.md_oracle as mo
        import oracle.neb_oracle as no
        from torchani_b200.calculator import HostCalculator
        self.fo, self.no = fo, no
        sp, x, cell, pbc = workload(name)
        self.B, self.n, self.A = x.shape[:3]
        m = self.n - 2
        self.serial = serial
        self.one = HostCalculator(model, sp[:1], cell=cell, pbc=pbc)
        self.calc = self.one if serial else HostCalculator(model, np.repeat(sp, m, 0), cell=cell, pbc=pbc)
        self.wrap = (lambda y: np.stack([mo.wrap(c, cell) for c in y])) if pbc else (lambda y: y)
        self.scale = np.where(sp[0] >= 0, fo.HARTREE_EV, 0.0)
        ends = x[:, [0, -1]].reshape(-1, self.A, 3)
        self.e_end = np.array([self._energy_forces(e[None], self.one)[0][0] for e in ends]).reshape(self.B, 2)
        self.par = fo.params(0.0)
        self.x, self.v = x.copy(), np.zeros_like(x[:, 1:-1])
        self.sc = [fo.init(self.par) for _ in range(self.B)]
        self.t = 0

    def _energy_forces(self, imgs, calc=None):
        e, f = (calc or self.calc).calculate(self.wrap(imgs))
        return np.asarray(e, dtype=np.float64).reshape(-1), np.asarray(f, dtype=np.float64).reshape(imgs.shape)

    def step(self):
        m, A = self.n - 2, self.A
        inner = self.x[:, 1:-1].reshape(-1, A, 3)
        if self.serial:
            ef = [self._energy_forces(y[None]) for y in inner]
            e, f = np.concatenate([a for a, _ in ef]), np.concatenate([b for _, b in ef])
        else:
            e, f = self._energy_forces(inner)
        e, f = e.reshape(self.B, m), f.reshape(self.B, m, A, 3) * self.scale[None, None, :, None]
        for b in range(self.B):
            E = np.concatenate([self.e_end[b, :1], e[b], self.e_end[b, 1:]])
            self.x[b], self.v[b], self.sc[b], _, _, _ = self.no.step(
                self.x[b], self.v[b], self.sc[b], E, f[b], 0.1, self.par, self.t, "aseneb", True,
                (self.scale != 0).astype(np.float64))
        self.t += 1


def host_arm(model, name, steps, serial):
    h = HostNEB(model, name, serial)
    for _ in range(3):
        h.step()

    def timed():
        t0 = time.perf_counter()
        for _ in range(steps):
            h.step()
        return (time.perf_counter() - t0) * 1e3 / steps
    return timed


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--workloads", default="mol26,mol26x32,water1k")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("neb_timing needs a GPU")
    from torchani_b200 import models
    model = models.ANI2x(seed=0)
    model = models.ANI(model.symbols, model.aev_computer, model.neural_networks, model.energy_shifter, False).cuda()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    result = {"device": torch.cuda.get_device_name(0), "nvidia_smi": smi, "steps": args.steps, "workloads": {}}
    for name in args.workloads.split(","):
        arms, nebs = {}, {}
        for K in (1, 10, 50):
            nebs[K], arms[f"device K={K}"] = device_arm(model, name, K, args.steps)
        host_steps = max(5, args.steps // 20)
        arms["host batched"] = host_arm(model, name, host_steps, False)
        arms["host serial"] = host_arm(model, name, host_steps, True)
        times = {k: [] for k in arms}
        for _ in range(args.reps):
            for k, fn in arms.items():
                times[k].append(fn())
        rec = {k: {"ms_per_step": statistics.median(v), "spread_ms": [min(v), max(v)]} for k, v in times.items()}
        sp, x, _, _ = workload(name)
        rec["atoms_per_force_step"] = int(x.shape[0] * (x.shape[1] - 2) * x.shape[2])
        rec["neb_launches_ms_per_step"] = launch_ms(nebs[50])
        result["workloads"][name] = rec
        print(name, json.dumps(rec, indent=1), flush=True)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "neb_timing.json"), "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
