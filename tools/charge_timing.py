#!/usr/bin/env python
"""Time the charge pass of an ANImbis-shaped model (models.ANIq) in the fused step.

Model: ANI-2x AEV and 8-member CELU ensemble (seeded weights, as bench.py), one set of charge networks with ANI-2x widths,
GELU, no biases, out_dim = 2 (seeded), the q^2-scaled normaliser with the weights of tests/golden/charges_mbis_*.npz.
Workloads: the 9 999-atom periodic water box and the GDB-like padded batch of 256 conformers.  Energy + forces,
Engine.run graph-replayed.  For each workload:

    step                 the step without charges
    step_charges_chained the step with charges, charge networks through ani_b200_mlp_forward (three launches)
    step_charges_step    the same through ani_b200_mlp_step(..., want_backward=0) (data-flow launch per window)
    forward_chained      the charge networks' forward alone (ani_b200_mlp_forward on the step's tiled AEVs)
    forward_step         the same through ani_b200_mlp_step(..., want_backward=0)
    charges_kernel       ani_b200_charges alone

The step arms alternate, CUDA events bracket K calls per repetition; the kernel-alone arms are K launches.  Before any
timing the charges of both forward entry points are compared (bitwise equal charges are not required; they must agree
to 1e-6 e).  Output: median and spread per arm in ms, the device name and power limit, as JSON in --out.

    python tools/charge_timing.py --out <dir> [--reps 20] [--k 20]
"""
from __future__ import annotations

import argparse
import ctypes as C
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


def build_model(dev):
    from torchani_b200 import electro, models, nn, synthetic
    w2x = synthetic.make_weights(models.SYMBOLS_2X, synthetic.DIMS_2X, 1008, 8, seed=1234)
    base = models.from_weight_lists("2x", w2x, periodic_table_index=False)
    qnets = nn.ChargeNetworks.like_2x(models.SYMBOLS_2X, 1008)
    g = torch.Generator().manual_seed(99)
    with torch.no_grad():
        for s in models.SYMBOLS_2X:
            for w, _ in qnets.atomics[s].linear_pairs():
                w.copy_((torch.rand(w.shape, generator=g) * 2 - 1) / w.shape[1] ** 0.5)
    rec = np.load(os.path.join(ROOT, "tests", "golden", "charges_mbis_small264_nopbc.npz"))
    norm = electro.ChargeNormalizer(models.SYMBOLS_2X, rec["norm_weights"].tolist(), True)
    m = models.ANIq(models.SYMBOLS_2X, base.aev_computer, base.neural_networks, base.energy_shifter, None, False,
                    qnets, norm)
    return m.to(dev).requires_grad_(False)


def timed(fn, k: int) -> float:
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(k):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / k


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--k", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        print("charge_timing: no CUDA device", file=sys.stderr)
        return 2
    from torchani_b200 import _lib, synthetic
    from torchani_b200._lib import check, ptr
    dev = torch.device("cuda:0")
    m = build_model(dev)
    eng = m.engine(dev)
    L = eng.lib
    _, idx, coords, cell, pbc = synthetic.water_box(3333, seed=0)
    sp_b, co_b = synthetic.conformer_batch(256)
    workloads = {"water_10k": (idx, coords, cell, True), "gdb_batch_256": (sp_b, co_b, None, False)}
    result = {"device": device_info(dev), "reps": args.reps, "k": args.k, "workloads": {}}
    ok = True
    for name, (sp, co, cl, periodic) in workloads.items():
        spd, cod = sp.to(dev), co.float().to(dev)
        cld = None if cl is None else cl.float().to(dev)
        ws, _ = eng._stage_inputs(spd, cod, cld, periodic)
        eng.charge_buffers(ws)
        qn, qp = eng.charges
        st = torch.cuda.current_stream(dev).cuda_stream

        def step(charges: bool, mode: str = "chained"):
            eng.charge_mlp = mode
            eng.run(ws, periodic, True, charges=charges)

        q = {}
        for mode in ("chained", "step"):
            step(True, mode)
            eng.check_status(ws)
            q[mode] = eng.charges_result(ws).charges.clone()
        diff = float((q["chained"] - q["step"]).abs().max())
        if not diff <= 1e-6:
            print(f"{name}: the two forward entry points disagree by {diff:.3e} e", file=sys.stderr)
            ok = False
            continue
        a1, a2, a3 = ws.q_act
        w, ms = qp.arrays()
        kernels = {
            "forward_chained": lambda: check(L.ani_b200_mlp_forward(
                C.byref(qn.model), ptr(ws.x), ws.rows_cap, ptr(ws.row_atom), ptr(ws.layout_info), ptr(ws.aev_blocks),
                ptr(a1), ptr(a2), ptr(a3), ptr(ws.q_raw), 0, ptr(ws.status), st)),
            "forward_step": lambda: check(L.ani_b200_mlp_step(
                C.byref(qn.model), ptr(ws.x), None, ws.rows_cap, ptr(ws.row_atom), ptr(ws.layout_info),
                ptr(ws.aev_blocks), ptr(a1), ptr(a2), ptr(a3), ptr(ws.q_raw), 0, ptr(ws.mlp_sync), ptr(ws.status), st)),
            "charges_kernel": lambda: check(L.ani_b200_charges(
                ptr(ws.q_raw), ptr(ws.row_of), ptr(ws.orig_to_sorted), ptr(ws.species_i32), ptr(ws.coords), ws.n_conf,
                ws.n_per_conf, w, qn.num_species, int(qp.scale_by_q2), 1, 0.0, ms, qp.frame, ptr(ws.charges),
                ptr(ws.dipoles), st)),
        }
        arms = {"step": lambda: step(False), "step_charges_chained": lambda: step(True, "chained"),
                "step_charges_step": lambda: step(True, "step")}
        for fn in list(arms.values()) + list(kernels.values()):   # warm-up, graph capture
            for _ in range(eng.graph_after + 3):
                fn()
        torch.cuda.synchronize()
        times = {k: [] for k in list(arms) + list(kernels)}
        for _ in range(args.reps):
            for k, fn in list(arms.items()) + list(kernels.items()):
                times[k].append(timed(fn, args.k))
        eng.check_status(ws)
        eng.charge_mlp = "chained"
        res = {k: {"median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v)} for k, v in times.items()}
        res["atoms"] = int((sp >= 0).sum())
        res["charge_launches"] = {"chained": 4, "step": L.ani_b200_mlp_step_windows(C.byref(qn.model), ws.rows_cap) + 1}
        result["workloads"][name] = res
        print(name, json.dumps({k: round(v["median_ms"], 4) for k, v in res.items() if isinstance(v, dict)
                                and "median_ms" in v}))
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "charge_timing.json"), "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps(result["device"]))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
