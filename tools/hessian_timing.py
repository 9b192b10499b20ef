#!/usr/bin/env python
"""Time ``models.ANI.energies_forces_hessians`` (ANI-2x-shaped x 8, the seeded weights of the golden fixtures) at
three molecule sizes: the first 20 and 100 atoms of the 1C17 chunk and the whole 312-atom chunk (open systems).

Per size: warm-up calls, then ``--reps`` timed calls (host clock around a call that ends in a device synchronise:
the ordinary step, the host planning of the chunks and every Hessian launch), and one call with
``Engine.profile = True`` that splits the Hessian's device time into its Jacobian, tangent network, geometric and
assembly launches (CUDA events around each, Engine.stage_events, summed over the chunks).  The flop count of the
tangent pass is 2 (ldx h1 + h1 h2 + h2 h3 + h3 h2 + h2 h1) per Jacobian row and active member (DESIGN.md 4.10).

Where oracle/_ref holds the reference's compiled package, the reference model with the same weights (its cuAEV path on
the GPU) is timed too, through ``torchani.grad.energies_forces_and_hessians`` -- after checking that its Hessian
agrees with ours (max |dH| <= 1e-3 max |H|); without it that arm is reported as absent.  Output: JSON in --out with the
device name and power limit.

    python tools/hessian_timing.py --out <dir> [--reps 5]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import oracle.ani_oracle as orc   # noqa: E402


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def timed(fn, reps: int) -> list:
    out = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1e3)
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/hessian_timing.py measures on a CUDA device; none is available")
    from torchani_b200 import models
    dev = torch.device("cuda:0")
    w64 = orc.make_weights(orc.SYMBOLS_2X, orc.DIMS_2X, 1008, 8, 1234, torch.float64)
    w32 = [{s: [(a.float(), b.float()) for a, b in layers] for s, layers in wm.items()} for wm in w64]
    model = models.from_weight_lists("2x", w32, device=dev, periodic_table_index=False)
    eng = model.engine(dev)
    z = np.load(os.path.join(ROOT, "tests", "golden", "1c17_chunk_hcnos_ani2x.npz"))
    species, coords = torch.tensor(z["species"]), torch.tensor(z["coords"], dtype=torch.float32)
    ref = None
    from oracle import ref_torchani
    if os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "torchani")):
        ref = ref_torchani.build_model(w64, "2x", device=dev, strategy="cuaev", periodic_table_index=False)
    result = {"card": card(), "sizes": []}
    for n in (20, 100, 312):
        sp, co = species[:, :n].to(dev), coords[:, :n].to(dev)
        call = lambda: model.energies_forces_hessians(sp, co)   # noqa: E731
        for _ in range(2):
            _, _, h = call()
        ms = timed(call, args.reps)
        eng.profile = True
        eng.stage_events.clear()
        call()
        torch.cuda.synchronize()
        stages = {k: sum(a.elapsed_time(b) for a, b in v) for k, v in eng.stage_events.items()
                  if k.startswith("hessian")}   # summed over the chunks
        eng.profile = False
        rows = 3 * int(eng.workspace(1, n).nbr_cnt[:n].sum())
        h1, h2, h3 = 256, 192, 160   # (the hydrogen network; the widest of ANI-2x)
        rec = {"atoms": n, "jacobian_rows": rows, "median_ms": float(np.median(ms)), "min_ms": float(min(ms)),
               "max_ms": float(max(ms)), "stages_ms": stages,
               "tangent_mflop_per_row_member_H": 2 * (1024 * h1 + h1 * h2 + h2 * h3 + h3 * h2 + h2 * h1) / 1e6}
        if ref is not None:
            torchani = ref_torchani.load()
            x = co.clone()
            out = torchani.grad.energies_forces_and_hessians(ref, sp, x)
            err = float((out.hessians - h).abs().max())
            rec["reference_max_abs_dH"] = err
            if err <= 1e-3 * float(h.abs().max()):
                rms = timed(lambda: torchani.grad.energies_forces_and_hessians(ref, sp, co.clone()), args.reps)
                rec["reference_median_ms"] = float(np.median(rms))
        result["sizes"].append(rec)
        print(json.dumps(rec))
    result["reference"] = "timed" if ref is not None else "absent (oracle/_ref not built)"
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "hessian_timing.json"), "w") as fh:
        json.dump(result, fh, indent=1)
    print(result["card"])


if __name__ == "__main__":
    main()
