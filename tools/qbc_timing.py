#!/usr/bin/env python
"""Time the query-by-committee step (Engine.run(..., members=True)) against the ordinary energy + force step, and
against the eager formulation it replaced.

Three arms, in one process, alternated, on the workloads of bench.py (water 1 k, water 10 k, the GDB batch of 256;
ANI-2x-shaped x8 ensemble with bench.py's seeded synthetic weights):

    step   the ordinary energy + force step (Engine.run), graph-replayed
    qbc    the QBC step: every member's forces from one AEV-backward launch and the statistics kernel, graph-replayed
    eager  the formulation before it, restated here: one want_backward=2 MLP step, then one single-slab
           ani_b200_aev_backward launch per member and the energy reduction, eagerly (no graph, no statistics)

Every arm is warmed up (eager uses and the graph capture happen before timing).  A 256 MiB buffer is overwritten
before every timed arm (L2 flush, untimed); CUDA events bracket each arm.  Before timing, the qbc arm's member
gradients are compared with the eager arm's (1e-5 of the largest component) and its mean gradient with the step's.
Output: median and spread per arm, the device name and power limit, as JSON in the directory given by --out.

    python tools/qbc_timing.py --out <dir> [--reps 20]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

WORKLOADS = ("water1k", "water10k", "gdb256")


def eager_members(eng, ws, pbc: bool, grads) -> None:
    """The eager formulation: preparation, AEV forward, ONE want_backward=2 MLP step, then ani_b200_aev_backward once
    per active member on its slab, and the energy reduction (grid modes 0 and 1 only, as used here)."""
    from torchani_b200._lib import MLPModel, ANI_MAX_MEMBERS, check, ptr
    from torchani_b200.engine import _grid_mode
    L, c, nets = eng.lib, eng.consts, eng.nets
    n, n_conf, n_per_conf = ws.n, ws.n_conf, ws.n_per_conf
    st = torch.cuda.current_stream().cuda_stream
    active = list(nets.active)
    model = MLPModel.from_buffer_copy(nets.model)
    for m in range(ANI_MAX_MEMBERS):
        model.member_scale[m] = 1.0 if m in active else 0.0
    grads.zero_()
    check(L.ani_b200_prepare_step(
        ptr(ws.coords), ptr(ws.species_i32), n_conf, n_per_conf, ptr(ws.cell) if pbc else None, int(pbc),
        _grid_mode(n_conf, pbc), c.rcr, ws.max_bins, ptr(ws.grid), ptr(ws.bin_start), ptr(ws.sorted_orig),
        ptr(ws.orig_to_sorted), ptr(ws.spos), ptr(ws.sbin), ptr(ws.bucket_ranges), 0, n, c.num_species, ws.rows_cap,
        ptr(ws.row_of), ptr(ws.row_atom), ptr(ws.tile_species), ptr(ws.layout_info), len(c.shf_r),
        len(c.shf_a) * len(c.shf_z), c.out_dim, nets.ldx, nets.col_pad, ptr(ws.aev_blocks), None, 0, None, 0,
        ptr(ws.bucket_species), ptr(ws.scratch), ptr(ws.status), st), "prepare_step")
    mask = ws.aev_blocks.data_ptr() + 4 * (ws.n_blocks + 1)
    check(L.ani_b200_aev_forward(
        C.byref(eng.params), ptr(ws.grid), ptr(ws.bin_start), ptr(ws.spos), ptr(ws.sbin), ptr(ws.bucket_ranges),
        ptr(ws.bucket_species), mask, n, 0, n, ptr(ws.row_of), ptr(ws.x), nets.ldx, 1, ptr(ws.nbr_cnt),
        ptr(ws.nbr_list), ws.nbr_cap, ptr(ws.status), st), "aev_forward")
    check(L.ani_b200_mlp_step(
        C.byref(model), ptr(ws.x), ptr(ws.dx_members), ws.rows_cap, ptr(ws.row_atom), ptr(ws.layout_info),
        ptr(ws.aev_blocks), ptr(ws.act1), ptr(ws.act2), ptr(ws.act3), ptr(ws.e_member), 2, ptr(ws.mlp_sync),
        ptr(ws.status), st), "mlp_step")
    for k, m in enumerate(active):
        check(L.ani_b200_aev_backward(
            C.byref(eng.params), ptr(ws.grid), ptr(ws.spos), ptr(ws.sorted_orig), mask, n, 0, n, ptr(ws.row_of),
            ws.dx_members[m].data_ptr(), nets.ldx, ptr(ws.nbr_cnt), ptr(ws.nbr_list), ws.nbr_cap, grads[k].data_ptr(),
            ptr(ws.status), 0, None, st), "aev_backward")
    check(L.ani_b200_reduce_energies(
        C.byref(model), ptr(ws.e_member), ws.rows_cap, ptr(ws.row_of), ptr(ws.orig_to_sorted), ptr(ws.species_i32),
        n, 0, n, n_conf, n_per_conf, None, ptr(ws.atomic), ptr(ws.member_atomic), ptr(ws.energies), st),
        "reduce_energies")


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=20, help="timed repetitions of each arm")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        print("qbc_timing: no CUDA device", file=sys.stderr)
        return 2
    from bench import make_workload
    from periodic_batch_timing import device_info
    from torchani_b200 import models
    from torchani_b200.engine import Engine
    from torchani_b200.synthetic import DIMS_2X, make_weights
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    weights = make_weights(models.SYMBOLS_2X, DIMS_2X, 1008, 8, seed=1234)
    model = models.from_weight_lists("2x", weights, device=dev, periodic_table_index=True)
    base = model.engine(dev)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    rows, ok = [], True
    for name in WORKLOADS:
        w = make_workload(name)
        eng = Engine(base.consts, base.nets, base.sae.tolist(), nbr_cap=base.nbr_cap)
        idx, co = w["idx"].to(dev), w["coords"].to(dev).float()
        pbc = w["pbc"] is not None
        ws = eng.workspace(*idx.shape)
        ws.species_i32.copy_(idx.reshape(-1))
        ws.coords.copy_(co.reshape(-1, 3))
        if pbc:
            ws.cell.copy_(w["cell"].to(dev).float().reshape(-1))
        eng.members_buffers(ws)
        M = len(eng.nets.active)
        grads = torch.zeros(M, ws.n, 3, device=dev)
        g_step = torch.zeros(ws.n, 3, device=dev)

        def step():
            eng.run(ws, pbc, True)

        def qbc():
            eng.run(ws, pbc, True, members=True)

        def eager():
            eager_members(eng, ws, pbc, grads)

        for _ in range(eng.graph_after + 3):
            step()
        g_step.copy_(ws.grad)
        for _ in range(eng.graph_after + 3):
            qbc()
        g_mean = ws.grad.clone()
        g_qbc = ws.grad_members[:M].clone()
        for _ in range(3):
            eager()
        eng.check_status(ws)
        torch.cuda.synchronize()
        scale = float(grads.abs().max())
        d_members = float((g_qbc - grads).abs().max())
        d_mean = float((g_mean - g_step).abs().max())
        row = {"workload": name, "atoms": w["n_atoms"], "n_conf": w["n_conf"], "members": M,
               "max_member_grad_diff": d_members, "max_mean_grad_diff": d_mean}
        if d_members > 1e-5 * scale or d_mean > 1e-5 * scale:
            row["error"] = "the arms disagree: not timed"
            ok = False
            rows.append(row)
            print(json.dumps(row), flush=True)
            continue
        times = {"step": [], "qbc": [], "eager": []}
        for _ in range(args.reps):
            for arm, fn in (("step", step), ("qbc", qbc), ("eager", eager)):
                flush.fill_(1)
                ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                ev0.record()
                fn()
                ev1.record()
                ev1.synchronize()
                times[arm].append(ev0.elapsed_time(ev1))
        eng.check_status(ws)
        for arm, t in times.items():
            row[arm] = {"median_ms": statistics.median(t), "min_ms": min(t), "max_ms": max(t)}
        row["qbc_over_step"] = row["qbc"]["median_ms"] / row["step"]["median_ms"]
        row["eager_over_qbc"] = row["eager"]["median_ms"] / row["qbc"]["median_ms"]
        rows.append(row)
        print(json.dumps(row), flush=True)
        del eng, ws
        torch.cuda.empty_cache()
    record = {"tool": "qbc_timing", **device_info(dev), "reps": args.reps,
              "method": "CUDA events around each arm, arms alternated, 256 MiB L2 flush before each (untimed); step "
                        "and qbc graph-replayed, eager without a graph", "rows": rows}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "qbc_timing.json"), "w") as fh:
        json.dump(record, fh, indent=1)
    print(json.dumps({k: v for k, v in record.items() if k != "rows"}))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
