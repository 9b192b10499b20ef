#!/usr/bin/env python
"""Time the explicit-row AEV forward: ``AEVComputer.compute_from_neighbors`` on a half pair list, graph-replayed.

Workload: the 9 999-atom periodic water box of bench.py (ANI-2x constants), its half pair list within Rcr from
``neighbors.cell_list``.  Two measurements, each a CUDA graph replayed between CUDA events after warm-up:

    call    the two launches compute_from_neighbors issues for the forward: ani_b200_pairs_to_rows (pairs ->
            per-atom rows) and ani_b200_aev_forward_rows, on buffers allocated once
    kernel  ani_b200_aev_forward_rows alone, 20 launches per graph on rows built once

Every figure is the median over --reps windows of --iters replays, with the smallest and largest window.  Output: JSON
in --out (times in microseconds, the device name and power limit), and with --save-aev the AEVs as a float32 .npy
file, for a comparison between builds.

    python tools/aev_rows_timing.py --out <dir> [--reps 7] [--iters 100] [--save-aev <file>]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


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


def time_graph(fn, reps: int, iters: int) -> dict:
    """Median / min / max over `reps` windows of the time per replay (us) of a graph of fn."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    for _ in range(10):
        g.replay()
    torch.cuda.synchronize()
    t = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            g.replay()
        b.record()
        b.synchronize()
        t.append(a.elapsed_time(b) * 1e3 / iters)
    return {"median_us": statistics.median(t), "min_us": min(t), "max_us": max(t)}


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--save-aev", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        print("aev_rows_timing: no CUDA device", file=sys.stderr)
        return 2
    from torchani_b200 import _lib, neighbors, synthetic
    from torchani_b200.aev import AEVComputer
    dev = torch.device("cuda:0")
    m = AEVComputer.like_2x().to(dev)
    _, idx, coords, cell, pbc = synthetic.water_box(3333, seed=0)
    sp, co = idx.to(dev), coords.to(dev)
    nb = neighbors.cell_list(m.constants.rcr, sp, co, cell.to(dev), pbc.to(dev))
    pairs, diff = nb.indices.contiguous(), nb.diff_vectors.float().contiguous()
    with torch.no_grad():
        aev = m.compute_from_neighbors(sp, co, nb)   # checks the status words once
    torch.cuda.synchronize()
    if args.save_aev:
        np.save(args.save_aev, aev.cpu().numpy())

    L, n, cap, D = _lib.lib(), sp.numel(), m.nbr_cap, m.constants.out_dim
    i32 = dict(dtype=torch.int32, device=dev)
    P = pairs.shape[1]
    row_start, row_j = torch.zeros(n + 1, **i32), torch.zeros(2 * P, **i32)
    row_d, scratch, status = torch.zeros(2 * P, 4, device=dev), torch.zeros(2 * n, **i32), torch.zeros(1, **i32)
    st = torch.cuda.current_stream().cuda_stream
    _lib.check(L.ani_b200_pairs_to_rows(pairs[0].data_ptr(), pairs[1].data_ptr(), diff.data_ptr(), P, n, cap,
                                        row_start.data_ptr(), row_j.data_ptr(), row_d.data_ptr(), scratch.data_ptr(),
                                        status.data_ptr(), st))
    spos = torch.zeros(n, 4, device=dev)
    spos[:, 3] = sp.reshape(-1).to(torch.int32).view(torch.float32)
    grid = torch.zeros(C.sizeof(_lib.Grid) // 4, **i32)
    grid[_lib.Grid.n_real.offset // 4] = n
    ident = torch.arange(n, **i32)
    out = torch.zeros(n, D, device=dev)
    params = m._params()

    def rows():
        L.ani_b200_pairs_to_rows(pairs[0].data_ptr(), pairs[1].data_ptr(), diff.data_ptr(), P, n, cap,
                                 row_start.data_ptr(), row_j.data_ptr(), row_d.data_ptr(), scratch.data_ptr(),
                                 status.data_ptr(), torch.cuda.current_stream().cuda_stream)

    def forward():
        L.ani_b200_aev_forward_rows(C.byref(params), grid.data_ptr(), spos.data_ptr(), row_start.data_ptr(),
                                    row_j.data_ptr(), row_d.data_ptr(), n, ident.data_ptr(), out.data_ptr(), D, 0, cap,
                                    status.data_ptr(), torch.cuda.current_stream().cuda_stream)

    def call():
        rows()
        forward()

    def kernel():
        for _ in range(20):
            forward()

    res = {"workload": f"water box, {n} atoms, {P} pairs within Rcr, nbr_cap {cap}", **device_info(dev),
           "call": time_graph(call, args.reps, args.iters)}
    k = time_graph(kernel, args.reps, max(args.iters // 10, 1))
    res["kernel"] = {key: v / 20 for key, v in k.items()}
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "aev_rows_timing.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    sys.exit(main())
