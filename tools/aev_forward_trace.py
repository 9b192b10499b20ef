"""Phase split of the CTA-staged AEV forward kernel (k_aev_forward_cta): clock64 cycles per phase and warp.

    python tools/aev_forward_trace.py [--molecules 3333]

Builds the library variant compiled with -DANI_AEV_FWD_TRACE=1 (torchani_b200/libani_b200_aevtrace.so) and runs one
water-box step with it.  Per phase it prints the median and p90 over the atoms' records (one
record per atom: its warp's time; every warp takes part in its whole CTA's staging), then the span of the launch and
the idle tail of the SMs: span end minus the last record end on each SM (median and max over SMs).
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PHASES = ["ranges", "count", "place", "compact", "list", "radial", "angular"]
WORDS = 16


def trace(n_mol: int) -> dict:
    sys.path.insert(0, ROOT)
    from torchani_b200 import build
    os.environ["ANI_B200_LIB"] = build.build(variant="aevtrace")   # read when torchani_b200._lib is imported
    import numpy as np
    import torch
    from torchani_b200 import _lib, synthetic
    from torchani_b200.engine import Engine, PackedNetworks, constants_2x

    dev = torch.device("cuda:0")
    consts = constants_2x()
    symbols = ("H", "C", "N", "O", "S", "F", "Cl")
    w = synthetic.make_weights(symbols, synthetic.DIMS_2X, 1008, 8, seed=1)
    nets = PackedNetworks([[wm[s] for s in symbols] for wm in w], consts.out_dim, dev)
    _, idx, coords, cell, _ = synthetic.water_box(n_mol, seed=0)
    eng = Engine(consts, nets, None, cuda_graph=False)
    sp, co, ce = idx.to(dev), coords.to(dev), cell.to(dev)
    for _ in range(5):
        eng.step(sp, co, ce, True)
    torch.cuda.synchronize()
    n = eng.workspace(*idx.shape).n
    buf = torch.zeros(n * WORDS, dtype=torch.int64, device=dev)
    _lib.check(_lib.lib().ani_b200_debug_aev_trace(buf.data_ptr()), "debug_aev_trace")
    eng.step(sp, co, ce, True)
    torch.cuda.synchronize()
    _lib.check(_lib.lib().ani_b200_debug_aev_trace(None), "debug_aev_trace")
    r = buf.view(-1, WORDS).cpu().numpy()
    atoms = allr = r[:n][r[:n, 8] != 0]
    ghz = float((allr[:, 11] - allr[:, 10]).sum() / (allr[:, 9] - allr[:, 8]).sum())  # cycles per ns
    us = lambda cyc: cyc / ghz / 1e3  # noqa: E731
    t0, t1 = int(allr[:, 8].min()), int(allr[:, 9].max())
    last = {}
    for row in allr:
        last[int(row[12])] = max(last.get(int(row[12]), 0), int(row[9]))
    tails = np.array([t1 - v for v in last.values()]) / 1e3
    life = atoms[:, 11] - atoms[:, 10]
    out = {"atoms": len(atoms), "sm_ghz": ghz, "span_us": (t1 - t0) / 1e3,
           "sms": len(last), "tail_idle_us": {"median": float(np.median(tails)), "max": float(tails.max())},
           "life_us": {"median": float(us(np.median(life))), "p90": float(us(np.percentile(life, 90)))},
           "staging_share": float(atoms[:, 0:3].sum() / life.sum()), "phases_us": {}}
    for k, name in enumerate(PHASES):
        out["phases_us"][name] = {"median": float(us(np.median(atoms[:, k]))),
                                  "p90": float(us(np.percentile(atoms[:, k], 90)))}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--molecules", type=int, default=3333)
    d = trace(ap.parse_args().molecules)
    print(f"== k_aev_forward_cta: {d['atoms']} atoms, span {d['span_us']:.1f} us, SM idle tail median "
          f"{d['tail_idle_us']['median']:.1f} / max {d['tail_idle_us']['max']:.1f} us over {d['sms']} SMs, "
          f"{d['sm_ghz']:.2f} GHz, staging (with its barriers) {100 * d['staging_share']:.0f} % of a warp's time")
    print(f"   per atom: life median {d['life_us']['median']:.2f} us, p90 {d['life_us']['p90']:.2f} us")
    for name in PHASES:
        v = d["phases_us"][name]
        print(f"   {name:8s} median {v['median']:7.2f} us   p90 {v['p90']:7.2f} us")
    print("   json " + json.dumps(d))


if __name__ == "__main__":
    main()
