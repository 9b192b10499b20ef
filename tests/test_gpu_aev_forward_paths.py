"""The two AEV forward kernels against each other, bit for bit.

``k_aev_forward_cta`` (the default on the bucket grid) stages a CTA's 27-bucket neighbourhood in shared memory;
``k_aev_forward`` (``ANI_B200_AEV_LEGACY=1``, and the explicit-row entry points) walks every atom's candidate ranges
itself and regroups the neighbours by species.  Both then run the same per-atom feature code on the same neighbour
order (species, range, position), so as long as nbr_cap holds they must agree exactly: plain and tiled AEVs,
neighbour counts and words, status, and one engine step's energies.  The step's gradient is summed with float atomics
by the AEV backward, so its last bits change from run to run of either kernel: it is compared at 1e-6 of its largest
component.

The switch is read once per process, so each side runs in a child process (this file as a script, under a timeout)
that saves its outputs to a temporary directory; the test compares them with ``torch.equal``.  The systems come from
the generators of ``test_gpu_aev.py``.
"""
import ctypes as C
import os
import subprocess
import sys
import typing as tp

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path[:0] = [p for p in (HERE, ROOT) if p not in sys.path]   # run as a script by the test below

import test_gpu_aev as ta  # noqa: E402

DEV = "cuda:0"


class Case(tp.NamedTuple):
    name: str
    cfg: str          # test_gpu_aev.CFG key (ShfA x ShfZ = 8 x 4 or 4 x 8)
    mode: int         # ani_grid::mode the engine must choose
    cap: int


CASES = [
    Case("cubic_8x4", "s8_r17", 0, 128),
    Case("cubic_4x8", "s3_r32", 0, 128),
    Case("skewed_8x4", "s7_r16", 0, 128),
    Case("skewed_4x8", "s7_r15", 0, 128),
    Case("open_batch", "s8_r17", 1, 128),
    Case("periodic_batch", "s3_r32", 2, 128),
    Case("conformer_cells", "s8_r17", 3, 128),
    Case("dense", "s7_r16", 0, 256),       # more than 768 candidates per CTA: several staging windows
]


def system(case: Case) -> tp.Tuple[torch.Tensor, torch.Tensor, tp.Optional[torch.Tensor]]:
    """(species, coords, cell) on the host; the last element of the configuration is absent everywhere."""
    S = ta.CFG[case.cfg].S
    present = list(range(S - 1))
    if case.name.startswith("cubic"):
        s = ta.random_box(240, 0.1, present, seed=3)
        return s.species, s.coords, s.cell
    if case.name.startswith("skewed"):
        s = ta.skewed_cell_system()
        return s.species % (S - 1), s.coords, s.cell
    if case.name == "dense":
        s = ta.random_box(1100, 0.3, present, seed=17)
        return s.species, s.coords, s.cell
    # batches of three conformers: the same cubic cell (mode 2), none (mode 1), or three different cells (mode 3)
    densities = (0.1, 0.08, 0.12) if case.mode == 3 else (0.1, 0.1, 0.1)
    boxes = [ta.random_box(200, d, present, seed=40 + k) for k, d in enumerate(densities)]
    sp = torch.cat([b.species for b in boxes])
    co = torch.cat([b.coords for b in boxes])
    if case.mode == 1:
        return sp, co, None
    if case.mode == 2:
        return sp, co, boxes[0].cell
    return sp, co, torch.stack([b.cell for b in boxes])


def outputs(case: Case) -> tp.Dict[str, torch.Tensor]:
    """Every output of the AEV forward entry point for one system, with and without the range table, plain and
    tiled, with the step's element mask (dead elements skipped) and with the composition-changed flag set; then one
    engine step with gradients."""
    from torchani_b200._lib import check, ptr
    from torchani_b200.engine import operand_buffer
    spec = ta.spec_of(ta.CFG[case.cfg])
    eng, _, _ = ta.make_engine(spec, nbr_cap=case.cap)
    sp, co, cell = (None if t is None else t.to(DEV) for t in system(case))
    pbc = cell is not None
    for _ in range(2):   # the second step sees an unchanged composition
        eng.step(sp, co, cell, pbc, want_grad=False)
    torch.cuda.synchronize()
    ws = eng.workspace(*sp.shape)
    assert eng.grid_info(ws).mode == case.mode
    n, ldx, L = ws.n, eng.nets.ldx, eng.lib
    mask = int(ws.aev_blocks[ws.n_blocks + 1].item())
    assert mask == (1 << (spec.num_species - 1)) - 1, "one element must be absent"
    masks = {"all": None, "mask": torch.tensor([mask, 0], dtype=torch.int32, device=DEV),
             "changed": torch.tensor([mask, 1], dtype=torch.int32, device=DEV)}
    lat = (ptr(ws.lattice),) if case.mode == 3 else ()
    forward = L.ani_b200_aev_forward_cells if lat else L.ani_b200_aev_forward
    tables = {"table": ws.bucket_ranges, "no_table": None}
    if case.mode == 1:
        tables = {"no_table": None}      # one bucket per conformer: no range table
    else:
        assert ws.bucket_ranges is not None
    if case.name == "dense":
        rng = ws.bucket_ranges.view(-1, 27, 2, 4)[:, :, 0, :2].contiguous().view(torch.int32).cpu()
        occupied = torch.unique(ws.sbin[:n].long().cpu())
        assert int((rng[..., 1] - rng[..., 0]).clamp(min=0).sum(1)[occupied].max()) > 768
    out = {}
    st = torch.cuda.current_stream().cuda_stream
    for tname, table in tables.items():
        for mname, m in masks.items():
            for layout in (0, 1):
                x = (torch.full((ws.rows_cap, ldx), ta.SENTINEL, device=DEV) if layout == 0
                     else operand_buffer(ws.rows_cap, ldx, DEV))
                cnt = torch.full((n,), -1, dtype=torch.int32, device=DEV)
                words = torch.full((n * ws.nbr_cap,), -1, dtype=torch.int32, device=DEV)
                status = torch.zeros(1, dtype=torch.int32, device=DEV)
                check(forward(C.byref(eng.params), ptr(ws.grid), ptr(ws.bin_start), ptr(ws.spos), ptr(ws.sbin),
                              ptr(table), None, ptr(m), n, 0, n, ptr(ws.row_of), ptr(x), ldx, layout, ptr(cnt),
                              ptr(words), ws.nbr_cap, ptr(status), *lat, st), "aev_forward")
                torch.cuda.synchronize()
                assert int(status.item()) == 0, (tname, mname, layout, int(status.item()))
                key = f"{tname}/{mname}/layout{layout}"
                out.update({f"{key}/aev": x.cpu(), f"{key}/nbr_cnt": cnt.cpu(), f"{key}/nbr_list": words.cpu(),
                            f"{key}/status": status.cpu()})
    res = eng.step(sp, co, cell, pbc, check=True)
    out["step/energies"] = res.energies.cpu()
    out["step/grad"] = res.grad.cpu()
    return out


def _dump(outdir: str) -> None:
    for case in CASES:
        torch.save(outputs(case), os.path.join(outdir, case.name + ".pt"))


@pytest.fixture(scope="module")
def dumps(tmp_path_factory):
    """{"staged": dir, "warp": dir} with one file of outputs per case from each kernel."""
    dirs = {}
    for side, legacy in (("staged", "0"), ("warp", "1")):
        d = tmp_path_factory.mktemp(side)
        env = dict(os.environ, ANI_B200_AEV_LEGACY=legacy)
        cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), str(d)]
        res = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
        assert res.returncode == 0, res.stdout[-4000:] + res.stderr[-4000:]
        dirs[side] = str(d)
    return dirs


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_warp_per_atom_search_matches_the_staged_kernel(dumps, case):
    a = torch.load(os.path.join(dumps["staged"], case.name + ".pt"))
    b = torch.load(os.path.join(dumps["warp"], case.name + ".pt"))
    assert a.keys() == b.keys()
    differ = [k for k in a if k != "step/grad" and not torch.equal(a[k], b[k])]
    assert not differ, f"{case.name}: the kernels differ in {differ}"
    g, h = a["step/grad"], b["step/grad"]
    assert float((g - h).abs().max()) <= 1e-6 * float(g.abs().max())


if __name__ == "__main__":
    _dump(sys.argv[1])
