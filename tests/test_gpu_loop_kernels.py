"""The device loop kernels on their own (csrc/md.cu, csrc/opt.cu, csrc/lbfgs.cu, csrc/md_common.cuh): the C-ABI entry
points driven directly, with no model, engine or force step, against the float64 oracles, step by step.

Each step the test computes a synthetic gradient from the device's current float64 positions (a quadratic with a
random SPD block-banded Hessian, a quartic term and one indefinite direction, so that L-BFGS meets pairs with y.s < 0),
rounds it to float32 and uploads it: device and oracle then see the same bits.  Every step is compared from the
device's own state before that step (read back, one oracle step, compare), so errors cannot compound; the kernels are
float64 in a fixed order without atomics, so positions, velocities, scalars and records agree with the oracle to
rounding (1e-12 relative), and a replay from a saved state gives the same bits (bar 0).

The shapes are where the kernels change form:
* MD, FIRE, cell FIRE: n_per_conf 1, 255, 256, 257 and 8193 (33 blocks of ANI_MD_BLOCK: the second pass over the
  per-block partials is lane-strided past 32 blocks);
* L-BFGS: n_per_conf 1, 31, 32, 33 and 1025 (33 tiles: the fmax and pmax partials' lane-strided loops), memory 1, 7,
  8, 9, 32, 33 and 128 (dot-sweep groups blockIdx.y >= 1 for rows >= 8, the direction sweep over eight warps for
  L > 8, the lane-strided triangular solves for L > 32, the row totals of rows = 129 > LB_SOLVE), run past a full and
  wrapped ring, with pairs skipped (y = 0 exactly) before and after the ring is full;
* n_conf 65535 with one atom each (the grid.y limit);
* distinct parameter rows per conformer (a kernel that read conformer 0's row, or the wrong stride, fails);
* open cells, one shared triclinic cell with a negative tilt, and the per-conformer lattice table
  (ANI_LATTICE_STRIDE), with positions several cells away on both sides;
* padding and fixed atoms, scattered and in the last block.
"""
import math

import mpmath
import numpy as np
import pytest
import torch

import oracle.cell_fire_oracle as cfo
import oracle.fire_oracle as fo
import oracle.lbfgs_oracle as lo
import oracle.md_oracle as mo
import oracle.npt_oracle as no

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
REL = 1e-12
INF = float("inf")


def _lib():
    from torchani_b200 import _lib
    return _lib


def L():
    return _lib().lib()


def ptr(t):
    return None if t is None else t.data_ptr()


def call(rc, what):
    assert rc == 0, f"{what}: {L().ani_b200_error_string(rc).decode()}"
    torch.cuda.synchronize()


def dev(a, dtype=torch.float64):
    return torch.as_tensor(np.ascontiguousarray(a)).to(device=DEV, dtype=dtype)


def h(t):
    return t.detach().cpu().numpy().copy()


def close(got, ref, what, rel=REL, scale=None):
    got, ref = np.asarray(got, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    s = np.abs(ref).max() if scale is None else scale
    err = np.abs(got - ref).max() if ref.size else 0.0
    assert err <= rel * max(s, 1e-300), f"{what}: {err:.3e} (scale {s:.3e})"


# ------------------------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------------------------
TRICLINIC = np.array([[11.0, 0.0, 0.0], [-3.25, 10.5, 0.0], [1.75, -2.5, 9.75]])   # negative tilts


def cells_for(mode, C):
    """(C, 3, 3) float32-exact cell rows of the cell mode, or None when open."""
    if mode == "open":
        return None
    if mode == "shared":
        return np.repeat(TRICLINIC[None], C, 0)
    return np.stack([TRICLINIC * (1.0 + 0.125 * c) + np.diag([0.0, 0.5 * c, -0.25 * c]) for c in range(C)])


def cell_args(mode, cells):
    """(the init's cells f32 and cell_mode, the step's cell argument f32, is it the lattice table)"""
    if mode == "open":
        return None, 0, None, False
    if mode == "shared":
        c = dev(cells[0].reshape(9), torch.float32)
        return c, 1, c, False
    per = dev(cells.reshape(-1, 9), torch.float32)
    table = np.concatenate([cells.reshape(-1, 9), np.linalg.inv(cells).reshape(-1, 9)], 1)
    return per, 2, dev(table, torch.float32), True


class Field:
    """The synthetic energy surface of (C, A) atoms: E = 1/2 d K d + kc/2 sum |d_i - d_(i+1)|^2 (a ring) + q/4 sum d^4
    - lam/2 (u.d)^2 with d = x - x0, K a random SPD 3 x 3 block per atom and u a unit vector per conformer (the
    indefinite direction).  ``grad`` is dE/dx rounded to float32."""

    def __init__(self, x0, rng, k=0.02, kc=0.005, q=0.002, lam=0.03):
        C, A, _ = x0.shape
        self.x0 = x0
        Q = np.linalg.qr(rng.standard_normal((A, 3, 3)))[0]
        self.K = np.einsum("aij,aj,akj->aik", Q, k * rng.uniform(0.5, 2.0, (A, 3)), Q)
        self.kc, self.q, self.lam = kc, q, lam
        u = rng.standard_normal((C, A, 3))
        self.u = u / np.sqrt((u * u).sum((1, 2), keepdims=True))

    def grad(self, x):
        d = x - self.x0
        g = np.einsum("aij,caj->cai", self.K, d) + self.q * d ** 3
        g += self.kc * (2.0 * d - np.roll(d, 1, 1) - np.roll(d, -1, 1))
        g -= self.lam * (d * self.u).sum((1, 2))[:, None, None] * self.u
        return g.astype(np.float32)


def positions(rng, C, A, cells, spread=8.0):
    """Random positions, each moved by a random whole number of cells in -3..3 along every lattice vector."""
    x = rng.uniform(0.0, spread, (C, A, 3))
    if cells is not None:
        x += np.einsum("cak,ckj->caj", rng.integers(-3, 4, (C, A, 3)).astype(np.float64), cells)
    return x


def padding(C, A, every=7, block=256):
    """Padding / fixed atoms: every ``every``-th atom, scattered, and one atom of the last ``block``-atom block (or tile)
    when it holds more than one, else one of the block before; the first atom of the last block is always real, so
    that every block writes nonzero partials and a second pass that missed block 33 (or tile 33) would show.  None
    with one atom."""
    pad = np.zeros((C, A), dtype=bool)
    if A > 1:
        pad[:, 3::every] = True
        first = (A - 1) // block * block
        pad[:, -1 if A - first > 1 else -2] = True
        pad[:, first] = False
    return pad


def hot_last_atom(field, A):
    """Move the minimum of the last atom 3 A away, so that it carries the largest force of its conformer (and, in
    L-BFGS, the largest step) for the first steps: the maxima over the blocks or tiles then come from the last one."""
    if A > 1:
        field.x0[:, -1] += 3.0


def check_coords(c32, before, x, cells, written):
    """The float32 coordinates: float32 of x wrapped into the cell (fractional coordinates minus their floor) for the
    atoms the step moved, within half a float32 ulp and the rounding of the wrap's float64 arithmetic (either image for an atom
    within 1e-12 of a face); unchanged for the others."""
    assert np.array_equal(c32[~written], before[~written]), "coordinates of atoms that did not move"
    for c in range(x.shape[0]):
        w = written[c]
        if not w.any():
            continue
        xc, got = x[c][w], c32[c][w].astype(np.float64)
        if cells is None:
            assert np.array_equal(c32[c][w], xc.astype(np.float32))
            continue
        inv = np.linalg.inv(cells[c])
        frac = xc @ inv
        n = np.round((xc - got) @ inv)
        near = np.abs(frac - np.round(frac)) < 1e-12
        assert ((n == np.floor(frac)) | (near & (np.abs(n - np.floor(frac)) <= 1))).all(), "wrong image"
        ref = xc - n @ cells[c]
        # float32 rounding to nearest: half an ulp of the result, plus the float64 rounding of the wrap itself
        tol = 0.5 * np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64) + 1e-14 * np.abs(xc).max()
        assert (np.abs(got - ref) <= tol).all(), np.abs(got - ref).max()


def snapshot(bufs):
    return [b.clone() for b in bufs]


def restore(bufs, saved):
    for b, s in zip(bufs, saved):
        b.copy_(s)
    torch.cuda.synchronize()


def bits(bufs):
    return [h(b.view(torch.uint8)) for b in bufs]


def same_bits(a, b):
    assert len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))


# ------------------------------------------------------------------------------------------------------------------
# 1. the Langevin noise against the Philox restatement of the oracle
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed, step", [(0, 0), (0x0123456789ABCDEF, 7), (2 ** 64 - 1, (3 << 32) + 5), (42, -1)])
def test_md_noise_matches_the_philox_restatement(seed, step):
    """ani_b200_md_noise and ani_b200_md_cell_noise against md_oracle.normal (Philox4x32-10, counter (step, atom,
    component), key the seed, Box-Muller's cosine branch) to 1e-14 max(1, |z|): the counter and key words, their
    halves and the atom / component mapping."""
    n = 3 * mo_block() + 5
    out = torch.zeros(n, 3, dtype=torch.float64, device=DEV)
    call(L().ani_b200_md_noise(seed, step, n, ptr(out), None), "md_noise")
    ref = mo.normal(np.uint64(seed), step, np.arange(n)[:, None], np.arange(3)[None])
    z = h(out)
    assert (np.abs(z - ref) <= 1e-14 * np.maximum(1.0, np.abs(ref))).all(), np.abs(z - ref).max()
    cn = torch.zeros(n, dtype=torch.float64, device=DEV)
    call(L().ani_b200_md_cell_noise(seed, step, n, ptr(cn), None), "md_cell_noise")
    ref = mo.normal(np.uint64(seed), step, np.arange(n), 3)
    assert (np.abs(h(cn) - ref) <= 1e-14 * np.maximum(1.0, np.abs(ref))).all()


def mo_block():
    return _lib().ANI_MD_BLOCK


# ------------------------------------------------------------------------------------------------------------------
# 2. MD: velocity Verlet and Langevin
# ------------------------------------------------------------------------------------------------------------------
class MD:
    """One ani_md_state on torch buffers, sized as the header and md.py size them."""

    def __init__(self, C, A, integrator, mode, seed=1, qbc=False, record_every=2, frame_slots=2, frame_v=True,
                 rows=3, zero_momentum=False):
        lib_ = _lib()
        rng = np.random.default_rng(seed)
        self.C, self.A, self.integrator, self.mode = C, A, integrator, mode
        self.cells = cells_for(mode, C)
        x = positions(rng, C, A, self.cells)
        self.field = Field(x + rng.normal(0, 0.2, x.shape), rng)
        self.pad = padding(C, A)
        mass = rng.uniform(1.0, 16.0, (C, A))
        self.inv = np.where(self.pad, 0.0, 1.0 / mass)
        v = np.where(self.pad[..., None], 0.0, rng.normal(0.0, 0.01, (C, A, 3)))
        par = np.zeros((C, lib_.ANI_MD_PARAMS))
        par[:, 0] = [0.5, 0.75, 1.25][:C] if C <= 3 else 0.5 + 0.25 * (np.arange(C) % 4)
        par[:, 1] = [300.0, 150.0, 600.0][:C] if C <= 3 else 300.0
        par[:, 2] = [0.01, 0.05, 0.2][:C] if C <= 3 else 0.02
        par[:, 3] = INF
        par[:, 4] = INF
        par[:, 5] = 3 * (~self.pad).sum(1)
        self.par = par
        n = C * A
        self.nb = -(-A // lib_.ANI_MD_BLOCK)
        self.x, self.v = dev(x), dev(v)
        self.inv_t, self.par_t = dev(self.inv.reshape(-1)), dev(par)
        self.counter = torch.zeros(2, dtype=torch.int64, device=DEV)
        self.stop = torch.full((C,), -1, dtype=torch.int64, device=DEV)
        self.trigger = torch.zeros(2, C, A, 3, dtype=torch.float64, device=DEV) if qbc else None
        self.rows, self.record_every, self.frame_slots, self.frame_v = rows, record_every, frame_slots, frame_v
        self.thermo = torch.zeros(rows, C, lib_.ANI_MD_THERMO, dtype=torch.float64, device=DEV)
        self.frames = torch.zeros(max(frame_slots, 1), 1 + frame_v, n, 3, dtype=torch.float64, device=DEV)
        self.partials = torch.zeros(C * self.nb * 2, dtype=torch.float64, device=DEV)
        self.coords = torch.zeros(C, A, 3, dtype=torch.float32, device=DEV)
        self.seed = 0x9E3779B97F4A7C15 ^ seed
        st = lib_.MDState()
        st.x, st.v, st.inv_mass, st.params = ptr(self.x), ptr(self.v), ptr(self.inv_t), ptr(self.par_t)
        st.counter, st.stop_step, st.trigger = ptr(self.counter), ptr(self.stop), ptr(self.trigger)
        st.thermo, st.frames, st.partials = ptr(self.thermo), ptr(self.frames), ptr(self.partials)
        st.seed, st.accel, st.kb = self.seed, mo.ACCEL, mo.KB
        st.n_conf, st.n_per_conf, st.integrator, st.thermo_rows = C, A, integrator, rows
        st.record_every, st.frame_slots, st.frame_velocities = record_every, frame_slots, int(frame_v)
        self.st = st
        self.init_cells, self.cell_mode, self.step_cell, self.table = cell_args(mode, self.cells)
        self.qbc = qbc
        self.qbc_t = dev(np.zeros(C)) if qbc else None
        self.fstd_t = torch.zeros(n, dtype=torch.float32, device=DEV) if qbc else None
        v0 = h(self.v)
        call(L().ani_b200_md_init(self.st_ref(), ptr(self.init_cells), self.cell_mode, int(zero_momentum),
                                  ptr(self.coords), None), "md_init")
        if zero_momentum:
            m = np.where(self.pad, 0.0, 1.0 / np.where(self.pad, 1.0, self.inv))
            p = (m[..., None] * v0).sum(1)
            ref = np.where(self.pad[..., None], v0, v0 - (p / m.sum(1)[:, None])[:, None])
            close(h(self.v), ref, "zero_momentum v")
            assert np.abs((m[..., None] * h(self.v)).sum(1)).max() <= 1e-12 * np.abs(m[..., None] * v0).sum((1, 2)).max()
        check_coords(h(self.coords), np.zeros((C, A, 3), np.float32), h(self.x), self.cells,
                     np.ones((C, A), dtype=bool))

    def st_ref(self):
        import ctypes
        return ctypes.byref(self.st)

    def buffers(self):
        out = [self.x, self.v, self.counter, self.stop, self.thermo, self.frames, self.coords]
        return out + ([self.trigger] if self.qbc else [])

    def launch(self, grad, energies, qbc=None, fstd=None):
        g = dev(grad.reshape(-1, 3), torch.float32)
        e = dev(energies)
        if self.qbc:
            self.qbc_t.copy_(dev(qbc))
            self.fstd_t.copy_(dev(fstd.reshape(-1), torch.float32))
        fn = L().ani_b200_md_step_cells if self.table else L().ani_b200_md_step
        call(fn(self.st_ref(), ptr(g), ptr(e), ptr(self.qbc_t), ptr(self.fstd_t), ptr(self.step_cell),
                ptr(self.coords), None), "md_step")


def md_oracle_step(md, t, x, v, stop, grad, energies, qbc=None, fstd=None):
    """One device MD step restated: returns x, v, the thermo row, the frame (x, v) or None, the conformers that stop."""
    C, A = md.C, md.A
    g = grad.astype(np.float64)
    frozen = stop >= 0
    dt = md.par[:, 0]
    v = v.copy()
    if t > 0:
        kicked = mo.kick(v, g, md.inv, dt[:, None])
        v[~frozen] = kicked[~frozen]
    ekin = mo.kinetic(v, md.inv)
    thermo = np.stack([np.full(C, float(t)), energies, ekin, 2.0 * ekin / (md.par[:, 5] * mo.KB)], 1)
    trip = np.zeros(C, dtype=bool)
    if qbc is not None:
        fm = np.where(md.pad, 0.0, fstd).max(1)
        trip = ~frozen & ((qbc > md.par[:, 3]) | (fm > md.par[:, 4]))
    frame = (x.copy(), v.copy()) if md.record_every and t % md.record_every == 0 else None
    x1, v1 = x.copy(), v.copy()
    for c in np.nonzero(~frozen & ~trip)[0]:
        noise = None
        if md.integrator == mo.LANGEVIN:
            flat = c * A + np.arange(A)
            noise = mo.normal(np.uint64(md.seed), t, flat[:, None], np.arange(3)[None])
        x1[c], v1[c] = mo.start(x[c], v[c], g[c], md.inv[c], dt[c], md.integrator, md.par[c, 1], md.par[c, 2], noise)
    return x1, v1, thermo, frame, trip


def md_compare_step(md, t, grad, energies, qbc=None, fstd=None):
    x, v, stop, c32 = h(md.x), h(md.v), h(md.stop), h(md.coords)
    assert h(md.counter)[0] == t
    x1, v1, thermo, frame, trip = md_oracle_step(md, t, x, v, stop, grad, energies, qbc, fstd)
    md.launch(grad, energies, qbc, fstd)
    xd, vd = h(md.x), h(md.v)
    close(xd, x1, f"x step {t}", scale=np.abs(x1).max())
    close(vd, v1, f"v step {t}", scale=np.abs(v1).max())
    frozen = (stop >= 0) | trip
    before = stop >= 0
    assert np.array_equal(xd[frozen], x[frozen]), "x of a stopped conformer"
    assert np.array_equal(vd[before], v[before]), "v of a conformer stopped before this step"
    assert np.array_equal(xd[md.pad], x[md.pad]) and np.array_equal(vd[md.pad], v[md.pad])
    row = h(md.thermo)[t % md.rows]
    assert (row[:, 0] == t).all() and np.array_equal(row[:, 1], energies)
    close(row[:, 2:], thermo[:, 2:], f"thermo step {t}")
    new_stop = np.where(trip, t, stop)
    assert np.array_equal(h(md.stop), new_stop)
    assert h(md.counter)[0] == t + 1
    if frame is not None:
        f = h(md.frames)[(t // md.record_every) % md.frame_slots]
        assert np.array_equal(f[0].reshape(x.shape), x)
        if md.frame_v:
            close(f[1].reshape(x.shape), frame[1], f"frame v step {t}")
    if trip.any():   # the trigger copy: x(t) and v(t) (after the final half kick), which the conformer keeps
        tr = h(md.trigger)
        for c in np.nonzero(trip)[0]:
            assert np.array_equal(tr[0, c], x[c]) and np.array_equal(tr[1, c], vd[c])
    moved = ~frozen[:, None] & ~md.pad
    check_coords(h(md.coords), c32, xd, md.cells, moved)
    return trip


MD_CASES = [  # n_conf, n_per_conf, integrator, cell mode
    (3, 1, mo.VERLET, "open"),
    (3, 255, mo.LANGEVIN, "shared"),
    (1, 256, mo.VERLET, "table"),
    (3, 257, mo.LANGEVIN, "table"),
    (3, 8193, mo.VERLET, "shared"),
    (3, 8193, mo.LANGEVIN, "table"),
    (1, 8193, mo.LANGEVIN, "open"),
]


@pytest.mark.parametrize("C, A, integrator, mode", MD_CASES)
def test_md_steps_against_the_oracle(C, A, integrator, mode):
    """Seven steps of ani_b200_md_step(_cells), each against md_oracle from the device's state before it: distinct dt,
    T and friction per conformer, the Langevin normals from the Philox restatement (not from md_noise), padding atoms,
    thermo_rows wrapping (3 rows, 7 steps), frames with record_every 2 in 2 slots (wrapping), 33-block conformers
    (n_per_conf 8193: the lane-strided second pass over the block partials); then the last four steps again from a
    saved state, bitwise."""
    md = MD(C, A, integrator, mode, seed=A + 7 * C + integrator, frame_v=(A % 2 == 1))
    rng = np.random.default_rng(5)
    grads, energies = [], []
    for t in range(7):
        if t == 3:
            saved = snapshot(md.buffers())
        g = md.field.grad(h(md.x))
        e = rng.normal(-40.0, 1.0, C)
        grads.append(g)
        energies.append(e)
        md_compare_step(md, t, g, e)
    first = bits(md.buffers())
    restore(md.buffers(), saved)
    for t in range(3, 7):
        md.launch(grads[t], energies[t])
    same_bits(bits(md.buffers()), first)


def test_md_zero_momentum_over_33_blocks():
    """ani_b200_md_init with zero_momentum at 8193 atoms per conformer (padding scattered and in the last block): v of
    the real atoms minus the total momentum over the total mass, and the coordinates of x."""
    MD(3, 8193, mo.VERLET, "shared", seed=3, zero_momentum=True)


def test_md_qbc_stop_in_block_33():
    """A QBC stop of conformer 1 by its largest force_stdev, which sits on atom 8192, alone in block 33: stop_step,
    the trigger copy of x(t), v(t), and a frozen conformer that stays bitwise constant while the others run; an
    energy-QBC stop of conformer 2 later.  Distinct thresholds per conformer."""
    md = MD(3, 8193, mo.LANGEVIN, "table", seed=11, qbc=True)
    assert not md.pad[:, -1].any()   # the stop atom (block 33) is real
    md.par[1, 4] = 0.5     # force-stdev threshold of conformer 1
    md.par[2, 3] = 0.25    # energy-QBC threshold of conformer 2
    md.par_t.copy_(dev(md.par))
    rng = np.random.default_rng(9)
    frozen_x = None
    for t in range(7):
        g = md.field.grad(h(md.x))
        fstd = rng.uniform(0.0, 0.4, (3, 8193)).astype(np.float32)
        qbc = np.array([0.0, 0.1, 0.5 if t >= 5 else 0.1])
        if t == 2:
            fstd[1, 8192] = 0.75
        trip = md_compare_step(md, t, g, rng.normal(size=3), qbc, fstd)
        if t == 2:
            assert trip.tolist() == [False, True, False]
            frozen_x, frozen_v = h(md.x)[1], h(md.v)[1]
        if t > 2:
            assert np.array_equal(h(md.x)[1], frozen_x) and np.array_equal(h(md.v)[1], frozen_v)
    assert h(md.stop).tolist() == [-1, 2, 5]


# ------------------------------------------------------------------------------------------------------------------
# 3. NPT: stochastic cell rescaling
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C, A, slots, per_conf", [(3, 257, 1, True), (1, 8193, 33, False), (3, 255, 64, True),
                                                   (3, 8193, 64, True)])
def test_npt_steps_against_the_oracle(C, A, slots, per_conf):
    """Six steps of ani_b200_md_step_npt, each against md_oracle + npt_oracle: mu from the restated cell noise
    (Philox counter (step, conformer, 3)), the virial slots (1, 33, 64: lane-strided past 32) summed, the master cell by
    step parity, cell_out, the {V, P_int} record, the frame cells, and the coordinates wrapped into the float32-rounded
    new cell; distinct T, dt, friction, P0, tau_p and beta_T per conformer."""
    lib_ = _lib()
    md = MD(C, A, mo.LANGEVIN, "table" if per_conf else "shared", seed=A + slots, frame_v=True)
    rng = np.random.default_rng(slots)
    stride = lib_.ANI_LATTICE_STRIDE
    master = torch.zeros(2, C, 9, dtype=torch.float64, device=DEV)
    master[0] = dev(md.cells.reshape(C, 9))
    md.v.mul_(0.1)   # a start near room temperature, so that mu stays near 1 over the steps
    bp = np.stack([no.BAR * np.array([1.0, 500.0, -200.0][:C]), np.array([100.0, 250.0, 60.0][:C]),
                   np.array([4.5e-5, 2.0e-5, 9e-6][:C]) / no.BAR], 1)
    bp_t = dev(bp)
    cell_out = torch.zeros(C, stride, dtype=torch.float32, device=DEV)
    virial = torch.zeros(C, slots, 9, dtype=torch.float64, device=DEV)
    record = torch.zeros(md.rows, C, lib_.ANI_MD_BARO, dtype=torch.float64, device=DEV)
    fcells = torch.zeros(md.frame_slots, C, 9, dtype=torch.float64, device=DEV)
    b = lib_.MDBarostat()
    b.master, b.params, b.cell_out, b.virial = ptr(master), ptr(bp_t), ptr(cell_out), ptr(virial)
    b.record, b.frame_cells, b.cell_stride, b.virial_slots = ptr(record), ptr(fcells), stride, slots
    import ctypes
    bufs = md.buffers() + [master, cell_out, record, fcells]
    grads, ws, es = [], [], []
    for t in range(6):
        if t == 3:
            saved = snapshot(bufs)
        x, v, c32 = h(md.x), h(md.v), h(md.coords)
        hc = h(master)[t % 2].reshape(C, 3, 3)
        other = h(master)[(t + 1) % 2]
        g = md.field.grad(x)
        W = rng.normal(0.0, 0.002, (C, slots, 9))
        virial.copy_(dev(W))
        e = rng.normal(size=C)
        grads.append(g)
        ws.append(W)
        es.append(e)
        x1, v1, thermo, frame, _ = md_oracle_step(md, t, x, v, -np.ones(C, np.int64), g, e)
        ekin = thermo[:, 2]
        xi = mo.normal(np.uint64(md.seed), t, np.arange(C), 3)
        Wt = W.sum(1).reshape(C, 3, 3)
        xs, vs, hn, vol, pint = no.cell_rescale(x1, v1, hc, ekin, Wt, md.par[:, 1], bp[:, 0], bp[:, 1], bp[:, 2],
                                                md.par[:, 0], xi)
        mov = ~md.pad[..., None]
        xs, vs = np.where(mov, xs, x1), np.where(mov, vs, v1)
        g_t = dev(g.reshape(-1, 3), torch.float32)
        call(L().ani_b200_md_step_npt(md.st_ref(), ctypes.byref(b), ptr(g_t), ptr(dev(e)), ptr(md.coords), None),
             "md_step_npt")
        xd = h(md.x)
        close(xd, xs, f"x step {t}")
        close(h(md.v), vs, f"v step {t}")
        m = h(master)
        assert np.array_equal(m[t % 2], hc.reshape(C, 9)), "the master slot of step t"
        close(m[(t + 1) % 2], hn.reshape(C, 9), f"master cell step {t}")
        assert not np.array_equal(m[(t + 1) % 2], other)
        out = h(cell_out)[:, :9]
        assert np.array_equal(out, m[(t + 1) % 2].astype(np.float32)), "cell_out"
        rec = h(record)[t % md.rows]
        close(rec[:, 0], vol, "V")
        close(rec[:, 1], pint, "P_int", scale=np.abs(pint).max() + np.abs(Wt).max() / vol.min())
        thm = h(md.thermo)[t % md.rows]
        close(thm[:, 2:], thermo[:, 2:], "thermo")
        if t % md.record_every == 0:
            fc = h(fcells)[(t // md.record_every) % md.frame_slots]
            assert np.array_equal(fc, hc.reshape(C, 9))
        check_coords(h(md.coords), c32, xd, out.astype(np.float64).reshape(C, 3, 3), ~md.pad)
    first = bits(bufs)
    restore(bufs, saved)
    for t in range(3, 6):
        virial.copy_(dev(ws[t]))
        g_t = dev(grads[t].reshape(-1, 3), torch.float32)
        call(L().ani_b200_md_step_npt(md.st_ref(), ctypes.byref(b), ptr(g_t), ptr(dev(es[t])), ptr(md.coords), None),
             "md_step_npt")
    same_bits(bits(bufs), first)


# ------------------------------------------------------------------------------------------------------------------
# 4. FIRE
# ------------------------------------------------------------------------------------------------------------------
class Opt:
    """One ani_opt_state on torch buffers (optimize.py's sizes)."""

    def __init__(self, C, A, mode, par, seed=1, rows=3, field_kw=None, fixed_every=5):
        lib_ = _lib()
        rng = np.random.default_rng(seed)
        self.C, self.A, self.mode = C, A, mode
        self.cells = cells_for(mode, C)
        x = positions(rng, C, A, self.cells)
        self.field = Field(x + rng.normal(0, 0.3, x.shape), rng, **(field_kw or {}))
        hot_last_atom(self.field, A)
        self.pad = padding(C, A, fixed_every)
        self.fs = np.where(self.pad, 0.0, fo.HARTREE_EV)
        self.par = par
        self.rows = rows
        self.x = dev(x)
        self.v = torch.zeros(C, A, 3, dtype=torch.float64, device=DEV)
        self.fs_t, self.par_t = dev(self.fs.reshape(-1)), dev(par)
        self.scalars = torch.zeros(2, C, lib_.ANI_OPT_SCALARS, dtype=torch.float64, device=DEV)
        self.counter = torch.zeros(2, dtype=torch.int64, device=DEV)
        self.conv = torch.full((C,), -1, dtype=torch.int64, device=DEV)
        self.record = torch.zeros(rows, C, lib_.ANI_OPT_RECORD, dtype=torch.float64, device=DEV)
        self.partials = torch.zeros(C * -(-A // lib_.ANI_MD_BLOCK) * 4, dtype=torch.float64, device=DEV)
        self.coords = torch.zeros(C, A, 3, dtype=torch.float32, device=DEV)
        st = lib_.OptState()
        st.x, st.v, st.force_scale, st.params = ptr(self.x), ptr(self.v), ptr(self.fs_t), ptr(self.par_t)
        st.scalars, st.counter, st.conv_step = ptr(self.scalars), ptr(self.counter), ptr(self.conv)
        st.record, st.partials = ptr(self.record), ptr(self.partials)
        st.n_conf, st.n_per_conf, st.record_rows = C, A, rows
        self.st = st
        self.init_cells, self.cell_mode, self.step_cell, self.table = cell_args(mode, self.cells)

    def ref(self):
        import ctypes
        return ctypes.byref(self.st)

    def init(self, reset=1):
        call(L().ani_b200_opt_init(self.ref(), ptr(self.init_cells), self.cell_mode, reset, ptr(self.coords), None),
             "opt_init")

    def buffers(self):
        return [self.x, self.v, self.scalars, self.counter, self.conv, self.record, self.coords]

    def launch(self, grad, energies):
        g, e = dev(grad.reshape(-1, 3), torch.float32), dev(energies)
        fn = L().ani_b200_opt_step_cells if self.table else L().ani_b200_opt_step
        call(fn(self.ref(), ptr(g), ptr(e), ptr(self.step_cell), ptr(self.coords), None), "opt_step")


FIRE_CASES = [(3, 1, "open"), (3, 255, "shared"), (1, 256, "table"), (3, 257, "table"), (3, 8193, "shared"),
              (3, 8193, "table")]


@pytest.mark.parametrize("C, A, mode", FIRE_CASES)
def test_fire_steps_against_the_oracle(C, A, mode):
    """24 steps of ani_b200_opt_step(_cells), each against fire_oracle from the device's state before it, with scripted
    gradients so that P > 0 holds for more than Nmin steps (dt grows to dtmax and a becomes a fa), P <= 0 resets
    (the gradient flips sign at steps 9 and 17), the maxstep clamp is on (conformer 0) and off (conformer 1),
    conformer 2 converges at step 0 and conformer 1 at step 20 (its gradient scaled by 1e-12), record_rows wraps (3
    rows), and opt_init with reset = 0 at step 12 keeps v, the scalars and the counter.  Distinct parameter rows per
    conformer (dt0, maxstep, dtmax, Nmin, finc, fdec, astart, fa, fmax).  The last 8 steps again from a saved state,
    bitwise."""
    par = np.stack([fo.params(0.0, dt=0.05, maxstep=1e-4, dtmax=0.09, n_min=2, finc=1.15, fdec=0.6, astart=0.2,
                              fa=0.95),
                    fo.params(1e-6, dt=0.02, maxstep=50.0, dtmax=0.04, n_min=3, finc=1.2, fdec=0.4, astart=0.15,
                              fa=0.9),
                    fo.params(1e9, dt=0.1, maxstep=0.2, dtmax=1.0)])[:C]
    opt = Opt(C, A, mode, par, seed=A + C)
    opt.init()
    sc = h(opt.scalars)[0]
    assert np.array_equal(sc, np.stack([par[:, 0], par[:, 6], np.zeros(C)], 1))
    check_coords(h(opt.coords), np.zeros((C, A, 3), np.float32), h(opt.x), opt.cells, np.ones((C, A), bool))
    seen = dict(grow=False, reset=False, clamp=False, free=False)
    grads = []
    for t in range(24):
        if t == 16:
            saved = snapshot(opt.buffers())
        if t == 12:
            before = [h(b) for b in (opt.v, opt.scalars, opt.counter, opt.x)]
            opt.init(reset=0)
            for a_, b_ in zip(before, (opt.v, opt.scalars, opt.counter, opt.x)):
                assert np.array_equal(a_, h(b_))
            check_coords(h(opt.coords), np.zeros((C, A, 3), np.float32), h(opt.x), opt.cells, np.ones((C, A), bool))
        x, v, sc, conv, c32 = h(opt.x), h(opt.v), h(opt.scalars)[t % 2], h(opt.conv), h(opt.coords)
        g = opt.field.grad(x)
        if t in (9, 17):
            g = -g
        if C > 1 and t == 20:
            g[1] *= np.float32(1e-12)
        grads.append(g)
        e = np.arange(C) + 0.5 * t
        ref = [fo.step(x[c], v[c], sc[c], g[c], opt.fs[c], par[c], t, conv[c] >= 0) for c in range(C)]
        opt.launch(g, e)
        xd, vd, scd = h(opt.x), h(opt.v), h(opt.scalars)[(t + 1) % 2]
        rec = h(opt.record)[t % opt.rows]
        for c, (x1, v1, s1, fmax, cv) in enumerate(ref):
            close(xd[c], x1, f"x step {t} conformer {c}", scale=np.abs(x1).max())
            close(vd[c], v1, f"v step {t} conformer {c}", scale=max(np.abs(v1).max(), 1e-300))
            close(scd[c], s1, f"scalars step {t} conformer {c}")
            assert rec[c, 0] == t and rec[c, 1] == e[c]
            close(rec[c, 2], fmax, "fmax")
            assert (h(opt.conv)[c] == t) == cv
            if conv[c] < 0 and not cv and t > 0:
                seen["grow"] |= s1[0] == par[c, 2] and s1[1] < par[c, 6]
                seen["reset"] |= s1[2] == 0 and sc[c][2] > 0
                dr = np.sqrt(((x1 - x[c]) ** 2).sum())   # the clamp makes the whole step exactly maxstep long
                seen["clamp" if abs(dr - par[c, 1]) <= 1e-9 * par[c, 1] else "free"] |= dr > 0
        frozen = conv >= 0
        assert np.array_equal(xd[frozen], x[frozen]) and np.array_equal(vd[frozen], v[frozen])
        written = ~(frozen | (h(opt.conv) == t))[:, None] & ~opt.pad
        check_coords(h(opt.coords), c32, xd, opt.cells, written)
    if C > 1:
        assert h(opt.conv).tolist() == [-1, 20, 0][:C]
        assert seen["grow"] and seen["reset"] and seen["clamp"] and seen["free"], seen
    first = bits(opt.buffers())
    restore(opt.buffers(), saved)
    for t in range(16, 24):
        opt.launch(grads[t], np.arange(C) + 0.5 * t)
    same_bits(bits(opt.buffers()), first)


# ------------------------------------------------------------------------------------------------------------------
# 5. variable-cell FIRE: the matrix exponential and its Frechet derivative
# ------------------------------------------------------------------------------------------------------------------
MP_DIGITS = 40


def expm3(a, e):
    """A float64 restatement of opt.cu's expm3: the Taylor series of [[a, e], [0, a]] / 2^s (13 terms, Horner), then
    s squarings, s = 0 for |a|_1 <= 1/4, else the exponent of 4 |a|_1.  Returns (expm(a), D_expm(a)[e]).

    The bar of the cell tests comes from this restatement against a 40-digit mpmath reference (20 random matrices per
    norm, error relative to the largest entry), measured on a CPU: <= 1e-15 up to |a|_1 = 1, 4e-15 at 7.5 and 3.4e-14
    at 40, for the exponential and the Frechet derivative alike.  The device runs the same operations in the same order
    (with fused multiply-adds), so 1e-12 of the largest entry leaves a margin of about 30 at |a|_1 = 40;
    ``test_expm3_restatement_error`` re-measures the restatement's side."""
    nrm = np.abs(a).sum(0).max()
    s = 0
    if nrm > 0.25:
        s = min(max(np.frexp(4.0 * nrm)[1], 0), 1100)
    sc = np.ldexp(1.0, -s)
    As, Es = a * sc, e * sc
    x, q = np.eye(3), np.zeros((3, 3))
    for n in range(13, 0, -1):
        t = As @ x
        q = (As @ q + Es @ x) / n
        x = t / n + np.eye(3)
    for _ in range(s):
        q = x @ q + q @ x
        x = x @ x
    return x, q


def mp_expm_frechet(a, e):
    """expm(a) and D_expm(a)[e] at MP_DIGITS digits: the blocks of expm([[a, e], [0, a]])."""
    with mpmath.workdps(MP_DIGITS):
        B = mpmath.zeros(6, 6)
        for i in range(3):
            for j in range(3):
                B[i, j] = B[i + 3, j + 3] = mpmath.mpf(float(a[i, j]))
                B[i, j + 3] = mpmath.mpf(float(e[i, j]))
        X = mpmath.expm(B)
        return (np.array([[float(X[i, j]) for j in range(3)] for i in range(3)]),
                np.array([[float(X[i, j + 3]) for j in range(3)] for i in range(3)]))


def log_norm_matrix(target, rng):
    """A symmetric 3 x 3 L with |L|_1 (the largest column sum of |L|, the norm expm3 tests) exactly ``target``: column
    0 is (target, 0, 0), the other two a randomly rotated diag(0.95, 0.9) target (column sums < target).  The spread
    of the eigenvalues is 0.1 target, so F = expm(L) stays well conditioned (cond 55 at 40) and G, which holds
    F^-T, carries no error of its own beyond float64 rounding."""
    th = rng.uniform(0.0, np.pi)
    rot = np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]])
    b = rot @ np.diag([0.95 * target, 0.9 * target]) @ rot.T
    b = 0.5 * (b + b.T)
    out = np.zeros((3, 3))
    out[0, 0] = target
    out[1:, 1:] = b
    assert np.abs(out).sum(0).max() == target
    return out


NORMS = [0.0, 0.1, 0.25, float(np.nextafter(0.25, 1.0)), 0.5, 1.0, 7.5, 40.0]


def test_expm3_restatement_error():
    """The restatement's error against mpmath at every norm of the cell tests stays within the table of expm3's
    docstring (times 3, for other random matrices)."""
    rng = np.random.default_rng(0)
    for target, bar in zip(NORMS, [1e-15] * 6 + [4e-15, 3.4e-14]):
        for _ in range(2):
            a, e = log_norm_matrix(target, rng), rng.standard_normal((3, 3))
            x, q = expm3(a, e)
            xr, qr = mp_expm_frechet(a, e)
            assert np.abs(x - xr).max() <= 3 * bar * np.abs(xr).max()
            assert np.abs(q - qr).max() <= 3 * bar * np.abs(qr).max()


@pytest.mark.parametrize("norm, projection", [(n, k % 3) for k, n in enumerate(NORMS)] + [(40.0, 0), (40.0, 2)])
def test_cell_fire_exponentials_against_mpmath(norm, projection):
    """ani_b200_opt_cell_step with the master slot {d, v_cell, F} written by the test, |d / c|_1 = ``norm`` (0 to 40:
    past 0.25 the scaling-and-squaring loop runs, its Frechet half included): cell_force against
    Phi = D_expm(L^T)[G] / c from mpmath at 40 digits, projected, the new master F against mpmath's expm of the new d,
    the FIRE step over the A + 3 rows against fire_oracle with that Phi, cell_out, the record and the coordinates;
    three conformers with distinct p0, c, FIRE rows and cells; two steps (the second from the device's own master).
    Bars: 1e-12 of the largest entry (see ``expm3``)."""
    lib_ = _lib()
    C = 3
    A = [1, 257, 8193][NORMS.index(norm) % 3]
    rng = np.random.default_rng(int(norm * 1000) + projection)
    par = np.stack([fo.params(0.0, dt=0.05, maxstep=0.05), fo.params(0.0, dt=0.02, maxstep=5.0, astart=0.2),
                    fo.params(0.0, dt=0.03, maxstep=0.3, fa=0.9)])
    opt = Opt(C, A, "open", par, seed=A, fixed_every=9)
    h0 = np.stack([TRICLINIC * (1.0 + 0.1 * c) for c in range(C)])
    cp = np.stack([np.array([0.01, 0.002, -0.005]) / mo.HARTREE_EV, np.array([1.0, 2.0, 0.5]),
                   np.full(3, mo.HARTREE_EV)], 1)   # {p0, c, unit} per conformer (c a power of two: d / c is L exactly)
    master = torch.zeros(2, C, lib_.ANI_OPT_CELL_MASTER, dtype=torch.float64, device=DEV)
    h0_t, cp_t = dev(h0.reshape(C, 9)), dev(cp)
    stride = 13
    cell_out = torch.zeros(C, stride, dtype=torch.float32, device=DEV)
    slots = 33
    virial = torch.zeros(C, slots, 9, dtype=torch.float64, device=DEV)
    cforce = torch.zeros(C, 9, dtype=torch.float64, device=DEV)
    crec = torch.zeros(opt.rows, C, lib_.ANI_OPT_CELL_RECORD, dtype=torch.float64, device=DEV)
    q = lib_.OptCell()
    q.master, q.h0, q.params, q.cell_out, q.virial = ptr(master), ptr(h0_t), ptr(cp_t), ptr(cell_out), ptr(virial)
    q.cell_force, q.record, q.cell_stride, q.virial_slots, q.projection = ptr(cforce), ptr(crec), stride, slots, \
        projection
    import ctypes
    qr = ctypes.byref(q)
    call(L().ani_b200_opt_cell_init(opt.ref(), qr, 1, ptr(opt.coords), None), "opt_cell_init")
    m0 = h(master)
    assert np.array_equal(m0[0, :, 18:], np.tile(np.eye(3).reshape(9), (C, 1)))
    # the test's master: d = c L, v_cell random, F = expm(L) (40 digits)
    m = np.zeros((C, 27))
    for c in range(C):
        Lm = log_norm_matrix(norm, rng)
        m[c, :9] = (cp[c, 1] * Lm).reshape(9)
        m[c, 9:18] = rng.normal(0.0, 0.01, 9)
        m[c, 18:] = mp_expm_frechet(m[c, :9].reshape(3, 3) / cp[c, 1], np.zeros((3, 3)))[0].reshape(9)
    master[0] = dev(m)
    for t in range(2):
        mt = h(master)[t % 2]
        u, v, sc, c32 = h(opt.x), h(opt.v), h(opt.scalars)[t % 2], h(opt.coords)
        g = opt.field.grad(u)   # (any function of the state: r = F u is ~1e18 A at |L|_1 = 40)
        W = rng.normal(0.0, 0.02, (C, slots, 9))
        virial.copy_(dev(W))
        e = rng.normal(size=C)
        gd, ed = dev(g.reshape(-1, 3), torch.float32), dev(e)
        call(L().ani_b200_opt_cell_step(opt.ref(), qr, ptr(gd), ptr(ed), ptr(opt.coords), None), "opt_cell_step")
        mn, phi_d, rec = h(master)[(t + 1) % 2], h(cforce), h(crec)[t % opt.rows]
        assert np.array_equal(h(master)[t % 2], mt)
        for c in range(C):
            d, vc, F = (mt[c, 9 * k:9 * k + 9].reshape(3, 3) for k in range(3))
            Lt = d.T / cp[c, 1]
            hh = h0[c] @ F.T
            vol = abs(np.linalg.det(hh))
            Wc = W[c].sum(0).reshape(3, 3)
            G = -(Wc + cp[c, 0] * vol * np.eye(3)) @ np.linalg.inv(F).T * cp[c, 2]
            phi = mp_expm_frechet(Lt, G)[1] / cp[c, 1]
            close(phi_d[c], cfo.project(phi, projection).reshape(9), f"cell_force |L|_1 {norm} conformer {c}",
                  scale=np.abs(phi).max())
            phi = phi_d[c].reshape(3, 3)
            close(rec[c], [vol, -np.trace(Wc) / (3.0 * vol), e[c] + cp[c, 0] * vol], "cell record")
            f = -g[c].astype(np.float64) * opt.fs[c][:, None]
            rows = np.vstack([u[c], d])
            vv = np.vstack([v[c], vc])
            x1, v1, s1, fmax, cv = fo.step(rows, vv, sc[c], -np.vstack([f @ F, phi]), np.ones(len(rows)), par[c], t)
            close(h(opt.x)[c], x1[:-3], f"u step {t}", scale=np.abs(x1[:-3]).max())
            close(mn[c, :9], x1[-3:].reshape(9), f"d step {t}", scale=np.abs(x1[-3:]).max())
            close(mn[c, 9:18], v1[-3:].reshape(9), f"v_cell step {t}", scale=np.abs(v1).max())
            close(h(opt.scalars)[(t + 1) % 2][c], s1, "scalars")
            Fn = mp_expm_frechet(mn[c, :9].reshape(3, 3) / cp[c, 1], np.zeros((3, 3)))[0]
            close(mn[c, 18:], Fn.reshape(9), f"F(t+1) |L|_1 {norm}", scale=np.abs(Fn).max())
            hn = h0[c] @ mn[c, 18:].reshape(3, 3).T
            out = h(cell_out)[c, :9].astype(np.float64)
            assert (np.abs(out - hn.reshape(9)) <= np.spacing(np.abs(hn.reshape(9)).astype(np.float32))).all()
        rn = np.einsum("cij,caj->cai", mn[:, 18:].reshape(C, 3, 3), h(opt.x))
        check_coords(h(opt.coords), c32, rn, h(cell_out)[:, :9].astype(np.float64).reshape(C, 3, 3), ~opt.pad)


# ------------------------------------------------------------------------------------------------------------------
# 6. L-BFGS
# ------------------------------------------------------------------------------------------------------------------
class Lbfgs:
    """One ani_lbfgs_state on torch buffers (optimize.py's sizes; M = memory + 1 ring slots)."""

    def __init__(self, C, A, memory, mode, par, seed=1, rows=3):
        lib_ = _lib()
        rng = np.random.default_rng(seed)
        self.C, self.A, self.mem, self.M, self.mode, self.par, self.rows = C, A, memory, memory + 1, mode, par, rows
        self.cells = cells_for(mode, C)
        x = positions(rng, C, A, self.cells)
        self.field = Field(x + rng.normal(0, 0.3, x.shape), rng, lam=0.08)
        hot_last_atom(self.field, A)
        self.pad = padding(C, A, 6, block=_lib().ANI_LBFGS_TILE)
        self.fs = np.where(self.pad, 0.0, fo.HARTREE_EV)
        z = lambda *s: torch.zeros(*s, dtype=torch.float64, device=DEV)   # noqa: E731
        M = self.M
        self.x, self.x_prev, self.g_prev, self.p = dev(x), z(C, A, 3), z(C, A, 3), z(C, A, 3)
        self.s, self.y, self.sy, self.yy = z(C, M, A, 3), z(C, M, A, 3), z(C, M, M), z(C, M, M)
        self.coef = z(C, 2, memory)
        self.iter = torch.zeros(C, 2, dtype=torch.int64, device=DEV)
        self.fs_t, self.par_t = dev(self.fs.reshape(-1)), dev(par)
        self.counter = torch.zeros(2, dtype=torch.int64, device=DEV)
        self.conv = torch.full((C,), -1, dtype=torch.int64, device=DEV)
        self.record = z(rows, C, lib_.ANI_LBFGS_RECORD)
        self.partials = z(lib_.lbfgs_partials(C, A, memory))
        self.coords = torch.zeros(C, A, 3, dtype=torch.float32, device=DEV)
        st = lib_.LbfgsState()
        for k in ("x", "x_prev", "g_prev", "s", "y", "sy", "yy", "coef", "p", "iter", "counter", "record", "partials"):
            setattr(st, k, ptr(getattr(self, k)))
        st.force_scale, st.params, st.conv_step = ptr(self.fs_t), ptr(self.par_t), ptr(self.conv)
        st.n_conf, st.n_per_conf, st.memory, st.record_rows = C, A, memory, rows
        self.st = st
        self.init_cells, self.cell_mode, self.step_cell, self.table = cell_args(mode, self.cells)
        import ctypes
        self.ref = ctypes.byref(self.st)
        call(L().ani_b200_lbfgs_init(self.ref, ptr(self.init_cells), self.cell_mode, 1, ptr(self.coords), None),
             "lbfgs_init")
        assert np.array_equal(h(self.x_prev), x) and not h(self.iter).any()

    def buffers(self):
        return [self.x, self.x_prev, self.g_prev, self.s, self.y, self.sy, self.yy, self.coef, self.p, self.iter,
                self.counter, self.conv, self.record, self.coords]

    def launch(self, grad, energies):
        g, e = dev(grad.reshape(-1, 3), torch.float32), dev(energies)
        fn = L().ani_b200_lbfgs_step_cells if self.table else L().ani_b200_lbfgs_step
        call(fn(self.ref, ptr(g), ptr(e), ptr(self.step_cell), ptr(self.coords), None), "lbfgs_step")

    def live(self, S, Y, it, c):
        """The live pairs of conformer c in chronological order: pair j in slot (head - L + j) % M."""
        head = int(it[c, 1])
        n = min(self.mem, head)
        slots = [(head - n + j) % self.M for j in range(n)]
        return slots, [S[c, k].reshape(-1) for k in slots], [Y[c, k].reshape(-1) for k in slots]


def lbfgs_compare_step(lb, t, g, e):
    C, mem = lb.C, lb.mem
    x, xp, gp, S, Y, it, conv = (h(b) for b in (lb.x, lb.x_prev, lb.g_prev, lb.s, lb.y, lb.iter, lb.conv))
    c32 = h(lb.coords)
    states, before = [], []
    for c in range(C):
        st = lo.State(mem)
        st.iteration = int(it[c, 0])
        slots, st.s, st.y = lb.live(S, Y, it, c)
        st.rho = [1.0 / float(np.dot(yy, ss)) for ss, yy in zip(st.s, st.y)]
        st.r0, st.g0 = xp[c], gp[c]
        states.append(st)
        before.append({k: (S[c, k].copy(), Y[c, k].copy()) for k in slots})
    ref = [lo.step(states[c], x[c], g[c], lb.fs[c], lb.par[c], conv[c] >= 0) for c in range(C)]
    lb.launch(g, e)
    xd, S2, Y2, it2, conv2, SY, YY, coef, p = (h(b) for b in (lb.x, lb.s, lb.y, lb.iter, lb.conv, lb.sy, lb.yy,
                                                              lb.coef, lb.p))
    rec = h(lb.record)[t % lb.rows]
    skipped = []
    for c, (x1, fmax, cv) in enumerate(ref):
        st = states[c]
        assert rec[c, 0] == t and rec[c, 1] == e[c]
        close(rec[c, 2], fmax, "fmax")
        assert (conv2[c] == t) == cv and (conv2[c] >= 0) == (conv[c] >= 0 or cv)
        if conv[c] >= 0 or cv:   # frozen: nothing of the conformer changes
            assert np.array_equal(xd[c], x[c]) and np.array_equal(it2[c], it[c])
            for k, (s0, y0) in before[c].items():
                assert np.array_equal(S2[c, k], s0) and np.array_equal(Y2[c, k], y0)
            continue
        # the pairs: the head advances exactly when the oracle appended one, and the live ring is the oracle's history
        nhead = int(it2[c, 1])
        assert it2[c, 0] == it[c, 0] + 1 and nhead - int(it[c, 1]) in (0, 1)
        slots, S_live, Y_live = lb.live(S2, Y2, it2, c)
        assert len(S_live) == len(st.s)
        for j in range(len(st.s)):
            assert np.array_equal(S_live[j], st.s[j]) and np.array_equal(Y_live[j], st.y[j]), (t, c, j)
        if nhead == int(it[c, 1]) and int(it[c, 0]) >= 1:
            skipped.append(c)
            for k, (s0, y0) in before[c].items():   # a skipped pair overwrites no live slot
                assert np.array_equal(S2[c, k], s0) and np.array_equal(Y2[c, k], y0)
        # SY (upper triangle, chronological) and YY against float64 products of the ring
        n = len(S_live)
        if n:
            Sm, Ym = np.array(S_live), np.array(Y_live)
            sy_ref, yy_ref = Sm @ Ym.T, Ym @ Ym.T
            nrm = np.sqrt((Sm * Sm).sum(1))[:, None] * np.sqrt((Ym * Ym).sum(1))[None]
            nyy = np.sqrt((Ym * Ym).sum(1))[:, None] * np.sqrt((Ym * Ym).sum(1))[None]
            sy_d, yy_d = SY[c][np.ix_(slots, slots)], YY[c][np.ix_(slots, slots)]
            iu = np.triu_indices(n)
            assert (np.abs(sy_d - sy_ref)[iu] <= REL * nrm[iu]).all(), "SY"
            assert (np.abs(yy_d - yy_ref) <= REL * nyy).all(), "YY"
        # the direction: the device's p against the two-loop recursion and the compact form, the bar 10 times their
        # spread, with a floor of the rounding of the device's sum p = -(H0 g + sum_j a_j s_j + b_j y_j): 2 (L + 4) eps
        # (2 L products and sums, and H0 (g force_scale)) times the largest sum of its terms' magnitudes (p cancels
        # terms far larger than itself at L = 128); then p
        # against the device's own coefficients
        gc = g[c].astype(np.float64) * lb.fs[c][:, None]
        h0 = lb.par[c, 2]
        p2 = lo.two_loop(st.s, st.y, st.rho, gc, h0)
        pc = lo.compact_direction(S_live, Y_live, gc, h0) if n else -h0 * gc.reshape(-1)
        terms = h0 * np.abs(gc.reshape(-1))
        if n:
            terms = terms + np.abs(np.array(S_live)).T @ np.abs(coef[c, 0, :n]) + \
                np.abs(np.array(Y_live)).T @ np.abs(coef[c, 1, :n])
        floor = 2.0 * (n + 4) * np.finfo(np.float64).eps * terms.max()
        bar = max(10.0 * np.abs(p2 - pc).max(), floor, 1e-15 * np.abs(pc).max())
        assert np.abs(p[c].reshape(-1) - pc).max() <= bar, (t, c, np.abs(p[c].reshape(-1) - pc).max(), bar)
        if n:
            a_d, b_d = coef[c, 0, :n], coef[c, 1, :n]
            assert np.abs(-(h0 * gc.reshape(-1) + Sm.T @ a_d + Ym.T @ b_d) - p[c].reshape(-1)).max() <= \
                1e-13 * (h0 * np.abs(gc).max() + np.abs(Sm.T * a_d).sum(1).max() + np.abs(Ym.T * b_d).sum(1).max())
            # a and b by their residuals in the device's own R = triu(SY) and YY: r = -b / H0 solves R r = u and a
            # solves R^T a = t = (D + H0 Y^T Y) r - H0 w.  A triangular substitution is componentwise backward stable,
            # |T x - rhs| <= L eps |T| |x|, and u, w are sums over 3 n_per_conf products, so each residual is bounded
            # by gam (|T| |x| + the absolute sums of its right-hand side), gam = 2 (L + 3 n_per_conf) eps.  Unlike a
            # forward error, this bound does not grow with the condition of R (poor at L = 128); a wrong
            # coefficient leaves a residual of the size of the right-hand side.
            gam = 2.0 * (n + 3 * lb.A) * np.finfo(np.float64).eps
            R = np.triu(sy_d)
            ga = np.abs(gc.reshape(-1))
            u, w = Sm @ gc.reshape(-1), Ym @ gc.reshape(-1)
            r_d = -b_d / h0
            res = np.abs(R @ r_d - u)
            assert (res <= gam * (np.abs(R) @ np.abs(r_d) + np.abs(Sm) @ ga)).all(), ("b", t, c)
            K = np.diag(np.diag(R)) + h0 * yy_d
            t_d = K @ r_d - h0 * w
            res = np.abs(R.T @ a_d - t_d)
            assert (res <= gam * (np.abs(R.T) @ np.abs(a_d) + np.abs(K) @ np.abs(r_d) + h0 * np.abs(Ym) @ ga)).all(), \
                ("a", t, c)
        longest = np.sqrt((p[c] ** 2).sum(1)).max()
        scale = lb.par[c, 0] / longest if longest >= lb.par[c, 0] else 1.0
        close(xd[c], x1, f"x step {t} conformer {c}", scale=np.abs(x1).max(),
              rel=REL + 2.0 * bar * lb.par[c, 1] / np.abs(x1).max())   # (the direction's error, and its clamp's)
        close(xd[c], x[c] + p[c] * scale * lb.par[c, 1], "x from the device's own direction", scale=np.abs(x1).max())
    written = (conv2 < 0)[:, None] & ~lb.pad
    check_coords(h(lb.coords), c32, xd, lb.cells, written)
    return skipped


LBFGS_CASES = [  # memory, n_conf, n_per_conf, cell mode
    (1, 3, 1, "open"),
    (7, 3, 31, "shared"),
    (8, 1, 32, "table"),
    (9, 3, 33, "table"),
    (32, 3, 1025, "open"),
    (33, 3, 33, "shared"),
    (128, 3, 1025, "table"),
]


@pytest.mark.parametrize("memory, C, A, mode", LBFGS_CASES)
def test_lbfgs_steps_against_the_oracle(memory, C, A, mode):
    """memory + 12 steps of ani_b200_lbfgs_step(_cells), each against lbfgs_oracle on lo.State rebuilt from the ring
    (pair j in slot (head - L + j) % (memory + 1)): x, the record, k, head, the live ring pair by pair, SY and YY
    against float64 products of the ring, the coefficients against the compact form, and the direction against both
    of the oracle's forms.  The ring fills and wraps (full-ring drop, spare slot, one-column SY / YY update); the same
    float32 gradient fed twice (y = 0, the pair skipped) at step 1 and, with the ring full, at step memory + 4;
    conformer 0 clamped (maxstep 0.02, damping 0.7), conformer 1 not (maxstep 10, damping 1.3, converging at step
    memory + 8), conformer 2 converged at step 0.  Paths: rows >= 8 (memory >= 8: dot-sweep groups blockIdx.y >= 1),
    L > 8 (the direction sweep over eight warps), L > 32 (lane-strided triangular solves), rows = 129 (memory 128:
    the row totals past LB_SOLVE), 33 tiles (n_per_conf 1025: lane-strided fmax / pmax partials).  The last 6 steps
    again from a saved state, bitwise."""
    par = np.stack([lo.params(0.0, maxstep=0.02, damping=0.7, alpha=50.0),
                    lo.params(1e-6, maxstep=10.0, damping=1.3, alpha=90.0),
                    lo.params(1e9)])[:C]
    lb = Lbfgs(C, A, memory, mode, par, seed=memory + A)
    steps = memory + 12
    skip = (1, memory + 4)
    grads, prev = [], None
    skipped_at = {}
    for t in range(steps):
        if t == steps - 6:
            saved = snapshot(lb.buffers())
        g = prev if t in skip else lb.field.grad(h(lb.x))
        if C > 1 and t == memory + 8:
            g = g.copy()
            g[1] *= np.float32(1e-12)
        grads.append(g)
        e = np.arange(C) - 0.25 * t
        skipped_at[t] = lbfgs_compare_step(lb, t, g, e)
        prev = g
    for t in skip:
        assert 0 in skipped_at[t], (t, skipped_at[t])
    assert int(h(lb.iter)[0, 1]) == steps - 1 - len(skip) and int(h(lb.iter)[0, 1]) > memory + 1
    if C > 1:
        assert h(lb.conv).tolist() == [-1, memory + 8, 0][:C]
        assert int(h(lb.iter)[1, 0]) == memory + 8 and int(h(lb.iter)[2, 0]) == 0
    first = bits(lb.buffers())
    restore(lb.buffers(), saved)
    for t in range(steps - 6, steps):
        lb.launch(grads[t], np.arange(C) - 0.25 * t)
    same_bits(bits(lb.buffers()), first)


# ------------------------------------------------------------------------------------------------------------------
# 7. 65535 conformers of one atom: the grid.y limit
# ------------------------------------------------------------------------------------------------------------------
def test_65535_conformers_one_step():
    """One step of MD (Verlet), FIRE and L-BFGS with n_conf = 65535 (the grid.y limit the entry points accept), one atom
    each and a distinct parameter row per conformer, against the oracles' formulas vectorised over the conformers."""
    C = 65535
    rng = np.random.default_rng(1)
    x = rng.normal(0.0, 3.0, (C, 1, 3))
    g = rng.normal(0.0, 0.05, (C, 1, 3)).astype(np.float32)
    e = rng.normal(size=C)
    # MD
    md = MD(C, 1, mo.VERLET, "open", seed=2)
    md.x.copy_(dev(x))
    v = h(md.v)
    md.launch(g, e)
    dt = md.par[:, 0][:, None, None]
    v1 = v - 0.5 * dt * mo.ACCEL * md.inv[..., None] * g
    close(h(md.x), x + dt * v1, "MD x")
    close(h(md.v), v1, "MD v")
    th = h(md.thermo)[0]
    close(th[:, 2], mo.kinetic(v, md.inv), "MD E_kin")
    assert np.array_equal(h(md.coords), h(md.x).astype(np.float32))
    # FIRE at step 0: v' = dt f, x + dt v' min(1, maxstep / |dr|)
    par = np.stack([fo.params(0.0, dt=0.05 + 0.001 * (c % 50), maxstep=0.01 + 0.02 * (c % 3)) for c in range(C)])
    opt = Opt(C, 1, "open", par, seed=3)
    opt.x.copy_(dev(x))
    opt.init()
    opt.launch(g, e)
    f = -g.astype(np.float64) * fo.HARTREE_EV
    dtc = par[:, 0][:, None, None]
    vn = dtc * f
    dr = dtc[:, 0, 0] * np.sqrt((vn ** 2).sum((1, 2)))
    sc = np.where(dr > par[:, 1], par[:, 1] / dr, 1.0)[:, None, None]
    close(h(opt.v), vn, "FIRE v")
    close(h(opt.x), x + dtc * sc * vn, "FIRE x")
    close(h(opt.record)[0][:, 2], np.sqrt((f ** 2).sum((1, 2))), "FIRE fmax")
    # L-BFGS at step 0: p = -H0 g, clamped to maxstep, damped
    lpar = np.stack([lo.params(0.0, maxstep=0.01 + 0.01 * (c % 4), damping=0.5 + 0.25 * (c % 3),
                               alpha=40.0 + c % 7) for c in range(C)])
    lb = Lbfgs(C, 1, 1, "open", lpar, seed=4)
    lb.x.copy_(dev(x))
    call(L().ani_b200_lbfgs_init(lb.ref, None, 0, 1, ptr(lb.coords), None), "lbfgs_init")
    lb.launch(g, e)
    gg = g.astype(np.float64) * fo.HARTREE_EV
    p = -lpar[:, 2][:, None, None] * gg
    ln = np.sqrt((p ** 2).sum((1, 2)))
    sc = np.where(ln >= lpar[:, 0], lpar[:, 0] / ln, 1.0)[:, None, None]
    close(h(lb.x), x + p * sc * lpar[:, 1][:, None, None], "L-BFGS x")
    assert (h(lb.iter)[:, 0] == 1).all() and (h(lb.iter)[:, 1] == 0).all()


def test_65535_conformers_npt_and_cell_fire():
    """One step of ani_b200_md_step_npt and of ani_b200_opt_cell_step with n_conf = 65535, one atom each and distinct
    parameter rows (dt, P0, tau_p, beta_T; the FIRE row, p0, c and h0), against md_oracle / npt_oracle and the cell-FIRE
    formulas vectorised over the conformers.  The cell step starts from F = I, where Phi = G / c."""
    import ctypes
    from scipy.linalg import expm
    lib_ = _lib()
    C = 65535
    rng = np.random.default_rng(2)
    g = rng.normal(0.0, 0.05, (C, 1, 3)).astype(np.float32)
    e = rng.normal(size=C)
    # NPT (Langevin): B A O A of step 0 (no final half kick at t = 0), then the cell rescaling
    md = MD(C, 1, mo.LANGEVIN, "shared", seed=5)
    md.v.mul_(0.1)
    x, v = h(md.x), h(md.v)
    master = torch.zeros(2, C, 9, dtype=torch.float64, device=DEV)
    master[0] = dev(md.cells.reshape(C, 9))
    k = np.arange(C)
    bp = np.stack([no.BAR * (1.0 + (k % 5)), 100.0 + (k % 7), 4.5e-5 / no.BAR * (1.0 + 0.1 * (k % 3))], 1)
    bp_t = dev(bp)
    cell_out = torch.zeros(C, 9, dtype=torch.float32, device=DEV)
    W = rng.normal(0.0, 0.002, (C, 1, 9))
    virial = dev(W)
    record = torch.zeros(md.rows, C, lib_.ANI_MD_BARO, dtype=torch.float64, device=DEV)
    fcells = torch.zeros(md.frame_slots, C, 9, dtype=torch.float64, device=DEV)
    b = lib_.MDBarostat()
    b.master, b.params, b.cell_out, b.virial = ptr(master), ptr(bp_t), ptr(cell_out), ptr(virial)
    b.record, b.frame_cells, b.cell_stride, b.virial_slots = ptr(record), ptr(fcells), 9, 1
    gd = dev(g.reshape(-1, 3), torch.float32)
    call(L().ani_b200_md_step_npt(md.st_ref(), ctypes.byref(b), ptr(gd), ptr(dev(e)), ptr(md.coords), None),
         "md_step_npt")
    dt, T, fr = (md.par[:, i][:, None, None] for i in range(3))
    im = md.inv[..., None]
    v1 = v - 0.5 * dt * mo.ACCEL * im * g.astype(np.float64)
    x1 = x + 0.5 * dt * v1
    cf = np.exp(-fr * dt)
    xi = mo.normal(np.uint64(md.seed), 0, k[:, None, None], np.arange(3)[None, None])
    v1 = cf * v1 + np.sqrt((1.0 - cf * cf) * mo.KB * T * mo.ACCEL * im) * xi
    x1 = x1 + 0.5 * dt * v1
    hc = md.cells
    xs, vs, hn, vol, pint = no.cell_rescale(x1, v1, hc, mo.kinetic(v, md.inv), W.sum(1).reshape(C, 3, 3),
                                            md.par[:, 1], bp[:, 0], bp[:, 1], bp[:, 2], md.par[:, 0],
                                            mo.normal(np.uint64(md.seed), 0, k, 3))
    close(h(md.x), xs, "NPT x")
    close(h(md.v), vs, "NPT v")
    close(h(master)[1], hn.reshape(C, 9), "NPT master cell")
    assert np.array_equal(h(cell_out), h(master)[1].astype(np.float32))
    close(h(record)[0][:, 0], vol, "NPT V")
    # cell FIRE from F = I, d = 0, v = 0
    par = np.stack([fo.params(0.0, dt=0.02 + 0.001 * (i % 30), maxstep=0.002 + 0.05 * (i % 2)) for i in range(C)])
    opt = Opt(C, 1, "open", par, seed=6)
    u = h(opt.x)
    h0 = TRICLINIC[None] * (1.0 + 0.01 * (k % 10))[:, None, None]
    cp = np.stack([0.001 * (k % 4) / mo.HARTREE_EV, 1.0 + 0.5 * (k % 3), np.full(C, mo.HARTREE_EV)], 1)
    mst = torch.zeros(2, C, lib_.ANI_OPT_CELL_MASTER, dtype=torch.float64, device=DEV)
    h0_t, cp_t = dev(h0.reshape(C, 9)), dev(cp)
    cout = torch.zeros(C, 9, dtype=torch.float32, device=DEV)
    Wc = rng.normal(0.0, 0.01, (C, 1, 9))
    vir = dev(Wc)
    cforce = torch.zeros(C, 9, dtype=torch.float64, device=DEV)
    crec = torch.zeros(opt.rows, C, lib_.ANI_OPT_CELL_RECORD, dtype=torch.float64, device=DEV)
    q = lib_.OptCell()
    q.master, q.h0, q.params, q.cell_out, q.virial = ptr(mst), ptr(h0_t), ptr(cp_t), ptr(cout), ptr(vir)
    q.cell_force, q.record, q.cell_stride, q.virial_slots, q.projection = ptr(cforce), ptr(crec), 9, 1, 0
    call(L().ani_b200_opt_cell_init(opt.ref(), ctypes.byref(q), 1, ptr(opt.coords), None), "opt_cell_init")
    call(L().ani_b200_opt_cell_step(opt.ref(), ctypes.byref(q), ptr(gd), ptr(dev(e)), ptr(opt.coords), None),
         "opt_cell_step")
    vol = np.abs(np.linalg.det(h0))
    G = -(Wc.reshape(C, 3, 3) + cp[:, 0, None, None] * vol[:, None, None] * np.eye(3)) * cp[:, 2, None, None]
    phi = G / cp[:, 1, None, None]
    close(h(cforce), phi.reshape(C, 9), "cell force at F = I")
    f = -g.astype(np.float64) * fo.HARTREE_EV
    rows = np.concatenate([f, phi], 1)   # (C, 4, 3): the atom row and the three cell rows
    dtc = par[:, 0][:, None, None]
    vn = dtc * rows
    dr = dtc[:, 0, 0] * np.sqrt((vn ** 2).sum((1, 2)))
    st = dtc * np.where(dr > par[:, 1], par[:, 1] / dr, 1.0)[:, None, None]
    m1 = h(mst)[1]
    close(h(opt.x), u + st * vn[:, :1], "cell FIRE u")
    close(m1[:, :9], (st * vn[:, 1:]).reshape(C, 9), "cell FIRE d")
    close(m1[:, 9:18], vn[:, 1:].reshape(C, 9), "cell FIRE v_cell")
    Fn = expm(m1[:, :9].reshape(C, 3, 3) / cp[:, 1, None, None])
    close(m1[:, 18:], Fn.reshape(C, 9), "cell FIRE F(t+1)")
    hn = np.einsum("cij,ckj->cik", h0, m1[:, 18:].reshape(C, 3, 3))
    out = h(cout).astype(np.float64)
    assert (np.abs(out - hn.reshape(C, 9)) <= 0.5 * np.spacing(np.abs(hn.reshape(C, 9)).astype(np.float32))
            + 1e-15 * np.abs(hn).max()).all()
    close(h(crec)[0][:, 0], vol, "cell FIRE V")
