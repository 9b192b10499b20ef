"""The float64 L-BFGS oracle (oracle/lbfgs_oracle.py): ASE's two-loop recursion against the compact representation the
device uses, the rules it restates (first step, clamp, damping, history), a problem with a known answer, and the
L-BFGS entry points of the C-ABI and the Python driver without a GPU (struct layout, argument checks that return before
any CUDA call)."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import oracle.fire_oracle as fo
import oracle.lbfgs_oracle as lo
from helpers import ROOT


def _history(rng, L, n, negative=0):
    """L random pairs in n dimensions with mostly positive curvature; the first ``negative`` have y.s < 0."""
    S, Y = [], []
    for i in range(L):
        s = rng.standard_normal(n)
        y = s * rng.uniform(0.5, 2.0) + 0.3 * rng.standard_normal(n)
        if i < negative:
            y = -y
        S.append(s)
        Y.append(y)
    return S, Y


def _inverse_hessian(S, Y, H0, n):
    rho = [1.0 / np.dot(y, s) for s, y in zip(S, Y)]
    return np.stack([-lo.two_loop(S, Y, rho, e, H0) for e in np.eye(n)], 1)


def test_two_loop_and_compact_forms_agree():
    """Random histories of L = 1..memory pairs (some with y.s < 0) and a ring that has wrapped: both forms give the same
    p to 1e-12 relative."""
    rng = np.random.default_rng(11)
    worst = 0.0
    for trial in range(200):
        n = int(rng.integers(6, 61))
        L = int(rng.integers(1, 20))
        S, Y = _history(rng, L, n, negative=int(rng.integers(0, 3)) if trial % 3 == 0 else 0)
        S, Y = [s for s, y in zip(S, Y) if np.dot(s, y) != 0], [y for s, y in zip(S, Y) if np.dot(s, y) != 0]
        g = rng.standard_normal(n)
        H0 = 1.0 / rng.uniform(10.0, 100.0)
        rho = [1.0 / np.dot(y, s) for s, y in zip(S, Y)]
        a, b = lo.two_loop(S, Y, rho, g, H0), lo.compact_direction(np.array(S), np.array(Y), g, H0)
        worst = max(worst, np.abs(a - b).max() / np.abs(a).max())
    assert worst <= 1e-12, worst
    # a wrapped history: memory 5 after 13 updates keeps the last 5 pairs in order
    st = lo.State(memory=5)
    x, g = rng.standard_normal((4, 3)), rng.standard_normal((4, 3))
    for _ in range(13):
        st.r0, st.g0, st.iteration = x, g, st.iteration + 1
        x = x + 0.1 * rng.standard_normal((4, 3))
        g = g + 0.3 * (x - st.r0) + 0.01 * rng.standard_normal((4, 3))
        lo.update(st, x, g)
    assert len(st.s) == 5
    a = lo.two_loop(st.s, st.y, st.rho, g, 1 / 70.0)
    b = lo.compact_direction(np.array(st.s), np.array(st.y), g, 1 / 70.0)
    assert np.abs(a - b).max() <= 1e-12 * np.abs(a).max()


def test_secant_condition_and_positive_definite():
    rng = np.random.default_rng(5)
    for L in (1, 3, 8):
        n = 12
        S, Y = _history(rng, L, n)
        assert all(np.dot(s, y) > 0 for s, y in zip(S, Y))
        H = _inverse_hessian(S, Y, 1 / 70.0, n)
        assert np.abs(H @ Y[-1] - S[-1]).max() <= 1e-12 * np.abs(S[-1]).max()
        assert np.abs(H - H.T).max() <= 1e-12 * np.abs(H).max()
        assert np.linalg.eigvalsh(0.5 * (H + H.T)).min() > 0
    # the compact form satisfies the same secant condition, also with y.s < 0 pairs in the history
    S, Y = _history(rng, 6, 12, negative=2)
    Hc = np.stack([-lo.compact_direction(np.array(S), np.array(Y), e, 1 / 70.0) for e in np.eye(12)], 1)
    assert np.abs(Hc @ Y[-1] - S[-1]).max() <= 1e-12 * np.abs(S[-1]).max()


def test_first_step_clamp_and_damping():
    """The first step is f / alpha; the clamp scales the whole step by maxstep over the LONGEST ATOM step, and applies
    from max_i |p_i| >= maxstep on; damping multiplies after the clamp."""
    rng = np.random.default_rng(2)
    x = rng.standard_normal((5, 3))
    g = rng.standard_normal((5, 3))
    big = lo.params(0.0, maxstep=100.0, alpha=70.0)
    x1, _, _ = lo.step(lo.State(), x, g, np.ones(5), big)
    assert np.allclose(x1 - x, -g / 70.0, rtol=1e-14, atol=1e-16)
    p = -g / 70.0
    longest = np.sqrt((p * p).sum(1)).max()
    assert longest < np.linalg.norm(p)   # the atom step, not the global norm, sets the clamp
    # exactly at maxstep: the factor applies (it is 1)
    at = lo.determine_step(p, longest)
    assert np.array_equal(at, p * (longest / longest))
    small = lo.params(0.0, maxstep=0.5 * longest)
    x2, _, _ = lo.step(lo.State(), x, g, np.ones(5), small)
    assert np.sqrt(((x2 - x) ** 2).sum(1)).max() == pytest.approx(0.5 * longest, rel=1e-14)
    damped = lo.params(0.0, maxstep=0.5 * longest, damping=0.3)
    x3, _, _ = lo.step(lo.State(), x, g, np.ones(5), damped)
    assert np.allclose(x3 - x, 0.3 * (x2 - x), rtol=1e-14, atol=1e-16)


def test_history_keeps_the_last_memory_pairs_and_skips_zero_curvature():
    rng = np.random.default_rng(9)
    st = lo.State(memory=3)
    par = lo.params(0.0, maxstep=0.05)
    x = fo.icosahedron() + 0.05 * rng.standard_normal((13, 3))
    xs, gs = [], []
    for t in range(7):
        g = fo.lj(x)[1]
        xs.append(x.copy())
        gs.append(g)
        x, _, _ = lo.step(st, x, g, np.ones(13), par)
    assert st.iteration == 7 and len(st.s) == 3
    for j in range(3):   # the pairs x(t+1) - x(t) of t = 3, 4, 5, oldest first
        t = 3 + j
        assert np.array_equal(st.s[j], (xs[t + 1] - xs[t]).reshape(-1))
        assert np.array_equal(st.y[j], (gs[t + 1] - gs[t]).reshape(-1))
    # a pair with y.s == 0 (no move and the same forces) is skipped: the history keeps its last pairs, no gap
    kept = [s.copy() for s in st.s]
    st.r0, st.g0 = x.copy(), fo.lj(x)[1]
    lo.update(st, x, st.g0)
    assert len(st.s) == 3 and all(np.array_equal(a, b) for a, b in zip(st.s, kept))


def test_fixed_atoms_do_not_move():
    rng = np.random.default_rng(4)
    x0 = fo.icosahedron() + 0.08 * rng.standard_normal((13, 3))
    scale = np.ones(13)
    scale[[0, 5]] = 0.0
    x, _, _ = lo.run(x0, fo.lj, lo.params(1e-3), 200, force_scale=scale)
    assert np.array_equal(x[[0, 5]], x0[[0, 5]])


def test_lj13_reaches_the_global_minimum_in_fewer_steps_than_fire():
    """The 64 perturbed icosahedra of the GPU tests (seed 2024, sigma 2.5 A, eps 0.5 eV, noise 0.08 sigma) reach
    E = -44.326801 eps at fmax 1e-3 eV / A, each in fewer steps than FIRE (float64 oracles of both)."""
    rng = np.random.default_rng(2024)
    sig, eps = 2.5, 0.5
    xs = [fo.icosahedron(sig) + 0.08 * sig * rng.standard_normal((13, 3)) for _ in range(64)]

    def eg(x):
        return fo.lj(x, sig, eps)
    steps = []
    for x0 in xs:
        x, e, t = lo.run(x0, eg, lo.params(1e-3), 1000)
        _, _, t_fire = fo.run(x0, eg, fo.params(1e-3), 1000)
        assert 0 < t < t_fire, (t, t_fire)
        assert e / eps == pytest.approx(fo.E_LJ13, abs=1e-6)
        steps.append(t)
    assert max(steps) <= 47, max(steps)   # the step budget test_gpu_lbfgs.py doubles


def test_lbfgs_state_layout_matches_header(tmp_path):
    from torchani_b200 import _lib
    prog = tmp_path / "lbfgs.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "ani_b200.h"\n'
                    'int main(){printf("%zu %zu %zu %zu %zu %zu %zu %d %d %d %d %zu\\n", sizeof(ani_lbfgs_state),'
                    ' offsetof(ani_lbfgs_state, iter), offsetof(ani_lbfgs_state, partials),'
                    ' offsetof(ani_lbfgs_state, n_conf), offsetof(ani_lbfgs_state, memory),'
                    ' offsetof(ani_lbfgs_state, record_rows), offsetof(ani_lbfgs_state, force_scale),'
                    ' ANI_LBFGS_PARAMS, ANI_LBFGS_RECORD, ANI_LBFGS_MAX_MEMORY, ANI_LBFGS_TILE,'
                    ' ANI_LBFGS_PARTIALS(3, 130, 100));return 0;}\n')
    exe = tmp_path / "lbfgs"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    out = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    S = _lib.LbfgsState
    assert out == [C.sizeof(S), S.iter.offset, S.partials.offset, S.n_conf.offset, S.memory.offset,
                   S.record_rows.offset, S.force_scale.offset, _lib.ANI_LBFGS_PARAMS, _lib.ANI_LBFGS_RECORD,
                   _lib.ANI_LBFGS_MAX_MEMORY, _lib.ANI_LBFGS_TILE, _lib.lbfgs_partials(3, 130, 100)]
    assert len(lo.PARAMS) == _lib.ANI_LBFGS_PARAMS
    assert _lib.ANI_LBFGS_RECORD == _lib.ANI_OPT_RECORD   # the drivers share the record layout


def test_lbfgs_argument_validation_without_gpu():
    """Bad arguments are rejected before any CUDA call (the pointers are host dummies)."""
    from torchani_b200 import _lib
    L = _lib.lib()
    buf = (C.c_char * 4096)()
    h = C.cast(buf, C.c_void_p).value
    names = [k for k, _ in _lib.LbfgsState._fields_ if k not in ("n_conf", "n_per_conf", "memory", "record_rows")]

    def state(**kw):
        s = _lib.LbfgsState()
        for k in names:
            setattr(s, k, h)
        s.n_conf, s.n_per_conf, s.memory, s.record_rows = 1, 4, 8, 4
        for k, v in kw.items():
            setattr(s, k, v)
        return s

    def step(s, grad=h, energies=h, coords=h):
        return L.ani_b200_lbfgs_step(C.byref(s), grad, energies, None, coords, None)

    for bad in [{k: None} for k in names] + [{"n_conf": 0}, {"n_per_conf": 0}, {"record_rows": 0}, {"memory": 0},
                                             {"memory": 129}, {"memory": -1}]:
        assert step(state(**bad)) == -1, bad
    assert step(state(), grad=None) == -1
    assert step(state(), energies=None) == -1
    assert step(state(), coords=None) == -1
    assert step(state(n_conf=70000)) != 0   # more conformers than a grid dimension holds
    assert L.ani_b200_lbfgs_step_cells(C.byref(state()), h, h, None, h, None) == -1   # no lattice table
    assert L.ani_b200_lbfgs_init(C.byref(state()), None, 1, 1, h, None) == -1   # a periodic mode without its cell
    assert L.ani_b200_lbfgs_init(C.byref(state()), h, 3, 1, h, None) == -1
    assert L.ani_b200_lbfgs_init(C.byref(state()), None, 0, 1, None, None) == -1
    assert L.ani_b200_lbfgs_init(C.byref(state(memory=200)), None, 0, 1, h, None) == -1
    assert L.ani_b200_lbfgs_init(C.byref(state(x_prev=None)), None, 0, 1, h, None) == -1


class _CpuModel:
    """Enough of a model for the driver's checks that come before any device work."""

    def buffers(self):
        import torch
        yield torch.zeros(1)


@pytest.mark.parametrize("kw,match", [
    (dict(memory=0), "memory"), (dict(memory=129), "memory"), (dict(memory=2.5), "memory"),
    (dict(alpha=0.0), "alpha"), (dict(alpha=math.inf), "alpha"), (dict(damping=-1.0), "damping"),
    (dict(damping=math.nan), "damping"), (dict(maxstep=0.0), "maxstep"), (dict(maxstep=math.inf), "maxstep"),
    (dict(steps_per_replay=0), "steps_per_replay")])
def test_lbfgs_parameter_rejections_without_gpu(kw, match):
    from torchani_b200 import optimize
    with pytest.raises(ValueError, match=match):
        optimize.LBFGS(_CpuModel(), np.zeros(3, dtype=np.int64), np.zeros((3, 3)), **kw)


def test_lbfgs_warns_on_a_large_maxstep_and_rejects_a_cpu_model():
    from torchani_b200 import optimize
    with pytest.warns(UserWarning, match="maximum step"):
        with pytest.raises(ValueError, match="CUDA"):
            optimize.LBFGS(_CpuModel(), np.zeros(3, dtype=np.int64), np.zeros((3, 3)), maxstep=1.5)
    with pytest.raises(ValueError, match="CUDA"):
        optimize.LBFGS(_CpuModel(), np.zeros(3, dtype=np.int64), np.zeros((3, 3)))
