"""The C-ABI library: loads, exports every symbol include/ani_b200.h declares, struct layouts
match the ctypes mirror, and argument validation works without a GPU (no compute calls)."""
import ctypes as C
import os
import re
import subprocess
import sys

import pytest

from helpers import ROOT

HEADER = os.path.join(ROOT, "include", "ani_b200.h")


def _declared_symbols():
    src = open(HEADER).read()
    return sorted(set(re.findall(r"\b(ani_b200_[a-z0-9_]+)\s*\(", src)))


def test_library_builds_and_exports_every_declared_symbol():
    from torchani_b200 import build
    lib_path = build.build()
    assert os.path.exists(lib_path)
    lib = C.CDLL(lib_path)
    declared = _declared_symbols()
    assert len(declared) >= 11
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in ani_b200.h but not exported"
    from torchani_b200 import _lib
    assert sorted(_lib.EXPORTED_SYMBOLS) == declared, "ctypes prototypes out of sync with the header"
    assert _lib.lib().ani_b200_abi_version() == 4


def test_struct_layouts_match_header(tmp_path):
    from torchani_b200 import _lib
    prog = tmp_path / "sz.c"
    prog.write_text(
        '#include <stdio.h>\n#include <stddef.h>\n#include "ani_b200.h"\n'
        'int main(){printf("%zu %zu %zu %zu %zu %zu %zu\\n", sizeof(ani_aev_params), sizeof(ani_grid),'
        ' sizeof(ani_mlp_species), sizeof(ani_mlp_model), offsetof(ani_grid, n_real),'
        ' offsetof(ani_mlp_model, sp), offsetof(ani_aev_params, cos_z));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    sizes = [int(v) for v in out]
    assert sizes == [C.sizeof(_lib.AEVParams), C.sizeof(_lib.Grid), C.sizeof(_lib.MLPSpecies),
                     C.sizeof(_lib.MLPModel), _lib.Grid.n_real.offset, _lib.MLPModel.sp.offset,
                     _lib.AEVParams.cos_z.offset]


def test_argument_validation_without_gpu():
    """Bad arguments are rejected before any CUDA call is made."""
    from torchani_b200 import _lib
    L = _lib.lib()
    assert L.ani_b200_error_string(0) == b"ok"
    assert b"argument" in L.ani_b200_error_string(-1)
    # null pointers
    assert L.ani_b200_build_cells(None, None, 1, 1, None, 0, 0, 5.1, 64, None, None, None, None, None, None,
                                  None, None, None, None) == -1
    assert L.ani_b200_aev_forward(None, None, None, None, None, None, None, None, 0, 0, 0, None, None, 0, 0, None, None,
                                  128, None, None) == -1
    # unsupported AEV configuration (ShfA x ShfZ must be 8x4 or 4x8) is reported as such
    p = _lib.AEVParams()
    p.num_species, p.n_shf_r, p.n_shf_a, p.n_shf_z = 7, 16, 5, 5
    p.rcr, p.rca, p.zeta = 5.1, 3.5, 14.1
    assert L.ani_b200_aev_forward(C.byref(p), None, None, None, None, None, None, None, 0, 0, 0, None, None, 0, 0, None,
                                  None, 128, None, None) == -2
    with pytest.raises(_lib.ANIB200Error):
        _lib.check(-2, "x")

    # member lists of the step terms: the arguments are valid except where a case says otherwise.  The pointers are
    # host dummies, so every call below must return before it touches CUDA; the pair and AEV-members calls with an
    # empty atom range (lo == hi) and a valid list return OK there, which shows the other cases fail on their lists.
    buf = (C.c_char * 4096)()
    h = C.cast(buf, C.c_void_p)
    ok_list = (C.c_int32 * 3)(0, 3, 7)
    lists = {"count above 16": (ok_list, 17), "index out of range": ((C.c_int32 * 2)(0, 16), 2),
             "negative index": ((C.c_int32 * 2)(-1, 0), 2), "null list": (None, 3)}
    pp = _lib.PairParams()
    pp.kind, pp.cutoff_fn, pp.num_species, pp.cutoff, pp.to_bohr = 0, 1, 7, 5.1, 1.8897
    dp = _lib.D3Params()
    dp.cutoff_fn, dp.num_species, dp.cutoff, dp.to_bohr = 1, 7, 8.0, 1.8897
    ap = _lib.AEVParams()
    ap.num_species, ap.n_shf_r, ap.n_shf_a, ap.n_shf_z, ap.cutoff_kind = 7, 16, 8, 4, 0
    ap.rcr, ap.rca, ap.zeta = 5.1, 3.5, 14.1

    def pair(members, n_members, lo=0, hi=4, member_atomic=h, grad_members=h):
        return L.ani_b200_pair_potential(C.byref(pp), h, h, h, 4, lo, hi, 1, 4, h, h, 32, h, h, h, h, member_atomic,
                                         grad_members, members, n_members, None)

    def d3(members, n_members, member_atomic=h, grad_members=h, cells=False, lattice=h):
        args = (C.byref(dp), h, h, h, h, h, 4, 0, 4, 1, 4, 1.0, h, h, h, h, h, h, member_atomic, grad_members, members,
                n_members, h)
        if cells:
            return L.ani_b200_dispersion_d3_cells(*args, lattice, None)
        return L.ani_b200_dispersion_d3(*args, None)

    def aev_members(members, n_members, lo=0, hi=4):
        return L.ani_b200_aev_backward_members(C.byref(ap), h, h, h, h, 4, lo, hi, h, h, 1008, 1008, members,
                                               n_members, h, h, 64, h, h, 0, None)

    def qbc(members, n_members):
        return L.ani_b200_ensemble_qbc(h, members, n_members, h, h, None, 1, 4, h, h, h, h, None)

    assert pair(ok_list, 3, hi=0) == 0
    assert aev_members(ok_list, 3, hi=0) == 0
    for case, (members, n_members) in lists.items():
        assert pair(members, n_members) == -1, case
        assert d3(members, n_members) == -1, case
        assert d3(members, n_members, cells=True) == -1, case
        assert aev_members(members, n_members) == -1, case
        assert qbc(members, n_members) == -1, case
    # member outputs with no members
    assert pair(None, 0, grad_members=None) == -1
    assert pair(None, 0, member_atomic=None) == -1
    assert d3(None, 0, grad_members=None) == -1
    assert d3(None, 0, member_atomic=None, cells=True) == -1
    # zero members where the call needs one
    assert aev_members(ok_list, 0) == -1
    assert qbc(ok_list, 0) == -1
    # the _cells form of D3 without its lattice table
    assert d3(ok_list, 3, cells=True, lattice=None) == -1

    # an MD step over more conformers than a grid's y extent holds
    st = _lib.MDState()
    for name in ("x", "v", "inv_mass", "params", "counter", "stop_step", "thermo", "partials"):
        setattr(st, name, h.value)
    st.accel, st.kb, st.integrator, st.thermo_rows = 1.0, 1.0, _lib.MD_VERLET, 1
    st.n_conf, st.n_per_conf = 65536, 1
    assert L.ani_b200_md_step(C.byref(st), h, h, None, None, None, h, None) == -2


def test_product_package_does_not_import_the_oracle():
    """The oracle is test infrastructure: nothing under torchani_b200/ may reference it."""
    pkg = os.path.join(ROOT, "torchani_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in text and "from oracle" not in text and "oracle." not in text, \
                    f"{f} uses the oracle"
    code = "import sys; import torchani_b200.models, torchani_b200.parallel; print(any(m.startswith('oracle') for m in sys.modules))"
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT, check=True)
    assert out.stdout.strip() == "False"
