"""The wgmma main loops of the MLP kernels, as compiled: every commit group is one run of wgmmas.

ptxas closes each branch inside a wgmma commit group with its own group boundary (the SASS `gsb0` flag).  A run-time
branch between `wgmma.fence` and `wgmma.commit_group` therefore turns one group into several, closed by an empty
HGMMA that carries the commit, and `wgmma.wait_group 1` (`WARPGROUP.DEPBAR.LE gsb0, 0x1`) then waits for all of
them: the tensor pipe drains at every K-block.  ptxas also reports a warpgroup.arrive it had to inject (C7519).
These checks read the library the build made; no GPU is needed."""
import os
import re
import shutil
import subprocess

import pytest

from torchani_b200 import build

KERNELS = ("k_mlp_resident", "k_gemm_wg")
EMPTY_COMMIT = re.compile(r"HGMMA\.64x8x16\.F16 RZ, gdesc\[URZ\]")


def _tools():
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    cuobjdump = shutil.which("cuobjdump") or os.path.join(os.path.dirname(nvcc), "cuobjdump")
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not found")
    return cuobjdump


def _kernels(cuobjdump, lib):
    """{mangled name: [SASS instruction lines]} of the MLP GEMM kernels in the library"""
    sass = subprocess.run([cuobjdump, "-sass", lib], capture_output=True, text=True, check=True).stdout
    out = {}
    for fn in re.split(r"\n\s*Function : ", sass)[1:]:
        name, body = fn.split("\n", 1)
        if any(k in name for k in KERNELS):
            out[name.strip()] = [ln for ln in body.split("\n") if re.match(r"\s*/\*[0-9a-f]{4,}\*/", ln)]
    return out


@pytest.mark.parametrize("variant", ["", "bf16x3"])
def test_every_wgmma_commit_group_is_one_run(variant):
    cuobjdump = _tools()
    lib = build.build(variant=variant)
    kernels = _kernels(cuobjdump, lib)
    expected = KERNELS if not variant else ("k_gemm_wg",)  # the 3 x bf16 build has no resident kernel
    for k in expected:
        assert any(k in name for name in kernels), f"{k} not found in {lib}"
    for name, lines in kernels.items():
        assert not any(EMPTY_COMMIT.search(ln) for ln in lines), f"{name}: empty HGMMA carrying a commit"
        open_group = False  # a group closed by gsb0 that no WARPGROUP.DEPBAR has waited on yet
        for ln in lines:
            if "WARPGROUP.DEPBAR" in ln:
                open_group = False
            elif "HGMMA" in ln and "gsb0" in ln:
                assert not open_group, f"{name}: two gsb0 HGMMAs without a WARPGROUP.DEPBAR between them:\n{ln}"
                open_group = True
    log = os.path.join(build.BUILD + ("_" + variant if variant else ""), "mlp.ptxas.log")
    injected = [ln for ln in open(log) if "C7519" in ln and any(k in ln for k in KERNELS)]
    assert not injected, "ptxas injected warpgroup.arrive:\n" + "".join(injected[:4])
