"""CPU-only checks of the build of k_cheb_conv_wide, the 640-thread 64 x 128 Chebyshev conv (csrc/cheb_umma.cu): it is
launched with the register count its setmaxnreg split assumes, that split is balanced, and its main loop issues one
128-column wgmma per K step instead of two 64-column ones."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "pose2mesh_release_b200", "csrc", "cheb_umma.cu")


def _cuobjdump():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    return tool


def _wide_kernels(tool, lib):
    """{mangled name: launch registers} of every k_cheb_conv_wide instantiation in the library."""
    out = subprocess.run([tool, "-res-usage", lib], capture_output=True, text=True).stdout
    found = re.findall(r"Function (\S*k_cheb_conv_wide\S*?):?\n[^\n]*REG:(\d+)", out)
    return {name: int(regs) for name, regs in found}


def _wide_constants():
    src = open(SRC).read()
    m = re.search(r"REGS_LAUNCH_W = (\d+), REGS_UTIL_W = (\d+), REGS_PROD_W = (\d+), REGS_EPI_W = (\d+)", src)
    t = re.search(r"NUM_THREADS_W = (\d+) \* 32", src)
    assert m and t, "register targets of the 64 x 128 layout not found"
    return (*(int(v) for v in m.groups()), int(t.group(1)) * 32)


def test_wide_conv_launches_with_the_registers_its_split_assumes():
    """setmaxnreg.inc draws on what the CTA's own setmaxnreg.dec released, so the split only balances if every
    instantiation is launched with REGS_LAUNCH_W (96) registers per thread; the host refuses to launch otherwise."""
    from pose2mesh_release_b200 import build

    tool = _cuobjdump()
    kernels = _wide_kernels(tool, build.build())
    assert len(kernels) >= 8, f"k_cheb_conv_wide instantiations: {sorted(kernels)}"
    launch = _wide_constants()[0]
    assert set(kernels.values()) == {launch} == {96}, kernels


def test_wide_conv_register_split_is_balanced():
    """640 threads at 96 registers fill the SM's 64 K (104 would not fit); the utility warpgroup (40) and the two
    producer warpgroups pay for the two MMA + epilogue warpgroups, whose m64n128 accumulator needs more than 90."""
    launch, util, prod, epi, threads = _wide_constants()
    assert threads == 640
    assert launch * threads <= 65536 < (launch + 8) * threads
    assert all(v % 8 == 0 and 24 <= v <= 256 for v in (launch, util, prod, epi))
    assert 2 * 128 * (epi - launch) <= 128 * (launch - util) + 2 * 128 * (launch - prod)
    assert epi >= 96


def test_wide_conv_main_loop_issues_m64n128():
    """Six wgmma per K-block (hi*Whi, lo*Whi, hi*Wlo, two k16 steps each), each over all 128 output columns: every
    instantiation carries exactly six HGMMA.64x128x16 and no 64-column HGMMA."""
    from pose2mesh_release_b200 import build

    tool = _cuobjdump()
    lib = build.build()
    kernels = _wide_kernels(tool, lib)
    assert kernels
    for name in kernels:
        sass = subprocess.run([tool, "-sass", "-fun", name, lib], capture_output=True, text=True).stdout
        hgmma = re.findall(r"HGMMA\.(\d+x\d+x\d+)", sass)
        assert hgmma.count("64x128x16") == 6 and set(hgmma) == {"64x128x16"}, (name, hgmma)
