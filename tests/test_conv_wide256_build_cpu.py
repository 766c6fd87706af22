"""CPU-only checks of the build of the 64 x 256 mode of k_cheb_conv_wide (csrc/cheb_umma.cu: 256 output columns per
CTA, both MMA warpgroups on one tile): it launches with the 96 registers the 640-thread setmaxnreg split assumes, and
each warpgroup issues six 128-column wgmma per K-block on its half of the weight block, with no 64-column wgmma."""
import os
import re
import shutil
import subprocess

import pytest


def _cuobjdump():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    return tool


def _pair_kernels(tool, lib):
    """{mangled name: launch registers} of every k_cheb_conv_wide<256, ...> instantiation in the library."""
    out = subprocess.run([tool, "-res-usage", lib], capture_output=True, text=True).stdout
    found = re.findall(r"Function (\S*k_cheb_conv_wideILi256E\S*?):?\n[^\n]*REG:(\d+)", out)
    return {name: int(regs) for name, regs in found}


def test_pair_conv_launches_with_96_registers():
    from pose2mesh_release_b200 import build

    tool = _cuobjdump()
    kernels = _pair_kernels(tool, build.build())
    # one ring depth (3 slots) x two T1 stagings, T1-given convs only
    assert len(kernels) == 2, sorted(kernels)
    assert set(kernels.values()) == {96}, kernels


def test_pair_conv_main_loop_issues_m64n128():
    """Both warpgroups run the one main loop, so the SASS holds the six HGMMA.64x128x16 of a K-block once."""
    from pose2mesh_release_b200 import build

    tool = _cuobjdump()
    lib = build.build()
    kernels = _pair_kernels(tool, lib)
    assert kernels
    for name in kernels:
        sass = subprocess.run([tool, "-sass", "-fun", name, lib], capture_output=True, text=True).stdout
        hgmma = re.findall(r"HGMMA\.(\d+x\d+x\d+)", sass)
        assert hgmma.count("64x128x16") == 6 and set(hgmma) == {"64x128x16"}, (name, hgmma)
