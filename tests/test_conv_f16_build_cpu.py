"""CPU-only checks of the build of the single-pass fp16 conv kernels (csrc/cheb_umma.cu: k_cheb_conv_f16_umma and
k_cheb_conv_f16_wide, cheb_conv_body with F16 = true): each launches with the register count its setmaxnreg split
assumes, and its main loop issues two k16 wgmma per K-block (per 64-row half in the 128 x 64 configuration) where the
fp16x3 instantiations issue six."""
import re
import shutil
import subprocess
import os

import pytest


def _cuobjdump():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    return tool


def _kernels(tool, lib, name):
    """{mangled name: launch registers} of every instantiation of kernel `name` in the library."""
    out = subprocess.run([tool, "-res-usage", lib], capture_output=True, text=True).stdout
    found = re.findall(r"Function (\S*" + name + r"I\S*?):?\n[^\n]*REG:(\d+)", out)
    return {n: int(regs) for n, regs in found}


def _hgmma(tool, lib, fn):
    sass = subprocess.run([tool, "-sass", "-fun", fn, lib], capture_output=True, text=True).stdout
    return re.findall(r"HGMMA\.(\d+x\d+x\d+)", sass)


def _configs(kernels):
    """(NC, NS, XS, MODE) of each instantiation, from its mangled template arguments."""
    return {tuple(int(v) for v in re.search(r"ILi(\d+)ELi(\d+)ELi(\d+)ELi(\d+)E", k).groups()) for k in kernels}


def test_f16_wide_conv_builds_ring_of_6_only_with_96_registers_and_two_m64n128():
    """64 x 128 and 64 x 256: the instantiations the eval forward can launch, at the 96 registers of the 640-thread
    split.  64 x 128: a ring of 6 slots with 1 or 2 T1 stages (T1 given) and 2 X stages (plain: only the isolated rows'
    GEMM, whose tiles hold one CSR entry per row); six fp16 slots fit wherever three fp16x3 slots do, and every tile
    family a conv runs on fits those, so no ring of 3 is built (cheb_umma.cu: launchable).  64 x 256: T1 given only."""
    from pose2mesh_release_b200 import build

    tool = _cuobjdump()
    lib = build.build()
    kernels = _kernels(tool, lib, "k_cheb_conv_f16_wide")
    assert _configs(kernels) == {(128, 6, 2, 1), (128, 6, 1, 1), (128, 6, 2, 0), (256, 3, 2, 1), (256, 3, 1, 1)}, \
        sorted(kernels)
    assert len(kernels) == 5, sorted(kernels)
    assert set(kernels.values()) == {96}, kernels
    for name in kernels:
        hgmma = _hgmma(tool, lib, name)
        assert hgmma.count("64x128x16") == 2 and set(hgmma) == {"64x128x16"}, (name, hgmma)


def test_f16_conv_umma_builds_two_x_stage_plain_only_with_80_registers_and_two_k16_per_half():
    """128 x 64: 1 or 2 T1 stages (T1 given) and the plain GEMM with 2 X stages only (the isolated rows' GEMM), at 80
    registers, two k16 wgmma per K-block and 64-row half."""
    from pose2mesh_release_b200 import build

    tool = _cuobjdump()
    lib = build.build()
    kernels = _kernels(tool, lib, "k_cheb_conv_f16_umma")
    assert _configs(kernels) == {(64, 3, 2, 1), (64, 3, 1, 1), (64, 3, 2, 0)}, sorted(kernels)
    assert len(kernels) == 3, sorted(kernels)
    assert set(kernels.values()) == {80}, kernels
    for name in kernels:
        hgmma = _hgmma(tool, lib, name)
        assert hgmma.count("64x64x16") == 4 and set(hgmma) == {"64x64x16"}, (name, hgmma)
