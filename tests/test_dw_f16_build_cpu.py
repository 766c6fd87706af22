"""CPU-only checks of the build of the single-pass fp16 weight gradient (csrc/cheb_umma.cu: k_cheb_dw_f16_umma,
cheb_dw_body with F16 = true): each instantiation launches with the registers of the 768-thread launch it shares with
k_cheb_dw_umma (no setmaxnreg split to rebalance, no spills), and issues one third of the matching fp16x3 kernel's
HGMMAs, all m64n32k16: one g T product per 16-row K step where fp16x3 issues g_hi T_hi, g_lo T_hi and g_hi T_lo."""
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


def _kernels(tool, lib, name):
    """{XS: (mangled name, registers, stack bytes)} of every instantiation of kernel `name` in the library."""
    out = subprocess.run([tool, "-res-usage", lib], capture_output=True, text=True).stdout
    found = re.findall(r"Function (\S*\d" + name + r"ILi(\d+)E\S*?):?\n[^\n]*REG:(\d+) STACK:(\d+)", out)
    return {int(xs): (n, int(regs), int(stack)) for n, xs, regs, stack in found}


def _hgmma(tool, lib, fn):
    sass = subprocess.run([tool, "-sass", "-fun", fn, lib], capture_output=True, text=True).stdout
    return re.findall(r"HGMMA\.(\d+x\d+x\d+)", sass)


def test_f16_dw_builds_both_x_stages_with_80_registers_and_a_third_of_the_hgmma():
    from pose2mesh_release_b200 import build

    tool = _cuobjdump()
    lib = build.build()
    f16 = _kernels(tool, lib, "k_cheb_dw_f16_umma")
    x3 = _kernels(tool, lib, "k_cheb_dw_umma")
    assert set(f16) == set(x3) == {1, 2}, (sorted(f16), sorted(x3))
    for xs in (1, 2):
        name, regs, stack = f16[xs]
        # __launch_bounds__(768, 1): 65536 / 768 rounded down to a multiple of 8, as the fp16x3 kernel
        assert regs == x3[xs][1] == 80, (name, regs, x3[xs][1])
        assert stack <= x3[xs][2], (name, stack, x3[xs][2])
        h16, h3 = _hgmma(tool, lib, name), _hgmma(tool, lib, x3[xs][0])
        assert set(h16) == set(h3) == {"64x32x16"}, (h16, h3)
        # three orders x 8 K steps per tile: 24 single-pass products, 72 at fp16x3
        assert 3 * len(h16) == len(h3) == 72, (len(h16), len(h3))
