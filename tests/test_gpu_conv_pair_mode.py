"""Every 256 -> 256 tensor-core conv of the SMPL- and MANO-size hierarchies runs in the 64 x 256 mode of
k_cheb_conv_wide (one CTA per 64-row tile for all 256 output columns, both MMA warpgroups reading one A block, a ring
of three 40 KB slots); the 128 -> 256 layer and every 128-wide one keep 128 columns per CTA.  What the layers compute
is checked against float64 by test_gpu_kernels_fp64.py and test_gpu_at_size.py; this pins which mode they run in."""
import ctypes as C

import pytest
import torch

import bench

pytestmark = pytest.mark.gpu


def tiling(lib, h, level, fin, fout):
    from pose2mesh_release_b200 import _lib

    out = (C.c_int32 * 3)()
    _lib.check(lib.p2m_debug_conv_tiling(h, level, fin, fout, out), "p2m_debug_conv_tiling")
    return dict(cols=out[0], ns=out[1], xs=out[2])


@pytest.mark.parametrize("mesh", ["smpl", "mano"])
def test_256_wide_layers_take_the_64x256_mode(mesh):
    from pose2mesh_release_b200 import _lib
    from pose2mesh_release_b200.meshnet import Pose2Mesh

    graph_L, _ = bench.build_problem(mesh)
    model = Pose2Mesh(5, 3, graph_L, joint_set="mano" if mesh == "mano" else "human36")
    model = model.to(torch.device("cuda:0")).set_precision("fp16x3").eval()
    hier, d = model._hier, torch.cuda.current_device()
    lib, h = _lib.load(), hier.handle(d)
    seen = set()
    for info in hier.layer_info(d):
        if info["fout"] not in (128, 256) or info["fin"] % 32 != 0:
            continue
        t = tiling(lib, h, info["level"], info["fin"], info["fout"])
        if t["cols"] == 0:  # not on the tensor cores (e.g. the joint graph)
            continue
        seen.add(info["fout"])
        if info["fin"] == info["fout"] == 256:
            assert t == dict(cols=256, ns=3, xs=2), (info, t)
        else:
            assert t["cols"] == 128 and t["ns"] in (3, 6), (info, t)
    assert 256 in seen and 128 in seen, seen
