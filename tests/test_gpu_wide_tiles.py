"""The 64-row x 128-column configuration of the wgmma conv (every T1-given and plain conv with Fout % 128 == 0) at the
places the width grid only touches in passing: the persistent CTA loop around its grid (all SMs for 128-wide layers,
half of them for 256-wide ones), levels with V % 64 == 0 but V % 128 != 0 (no TMA boxes, tiles end on a 64-row
boundary), 256 -> 256 forward and backward, and the padding-elision index-list families of a full-size level whose
connected row count is not a multiple of 64.  Every case asserts kernel_status == 0."""
import ctypes as C

import numpy as np
import pytest
import torch

import graphs as G
from helpers import CASES
from test_gpu_kernels_fp64 import check_bwd, check_fwd, conv_path, expect_tc, level, make_layer, run

pytestmark = pytest.mark.gpu


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("fin,fout", [(128, 128), (32, 256)], ids=lambda v: str(v))
def test_persistent_loop_64_row_tiles(fin, fout):
    """V = 64: one 64-row tile per mesh, so n_tiles = B and the grid is min(B, SMs / (fout / 128)): n_tiles = 1, grid - 1,
    grid, grid + 1 and 3 grid + 5 make every CTA run 0, 1, 2 or 4 tiles (6-slot ring phases wrap mid-tile)."""
    L = G.get("V64")
    grid = sms() // (fout // 128)
    for B in (1, grid - 1, grid, grid + 1, 3 * grid + 5):
        x, W, b = make_layer(64, B, fin, fout, seed=B + fout)
        dz = np.random.default_rng(B).standard_normal((B, 64, fout)).astype(np.float32)
        y, dx, dW, db, p = run(L, x, W, b, "fp16x3", dz if B in (grid + 1, 3 * grid + 5) else None)
        expect_tc(p, "fp16x3", fin, fout, 64)
        check_fwd(f"V64 B={B} {fin}->{fout}", L, x, W, b, "fp16x3", y)
        if dx is not None:
            check_bwd(f"V64 B={B} {fin}->{fout}", L, x, W, dz, "fp16x3", dx, dW, db)


def test_persistent_loop_two_tiles_per_mesh():
    """V = 128 (TMA boxes of 64 rows): two tiles per mesh, n_tiles = 2 B around the all-SM grid of a 128-wide layer."""
    L = G.get("V128")
    grid = sms()
    for B in (grid // 2, grid // 2 + 1, (3 * grid + 5) // 2):
        x, W, b = make_layer(128, B, 128, 128, seed=B)
        dz = np.random.default_rng(B).standard_normal((B, 128, 128)).astype(np.float32)
        y, dx, dW, db, p = run(L, x, W, b, "fp16x3", dz)
        expect_tc(p, "fp16x3", 128, 128, 128)
        check_fwd(f"V128 B={B}", L, x, W, b, "fp16x3", y)
        check_bwd(f"V128 B={B}", L, x, W, dz, "fp16x3", dx, dW, db)


@pytest.mark.parametrize("name", ["V1088", "far"])
@pytest.mark.parametrize("fin,fout", [(64, 128), (128, 128), (256, 256)], ids=lambda v: str(v))
def test_v_multiple_of_64_not_128(name, fin, fout):
    """V = 1088 = 17 * 64: the 64-row tiles end exactly at V, the 128-row ones do not, and no own-row TMA box is used."""
    L = G.get(name)
    V = L.shape[0]
    assert V % 64 == 0 and V % 128 != 0
    x, W, b = make_layer(V, 3, fin, fout, seed=V + fin + fout)
    dz = np.random.default_rng(fout).standard_normal((3, V, fout)).astype(np.float32)
    y, dx, dW, db, p = run(L, x, W, b, "fp16x3", dz)
    expect_tc(p, "fp16x3", fin, fout, V)
    assert p["tma"] == 0
    check_fwd(f"{name} {fin}->{fout}", L, x, W, b, "fp16x3", y)
    check_bwd(f"{name} {fin}->{fout}", L, x, W, dz, "fp16x3", dx, dW, db)


@pytest.mark.parametrize("lvl", ["tma", "ragged"])
def test_256_to_256_forward_and_backward(lvl):
    L = level(lvl)
    V = L.shape[0]
    x, W, b = make_layer(V, 4, 256, 256, seed=256 + V)
    dz = np.random.default_rng(V).standard_normal((4, V, 256)).astype(np.float32)
    y, dx, dW, db, p = run(L, x, W, b, "fp16x3", dz)
    expect_tc(p, "fp16x3", 256, 256, V)
    check_fwd(f"256->256 {lvl}", L, x, W, b, "fp16x3", y)
    check_bwd(f"256->256 {lvl}", L, x, W, dz, "fp16x3", dx, dW, db)


def _per_mesh_rel_err(y, ref):
    y, ref = y.detach().double().cpu(), ref.detach().double().cpu()
    d = (y - ref).abs().flatten(1).max(dim=1).values
    s = ref.abs().flatten(1).max(dim=1).values.clamp_min(1e-30)
    return float((d / s).max())


def test_index_list_tiles_with_ragged_row_count():
    """The full-size SMPL hierarchy: the finest level's 6890 connected rows (real_tiles) are 107 full 64-row tiles and
    one of 42 rows; its isolated rows run as plain GEMMs on the representative / isolated families.  Elision forced on,
    off, and the default (with duplicate elimination) must agree, in eval and train mode."""
    from pose2mesh_release_b200 import _lib
    from pose2mesh_release_b200 import graph as pg
    from pose2mesh_release_b200.meshnet import Pose2Mesh

    n, seed, levels, _ = CASES["smpl_like"]
    face = pg.synthetic_sphere_faces(n, seed)
    _, graph_L, _, _ = pg.build_coarse_graphs(face, 17, pg.H36M_SKELETON, pg.H36M_FLIP_PAIRS, levels=levels)
    torch.manual_seed(123)
    model = Pose2Mesh(5, 3, graph_L, joint_set="human36").to(torch.device("cuda:0")).set_precision("fp16x3").eval()
    hier, d = model._hier, torch.cuda.current_device()
    out = (C.c_int32 * 9)()
    _lib.check(_lib.load().p2m_debug_conv_path(hier.handle(d), 0, 128, 128, out), "p2m_debug_conv_path")
    V, n_iso = graph_L[0].shape[0], out[8]
    assert n_iso > 0 and (V - n_iso) % 64 != 0, (V, n_iso)
    x = torch.randn(6, 17, 5, generator=torch.Generator().manual_seed(2)).to(torch.device("cuda:0"))
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    res = {}
    try:
        for mode in (0, 1, 2):
            hier.set_debug(d, elide_padding=mode)
            with torch.no_grad():
                model.eval()
                y_eval = model(x)
                model.train()
                y_train = model(x)
            model.load_state_dict(sd)  # undo the running-stat update
            res[mode] = (y_eval, y_train)
        assert hier.kernel_status(d) == 0
    finally:
        hier.set_debug(d, elide_padding=1, dedup_padding=True)
        model.eval()
    for mode in (1, 2):
        assert _per_mesh_rel_err(res[mode][0], res[0][0]) < 2e-5, mode
        assert _per_mesh_rel_err(res[mode][1], res[0][1]) < 2e-5, mode
