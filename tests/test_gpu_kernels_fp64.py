"""The wgmma conv, dW and dense-GEMM kernels element-wise against float64 (tests/fp64_ref.py), through the public
module and the C ABI, at both precisions: every supported width, the persistent CTA loop, the graph families of
tests/graphs.py, input / weight / gradient scales, and two metamorphic properties that need no reference.

Every case asserts kernel_status == 0 and, through p2m_debug_conv_path, that it ran on the path it is named after.
The worst error-to-bound ratio per precision and the module's wall time are written to the JSON file named by
P2M_FP64_REPORT (if set) when the module finishes."""
import ctypes as C
import json
import os
import time

import numpy as np
import pytest
import torch

import fp64_ref as R
import graphs as G
from helpers import graph_from_fixture

pytestmark = pytest.mark.gpu

PRECISIONS = ["fp32", "fp16x3"]
_WORST = {"fp32": [0.0, ""], "fp16x3": [0.0, ""]}


@pytest.fixture(scope="module", autouse=True)
def _report():
    t0 = time.time()
    yield
    out = os.environ.get("P2M_FP64_REPORT")
    if out:
        with open(out, "w") as f:
            json.dump({"wall_s": time.time() - t0, "worst_ratio": _WORST}, f, indent=1)


def dev():
    return torch.device("cuda:0")


def level(name):
    """Sphere-hierarchy levels: 'tma' = V 1024 (smpl_small level 1), 'ragged' = V 1088 (mano_like level 0)."""
    fx, i = {"tma": ("smpl_small", 1), "ragged": ("mano_like", 0)}[name]
    return graph_from_fixture(fx)[0][i]


def conv_path(gh, fin, fout):
    from pose2mesh_release_b200 import _lib

    out = (C.c_int32 * 9)()
    _lib.check(_lib.load().p2m_debug_conv_path(gh.handle(0), 0, fin, fout, out), "p2m_debug_conv_path")
    return dict(zip(("conv", "conv_xs", "dw", "dw_xs", "dt", "dt_xs", "tma", "max_h1", "n_iso"), list(out)))


def run(L, x, W, b, precision, dz=None, sm_cap=0):
    """graph_conv_cheby's linear part on the GPU: returns (y, dx, dW, db, path) as float64 numpy (grads None without dz).
    sm_cap > 0: the persistent tensor-core grids are sized for that many SMs (p2m_debug_set_sm_count)."""
    from pose2mesh_release_b200 import _lib
    from pose2mesh_release_b200 import cheby_graph_conv as cgc

    cgc.set_default_precision(precision)
    gh = cgc.graph_handle(L)
    try:
        _lib.check(_lib.load().p2m_debug_set_sm_count(gh.handle(0), sm_cap), "set_sm_count")
        xg = torch.as_tensor(np.asarray(x, np.float32)).to(dev()).requires_grad_(dz is not None)
        Wg = torch.as_tensor(np.asarray(W, np.float32)).to(dev()).requires_grad_(dz is not None)
        bg = torch.as_tensor(np.asarray(b, np.float32)).to(dev()).requires_grad_(dz is not None)
        y = cgc.ChebConvLinear.apply(xg, Wg, bg, gh)
        grads = (None, None, None)
        if dz is not None:
            y.backward(torch.as_tensor(np.asarray(dz, np.float32)).to(dev()))
            grads = tuple(t.grad.double().cpu().numpy() for t in (xg, Wg, bg))
        assert gh.kernel_status(0) == 0, "a tensor-core kernel timed out on an mbarrier"
        p = conv_path(gh, x.shape[2], W.shape[0])
    finally:
        _lib.check(_lib.load().p2m_debug_set_sm_count(gh.handle(0), 0), "set_sm_count")
        cgc.set_default_precision("fp32")
    return (y.detach().double().cpu().numpy(),) + grads + (p,)


def check(what, precision, got, ref, bound):
    r = R.bound_ratio(got, ref, bound)
    if r > _WORST[precision][0]:
        _WORST[precision] = [r, what]
    assert r <= 1.0, f"{what}: max |err| / bound = {r:.3g}"


def make_layer(V, B, fin, fout, seed, x_scale=1.0, w_scale=1.0, zero_bias=False):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((B, V, fin)) * x_scale).astype(np.float32)
    W = ((rng.random((fout, 3 * fin)) * 2 - 1) * np.sqrt(2.0 / (3 * fin + fout)) * w_scale).astype(np.float32)
    b = np.zeros(fout, np.float32) if zero_bias else (rng.standard_normal(fout) * 0.1).astype(np.float32)
    return x, W, b


def check_fwd(tag, L, x, W, b, precision, y):
    check(tag + "/y", precision, y, R.cheb_conv_fwd(x, L, W, b), R.cheb_conv_fwd_bound(x, L, W, b, precision))


def check_bwd(tag, L, x, W, dz, precision, dx, dW, db):
    rdx, rdW, rdb = R.cheb_conv_bwd(x, L, W, dz)
    bdx, bdW, bdb = R.cheb_conv_bwd_bound(x, L, W, dz, precision)
    check(tag + "/dx", precision, dx, rdx, bdx)
    check(tag + "/dW", precision, dW, rdW, bdW)
    check(tag + "/db", precision, db, rdb, bdb)


def expect_tc(p, precision, fin, fout, V):
    tc = precision == "fp16x3" and fin % 32 == 0
    assert p["conv"] == tc and p["dw"] == tc, p
    assert p["dt"] == (tc and fin in (64, 128, 256)), p
    if tc:
        assert p["tma"] == (V % 128 == 0), p


# ------------------------------------------------------------------------------------------------------ width grid
WIDTHS = [(fin, fout) for fin in (32, 64, 96, 128, 160, 192, 224, 256) for fout in (64, 128, 256)] + \
         [(5, 64), (20, 128)]   # SIMT controls


@pytest.mark.parametrize("lvl", ["tma", "ragged"])
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("fin,fout", WIDTHS, ids=lambda v: str(v))
def test_width_grid_forward_and_backward(fin, fout, precision, lvl):
    L = level(lvl)
    V = L.shape[0]
    x, W, b = make_layer(V, 1, fin, fout, seed=fin * 1000 + fout)
    dz = np.random.default_rng(fout).standard_normal((1, V, fout)).astype(np.float32)
    y, dx, dW, db, p = run(L, x, W, b, precision, dz)
    expect_tc(p, precision, fin, fout, V)
    tag = f"width {fin}->{fout} {lvl}"
    check_fwd(tag, L, x, W, b, precision, y)
    check_bwd(tag, L, x, W, dz, precision, dx, dW, db)


# ------------------------------------------------------------------------------------------------- persistent loop
PERSISTENT_CAP = 8   # SMs the grids are sized for: independent of the part's own count


@pytest.mark.parametrize("fin,fout", [(64, 64), (128, 128), (32, 256), (256, 256)], ids=lambda v: str(v))
def test_persistent_cta_loop(fin, fout):
    """V = 128 is one 128-row tile per mesh (Fout = 64) or two 64-row tiles (Fout % 128 == 0; 32 -> 256 as two
    128-column slices, 256 -> 256 in the 64 x 256 mode), so n_tiles = B or 2 B, on a grid capped at 8 SMs: grid.x =
    min(n_tiles, 8 / column slices), read back from the launch log.  B = 1, 7, 8, 9 and 29 make each CTA run from 1 to
    15 tiles (ring slots and mbarrier phases reused).  tests/test_gpu_persistent_tiles_fp64.py covers every
    configuration."""
    from pose2mesh_release_b200 import _lib

    L = G.get("V128")
    most = 0
    for B in (1, 7, 8, 9, 29):
        x, W, b = make_layer(128, B, fin, fout, seed=B)
        dz = np.random.default_rng(B).standard_normal((B, 128, fout)).astype(np.float32)
        _lib.conv_log(reset=True)
        y, dx, dW, db, p = run(L, x, W, b, "fp16x3", dz if B in (9, 29) else None, sm_cap=PERSISTENT_CAP)
        conv = next(e for e in _lib.conv_log(reset=True) if e["kind"] == "conv")
        assert conv["grid_x"] == min(conv["n_tiles"], max(1, PERSISTENT_CAP // conv["grid_y"])), conv
        most = max(most, conv["tiles_per_cta"])
        expect_tc(p, "fp16x3", fin, fout, 128)
        check_fwd(f"persistent B={B} {fin}->{fout}", L, x, W, b, "fp16x3", y)
        if dx is not None:
            check_bwd(f"persistent B={B} {fin}->{fout}", L, x, W, dz, "fp16x3", dx, dW, db)
    assert most >= 4, most


# ------------------------------------------------------------------------------------------------- graph families
# what p2m_debug_conv_path must report for Fin = Fout = 64 at fp16x3 (None = not checked)
FAMILY_PATH = {
    "V1": dict(conv=1, tma=0), "V64": dict(conv=1, tma=0), "V127": dict(conv=1, tma=0), "V128": dict(conv=1, tma=1),
    "V129": dict(conv=1, tma=0), "V1088": dict(conv=1, tma=0), "V2048": dict(conv=1, tma=1),
    "band8": dict(conv=1, conv_xs=2), "band12": dict(conv=1, conv_xs=2), "band14": dict(conv=1, conv_xs=2),
    "band16": dict(conv=1, conv_xs=1), "band20": dict(conv=1, conv_xs=1, dw=0),
    "h1_256": dict(conv=1, max_h1=256), "h1_257": dict(conv=0, dw=0, max_h1=257),
    "far": dict(conv=1, tma=0), "hub": dict(conv=1), "empty_rows": dict(conv=1),
    "iso_uniform": dict(conv=1, n_iso=512), "iso_two_diag": dict(conv=1, n_iso=0),
    "dense": dict(conv=0, dw=0, dt=0, max_h1=0),
}


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", sorted(FAMILY_PATH))
def test_graph_family(name, precision):
    L = G.get(name)
    V = L.shape[0]
    x, W, b = make_layer(V, 2, 64, 64, seed=V)
    dz = np.random.default_rng(V + 1).standard_normal((2, V, 64)).astype(np.float32)
    y, dx, dW, db, p = run(L, x, W, b, precision, dz)
    if precision == "fp16x3":
        for k, v in FAMILY_PATH[name].items():
            assert p[k] == v, (k, p)
    else:
        assert p["conv"] == p["dw"] == p["dt"] == 0
    check_fwd(name, L, x, W, b, precision, y)
    check_bwd(name, L, x, W, dz, precision, dx, dW, db)
    # the same matrix as a torch COO tensor with every entry stored twice: graph_handle coalesces it
    y2 = run(G.torch_coo_with_duplicates(L), x, W, b, precision)[0]
    assert np.array_equal(y, y2)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_nonsymmetric_laplacian(precision):
    """The forward is right for any L~; the backward needs L~^T, which the kernels only have for a symmetric L~:
    it must refuse rather than return a gradient for L~."""
    L = G.get("nonsymmetric")
    V = L.shape[0]
    x, W, b = make_layer(V, 2, 64, 64, seed=3)
    y = run(L, x, W, b, precision)[0]
    check_fwd("nonsymmetric", L, x, W, b, precision, y)
    dz = np.ones((2, V, 64), np.float32)
    with pytest.raises(RuntimeError, match="symmetric"):
        run(L, x, W, b, precision, dz)


# ------------------------------------------------------------------------------------------------------------ scales
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("e", [-24, -16, -12, 0, 12, 15, 20])
def test_input_scale(e, precision):
    L = level("tma")
    x, W, b = make_layer(L.shape[0], 2, 64, 128, seed=5, x_scale=2.0 ** e)
    y, *_, p = run(L, x, W, b, precision)
    expect_tc(p, precision, 64, 128, L.shape[0])
    check_fwd(f"x*2^{e}", L, x, W, b, precision, y)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_mixed_row_magnitudes_and_zero_rows(precision):
    L = level("ragged")
    V = L.shape[0]
    x, W, b = make_layer(V, 2, 96, 64, seed=6)
    rng = np.random.default_rng(7)
    x = (x * 2.0 ** rng.uniform(-8, 8, size=(2, V, 1))).astype(np.float32)
    x[:, 130:200] = 0.0                                  # all-zero rows inside a tile
    dz = (rng.standard_normal((2, V, 64)) * 2.0 ** rng.uniform(-8, 8, size=(2, V, 1))).astype(np.float32)
    y, dx, dW, db, p = run(L, x, W, b, precision, dz)
    expect_tc(p, precision, 96, 64, V)
    check_fwd("mixed rows", L, x, W, b, precision, y)
    check_bwd("mixed rows", L, x, W, dz, precision, dx, dW, db)
    # an all-zero input returns the bias exactly
    y0 = run(L, np.zeros_like(x), W, b, precision)[0]
    assert np.array_equal(y0, np.broadcast_to(b.astype(np.float64), y0.shape))


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("e", [-8, 6, 14])
def test_weight_scale(e, precision):
    """max |w| ~ 1400 at e = 14: beyond fp16's range after a fixed 2^6 packing scale."""
    L = level("tma")
    x, W, b = make_layer(L.shape[0], 1, 64, 64, seed=8, w_scale=2.0 ** e)
    dz = np.random.default_rng(9).standard_normal((1, L.shape[0], 64)).astype(np.float32)
    y, dx, dW, db, p = run(L, x, W, b, precision, dz)
    expect_tc(p, precision, 64, 64, L.shape[0])
    check_fwd(f"w*2^{e}", L, x, W, b, precision, y)
    check_bwd(f"w*2^{e}", L, x, W, dz, precision, dx, dW, db)


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("s", [1e-8, 1e-4, 1.0, 1e4])
def test_gradient_scale(s, precision):
    L = level("ragged")
    x, W, b = make_layer(L.shape[0], 2, 128, 128, seed=10)
    dz = (np.random.default_rng(11).standard_normal((2, L.shape[0], 128)) * s).astype(np.float32)
    _, dx, dW, db, p = run(L, x, W, b, precision, dz)
    expect_tc(p, precision, 128, 128, L.shape[0])
    check_bwd(f"dz*{s:g}", L, x, W, dz, precision, dx, dW, db)


# ------------------------------------------------------------------------------------------------------- metamorphic
@pytest.mark.parametrize("precision", PRECISIONS)
def test_power_of_two_scaling_is_exact(precision):
    """With b = 0: conv(2^e x) == 2^e conv(x) and conv(x; 2^e W) == 2^e conv(x; W), bitwise, where fp32 itself neither
    underflows nor overflows."""
    L = level("tma")
    x, W, b = make_layer(L.shape[0], 2, 64, 64, seed=12, zero_bias=True)
    y = run(L, x, W, b, precision)[0]
    for e in (-12, -6, 6, 12):
        ys = run(L, (x * 2.0 ** e).astype(np.float32), W, b, precision)[0]
        assert np.array_equal(ys, y * 2.0 ** e), ("x", e)
        yw = run(L, x, (W * 2.0 ** e).astype(np.float32), b, precision)[0]
        assert np.array_equal(yw, y * 2.0 ** e), ("W", e)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_mesh_output_independent_of_batch_position(precision):
    """y(x)[b] == y(x[b:b+1])[0] and a permuted batch gives the permuted output, bitwise: a tile's K order does not
    depend on which CTA runs it or on what that CTA ran before (B = 40 meshes of 8 tiles: 2-3 tiles per CTA)."""
    L = level("tma")
    x, W, b = make_layer(L.shape[0], 40, 64, 128, seed=13)
    y = run(L, x, W, b, precision)[0]
    for i in (0, 1, 17, 39):
        assert np.array_equal(run(L, x[i:i + 1], W, b, precision)[0][0], y[i]), i
    perm = np.random.default_rng(14).permutation(40)
    assert np.array_equal(run(L, x[perm], W, b, precision)[0], y[perm])


# ------------------------------------------------------------------------------------------------------- dense GEMM
def _posenet(J, H, seed):
    from pose2mesh_release_b200.posenet import LinearModel

    torch.manual_seed(seed)
    m = LinearModel(J, H, num_stage=2, p_dropout=0.5)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for st in m.linear_stages:
            for bn in (st.batch_norm1, st.batch_norm2):
                bn.weight.copy_(torch.rand(H, generator=g) + 0.5)
                bn.bias.copy_(torch.randn(H, generator=g) * 0.5)
                bn.running_mean.copy_(torch.randn(H, generator=g) * 0.5)
                bn.running_var.copy_(torch.rand(H, generator=g) + 0.5)
    return m.to(dev()).eval()


POSENET = [(H, B, J) for H in (64, 128, 192) for B in (1, 127, 128, 129, 300) for J in (17, 24)] + \
          [(4096, B, J) for B in (1, 129) for J in (17, 24)]


@pytest.mark.parametrize("H,B,J", POSENET, ids=lambda v: str(v))
def test_posenet_dense_gemm(H, B, J):
    """p2m_posenet_forward: every H here is a multiple of 64, so the H x H GEMMs run on the tensor cores; 3J = 51 <= 64
    also puts the output layer there (zero-padded to 64 columns), 3J = 72 keeps it on the fp32 SIMT GEMM."""
    m = _posenet(J, H, seed=H + B + J)
    x = torch.randn(B, 2 * J, generator=torch.Generator().manual_seed(B))
    with torch.no_grad():
        y = m.forward_native(x.to(dev())).double().cpu().numpy()
    sd = {k: v.detach().cpu().numpy() for k, v in m.state_dict().items() if v.is_floating_point()}
    ref, bound = R.posenet_forward(sd, x.numpy(), 2, precision="fp16x3",
                                   last_precision="fp16x3" if 3 * J <= 64 else "fp32")
    check(f"posenet H={H} B={B} J={J}", "fp16x3", y, ref, bound)
