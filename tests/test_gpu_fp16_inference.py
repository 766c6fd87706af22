"""The single-pass fp16 precision (P2M_PREC_FP16_TC, inference only) on the device.

1. Single layer (p2m_cheb_conv_fwd) against float64: every width of the three kernel configurations (128 x 64,
   64 x 128, 64 x 256), the graph families of tests/graphs.py, the persistent CTA loop.  Every element lies within
   fp64_ref's bound at "fp16" (SPLIT16 = 2^-10 + 2^-22), and at least one element of each case lies beyond
   the fp16x3 bound: the single pass is what ran.
2. The eval network layer by layer (test_gpu_network_fp64.check_eval on an fp16 net), each layer from its own captured
   input: elision 0 / 1 / 2 (index-list tiles and the isolated rows' combined-weight GEMM), the virtual unpool,
   residuals, the fused head, dedup.
3. Full size (SMPL hierarchy, B = 256): finite, two runs, forward_vertices and CUDA-graph replay equal to the plain
   forward bit for bit, batch split and elision / dedup within a tolerance derived from SPLIT16, the per-mesh deviation
   from the float64 oracle on test_gpu_parity's 32-mesh sample (written to P2M_FP16_REPORT if set).
4. Refusal: training forwards and backwards raise and leave the BatchNorm running statistics untouched; back at fp16x3
   the results are bitwise those of a model that never left it.
Every test ends with kernel_status == 0."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

import fp64_ref as R
import graphs as G
from helpers import CASES, graph_from_fixture

pytestmark = pytest.mark.gpu


def dev():
    return torch.device("cuda:0")


def level(name):
    fx, i = {"tma": ("smpl_small", 1), "ragged": ("mano_like", 0)}[name]
    return graph_from_fixture(fx)[0][i]


def make_layer(V, B, fin, fout, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((B, V, fin)).astype(np.float32)
    W = ((rng.random((fout, 3 * fin)) * 2 - 1) * np.sqrt(2.0 / (3 * fin + fout))).astype(np.float32)
    b = (rng.standard_normal(fout) * 0.1).astype(np.float32)
    return x, W, b


def conv_info(gh, fin, fout):
    from pose2mesh_release_b200 import _lib

    lib = _lib.load()
    path, til = (C.c_int32 * 9)(), (C.c_int32 * 3)()
    _lib.check(lib.p2m_debug_conv_path(gh.handle(0), 0, fin, fout, path), "conv_path")
    _lib.check(lib.p2m_debug_conv_tiling(gh.handle(0), 0, fin, fout, til), "conv_tiling")
    return int(path[0]), tuple(til)


def run_layer(L, x, W, b, sm_cap=0):
    """p2m_cheb_conv_fwd at fp16: (y as float64, on tensor cores, (cols, ns, xs)).  sm_cap > 0: the persistent
    tensor-core grids are sized for that many SMs (p2m_debug_set_sm_count)."""
    from pose2mesh_release_b200 import _lib
    from pose2mesh_release_b200 import cheby_graph_conv as cgc

    cgc.set_default_precision("fp16")
    gh = cgc.graph_handle(L)
    try:
        _lib.check(_lib.load().p2m_debug_set_sm_count(gh.handle(0), sm_cap), "set_sm_count")
        with torch.no_grad():
            y = cgc.ChebConvLinear.apply(torch.as_tensor(x).to(dev()), torch.as_tensor(W).to(dev()),
                                         torch.as_tensor(b).to(dev()), gh)
        torch.cuda.synchronize()
        assert gh.kernel_status(0) == 0, "a tensor-core kernel timed out on an mbarrier"
        tc, til = conv_info(gh, x.shape[2], W.shape[0])
    finally:
        _lib.check(_lib.load().p2m_debug_set_sm_count(gh.handle(0), 0), "set_sm_count")
        cgc.set_default_precision("fp16x3")
    return y.double().cpu().numpy(), tc, til


def check_single_pass(tag, L, x, W, b, y, on_tc=True):
    L = L.tocsr().astype(np.float32).astype(np.float64)
    ref = R.cheb_conv_fwd(x, L, W, b)
    err = np.abs(y - ref)
    r16 = float((err / R.cheb_conv_fwd_bound(x, L, W, b, "fp16")).max())
    assert r16 <= 1.0, f"{tag}: max |err| / fp16 bound = {r16:.3g}"
    if on_tc:
        r3 = float((err / R.cheb_conv_fwd_bound(x, L, W, b, "fp16x3")).max())
        assert r3 > 1.0, f"{tag}: within the fp16x3 bound ({r3:.3g}): the single pass did not run"


# ------------------------------------------------------------------------------------------------------ 1. one layer
WIDTHS = [(fin, fout) for fin in (32, 64, 96, 128, 160, 192, 224, 256) for fout in (64, 128, 256)]


@pytest.mark.parametrize("lvl", ["tma", "ragged"])
@pytest.mark.parametrize("fin,fout", WIDTHS, ids=lambda v: str(v))
def test_single_layer_width_grid(fin, fout, lvl):
    L = level(lvl)
    x, W, b = make_layer(L.shape[0], 1, fin, fout, seed=fin * 1000 + fout)
    y, tc, til = run_layer(L, x, W, b)
    assert tc == 1
    assert til[0] == (256 if fin == fout == 256 else (64 if fout == 64 else 128)), til
    check_single_pass(f"width {fin}->{fout} {lvl}", L, x, W, b, y)


SYMMETRIC_FAMILIES = ["V1", "V64", "V127", "V128", "V129", "V1088", "V2048", "band8", "band12", "band14", "band16",
                      "band20", "h1_256", "h1_257", "far", "hub", "empty_rows", "iso_uniform", "iso_two_diag", "dense"]


@pytest.mark.parametrize("fin,fout", [(64, 64), (128, 128), (256, 256)], ids=lambda v: str(v))
@pytest.mark.parametrize("name", SYMMETRIC_FAMILIES)
def test_single_layer_graph_family(name, fin, fout):
    L = G.get(name)
    x, W, b = make_layer(L.shape[0], 2, fin, fout, seed=L.shape[0] + fin)
    y, tc, _ = run_layer(L, x, W, b)
    check_single_pass(f"{name} {fin}->{fout}", L, x, W, b, y, on_tc=bool(tc))


@pytest.mark.parametrize("fin,fout", [(64, 64), (128, 128), (256, 256)], ids=lambda v: str(v))
def test_single_layer_persistent_cta_loop(fin, fout):
    """V = 128: n_tiles = B (128 x 64) or 2 B (64-row tiles; 256 -> 256 in the 64 x 256 mode, one column slice), on a
    grid capped at 8 SMs (grid.x = min(n_tiles, 8), read back from the launch log): B = 1, 7, 9 and 29 make each CTA
    run from 1 to 8 tiles.
    tests/test_gpu_persistent_tiles_fp64.py covers every configuration."""
    from pose2mesh_release_b200 import _lib

    L = G.get("V128")
    grid = 8
    most = 0
    for B in (1, 7, 9, 29):
        x, W, b = make_layer(128, B, fin, fout, seed=B)
        _lib.conv_log(reset=True)
        y, tc, _ = run_layer(L, x, W, b, sm_cap=grid)
        conv = next(e for e in _lib.conv_log(reset=True) if e["kind"] == "conv")
        assert conv["grid_x"] == min(conv["n_tiles"], max(1, grid // conv["grid_y"])) and conv["f16"] == 1, conv
        most = max(most, conv["tiles_per_cta"])
        assert tc == 1
        check_single_pass(f"persistent B={B} {fin}->{fout}", L, x, W, b, y)
    assert most >= 4, most


# ------------------------------------------------------------------------------------------- 2. network, layer by layer
EVAL_CASES = [(name, elide, B) for name in ("smpl_small", "mano_like", "custom") for elide, B in ((0, 3), (1, 1), (2, 3))]


@pytest.mark.parametrize("name,elide,B", EVAL_CASES, ids=lambda v: str(v))
def test_eval_network_layer_by_layer(name, elide, B):
    import test_gpu_network_fp64 as N

    net = N.Net(name, "fp16", seed=31 + B + elide, open_relus=False)
    x, _ = N.train_inputs(net, B, seed=5 + elide)
    tag = f"{name} fp16 eval elide={elide} B={B}"
    y, yf, act, fc_out = N.check_eval(net, tag, x, elide)
    # at least one tensor-core layer beyond the fp16x3 bound: the single pass is what ran
    beyond = 0
    for li in range(net.n_layers):
        if net.route(li, B)["tc"]:
            inp, block_in = N.layer_input(net, li, x, fc_out, act)
            ref, b3 = N.eval_layer(net, li, inp, block_in, "fp16x3")
            beyond += int((np.abs(act[li] - ref) > b3).any())
    assert beyond >= 1, f"{tag}: no tensor-core layer beyond the fp16x3 bound"
    # dedup on against off: the representative rows are computed by the same GEMM, bit for bit
    for fuse in (False, True):
        yd, _ = N.forward_eval(net, x, elide, dedup=True, fuse=fuse, capture=False)
        assert np.array_equal(yd, y if not fuse else yf), (tag, "dedup", fuse)
    assert net.hier.kernel_status(0) == 0


# ------------------------------------------------------------------------------------------------- 3. full size
def smpl_model(precision):
    from oracle import meshnet_oracle as mo
    from pose2mesh_release_b200 import graph as pg
    from pose2mesh_release_b200.meshnet import Pose2Mesh

    n, seed, levels, _ = CASES["smpl_like"]
    face = pg.synthetic_sphere_faces(n, seed)
    _, graph_L, _, perm_rev = pg.build_coarse_graphs(face, 17, pg.H36M_SKELETON, pg.H36M_FLIP_PAIRS, levels=levels)
    torch.manual_seed(123)
    model = Pose2Mesh(5, 3, graph_L, joint_set="human36")
    sd = mo.randomize_bn_({k: v.detach().clone() for k, v in model.state_dict().items()}, seed=7)
    model.load_state_dict(sd)
    return model.to(dev()).set_precision(precision).eval(), sd, graph_L, perm_rev, n


def per_mesh(y, ref):
    y, ref = y.detach().double().cpu(), ref.detach().double().cpu()
    d = (y - ref).abs().flatten(1).max(dim=1).values
    s = ref.abs().flatten(1).max(dim=1).values.clamp_min(1e-30)
    return d / s


# Two fp16 forwards of one mesh that round differently: elision and dedup change how the isolated rows' weights are
# rounded (the combined W0 + c W1 + (2c^2 - 1) W2 once, not each order), and a batch split changes the fc's operand
# scale (found over the whole batch: its outputs may differ in the last bits, which the next conv's fp16 rounding can
# turn into one fp16 step).  Per layer the two differ by at most the two forwards' rounding, 2 SPLIT16 relative,
# compounded through the 21 layers of the SMPL plan at O(1) gain per layer: 21 * 2 * SPLIT16 = 4.1e-2 per mesh of
# max|y| is the ceiling.  (fp16x3 holds a batch split to 1e-6: its split keeps those last bits.)
ROUNDING_TOL = 21 * 2 * R.SPLIT16
PARITY_CEILING = 5e-2   # a chosen limit against layout or indexing bugs, not a derived bound
PICK = sorted({0, 1, 2, 3, 36, 37, 73, 74, 110, 111, 127, 128, 131, 147, 148, 149, 184, 185, 221, 222, 254, 255}
              | set(range(9, 256, 25)) | {200})


def test_full_size_smpl_b256():
    from oracle import meshnet_oracle as mo

    model, sd, graph_L, perm_rev, n = smpl_model("fp16")
    hier, d = model._hier, torch.cuda.current_device()
    B = 256
    x = torch.randn(B, 17, 5, generator=torch.Generator().manual_seed(0)).to(dev())
    with torch.no_grad():
        y = model(x)
        y2 = model(x)
        y_split = torch.cat([model(x[:100]), model(x[100:])])
        verts = model.forward_vertices(x, perm_rev, n)
    assert y.shape == (B, 12288, 3) and torch.isfinite(y).all()
    assert torch.equal(y, y2), "two runs differ"
    assert float(per_mesh(y_split, y).max()) < ROUNDING_TOL
    real = torch.as_tensor(np.asarray(perm_rev[:n])).to(dev())
    assert torch.equal(verts, y[:, real])
    # CUDA-graph replay equals eager
    xs = x.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.no_grad():
        model(xs)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g), torch.no_grad():
        yg = model(xs)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(yg, y), "CUDA-graph replay differs from the eager forward"
    # elision 0 / 2 and dedup off against the default
    try:
        for mode, dedup in ((0, True), (2, True), (1, False)):
            hier.set_debug(d, elide_padding=mode, dedup_padding=dedup)
            with torch.no_grad():
                ym = model(x)
            assert float(per_mesh(ym, y).max()) < ROUNDING_TOL, (mode, dedup)
    finally:
        hier.set_debug(d, elide_padding=1, dedup_padding=True)
    # per-mesh deviation from the float64 oracle on test_gpu_parity's sample
    laps = [t.to(torch.float64) for t in mo.laplacians_to_torch(graph_L)]
    sd64 = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
    with torch.no_grad():
        yo = mo.forward(sd64, laps, x[PICK].cpu().double(), training=False)
    dev_mesh = per_mesh(y[PICK], yo)
    with torch.no_grad():
        y3 = smpl_model("fp16x3")[0](x)
    dev_x3 = per_mesh(y, y3)
    out = os.environ.get("P2M_FP16_REPORT")
    if out:
        with open(out, "w") as f:
            json.dump({"per_mesh_vs_fp64_oracle": {"max": float(dev_mesh.max()), "median": float(dev_mesh.median()),
                                                   "all": [float(v) for v in dev_mesh]},
                       "per_mesh_vs_fp16x3": {"max": float(dev_x3.max()), "median": float(dev_x3.median())},
                       "meshes": PICK}, f, indent=1)
    assert float(dev_mesh.max()) < PARITY_CEILING, float(dev_mesh.max())
    assert float(dev_x3.max()) > 1e-5, "fp16 and fp16x3 agree to fp16x3 accuracy: the single pass did not run"
    assert hier.kernel_status(d) == 0


# --------------------------------------------------------------------------------------------------- 4. refusal
def test_training_and_backward_refused():
    from pose2mesh_release_b200 import cheby_graph_conv as cgc
    from pose2mesh_release_b200.meshnet import Pose2Mesh

    mats, _ = graph_from_fixture("smpl_small")
    torch.manual_seed(5)
    ref = Pose2Mesh(5, 3, mats, joint_set="human36").to(dev()).set_precision("fp16x3")
    torch.manual_seed(5)
    model = Pose2Mesh(5, 3, mats, joint_set="human36").to(dev()).set_precision("fp16")
    x = torch.randn(4, 17, 5, generator=torch.Generator().manual_seed(1)).to(dev())
    before = {k: v.clone() for k, v in model.state_dict().items()}
    buffers = dict(model.named_buffers())
    # module: a train-mode forward
    model.train()
    with pytest.raises(RuntimeError, match="fp16"):
        model(x)
    # module: a backward (of a train-mode forward taken at fp16x3, called after switching to fp16)
    model.set_precision("fp16x3")
    y = model(x)
    with torch.no_grad():                       # that forward did update the running statistics: restore them
        for k, v in buffers.items():
            v.copy_(before[k])
    model.set_precision("fp16")
    with pytest.raises(RuntimeError, match="fp16"):
        y.sum().backward()
    for k, v in model.state_dict().items():
        assert torch.equal(v, before[k]), k
    # single-layer functional: a training-mode BatchNorm, and a backward
    L = mats[1]
    V = L.shape[0]
    cl = torch.nn.Linear(3 * 64, 64).to(dev())
    bn = torch.nn.BatchNorm1d(64).to(dev()).train()
    bn_before = {k: v.clone() for k, v in bn.state_dict().items()}
    xi = torch.randn(2, V, 64, device=dev(), requires_grad=True)
    cgc.set_default_precision("fp16")
    try:
        with pytest.raises(RuntimeError, match="fp16"):
            cgc.graph_conv_cheby(xi, cl, bn, L, 64, 3)
        yi = cgc.graph_conv_cheby(xi, cl, None, L, 64, 3)
        with pytest.raises(RuntimeError, match="fp16"):
            yi.sum().backward()
        assert cgc.graph_handle(L).kernel_status(0) == 0
    finally:
        cgc.set_default_precision("fp16x3")
    for k, v in bn.state_dict().items():
        assert torch.equal(v, bn_before[k]), k
    # back at fp16x3: bitwise the model that never left it
    model.set_precision("fp16x3").eval()
    ref.eval()
    with torch.no_grad():
        assert torch.equal(model(x), ref(x))
    assert model._hier.kernel_status(0) == 0
