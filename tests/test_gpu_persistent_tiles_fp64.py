"""The tensor-core conv's persistent tile loop against float64, with CTAs running one to many tiles.

Every tensor-core conv, dW and dense-GEMM launch walks tiles blockIdx.x, blockIdx.x + gridDim.x, ... over a grid
of min(n_tiles, SMs / column slices), and carries state from one tile to the next: the A/B ring slots and their
mbarrier phases, the X / T1 stage counter, the double-buffered tile-metadata blob, in the 64 x 128 configuration the
tile alternation between the two MMA + epilogue warpgroups and the staging buffer they hand over, in the 64 x 256 mode
the two epilogues taking turns.  At the test sizes of the other modules a CTA mostly runs one tile, so
p2m_debug_set_sm_count caps the grid (as on a part with fewer SMs): the same kernels run, each CTA takes more tiles.
p2m_debug_conv_log reports which instantiation ran and with how many tiles per CTA.

1. Single layer (p2m_cheb_conv_fwd / _bwd): every kernel configuration at caps that give each CTA 1, 2, 3 and all
   (>= 8) of its launch's tiles, with grids that are multiples of and coprime to the level's tile-pattern count.
   y, dx, dW and db against fp64_ref's bounds at fp16x3, y at single-pass fp16.
2. The network schedules (eval at elision 0 / 1 / 2 with the fused head off and on, training forward and backward
   with and without dx) at caps 1 and 3, every layer from its captured inputs.
3. Coverage: every instantiation launch_n can select ran with >= 4 tiles on some CTA (see REACHABLE).

Metamorphic, needing no bound: a tile's K order does not depend on which CTA or warpgroup runs it, so y, dx and every
captured activation are bitwise equal across caps and to the uncapped run.  The weight gradients are reduced across
CTAs and are held to their bounds only.  Every case asserts kernel_status == 0."""
import math

import numpy as np
import pytest
import torch

import fp64_ref as R
import graphs as G
from helpers import graph_from_fixture

pytestmark = pytest.mark.gpu

# (kind, output columns per CTA, ring slots, X / T1 stages, MODE, single-pass fp16) -> most tiles one CTA ran
_SEEN = {}
_RAN = set()


def dev():
    return torch.device("cuda:0")


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def lib():
    from pose2mesh_release_b200 import _lib

    return _lib


@pytest.fixture(scope="module", autouse=True)
def _fresh_log():
    clear_log()   # launches of earlier modules count for nothing here


def clear_log():
    lib().load().p2m_debug_conv_log_reset()


def read_log():
    """The launches logged since the last read or clear (the log is reset), recorded into _SEEN."""
    log = lib().conv_log(reset=True)
    for e in log:
        k = (e["kind"], e["nc"], e["ns"], e["xs"], e["mode"], e["f16"])
        _SEEN[k] = max(_SEEN.get(k, 0), e["tiles_per_cta"])
    return log


def same_launches(a, b):
    """Two runs issued the same kernels on the same tiles (only grid.x differs)."""
    strip = lambda log: [tuple(v for k, v in e.items() if k not in ("grid_x", "tiles_per_cta")) for e in log]
    return strip(a) == strip(b)


# ----------------------------------------------------------------------------------------------------- 1. one layer
def level(name):
    if name in ("tma", "ragged"):
        fx, i = {"tma": ("smpl_small", 1), "ragged": ("mano_like", 0)}[name]
        return graph_from_fixture(fx)[0][i]
    return G.get(name)


def make_layer(V, B, fin, fout, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((B, V, fin)).astype(np.float32)
    W = ((rng.random((fout, 3 * fin)) * 2 - 1) * np.sqrt(2.0 / (3 * fin + fout))).astype(np.float32)
    b = (rng.standard_normal(fout) * 0.1).astype(np.float32)
    dz = rng.standard_normal((B, V, fout)).astype(np.float32)
    return x, W, b, dz


def run_layer(L, x, W, b, precision, cap, dz=None):
    """The layer on the GPU with the grid capped at `cap` SMs (0 = none): (y, dx, dW, db, log) as float64 numpy."""
    from pose2mesh_release_b200 import cheby_graph_conv as cgc

    _lib = lib()
    cgc.set_default_precision(precision)
    gh = cgc.graph_handle(L)
    h = gh.handle(0)
    try:
        _lib.check(_lib.load().p2m_debug_set_sm_count(h, cap), "set_sm_count")
        clear_log()
        xg = torch.as_tensor(x).to(dev()).requires_grad_(dz is not None)
        Wg = torch.as_tensor(W).to(dev()).requires_grad_(dz is not None)
        bg = torch.as_tensor(b).to(dev()).requires_grad_(dz is not None)
        with torch.set_grad_enabled(dz is not None):
            y = cgc.ChebConvLinear.apply(xg, Wg, bg, gh)
        grads = (None, None, None)
        if dz is not None:
            y.backward(torch.as_tensor(dz).to(dev()))
            grads = tuple(t.grad.double().cpu().numpy() for t in (xg, Wg, bg))
        torch.cuda.synchronize()
        assert gh.kernel_status(0) == 0, "a tensor-core kernel timed out on an mbarrier"
        log = read_log()
    finally:
        _lib.check(_lib.load().p2m_debug_set_sm_count(h, 0), "set_sm_count")
        cgc.set_default_precision("fp16x3")
    return (y.detach().double().cpu().numpy(),) + grads + (log,)


def grids(n_tiles, n_slices, P):
    """grid.x values that give each CTA 1, 2, 3 and all of the launch's tiles, one a multiple of the tile-pattern count
    P (every CTA sees the same blob sizes tile after tile) and one coprime to it (they change)."""
    gmax = min(sms() // n_slices, n_tiles)
    out = {min(gmax, math.ceil(n_tiles / k)) for k in (1, 2, 3)} | {1}
    if P <= gmax:
        out.add(P * max(1, min(gmax // P, n_tiles // P // 2)))
    out.add(next(g for g in range(2, gmax + 1) if math.gcd(g, P) == 1))
    return sorted(out)


# (id, level, fin, fout, B, precision, backward, forward conv's (columns per CTA, ring slots, T1 stages))
LAYERS = [
    ("128x64 64->64", "V128", 64, 64, 12, "fp16x3", True, (64, 3, 2)),
    ("128x64 96->64 ragged", "ragged", 96, 64, 3, "fp16x3", True, (64, 3, 2)),
    ("128x64 64->64 one X stage", "band16", 64, 64, 2, "fp16x3", True, (64, 3, 1)),
    ("64x128 128->128", "tma", 128, 128, 2, "fp16x3", True, (128, 6, 2)),
    ("64x128 32->128 ragged", "ragged", 32, 128, 2, "fp16x3", True, (128, 6, 2)),   # 3 K-blocks: half the ring
    ("64x128 128->128 one T1 stage", "band14", 128, 128, 2, "fp16x3", True, (128, 6, 1)),
    ("64x128 128->128 ring of 3", "band18", 128, 128, 2, "fp16x3", True, (128, 3, 2)),
    ("64x128 128->128 ring of 3 one T1 stage", "clique12", 128, 128, 4, "fp16x3", True, (128, 3, 1)),
    # and its backward's dT GEMMs (plain, 128 columns) with a ring of 3 and one X stage
    ("64x128 128->128 plain ring of 3 one X stage", "twoclique49", 128, 128, 6, "fp16x3", True, (128, 3, 1)),
    ("64x128 128->256 two slices", "tma", 128, 256, 2, "fp16x3", True, (128, 6, 2)),
    ("64x256 256->256", "tma", 256, 256, 2, "fp16x3", True, (256, 3, 2)),
    ("64x256 256->256 one T1 stage", "band21", 256, 256, 2, "fp16x3", True, (256, 3, 1)),
    ("fp16 128x64 64->64", "V128", 64, 64, 12, "fp16", False, (64, 3, 2)),
    ("fp16 128x64 96->64 ragged", "ragged", 96, 64, 3, "fp16", False, (64, 3, 2)),
    ("fp16 128x64 64->64 one X stage", "farband20", 64, 64, 3, "fp16", False, (64, 3, 1)),
    ("fp16 64x128 128->128", "tma", 128, 128, 2, "fp16", False, (128, 6, 2)),
    ("fp16 64x128 32->128 ragged", "ragged", 32, 128, 2, "fp16", False, (128, 6, 2)),
    ("fp16 64x128 128->128 one T1 stage", "clique12", 128, 128, 4, "fp16", False, (128, 6, 1)),
    ("fp16 64x128 128->256 two slices", "tma", 128, 256, 2, "fp16", False, (128, 6, 2)),
    ("fp16 64x256 256->256", "tma", 256, 256, 2, "fp16", False, (256, 3, 2)),
    ("fp16 64x256 256->256 one T1 stage", "clique14", 256, 256, 4, "fp16", False, (256, 3, 1)),
]


def layer_refs(L, x, W, b, dz, precision):
    """name -> (float64 reference, bound) of y and, with dz, of dx, dW and db, on the Laplacian's fp32 values as the
    device holds them."""
    L = L.tocsr().astype(np.float32).astype(np.float64)
    out = {"y": (R.cheb_conv_fwd(x, L, W, b), R.cheb_conv_fwd_bound(x, L, W, b, precision))}
    if dz is not None:
        refs = R.cheb_conv_bwd(x, L, W, dz)
        bounds = R.cheb_conv_bwd_bound(x, L, W, dz, precision)
        out.update(zip(("dx", "dW", "db"), zip(refs, bounds)))
    return out


def check_layer(tag, refs, got):
    for name, value in got.items():
        ref, bound = refs[name]
        r = R.bound_ratio(value, ref, bound)
        assert r <= 1.0, f"{tag} {name}: max |err| / bound = {r:.3g}"


@pytest.mark.parametrize("case", LAYERS, ids=lambda c: c[0])
def test_single_layer_tiles_per_cta(case):
    """The uncapped run against float64; at every grid, y and dx bitwise equal to it and dW, db (reduced across
    CTAs) against float64."""
    tag, lvl, fin, fout, B, precision, bwd, tiling = case
    L = level(lvl)
    V = L.shape[0]
    x, W, b, dz = make_layer(V, B, fin, fout, seed=V + fin * 7 + fout)
    dz = dz if bwd else None
    y0, dx0, dW0, db0, log0 = run_layer(L, x, W, b, precision, 0, dz)
    conv0 = next(e for e in log0 if e["kind"] == "conv")
    assert (conv0["nc"], conv0["ns"], conv0["xs"], conv0["mode"], conv0["f16"]) == \
        tiling + (1, int(precision == "fp16")), (tag, conv0)
    n_tiles, n_slices = conv0["n_tiles"], conv0["grid_y"]
    P = n_tiles // B
    refs = layer_refs(L, x, W, b, dz, precision)
    check_layer(f"{tag} uncapped", refs, dict(y=y0, dx=dx0, dW=dW0, db=db0) if bwd else dict(y=y0))
    per_cta = set()
    for g in grids(n_tiles, n_slices, P):
        y, dx, dW, db, log = run_layer(L, x, W, b, precision, g * n_slices, dz)
        conv = next(e for e in log if e["kind"] == "conv")
        assert conv["grid_x"] == g and conv["tiles_per_cta"] == math.ceil(n_tiles / g), (tag, g, conv)
        assert same_launches(log, log0), (tag, g)
        per_cta.add(conv["tiles_per_cta"])
        t = f"{tag} grid {g} ({conv['tiles_per_cta']} tiles per CTA)"
        assert np.array_equal(y, y0), t + ": y differs from the uncapped run"
        if bwd:
            assert np.array_equal(dx, dx0), t + ": dx differs from the uncapped run"
            check_layer(t, refs, dict(dW=dW, db=db))
    assert {1, 2, 3} <= per_cta and max(per_cta) >= 8, (tag, sorted(per_cta))
    _RAN.add(tag)


# ---------------------------------------------------------------------------------------------- 2. network schedules
NETS = ["custom", "mano_like", "smpl_small"]
CAPS = (1, 3)


def set_cap(net, cap):
    net.hier.set_debug(0, sm_count=cap)


def captured_equal(tag, a, b):
    """Every captured tensor of two runs bitwise equal (lists: per layer, None where not captured)."""
    assert a.keys() == b.keys()
    for k in a:
        va, vb = a[k], b[k]
        if isinstance(va, list):
            for li, (ta, tb) in enumerate(zip(va, vb)):
                # (equal_nan: a layer whose output the fused head replaced is never written)
                assert (ta is None) == (tb is None) and (ta is None or np.array_equal(ta, tb, equal_nan=True)), \
                    (tag, k, li)
        else:
            assert np.array_equal(va, vb, equal_nan=True), (tag, k)


@pytest.mark.parametrize("precision", ["fp16x3", "fp16"])
@pytest.mark.parametrize("name", NETS)
def test_eval_network_capped(name, precision):
    """Eval forward at elision 0 / 1 / 2, fused head off and on, dedup off: at caps 1 and 3 every captured layer output
    and the result are bitwise those of the uncapped run; at cap 1 every layer is checked against float64."""
    import test_gpu_network_fp64 as N

    B = 3
    net = N.Net(name, precision, seed=41, open_relus=False)
    try:
        for elide in (0, 1, 2):
            x, _ = N.train_inputs(net, B, seed=7 + elide)
            tag = f"{name} {precision} eval elide={elide}"
            base = {}
            for cap in (0,) + CAPS:
                set_cap(net, cap)
                for fuse in (False, True):
                    clear_log()
                    y, c = N.forward_eval(net, x, elide, dedup=False, fuse=fuse)
                    log = read_log()
                    if cap == 0:
                        base[fuse] = (y, c, log)
                        continue
                    t = f"{tag} fuse={fuse} cap={cap}"
                    assert same_launches(log, base[fuse][2]), t
                    assert all(e["grid_x"] <= cap for e in log), t
                    assert np.array_equal(y, base[fuse][0]), t + ": y differs from the uncapped run"
                    captured_equal(t, c, base[fuse][1])
                if cap == 1:
                    N.check_eval(net, f"{tag} cap=1", x, elide)
    finally:
        set_cap(net, 0)
    assert net.hier.kernel_status(0) == 0
    _RAN.add(("eval", name, precision))


@pytest.mark.parametrize("need_dx", [True, False])
@pytest.mark.parametrize("name", NETS)
def test_train_network_capped(name, need_dx):
    """Training forward and backward at fp16x3 (open ReLUs): at caps 1 and 3 every captured forward and backward tensor
    (z, a, fc_out, g_a, g_z, dx, fc_dx) and y are bitwise those of the uncapped run, and every layer, weight
    gradients included, is checked against float64 (the weight gradients are reduced across CTAs)."""
    import test_gpu_network_fp64 as N

    B = 3
    net = N.Net(name, "fp16x3", seed=53, open_relus=True)
    x, tgt = N.train_inputs(net, B, seed=11)
    try:
        clear_log()
        cap0, _, _, y0 = N.forward_train_backward(net, x, tgt, need_dx)
        log0 = read_log()
        for cap in CAPS:
            set_cap(net, cap)
            # a capped CTA accumulates a dW element over the rows of many tiles in fp32, where dW's partial sums keep
            # one sign: fp64_ref's sqrt-growth accumulation term (a grid of many CTAs) need not hold there, n u of
            # that chain does (N.dw_chain, per layer)
            net.sm_cap = cap
            c, grads, bufs, y = N.forward_train_backward(net, x, tgt, need_dx)
            log = read_log()
            t = f"{name} train dx={need_dx} cap={cap}"
            assert same_launches(log, log0), t
            assert np.array_equal(y, y0), t + ": y differs from the uncapped run"
            captured_equal(t, c, cap0)
            N.check_train(net, t, x, y, c, grads, bufs, need_dx)
    finally:
        set_cap(net, 0)
        net.sm_cap = 0
    assert net.hier.kernel_status(0) == 0
    _RAN.add(("train", name, need_dx))


# ----------------------------------------------------------------------------------------------------- 3. coverage
# Every (kind, columns per CTA, ring slots, X / T1 stages, MODE, fp16) launch_n and launch_umma_dw can select, derived
# from conv_cfg / conv_cols over conv_smem (and dw_smem) for staged-row counts and blob sizes up to
# umma_conv_supported's limits, and confirmed from the log of the graphs above.  Left out:
# - (conv, 64, 3, 1, MODE 0): the plain 128 x 64 GEMM always gets two X stages.  A supported level has
#   conv_smem(64, 3, 1, MODE 1) <= 227 KB, and that is the plain size with one stage plus max_h1 * 128 bytes of T1
#   stage, max_h1 >= 128 rows: at least the 16 KB a second X stage of the plain GEMM needs.
# - single-pass fp16 at MODE 0 with fewer than the most slots and stages: its only plain GEMM is the isolated rows'
#   combined-weight GEMM, whose tiles stage their own rows only (one CSR entry per row).
# - the 64 x 256 mode at MODE 0: conv_cols takes it for T1-given convs only.
# - single-pass fp16 with the 64 x 128 ring of 3 (k_cheb_conv_f16_wide<128, 3, *, *>, either MODE): dead code on the
#   consecutive tiles.  Six fp16 slots, 6 (64 + 128) 64 B, are the 73728 B of three fp16x3 slots, and the only other
#   term of conv_smem that depends on the slot count is the barrier map, 8 (2 NS + 2 XS + 6): 48 B more at NS = 6.
#   Every other term is a multiple of 128 B, and the fixed small ones (barriers at NS = 3, XS = 1: 112; flags 16;
#   residual mbarriers 32; slack 1184) sum to 1344 = 64 mod 128, so conv_smem(128, 3, 1, MODE) <= 227 KB, which
#   umma_conv_supported requires at fp16x3, means <= 227 KB - 64, and six fp16 slots with one stage fit with 16 B to
#   spare: conv_cfg never goes below six.  build_umma_level_meta holds the padding elision's index-list tiles to the
#   same limit, so those instantiations are not built (cheb_umma.cu: launchable).
REACHABLE = {
    ("conv", 64, 3, 2, 1, 0), ("conv", 64, 3, 1, 1, 0), ("conv", 128, 6, 2, 1, 0), ("conv", 128, 6, 1, 1, 0),
    ("conv", 128, 3, 2, 1, 0), ("conv", 128, 3, 1, 1, 0), ("conv", 256, 3, 2, 1, 0), ("conv", 256, 3, 1, 1, 0),
    ("conv", 64, 3, 2, 0, 0), ("conv", 128, 6, 2, 0, 0), ("conv", 128, 6, 1, 0, 0), ("conv", 128, 3, 2, 0, 0),
    ("conv", 128, 3, 1, 0, 0),
    ("conv", 64, 3, 2, 1, 1), ("conv", 64, 3, 1, 1, 1), ("conv", 128, 6, 2, 1, 1), ("conv", 128, 6, 1, 1, 1),
    ("conv", 256, 3, 2, 1, 1), ("conv", 256, 3, 1, 1, 1),
    ("conv", 64, 3, 2, 0, 1), ("conv", 128, 6, 2, 0, 1),
    ("dw", 64, 3, 2, 1, 0), ("dw", 64, 3, 1, 1, 0),
}


def test_every_instantiation_ran_multi_tile():
    """Over this module's cases: every reachable instantiation ran with >= 4 tiles on one CTA (with 64 x 128 tile
    alternation: >= 2 on each MMA warpgroup)."""
    if len(_RAN) < len(LAYERS) + 2 * len(NETS) * 2:
        pytest.skip("reads the launches of the module's other tests: run the whole module")
    print("tiles per CTA:", {k: _SEEN[k] for k in sorted(_SEEN)})
    short = {k: _SEEN.get(k, 0) for k in REACHABLE if _SEEN.get(k, 0) < 4}
    assert not short, f"ran with fewer than 4 tiles on every CTA (0 = never ran): {short}"
    unknown = {k for k in _SEEN if k[0] != "gemm"} - REACHABLE
    assert not unknown, f"instantiations outside REACHABLE ran: {unknown}"
