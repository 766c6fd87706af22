"""Padding-vertex elision's index-list tiles against float64, at their shared-memory limits.

Where a level's isolated rows are elided, a tensor-core conv runs its connected rows on DevLevel::real_tiles (the
connected rows packed 128 and 64 to a tile) and its isolated rows through a plain GEMM on iso_tiles, or on the class
representatives' rep_tiles (eval with dedup); backward-data does the same on dz.  A connected-row tile carries a larger
halo and metadata blob than the consecutive tiles, which hold the isolated rows too, so it reaches configurations of
launch_n the consecutive tiles do not, and past the shared-memory limit build_umma_level_meta keeps no families and the
level runs on its consecutive tiles.

Each hierarchy of graphs.ELISION (a padded level, a level of half its size, the joint graph) runs the network schedules
of test_gpu_network_fp64 (eval with the fused head off and on and dedup off and on, the training forward and backward
with dX) at elision 0, 1 and 2, with the persistent grids at the device's SM count and capped, so that CTAs run several
index-list tiles.  Every captured layer is held to fp64_ref's bounds from its own captured inputs.  Each
case asserts its routes (p2m_debug_layer_route) against the elision rule, and the conv log against the configurations
p2m_debug_tile_families reports for the family each elided conv runs on."""
import numpy as np
import pytest
import torch

import graphs as G
import test_gpu_network_fp64 as N

pytestmark = pytest.mark.gpu

FAMILIES = list(G.ELISION)
# (kind, output columns per CTA, ring slots, X / T1 stages, MODE, fp16) -> most tiles one CTA ran on index-list tiles
_SEEN = {}
_RAN = set()
CAP = 3   # SMs of the capped grids: each CTA runs several of a launch's tiles


def lib():
    from pose2mesh_release_b200 import _lib

    return _lib


def families(net, level, fin, fout):
    return lib().tile_families(net.hier.handle(0), level, fin, fout)


def elided(mode, n_iso, V, rows, width):
    """p2m_api.cu's elided(): the rule the network schedules route a conv by."""
    return mode > 0 and n_iso > 0 and rows >= 2 * width and (mode >= 2 or 5 * n_iso >= 2 * V)


def n_iso(net, level):
    """The level's isolated rows if it has the tile families (else 0: nothing to elide)."""
    f = families(net, level, 64, 64)
    if f["real"][128]["n_pattern"] == 0:
        return 0
    L = net.levels[level].tocsr()
    one = np.diff(L.indptr) == 1
    return int(np.count_nonzero(one & (L.indices[L.indptr[:-1]] == np.arange(L.shape[0]))))


def conv_cfg(net, level, fin, fout, family, cfg):
    """(columns per CTA, ring slots, X stages) the hook reports for a conv fin -> fout on `family`'s tiles."""
    f = families(net, level, fin, fout)[family]
    return f[128 if fout == 64 else 64][cfg]


def check_routes(net, tag, B, mode, need_dx=True, train=False):
    """Every layer's route against the elision rule; returns the (family, cfg) configurations the elided convs must
    have launched with, as conv-log keys."""
    want = set()
    f16 = int(net.precision == "fp16")
    for li, L in enumerate(net.layers):
        lvl, V = L["level"], net.V(li)
        r = net.route(li, B, need_dx)
        ni = n_iso(net, lvl)
        assert r["elide"] == (r["tc"] and elided(mode, ni, V, B * V, L["fout"])), (tag, li, r)
        if train:
            assert r["dx_elide"] == (r["tc_dx"] and elided(mode, ni, V, B * V, L["fin"])), (tag, li, r)
        prec = "fp16" if f16 else "fp16x3"
        if r["elide"]:
            nc, ns, xs = conv_cfg(net, lvl, L["fin"], L["fout"], "real", "t1_" + prec)
            assert ns > 0, (tag, li, "elided onto a family that does not fit")
            want.add(("conv", nc, ns, xs, 1, f16))
        if train and r["dx_elide"]:
            nc, ns, xs = conv_cfg(net, lvl, L["fout"], L["fin"], "real", "t1_fp16x3")
            want.add(("conv", nc, ns, xs, 1, 0))
    return want


def read_log(tag, want, capped):
    log = lib().conv_log(reset=True)
    got = {}
    for e in log:
        k = (e["kind"], e["nc"], e["ns"], e["xs"], e["mode"], e["f16"])
        got[k] = max(got.get(k, 0), e["tiles_per_cta"])
    missing = want - set(got)
    assert not missing, (tag, "elided convs did not launch with the configurations their family reports", missing)
    if capped:
        for k in want:
            _SEEN[k] = max(_SEEN.get(k, 0), got[k])
        for k, v in got.items():   # the isolated rows' plain GEMMs (MODE 0 on iso_tiles / rep_tiles)
            if k[0] == "conv" and k[4] == 0 and want:
                _SEEN[k] = max(_SEEN.get(k, 0), v)
    return log


# ------------------------------------------------------------------------------------------------- the families
# family -> the padded level's (real_tiles at 128 rows: n_pattern, max_h1), and per conv (fin, fout) the T1-given
# fp16x3 configuration on its connected-row tiles; None: build_umma_level_meta keeps no families
EXPECT = {
    "el_h1_256": ((4, 256), {(256, 64): (64, 3, 2), (128, 256): (128, 6, 2)}),
    "el_h1_257": None,
    "el_clique24": ((4, 145), {(128, 256): (128, 6, 1), (256, 64): (64, 3, 2)}),
    "el_clique40": ((4, 160), {(128, 256): (128, 3, 2), (256, 256): (256, 3, 1), (256, 64): (64, 3, 1)}),
    "el_clique48": None,
    "el_ragged": ((5, 142), {}),
    "el_real128": ((1, 128), {}),
    "el_real129": ((2, 130), {}),
    "el_iso255": ((4, 142), {}),
    "el_iso256": ((3, 142), {}),
    "el_iso257": ((3, 142), {}),
    "el_rows2w": ((1, 128), {}),
}


@pytest.mark.parametrize("name", FAMILIES)
def test_families_and_routes(name):
    """The hook's report of the padded level: which families exist, their sizes and the configurations each family
    was built to reach; a level without families runs every conv on its consecutive tiles (elide off at every mode)."""
    net = N.Net(name, "fp16x3", seed=1, open_relus=True)
    f = families(net, 0, 256, 64)
    cons = f["consecutive"][128]
    assert cons["n_pattern"] > 0 and cons["t1_fp16x3"][1] > 0, (name, cons)
    exp = EXPECT[name]
    if exp is None:
        assert all(f[k][t]["n_pattern"] == 0 for k in ("real", "iso", "rep") for t in (128, 64)), (name, f)
        for mode in (1, 2):
            net.hier.set_debug(0, elide_padding=mode)
            for li in range(net.n_layers):
                if net.layers[li]["level"] == 0:
                    r = net.route(li, 4)
                    assert not r["elide"] and not r["dx_elide"], (name, mode, li, r)
        return
    (P, h1), cfgs = exp
    real = f["real"][128]
    assert (real["n_pattern"], real["max_h1"]) == (P, h1), (name, real)
    for (fin, fout), want in cfgs.items():
        assert conv_cfg(net, 0, fin, fout, "real", "t1_fp16x3") == want, (name, fin, fout)
    # six fp16 slots and both stages of the isolated rows' plain GEMM wherever three fp16x3 slots fit
    for fam in ("real", "iso", "rep"):
        for fin, fout in ((128, 256), (256, 64)):
            t = families(net, 0, fin, fout)[fam][128 if fout == 64 else 64]
            if t["n_pattern"]:
                assert t["t1_fp16"][1] == (6 if fout != 64 else 3), (name, fam, t)
                if fam != "real":
                    assert t["plain_fp16"][1:] == ((6, 2) if fout != 64 else (3, 2)), (name, fam, t)


# ------------------------------------------------------------------------------------------------------ eval
EVAL_B = {"el_rows2w": 2}   # B V = 512 = 2 x 256: the 256-wide convs elide at B = 2 (at B = 1 they do not)
# elision 2 with the grids capped; fp32 runs no tensor-core conv, so it elides nothing at any mode: one run
MODES = {"fp16x3": (0, 1, 2), "fp16": (0, 1, 2), "fp32": (2,)}


@pytest.mark.parametrize("precision", ["fp16x3", "fp16", "fp32"])
@pytest.mark.parametrize("name", FAMILIES)
def test_eval_layer_by_layer(name, precision):
    """Eval forward at elision 0 / 1 / 2 (capped at 2): every layer (fused head off, then the fused head) from
    its captured input; dedup on (the isolated rows' GEMM on rep_tiles) bitwise equal to dedup off (on iso_tiles)."""
    B = EVAL_B.get(name, 1)
    net = N.Net(name, precision, seed=17, open_relus=False)
    try:
        for mode in MODES[precision]:
            x, _ = N.train_inputs(net, B, seed=3 + mode)
            cap = CAP if mode == 2 else 0
            net.hier.set_debug(0, elide_padding=mode, sm_count=cap)
            tag = f"{name} {precision} eval elide={mode} cap={cap}"
            lib().conv_log(reset=True)
            want = check_routes(net, tag, B, mode) if precision != "fp32" else set()
            y, yf, _, _ = N.check_eval(net, tag, x, mode)
            read_log(tag, want, cap > 0)
            for fuse in (False, True):
                yd, _ = N.forward_eval(net, x, mode, dedup=True, fuse=fuse, capture=False)
                assert np.array_equal(yd, y if not fuse else yf), (tag, "dedup", fuse)
            read_log(tag, set(), cap > 0)
            assert net.hier.kernel_status(0) == 0, tag
    finally:
        net.hier.set_debug(0, sm_count=0)
    _RAN.add(("eval", name, precision))


# ----------------------------------------------------------------------------------------------------- training
def mse(y, tgt):
    """The loss of the training cases: with the L1 loss, the 64-wide BatchNorm in front of the head sums 1024 rows of
    one magnitude (|dL/dy| constant), where fp64_ref's sqrt-growth model of the statistics sums (stat_allowance) does
    not hold for dbeta (up to 1.2 x its bound, at elision 0 and in fp32 as well: not a tile path).  A squared error's
    gradient varies from row to row."""
    return ((y - tgt) ** 2).mean()


@pytest.mark.parametrize("precision", ["fp16x3", "fp32"])
@pytest.mark.parametrize("name", FAMILIES)
def test_train_layer_by_layer(name, precision):
    """Training forward and backward with dX at elision 0 / 1 / 2 (capped at elision 2): every layer from its captured
    inputs, the backward-data convs on the connected-row tiles where dx_elide."""
    B = EVAL_B.get(name, 1)
    net = N.Net(name, precision, seed=29, open_relus=True)
    try:
        for mode in MODES[precision]:
            cap = CAP if mode == 2 else 0
            net.hier.set_debug(0, elide_padding=mode, sm_count=cap)
            net.sm_cap = cap
            tag = f"{name} {precision} train elide={mode} cap={cap}"
            x, tgt = N.train_inputs(net, B, seed=5 + mode)
            lib().conv_log(reset=True)
            want = check_routes(net, tag, B, mode, train=True) if precision != "fp32" else set()
            cap_, grads, bufs, y = N.forward_train_backward(net, x, tgt, True, loss_fn=mse)
            read_log(tag, want, cap > 0)
            N.check_train(net, tag, x, y, cap_, grads, bufs, True)
    finally:
        net.hier.set_debug(0, sm_count=0)
        net.sm_cap = 0
    _RAN.add(("train", name, precision))


# ----------------------------------------------------------------------------------------------------- coverage
# Every instantiation launch_n can select on an index-list family (real_tiles: T1-given; iso_tiles / rep_tiles:
# plain), and the families above that reach it with >= 2 tiles on some CTA.  Not reachable there:
# - the plain GEMM with fewer than the deepest ring and both X stages: it runs on the isolated rows' tiles, one CSR
#   entry per row (blobs of at most 2176 bytes);
# - a 64 x 128 T1-given conv with a ring of 3 and one T1 stage (conv, 128, 3, 1): its 64-row family would need blobs
#   over ~45 KB, and the 128-row family of the same connected rows (twice the rows) would then not fit the 128 x 64
#   ring, so build_umma_level_meta keeps no families;
# - single-pass fp16 below six 64 x 128 slots: six fp16 slots fit wherever three fp16x3 slots do, and a family is
#   kept only where those fit (launchable<> in cheb_umma.cu: those instantiations are not built).
ON_INDEX_TILES = {
    ("conv", 64, 3, 2, 1, 0): "el_h1_256", ("conv", 64, 3, 1, 1, 0): "el_clique40",
    ("conv", 128, 6, 2, 1, 0): "el_h1_256", ("conv", 128, 6, 1, 1, 0): "el_clique24",
    ("conv", 128, 3, 2, 1, 0): "el_clique40", ("conv", 256, 3, 2, 1, 0): "el_h1_256",
    ("conv", 256, 3, 1, 1, 0): "el_clique40",
    ("conv", 64, 3, 2, 0, 0): "el_h1_256", ("conv", 128, 6, 2, 0, 0): "el_h1_256",
    ("conv", 64, 3, 2, 1, 1): "el_h1_256", ("conv", 128, 6, 2, 1, 1): "el_h1_256",
    ("conv", 256, 3, 2, 1, 1): "el_h1_256",
    ("conv", 64, 3, 2, 0, 1): "el_h1_256", ("conv", 128, 6, 2, 0, 1): "el_h1_256",
}


def test_index_tile_instantiations_ran_multi_tile():
    """Over this module's cases: every instantiation of ON_INDEX_TILES ran on index-list tiles with >= 2 tiles on some
    CTA, nothing outside it ran there, and the families' hook reports agree with the list."""
    if len(_RAN) < 5 * len(FAMILIES):
        pytest.skip("reads the launches of the module's other tests: run the whole module")
    print("tiles per CTA on index-list tiles:", {k: _SEEN[k] for k in sorted(_SEEN)})
    short = {k: _SEEN.get(k, 0) for k in ON_INDEX_TILES if _SEEN.get(k, 0) < 2}
    assert not short, f"ran with fewer than 2 tiles on every CTA (0 = never ran): {short}"
    unknown = set(_SEEN) - set(ON_INDEX_TILES)
    assert not unknown, f"instantiations outside ON_INDEX_TILES ran on index-list tiles: {unknown}"
    for k, name in ON_INDEX_TILES.items():
        if k[4] != 1 or k[5] != 0:
            continue
        net = N.Net(name, "fp16x3", seed=1, open_relus=True)
        fin, fout = {64: (256, 64), 128: (128, 256), 256: (256, 256)}[k[1]]
        assert ("conv",) + conv_cfg(net, 0, fin, fout, "real", "t1_fp16x3") + (1, 0) == k, (k, name)
