"""Float64 CPU restatement of the device rule of the training inputs (pose2mesh_release_b200/inputs.py):

    synthesize_pose      lib/noise_utils.py:17-285 (num_overlap = 0, near_joints all zero) on the counter-based stream
                         of include/p2m_b200.h, with the shortcuts DESIGN.md §4.3 (dataset inputs) argues are exact
                         in distribution
    generate_syn_error   data/Human36M/dataset.py:143-155 on the same stream
    training_pose2d      the train branch of the datasets' replace_joint_img and the crop / normalisation around it
                         (data/Human36M/dataset.py:359-392,436-445), and with box_joints the test-split branch (:446-452)

The random stream is the library's, not numpy's: the device is restated draw for draw, so the device must agree with
this module to rounding, while tests/golden/inputs.npz (the unmodified reference over many seeds) pins the distribution.
The joints are visited in the reference's order j = 0 .. 16; the device runs them in two phases (DESIGN.md §4.3,
dataset inputs), which gives the same result.  Vectorised over the batch, written joint by joint.
"""
from __future__ import annotations

import numpy as np

# COCO keypoint OKS sigmas (cfg.kps_sigmas, lib/noise_utils.py:9-11; the COCO benchmark's published constants)
KPS_SIGMAS_X10 = (.26, .25, .25, .35, .35, .79, .79, .72, .72, .62, .62, 1.07, 1.07, .87, .87, .89, .89)
NUM_KPS = 17
KPS_SYMMETRY = ((1, 2), (3, 4), (5, 6), (7, 8), (9, 10), (11, 12), (13, 14), (15, 16))
N = 500
INPUT_SHAPE = (384, 288)

# stream ids: 16 * joint + purpose (include/p2m_b200.h)
JITTER, GOOD, INV, MISS_GT, MISS_INV, MISS_PICK, CHOICE, GAUSS, KEEP = range(9)
CHUNK = 32      # draws per step of the first-survivor search (one warp on the device)


def pair_of(j: int):
    for q, w in KPS_SYMMETRY:
        if j == q:
            return w
        if j == w:
            return q
    return None


# --------------------------------------------------------------------------------------------- the random stream
def philox4x32_10(ctr, key):
    """Philox4x32-10 (Salmon et al., SC'11), the algorithm of tests/posenet_train_ref.py.  ctr: four uint32 arrays (or
    ints), key: two ints.  Returns four uint64 arrays holding uint32 values."""
    c = [np.asarray(v, np.uint64) & np.uint64(0xFFFFFFFF) for v in ctr]
    c = np.broadcast_arrays(*c)
    k = [int(v) & 0xFFFFFFFF for v in key]
    m0, m1, mask, s32 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57), np.uint64(0xFFFFFFFF), np.uint64(32)
    for _ in range(10):
        p0, p1 = m0 * c[0], m1 * c[2]
        c = [(p1 >> s32) ^ c[1] ^ np.uint64(k[0]), p1 & mask, (p0 >> s32) ^ c[3] ^ np.uint64(k[1]), p0 & mask]
        k = [(k[0] + 0x9E3779B9) & 0xFFFFFFFF, (k[1] + 0xBB67AE85) & 0xFFFFFFFF]
    return c


def _u53(hi, lo):
    """A float64 uniform on [0, 1) from two words: 27 high bits of one, 26 of the other (numpy's random_double)."""
    return ((hi >> np.uint64(5)).astype(np.float64) * 67108864.0 + (lo >> np.uint64(6)).astype(np.float64)) \
        / 9007199254740992.0


def uniforms(seed, b, sid: int, d):
    """The two float64 uniforms of counter (d, sid, b, seed[1]) under key seed[0]; b and d broadcast."""
    s0, s1 = (int(v) & 0xFFFFFFFFFFFFFFFF for v in seed)
    w = philox4x32_10((d, sid, b, s1 & 0xFFFFFFFF), (s0 & 0xFFFFFFFF, s0 >> 32))
    return _u53(w[0], w[1]), _u53(w[2], w[3])


def pick_index(u, n):
    """floor(u n) clamped to n - 1 (u n can round up to n)."""
    return np.minimum(np.floor(u * n), n - 1).astype(np.int64)


# --------------------------------------------------------------------------------------------- candidate points
def _points(seed, b, sid, d, src, rlo, rhi):
    """Draws d ([n]) of stream sid for samples b ([B]): angle ~ U(0, 2 pi), r ~ U(rlo, rhi) around src [B, 2]."""
    ua, ur = uniforms(seed, b[:, None], sid, d[None, :])
    angle = 2 * np.pi * ua
    r = rlo[:, None] + (rhi - rlo)[:, None] * ur
    return src[:, 0:1] + r * np.cos(angle), src[:, 1:2] + r * np.sin(angle), r


def _far(x, y, other, has_other, thr):
    """noise_utils' dist_mask: distance to the other source > thr (no other source: every draw passes)."""
    d = np.sqrt((other[:, 0:1] - x) ** 2 + (other[:, 1:2] - y) ** 2)
    return ~has_other[:, None] | (d > thr)


def first_survivor(seed, b, sid, n_draw, src, rlo, rhi, other, has_other, by_radius=True, thr=None):
    """The first of draws 0 .. n_draw - 1 that passes the mask (distance to `other` > r, or > thr): in distribution
    the reference's uniformly chosen survivor of n_draw draws.  -> found [B], x [B], y [B]."""
    B = len(b)
    found, X, Y = np.zeros(B, bool), np.zeros(B), np.zeros(B)
    for start in range(0, n_draw, CHUNK):
        act = np.nonzero(~found)[0]
        if len(act) == 0:
            break
        d = np.arange(start, min(start + CHUNK, n_draw), dtype=np.uint64)
        x, y, r = _points(seed, b[act], sid, d, src[act], rlo[act], rhi[act])
        ok = _far(x, y, other[act], has_other[act], r if by_radius else thr[act][:, None])
        hit = ok.any(axis=1)
        first = np.argmax(ok, axis=1)
        rows = act[hit]
        found[rows] = True
        X[rows], Y[rows] = x[hit, first[hit]], y[hit, first[hit]]
    return found, X, Y


def _miss_source(seed, b, sid, src, rlo, rhi, other, has_other, thr, need):
    """4 N draws around src for the samples `need`; the others pass every draw (the sources are farther apart than
    ks10 + ks50, or there is no other source).  -> survivors count [B] and the draws / masks of `need`."""
    B = len(b)
    count = np.full(B, 4 * N, np.int64)
    idx = np.nonzero(need)[0]
    if len(idx) == 0:
        return count, idx, None
    d = np.arange(4 * N, dtype=np.uint64)
    x, y, _ = _points(seed, b[idx], sid, d, src[idx], rlo[idx], rhi[idx])
    ok = _far(x, y, other[idx], has_other[idx], thr[idx][:, None])
    count[idx] = ok.sum(axis=1)
    return count, idx, (x, y, ok)


def _kth(seed, b, sid, k, src, rlo, rhi, drawn, rows):
    """The k-th survivor (0-based) of a source for the samples `rows`: from the draws where they were counted, else
    draw k itself (every draw survives)."""
    x, y = np.zeros(len(b)), np.zeros(len(b))
    counted = np.zeros(len(b), bool)
    if drawn[2] is not None:
        dx, dy, ok = drawn[2]
        sel = np.isin(drawn[0], rows)
        r = drawn[0][sel]
        at = np.argmax(np.cumsum(ok[sel], axis=1) > k[r][:, None], axis=1)
        x[r], y[r] = dx[sel, at], dy[sel, at]
        counted[r] = True
    r = rows[~counted[rows]]
    if len(r):
        ua, ur = uniforms(seed, b[r], sid, k[r].astype(np.uint64))
        rad = rlo[r] + (rhi[r] - rlo[r]) * ur
        x[r] = src[r, 0] + rad * np.cos(2 * np.pi * ua)
        y[r] = src[r, 1] + rad * np.sin(2 * np.pi * ua)
    return x, y


# --------------------------------------------------------------------------------------------- synthesize_pose
def radii(area):
    """get_dist_wrt_ks for d = 0.10, 0.50, 0.85: [B, 17] each."""
    sig = np.array(KPS_SIGMAS_X10) / 10.0
    var = (sig * 2) ** 2
    area = np.asarray(area, np.float64)[:, None]
    return tuple(np.sqrt(-2 * area * var[None, :] * np.log(ks)) for ks in (0.10, 0.50, 0.85))


def tier_probs(j: int, num_valid):
    """(jitter, miss, inv) probabilities of joint j for each sample's visible-joint count [B]."""
    if j == 0 or 13 <= j <= 16:
        jit = (0.15, 0.10)
    elif 1 <= j <= 10:
        jit = (0.20, 0.15)
    else:
        jit = (0.25, 0.20)
    jitter = np.where(num_valid <= 10, jit[0], jit[1])
    if j <= 4:
        ms = (0.15, 0.10, 0.02)
    elif j in (5, 6, 15, 16):
        ms = (0.20, 0.13, 0.05)
    else:
        ms = (0.25, 0.15, 0.10)
    miss = np.where(num_valid <= 5, ms[0], np.where(num_valid <= 10, ms[1], ms[2]))
    inv = 0.01 if j <= 4 else (0.03 if j <= 10 else 0.06)
    return jitter, miss, np.full(len(num_valid), inv)


def synthesize_pose(joints, area, seed, sample_index=None, trace=None):
    """joints [B, 17, 3] (x, y, visibility), area [B] -> [B, 17, 3] float64 rows (x, y, 1) or (0, 0, 0).
    sample_index [B]: each sample's index in the device call (default 0 .. B-1).  trace (a dict, optional) receives
    per joint j: 'inv_j' [B, 2] and 'has_inv_j' [B], the inv source joint j used."""
    joints = np.asarray(joints, np.float64)
    B = joints.shape[0]
    b = np.arange(B, dtype=np.uint64) if sample_index is None else np.asarray(sample_index, np.uint64)
    ks10, ks50, ks85 = radii(area)
    synth = joints.copy()
    num_valid = np.sum(joints[:, :, 2] > 0, axis=1)
    zero = np.zeros(B)
    for j in range(NUM_KPS):
        sid = 16 * j
        gt = synth[:, j, :2].copy()
        p = pair_of(j)
        has_inv = np.zeros(B, bool) if p is None else joints[:, p, 2] > 0   # the ORIGINAL visibility
        inv = np.zeros((B, 2)) if p is None else synth[:, p, :2].copy()      # phase 2: the partner's synthesized row
        if trace is not None:
            trace[f"inv_{j}"], trace[f"has_inv_{j}"] = np.where(has_inv[:, None], inv, 0.0), has_inv.copy()
        jitter_prob, miss_prob, inv_prob = tier_probs(j, num_valid)
        k10, k50, k85 = ks10[:, j], ks50[:, j], ks85[:, j]

        # jitter: N draws, r ~ U(ks85, ks50) around gt, kept if farther than r from inv
        jit_ok, jx, jy = first_survivor(seed, b, sid + JITTER, N, gt, k85, k50, inv, has_inv)

        # miss: 4N draws per source, r ~ U(ks50, ks10), kept if farther than ks50 from the other source; the pick is
        # the gt source with probability S0 / (S0 + S1 // 4), then a uniform survivor of the chosen source
        sep = np.sqrt((gt[:, 0] - inv[:, 0]) ** 2 + (gt[:, 1] - inv[:, 1]) ** 2)
        need = has_inv & ~(sep > (k10 + k50) * (1 + 1e-9))
        s0, rows0, d0 = _miss_source(seed, b, sid + MISS_GT, gt, k50, k10, inv, has_inv, k50, need)
        s1, rows1, d1 = _miss_source(seed, b, sid + MISS_INV, inv, k50, k10, gt, has_inv, k50, need)
        s1 = np.where(has_inv, s1, 0)
        tot = s0 + s1 // 4
        miss_ok = tot > 0                              # S0 = 0 and S1 < 4: absent (the reference raises there)
        ua, ub = uniforms(seed, b, sid + MISS_PICK, 0)
        kk = pick_index(ua, np.maximum(tot, 1))
        from_gt = kk < s0
        k_gt = kk
        k_inv = pick_index(ub, np.maximum(s1, 1))
        mx, my = np.zeros(B), np.zeros(B)
        r_gt = np.nonzero(miss_ok & from_gt)[0]
        r_inv = np.nonzero(miss_ok & ~from_gt)[0]
        gx_, gy_ = _kth(seed, b, sid + MISS_GT, k_gt, gt, k50, k10, (rows0, None, d0), r_gt)
        ix_, iy_ = _kth(seed, b, sid + MISS_INV, k_inv, inv, k50, k10, (rows1, None, d1), r_inv)
        mx[r_gt], my[r_gt] = gx_[r_gt], gy_[r_gt]
        mx[r_inv], my[r_inv] = ix_[r_inv], iy_[r_inv]

        # inv: N draws around inv (only with a visible pair), r ~ U(0, ks50), kept if farther than r from gt
        inv_ok, vx, vy = first_survivor(seed, b, sid + INV, N, inv, zero, k50, gt, np.ones(B, bool))
        inv_ok &= has_inv

        # good: N // 4 draws, r ~ U(0, ks85) around gt, kept if farther than r from inv
        good_prob = 1 - (jitter_prob + miss_prob + inv_prob + 0)
        good_ok, ox, oy = first_survivor(seed, b, sid + GOOD, N // 4, gt, zero, k85, inv, has_inv)

        # an absent candidate has probability 0; the rest are renormalised and one is drawn
        jitter_prob = np.where(jit_ok, jitter_prob, 0.0)
        miss_prob = np.where(miss_ok, miss_prob, 0.0)
        inv_prob = np.where(inv_ok, inv_prob, 0.0)
        good_prob = np.where(good_ok, good_prob, 0.0)
        normalizer = jitter_prob + miss_prob + inv_prob + 0 + good_prob
        uc, _ = uniforms(seed, b, sid + CHOICE, 0)
        t = uc * normalizer
        c1 = jitter_prob
        c2 = c1 + miss_prob
        c3 = c2 + inv_prob
        cand = [(jit_ok, jx, jy, t < c1), (miss_ok, mx, my, t < c2), (inv_ok, vx, vy, t < c3), (good_ok, ox, oy, None)]
        out = np.zeros((B, 3))
        done = normalizer == 0                         # every candidate absent: the row is zeroed
        last_x, last_y = np.zeros(B), np.zeros(B)       # the last present candidate takes a t at the top of the range
        for ok, cx, cy, _ in cand:
            last_x, last_y = np.where(ok, cx, last_x), np.where(ok, cy, last_y)
        for ok, cx, cy, below in cand[:3]:
            take = ~done & ok & below
            out[take, 0], out[take, 1], out[take, 2] = cx[take], cy[take], 1.0
            done |= take
        rest = ~done
        out[rest, 0], out[rest, 1], out[rest, 2] = last_x[rest], last_y[rest], 1.0
        synth[:, j] = out.astype(np.float32)           # the device's rows are float32, as the datasets' arrays
    return synth


# --------------------------------------------------------------------------------------------- Human3.6M errors
def generate_syn_error(table, B: int, seed, sample_index=None):
    """table: (mean [17, 2], std [17, 2], weight [17]) float64 -> noise [B, 17, 2] float32, kept rows only."""
    mean, std, weight = (np.asarray(a, np.float64) for a in table)
    b = np.arange(B, dtype=np.uint64) if sample_index is None else np.asarray(sample_index, np.uint64)
    noise = np.zeros((B, 17, 2), np.float32)
    for i in range(17):
        u1, u2 = uniforms(seed, b, 16 * i + GAUSS, 0)
        rad = np.sqrt(-2.0 * np.log(1.0 - u1))
        z0, z1 = rad * np.cos(2 * np.pi * u2), rad * np.sin(2 * np.pi * u2)
        x = (mean[i, 0] + std[i, 0] * z0).astype(np.float32)
        y = (mean[i, 1] + std[i, 1] * z1).astype(np.float32)
        prob, _ = uniforms(seed, b, 16 * i + KEEP, 0)
        keep = np.float64(np.float32(weight[i])) > prob
        noise[:, i, 0] = np.where(keep, x, np.float32(0))
        noise[:, i, 1] = np.where(keep, y, np.float32(0))
    return noise


# --------------------------------------------------------------------------------------------- crop and normalise
def crop_map(box_joints, input_shape=INPUT_SHAPE):
    """k_normalize_pose2d's box: get_bbox -> process_bbox -> the rot-0 affine map, per sample, in its float32 /
    float64 steps.  box_joints [B, Jb, 2] float32 -> dict of [B] arrays (ccx, ccy float32; sc float64; tight and
    processed box sizes)."""
    p = np.asarray(box_joints, np.float32)
    in_h, in_w = input_shape
    xmin, xmax = p[:, :, 0].min(1).astype(np.float64), p[:, :, 0].max(1).astype(np.float64)
    ymin, ymax = p[:, :, 1].min(1).astype(np.float64), p[:, :, 1].max(1).astype(np.float64)
    xc, w = (xmin + xmax) / 2.0, xmax - xmin
    yc, h = (ymin + ymax) / 2.0, ymax - ymin
    bx, by, bw, bh = (v.astype(np.float32) for v in (xc - 0.5 * w, yc - 0.5 * h, w, h))
    f = np.float32
    w = (bx + (bw - f(1))) - bx
    h = (by + (bh - f(1))) - by
    cx, cy = bx + w / f(2), by + h / f(2)
    aspect = f(in_w) / f(in_h)
    grow_h = w > aspect * h
    grow_w = ~grow_h & (w < aspect * h)
    h = np.where(grow_h, w / aspect, h).astype(np.float32)
    w = np.where(grow_w, h * aspect, w).astype(np.float32)
    x0, y0 = cx - w / f(2), cy - h / f(2)
    ccx, ccy = x0 + w * f(0.5), y0 + h * f(0.5)
    s1y = ccy + w * f(-0.5)
    d1y = f(in_h * 0.5) + f(in_w * -0.5)
    sc = (np.float64(d1y) - in_h * 0.5) / (s1y.astype(np.float64) - ccy.astype(np.float64))
    tight_w = (bx + bw).astype(np.float64) - bx        # replace_joint_img's xmax - xmin (xmax = x + w in float32)
    tight_h = (by + bh).astype(np.float64) - by
    return {"ccx": ccx, "ccy": ccy, "sc": sc, "tight_w": tight_w, "tight_h": tight_h,
            "crop_w": w.astype(np.float64), "crop_h": h.astype(np.float64)}


def crop_points(m, joints_px, input_shape=INPUT_SHAPE):
    """joints_px [B, J, 2] through the map -> float32 crop pixels [B, J, 2]."""
    in_h, in_w = input_shape
    p = np.asarray(joints_px, np.float32).astype(np.float64)
    tx = (p[:, :, 0] - m["ccx"].astype(np.float64)[:, None]) * m["sc"][:, None] + in_w * 0.5
    ty = (p[:, :, 1] - m["ccy"].astype(np.float64)[:, None]) * m["sc"][:, None] + in_h * 0.5
    return np.stack([tx, ty], -1).astype(np.float32)


def crop_area(m, area_box: str):
    """replace_joint_img's area: the tight box ('tight') or the processed box ('crop', MuCo) mapped into the crop."""
    w, h = (m["tight_w"], m["tight_h"]) if area_box == "tight" else (m["crop_w"], m["crop_h"])
    return (m["sc"] * w) * (m["sc"] * h)


def normalize(crop, input_shape=INPUT_SHAPE):
    """/ input size, then zero mean and unit (population) std per pose and coordinate."""
    in_h, in_w = input_shape
    u = crop.astype(np.float64) / np.array([in_w, in_h], np.float64)
    mu = u.mean(axis=1, keepdims=True)
    sd = np.sqrt(((u - mu) ** 2).mean(axis=1, keepdims=True))
    return (u - mu) / sd


def training_pose2d(joints_px, noise: str, seed=None, table=None, area_box="tight", box_joints=None,
                    input_shape=INPUT_SHAPE):
    """The device's training_pose2d: noise 'none' | 'coco' (rows 0-16 synthesized, every joint visible) | 'h36m'.
    -> (pose2d [B, J, 2] float64, crop [B, J, 2] float32 after the noise)."""
    joints_px = np.asarray(joints_px, np.float32)
    B = joints_px.shape[0]
    m = crop_map(joints_px if box_joints is None else box_joints, input_shape)
    crop = crop_points(m, joints_px, input_shape)
    in_h, in_w = input_shape
    if noise == "coco":
        j17 = np.concatenate([crop[:, :17].astype(np.float64), np.ones((B, 17, 1))], axis=2)
        crop = crop.copy()
        crop[:, :17] = synthesize_pose(j17, crop_area(m, area_box), seed)[:, :, :2].astype(np.float32)
    elif noise == "h36m":
        err = generate_syn_error(table, B, seed)
        scale = np.array([in_w, in_h], np.float32)
        crop = crop + (err / np.float32(256)) * scale
    return normalize(crop, input_shape), crop


# --------------------------------------------------------------------------------------------- outcome cells
N_RAD = 8
N_CELL = 5 * N_RAD + 2           # five annuli x N_RAD radial bins, zeroed, elsewhere
GRID = 12
N_CELL_2D = GRID * GRID + 2      # offset from gt / ks10 on a GRID x GRID grid over [-1.5, 1.5]^2, zeroed, outside


def outcome_cells(out, joints, area):
    """The cell of each synthesized row, for comparing distributions: out [M, 17, 3], joints [17, 3], area (scalar).
    The annuli around the joint's own coordinate (good [0, ks85), jitter [ks85, ks50), miss [ks50, ks10]) and, with a
    visible pair, around the inv source the joint used (inv [0, ks50), miss [ks50, ks10]) are tested in that order;
    within an annulus, N_RAD equal radial bins.  -> [M, 17] int."""
    out = np.asarray(out, np.float64)
    joints = np.asarray(joints, np.float64)
    M = out.shape[0]
    k10, k50, k85 = (r[0] for r in radii(np.array([area])))
    cells = np.full((M, NUM_KPS), N_CELL - 1, np.int64)
    for j in range(NUM_KPS):
        p = pair_of(j)
        gt = joints[j, :2]
        dg = np.hypot(out[:, j, 0] - gt[0], out[:, j, 1] - gt[1])
        rings = [(dg, 0.0, k85[j]), (dg, k85[j], k50[j]), (dg, k50[j], k10[j])]
        if p is not None and joints[p, 2] > 0:
            inv = out[:, p, :2] if j % 2 == 0 else np.broadcast_to(joints[p, :2], (M, 2))
            di = np.hypot(out[:, j, 0] - inv[:, 0], out[:, j, 1] - inv[:, 1])
            rings += [(di, 0.0, k50[j]), (di, k50[j], k10[j])]
        done = out[:, j, 2] == 0
        cells[done, j] = N_CELL - 2
        for a, (d, lo, hi) in enumerate(rings):
            hit = ~done & (d >= lo) & (d <= hi * (1 + 1e-12))
            rb = np.clip(((d - lo) / (hi - lo) * N_RAD).astype(np.int64), 0, N_RAD - 1)
            cells[hit, j] = a * N_RAD + rb[hit]
            done |= hit
    return cells


def offset_cells(out, joints, area):
    """The cell of each synthesized row's offset from the joint's coordinate over ks10 (close sources). -> [M, 17]."""
    out = np.asarray(out, np.float64)
    joints = np.asarray(joints, np.float64)
    k10 = radii(np.array([area]))[0][0]
    off = (out[:, :, :2] - joints[None, :, :2]) / k10[None, :, None]
    g = np.floor((off + 1.5) / 3.0 * GRID).astype(np.int64)
    inside = (g >= 0).all(-1) & (g < GRID).all(-1)
    cells = np.where(inside, np.clip(g[..., 1], 0, GRID - 1) * GRID + np.clip(g[..., 0], 0, GRID - 1), GRID * GRID + 1)
    return np.where(out[:, :, 2] == 0, GRID * GRID, cells)


def histogram(cells, n_cell):
    """[M, 17] cells -> [17, n_cell] counts."""
    return np.stack([np.bincount(cells[:, j], minlength=n_cell) for j in range(cells.shape[1])])
