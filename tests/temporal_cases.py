"""The cases of tests/golden/temporal.npz (made by tests/golden/make_golden_temporal.py from the unmodified reference).

The inputs are not stored: they are rebuilt here from PCG64's raw bit stream (stable across numpy versions) with exact
float64 arithmetic, and the fixture pins a digest of every input so a drift in this builder is caught.  Outputs that
must match bit for bit are pinned by digest (dtype, shape and bytes, with NaN payloads and zero signs made canonical,
as np.array_equal(..., equal_nan=True) compares); outputs held to a tolerance are stored as arrays.
"""
import functools
import hashlib
import os

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "temporal.npz")
PAIRS = ((0.004, 0.7), (0.004, 0.005), (1.0, 0.0), (0.1, 10.0))
VIS_VARIANTS = ("none", "random", "first", "last", "all")
VIDEO_LENGTHS = (1, 2, 3, 50, 400, 1000)
VIDEO_ORDER = (3, 0, 5, 1, 4, 2)     # the videos lie in the frame array in this order


def uniform(seed: int, n: int) -> np.ndarray:
    """n float64 values in [0, 1) from the top 53 bits of PCG64(seed)'s raw output."""
    raw = np.random.PCG64(seed).random_raw(n)
    return (raw >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def walk(seed: int, shape, dtype, step=8.0, scale=300.0) -> np.ndarray:
    """Random-walk motion in mm along axis 0: a start in [-scale, scale) plus steps in [-step, step)."""
    m, n = int(np.prod(shape[1:])), int(np.prod(shape))
    u = uniform(seed, m + n)
    start = (u[:m] - 0.5) * (2.0 * scale)
    steps = ((u[m:] - 0.5) * (2.0 * step)).reshape(shape)
    return (start.reshape(shape[1:]) + np.cumsum(steps, axis=0)).astype(dtype)


def noisy(seed: int, x: np.ndarray, amp: float) -> np.ndarray:
    return (x + (uniform(seed, x.size).reshape(x.shape) - 0.5) * (2.0 * amp)).astype(x.dtype)


def digest(a) -> str:
    a = np.ascontiguousarray(a)
    if a.dtype.kind == "f":
        a = a.copy()
        a[np.isnan(a)] = np.nan
        a[a == 0] = 0
    h = hashlib.sha256(f"{a.dtype.str}{a.shape}".encode())
    h.update(a.tobytes())
    return h.hexdigest()


# ------------------------------------------------------------------------------------------------ smoothing
def smoothing_inputs():
    """[x]: every smoothing input, float32 and float64."""
    xs = []
    for d, dt in enumerate((np.float32, np.float64)):
        for n in (1, 2, 3, 17):
            for J in (14, 17, 24):
                xs.append(walk(1000 * d + 10 * n + J, (n, J, 3), dt))
        xs.append(walk(1000 * d + 500, (1000, 14, 3), dt))
        xs.append(np.full((30, 14, 3), 123.25, dt))                                           # constant
        xs.append(np.where(np.arange(30)[:, None, None] < 15, 0.0, 100.0).repeat(14, 1).repeat(3, 2).astype(dt))
        s = walk(1000 * d + 600, (30, 14, 3), dt)                                             # one NaN, one inf
        s[12, 3, 1] = np.nan
        s[17, 5, 2] = np.inf
        xs.append(s)
    xs.append(walk(2000, (40, 778, 3), np.float32, step=2.0))                                # a MANO-size mesh
    return xs


def smoothing_cases():
    """[(input index, min_cutoff, beta)]: every input under every pair, the mesh under the default pair."""
    n_in = len(smoothing_inputs())
    return [(k, mc, b) for k in range(n_in - 1) for mc, b in PAIRS] + [(n_in - 1, 0.004, 0.7)]


def nonuniform_case(dt):
    """(x [60, 14, 3], t [60]) for one OneEuroFilter run at non-uniform times."""
    tag = 0 if dt == np.float32 else 1
    x = walk(3000 + tag, (60, 14, 3), dt)
    t = np.concatenate([[0.0], np.cumsum(0.25 + 1.75 * uniform(3010 + tag, 59))]).astype(dt)
    return x, t


# ------------------------------------------------------------------------------------------------ accel
def accel_sequences():
    """[(gt, pred, {variant: vis or None})] for N in {1, 2, 3, 4, 500} at J = 14 and N = 40 at J = 17, 24."""
    specs = [(dt, n, 14) for dt in (np.float32, np.float64) for n in (1, 2, 3, 4, 500)]
    specs += [(dt, 40, J) for dt in (np.float32, np.float64) for J in (17, 24)]
    out = []
    for i, (dt, n, J) in enumerate(specs):
        gt = walk(4000 + i, (n, J, 3), dt)
        pred = noisy(4100 + i, gt, 35.0)
        variants = {"none": None, "random": uniform(4200 + i, n) > 0.15, "first": np.arange(n) > 0,
                    "last": np.arange(n) < n - 1, "all": np.zeros(n, bool)}
        out.append((gt, pred, variants))
    return out


def accel_cases():
    """[(sequence index, gt, pred, variant, vis or None)]."""
    return [(i, gt, pred, v, vis) for i, (gt, pred, variants) in enumerate(accel_sequences())
            for v, vis in variants.items()]


# ------------------------------------------------------------------------------------------------ video block
def video_set():
    """(pred_j3d, gt_j3d [1456, 14, 3] float32 in mm, masks [6, 1456]): six 3DPW-like videos, pred = gt + noise."""
    total = sum(VIDEO_LENGTHS)
    starts, pos = {}, 0
    for v in VIDEO_ORDER:
        starts[v] = pos
        pos += VIDEO_LENGTHS[v]
    masks = np.zeros((len(VIDEO_LENGTHS), total), bool)
    gt = np.zeros((total, 14, 3), np.float32)
    for v, n in enumerate(VIDEO_LENGTHS):
        masks[v, starts[v]:starts[v] + n] = True
        gt[masks[v]] = walk(5000 + v, (n, 14, 3), np.float32)
    pred = noisy(5100, gt, 70.0)
    return pred, gt, masks


# ------------------------------------------------------------------------------------------------ fixture
@functools.lru_cache(maxsize=1)
def fixture():
    with np.load(PATH) as z:
        return {k: z[k] for k in z.files}


def input_digests():
    """Digests of every rebuilt input, in the fixture's key order."""
    out = {f"in{k}": digest(x) for k, x in enumerate(smoothing_inputs())}
    for dt, tag in ((np.float32, "f32"), (np.float64, "f64")):
        x, t = nonuniform_case(dt)
        out[f"ou_{tag}_x"], out[f"ou_{tag}_t"] = digest(x), digest(t)
    for i, (gt, pred, variants) in enumerate(accel_sequences()):
        out[f"ac{i}_gt"], out[f"ac{i}_pred"] = digest(gt), digest(pred)
        for v, vis in variants.items():
            if vis is not None:
                out[f"ac{i}_{v}_vis"] = digest(vis)
    pred, gt, masks = video_set()
    out.update({"vid_pred": digest(pred), "vid_gt": digest(gt), "vid_masks": digest(masks)})
    return out
