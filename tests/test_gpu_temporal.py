"""The temporal metrics on the GPU (SURVEY.md §8 row f8, pose2mesh_release_b200.temporal) against

  * the unmodified reference (tests/golden/temporal.npz): smoothing and per-window acceleration errors bit for bit,
    video means and totals within 1e-6 relative, per-frame PA-MPJPE within 1e-6 of the frame's max |gt|;
  * oracle/temporal_oracle.py, the kernels' arithmetic in numpy: bit for bit on ragged batches."""
import numpy as np
import pytest
import torch

import temporal_cases as tc
from oracle import temporal_oracle as to
from pose2mesh_release_b200 import _lib
from pose2mesh_release_b200 import temporal as T

pytestmark = pytest.mark.gpu


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def host(t):
    return t.cpu().numpy()


def same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b, equal_nan=True)


def walk(rng, shape, dtype):
    return (rng.standard_normal(shape[1:]) * 300 + np.cumsum(rng.standard_normal(shape) * 8, 0)).astype(dtype)


def launches(fn):
    _lib.load().p2m_launch_count_reset()
    out = fn()
    return out, _lib.load().p2m_launch_count()


# ------------------------------------------------------------------------------------------------ reference fixture
def _smoothing_items():
    """[(x, min_cutoff, beta, reference digest)]."""
    z, xs = tc.fixture(), tc.smoothing_inputs()
    return [(xs[k], mc, b, str(z[f"sm{i}_digest"])) for i, (k, mc, b) in enumerate(tc.smoothing_cases())]


def test_smooth_pose_matches_reference_bitwise():
    for i, (x, mc, b, ref) in enumerate(_smoothing_items()):
        got = host(T.smooth_pose(cuda(x), min_cutoff=mc, beta=b))
        assert same(got, to.one_euro(x, mc, b)) and tc.digest(got) == ref, i


def test_smooth_sequences_batches_every_fixture_case_per_parameter_pair():
    by_pair = {}
    for x, mc, b, ref in _smoothing_items():
        by_pair.setdefault((x.dtype, x.shape[1:], mc, b), []).append((x, ref))
    for (dt, shape, mc, b), items in by_pair.items():
        xs = np.concatenate([x for x, _ in items])
        got, n = launches(lambda: T.smooth_sequences(cuda(xs), [len(x) for x, _ in items], mc, b))
        assert n == 1
        parts = np.split(host(got), np.cumsum([len(x) for x, _ in items])[:-1])
        assert [tc.digest(p) for p in parts] == [ref for _, ref in items], (dt, shape, mc, b)


def test_compute_error_accel_matches_reference_bitwise():
    z = tc.fixture()
    for i, gt, pred, v, vis in tc.accel_cases():
        got = host(T.compute_error_accel(cuda(gt), cuda(pred), None if vis is None else cuda(vis)))
        assert tc.digest(got) == str(z[f"ac{i}_{v}_digest"]), (i, v)


def test_accel_errors_per_window_and_means_batched():
    z = tc.fixture()
    for dt in (np.float32, np.float64):
        for J in (14, 17, 24):
            cases = [c for c in tc.accel_cases() if c[1].dtype == dt and c[1].shape[1] == J and c[3] == "random"]
            gt = np.concatenate([c[1] for c in cases])
            pred = np.concatenate([c[2] for c in cases])
            vis = np.concatenate([c[4] for c in cases])
            lengths = [len(c[1]) for c in cases]
            (pw, valid, mean), n = launches(lambda: T.accel_errors(cuda(gt), cuda(pred), lengths, cuda(vis)))
            assert n <= 2
            ref = [to.accel_error(c[1], c[2], c[4]) for c in cases]
            assert same(host(pw), np.concatenate([r[0] for r in ref]))
            assert np.array_equal(host(valid), np.concatenate([r[1] for r in ref]))
            wins = np.concatenate([[0], np.cumsum([max(n - 2, 0) for n in lengths])])
            for k, (i, *_, v, _) in enumerate(cases):
                seg = slice(wins[k], wins[k + 1])
                assert tc.digest(host(pw)[seg][host(valid)[seg]]) == str(z[f"ac{i}_{v}_digest"]), (i, v)
            want = np.array([r[0][r[1]].astype(np.float64).mean() if r[1].any() else np.nan for r in ref])
            np.testing.assert_allclose(host(mean), want, rtol=1e-6)
            assert (np.isnan(host(mean)) == np.isnan(want)).all()


@pytest.mark.parametrize("smooth", [True, False])
def test_evaluate_video_matches_reference_block(smooth):
    z = tc.fixture()
    tag = "smooth" if smooth else "raw"
    pred_j3d, gt_j3d, masks = tc.video_set()
    masks = list(masks)
    out, n = launches(lambda: T.evaluate_video(cuda(pred_j3d), cuda(gt_j3d), masks, smooth=smooth))
    assert n <= (9 if smooth else 8)
    acc, mpjpe = host(out["accel_error"]), host(out["mpjpe"])
    np.testing.assert_allclose(acc, z[f"vid_{tag}_accel"], rtol=1e-6)
    assert (np.isnan(acc) == np.isnan(z[f"vid_{tag}_accel"])).all()
    np.testing.assert_allclose(mpjpe, z[f"vid_{tag}_mpjpe"], rtol=1e-6)
    np.testing.assert_allclose(float(out["mpjpe_total"]), float(z[f"vid_{tag}_mpjpe_total"]), rtol=1e-6)
    assert np.isnan(float(out["accel_error_total"])) and np.isnan(z[f"vid_{tag}_accel_total"])
    np.testing.assert_allclose(float(out["pa_mpjpe_total"]), float(z[f"vid_{tag}_pa_total"]), rtol=1e-6)
    if smooth:
        pa = host(out["pa_mpjpe"])
        scale = np.abs(gt_j3d[np.concatenate([np.flatnonzero(m) for m in masks])]).max(axis=(1, 2))
        assert pa.shape == z["vid_smooth_pa"].shape
        assert (np.abs(pa - z["vid_smooth_pa"]) <= 1e-6 * scale[:, None]).all()
    # the videos with windows only: the accel total is then finite
    keep = [v for v, m in enumerate(masks) if m.sum() >= 3]
    out = T.evaluate_video(cuda(pred_j3d), cuda(gt_j3d), [masks[v] for v in keep], smooth=smooth)
    ref_acc = z[f"vid_{tag}_accel"][keep]
    np.testing.assert_allclose(float(out["accel_error_total"]), np.mean(ref_acc.astype(np.float64)), rtol=1e-6)


def test_evaluate_video_index_arrays_equal_masks():
    pred_j3d, gt_j3d, masks = tc.video_set()
    a = T.evaluate_video(cuda(pred_j3d), cuda(gt_j3d), list(masks))
    b = T.evaluate_video(cuda(pred_j3d), cuda(gt_j3d), [np.flatnonzero(m) for m in masks])
    for k in a:
        assert torch.equal(a[k].nan_to_num(-1), b[k].nan_to_num(-1)), k


# ------------------------------------------------------------------------------------------------ kernel order at size
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_ragged_3dpw_sized_batch_bitwise(dtype):
    rng = np.random.default_rng(7)
    lengths = [1, 2] + list(rng.integers(600, 1300, 35))
    lengths[-1] += 35000 - sum(lengths)
    x = walk(rng, (sum(lengths), 14, 3), dtype)
    gt = (x + rng.standard_normal(x.shape) * 30).astype(dtype)
    y = host(T.smooth_sequences(cuda(x), lengths, 0.004, 0.7))
    pw, valid, _ = T.accel_errors(cuda(gt), cuda(y), lengths)
    off = np.concatenate([[0], np.cumsum(lengths)])
    win = []
    for s in range(len(lengths)):
        seg = slice(off[s], off[s + 1])
        assert same(y[seg], to.one_euro(x[seg], 0.004, 0.7)), s
        win.append(to.accel_error(gt[seg], y[seg])[0])
    assert same(host(pw), np.concatenate(win)) and host(valid).all()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_smpl_mesh_frames_bitwise(dtype):
    rng = np.random.default_rng(11)
    lengths = [1, 2, 37, 60]
    x = walk(rng, (sum(lengths), 6890, 3), dtype)
    y = host(T.smooth_sequences(cuda(x), lengths, 0.004, 0.7))
    off = np.concatenate([[0], np.cumsum(lengths)])
    for s in range(len(lengths)):
        seg = slice(off[s], off[s + 1])
        assert same(y[seg], to.one_euro(x[seg], 0.004, 0.7)), s


# ------------------------------------------------------------------------------------------------ properties
def test_deterministic_and_independent_of_batch_order():
    rng = np.random.default_rng(3)
    lengths = [5, 300, 1, 80, 2, 41]
    x = walk(rng, (sum(lengths), 14, 3), np.float32)
    gt = (x + rng.standard_normal(x.shape) * 30).astype(np.float32)
    off = np.concatenate([[0], np.cumsum(lengths)])
    videos = [np.arange(off[s], off[s + 1]) for s in range(len(lengths))]
    a = T.evaluate_video(cuda(x), cuda(gt), videos)
    b = T.evaluate_video(cuda(x), cuda(gt), videos)
    perm = [3, 0, 5, 2, 4, 1]
    c = T.evaluate_video(cuda(x), cuda(gt), [videos[p] for p in perm])
    for k in ("accel_error", "mpjpe"):
        assert torch.equal(a[k].nan_to_num(-1), b[k].nan_to_num(-1))
        assert torch.equal(a[k][perm].nan_to_num(-1), c[k].nan_to_num(-1)), k
    pa_a = torch.split(a["pa_mpjpe"], lengths)
    pa_c = torch.split(c["pa_mpjpe"], [lengths[p] for p in perm])
    for i, p in enumerate(perm):
        assert torch.equal(pa_a[p], pa_c[i])
    ys = T.smooth_sequences(cuda(x), lengths, 0.004, 0.7)
    yp = T.smooth_sequences(cuda(np.concatenate([x[off[p]:off[p + 1]] for p in perm])), [lengths[p] for p in perm],
                            0.004, 0.7)
    assert torch.equal(torch.cat([ys[off[p]:off[p + 1]] for p in perm]), yp)


def test_nan_stays_in_its_channel_and_video():
    rng = np.random.default_rng(4)
    lengths = [50, 60]
    x = walk(rng, (110, 14, 3), np.float64)
    x[20, 4, 1] = np.nan
    y = host(T.smooth_sequences(cuda(x), lengths, 0.004, 0.7))
    assert np.isnan(y[20:50, 4, 1]).all() and np.isfinite(y[:20]).all()
    mask = np.ones_like(y, bool)
    mask[20:50, 4, 1] = False
    assert np.isfinite(y[mask]).all()
    assert same(y, np.concatenate([to.one_euro(x[:50], 0.004, 0.7), to.one_euro(x[50:], 0.004, 0.7)]))


def test_empty_and_invisible_videos_give_nan():
    rng = np.random.default_rng(5)
    gt = walk(rng, (20, 14, 3), np.float32)
    pred = (gt + 10).astype(np.float32)
    vis = np.ones(20, bool)
    vis[10:20] = False
    _, _, mean = T.accel_errors(cuda(gt), cuda(pred), [0, 10, 10, 0], cuda(vis))
    m = host(mean)
    assert np.isnan(m[0]) and np.isfinite(m[1]) and np.isnan(m[2]) and np.isnan(m[3])
    out = T.evaluate_video(cuda(pred), cuda(gt), [np.arange(10), np.array([], np.int64)])
    assert np.isnan(host(out["mpjpe"])[1]) and np.isnan(host(out["accel_error"])[1])
    assert np.isfinite(host(out["mpjpe"])[0])


# ------------------------------------------------------------------------------------------------ argument errors
def test_argument_errors():
    x = torch.zeros((10, 14, 3), device="cuda:0")
    with pytest.raises(RuntimeError):
        T.smooth_pose(x.cpu())
    with pytest.raises(ValueError):
        T.smooth_pose(x[:0])
    with pytest.raises(ValueError):
        T.smooth_pose(x.half())
    with pytest.raises(ValueError):
        T.smooth_sequences(x, [4, 5], 0.004, 0.7)            # offsets do not cover the input
    with pytest.raises(ValueError):
        T.smooth_sequences(x, [11, -1], 0.004, 0.7)
    with pytest.raises(ValueError):
        T.compute_error_accel(x, x[:, :13])                   # shape mismatch
    with pytest.raises(ValueError):
        T.compute_error_accel(x, x.double())
    with pytest.raises(RuntimeError):
        T.compute_error_accel(x.cpu(), x.cpu())
    with pytest.raises(ValueError):
        T.compute_error_accel(x, x, torch.ones(9, dtype=torch.bool, device="cuda:0"))   # vis length != N
    with pytest.raises(RuntimeError):
        T.compute_error_accel(x, x, torch.ones(10, dtype=torch.bool))
    with pytest.raises(ValueError):
        T.accel_errors(x, x, [3, 3])
    with pytest.raises(ValueError):
        T.evaluate_video(x, x, [np.array([0, 10])])          # frame index out of range
    with pytest.raises(ValueError):
        T.evaluate_video(x, x, [np.ones(9, bool)])            # mask length != frames
    with pytest.raises(ValueError):
        T.accel_errors(torch.zeros((10, 33, 3), device="cuda:0"), torch.zeros((10, 33, 3), device="cuda:0"), [10])
