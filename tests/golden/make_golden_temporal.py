#!/usr/bin/env python
"""Golden vectors of the reference's temporal metrics, produced by the UNMODIFIED reference functions
smooth_utils.smooth_pose / OneEuroFilter (lib/smooth_utils.py:5-72), coord_utils.compute_error_accel
(lib/coord_utils.py:194-222) and coord_utils.rigid_align (:146-149), imported through oracle/ref_shim.py.

    P2M_REFERENCE_ROOT=/path/to/Pose2Mesh_RELEASE python tests/golden/make_golden_temporal.py -> temporal.npz

The inputs are rebuilt by tests/temporal_cases.py from a bit-stable generator; the file pins their digests
(digest_<input>) and the digests of the reference's bit-exact outputs:

  sm{i}_digest        smooth_pose on every case of temporal_cases.smoothing_cases() (float32 and float64, four
                      (min_cutoff, beta) pairs, N in {1, 2, 3, 17, 1000} over 14-, 17- and 24-joint frames, constant,
                      step, NaN and inf signals, a 40 x 778 x 3 mesh sequence)
  ou_{f32,f64}_digest one OneEuroFilter run at non-uniform times
  ac{i}_{v}_digest    compute_error_accel's compacted errors per sequence and visibility variant (none, random,
                      first / last / all frames invisible)

Video (vid_*): six synthetic 3DPW-like videos in mm, smoothed and raw.  The video block of PW3D.evaluate
(data/PW3D/dataset.py:387-415) sits inside a string literal in the reference and cannot be called, so its lines are
restated here around the unmodified smooth_pose, compute_error_accel and rigid_align; its per-video means, totals and
(smoothed) per-frame PA-MPJPE are stored as arrays, since the tests hold them to a tolerance.

The archive is written with fixed zip timestamps, so running the generator twice gives the same bytes.
"""
import io
import os
import sys
import warnings
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

import temporal_cases as tc  # noqa: E402
from oracle import ref_shim  # noqa: E402


def load_reference():
    ref_shim.load("human36")
    import coord_utils  # noqa: E402  (reference module, lib/coord_utils.py)
    import smooth_utils  # noqa: E402  (reference module, lib/smooth_utils.py)

    return smooth_utils, coord_utils


def save(path, arrays):
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for key in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(arrays[key]), allow_pickle=False)
            info = zipfile.ZipInfo(key + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())


def main():
    smooth_utils, coord_utils = load_reference()
    out = {"numpy_version": np.array(np.__version__)}
    out.update({f"digest_{k}": np.array(v) for k, v in tc.input_digests().items()})
    with warnings.catch_warnings(), np.errstate(all="ignore"):
        warnings.simplefilter("ignore")
        # ---- smoothing
        inputs = tc.smoothing_inputs()
        cases = tc.smoothing_cases()
        for i, (k, mc, b) in enumerate(cases):
            y = smooth_utils.smooth_pose(inputs[k].copy(), min_cutoff=mc, beta=b)
            assert y.dtype == inputs[k].dtype
            out[f"sm{i}_digest"] = np.array(tc.digest(y))
        out["sm_cases"] = np.array(cases, np.float64)
        for dt, tag in ((np.float32, "f32"), (np.float64, "f64")):
            x, t = tc.nonuniform_case(dt)
            f = smooth_utils.OneEuroFilter(np.full_like(x[0], t[0]), x[0], min_cutoff=0.004, beta=0.7)
            y = np.empty_like(x)
            y[0] = x[0]
            for i in range(1, len(x)):
                y[i] = f(np.full_like(x[i], t[i]), x[i])
            out[f"ou_{tag}_digest"] = np.array(tc.digest(y))

        # ---- acceleration error
        for i, gt, pred, v, vis in tc.accel_cases():
            e = coord_utils.compute_error_accel(gt.copy(), pred.copy(), None if vis is None else vis.copy())
            assert e.dtype == gt.dtype
            out[f"ac{i}_{v}_digest"] = np.array(tc.digest(e))

        # ---- the video block, restated around the unmodified functions
        pred_j3d, gt_j3d, masks = tc.video_set()
        for smooth in (True, False):
            accel_error, mpjpe_list, pa_mpjpe_list = [], [], []
            for vid_idx in masks:
                pred, gt = pred_j3d[vid_idx], gt_j3d[vid_idx]
                if smooth:
                    pred = smooth_utils.smooth_pose(pred, min_cutoff=0.004, beta=0.005)
                vid_acc_err = coord_utils.compute_error_accel(gt, pred)
                vid_acc_err = np.mean(vid_acc_err)
                accel_error.append(vid_acc_err)
                mpjpe = np.sqrt(np.sum((pred - gt) ** 2, 2))
                mpjpe_list.append(np.mean(mpjpe))
                for idx in range(len(pred)):
                    pa_pred = coord_utils.rigid_align(pred[idx], gt[idx])
                    pa_mpjpe = np.sqrt(np.sum((pa_pred - gt[idx]) ** 2, 1))
                    pa_mpjpe_list.append(pa_mpjpe)
            tag = "smooth" if smooth else "raw"
            out.update({f"vid_{tag}_accel": np.array(accel_error), f"vid_{tag}_mpjpe": np.array(mpjpe_list),
                        f"vid_{tag}_accel_total": np.mean(accel_error), f"vid_{tag}_mpjpe_total": np.mean(mpjpe_list),
                        f"vid_{tag}_pa_total": np.mean(pa_mpjpe_list)})
            if smooth:
                out["vid_smooth_pa"] = np.array(pa_mpjpe_list)
    path = os.path.join(HERE, "temporal.npz")
    save(path, out)
    print("wrote", path, os.path.getsize(path))


if __name__ == "__main__":
    main()
