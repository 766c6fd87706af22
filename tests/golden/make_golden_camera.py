#!/usr/bin/env python
"""Golden vectors for the demo's camera fit, produced by the UNMODIFIED reference functions:

    P2M_REFERENCE_ROOT=<checkout> python tests/golden/make_golden_camera.py   ->  tests/golden/camera_fit.npz

Reference functions used as they are (through oracle/ref_shim.py): coord_utils.get_bbox / process_bbox,
aug_utils.j2d_processing, models.project_net.get_model(500) and torch.optim.Adam.  demo/run.py itself cannot be
imported (it needs pyrender through its renderer), so the body of its loop (run.py:176-189, batch 1, CPU float32,
one thread) and convert_crop_cam_to_orig_img (run.py:24-43) are restated here line for line.

Cases, in order:
  0        the demo's own input (demo/h36m_joint_input.npy, int64) with the joints FlatPose2Mesh regresses from it:
           PoseNet and MeshNet of pose2mesh_net.get_model(17, smpl_small graph) under torch.manual_seed(123), BatchNorm
           statistics randomised with seed 3, the joint regressor torch.rand(17, 1200) (seed 6) normalised per row,
           all through the CPU oracles (oracle/demo_oracle.py, oracle/meshnet_oracle.py);
  1-31     17-joint H36M-style inputs [17, 2] (odd cases int64, even cases float64), projections of seeded 3-D joints
           through a seeded camera plus 3 px of noise;
  32-63    coco-style inputs [19, 3] float64: 17 joints with confidences, pelvis and neck appended (run.py:127-146);
  64       exact zero residuals: an int64 pose (integer crop targets) and 3-D joints chosen so that the initial camera
           (1, 0, 0) reproduces every target exactly in float32.
Every case draws its init from torch.rand((1, 3)) by constructing OptimzeCamLayer (torch.manual_seed(2024) first);
case 64 then sets its camera to (1, 0, 0).  Each case is fitted twice: as given, and with the float32 target scaled by
(1 + 2^-23) (one ulp); the spread of the two is the GPU tolerance's basis.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

from oracle import ref_shim  # noqa: E402

COCO_NAMES = ('Nose', 'L_Eye', 'R_Eye', 'L_Ear', 'R_Ear', 'L_Shoulder', 'R_Shoulder', 'L_Elbow', 'R_Elbow', 'L_Wrist',
              'R_Wrist', 'L_Hip', 'R_Hip', 'L_Knee', 'R_Knee', 'L_Ankle', 'R_Ankle', 'Pelvis', 'Neck')
CROP = 500


def add_pelvis_neck(j):
    """run.py:127-146 (add_pelvis, add_neck) on a [17, 3] coco pose."""
    out = j
    for a, b in (("L_Hip", "R_Hip"), ("L_Shoulder", "R_Shoulder")):
        ia, ib = COCO_NAMES.index(a), COCO_NAMES.index(b)
        p = (out[ia, :] + out[ib, :]) * 0.5
        p[2] = out[ia, 2] * out[ib, 2]
        out = np.concatenate((out, p.reshape(1, 3)))
    return out


def demo_joints(joint_input):
    from helpers import graph_from_fixture
    from oracle import demo_oracle as do
    from oracle import meshnet_oracle as mo
    from pose2mesh_release_b200 import pose2mesh_net

    mats, zg = graph_from_fixture("smpl_small")
    torch.manual_seed(123)
    flat = pose2mesh_net.get_model(17, mats)
    sd = {k: v.detach().clone() for k, v in flat.state_dict().items()}
    mo.randomize_bn_({("bn." + k): v for k, v in sd.items() if "batch_norm" in k or ".bn." in k}, seed=3)
    sd_p = {k[len("pose_lifter."):]: v for k, v in sd.items() if k.startswith("pose_lifter.")}
    sd_m = {k[len("pose2mesh."):]: v for k, v in sd.items() if k.startswith("pose2mesh.")}
    pose2d = torch.from_numpy(do.normalize_pose2d(joint_input))[None]
    jr = torch.rand(17, 1200, generator=torch.Generator().manual_seed(6))
    jr = jr / jr.sum(1, keepdim=True)
    with torch.no_grad():
        p3 = do.posenet_forward(sd_p, pose2d.reshape(1, -1))
        mesh = mo.forward(sd_m, mo.laplacians_to_torch(mats), do.flat_pose2mesh_input(pose2d, p3), training=False)
        _, joints = do.regress_joints(mesh, np.asarray(zg["perm_reverse"]), 1200, jr)
    return joints[0].numpy().astype(np.float32)


def synthetic_cases(n_h36m=31, n_coco=32):
    g = np.random.default_rng(77)
    inputs, p3ds = [], []
    for i in range(n_h36m + n_coco):
        p3d = (g.normal(0, 0.3, (17, 3))).astype(np.float32)
        s, t = g.uniform(0.6, 1.3), g.normal(0, 0.1, 2)
        S, O = g.uniform(80, 300), g.uniform(100, 600, 2)
        px = (p3d[:, :2] + t) * s * S + O + g.normal(0, 3, (17, 2))
        if i < n_h36m:
            inputs.append(np.round(px).astype(np.int64) if i % 2 == 0 else px.astype(np.float64))
        else:
            conf = g.uniform(0.05, 1.0, (17, 1))
            inputs.append(add_pelvis_neck(np.concatenate([px, conf], 1).astype(np.float64)))
        p3ds.append(p3d)
    return inputs, p3ds


def zero_residual_case():
    """A 17-joint layout for case 64 (its x, y are replaced by exact preimages of the reference's targets)."""
    k = np.arange(17)
    p3d = np.zeros((17, 3), np.float32)
    p3d[:, 0], p3d[:, 1] = (k - 8) / 8.0, ((k * 5) % 17 - 8) / 8.0
    return p3d


def reference_fit(p3d, target_f32, init):
    """run.py:161-189 on CPU with the reference's OptimzeCamLayer and torch.optim.Adam (batch 1)."""
    from models import project_net

    with torch.random.fork_rng():       # the global generator advances once per case, in main() only
        net = project_net.get_model(crop_size=CROP)
    with torch.no_grad():
        net.cam_param.copy_(torch.from_numpy(init[None]))
    pred_3d_joint = torch.from_numpy(p3d[None])
    target_joint = torch.from_numpy(target_f32[None, :, :2])
    criterion = torch.nn.L1Loss()
    optimizer = torch.optim.Adam(net.parameters(), lr=0.1)
    net.train()
    for j in range(0, 1500):
        pred_2d_joint = net(pred_3d_joint.detach())
        loss = criterion(pred_2d_joint, target_joint[:, :17, :])
        optimizer.zero_grad()
        loss.backward()
        optimizer.step()
        if j == 500:
            for param_group in optimizer.param_groups:
                param_group['lr'] = 0.05
        if j == 1000:
            for param_group in optimizer.param_groups:
                param_group['lr'] = 0.001
    with torch.no_grad():
        final = criterion(net(pred_3d_joint), target_joint[:, :17, :]).item()
    return net.cam_param[0].detach().numpy().copy(), np.float32(final)


def convert_crop_cam_to_orig_img(cam, bbox, img_width, img_height):
    """run.py:24-43, unchanged."""
    x, y, w, h = bbox[:, 0], bbox[:, 1], bbox[:, 2], bbox[:, 3]
    cx, cy, h = x + w / 2, y + h / 2, h
    hw, hh = img_width / 2., img_height / 2.
    sx = cam[:, 0] * (1. / (img_width / h))
    sy = cam[:, 0] * (1. / (img_height / h))
    tx = ((cx - hw) / hw / sx) + cam[:, 1]
    ty = ((cy - hh) / hh / sy) + cam[:, 2]
    return np.stack([sx, sy, tx, ty]).T


def main():
    torch.set_num_threads(1)
    ref_shim.load("human36")
    import aug_utils  # noqa: E402  (reference modules)
    import coord_utils  # noqa: E402
    from models import project_net  # noqa: E402

    joint_demo = np.load(os.path.join(ref_shim.REF_ROOT, "demo", "h36m_joint_input.npy"))
    inputs, p3ds = synthetic_cases()
    inputs = [joint_demo] + inputs
    p3ds = [demo_joints(joint_demo)] + p3ds
    # case 64: an int64 pose; its 3-D joints are fitted to the reference's crop target below
    zp = zero_residual_case()
    zero_in = np.round((zp[:, :2].astype(np.float64) * 250 + 250) * 0.8 + 40.0).astype(np.int64)   # integer targets
    inputs.append(zero_in)
    p3ds.append(zp)
    torch.manual_seed(2024)
    n = len(inputs)
    out = {k: [] for k in ("bbox", "target", "cam", "loss", "cam_pert", "loss_pert", "orig_cam", "init", "img_wh")}
    for i in range(n):
        joint_input = inputs[i]
        init = project_net.get_model(crop_size=CROP).cam_param.detach()[0].numpy().copy()   # torch.rand((1, 3))
        bbox1 = coord_utils.process_bbox(coord_utils.get_bbox(joint_input).copy(), aspect_ratio=1.0, scale=1.25)
        target, _ = aug_utils.j2d_processing(joint_input.copy(), (CROP, CROP), bbox1, 0, 0, None)
        p3d = p3ds[i]
        if i == n - 1:
            # rebuild the 3-D joints from the reference's target so the residuals at (1, 0, 0) are exactly zero
            p3d = p3d.copy()
            for idx in np.ndindex(17, 2):
                t = np.float32(target[idx])
                p0 = np.float32((np.float64(t) - 250) / 250)
                cands = [p0] + [np.nextafter(p0, np.float32(d * np.inf), dtype=np.float32) for d in (1, -1)]
                p3d[idx] = next(c for c in cands if np.float32(np.float32(c * np.float32(250)) + np.float32(250)) == t)
            assert np.array_equal((torch.from_numpy(p3d[None, :, :2]) * 1.0 * 250 + 250).numpy()[0], target[:, :2])
            p3ds[i] = p3d
            init = np.array([1, 0, 0], np.float32)
        cam, loss = reference_fit(p3d, target.astype(np.float32), init)
        tp = (torch.from_numpy(target[:, :2].astype(np.float32)) * (1 + 2 ** -23)).numpy()
        cam_p, loss_p = reference_fit(p3d, tp, init)
        wh = np.array([int(np.max(joint_input[:, 0]) * 1.5), int(np.max(joint_input[:, 1]) * 1.5)])   # run.py:232
        orig = convert_crop_cam_to_orig_img(cam[None], np.asarray(bbox1, np.float32)[None], int(wh[0]), int(wh[1]))
        for k, v in (("bbox", bbox1), ("target", target[:, :2]), ("cam", cam), ("loss", loss), ("cam_pert", cam_p),
                     ("loss_pert", loss_p), ("orig_cam", orig[0]), ("init", init), ("img_wh", wh)):
            out[k].append(np.asarray(v))
        print(i, joint_input.dtype, joint_input.shape, cam, loss, "spread", np.abs(cam - cam_p).max())
    arrays = {k: np.stack(v) for k, v in out.items() if k != "target"}
    arrays["bbox"] = arrays["bbox"].astype(np.float32)
    arrays["orig_cam"] = arrays["orig_cam"].astype(np.float32)
    # inputs of different row counts / dtypes: stored per group
    arrays["joints_demo"] = inputs[0]
    arrays["joints_h36m_int"] = np.stack([inputs[i] for i in range(1, 32) if inputs[i].dtype == np.int64])
    arrays["joints_h36m_f64"] = np.stack([inputs[i] for i in range(1, 32) if inputs[i].dtype == np.float64])
    arrays["joints_coco"] = np.stack(inputs[32:64])
    arrays["joints_zero"] = inputs[64]
    arrays["kind"] = np.array([0] + [1 if inputs[i].dtype == np.int64 else 2 for i in range(1, 32)] + [3] * 32 + [4])
    arrays["target_17"] = np.stack([t[:17] for t in out["target"]]).astype(np.float32)
    arrays["target_coco"] = np.stack(out["target"][32:64]).astype(np.float32)
    arrays["pred_joints3d"] = np.stack(p3ds).astype(np.float32)
    path = os.path.join(HERE, "camera_fit.npz")
    np.savez_compressed(path, **arrays)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
