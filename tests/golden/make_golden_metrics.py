#!/usr/bin/env python
"""Golden vectors of the reference's evaluation metrics, produced by the UNMODIFIED reference functions:
coord_utils.rigid_transform_3D / rigid_align (lib/coord_utils.py:127-149) and the compute_joint_err /
compute_both_err methods of Human36M, PW3D and SURREAL (data/*/dataset.py), called unbound on a stub `self` that
carries human36_eval_joint.  The dataset modules are imported with the packages they need for loading data but not
for these methods (pycocotools, transforms3d, smpl, ...) stubbed in sys.modules.  Also stores the reference's
J_regressor_h36m_correct.npy (a data file), so the end-to-end tests use a real regressor with its real row sums.

    P2M_REFERENCE_ROOT=/path/to/Pose2Mesh_RELEASE python tests/golden/make_golden_metrics.py -> eval_metrics.npz

Every input is float32-representable (the GPU gets the same values).  Procrustes case i: rt{i}_A, rt{i}_B [n, 3],
rt{i}_c, rt{i}_R, rt{i}_t and rt{i}_aligned on the rows rt{i}_rows (all rows up to n = 778, a seeded 256 of them
above, to keep the file small).  The per-point float32 errors ({set}_joint_pp, {set}_mesh_pp) restate the reference's
expression (np.power(np.power(p - g, 2).sum(axis=2), 0.5) after the torch root subtraction); the generator checks
that their float32 mean is bit for bit the reference method's return value.
"""
import importlib.util
import os
import sys
import types
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import ref_shim  # noqa: E402

H36M_EVAL_JOINT = (1, 2, 3, 4, 5, 6, 8, 10, 11, 12, 13, 14, 15, 16)


def _stub(name):
    mod = types.ModuleType(name)
    mod.__path__ = []
    mod.__getattr__ = lambda attr: (lambda *a, **k: None)
    sys.modules[name] = mod


def load_reference():
    ref_shim.load("human36")
    for name in ("transforms3d", "pycocotools", "pycocotools.coco", "smpl", "noise_utils", "aug_utils", "vis",
                 "funcs_utils", "smooth_utils", "Human36M", "Human36M.noise_stats"):
        try:
            if name in sys.modules:
                continue
            if name.split(".")[0] in ("Human36M",):
                raise ImportError
            __import__(name)
        except Exception:
            _stub(name)
    import coord_utils  # noqa: E402  (reference module, lib/coord_utils.py)

    classes = {}
    for ds, cls in (("Human36M", "Human36M"), ("PW3D", "PW3D"), ("SURREAL", "SURREAL")):
        path = os.path.join(ref_shim.REF_ROOT, "data", ds, "dataset.py")
        spec = importlib.util.spec_from_file_location(f"ref_dataset_{ds}", path)
        mod = importlib.util.module_from_spec(spec)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            spec.loader.exec_module(mod)
        classes[ds] = getattr(mod, cls)
    return coord_utils, classes


def f32(x):
    return np.asarray(x, dtype=np.float32).astype(np.float64)


def random_rotation(rng):
    q, r = np.linalg.qr(rng.standard_normal((3, 3)))
    q = q * np.sign(np.diag(r))
    return q if np.linalg.det(q) > 0 else -q


def procrustes_cases(rng):
    cases = []
    for scale in (1000.0, 1.0):
        for n in (14, 17, 778, 6890):
            A = f32(rng.standard_normal((n, 3)) * 0.3 * scale + rng.standard_normal(3) * scale)
            s = rng.uniform(0.7, 1.4)
            B = f32(s * A @ random_rotation(rng).T + rng.standard_normal(3) * scale
                    + 0.02 * scale * rng.standard_normal((n, 3)))
            cases.append((f"similarity_n{n}_{'mm' if scale > 1 else 'm'}", A, B))
    A = f32(rng.standard_normal((17, 3)) * 300.0)
    mirrored = A * np.array([-1.0, 1.0, 1.0]) + f32(5.0 * rng.standard_normal((17, 3)))
    cases.append(("mirrored", A, f32(mirrored)))
    cases.append(("identical", A, A.copy()))
    P = f32(np.concatenate([rng.standard_normal((17, 2)) * 300.0, np.zeros((17, 1))], axis=1))
    cases.append(("planar", P, f32(P @ random_rotation(rng).T * 1.1 + 40.0 + rng.standard_normal((17, 3)))))
    k = np.arange(-8, 9, dtype=np.float64)[:, None]
    L = f32(np.array([10.0, -20.0, 5.0]) + k * np.array([1.0, 2.0, -3.0]))
    cases.append(("collinear", L, f32(rng.standard_normal((17, 3)) * 100.0)))
    cases.append(("all_equal", f32(np.tile([1.5, -2.0, 3.25], (17, 1))), f32(rng.standard_normal((17, 3)))))
    return cases


def per_point_f32(pred, gt, root_p, root_g, subset):
    """The reference's expression: torch root subtraction, float32 numpy distances (dataset.py:455-462)."""
    p = (torch.from_numpy(pred) - torch.from_numpy(root_p)).numpy()
    g = (torch.from_numpy(gt) - torch.from_numpy(root_g)).numpy()
    if subset is not None:
        p, g = p[:, subset, :], g[:, subset, :]
    return np.power((np.power((p - g), 2)).sum(axis=2), 0.5)


if __name__ == "__main__":
    coord_utils, classes = load_reference()
    rng = np.random.default_rng(2024)
    out = {}
    names = []
    for i, (name, A, B) in enumerate(procrustes_cases(rng)):
        with warnings.catch_warnings(), np.errstate(all="ignore"):
            warnings.simplefilter("ignore")
            c, R, t = coord_utils.rigid_transform_3D(A.copy(), B.copy())
            aligned = coord_utils.rigid_align(A.copy(), B.copy())
        if name == "mirrored":  # the reference's det R < 0 branch must be taken on this case
            H = (A - A.mean(0)).T @ (B - B.mean(0)) / len(A)
            U, _, Vh = np.linalg.svd(H)
            assert np.linalg.det(Vh.T @ U.T) < 0, "mirrored case does not take the det < 0 branch"
        if name == "all_equal":
            assert np.isnan(c) and np.isnan(aligned).all()
        rows = np.arange(len(A)) if len(A) <= 778 else np.sort(rng.choice(len(A), 256, replace=False))
        out.update({f"rt{i}_A": A.astype(np.float32), f"rt{i}_B": B.astype(np.float32), f"rt{i}_c": np.float64(c),
                    f"rt{i}_R": R, f"rt{i}_t": t, f"rt{i}_rows": rows.astype(np.int32),
                    f"rt{i}_aligned": aligned[rows]})
        names.append(name)
    out["rt_names"] = np.array(names)

    stub = types.SimpleNamespace(human36_eval_joint=H36M_EVAL_JOINT)
    # (set, class, batch, n_joint, n_vertex, joint-err root, joint-err subset, both-err subset)
    sets = [("h36m", "Human36M", 2, 17, 1500, 0, H36M_EVAL_JOINT, H36M_EVAL_JOINT),
            ("pw3d", "PW3D", 2, 24, 778, -2, None, H36M_EVAL_JOINT),
            ("surreal", "SURREAL", 2, 17, 1000, 0, None, None)]
    for tag, cls, B, nj, nv, root, jsub, bsub in sets:
        pj = (rng.standard_normal((B, nj, 3)) * 300.0 + [0.0, 0.0, 4000.0]).astype(np.float32)
        gj = (pj + rng.standard_normal((B, nj, 3)) * 40.0).astype(np.float32)
        pm = (rng.standard_normal((B, nv, 3)) * 300.0 + [0.0, 0.0, 4000.0]).astype(np.float32)
        gm = (pm + rng.standard_normal((B, nv, 3)) * 40.0).astype(np.float32)
        C = classes[cls]
        jerr = C.compute_joint_err(stub, torch.from_numpy(pj), torch.from_numpy(gj))
        both_j, both_m = C.compute_both_err(stub, torch.from_numpy(pm), torch.from_numpy(gm), torch.from_numpy(pj),
                                            torch.from_numpy(gj))
        r = root % nj
        pp_joint = per_point_f32(pj, gj, pj[:, r:r + 1], gj[:, r:r + 1], list(jsub) if jsub else None)
        pp_bj = per_point_f32(pj, gj, pj[:, :1], gj[:, :1], list(bsub) if bsub else None)
        pp_mesh = per_point_f32(pm, gm, pj[:, :1], gj[:, :1], None)
        assert pp_joint.dtype == np.float32 and pp_joint.mean() == jerr
        assert pp_bj.mean() == both_j and pp_mesh.mean() == both_m
        out.update({f"{tag}_pred_joint": pj, f"{tag}_gt_joint": gj, f"{tag}_pred_mesh": pm, f"{tag}_gt_mesh": gm,
                    f"{tag}_joint_root": np.int32(root),
                    f"{tag}_joint_subset": np.array(jsub if jsub else [], dtype=np.int32),
                    f"{tag}_both_subset": np.array(bsub if bsub else [], dtype=np.int32),
                    f"{tag}_joint_err": np.float64(jerr), f"{tag}_both_joint_err": np.float64(both_j),
                    f"{tag}_both_mesh_err": np.float64(both_m),
                    f"{tag}_joint_pp": pp_joint, f"{tag}_both_joint_pp": pp_bj, f"{tag}_mesh_pp": pp_mesh})
    out["J_regressor_h36m"] = np.load(os.path.join(ref_shim.REF_ROOT, "data", "Human36M",
                                                   "J_regressor_h36m_correct.npy"))
    path = os.path.join(HERE, "eval_metrics.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path))
