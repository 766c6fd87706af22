#!/usr/bin/env python
"""Golden statistics of the training inputs' synthetic detector errors, produced from the UNMODIFIED reference:

    P2M_REFERENCE_ROOT=<checkout> python tests/golden/make_golden_inputs.py   ->  tests/golden/inputs.npz

synthesize_pose is the reference's lib/noise_utils.py, imported as it is (its only missing dependency, easydict, gets a
three-line shim).  Each case (joints [17, 3] in crop pixels, area) is run M times under np.random.seed / random.seed,
one call per sample as the datasets make it, and only the per-joint outcome statistics are stored (counts, not
samples): oracle/inputs_oracle.py's outcome_cells (annulus and radial bin) and offset_cells (offset from the joint over
ks10 on a grid, for sources that overlap).  Human36M.generate_syn_error (data/Human36M/dataset.py:143-155) is restated
below line for line (RESTATEMENT markers; the dataset module needs pycocotools) and run over M_H36M samples; its table
is the reference's data/Human36M/noise_stats.py, stored as data.

Keys: case_names [C], case_joints [C, 17, 3], case_area [C], M, ref_cells [C, 17, N_CELL], ref_offsets [C, 17,
N_CELL_2D] (int64 counts); kps_sigmas [17] (cfg.kps_sigmas); error_joint [17] (str), error_mean, error_std [17, 2],
error_weight [17] in noise_stats' order; h36m_joints_name [17] (Human36M's joint order, which get_stat sorts by);
h36m_M, h36m_kept [17], h36m_sum, h36m_sumsq [17, 2] (float64 sums over the kept draws, get_stat order).
"""
import multiprocessing as mp
import os
import random
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import inputs_oracle as io  # noqa: E402

REF = os.environ.get("P2M_REFERENCE_ROOT", "")
M = 5000
WORKERS = 8
M_H36M = 100000
H36M_JOINTS_NAME = ('Pelvis', 'R_Hip', 'R_Knee', 'R_Ankle', 'L_Hip', 'L_Knee', 'L_Ankle', 'Torso', 'Neck', 'Nose',
                    'Head', 'L_Shoulder', 'L_Elbow', 'L_Wrist', 'R_Shoulder', 'R_Elbow', 'R_Wrist')  # dataset.py:53-55

# a person in the 288 x 384 crop; at area 900 every symmetric pair is more than 2 ks10 apart
SKELETON = np.array([[144, 60], [156, 50], [132, 50], [172, 58], [116, 58], [190, 110], [98, 110], [215, 170],
                     [73, 170], [230, 230], [58, 230], [175, 230], [113, 230], [180, 300], [108, 300], [185, 365],
                     [103, 365]], np.float64)


def cases():
    def pose(visible, moves=()):
        j = np.zeros((17, 3))
        j[:, :2] = SKELETON
        j[list(visible), 2] = 1.0
        for k, xy in moves:
            j[k, :2] = xy
        return j

    every = range(17)
    return [
        ("all_visible", pose(every), 900.0),
        ("le10_visible", pose([0, 1, 3, 5, 6, 7, 11, 12, 13, 15]), 900.0),
        ("le5_visible", pose([0, 5, 6, 11, 16]), 900.0),
        ("invisible_partners", pose([j for j in every if j not in (2, 8, 12, 16)]), 900.0),
        # shoulders 6 px and hips 8 px apart: well inside ks10 (10.2 and 13.8 px), the sources overlap
        ("close_pairs", pose(every, [(5, (147, 110)), (6, (141, 110)), (11, (148, 230)), (12, (140, 230))]), 900.0),
    ]


def _import_noise_utils():
    shim = types.ModuleType("easydict")
    shim.EasyDict = type("EasyDict", (dict,), {"__getattr__": dict.__getitem__, "__setattr__": dict.__setitem__})
    sys.modules["easydict"] = shim
    sys.path.insert(0, os.path.join(REF, "lib"))
    import noise_utils
    return noise_utils


def _run(args):
    joints, area, seed, n = args
    nu = _import_noise_utils()
    np.random.seed(seed)
    random.seed(seed)
    return np.stack([nu.synthesize_pose(joints.copy(), area, num_overlap=0) for _ in range(n)])


# ---- RESTATEMENT of Human36M.generate_syn_error (data/Human36M/dataset.py:143-155) --------------------------------
def generate_syn_error(human36_error_distribution, human36_joint_num=17):
    noise = np.zeros((human36_joint_num, 2), dtype=np.float32)
    weight = np.zeros(human36_joint_num, dtype=np.float32)
    for i, ed in enumerate(human36_error_distribution):
        noise[i, 0] = np.random.normal(loc=ed['mean'][0], scale=ed['std'][0])
        noise[i, 1] = np.random.normal(loc=ed['mean'][1], scale=ed['std'][1])
        weight[i] = ed['weight']

    prob = np.random.uniform(low=0.0, high=1.0, size=human36_joint_num)
    weight = (weight > prob)
    noise = noise * weight[:, None]

    return noise, weight
# ---- end RESTATEMENT -----------------------------------------------------------------------------------------------


def main():
    if not REF or not os.path.isdir(os.path.join(REF, "lib")):
        raise SystemExit("set P2M_REFERENCE_ROOT to a Pose2Mesh_RELEASE checkout")
    nu = _import_noise_utils()
    sys.path.insert(0, os.path.join(REF, "data", "Human36M"))
    from noise_stats import error_distribution

    out = {}
    cs = cases()
    out["case_names"] = np.array([c[0] for c in cs])
    out["case_joints"] = np.stack([c[1] for c in cs])
    out["case_area"] = np.array([c[2] for c in cs])
    out["M"] = np.int64(M)
    cells, offs = [], []
    with mp.Pool(WORKERS) as pool:
        for ci, (name, joints, area) in enumerate(cs):
            per = M // WORKERS
            parts = pool.map(_run, [(joints, area, 1000 * ci + w, per) for w in range(WORKERS)])
            res = np.concatenate(parts)
            cells.append(io.histogram(io.outcome_cells(res, joints, area), io.N_CELL))
            offs.append(io.histogram(io.offset_cells(res, joints, area), io.N_CELL_2D))
            print(name, "zeroed per joint:", cells[-1][:, io.N_CELL - 2].tolist(), flush=True)
    out["ref_cells"], out["ref_offsets"] = np.stack(cells), np.stack(offs)
    out["kps_sigmas"] = np.asarray(nu.cfg.kps_sigmas, np.float64)

    out["error_joint"] = np.array([ed["Joint"] for ed in error_distribution])
    out["error_mean"] = np.array([ed["mean"] for ed in error_distribution], np.float64)
    out["error_std"] = np.array([ed["std"] for ed in error_distribution], np.float64)
    out["error_weight"] = np.array([ed["weight"] for ed in error_distribution], np.float64)
    out["h36m_joints_name"] = np.array(H36M_JOINTS_NAME)
    ordered = [next(ed for ed in error_distribution if ed["Joint"] == j) for j in H36M_JOINTS_NAME]  # get_stat
    np.random.seed(7)
    kept = np.zeros(17, np.int64)
    s, ss = np.zeros((17, 2)), np.zeros((17, 2))
    for _ in range(M_H36M):
        noise, w = generate_syn_error(ordered)
        kept += w
        s += np.where(w[:, None], noise, 0).astype(np.float64)
        ss += np.where(w[:, None], noise.astype(np.float64) ** 2, 0)
    out["h36m_M"], out["h36m_kept"], out["h36m_sum"], out["h36m_sumsq"] = np.int64(M_H36M), kept, s, ss
    path = os.path.join(HERE, "inputs.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
