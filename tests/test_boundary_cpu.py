"""CPU-only checks of the drop-in boundary: library loads and exports the C ABI, the module has the
reference's state_dict surface and initialiser, the native graph builder reproduces the reference's
hierarchy, the product path refuses to run without a GPU, and nothing in the product imports oracle/."""
import ast
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from helpers import CASES, graph_from_fixture, load_npz, tensor_digest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_loads_and_exports_header_symbols():
    from pose2mesh_release_b200 import _lib

    lib = _lib.load()
    header = open(os.path.join(ROOT, "include", "p2m_b200.h")).read()
    declared = set(re.findall(r"\b(p2m_[a-z0-9_]+)\s*\(", header))
    assert declared, "no declarations parsed"
    for name in sorted(declared):
        assert hasattr(lib, name), f"{name} declared in include/p2m_b200.h but not exported"
    assert set(_lib.EXPORTS) == declared
    assert b"sm_90a" in lib.p2m_version()


STATELESS = ["p2m_posenet_forward", "p2m_regress_joints", "p2m_normalize_pose2d", "p2m_mesh_losses", "p2m_coord_loss",
             "p2m_rigid_align", "p2m_point_errors", "p2m_nearest_distances", "p2m_align_w_scale", "p2m_pck_accumulate",
             "p2m_one_euro_smooth", "p2m_accel_error", "p2m_segment_mean", "p2m_fit_camera", "p2m_crop_cam_to_orig",
             "p2m_render_meshes"]


def _host_args(lib, keep):
    """The arguments (stream excluded) of every stateless entry point: valid sizes, and a zeroed host (numpy) array in
    every data-array slot.  Host-side tables (subsets, offsets, thresholds, schedules) are what they always are."""
    from pose2mesh_release_b200 import _lib

    def h(*shape, dtype=np.float32):
        a = np.zeros(shape, dtype)
        keep.append(a)
        return a.ctypes.data

    f64, i32, u8 = np.float64, np.int32, np.uint8
    F32 = _lib.P2M_DTYPE_F32
    B, J, V, F, H = 2, 4, 8, 3, 64        # batch, joints, vertices, faces, PoseNet width
    off = (C.c_int64 * 2)(0, 4)          # one sequence of four frames: two acceleration windows
    thr = (C.c_double * 2)(0.1, 0.2)
    lr_steps, lr_values = (C.c_int32 * 1)(0), (C.c_double * 1)(0.1)
    posenet = _lib.PoseNetParams(num_joint=J, hidden=H, num_stage=0, w1_w=h(H, 2 * J), w1_b=h(H), w2_w=h(3 * J, H),
                                 w2_b=h(3 * J))
    keep += [off, thr, lr_steps, lr_values, posenet]
    ws_pose, ws_render = lib.p2m_posenet_workspace_bytes(B, H), lib.p2m_render_workspace_bytes(1, 4, 4)
    return {
        "p2m_posenet_forward": (C.byref(posenet), h(B, 2 * J), h(B, 3 * J), h(B, J, 5), B, h(ws_pose, dtype=u8),
                                ws_pose),
        "p2m_regress_joints": (h(J, V), h(B, V, 3), h(B, J, 3), B, J, V, 3),
        "p2m_normalize_pose2d": (h(B, J, 2), h(B, J, 2), B, J, 384, 288, 0),
        "p2m_mesh_losses": (h(B, V, 3), h(B, V, 3), h(F, 3, dtype=i32), B, V, F, h(2), h(2, dtype=f64), h(B, V, 3)),
        "p2m_coord_loss": (h(B, J, 3), h(B, J, 3), h(B, J, 3), B * J * 3, h(1), h(1, dtype=f64), h(B, J, 3)),
        "p2m_rigid_align": (h(B, V, 3), h(B, V, 3), B, V, None, 0, h(B, 13, dtype=f64), h(B, V, 3), h(B, V),
                            h(B + 1, dtype=f64)),
        "p2m_point_errors": (h(B, V, 3), h(B, V, 3), h(B, 3), h(B, 3), B, V, None, 0, 0, h(B, V), h(B + 1, dtype=f64)),
        "p2m_nearest_distances": (F32, h(B, V, 3), h(B, V, 3), B, V, V, thr, 2, h(B, V, dtype=f64), h(B, V, dtype=f64),
                                  h(B, 2, 2, dtype=np.int64), h(B, 2, 2, dtype=f64), h(B, 2, dtype=f64)),
        "p2m_align_w_scale": (h(B, V, 3), h(B, V, 3), B, V, F32, h(B, V, 3), h(B, V, dtype=f64)),
        "p2m_pck_accumulate": (None, h(B * V, 3), h(B * V, 3), B * V, thr, 2, h(B * V, dtype=f64),
                               h(2, dtype=np.int64)),
        "p2m_one_euro_smooth": (F32, h(4, J, 3), h(4, J, 3), J * 3, off, 1, 4, 1.0, 0.0, 1.0),
        "p2m_accel_error": (F32, h(4, J, 3), h(4, J, 3), J, off, 1, 4, h(4, dtype=u8), h(2), h(2, dtype=u8),
                            h(1, dtype=f64)),
        "p2m_segment_mean": (F32, h(4, 3), 3, off, 1, 4, h(4, dtype=u8), h(1, dtype=f64)),
        "p2m_fit_camera": (h(B, J, 2, dtype=f64), 2, _lib.P2M_CAM_INPUT_F64, J, h(B, J, 3), J, h(B, 3), B, 500, 10,
                           lr_steps, lr_values, 1, h(B, 2), h(B, 3), h(B, 4), h(B, J, 2), h(B), h(B, 4)),
        "p2m_crop_cam_to_orig": (h(B, 3), h(B, 4), h(B, 2), B, h(B, 4)),
        "p2m_render_meshes": (h(B, V, 3), B, V, h(F, 3, dtype=i32), F, h(B, 4), h(B, 3), h(B, dtype=i32),
                              h(1, 4, 4, 3, dtype=u8), 1, 4, 4, h(1, 4, 4, 3, dtype=u8), h(1, 4, 4, dtype=i32),
                              h(1, 4, 4, dtype=i32), h(1, 4, 4), h(ws_render // 8, dtype=np.uint64), ws_render),
    }


@pytest.mark.parametrize("name", STATELESS)
def test_stateless_entry_point_rejects_host_arrays(name):
    """A stateless entry point runs on the device of its data arrays, so it checks them before any CUDA work: host
    memory in every data-array slot is P2M_ERR_INVALID naming the call.  Skipped with a GPU, where an entry point
    without the check would launch kernels on host pointers."""
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from pose2mesh_release_b200 import _lib

    lib = _lib.load()
    keep = []
    status = getattr(lib, name)(*_host_args(lib, keep)[name], None)
    msg = lib.p2m_last_error().decode()
    assert status == 1, (status, msg)
    assert name[len("p2m_"):] in msg and "device memory" in msg, msg


def test_conv_kernel_register_split_is_balanced_in_the_build():
    """k_cheb_conv_umma redistributes registers between its warpgroups with setmaxnreg (csrc/cheb_umma.cu: REGS_*): the
    epilogue's setmaxnreg.inc draws on exactly what the utility warpgroup's setmaxnreg.dec released, which only works
    out if every instantiation is LAUNCHED with 80 registers per thread.  The host refuses to launch otherwise
    (check_launch_regs); this catches such a build here, without a GPU."""
    import shutil
    import subprocess

    from pose2mesh_release_b200 import build

    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    lib = build.build()
    out = subprocess.run([cuobjdump, "-res-usage", lib], capture_output=True, text=True).stdout
    regs = re.findall(r"Function [^\n]*k_cheb_conv_umma[^\n]*\n[^\n]*REG:(\d+)", out)
    assert len(regs) >= 4, f"conv kernel instantiations not found in {lib}"
    assert set(regs) == {"80"}, f"launch register counts of k_cheb_conv_umma: {sorted(set(regs))}"
    src = open(os.path.join(ROOT, "pose2mesh_release_b200", "csrc", "cheb_umma.cu")).read()
    m = re.search(r"REGS_LAUNCH = (\d+), REGS_UTIL = (\d+), REGS_EPI = (\d+)", src)
    launch, util, epi = (int(v) for v in m.groups())
    assert launch == 80 and epi - launch <= launch - util and util % 8 == 0 and epi % 8 == 0


def test_build_refuses_a_listed_source_that_does_not_exist(monkeypatch):
    """A stale name in build.SOURCES (a renamed file) would otherwise give a library without that file's symbols, which
    fails only when they are looked up: build() raises before any compiler runs."""
    import subprocess

    from pose2mesh_release_b200 import build

    def compiler(*args, **kwargs):
        raise AssertionError(f"a compiler ran: {args}")

    monkeypatch.setattr(build, "SOURCES", build.SOURCES + ["no_such_file.cu"])
    monkeypatch.setattr(subprocess, "Popen", compiler)
    monkeypatch.setattr(subprocess, "run", compiler)
    with pytest.raises(FileNotFoundError, match="no_such_file.cu"):
        build.build(force=True)


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "pose2mesh_release_b200")
    for fn in os.listdir(pkg):
        if not fn.endswith(".py"):
            continue
        tree = ast.parse(open(os.path.join(pkg, fn)).read())
        for node in ast.walk(tree):
            names = []
            if isinstance(node, ast.Import):
                names = [a.name for a in node.names]
            elif isinstance(node, ast.ImportFrom):
                names = [node.module or ""]
            assert not any(n.split(".")[0] == "oracle" for n in names), f"{fn} imports oracle"


@pytest.mark.parametrize("name", ["smpl_small", "mano_like"])
def test_module_state_dict_surface_and_init(name):
    from pose2mesh_release_b200.meshnet import Pose2Mesh

    n, seed, levels, mano = CASES[name]
    z = load_npz(f"meshnet_{name}.npz")
    mats, _ = graph_from_fixture(name)
    n_before = len(mats)
    torch.manual_seed(123)
    model = Pose2Mesh(5, 3, mats, joint_set="mano" if mano else "human36")
    assert len(mats) == n_before, "caller's list must not be mutated"
    sd = model.state_dict()
    assert sorted(sd.keys()) == [str(k) for k in z["keys"]]
    assert sum(p.numel() for p in model.parameters()) == int(z["n_param"])
    for k, v in sd.items():
        assert tuple(v.shape) == tuple(z["shape/" + k]), k
        np.testing.assert_allclose(tensor_digest(v), z["init/" + k], rtol=1e-12, atol=0, err_msg=k)
    last = len(model.cl) - 1
    assert model.bn[last] is None and f"bn.{last}.weight" not in sd
    # reference-style checkpoints load (keys identical), incl. the DataParallel 'module.'-stripped form
    model.load_state_dict({k: v.clone() for k, v in sd.items()})


def test_forward_refuses_cpu_tensors():
    from pose2mesh_release_b200.meshnet import Pose2Mesh

    mats, _ = graph_from_fixture("mano_like")
    model = Pose2Mesh(5, 3, mats, joint_set="mano")
    with pytest.raises(RuntimeError, match="CUDA"):
        model(torch.zeros(1, 21, 5))


@pytest.mark.parametrize("name", ["smpl_small", "mano_like", "smpl_like"])
def test_native_graph_builder_matches_reference_fixture(name):
    import hashlib

    from pose2mesh_release_b200 import graph as pg

    def sha(a):
        return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()

    n, seed, levels, mano = CASES[name]
    z = load_npz(f"graph_{name}.npz")
    face = pg.synthetic_sphere_faces(n, seed)
    j, sk, fp = (21, pg.MANO_SKELETON, pg.MANO_HORI_CONN) if mano else (17, pg.H36M_SKELETON, pg.H36M_FLIP_PAIRS)
    adj, lap, perm, perm_rev = pg.build_coarse_graphs(face, j, sk, fp, levels=levels)
    assert np.array_equal(np.asarray(perm_rev), z["perm_reverse"])
    for i, m in enumerate(lap):
        c = m.tocsr()
        c.sort_indices()
        assert c.nnz == int(z[f"L{i}_nnz"])
        assert sha(c.indptr.astype(np.int64)) == str(z[f"L{i}_indptr_sha"])
        assert sha(c.indices.astype(np.int64)) == str(z[f"L{i}_indices_sha"])
        ref = z[f"L{i}_data32_sum"]
        assert abs(np.abs(c.data.astype(np.float32)).astype(np.float64).sum() - ref[1]) <= 1e-6 * ref[1]


def test_compute_perm_known_answer_native():
    from pose2mesh_release_b200 import graph as pg

    got = pg.compute_perm([np.array([4, 1, 1, 2, 2, 3, 0, 0, 3]), np.array([2, 1, 0, 1, 0])])
    assert got == [[3, 4, 0, 9, 1, 2, 5, 8, 6, 7, 10, 11], [2, 4, 1, 3, 0, 5], [0, 1, 2]]   # lib/coarsening.py:261-262


def test_model_create_without_gpu_fails_loudly():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from pose2mesh_release_b200.meshnet import Pose2Mesh

    mats, _ = graph_from_fixture("mano_like")
    model = Pose2Mesh(5, 3, mats, joint_set="mano")
    with pytest.raises(RuntimeError, match="no usable CUDA device|no CPU path"):
        model._hier.handle(0)
