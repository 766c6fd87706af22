"""The float64 body-model oracle (tests/body_model_oracle.py) against golden vectors of the unmodified reference layers
(tests/golden/body_model.npz, made by tests/golden/make_golden_body_model.py), the synthetic models' digests, mutated
oracles that the bound must reject, and the host-side behaviour of pose2mesh_release_b200.body_model."""
import numpy as np
import pytest
import torch
from torch.nn import Module

import body_model_oracle as bo
import body_models as bm
from helpers import load_npz
from pose2mesh_release_b200.body_model import ManoLayer, SMPLLayer

Z = load_npz("body_model.npz")
CASES = [str(s) for s in Z["cases"]]
BOUND = 2e-6  # of the sample's max |coordinate|; the reference's own fp32 rounding is below 1e-6 on these models


def models():
    out = {"smpl": bm.smpl_model()}
    for side in ("right", "left"):
        for flat in (False, True):
            out[f"mano_{side}" + ("_flat" if flat else "")] = bm.mano_model(side, flat)
    return out


MODELS = models()


def case(name):
    g = lambda k: Z[f"{name}__{k}"] if f"{name}__{k}" in Z.files else None  # noqa: E731
    center = int(Z[f"{name}__center"])
    return dict(model=str(Z[f"{name}__model"]), pose=g("pose"), betas=g("betas"), trans=g("trans"),
                center=None if center < 0 else center, rows=g("rows"), verts=g("verts"), joints=g("joints"))


def run_oracle(c, **mut):
    m = MODELS[c["model"]]
    fwd = bo.smpl_forward if c["model"] == "smpl" else bo.mano_forward
    return fwd(m, c["pose"], c["betas"], c["trans"], c["center"], **mut)


def ratio(c, verts, joints):
    """Worst error over the stored rows and joints, per sample in units of the sample's max |coordinate|."""
    v = verts[:, c["rows"]]
    scale = np.maximum(np.abs(c["verts"]).max(axis=(1, 2)), np.abs(c["joints"]).max(axis=(1, 2)))
    err = np.maximum(np.abs(v - c["verts"]).max(axis=(1, 2)), np.abs(joints - c["joints"]).max(axis=(1, 2)))
    return float(np.max(err / scale))


@pytest.mark.parametrize("name", sorted(MODELS))
def test_model_digest(name):
    assert bm.digest(MODELS[name]) == str(Z[f"digest_{name}"])


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference(name):
    c = case(name)
    assert ratio(c, *run_oracle(c)) <= BOUND


def _fails_somewhere(names, **mut):
    return max(ratio(case(n), *run_oracle(case(n), **mut)) for n in names)


def test_bound_rejects_dropped_pose_blend():
    assert _fails_somewhere(["smpl_random", "mano_right_random"], pose_blend=False) > 10 * BOUND


def test_bound_rejects_ignored_model_betas():
    assert _fails_somewhere(["smpl_zero_betas"], model_fallback=False) > 10 * BOUND
    assert _fails_somewhere(["smpl_no_betas"], model_fallback=False) <= BOUND  # absent betas need no fallback rule


def test_bound_rejects_missing_hands_mean():
    assert _fails_somewhere(["mano_right_random", "mano_left_random"], hands_mean=False) > 10 * BOUND


def test_bound_rejects_tf32_basis():
    assert _fails_somewhere(["smpl_random", "smpl_angles"], basis_round=bo.tf32_round) > BOUND


def test_bound_rejects_wrong_tip_vertex():
    assert _fails_somewhere(["mano_right_random"], tips=(745, 317, 445, 556, 673)) > 10 * BOUND
    assert _fails_somewhere(["mano_left_random"], tips=(745, 317, 444, 556, 673)) > 10 * BOUND


def test_zero_pose_rotation_is_identity():
    R = bo.rodrigues(np.zeros((3, 3)))
    assert np.array_equal(R, np.broadcast_to(np.eye(3), (3, 3, 3)))


def _smpl():
    m = MODELS["smpl"]
    return SMPLLayer(m["v_template"], m["shapedirs"], m["posedirs"], m["J_regressor"], m["weights"], m["parents"],
                     m["betas"])


def test_cpu_tensors_refused():
    layer = _smpl()
    with pytest.raises(RuntimeError, match="CUDA"):
        layer(torch.zeros(2, 72))
    m = MODELS["mano_right"]
    mano = ManoLayer(m["v_template"], m["shapedirs"], m["posedirs"], m["J_regressor"], m["weights"], m["betas"],
                     m["hands_mean"], flat_hand_mean=False)
    with pytest.raises(RuntimeError, match="CUDA"):
        mano(torch.zeros(2, 48))


def test_unsupported_mano_modes():
    m = MODELS["mano_right"]
    args = (m["v_template"], m["shapedirs"], m["posedirs"], m["J_regressor"], m["weights"], m["betas"], m["hands_mean"])
    for kw in ({"use_pca": True}, {"root_rot_mode": "ortho6d"}, {"joint_rot_mode": "rotmat"}, {"side": "middle"}):
        with pytest.raises(ValueError):
            ManoLayer(*args, **kw)
    layer = ManoLayer(*args)
    with pytest.raises(ValueError, match="root_palm"):
        layer(torch.zeros(1, 48), root_palm=torch.Tensor([1]))
    with pytest.raises(ValueError, match="share_betas"):
        layer(torch.zeros(1, 48), share_betas=torch.Tensor([1]))


def test_requires_grad_refused():
    with pytest.raises(RuntimeError, match="requires grad"):
        _smpl()(torch.zeros(1, 72, requires_grad=True))


class _StandIn(Module):
    """A stand-in for the reference layer classes: only the buffers and attributes forward reads."""


def test_from_reference_copies_every_buffer():
    m = MODELS["smpl"]
    ref = bm.smpl_reference_layer(_StandIn, m, center_idx=3, gender="female")
    layer = SMPLLayer.from_reference(ref)
    for name, buf in ref.named_buffers():
        if name != "th_faces":
            assert torch.equal(getattr(layer, name), buf), name
    assert ref.kintree_parents[0] == bm.SMPL_PKL_ROOT_PARENT  # the real pkl's root entry, ignored by the reference
    assert layer.kintree_parents == [-1] + ref.kintree_parents[1:] and layer.center_idx == 3 and layer.gender == "female"
    for flat in (False, True):
        mm = bm.mano_model("left", flat)
        ref = bm.mano_reference_layer(_StandIn, mm, center_idx=9, flat_hand_mean=flat)
        layer = ManoLayer.from_reference(ref)
        for name, buf in ref.named_buffers():
            if name not in ("th_faces", "th_selected_comps"):
                assert torch.equal(getattr(layer, name), buf), name
        assert layer.side == "left" and layer.flat_hand_mean == flat and layer.center_idx == 9
        assert np.array_equal(layer.th_hands_mean[0].numpy(), mm["hands_mean"])


def test_smpl_root_parent_entry_is_ignored():
    """The root's parent entry is never read by SMPL_Layer.forward; -1, 2^32 - 1 or anything else give the same tree."""
    m = MODELS["smpl"]
    for root in (-1, bm.SMPL_PKL_ROOT_PARENT, 0):
        ref = bm.smpl_reference_layer(_StandIn, m, root_parent=root)
        assert SMPLLayer.from_reference(ref).kintree_parents == list(bm.SMPL_PARENTS)
    pkl_row = np.array([bm.SMPL_PKL_ROOT_PARENT] + list(bm.SMPL_PARENTS[1:]), dtype=np.uint32)
    layer = SMPLLayer(m["v_template"], m["shapedirs"], m["posedirs"], m["J_regressor"], m["weights"], pkl_row,
                      m["betas"])
    assert layer.kintree_parents == list(bm.SMPL_PARENTS)
