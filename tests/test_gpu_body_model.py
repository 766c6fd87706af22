"""The batched body-model layers (pose2mesh_release_b200.body_model) on the GPU, through the public modules:

  * accuracy against the float64 oracle (4e-6 of each sample's max |coordinate|) and against the unmodified
    reference's float32 outputs in tests/golden/body_model.npz (5e-6), for SMPL at B in {1, 15, 16, 17, 256, 1000}
    (the 16-sample groups' edges), MANO at B in {1, 1024} and every quirk case of the fixture;
  * bitwise determinism, batch-position invariance, NaN isolation and CUDA-graph replay; at most three launches;
  * argument errors, the drop-in from_reference path, and targets fed to MeshLosses / evaluate_meshes.
"""
import os
import sys

import numpy as np
import pytest
import torch
from torch.nn import Module

import body_model_oracle as bo
import body_models as bm
from test_body_model_cpu import CASES, MODELS, case

from pose2mesh_release_b200 import _lib
from pose2mesh_release_b200.body_model import ManoLayer, SMPLLayer, _BodyModel

pytestmark = pytest.mark.gpu
ORACLE_BOUND = 4e-6
GOLDEN_BOUND = 5e-6


def dev():
    return torch.device("cuda:0")


def smpl_layer(center_idx=None):
    m = MODELS["smpl"]
    return SMPLLayer(m["v_template"], m["shapedirs"], m["posedirs"], m["J_regressor"], m["weights"], m["parents"],
                     m["betas"], center_idx=center_idx)


def mano_layer(key, center_idx=None):
    m = MODELS[key]
    return ManoLayer(m["v_template"], m["shapedirs"], m["posedirs"], m["J_regressor"], m["weights"], m["betas"],
                     m["hands_mean"], center_idx=center_idx, flat_hand_mean=key.endswith("_flat"), side=m["side"])


def layer_for(key, center_idx=None):
    return smpl_layer(center_idx) if key == "smpl" else mano_layer(key, center_idx)


def cuda(a):
    return None if a is None else torch.as_tensor(np.asarray(a, np.float32)).to(dev())


def run(layer, pose, betas=None, trans=None):
    kw = {}
    if betas is not None:
        kw["th_betas"] = cuda(betas)
    if trans is not None:
        kw["th_trans"] = cuda(trans)
    v, j = layer(cuda(pose), **kw)
    torch.cuda.synchronize()
    return v.cpu().numpy().astype(np.float64), j.cpu().numpy().astype(np.float64)


def worst(got, ref):
    """Largest per-sample error in units of the sample's max |coordinate| (vertices and joints together)."""
    (gv, gj), (rv, rj) = got, ref
    scale = np.maximum(np.abs(rv).max(axis=(1, 2)), np.abs(rj).max(axis=(1, 2)))
    err = np.maximum(np.abs(gv - rv).max(axis=(1, 2)), np.abs(gj - rj).max(axis=(1, 2)))
    return float(np.max(err / scale))


def oracle(key, pose, betas=None, trans=None, center_idx=None):
    fwd = bo.smpl_forward if key == "smpl" else bo.mano_forward
    return fwd(MODELS[key], pose, betas, trans, center_idx)


def random_inputs(key, B, seed):
    rng = np.random.RandomState(seed)
    width = 72 if key == "smpl" else 48
    pose = rng.normal(0.0, 0.6, (B, width)).astype(np.float32)
    betas = rng.normal(0.0, 1.5, (B, 10)).astype(np.float32)
    trans = rng.normal(0.0, 0.5 if key == "smpl" else 0.1, (B, 3)).astype(np.float32)
    return pose, betas, trans


# ------------------------------------------------------------------------------------------------ accuracy
@pytest.mark.parametrize("name", CASES)
def test_golden_case(name):
    c = case(name)
    layer = layer_for(c["model"], c["center"])
    got = run(layer, c["pose"], c["betas"], c["trans"])
    assert worst(got, oracle(c["model"], c["pose"], c["betas"], c["trans"], c["center"])) <= ORACLE_BOUND
    rows = c["rows"]
    assert worst((got[0][:, rows], got[1]), (c["verts"], c["joints"])) <= GOLDEN_BOUND


@pytest.mark.parametrize("B", [1, 15, 16, 17, 256, 1000])
def test_smpl_batch_sizes(B):
    pose, betas, trans = random_inputs("smpl", B, seed=B)
    assert worst(run(smpl_layer(), pose, betas, trans), oracle("smpl", pose, betas, trans)) <= ORACLE_BOUND


@pytest.mark.parametrize("B", [1, 1024])
@pytest.mark.parametrize("key", ["mano_right", "mano_left_flat"])
def test_mano_batch_sizes(key, B):
    pose, betas, trans = random_inputs(key, B, seed=B + 7)
    assert worst(run(mano_layer(key), pose, betas, trans), oracle(key, pose, betas, trans)) <= ORACLE_BOUND


def test_zero_pose_is_rest_pose():
    """A zero pose gives R = I exactly: no NaN, and the pose blend is exactly zero."""
    layer = smpl_layer()
    v, j = run(layer, np.zeros((2, 72)), np.zeros((2, 10)))
    assert np.isfinite(v).all() and np.isfinite(j).all()
    assert worst((v, j), oracle("smpl", np.zeros((2, 72)))) <= ORACLE_BOUND


def test_center_on_tip_vertex_is_exactly_zero():
    layer = mano_layer("mano_right", center_idx=4)  # output joint 4: the thumb tip, a vertex
    pose, betas, _ = random_inputs("mano_right", 3, seed=5)
    v, j = run(layer, pose, betas)
    assert np.all(j[:, 4] == 0.0) and np.all(v[:, 745] == 0.0)


# ------------------------------------------------------------------------------------------------ determinism
def test_bitwise_deterministic():
    layer = smpl_layer()
    pose, betas, trans = random_inputs("smpl", 64, seed=1)
    a, b = run(layer, pose, betas, trans), run(layer, pose, betas, trans)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


@pytest.mark.parametrize("key", ["smpl", "mano_right"])
def test_batch_position_invariance(key):
    layer = layer_for(key)
    pose, betas, trans = random_inputs(key, 256, seed=3)
    ref = run(layer, pose[:1], betas[:1], trans[:1])
    for pos in (0, 15, 16, 17, 255):
        p, b, t = pose.copy(), betas.copy(), trans.copy()
        p[pos], b[pos], t[pos] = pose[0], betas[0], trans[0]
        got = run(layer, p, b, t)
        assert np.array_equal(got[0][pos], ref[0][0]) and np.array_equal(got[1][pos], ref[1][0]), pos
    for B in (17, 40):  # the same sample in a smaller batch
        got = run(layer, pose[:B], betas[:B], trans[:B])
        assert np.array_equal(got[0][0], ref[0][0]) and np.array_equal(got[1][0], ref[1][0])


def test_nan_isolation():
    layer = smpl_layer()
    pose, betas, trans = random_inputs("smpl", 40, seed=4)
    ref = run(layer, pose, betas, trans)
    bad = pose.copy()
    bad[17, 5] = np.nan
    got = run(layer, bad, betas, trans)
    keep = np.arange(40) != 17
    assert np.array_equal(got[0][keep], ref[0][keep]) and np.array_equal(got[1][keep], ref[1][keep])
    assert np.isnan(got[0][17]).all()


def test_cuda_graph_replay_matches_eager():
    layer = smpl_layer(center_idx=0)
    pose, betas, trans = (cuda(a) for a in random_inputs("smpl", 32, seed=6))
    zero = torch.zeros_like(trans)
    eager = [t.clone() for t in layer(pose, betas, zero)] + [t.clone() for t in layer(pose, betas, trans)]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):  # warm-up: the handle is created outside the capture
        layer(pose, betas, trans)
    torch.cuda.current_stream().wait_stream(s)
    trans_in = trans.clone()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = layer(pose, betas, trans_in)
    for t in (zero, trans):  # the device-side trans test follows the data at replay
        trans_in.copy_(t)
        g.replay()
        torch.cuda.synchronize()
        ev = eager[:2] if t is zero else eager[2:]
        assert torch.equal(out[0], ev[0]) and torch.equal(out[1], ev[1])


@pytest.mark.parametrize("key", ["smpl", "mano_right"])
def test_at_most_three_launches(key):
    layer = layer_for(key)
    pose, betas, trans = (cuda(a) for a in random_inputs(key, 8, seed=2))
    layer(pose, betas, trans)
    lib = _lib.load()
    lib.p2m_launch_count_reset()
    layer(pose, betas, trans)
    assert lib.p2m_launch_count() <= 3


# ------------------------------------------------------------------------------------------------ quirks
def test_smpl_zero_betas_batch_uses_model_betas_on_device():
    layer = smpl_layer()
    pose, betas, trans = random_inputs("smpl", 5, seed=9)
    zero = np.zeros_like(betas)
    got = run(layer, pose, zero, trans)
    assert worst(got, oracle("smpl", pose, None, trans)) <= ORACLE_BOUND
    one = zero.copy()
    one[3, 2] = 0.5  # one non-zero value anywhere: every sample uses its own betas
    assert worst(run(layer, pose, one, trans), oracle("smpl", pose, one, trans)) <= ORACLE_BOUND
    nan = zero.copy()
    nan[1, 0] = np.nan  # NaN counts as non-zero, as in the reference
    got = run(layer, pose, nan, trans)
    assert np.isnan(got[0][1]).all()
    ref = bo.smpl_forward(MODELS["smpl"], pose, zero, trans, model_fallback=False)  # the given (zero) betas
    keep = [0, 2, 3, 4]
    assert worst((got[0][keep], got[1][keep]), (ref[0][keep], ref[1][keep])) <= ORACLE_BOUND


@pytest.mark.parametrize("B", [4000, 40000])
def test_batch_flags_see_the_last_sample(B):
    """The batch-wide tests are split over several CTAs at these sizes; one non-zero value in the last sample alone must
    switch every sample to its given betas and to translation instead of centring."""
    layer = smpl_layer(center_idx=0)
    rng = np.random.RandomState(B)
    pose = cuda(rng.normal(0.0, 0.6, (B, 72)))
    zero_b, zero_t = torch.zeros(B, 10, device=dev()), torch.zeros(B, 3, device=dev())
    last_b, last_t = zero_b.clone(), zero_t.clone()
    last_b[-1, 3], last_t[-1, 1] = 0.7, 0.2
    p0 = pose[:1].cpu().numpy()
    m = MODELS["smpl"]
    for betas, trans, ref in ((zero_b, zero_t, bo.smpl_forward(m, p0, None, None, 0)),
                              (last_b, last_t, bo.smpl_forward(m, p0, np.zeros((1, 10)), np.zeros((1, 3)), None,
                                                               model_fallback=False))):
        v, j = layer(pose, betas, trans)
        got = (v[:1].cpu().numpy().astype(np.float64), j[:1].cpu().numpy().astype(np.float64))
        assert worst(got, ref) <= ORACLE_BOUND
        del v, j


def test_mano_explicit_zero_betas_used_as_given():
    layer = mano_layer("mano_right")
    pose, betas, trans = random_inputs("mano_right", 4, seed=10)
    zero = np.zeros_like(betas)
    got = run(layer, pose, zero, trans)
    assert worst(got, oracle("mano_right", pose, zero, trans)) <= ORACLE_BOUND
    assert worst(run(layer, pose, None, trans), oracle("mano_right", pose, None, trans)) <= ORACLE_BOUND


@pytest.mark.parametrize("key,center", [("smpl", 0), ("smpl", 7), ("mano_left", 0), ("mano_right", 9),
                                        ("mano_right", -1)])
def test_zero_trans_centres(key, center):
    layer = layer_for(key, center)
    pose, betas, trans = random_inputs(key, 3, seed=11)
    zero = np.zeros_like(trans)
    ref_center = center % (24 if key == "smpl" else 21)
    assert worst(run(layer, pose, betas, zero), oracle(key, pose, betas, zero, ref_center)) <= ORACLE_BOUND
    assert worst(run(layer, pose, betas), oracle(key, pose, betas, None, ref_center)) <= ORACLE_BOUND
    # a non-zero trans in any sample: trans is added everywhere and nothing is centred
    some = zero.copy()
    some[2, 1] = 0.25
    assert worst(run(layer, pose, betas, some), oracle(key, pose, betas, some, ref_center)) <= ORACLE_BOUND


# ------------------------------------------------------------------------------------------------ errors
def test_argument_errors():
    layer = smpl_layer()
    pose, betas, trans = (cuda(a) for a in random_inputs("smpl", 4, seed=12))
    with pytest.raises(ValueError):
        layer(pose, betas[:3])
    with pytest.raises(ValueError):
        layer(pose[:, :69], betas)
    with pytest.raises(ValueError):
        layer(pose, betas, trans[:2])
    with pytest.raises(ValueError):
        layer(pose[:0])
    with pytest.raises(RuntimeError, match="requires grad"):
        layer(pose.clone().requires_grad_(True), betas)
    with pytest.raises(RuntimeError, match="requires grad"):
        layer(pose, betas.clone().requires_grad_(True))
    mano = mano_layer("mano_right")
    with pytest.raises(ValueError):
        mano(cuda(np.zeros((2, 45))))
    with pytest.raises(ValueError, match="root_palm"):
        mano(cuda(np.zeros((2, 48))), root_palm=torch.Tensor([1]))
    with pytest.raises(ValueError):
        bm_args = MODELS["mano_right"]
        ManoLayer(bm_args["v_template"], bm_args["shapedirs"], bm_args["posedirs"], bm_args["J_regressor"],
                  bm_args["weights"], bm_args["betas"], bm_args["hands_mean"], use_pca=True)


def _create_error(parents=None, joint_map=None, poison=None):
    m = dict(MODELS["smpl"])
    if poison:
        m[poison] = m[poison].copy()
        m[poison].flat[5] = np.inf
    parents = list(m["parents"]) if parents is None else parents
    jm = list(range(24)) if joint_map is None else joint_map
    layer = _BodyModel(m["v_template"], m["shapedirs"], m["posedirs"], m["J_regressor"], m["weights"], parents,
                       m["betas"], None, jm, 1.0, None)
    with pytest.raises(RuntimeError, match="p2m_body_model_create") as e:
        layer.handle(0)
    return str(e.value)


def test_create_rejects_bad_models():
    p = list(MODELS["smpl"]["parents"])
    assert "parents[0]" in _create_error(parents=[0] + p[1:])
    assert "topological" in _create_error(parents=p[:5] + [7] + p[6:])
    assert "topological" in _create_error(parents=p[:5] + [5] + p[6:])
    assert "joint_map" in _create_error(joint_map=list(range(23)) + [24])
    assert "joint_map" in _create_error(joint_map=list(range(23)) + [-6891])
    assert "non-finite" in _create_error(poison="posedirs")
    assert "non-finite" in _create_error(poison="weights")


# ------------------------------------------------------------------------------------------------ drop-in
class _OracleStandIn(Module):
    """Stands in for the reference layer classes when the reference is not importable: built like the golden
    generator builds SMPL_Layer / ManoLayer (tests/body_models.py), its forward is the oracle on its own buffers."""

    def forward(self, pose, th_betas=None, th_trans=None):
        model = {k: getattr(self, "th_" + k).numpy() for k in ("shapedirs", "posedirs", "J_regressor", "weights")}
        model.update(v_template=self.th_v_template.numpy()[0], betas=self.th_betas.numpy()[0])
        b = None if th_betas is None else th_betas.numpy()
        t = None if th_trans is None else th_trans.numpy()
        if hasattr(self, "th_hands_mean"):
            model.update(hands_mean=self.th_hands_mean.numpy()[0], side=self.side)
            out = bo.mano_forward(model, pose.numpy(), b, t, self.center_idx)
        else:
            model["parents"] = np.array([-1] + list(self.kintree_parents[1:]))  # forward never reads the root's entry
            out = bo.smpl_forward(model, pose.numpy(), b, t, self.center_idx)
        return tuple(torch.from_numpy(o.astype(np.float32)) for o in out)


def _reference_classes():
    root = os.environ.get("P2M_REFERENCE_ROOT", "")
    if root and os.path.isdir(os.path.join(root, "smplpytorch")):
        sys.path[:0] = [os.path.join(root, "smplpytorch"), os.path.join(root, "manopth")]
        from manopth.manolayer import ManoLayer as RefMano
        from smplpytorch.pytorch.smpl_layer import SMPL_Layer as RefSMPL
        return RefSMPL, RefMano
    return _OracleStandIn, _OracleStandIn


@pytest.mark.parametrize("key,center", [("smpl", None), ("smpl", 0), ("mano_right", None), ("mano_left_flat", 9)])
def test_from_reference_drop_in(key, center):
    ref_smpl, ref_mano = _reference_classes()
    m = MODELS[key]
    if key == "smpl":
        ref = bm.smpl_reference_layer(ref_smpl, m, center_idx=center)
    else:
        ref = bm.mano_reference_layer(ref_mano, m, center_idx=center, flat_hand_mean=key.endswith("_flat"))
    layer = (SMPLLayer if key == "smpl" else ManoLayer).from_reference(ref)
    pose, betas, trans = random_inputs(key, 6, seed=13)
    if center is not None:
        trans = np.zeros_like(trans)
    with torch.no_grad():
        rv, rj = ref(torch.from_numpy(pose), th_betas=torch.from_numpy(betas), th_trans=torch.from_numpy(trans))
    got = run(layer, pose, betas, trans)
    assert worst(got, (rv.double().numpy(), rj.double().numpy())) <= GOLDEN_BOUND


class _BuffersOnly(Module):
    """A layer object carrying only the buffers and attributes the reference layers hold (no forward)."""


@pytest.mark.parametrize("name", CASES)
def test_from_reference_matches_reference_outputs(name):
    """from_reference on a layer built exactly as the golden generator built the unmodified SMPL_Layer / ManoLayer
    (SMPL's root parent entry 2^32 - 1, as in the pkl), against that reference layer's own float32 outputs."""
    c = case(name)
    m = MODELS[c["model"]]
    if c["model"] == "smpl":
        ref = bm.smpl_reference_layer(_BuffersOnly, m, center_idx=c["center"])
        layer = SMPLLayer.from_reference(ref)
    else:
        ref = bm.mano_reference_layer(_BuffersOnly, m, center_idx=c["center"],
                                      flat_hand_mean=c["model"].endswith("_flat"))
        layer = ManoLayer.from_reference(ref)
    got = run(layer, c["pose"], c["betas"], c["trans"])
    assert worst((got[0][:, c["rows"]], got[1]), (c["verts"], c["joints"])) <= GOLDEN_BOUND


# ------------------------------------------------------------------------------------------------ handles
def test_handles_of_different_sizes_in_any_order():
    """SMPL and MANO handles need different shared-memory sizes; using them interleaved, and creating the smaller model
    after the larger one, must work in every order."""
    pose_s, betas_s, trans_s = random_inputs("smpl", 20, seed=21)
    pose_m, betas_m, trans_m = random_inputs("mano_right", 20, seed=22)
    ref_s, ref_m = oracle("smpl", pose_s, betas_s, trans_s), oracle("mano_right", pose_m, betas_m, trans_m)
    mano = mano_layer("mano_right")
    assert worst(run(mano, pose_m, betas_m, trans_m), ref_m) <= ORACLE_BOUND  # MANO handle first
    smpl = smpl_layer()
    first = run(smpl, pose_s, betas_s, trans_s)
    assert worst(first, ref_s) <= ORACLE_BOUND
    mano2 = mano_layer("mano_right")  # a MANO handle created after the SMPL one
    for _ in range(2):
        assert worst(run(mano2, pose_m, betas_m, trans_m), ref_m) <= ORACLE_BOUND
        again = run(smpl, pose_s, betas_s, trans_s)
        assert np.array_equal(again[0], first[0]) and np.array_equal(again[1], first[1])
        assert worst(run(mano, pose_m, betas_m, trans_m), ref_m) <= ORACLE_BOUND


def test_load_state_dict_rebuilds_the_handle():
    layer = smpl_layer()
    pose, _, trans = random_inputs("smpl", 4, seed=23)
    run(layer, pose, None, trans)  # the handle now exists on this device
    m2 = dict(MODELS["smpl"], betas=(MODELS["smpl"]["betas"] * -1.5).astype(np.float32))
    sd = layer.state_dict()
    sd["th_betas"] = torch.from_numpy(m2["betas"])[None]
    layer.load_state_dict(sd)
    assert worst(run(layer, pose, None, trans), bo.smpl_forward(m2, pose, None, trans)) <= ORACLE_BOUND
    layer.th_v_template[0, :, 1] += 0.5  # an in-place edit reaches the device after refresh()
    layer.refresh()
    m3 = dict(m2, v_template=layer.th_v_template[0].numpy())
    assert worst(run(layer, pose, None, trans), bo.smpl_forward(m3, pose, None, trans)) <= ORACLE_BOUND


# ------------------------------------------------------------------------------------------------ end to end
def test_targets_feed_losses_and_metrics():
    from pose2mesh_release_b200 import graph as pg
    from pose2mesh_release_b200 import loss as L
    from pose2mesh_release_b200 import metrics

    layer = smpl_layer()
    pose, betas, trans = random_inputs("smpl", 64, seed=14)
    gv_dev, _ = layer(cuda(pose), cuda(betas), cuda(trans))
    gv_ref = cuda(oracle("smpl", pose, betas, trans)[0])
    g = torch.Generator().manual_seed(15)
    pred = gv_ref + 0.02 * torch.randn(gv_ref.shape, generator=g).to(dev())
    face = pg.synthetic_sphere_faces(6890, 2)
    ln_d, le_d = L.MeshLosses(face)(pred, gv_dev)
    ln_r, le_r = L.MeshLosses(face)(pred, gv_ref)
    assert abs(ln_d.item() - ln_r.item()) < 1e-5 and abs(le_d.item() - le_r.item()) < 1e-5
    Jm = torch.as_tensor(MODELS["smpl"]["J_regressor"])
    a = metrics.evaluate_meshes(pred * 1000, gv_dev * 1000, Jm, 0, Jm, 0)
    b = metrics.evaluate_meshes(pred * 1000, gv_ref * 1000, Jm, 0, Jm, 0)
    scale = float(gv_ref.abs().max()) * 1000
    for k in a:
        assert float((a[k] - b[k]).abs().max()) / scale <= 1e-5, k
