"""The float64 gradient restatement (tests/body_model_grad_ref.py) against the unmodified reference layers' autograd
(tests/golden/body_model_grad.npz, made by tests/golden/make_golden_body_model_grad.py), the models' digests, mutated
gradients that the GPU bound must reject, and the default layers' refusal of inputs that require grad."""
import numpy as np
import pytest
import torch

import body_model_grad_ref as gr
import body_models as bm
from golden.make_golden_body_model_grad import MODES, cotangents
from helpers import load_npz
from pose2mesh_release_b200.body_model import ManoLayer, SMPLLayer

Z = load_npz("body_model_grad.npz")
CASES = [str(s) for s in Z["cases"]]
MODELS = {"smpl": bm.smpl_model()}
for _side in ("right", "left"):
    for _flat in (False, True):
        MODELS[f"mano_{_side}" + ("_flat" if _flat else "")] = bm.mano_model(_side, _flat)

# The GPU's bound, per sample and per gradient tensor, in units of that tensor's largest |entry| in the sample.
# fp32 (unit roundoff u = 6e-8) with fixed-order sums of many terms: the pose and betas gradients collect
# dcoef = dx basis^T over 3 V = 20670 columns and dA_j over up to 6890 vertices.  Rounding errors of independent terms
# grow like a random walk, u sqrt(n) per unit of result: 6e-8 * sqrt(20670) ~ 8.6e-6, so the bound is 1e-5.  (The
# forward's bound is 4e-6; on an H100 the worst case measured here is 1.5e-6.)
GRAD_BOUND = 1e-5


def case(name):
    g = lambda k: Z[f"{name}__{k}"] if f"{name}__{k}" in Z.files else None  # noqa: E731
    center = int(Z[f"{name}__center"])
    mk = str(Z[f"{name}__model"])
    out = dict(model=mk, kind="smpl" if mk == "smpl" else "mano", pose=g("pose"), betas=g("betas"), trans=g("trans"),
               center=None if center < 0 else center, seed=int(Z[f"{name}__seed"]), grads={})
    for mode in MODES:
        out["grads"][mode] = tuple(g(f"{mode}__{k}") for k in ("pose", "betas", "trans"))
    return out


def case_cotangents(c, mode):
    B = c["pose"].shape[0]
    return cotangents(c["seed"], B, 6890 if c["kind"] == "smpl" else 778, 24 if c["kind"] == "smpl" else 21, mode)


def grad_ratio(got, ref):
    """Worst error per sample and per gradient tensor, in units of that tensor's largest |entry| in the sample.  A
    tensor that is None must be None; an all-zero reference must be matched exactly."""
    worst = 0.0
    for g, r in zip(got, ref):
        assert (g is None) == (r is None)
        if r is None:
            continue
        g, r = np.asarray(g, np.float64).reshape(len(r), -1), np.asarray(r, np.float64).reshape(len(r), -1)
        scale = np.abs(r).max(axis=1)
        err = np.abs(g - r).max(axis=1)
        zero = scale == 0
        assert np.all(err[zero] == 0), "non-zero gradient where the reference has none"
        if (~zero).any():
            worst = max(worst, float(np.max(err[~zero] / scale[~zero])))
    return worst


def restated(c, mode, **mut):
    gv, gj = case_cotangents(c, mode)
    return gr.vjp(c["kind"], MODELS[c["model"]], c["pose"], c["betas"], c["trans"], c["center"], gv, gj, **mut)[2:]


@pytest.mark.parametrize("name", sorted(MODELS))
def test_model_digest(name):
    assert bm.digest(MODELS[name]) == str(Z[f"digest_{name}"])


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", CASES)
def test_restatement_matches_reference(name, mode):
    c = case(name)
    assert grad_ratio(restated(c, mode), c["grads"][mode]) <= 1e-11


def _worst(names, mode="both", **mut):
    return max(grad_ratio(restated(case(n), mode, **mut), case(n)["grads"][mode]) for n in names)


def test_bound_rejects_dropped_pose_blend():
    assert _worst(["smpl_random", "mano_right_random"], pose_blend=False) > 10 * GRAD_BOUND


def test_bound_rejects_dropped_centre_gradient():
    assert _worst(["smpl_center_no_trans", "mano_center_zero_trans", "mano_center_tip"], centre_grad=False) > \
        10 * GRAD_BOUND


def test_bound_rejects_betas_gradient_under_zero_rule():
    with pytest.raises(AssertionError, match="non-zero gradient"):
        _worst(["smpl_zero_betas"], leak_betas=True)


def test_bound_rejects_dropped_joints_path():
    assert _worst(["smpl_random", "mano_left_random"], mode="joints", joints_path=False) > 10 * GRAD_BOUND


def test_bound_rejects_untransposed_dx():
    assert _worst(["smpl_random", "mano_right_random"], mode="verts", transpose_dx=False) > 10 * GRAD_BOUND


def test_quaternion_renormalisation_term_is_below_fp32():
    """quat2mat divides by |q|, and |q| = 1 up to the 1e-8 offset in the angle, so the renormalisation's Jacobian
    changes the gradient by far less than fp32 can resolve -- even at the fixture's angles near 0.  Dropping it cannot
    be told apart from keeping it, by this bound or any fp32 one; the kernel keeps it, as autograd does."""
    assert _worst(["smpl_angles", "smpl_zero_pose", "mano_angles"], renorm=False) < 1e-6


def _smpl(**kw):
    m = MODELS["smpl"]
    return SMPLLayer(m["v_template"], m["shapedirs"], m["posedirs"], m["J_regressor"], m["weights"], m["parents"],
                     m["betas"], **kw)


def test_default_layers_refuse_grad():
    with pytest.raises(RuntimeError, match="requires grad"):
        _smpl()(torch.zeros(1, 72, requires_grad=True))
    m = MODELS["mano_right"]
    mano = ManoLayer(m["v_template"], m["shapedirs"], m["posedirs"], m["J_regressor"], m["weights"], m["betas"],
                     m["hands_mean"])
    with pytest.raises(RuntimeError, match="requires grad"):
        mano(torch.zeros(1, 48), th_betas=torch.zeros(1, 10, requires_grad=True))
    assert not _smpl().differentiable and _smpl(differentiable=True).differentiable


def test_from_reference_keyword():
    ref = bm.smpl_reference_layer(torch.nn.Module, MODELS["smpl"])
    assert SMPLLayer.from_reference(ref, differentiable=True).differentiable
    assert not SMPLLayer.from_reference(ref).differentiable
    mref = bm.mano_reference_layer(torch.nn.Module, MODELS["mano_left"])
    assert ManoLayer.from_reference(mref, differentiable=True).differentiable
