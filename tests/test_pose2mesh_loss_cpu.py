"""The Trainer's objective (lib/core/base.py:129-143) on CPU: the float64 oracle (tests/pose2mesh_loss_oracle.py)
against the unmodified reference's values and gradients (tests/golden/pose2mesh_loss.npz), and install()'s opt-in
rebinding of the reference's loss module (core.loss)."""
import os
import sys
import types

import numpy as np
import pytest
import torch

from helpers import load_npz

CASES = ("smpl", "mano")
INPUTS = ("cam_mesh", "lift_pose", "gt_mesh", "gt_reg3dpose", "gt_lift3dpose", "mesh_valid", "reg3dpose_valid",
          "lift3dpose_valid")


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("edge", (False, True))
def test_oracle_matches_reference_golden(case, edge):
    import pose2mesh_loss_oracle as lo

    z = load_npz("pose2mesh_loss.npz")
    x = {k: torch.from_numpy(z[f"{case}/{k}"]).double() for k in INPUTS}
    x["cam_mesh"].requires_grad_(True)
    x["lift_pose"].requires_grad_(True)
    face, perm = z[f"{case}/face"], z[f"{case}/perm_reverse"]
    loss, terms = lo.pose2mesh_loss(*(x[k] for k in INPUTS), face, torch.from_numpy(z[f"{case}/joint_regressor"]).double(),
                                    perm, weights=tuple(z["weights"]), edge=edge)
    loss.backward()
    tag = f"{case}/edge{int(edge)}"
    np.testing.assert_allclose(terms.detach().numpy(), z[f"{tag}/terms"], rtol=1e-12, atol=0)
    assert abs(float(loss.detach()) - float(z[f"{tag}/loss"])) <= 1e-12 * abs(float(z[f"{tag}/loss"]))
    if not edge:
        assert float(terms[2].detach()) == 0.0
    nv = int(face.max()) + 1
    g = x["cam_mesh"].grad.numpy()
    pad = np.ones(g.shape[1], bool)
    pad[perm[:nv]] = False
    assert not g[:, pad].any()
    for got, ref in ((g[:, perm[:nv]], z[f"{tag}/grad_mesh"]), (x["lift_pose"].grad.numpy(), z[f"{tag}/grad_lift"])):
        # the golden gradients are float64 values rounded to float32
        np.testing.assert_allclose(got, ref, rtol=2 ** -23, atol=1e-30)


def test_golden_covers_zero_masks_and_regressor_gaps():
    z = load_npz("pose2mesh_loss.npz")
    for case in CASES:
        jr = z[f"{case}/joint_regressor"]
        assert (jr == 0).all(1).any() and (jr == 0).all(0).any()
        assert (z[f"{case}/mesh_valid"] == 0).any()
    for k in ("mesh_valid", "reg3dpose_valid", "lift3dpose_valid"):
        m = z[f"mano/{k}"]
        assert (m.reshape(len(m), -1) == 0).all(1).any()


# ---- install(replace_losses=True)


def _stand_in_core_loss():
    core = types.ModuleType("core")
    core.__path__ = []
    loss = types.ModuleType("core.loss")
    for name in ("CoordLoss", "NormalVectorLoss", "EdgeLengthLoss", "LaplacianLoss"):
        setattr(loss, name, type(name, (torch.nn.Module,), {}))
    loss.get_loss = lambda faces: (loss.CoordLoss(),)
    base = types.ModuleType("core.base")
    base.get_loss = loss.get_loss                          # `from core.loss import get_loss` (base.py:14)
    core.loss, core.base = loss, base
    return {"core": core, "core.loss": loss, "core.base": base}


@pytest.fixture()
def reference(request):
    from test_install_cpu import STAND_INS, _stand_in_reference

    names = STAND_INS + ("core", "core.loss", "core.base")
    saved = {name: sys.modules.get(name) for name in names}
    mods = {**_stand_in_reference(), **_stand_in_core_loss()}
    if request.param == "reference":                      # the unmodified lib/core/loss.py in place of the stand-in
        from oracle import ref_shim

        if not ref_shim.available():
            pytest.skip("P2M_REFERENCE_ROOT not set")
        import importlib.util

        path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_golden_loss.py")
        spec = importlib.util.spec_from_file_location("make_golden_loss", path)
        maker = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(maker)
        mods["core.loss"] = maker.load_ref_loss()
        mods["core.base"].get_loss = mods["core.loss"].get_loss
    sys.modules.update(mods)
    import pose2mesh_release_b200.install as inst

    try:
        yield mods["core.loss"], mods["core.base"], inst
    finally:
        inst.uninstall()
        for name, mod in saved.items():
            if mod is None:
                sys.modules.pop(name, None)
            else:
                sys.modules[name] = mod


@pytest.mark.parametrize("reference", ("stand_in", "reference"), indirect=True)
def test_install_replace_losses_rebinds_and_uninstall_restores(reference):
    ref_loss, base, inst = reference
    from pose2mesh_release_b200 import loss as my_loss

    names = ("CoordLoss", "NormalVectorLoss", "EdgeLengthLoss", "get_loss")
    orig = {n: getattr(ref_loss, n) for n in names}
    laplacian = ref_loss.LaplacianLoss
    inst.install()                                          # the default leaves the losses alone
    assert {n: getattr(ref_loss, n) for n in names} == orig and base.get_loss is orig["get_loss"]
    inst.uninstall()
    inst.install(replace_losses=True)
    for n in names:
        assert getattr(ref_loss, n) is getattr(my_loss, n)
    assert base.get_loss is my_loss.get_loss and ref_loss.LaplacianLoss is laplacian
    inst.install(replace_losses=True)                       # idempotent
    inst.uninstall()
    assert {n: getattr(ref_loss, n) for n in names} == orig and base.get_loss is orig["get_loss"]
