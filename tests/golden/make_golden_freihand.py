#!/usr/bin/env python
"""Golden 21-row MANO evaluation regressor, produced by the UNMODIFIED reference: lib/_mano.py's MANO.__init__ runs as
written on the seeded synthetic right-hand MANO model of tests/body_models.py.  Only two things are replaced: MANO.get_layer
(the real one loads the licence-gated pkl) returns tests/body_models.py:mano_reference_layer, the bypass
make_golden_body_model.py uses, and `core.config` is a stub module (the real one needs easydict; get_layer, the only
reader of cfg, is replaced).

    P2M_REFERENCE_ROOT=/path/to/Pose2Mesh_RELEASE python tests/golden/make_golden_freihand.py -> freihand_regressor.npz

Keys: joint_regressor [21, 778] float32 (MANO.joint_regressor), J_regressor [16, 778] float32 (the layer's
th_J_regressor it was built from), model_digest (body_models.digest of the model).
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import body_models as bm  # noqa: E402

REF = os.environ.get("P2M_REFERENCE_ROOT", "")


def main():
    if not os.path.isfile(os.path.join(REF, "lib", "_mano.py")):
        raise SystemExit("set P2M_REFERENCE_ROOT to a Pose2Mesh_RELEASE checkout")
    sys.path[:0] = [os.path.join(REF, "lib"), os.path.join(REF, "manopth")]
    core = types.ModuleType("core")
    core.__path__ = []
    config = types.ModuleType("core.config")
    config.cfg = types.SimpleNamespace(mano_dir="")
    core.config = config
    sys.modules.setdefault("core", core)
    sys.modules.setdefault("core.config", config)
    import _mano  # noqa: E402  (reference module)
    from manopth.manolayer import ManoLayer

    model = bm.mano_model("right")
    _mano.MANO.get_layer = lambda self: bm.mano_reference_layer(ManoLayer, model)
    mano = _mano.MANO()
    Z = {"joint_regressor": np.ascontiguousarray(mano.joint_regressor, dtype=np.float32),
         "J_regressor": np.ascontiguousarray(mano.layer.th_J_regressor.numpy(), dtype=np.float32),
         "model_digest": np.array(bm.digest(model))}
    assert Z["joint_regressor"].shape == (21, 778) and mano.joint_regressor.dtype == np.float32
    path = os.path.join(HERE, "freihand_regressor.npz")
    np.savez_compressed(path, **Z)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
