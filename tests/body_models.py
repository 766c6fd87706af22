"""Seeded synthetic body models of SMPL's and MANO's real sizes.

The real SMPL / MANO models are licence-gated, so the tests use stand-ins with the same buffer layouts, sizes and
value scales.  A model is regenerated from its seed (np.random.RandomState, whose stream is stable across numpy
versions), never stored; `digest` pins the generator, and the golden fixture records each model's digest.

    smpl_model()              V=6890, J=24, S=10, P=207, SMPL's kinematic tree, metres
    mano_model(side, flat)    V=778,  J=16, S=10, P=135, with hands_mean (zero when flat_hand_mean)
"""
from __future__ import annotations

import hashlib

import numpy as np

SMPL_PARENTS = (-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 20, 21)
# the chain ManoLayer.forward hard-codes (lev1/2/3_idxs, manolayer.py), not the pkl's kintree_table
MANO_PARENTS = (-1, 0, 1, 2, 0, 4, 5, 0, 7, 8, 0, 10, 11, 0, 13, 14)
MANO_TIPS = {"right": (745, 317, 444, 556, 673), "left": (745, 317, 445, 556, 673)}
MANO_REORDER = (0, 13, 14, 15, 16, 1, 2, 3, 17, 4, 5, 6, 18, 10, 11, 12, 19, 7, 8, 9, 20)

BUFFERS = ("v_template", "shapedirs", "posedirs", "J_regressor", "weights", "betas")


def _model(rng: np.random.RandomState, V: int, J: int, S: int, size: float, n_reg: int = 20) -> dict:
    P = 9 * (J - 1)
    half = np.array([0.35, 0.85, 0.15]) * size
    v_template = rng.uniform(-1.0, 1.0, (V, 3)) * half
    shapedirs = rng.normal(0.0, 1e-2 * size, (V, 3, S))
    posedirs = rng.normal(0.0, 1e-3 * size, (V, 3, P))
    J_regressor = np.zeros((J, V))
    for j in range(J):
        idx = rng.choice(V, n_reg, replace=False)
        J_regressor[j, idx] = rng.uniform(0.1, 1.0, n_reg)
    J_regressor /= J_regressor.sum(1, keepdims=True)
    weights = np.zeros((V, J))
    for v in range(V):
        n = rng.randint(1, 5)
        idx = rng.choice(J, n, replace=False)
        weights[v, idx] = rng.uniform(0.05, 1.0, n)
    weights /= weights.sum(1, keepdims=True)
    betas = rng.normal(0.0, 0.8, S)  # non-zero, so the model-beta fallback is visible
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)  # noqa: E731
    return {"v_template": f32(v_template), "shapedirs": f32(shapedirs), "posedirs": f32(posedirs),
            "J_regressor": f32(J_regressor), "weights": f32(weights), "betas": f32(betas)}


def smpl_model(seed: int = 0) -> dict:
    m = _model(np.random.RandomState(seed), 6890, 24, 10, 1.0)
    m["parents"] = np.array(SMPL_PARENTS, dtype=np.int32)
    return m


def mano_model(side: str = "right", flat_hand_mean: bool = False, seed: int = 1) -> dict:
    """Both sides share one seeded model (only the tip vertices differ, as in ManoLayer)."""
    rng = np.random.RandomState(seed)
    m = _model(rng, 778, 16, 10, 0.12)
    hands_mean = rng.normal(0.0, 0.3, 45).astype(np.float32)
    m["hands_mean"] = np.zeros(45, np.float32) if flat_hand_mean else hands_mean
    m["parents"] = np.array(MANO_PARENTS, dtype=np.int32)
    m["side"] = side
    return m


def digest(model: dict) -> str:
    h = hashlib.sha256()
    for k in BUFFERS + ("hands_mean", "parents"):
        if k in model:
            a = np.ascontiguousarray(model[k])
            h.update(k.encode())
            h.update(str(a.dtype).encode() + str(a.shape).encode())
            h.update(a.tobytes())
    return h.hexdigest()


def _layer(cls, model, attrs):
    """An instance of `cls` (the reference's SMPL_Layer / ManoLayer, or any Module subclass) carrying the model's
    buffers under the reference's names, built with __new__ + Module.__init__ so that only the chumpy pkl loader is
    bypassed."""
    import torch
    from torch.nn import Module

    layer = cls.__new__(cls)
    Module.__init__(layer)
    for k, v in attrs.items():
        setattr(layer, k, v)
    t = lambda a: torch.tensor(np.asarray(a, np.float32))  # noqa: E731
    layer.register_buffer("th_betas", t(model["betas"])[None])
    layer.register_buffer("th_shapedirs", t(model["shapedirs"]))
    layer.register_buffer("th_posedirs", t(model["posedirs"]))
    layer.register_buffer("th_v_template", t(model["v_template"])[None])
    layer.register_buffer("th_J_regressor", t(model["J_regressor"]))
    layer.register_buffer("th_weights", t(model["weights"]))
    layer.register_buffer("th_faces", torch.zeros((1, 3), dtype=torch.long))
    return layer


SMPL_PKL_ROOT_PARENT = 2 ** 32 - 1  # what kintree_table[0][0] holds in the SMPL pkl (an unsigned -1)


def smpl_reference_layer(cls, model, center_idx=None, gender="neutral", root_parent=SMPL_PKL_ROOT_PARENT):
    """SMPL_Layer takes kintree_parents from the pkl's kintree_table[0], whose root entry is 2^32 - 1; forward never
    reads it.  The stand-in carries the same value unless root_parent says otherwise."""
    parents = [int(root_parent)] + [int(p) for p in model["parents"][1:]]
    return _layer(cls, model, {"center_idx": center_idx, "gender": gender, "kintree_parents": parents,
                               "num_joints": len(model["parents"])})


def mano_reference_layer(cls, model, center_idx=None, flat_hand_mean=False):
    import torch

    layer = _layer(cls, model, {"center_idx": center_idx, "robust_rot": False, "rot": 3, "flat_hand_mean": flat_hand_mean,
                                "side": model["side"], "use_pca": False, "joint_rot_mode": "axisang",
                                "root_rot_mode": "axisang", "ncomps": 45,
                                "kintree_parents": [int(p) for p in model["parents"]]})
    layer.register_buffer("th_hands_mean", torch.tensor(np.asarray(model["hands_mean"], np.float32))[None])
    layer.register_buffer("th_selected_comps", torch.eye(45))
    return layer


def random_axisang(rng: np.random.RandomState, n: int, lo: float, hi: float) -> np.ndarray:
    """n axis-angle vectors with random axes and angles log-uniform in [lo, hi]."""
    axis = rng.normal(size=(n, 3))
    axis /= np.linalg.norm(axis, axis=1, keepdims=True)
    ang = np.exp(rng.uniform(np.log(lo), np.log(hi), (n, 1)))
    return axis * ang
