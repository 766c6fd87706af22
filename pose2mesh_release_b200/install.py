"""Drop the native MeshNet into a running copy of the reference (SURVEY.md §8b).

    import __init_path                      # the reference's sys.path hack (main/__init_path.py)
    import pose2mesh_release_b200.install as p2m; p2m.install()
    import core.base                        # Trainer / Tester now build the native MeshNet

``install()`` rebinds ``models.meshnet.Pose2Mesh`` / ``get_model``,
``models.backbones.cheby_graph_conv.graph_conv_cheby`` and ``models.posenet.LinearModel`` / ``get_model`` (the
PoseNet in front of MeshNet: the reference's own ``FlatPose2Mesh`` then runs both halves natively in eval mode) and
swaps ``graph_utils.build_coarse_graphs`` for the native-matching builder; ``install(replace_losses=True)`` also rebinds
``core.loss.CoordLoss`` / ``NormalVectorLoss`` / ``EdgeLengthLoss`` / ``get_loss`` (and ``core.base``'s imported
``get_loss``) to the native losses, so the Trainer no longer copies the face table from host memory twice per step;
``install(replace_optimizer=True)`` rebinds ``funcs_utils.get_optimizer`` (and ``core.base``'s imported one) to one
that builds the native ``optim.RMSprop`` for ``cfg.TRAIN.optimizer == 'rmsprop'``.  ``uninstall()`` restores the
originals.  Nothing in the reference tree is modified on disk.
"""
from __future__ import annotations

import importlib
import sys

_saved = {}
_rebound = []  # (module, attribute, original) for `from graph_utils import build_coarse_graphs`-style holders


def _rebind_holders(original, replacement):
    """Modules imported BEFORE install() that did ``from graph_utils import build_coarse_graphs`` (the
    reference's datasets and demo/run.py do) hold their own reference to the original function: patch
    those bindings too, so that the overlay is never half applied."""
    for name, mod in list(sys.modules.items()):
        if mod is None or name.startswith("pose2mesh_release_b200"):
            continue
        try:
            items = list(vars(mod).items())
        except TypeError:
            continue
        for attr, val in items:
            if val is original:
                setattr(mod, attr, replacement)
                _rebound.append((mod, attr, original))


_LOSS_NAMES = ("CoordLoss", "NormalVectorLoss", "EdgeLengthLoss", "get_loss")


def _native_get_optimizer(original):
    """funcs_utils.get_optimizer (lib/funcs_utils.py:78-99) with the native RMSprop, built with the same arguments,
    for cfg.TRAIN.optimizer == 'rmsprop'; for every other optimizer, what `original` returns.  cfg is the one
    `original` reads (funcs_utils' ``from core.config import cfg``)."""
    def get_optimizer(model):
        cfg = original.__globals__["cfg"]
        if cfg.TRAIN.optimizer == "rmsprop":
            from .optim import RMSprop

            return RMSprop(model.parameters(), lr=cfg.TRAIN.lr)
        return original(model=model)

    return get_optimizer


def install(replace_graph_builder: bool = True, replace_losses: bool = False, replace_optimizer: bool = False):
    from . import cheby_graph_conv as my_conv
    from . import graph as my_graph
    from . import meshnet as my_meshnet
    from . import posenet as my_posenet

    ref_posenet = importlib.import_module("models.posenet")
    _saved.setdefault("posenet", (ref_posenet.LinearModel, ref_posenet.get_model))
    ref_posenet.LinearModel = my_posenet.LinearModel
    ref_posenet.get_model = my_posenet.get_model
    ref_meshnet = importlib.import_module("models.meshnet")
    ref_conv = importlib.import_module("models.backbones.cheby_graph_conv")
    _saved.setdefault("meshnet", (ref_meshnet.Pose2Mesh, ref_meshnet.get_model, ref_meshnet.graph_conv_cheby))
    _saved.setdefault("conv", ref_conv.graph_conv_cheby)
    ref_meshnet.Pose2Mesh = my_meshnet.Pose2Mesh
    ref_meshnet.get_model = my_meshnet.get_model
    ref_meshnet.graph_conv_cheby = my_conv.graph_conv_cheby
    ref_conv.graph_conv_cheby = my_conv.graph_conv_cheby
    if replace_graph_builder:
        ref_gu = importlib.import_module("graph_utils")
        _saved.setdefault("graph", ref_gu.build_coarse_graphs)
        _rebind_holders(_saved["graph"], my_graph.build_coarse_graphs)   # includes graph_utils itself
        ref_gu.build_coarse_graphs = my_graph.build_coarse_graphs
    _rebind_holders(_saved["conv"], my_conv.graph_conv_cheby)
    if replace_losses:
        from . import loss as my_loss

        ref_loss = importlib.import_module("core.loss")
        _saved.setdefault("loss", {name: getattr(ref_loss, name) for name in _LOSS_NAMES})
        for name, original in _saved["loss"].items():
            _rebind_holders(original, getattr(my_loss, name))               # includes core.loss itself
    if replace_optimizer and "optimizer" not in _saved:
        ref_fu = importlib.import_module("funcs_utils")
        _saved["optimizer"] = ref_fu.get_optimizer
        _rebind_holders(_saved["optimizer"], _native_get_optimizer(_saved["optimizer"]))  # funcs_utils, core.base


def uninstall():
    while _rebound:
        mod, attr, original = _rebound.pop()
        setattr(mod, attr, original)
    if "meshnet" in _saved:
        ref_meshnet = importlib.import_module("models.meshnet")
        ref_meshnet.Pose2Mesh, ref_meshnet.get_model, ref_meshnet.graph_conv_cheby = _saved.pop("meshnet")
    if "posenet" in _saved:
        ref_posenet = importlib.import_module("models.posenet")
        ref_posenet.LinearModel, ref_posenet.get_model = _saved.pop("posenet")
    if "conv" in _saved:
        importlib.import_module("models.backbones.cheby_graph_conv").graph_conv_cheby = _saved.pop("conv")
    if "graph" in _saved:
        importlib.import_module("graph_utils").build_coarse_graphs = _saved.pop("graph")
    if "optimizer" in _saved:
        importlib.import_module("funcs_utils").get_optimizer = _saved.pop("optimizer")
    if "loss" in _saved:
        ref_loss = importlib.import_module("core.loss")
        for name, original in _saved.pop("loss").items():
            setattr(ref_loss, name, original)
