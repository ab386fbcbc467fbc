"""lt_b200 -- H100-native (sm_90a) implementation of the volumetric-triangulation hot path of
karfly/learnable-triangulation-pytorch, behind the reference's own nn.Module / op interface.

Import as `lt_b200` (the directory name `learnable-triangulation-pytorch_b200` is not a valid
Python identifier; `lt_b200.py` at the repo root is the import shim).

    from lt_b200 import VolumetricTriangulationNet          # drop-in for mvn.models.triangulation
    from lt_b200 import op                                   # drop-in for mvn.utils.op (two ops)
    lt_b200.install()                                        # or: patch an imported reference `mvn` in place
"""
from . import loss, multiview, op, pipeline, pose_resnet, v2v, volumetric  # noqa: F401
from .multiview import Camera  # noqa: F401
from .train_graph import TrainStep  # noqa: F401
from .triangulation import (AlgebraicTriangulationNet, RANSACTriangulationNet, TwoStageTriangulationNet,  # noqa: F401
                            VolumetricTriangulationNet)
from .v2v import V2VModel  # noqa: F401

__version__ = "0.1.0"


def install(mvn_package=None):
    """Swap the reference's models, their custom ops, the keypoint criteria and the volumetric cross-entropy loss for the native
    ones.

    `mvn_package` is the already-imported reference package (`import mvn`); if None it is imported.
    After this, the reference `train.py` (which does `from mvn.models.triangulation import
    VolumetricTriangulationNet` and `from mvn.models.loss import KeypointsMSELoss, ..., VolumetricCELoss` at import time) picks up the
    native implementation unchanged.
    """
    import importlib
    if mvn_package is None:
        mvn_package = importlib.import_module("mvn")
    tri = importlib.import_module(mvn_package.__name__ + ".models.triangulation")
    ref_op = importlib.import_module(mvn_package.__name__ + ".utils.op")
    ref_loss = importlib.import_module(mvn_package.__name__ + ".models.loss")
    for name in ("KeypointsMSELoss", "KeypointsMSESmoothLoss", "KeypointsMAELoss", "KeypointsL2Loss", "VolumetricCELoss"):
        setattr(ref_loss, name, getattr(loss, name))
    tri.VolumetricTriangulationNet = VolumetricTriangulationNet
    tri.AlgebraicTriangulationNet = AlgebraicTriangulationNet
    tri.RANSACTriangulationNet = RANSACTriangulationNet
    ref_op.integrate_tensor_2d = op.integrate_tensor_2d
    ref_op.unproject_heatmaps = op.unproject_heatmaps
    ref_op.integrate_tensor_3d_with_coordinates = op.integrate_tensor_3d_with_coordinates
    return mvn_package
