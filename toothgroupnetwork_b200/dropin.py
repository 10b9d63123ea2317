"""Make the reference's import paths resolve to this package.

    import toothgroupnetwork_b200.dropin as dropin
    dropin.install()
    from models.modules import pointnet_pp        # reference code, unmodified

After ``install()`` the modules the reference's callers import
(``blocks.py:6``, ``heads.py:6``, ``basic_operators.py:4``, ``gen_utils.py:8``, ``pointnet_pp.py:3``,
``tsg_centroid_module.py:3``, ``tsg_seg_module.py:3``, ``tsegnet.py:8``, ``tgn_loss.py:4``,
``tsg_loss.py:2`` ...) are served from here:

    external_libs.pointops.functions.pointops      -> toothgroupnetwork_b200.pointops
    external_libs.pointnet2_utils.pointnet2_utils  -> toothgroupnetwork_b200.pointnet2_utils
    pointops_cuda                                  -> toothgroupnetwork_b200.pointops_cuda

Existing ``external_libs`` packages on ``sys.path`` (the reference checkout) keep serving every
other submodule (``external_libs.scheduler`` ...): only the three names above are overridden.
"""
from __future__ import annotations

import importlib
import sys
import types

_TARGETS = {
    "external_libs.pointops.functions.pointops": "toothgroupnetwork_b200.pointops",
    "external_libs.pointnet2_utils.pointnet2_utils": "toothgroupnetwork_b200.pointnet2_utils",
    "pointops_cuda": "toothgroupnetwork_b200.pointops_cuda",
}


def _ensure_package(name: str) -> types.ModuleType:
    if name in sys.modules:
        return sys.modules[name]
    try:
        return importlib.import_module(name)
    except Exception:
        pkg = types.ModuleType(name)
        pkg.__path__ = []          # namespace-like package
        sys.modules[name] = pkg
        if "." in name:
            parent, _, child = name.rpartition(".")
            setattr(_ensure_package(parent), child, pkg)
        return pkg


def install() -> None:
    for alias, target in _TARGETS.items():
        mod = importlib.import_module(target)
        if "." in alias:
            parent, _, child = alias.rpartition(".")
            setattr(_ensure_package(parent), child, mod)
        sys.modules[alias] = mod


def accelerate_ops_utils(ops_utils_module=None) -> None:
    """Optional: also replace the host-side crop search of the reference's ``ops_utils`` (sklearn KDTree.query(k=3072),
    ops_utils.py:146-161, and the gather :198-218) with the GPU versions of ``toothgroupnetwork_b200.crops``.  Call after
    ``install()``; imports ``ops_utils`` from ``sys.path`` when no module is passed."""
    from . import clustering, crops
    if ops_utils_module is None:
        ops_utils_module = importlib.import_module("ops_utils")
    crops.accelerate(ops_utils_module)
    clustering.accelerate(ops_utils_module)        # DBSCAN + noise vote of get_clustering_labels (ops_utils.py:86-144)
    for name in ("models.modules.tsegnet", "inference_pipelines.inference_pipeline_tsegnet"):
        if name in sys.modules:                     # their own ``from sklearn.cluster import DBSCAN`` (tsegnet.py:7,59)
            clustering.accelerate_dbscan(sys.modules[name])


def accelerate_kmeans(module=None) -> None:
    """Optional: point the ``KMeans`` name of the reference's ``ops_utils`` (``clustering_points(method="kmeans")`` and
    ``find_k_kmeans``, ops_utils.py:32) at ``toothgroupnetwork_b200.clustering.KMeans``, which fits on the GPU with scikit-learn's
    labels.  Imports ``ops_utils`` from ``sys.path`` when no module is passed."""
    from . import clustering
    if module is None:
        module = importlib.import_module("ops_utils")
    clustering.accelerate_kmeans(module)


def accelerate_blocks(blocks_module=None) -> None:
    """Optional: run the no-grad forwards of the reference's ``PointTransformerLayer`` / ``TransitionDown``
    (models/modules/cbl_point_transformer/blocks.py:31-44, :59-79) on the fused kernels of
    ``toothgroupnetwork_b200.blocks_fused``; under autograd the reference's own code keeps running."""
    from . import blocks_fused
    if blocks_module is None:
        blocks_module = importlib.import_module("models.modules.cbl_point_transformer.blocks")
    blocks_fused.accelerate(blocks_module)


def accelerate_decoder(blocks_module=None, heads_module=None) -> None:
    """Optional: run the no-grad forwards of the reference's ``TransitionUp`` (both forms) and ``MultiHead``
    (models/modules/cbl_point_transformer/blocks.py:92-111, heads.py:53-61) on the layer chain and ``csrc/pt_head.cu`` through
    ``toothgroupnetwork_b200.blocks_fused``; under autograd, and for packed clouds of unequal sizes in the head form, the
    reference's own code keeps running.  Imports both modules from ``sys.path`` when none is passed."""
    from . import blocks_fused
    if blocks_module is None and heads_module is None:
        blocks_module = importlib.import_module("models.modules.cbl_point_transformer.blocks")
        heads_module = importlib.import_module("models.modules.cbl_point_transformer.heads")
    blocks_fused.accelerate_decoder(blocks_module, heads_module)


def accelerate_transformer_blocks(blocks_module=None) -> None:
    """Optional: run the no-grad forward of the reference's ``PointTransformerBlock`` (models/modules/cbl_point_transformer/
    blocks.py:114-135: linear1, its BatchNorms, the transformer layer, linear3 and the residual) on the layer chain,
    ``csrc/pt_layer.cu``, ``csrc/pt_head.cu`` and ``csrc/pt_block.cu`` through ``toothgroupnetwork_b200.blocks_fused``, at the
    widths where that is measured to be faster (``blocks_fused.BLOCK_FUSED_MAX_C``); under autograd, at wider blocks and for
    shapes the kernels do not take, the class's previous forward keeps running.  Imports the module from ``sys.path`` when none
    is passed."""
    from . import blocks_fused
    if blocks_module is None:
        blocks_module = importlib.import_module("models.modules.cbl_point_transformer.blocks")
    blocks_fused.accelerate_blocks(blocks_module)


def accelerate_inference_pipeline(module=None) -> None:
    """Optional: run the boundary detection and resampling between the two networks of a tgnet inference
    (``InferencePipeLine.get_boundary_sampled_feats``, inference_pipelines/inference_pipeline_tgn.py:289-330: float64 KDTree kNN,
    label vote, random boundary subset, FPS) on the GPU through ``toothgroupnetwork_b200.boundary``.  Imports
    ``inference_pipelines.inference_pipeline_tgn`` from ``sys.path`` when no module is passed."""
    from . import boundary
    if module is None:
        module = importlib.import_module("inference_pipelines.inference_pipeline_tgn")
    boundary.accelerate(module)


def accelerate_label_transfer(module=None, ties: str = "host") -> None:
    """Optional: answer the float64 ``KDTree.query`` calls of the inference pipelines' label transfers on the GPU through
    ``toothgroupnetwork_b200.neighbors.KDTree`` (the boundary clusters and the final transfer to the mesh,
    inference_pipeline_tgn.py:107-114, :137-140; the final transfers of inference_pipeline_tsegnet.py:72-74 and
    inference_pipeline_sem.py:37-39), with the same indices and distances.  Rows with exactly tied distances are answered by
    scikit-learn's query code on a device-built tree (ties="host"), or by the same depth-first walk on the device
    (ties="device": ``neighbors.DeviceKDTree``, only the rows the walk flags reach the host).  Swaps the ``KDTree`` name of
    ``inference_pipelines.inference_pipeline_tgn`` (imported from ``sys.path`` when no module is passed), and of the tsegnet and
    sem pipelines when they are already imported.  ``ops_utils`` keeps its own: ``accelerate_ops_utils`` replaces its queries."""
    from . import neighbors
    if module is None:
        module = importlib.import_module("inference_pipelines.inference_pipeline_tgn")
    neighbors.accelerate(module, ties)
    for name in ("inference_pipelines.inference_pipeline_tsegnet", "inference_pipelines.inference_pipeline_sem"):
        if name in sys.modules:
            neighbors.accelerate(sys.modules[name], ties)


def accelerate_dgcnn(module=None) -> None:
    """Optional: answer the feature-space kNN of the DGCNN model (``knn`` of models/modules/dgcnn.py:4-10, called three times per
    forward by ``get_graph_feature``) with the exact kernel of ``toothgroupnetwork_b200.dgcnn``: the same indices without the
    N x N matrix.  Inputs the kernel does not reproduce stay on the module's own ``knn``.  Imports ``models.modules.dgcnn`` from
    ``sys.path`` when no module is passed."""
    from . import dgcnn
    if module is None:
        module = importlib.import_module("models.modules.dgcnn")
    dgcnn.accelerate(module)


def accelerate_dgcnn_forward(module=None, running_stats: bool = False) -> None:
    """Optional: run the no-grad forward of the DGCNN model (``DGCnnModule.forward``, models/modules/dgcnn.py:96-134) on the
    tensor-core layer chain of ``toothgroupnetwork_b200.dgcnn``: the EdgeConv gathers, BatchNorm, LeakyReLU and the neighbour max
    without the (B, 2C, N, k) tensors.  Under autograd the reference's own forward runs.  By default only train-mode BatchNorm
    (batch statistics) takes the fused path; ``running_stats=True`` also sends eval-mode calls (``module.eval()``, as the
    validation and test phases run) to it, their running-statistics layers on promoted tensor-core accumulation; a later call
    with True turns that on for an already-wrapped class.  Imports ``models.modules.dgcnn`` from ``sys.path`` when no module is
    passed."""
    from . import dgcnn
    if module is None:
        module = importlib.import_module("models.modules.dgcnn")
    dgcnn.accelerate_forward(module, running_stats=running_stats)


def accelerate_pointnet_forward(module=None, running_stats: bool = False) -> None:
    """Optional: run the no-grad forward of the PointNet model (``get_model.forward``, models/modules/pointnet.py:23-35) on the
    tensor-core layer chain of ``toothgroupnetwork_b200.pointnet``: both learned transforms, BatchNorm and the max over the points
    without the (B, 2176, N) concatenation.  ``PointFirstModule`` calls ``get_model``, so the sem pipeline uses it too.  Under
    autograd the reference's own forward runs.  By default only train-mode BatchNorm (batch statistics) takes the fused path;
    ``running_stats=True`` also sends eval-mode calls (validation and test phases) to it, their running-statistics layers on
    promoted tensor-core accumulation; a later call with True turns that on for an already-wrapped class.  Imports
    ``models.modules.pointnet`` from ``sys.path`` when no module is passed."""
    from . import pointnet
    if module is None:
        module = importlib.import_module("models.modules.pointnet")
    pointnet.accelerate_forward(module, running_stats=running_stats)


def uninstall() -> None:
    for alias in _TARGETS:
        sys.modules.pop(alias, None)
