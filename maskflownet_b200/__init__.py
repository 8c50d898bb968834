"""maskflownet_b200 -- Hopper-native (sm_90a) implementation of the MaskFlownet hot path:
the local correlation cost volume and the flow-guided deformable feature warp x occlusion mask that feeds it.

  maskflownet_b200.ops      tensor-level operators backed by libmaskflow_b200.so (C ABI: include/maskflow_b200.h)
  maskflownet_b200.mx       torch-backed shim of the MXNet `F` / gluon `nn` namespaces the reference's
                            network/MaskFlownet.py and network/layer.py are written against
  maskflownet_b200.network  host-side mirror of the reference's model graph that calls the fused operators
  maskflownet_b200.losses   MultiscaleEpe on the fused kernels (network/MaskFlownet.py:563-611)
  maskflownet_b200.augment  GeometryAugmentation / ColorAugmentation with the reference's constructor arguments (augmentation.py)
  maskflownet_b200.pipeline PipelineFlownet: train_batch / do_batch / validate / predict (network/pipeline.py:19-223)
  maskflownet_b200.video    VideoFlowPredictor: a video -> one colour-coded flow per frame pair, one CUDA graph per size
  maskflownet_b200.dist     batch sharding + the one gradient all-reduce;  .params  reader of the reference's checkpoints
"""
from . import _lib  # noqa: F401
from ._lib import MaskflowError  # noqa: F401

__version__ = "0.1.0"
