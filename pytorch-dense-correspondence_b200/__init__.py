"""pytorch-dense-correspondence_b200 -- the H100-native (sm_90a) implementation of the dense-descriptor training
hot path of RobotLocomotion/pytorch-dense-correspondence: Resnet34_8s forward/backward and the pixelwise
contrastive loss, behind the reference's own Python API.  Import as ``pdc_b200`` (see pdc_b200.py at the repo
root; the directory name itself is not a valid Python identifier).

Everything numerical happens in ``libddn_b200.so`` (C ABI in include/ddn_b200.h); importing this package
raises if that library is missing -- there is no CPU / PyTorch fallback.
"""
from . import _native
from .resnet_dilated import Resnet34_8s, Resnet50_8s, set_default_precision
from .dense_correspondence_network import DenseCorrespondenceNetwork
from .pixelwise_contrastive_loss import PixelwiseContrastiveLoss, DEFAULT_LOSS_CONFIG
from . import loss_composer
from .loss_composer import SpartanDatasetDataType
from .fused_adam import FusedAdam, adjust_learning_rate
from . import ops, synthetic, data_parallel, sampling, evaluation
from .evaluation import (DenseCorrespondenceEvaluation, match_statistics, quantitative_analysis_on_pair, descriptor_statistics,
                         descriptor_statistics_over_images, save_descriptor_statistics, across_object_analysis)

__all__ = ["Resnet34_8s", "Resnet50_8s", "DenseCorrespondenceNetwork", "PixelwiseContrastiveLoss", "loss_composer",
           "SpartanDatasetDataType", "DEFAULT_LOSS_CONFIG", "set_default_precision", "FusedAdam", "adjust_learning_rate", "ops", "synthetic", "data_parallel", "sampling",
           "evaluation", "DenseCorrespondenceEvaluation", "match_statistics", "quantitative_analysis_on_pair",
           "descriptor_statistics", "descriptor_statistics_over_images", "save_descriptor_statistics", "across_object_analysis"]
