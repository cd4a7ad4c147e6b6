"""Shim for dense_correspondence/loss_functions/pixelwise_contrastive_loss.py -> this project's implementation."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import _load  # noqa: F401
from pdc_b200.pixelwise_contrastive_loss import PixelwiseContrastiveLoss  # noqa: F401
