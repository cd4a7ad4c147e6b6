"""Shim for pytorch_segmentation_detection/models/resnet_dilated.py -> this project's implementation (Resnet34_8s and Resnet50_8s)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import _load  # noqa: F401
from pdc_b200.resnet_dilated import Resnet34_8s, Resnet50_8s  # noqa: F401
