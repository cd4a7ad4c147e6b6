"""Shim for dense_correspondence/loss_functions/loss_composer.py -> this project's implementation."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import _load  # noqa: F401
from pdc_b200.loss_composer import *  # noqa: F401,F403
from pdc_b200.loss_composer import get_loss, get_within_scene_loss, get_different_object_loss, zero_loss, is_zero_loss  # noqa: F401
