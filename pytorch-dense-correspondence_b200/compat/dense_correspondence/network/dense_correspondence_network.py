"""Shim for dense_correspondence/network/dense_correspondence_network.py -> this project's implementation."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import _load  # noqa: F401
from pdc_b200.dense_correspondence_network import DenseCorrespondenceNetwork  # noqa: F401
