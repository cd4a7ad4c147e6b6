"""Loads the REAL reference backbone by file path from the reference checkout (PDC_REFERENCE_ROOT).

TEST INFRASTRUCTURE.  The tests must not need the reference checkout, so nothing they run
may call this; oracle/make_golden.py uses it to write tests/golden/.

Recipe (SURVEY.md appendix D): exec the vendored torchvision-fork resnet.py and
pytorch_segmentation_detection/models/resnet_dilated.py unmodified, with (1) a shim module bound
as ``torchvision.models`` while resnet_dilated.py loads, because the fork package as a whole does
not import under Pillow>=7, and (2) ``model_zoo.load_url`` patched to return a freshly initialised
state dict, because the ImageNet checkpoint rd.py:292-295 insists on is not available offline.
"""
import importlib.util
import os
import sys
import types

from oracle.build_ref import REF_ROOT
_PSD = os.path.join(REF_ROOT, "external", "pytorch-segmentation-detection") if REF_ROOT else None
TV_RESNET = os.path.join(_PSD, "vision", "torchvision", "models", "resnet.py") if _PSD else None
RESNET_DILATED = os.path.join(_PSD, "pytorch_segmentation_detection", "models", "resnet_dilated.py") if _PSD else None


def reference_available():
    return _PSD is not None and os.path.isfile(TV_RESNET) and os.path.isfile(RESNET_DILATED)


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


_cache = {}


def load_reference_modules():
    if "rd" in _cache:
        return _cache["tv"], _cache["rd"]
    import torchvision
    tv = _load("ref_tv_resnet", TV_RESNET)
    tv.model_zoo.load_url = lambda url, *a, **k: tv.ResNet(tv.BasicBlock, [3, 4, 6, 3]).state_dict() \
        if "resnet34" in url else tv.ResNet(tv.BasicBlock, [2, 2, 2, 2]).state_dict()
    shim = types.ModuleType("torchvision.models")
    for n in ("resnet18", "resnet34", "resnet50", "resnet101", "resnet152"):
        setattr(shim, n, getattr(tv, n))
    real = sys.modules.get("torchvision.models")
    real_attr = getattr(torchvision, "models", None)
    sys.modules["torchvision.models"] = shim
    torchvision.models = shim
    try:
        rd = _load("ref_resnet_dilated", RESNET_DILATED)
    finally:
        if real is not None:
            sys.modules["torchvision.models"] = real
        if real_attr is not None:
            torchvision.models = real_attr
    _cache["tv"], _cache["rd"] = tv, rd
    return tv, rd


def reference_resnet34_8s(D, state_dict=None):
    """The reference's own Resnet34_8s(num_classes=D) (rd.py:283-322), optionally with weights loaded."""
    _, rd = load_reference_modules()
    net = rd.Resnet34_8s(num_classes=D)
    if state_dict is not None:
        net.load_state_dict(state_dict, strict=True)
    return net
