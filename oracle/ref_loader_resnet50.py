"""Loads the REAL reference Resnet50_8s (rd.py:399-435 over the fork's Bottleneck, resnet.py:72-109) from the reference
checkout (PDC_REFERENCE_ROOT), through oracle/ref_loader.py's recipe.

TEST INFRASTRUCTURE: only oracle/make_golden_resnet50.py calls this.  rd.Resnet50_8s insists on the ImageNet checkpoint
(``pretrained=True``), which is not available offline; while the module is built, ``model_zoo.load_url`` of the fork's
resnet.py returns a seeded ``ResNet(Bottleneck, [3, 4, 6, 3]).state_dict()`` instead, and the oracle's weights are loaded
on top of it.
"""
import torch

from oracle.ref_loader import load_reference_modules, reference_available  # noqa: F401


def reference_resnet50_8s(D, state_dict=None, seed=0):
    """The reference's own Resnet50_8s(num_classes=D), optionally with weights loaded."""
    tv, rd = load_reference_modules()
    saved = tv.model_zoo.load_url

    def stand_in(url, *a, **k):
        assert "resnet50" in url, url
        g = torch.random.get_rng_state()
        torch.manual_seed(seed)
        sd = tv.ResNet(tv.Bottleneck, [3, 4, 6, 3]).state_dict()
        torch.random.set_rng_state(g)
        return sd
    tv.model_zoo.load_url = stand_in
    try:
        net = rd.Resnet50_8s(num_classes=D)
    finally:
        tv.model_zoo.load_url = saved
    if state_dict is not None:
        net.load_state_dict(state_dict, strict=True)
    return net
