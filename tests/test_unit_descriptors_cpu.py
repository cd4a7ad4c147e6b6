"""CPU: unit-length descriptors (the reference's ``normalize`` option per pixel) -- the float64 restatement against the
executed reference's fixture, every ABI refusal before a launch, the unit flag of the low-resolution tag, and the
ValueError of ``forward_pair(..., per_pixel_normalize=True)`` on a network built without ``normalize``."""
import ctypes
import os

import numpy as np
import pytest
import torch

import pdc_b200
from pdc_b200 import _native as N
from pdc_b200 import resnet_dilated
from oracle import loss_oracle as LO
from oracle import unit_descriptor_oracle as UO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IDX_KEYS = ("matches_a", "matches_b", "masked_a", "masked_b", "background_a", "background_b", "blind_a", "blind_b")


def load_case(name):
    g = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))
    cfg = dict(LO.DEFAULT_LOSS_CONFIG)
    for k, v in zip(g["cfg_keys"], g["cfg_vals"]):
        cfg[str(k)] = type(cfg[str(k)])(v)
    return g, cfg


@pytest.mark.parametrize("name", ["loss_unit_d4", "loss_unit_d16"])
def test_float64_oracle_matches_executed_reference(name):
    g, cfg = load_case(name)
    H, W = int(g["H"]), int(g["W"])
    five, (dA, dB) = UO.unit_loss(g["low_a"], g["low_b"], H, W, {k: g[k] for k in IDX_KEYS}, cfg)
    # the reference ran in float32 (its upsample, norm and loss); the restatement in float64
    np.testing.assert_allclose(five, g["five"], rtol=2e-5, atol=1e-7)
    for got, ref in ((dA, g["dA"]), (dB, g["dB"])):
        got = got.numpy()
        assert np.linalg.norm(got - ref) <= 1e-4 * np.linalg.norm(ref)
    # the hard-negative counts of the same unit descriptors
    D = g["low_a"].shape[1]
    ya = UO.unit_upsample(g["low_a"], H, W)[0].reshape(D, -1).T.numpy()
    yb = UO.unit_upsample(g["low_b"], H, W)[0].reshape(D, -1).T.numpy()
    _, counts = LO.np_within_scene_loss(ya, yb, {k: g[k] for k in IDX_KEYS}, cfg, W)
    assert tuple(counts) == tuple(g["counts"])


def test_unit_upsample_oracle_has_unit_norm_and_nan_at_zero():
    low = torch.randn(2, 5, 4, 6, dtype=torch.float64)
    low[1, :, 0, 0] = 0.0
    y = UO.unit_upsample(low, 32, 48)
    n = y.norm(dim=1)
    assert torch.isnan(n[1, 0, 0])
    n[1, 0, 0] = 1.0
    assert torch.allclose(n, torch.ones_like(n), atol=1e-12)


def _cpu_network(normalize):
    return pdc_b200.DenseCorrespondenceNetwork(resnet_dilated.Resnet34_8s(num_classes=3), 3, image_width=48, image_height=32,
                                               normalize=normalize)


FAKE = ctypes.c_void_p(1 << 20)       # never dereferenced: every call below is refused first


def test_lowres_v2_refusals_launch_nothing():
    terms = (N.LossTerm * 1)()
    terms[0].idx_a = terms[0].idx_b = 1 << 20
    terms[0].n = 4
    terms[0].kind = N.TERM_MATCH

    def fwd(flags=N.LOWRES_UNIT, la=FAKE, D=4, h=6, w=8, H=48, W=64, sums=FAKE, n_terms=1):
        return N.lib.ddn_contrastive_terms_forward_lowres_v2(la, FAKE, 1, h, w, H, W, D, terms, n_terms, sums, FAKE, flags, None)

    def bwd(flags=N.LOWRES_UNIT, la=FAKE, D=4, h=6, w=8, H=48, W=64, scratch=FAKE, n_terms=1):
        return N.lib.ddn_contrastive_terms_backward_lowres_v2(la, FAKE, 1, h, w, H, W, D, terms, n_terms, FAKE, None, FAKE, FAKE,
                                                              scratch, flags, None)

    before = N.launch_count()
    for kw in (dict(flags=2), dict(flags=-1), dict(flags=1 << 8), dict(la=None), dict(D=0), dict(D=33), dict(h=0),
               dict(H=5), dict(W=7), dict(n_terms=0), dict(n_terms=9)):
        assert fwd(**kw) == -1, kw
        assert bwd(**kw) == -1, kw
    assert fwd(sums=None) == -1
    assert bwd(scratch=None) == -1
    assert bwd(la=ctypes.c_void_p((1 << 20) + 4)) == -1         # the backward's float4 / fp64 accesses need 16-byte alignment
    assert N.launch_count() == before


def test_net_v2_refusals_launch_nothing():
    arch, B, H, W, D = N.ARCH_RESNET34_8S, 2, 64, 96, 4
    base = N.lib.ddn_net_workspace_bytes_v2(arch, B, H, W, D, N.MODE_TRAIN, N.PRECISION_BF16X3, 0)
    assert base == N.lib.ddn_net_workspace_bytes(arch, B, H, W, D, N.MODE_TRAIN, N.PRECISION_BF16X3)
    unit = N.lib.ddn_net_workspace_bytes_v2(arch, B, H, W, D, N.MODE_TRAIN, N.PRECISION_BF16X3, N.NET_UNIT_DESCRIPTORS)
    assert unit >= base + 4 * B * D * H * W                       # the backward's cotangent through the normalisation
    # inference keeps nothing for a backward: the flag costs no workspace there
    assert N.lib.ddn_net_workspace_bytes_v2(arch, B, H, W, D, N.MODE_INFER, N.PRECISION_BF16X3, N.NET_UNIT_DESCRIPTORS) == \
        N.lib.ddn_net_workspace_bytes(arch, B, H, W, D, N.MODE_INFER, N.PRECISION_BF16X3)
    for flags in (2, -1, 1 << 4):
        assert N.lib.ddn_net_workspace_bytes_v2(arch, B, H, W, D, N.MODE_TRAIN, N.PRECISION_BF16X3, flags) == 0
    ws = ctypes.c_void_p(1 << 24)

    def fwd(flags=N.NET_UNIT_DESCRIPTORS, x=FAKE, nbytes=unit, D_=D, H_=H, groups=2):
        return N.lib.ddn_net_forward_v2(arch, x, FAKE, FAKE, FAKE, ws, nbytes, B, H_, W, D_, N.MODE_TRAIN, groups, 0.1, 1e-5,
                                        N.PRECISION_BF16X3, FAKE, flags, None)

    def bwd(flags=N.NET_UNIT_DESCRIPTORS, dy=FAKE, nbytes=unit, D_=D, H_=H, groups=2):
        return N.lib.ddn_net_backward_v2(arch, dy, None, FAKE, FAKE, ws, nbytes, B, H_, W, D_, N.MODE_TRAIN, groups, 1e-5,
                                         N.PRECISION_BF16X3, flags, N.NO_BUCKET_CALLBACK, None, None)

    before = N.launch_count()
    for kw in (dict(flags=2), dict(flags=-1), dict(D_=33), dict(H_=60), dict(groups=3)):
        assert fwd(**kw) == -1, kw
        assert bwd(**kw) == -1, kw
    assert fwd(x=None) == -1 and bwd(dy=None) == -1
    assert fwd(nbytes=base) == -2                                 # the unit plan needs more than the plain one
    assert bwd(nbytes=base) == -2
    assert N.launch_count() == before


def test_unit_upsample_refusals_launch_nothing():
    def fwd(x=FAKE, y=FAKE, N_=2, D=4, h=4, w=6, H=32, W=48):
        return N.lib.ddn_upsample_bilinear_unit_forward(x, y, N_, D, h, w, H, W, None)

    def bwd(x=FAKE, dy=FAKE, dx=FAKE, scratch=FAKE, N_=2, D=4, h=4, w=6, H=32, W=48):
        return N.lib.ddn_upsample_bilinear_unit_backward(x, dy, dx, scratch, N_, D, h, w, H, W, None)

    before = N.launch_count()
    for kw in (dict(x=None), dict(N_=0), dict(D=0), dict(D=33), dict(h=0), dict(W=-1)):
        assert fwd(**kw) == -1, kw
        assert bwd(**kw) == -1, kw
    assert fwd(y=None) == -1
    assert bwd(dy=None) == -1 and bwd(dx=None) == -1 and bwd(scratch=None) == -1
    assert N.launch_count() == before


def test_unit_flag_of_the_tag():
    low = torch.zeros(1, 12, 3)
    y = torch.zeros(1, 3, 32, 48)
    resnet_dilated.attach_lowres(y, low, 32, 48)
    assert resnet_dilated.lowres_of(y)[4] is False
    resnet_dilated.attach_lowres(y, low, 32, 48, unit=True)
    tag = resnet_dilated.lowres_of(y)
    assert tag[0] is low and tag[1:3] == (32, 48) and tag[4] is True
    # process_network_output keeps the tag, unit flag included (a view: same version counter)
    dcn = _cpu_network(normalize=True)
    p = dcn.process_network_output(y, 1)
    assert resnet_dilated.lowres_of(p)[4] is True and resnet_dilated.lowres_of(p)[0] is low
    # an in-place edit drops it
    y.add_(1.0)
    assert resnet_dilated.lowres_of(y) is None and resnet_dilated.lowres_of(p) is None


def test_fused_route_needs_matching_unit_flags():
    from pdc_b200 import loss_composer
    H, W = 32, 48
    low_a, low_b = torch.zeros(1, 24, 3), torch.zeros(1, 24, 3)
    pa, pb = torch.zeros(1, H * W, 3), torch.zeros(1, H * W, 3)
    resnet_dilated.attach_lowres(pa, low_a, H, W, unit=True)
    resnet_dilated.attach_lowres(pb, low_b, H, W, unit=True)
    r = loss_composer._fused_lowres(pa, pb, W)
    assert r[0] is low_a and r[1] is low_b and r[2] == (4, 6, H, W) and r[3] is True
    resnet_dilated.attach_lowres(pb, low_b, H, W, unit=False)
    assert loss_composer._fused_lowres(pa, pb, W) is None       # a mixed pair takes the generic gather
    resnet_dilated.attach_lowres(pa, low_a, H, W)
    assert loss_composer._fused_lowres(pa, pb, W)[3] is False


def test_per_pixel_normalize_needs_a_normalizing_network():
    dcn = _cpu_network(normalize=False)
    img = torch.zeros(1, 3, 32, 48)
    with pytest.raises(ValueError, match="normalize"):
        dcn.forward_pair(img, img, per_pixel_normalize=True)
