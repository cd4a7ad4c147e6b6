"""GPU: the tensor-core weight gradient at the sizes the training benchmark runs (16 images of 60x80, 1200 k-blocks of 64
pixels), where the persistent kernel splits the pixels into many chunks, and layer1 (16 images of 120x160), where each CTA of
the halo kernel keeps one fp32 accumulator over ~18 tiles, against the fp32 FFMA instrument on the same GPU."""
import functools

import pytest
import torch

from pdc_b200 import ops, _native as N

pytestmark = pytest.mark.gpu
DEV = "cuda"

WGRAD_CASES = [
    # N, H, W, Cin, Cout, k, stride, pad, dil
    (16, 60, 80, 512, 512, 3, 1, 4, 4),     # layer4 3x3: 144 tiles, half of all weight-gradient MACs
    (16, 60, 80, 256, 512, 3, 1, 4, 4),     # layer4.0.conv1
    (16, 60, 80, 256, 256, 3, 1, 2, 2),     # layer3 3x3
    (16, 60, 80, 128, 256, 1, 1, 0, 1),     # layer3.0.downsample
    (16, 60, 80, 256, 512, 1, 1, 0, 1),     # layer4.0.downsample
    (16, 120, 160, 64, 128, 3, 2, 1, 1),    # layer2.0.conv1: 64-channel tiles, stride 2
    (16, 120, 160, 64, 64, 3, 1, 1, 1),     # layer1 3x3: wgrad64_halo_kernel, ~18 tiles per CTA in one fp32 accumulator
]
TOL = {"bf16x3": 2e-5, "bf16": 8e-3}
PREC = {"bf16x3": N.PRECISION_BF16X3, "bf16": N.PRECISION_BF16}


def rel(a, b):
    a = a.double(); b = b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


@functools.lru_cache(maxsize=2)
def operands(case):
    n, h, w, cin, cout, k, s, p, d = case
    g = torch.Generator(device=DEV).manual_seed(sum(case))
    x = torch.randn(n, h, w, cin, generator=g, device=DEV)
    wt = torch.randn(cout, cin, k, k, generator=g, device=DEV) * (2.0 / (k * k * cin)) ** 0.5
    ho = (h + 2 * p - d * (k - 1) - 1) // s + 1
    wo = (w + 2 * p - d * (k - 1) - 1) // s + 1
    dy = torch.randn(n, ho, wo, cout, generator=g, device=DEV)
    _, dw_ref = ops.conv2d_backward(x, wt, dy, s, p, d, need_dx=False, precision=N.PRECISION_FP32_SIMT)
    return x, wt, dy, dw_ref


def wgrad(case, precision):
    _, _, _, _, _, _, s, p, d = case
    x, wt, dy, _ = operands(case)
    _, dw = ops.conv2d_backward(x, wt, dy, s, p, d, need_dx=False, precision=PREC[precision])
    return dw


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
@pytest.mark.parametrize("case", WGRAD_CASES)
def test_wgrad_at_training_size(case, precision):
    err = rel(wgrad(case, precision), operands(case)[3])
    assert err <= TOL[precision], err


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_wgrad_with_reserved_sms(precision):
    """Fewer workers: a smaller persistent grid and a different chunk count, same accuracy."""
    case = WGRAD_CASES[0]
    assert N.lib.ddn_set_reserved_sms(8) == 0
    try:
        dw = wgrad(case, precision)
    finally:
        assert N.lib.ddn_set_reserved_sms(0) == 0
    err = rel(dw, operands(case)[3])
    assert err <= TOL[precision], err


@pytest.mark.parametrize("case", [WGRAD_CASES[0], WGRAD_CASES[5], WGRAD_CASES[6]])
def test_wgrad_is_deterministic(case):
    a = wgrad(case, "bf16x3")
    b = wgrad(case, "bf16x3")
    assert torch.equal(a, b)
