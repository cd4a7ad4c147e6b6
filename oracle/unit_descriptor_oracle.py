"""Float64 restatement of the reference's ``normalize`` option under its loss (dense_correspondence_network.py:256-259 on a
batch of one, then loss_composer.get_loss), starting from the map the upsample blends.

    res = upsample_bilinear(low, align_corners=True)      resnet_dilated.py:320 (source coordinates in fp32, as there)
    y   = res / ||res||_2 over the channels, per pixel     net.py:256-259 (N == 1)
    five = get_loss(y)                                    oracle/loss_oracle.py (the restated reference loss)

``unit_upsample`` is the descriptor image the network writes with per-pixel normalisation; ``unit_loss`` gives the five loss
values and the gradients with respect to the un-normalised ``res`` of both images, the quantities
tests/golden/loss_unit_d*.npz stores from the executed reference (oracle/make_golden_unit.py).
"""
import numpy as np
import torch

from oracle import loss_oracle as LO
from oracle.resnet34_8s_oracle import process_network_output


def _source(n_in, n_out):
    """Source cells and weight of every output index, computed in fp32 as the reference's fp32 upsample computes them
    (ATen upsample_bilinear2d, align_corners=True: scale = (in-1)/(out-1), r = scale * dst, lambda = r - (int)r)."""
    scale = np.float32(n_in - 1) / np.float32(n_out - 1) if n_out > 1 else np.float32(0.0)
    r = (scale * np.arange(n_out, dtype=np.float32)).astype(np.float32)
    i0 = np.minimum(r.astype(np.int64), n_in - 1)
    i1 = np.where(i0 < n_in - 1, i0 + 1, i0)
    lam = (r - i0.astype(np.float32)).astype(np.float32)
    return torch.from_numpy(i0), torch.from_numpy(i1), torch.from_numpy(lam.astype(np.float64))


def upsample(low, H, W):
    """[N, D, h, w] -> [N, D, H, W] bilinear, align_corners=True (nn.functional.upsample_bilinear): the reference's source
    coordinates (fp32), the blend in low's dtype; differentiable."""
    h, w = low.shape[2], low.shape[3]
    h0, h1, lh = _source(h, H)
    w0, w1, lw = _source(w, W)
    lh = lh.to(low.dtype).view(1, 1, H, 1); lw = lw.to(low.dtype).view(1, 1, 1, W)
    r0, r1 = low.index_select(2, h0), low.index_select(2, h1)
    top = (1 - lw) * r0.index_select(3, w0) + lw * r0.index_select(3, w1)
    bot = (1 - lw) * r1.index_select(3, w0) + lw * r1.index_select(3, w1)
    return (1 - lh) * top + lh * bot


def unit_upsample(low, H, W):
    """Float64 unit descriptors [N, D, H, W] of the low-resolution maps [N, D, h, w] (every image and pixel on its own)."""
    res = upsample(torch.as_tensor(low).double(), H, W)
    return res / res.norm(dim=1, keepdim=True)


def unit_loss(low_a, low_b, H, W, idx, cfg):
    """-> (five floats, (dA, dB) float64 [1, D, H, W]) for one pair of [1, D, h, w] maps; ``idx``: dict of 1-D int64 index
    arrays as the fixtures store them (blind_* = [-1] when there are none)."""
    ra = upsample(torch.as_tensor(low_a).double(), H, W).requires_grad_()
    rb = upsample(torch.as_tensor(low_b).double(), H, W).requires_grad_()
    D = ra.shape[1]
    ya = ra / ra.norm(dim=1, keepdim=True)
    yb = rb / rb.norm(dim=1, keepdim=True)
    pa, pb = process_network_output(ya, 1, D, H, W), process_network_output(yb, 1, D, H, W)
    t = {k: torch.from_numpy(np.asarray(v)).long() for k, v in idx.items()}
    pcl = LO.TorchPixelwiseContrastiveLoss([H, W], dict(cfg))
    five = LO.get_loss(pcl, torch.tensor([LO.SpartanDatasetDataType.SINGLE_OBJECT_WITHIN_SCENE]), pa, pb,
                       t["matches_a"], t["matches_b"], t["masked_a"], t["masked_b"], t["background_a"], t["background_b"],
                       t["blind_a"], t["blind_b"])
    five[0].reshape(()).backward()
    return [float(v) for v in five], (ra.grad, rb.grad)
