"""The inputs and calls on which the oracle restatements are compared with the reference's own code.

TEST INFRASTRUCTURE.  oracle/make_golden.py runs every case below on the EXECUTED reference (oracle/build_ref.py,
oracle/ref_loader.py) and stores the results in tests/golden/reference_checks.npz; tests/test_oracle_ref_cpu.py and
tests/test_oracle_cpu.py run the same cases on the restatements (oracle/loss_oracle.py, oracle/resnet34_8s_oracle.py) and
compare with the stored results, so that the comparison needs nothing outside the repository.

Every case returns a flat {key: numpy array} dict (nested tuples / lists of results get keys "name/i/j").
"""
import numpy as np
import torch

from oracle import loss_oracle as LO
from oracle.resnet34_8s_oracle import process_network_output


def flatten(prefix, x, out):
    if isinstance(x, torch.Tensor):
        out[prefix] = x.detach().numpy().copy()
    elif isinstance(x, (tuple, list)):
        for i, v in enumerate(x):
            flatten("%s/%d" % (prefix, i), v, out)
    else:
        out[prefix] = np.array(x)
    return out


def _run(pcl, get_loss, A, B, idx, match_type=0):
    A = A.clone().requires_grad_(); B = B.clone().requires_grad_()
    _, D, H, W = A.shape
    pa, pb = process_network_output(A, 1, D, H, W), process_network_output(B, 1, D, H, W)
    five = get_loss(pcl, torch.tensor([match_type]), pa, pb, idx["matches_a"], idx["matches_b"], idx["masked_a"], idx["masked_b"],
                    idx["background_a"], idx["background_b"], idx["blind_a"], idx["blind_b"])
    five[0].reshape(()).backward()
    return [float(t) for t in five], A.grad, B.grad


def every_loss_method(pcl_cls):
    """Every public method of PixelwiseContrastiveLoss (pixelwise_contrastive_loss.py:35-411) on one seeded input."""
    H, W, D, P = 12, 20, 5, 240
    gen = torch.Generator().manual_seed(3)
    A = 0.3 * torch.randn(1, P, D, generator=gen); B = 0.3 * torch.randn(1, P, D, generator=gen)
    ma = torch.randint(0, P, (7,), generator=gen); mb = torch.randint(0, P, (7,), generator=gen)
    na = ma.repeat_interleave(4); nb = torch.randint(0, P, (28,), generator=gen)
    cfg = dict(LO.DEFAULT_LOSS_CONFIG, M_descriptor=0.6)
    o = pcl_cls([H, W], dict(cfg))
    out = {}
    flatten("match_loss", o.match_loss(A, B, ma, mb), out)
    for inv in (False, True):
        flatten("non_match_descriptor_loss/%d" % inv, o.non_match_descriptor_loss(A, B, na, nb, M=0.6, invert=inv), out)
        flatten("non_match_loss_descriptor_only/%d" % inv, o.non_match_loss_descriptor_only(A, B, na, nb, M_descriptor=0.6, invert=inv), out)
    flatten("non_match_loss_with_l2_pixel_norm", o.non_match_loss_with_l2_pixel_norm(A, B, mb, na, nb, M_descriptor=0.6, M_pixel=7), out)
    flatten("l2_pixel_loss", o.l2_pixel_loss(mb, nb, M_pixel=7), out)
    flatten("flattened_pixel_locations_to_u_v", o.flattened_pixel_locations_to_u_v(nb.unsqueeze(1)), out)
    for l2 in (False, True):
        flatten("get_loss_matched_and_non_matched_with_l2/%d" % l2,
                o.get_loss_matched_and_non_matched_with_l2(A, B, ma, mb, na, nb, use_l2_pixel_loss=l2), out)
    flatten("get_triplet_loss", o.get_triplet_loss(A, B, ma, mb, na, nb, 0.1), out)
    flatten("get_loss_original", o.get_loss_original(A, B, ma, mb, na, nb), out)
    # single-element index tensors (the unsqueeze branch, pcl.py:161-163,199-201) and identical descriptors (d = 0)
    one, two = torch.tensor([7]), torch.tensor([11])
    flatten("match_loss_single", o.match_loss(A, B, one, two), out)
    flatten("non_match_descriptor_loss_single", o.non_match_descriptor_loss(A, B, one, two, M=100.0), out)
    Z = torch.zeros(1, P, D)
    flatten("non_match_loss_descriptor_only_zero", o.non_match_loss_descriptor_only(Z, Z, na, nb, M_descriptor=0.5), out)
    return out


COMPOSER_OVERRIDES = ({}, {"scale_by_hard_negatives": False}, {"scale_by_hard_negatives_DIFFERENT_OBJECT": False},
                      {"M_masked": 1e-6, "M_background": 1e-6})      # the last: zero hard negatives -> max(h, 1)
COMPOSER_MATCH_TYPES = (0, 2, 3, 4)                                  # within-scene, different-object, multi, synthetic multi


def composer_inputs():
    H, W, D, P = 10, 16, 3, 160
    gen = torch.Generator().manual_seed(9)
    A = 0.3 * torch.randn(1, D, H, W, generator=gen); B = 0.3 * torch.randn(1, D, H, W, generator=gen)
    ma = torch.randint(0, P, (6,), generator=gen); mb = torch.randint(0, P, (6,), generator=gen)
    idx = dict(matches_a=ma, matches_b=mb, masked_a=ma.repeat_interleave(3), masked_b=torch.randint(0, P, (18,), generator=gen),
               background_a=ma.repeat_interleave(2), background_b=torch.randint(0, P, (12,), generator=gen),
               blind_a=torch.randint(0, P, (9,), generator=gen), blind_b=torch.randint(0, P, (9,), generator=gen))
    return A, B, idx


def composer_branches(pcl_cls, get_loss, empty_tensor):
    """loss_composer.get_loss over every configuration / match type above, the blind sentinel [-1], and the exception the
    across-scene (NameError / UnboundLocalError) and an unknown (ValueError) match type raise."""
    A, B, idx = composer_inputs()
    H, W = A.shape[2:]
    out = {}
    for i, over in enumerate(COMPOSER_OVERRIDES):
        cfg = dict(LO.DEFAULT_LOSS_CONFIG); cfg.update(over)
        for mt in COMPOSER_MATCH_TYPES:
            five, dA, dB = _run(pcl_cls([H, W], dict(cfg)), get_loss, A, B, idx, mt)
            flatten("cfg%d/mt%d" % (i, mt), [np.array(five), dA, dB], out)
    idx_e = dict(idx, blind_a=empty_tensor(), blind_b=empty_tensor())
    five, _, _ = _run(pcl_cls([H, W], dict(LO.DEFAULT_LOSS_CONFIG)), get_loss, A, B, idx_e, 0)
    out["sentinel/five"] = np.array(five)
    out["empty_tensor"] = empty_tensor().numpy().copy()
    for name, mt in (("across_scene", 1), ("unknown", 9)):
        try:
            _run(pcl_cls([H, W], dict(LO.DEFAULT_LOSS_CONFIG)), get_loss, A, B, idx, mt)
            out["raises/" + name] = np.array("")
        except Exception as e:        # the type is the result here
            out["raises/" + name] = np.array(type(e).__name__)
    return out


def sampler_inputs():
    H, W, k = 30, 40, 5
    gen = torch.Generator().manual_seed(4)
    ma = torch.randint(0, H * W, (11,), generator=gen)
    n = len(ma) * k
    ru, rv = torch.rand(n, generator=gen), torch.rand(n, generator=gen)
    mask = torch.zeros(H, W); mask[5:20, 8:30] = 1.0
    return H, W, k, ma, ru, rv, (mask, None, torch.zeros(H, W))


def reprojection_scene():
    """A ray-cast plane seen from two poses, with no-return pixels (depth 0) in A and an occluder in front of the plane in B."""
    H, W, n = 120, 160, 900
    K = np.array([[133.4, 0, 79.8], [0, 133.7, 59.1], [0, 0, 1.0]])

    def pose(rx, ry, t):
        cx, sx, cy, sy = np.cos(rx), np.sin(rx), np.cos(ry), np.sin(ry)
        Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]); Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
        T = np.eye(4); T[:3, :3] = Ry.dot(Rx); T[:3, 3] = t
        return T
    pa, pb = pose(0.01, -0.02, [0, 0, 0]), pose(-0.04, 0.1, [0.15, -0.03, 0.04])
    nrm, d0 = np.array([-0.1, 0.05, 1.0]), 1.2

    def render(T):
        us, vs = np.meshgrid(np.arange(W), np.arange(H))
        rays = np.linalg.inv(K).dot(np.stack([us.ravel(), vs.ravel(), np.ones(H * W)]))
        s = (d0 - nrm.dot(T[:3, 3])) / nrm.dot(T[:3, :3].dot(rays))
        return (s * 1000.0).reshape(H, W)
    da = np.round(render(pa)).astype(np.uint16); db = np.round(render(pb)).astype(np.uint16)
    da[10:30, 20:50] = 0
    db[60:80, 100:130] = 300
    mask = np.zeros((H, W), dtype=np.float32); mask[5:110, 10:150] = 1.0
    ru = torch.rand(n, generator=torch.Generator().manual_seed(8))
    return da, pa, db, pb, mask, ru, K, n
