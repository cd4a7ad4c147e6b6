"""GPU: unit-length descriptors -- the reference's ``normalize`` option (dense_correspondence_network.py:256-259) per pixel,
written by the upsample kernel (DDN_NET_UNIT_DESCRIPTORS) and applied to every sampled descriptor by the loss fused with the
upsample (DDN_LOWRES_UNIT).

* forward_pair(..., per_pixel_normalize=True) images against a float64 restatement of the network's own low-resolution map,
  at 64x96 and 640x480, B = 1 and 8, D in {1, 3, 4, 16, 32}; norms are 1 to fp32 rounding;
* at B = 1 forward / forward_pair return today's values bit for bit and carry the unit tag; the fused loss equals the
  generic full-resolution path and the executed reference's fixtures (tests/golden/loss_unit_d*.npz);
* at B = 8 the fused unit loss equals the generic gather on the torch-normalised images for every term kind, ragged
  lengths and a mixed pair-type batch;
* parameter gradients through the normalisation against float64 (both backbones at 64x96, Resnet34_8s at 640x480);
* the full-resolution cotangent (a triplet loss) against autograd through torch's normalisation, and the standalone unit
  upsample entry points (zero descriptor -> NaN);
* no host synchronisation in a fused unit step, the same launch count at B = 1 and 8, two steps bit-identical."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import pdc_b200
from pdc_b200 import _native as N
from pdc_b200 import loss_composer, resnet_dilated, synthetic
from pdc_b200 import sampling as S
from pdc_b200.loss_composer import SpartanDatasetDataType as T
from oracle import loss_oracle as LO
from oracle import resnet34_8s_oracle as R34
from oracle import resnet50_8s_oracle as R50
from oracle import unit_descriptor_oracle as UO

pytestmark = pytest.mark.gpu
DEV = "cuda"
IDX_KEYS = ("matches_a", "matches_b", "masked_a", "masked_b", "background_a", "background_b", "blind_a", "blind_b")
BATCH_KEYS = [k % s for k in ("matches_%s", "masked_non_matches_%s", "background_non_matches_%s", "blind_non_matches_%s")
              for s in "ab"]


def rel(x, y):
    x = x.detach().double().cpu(); y = y.detach().double().cpu()
    return float((x - y).norm() / max(float(y.norm()), 1e-30))


def network(D, H, W, backbone="Resnet34_8s", normalize=True):
    dcn = pdc_b200.DenseCorrespondenceNetwork.from_config(
        {"descriptor_dimension": D, "image_width": W, "image_height": H, "normalize": normalize,
         "backbone": {"model_class": "Resnet", "resnet_name": backbone}}, load_stored_params=False)
    oracle = (R34 if backbone == "Resnet34_8s" else R50).seeded_oracle(D=D, seed=0)
    dcn.fcn.load_state_dict(oracle.state_dict())
    return dcn


def unit_bound(low64, H, W):
    """Per-pixel bound on |fp32 unit descriptor - float64|: the fp32 blend errs by a few ulps of the blended magnitudes
    sum_k w_k |low_k|, and the division by ||x|| scales that error by 1 / ||x||, so pixels whose blend nearly cancels are
    ill-conditioned in any fp32 evaluation (the reference's included)."""
    x = UO.upsample(low64, H, W)
    a = UO.upsample(low64.abs(), H, W)
    return 1e-6 * (1.0 + a.norm(dim=1, keepdim=True) / x.norm(dim=1, keepdim=True))


def low_nchw(tag, B, D):
    low, H, W = tag[0], tag[1], tag[2]
    return low.detach().view(B, H // 8, W // 8, D).permute(0, 3, 1, 2)


# ---------------------------------------------------------------------------------------------------------------- images
@pytest.mark.parametrize("H,W", [(64, 96), (480, 640)])
@pytest.mark.parametrize("B", [1, 8])
@pytest.mark.parametrize("D", [1, 3, 4, 16, 32])
def test_unit_images_vs_float64(H, W, B, D):
    dcn = network(D, H, W)
    dcn.train()
    g = torch.Generator().manual_seed(D * 100 + B)
    a = torch.randn(B, 3, H, W, generator=g).to(DEV); b = torch.randn(B, 3, H, W, generator=g).to(DEV)
    with torch.no_grad():
        ya, yb = dcn.forward_pair(a, b, per_pixel_normalize=True)
    for y in (ya, yb):
        tag = resnet_dilated.lowres_of(y)
        assert tag is not None and tag[4] is True
        low64 = low_nchw(tag, B, D).cpu().double()
        ref = UO.unit_upsample(low64, H, W)
        got = y.detach().double().cpu()
        assert bool(((got - ref).abs() <= unit_bound(low64, H, W)).all()), float((got - ref).abs().max())
        n = got.norm(dim=1)
        assert float((n - 1).abs().max()) < 1e-6 * max(1.0, D ** 0.5)


# ---------------------------------------------------------------------------------------------------------- batch of one
def test_batch_one_keeps_todays_values_and_takes_the_fused_unit_loss():
    D, H, W = 4, 64, 96
    dcn = network(D, H, W)
    dcn.train()
    data = synthetic.make_pair_batch(1, H, W, 40, 120, 120, 30, seed=7)
    d = {k: (v.to(DEV) if v is not None else None) for k, v in data.items()}
    with torch.no_grad():
        raw = dcn.fcn(d["img_a"])
        want = raw / torch.norm(raw, 2, 1)
        got = dcn.forward(d["img_a"])
        assert torch.equal(got, want)
        assert resnet_dilated.lowres_of(got)[4] is True
        raw = dcn.fcn(torch.cat([d["img_a"], d["img_b"]], 0), bn_groups=2)
        wa, wb = raw[:1] / torch.norm(raw[:1], 2, 1), raw[1:] / torch.norm(raw[1:], 2, 1)
        ga, gb = dcn.forward_pair(d["img_a"], d["img_b"])
        assert torch.equal(ga, wa) and torch.equal(gb, wb)
        assert resnet_dilated.lowres_of(ga)[4] is True and resnet_dilated.lowres_of(gb)[4] is True
    # the fused unit loss on these tensors vs the generic gather on copies of them (no tag), gradients at the low map
    cfg = dict(LO.DEFAULT_LOSS_CONFIG, M_masked=1.5, M_background=1.2)
    res = []
    for fused in (True, False):
        ya, yb = dcn.forward_pair(d["img_a"], d["img_b"])
        pa, pb = dcn.process_network_output(ya, 1), dcn.process_network_output(yb, 1)
        if not fused:
            pa, pb = pa.clone(), pb.clone()
        assert (loss_composer._fused_lowres(pa, pb, W) is not None) == fused
        pcl = pdc_b200.PixelwiseContrastiveLoss(dcn.image_shape, dict(cfg))
        five = loss_composer.get_loss(pcl, torch.zeros(1, dtype=torch.int64), pa, pb, d["matches_a"], d["matches_b"],
                                      d["masked_a"], d["masked_b"], d["background_a"], d["background_b"], d["blind_a"],
                                      d["blind_b"])
        five[0].backward()
        res.append(([float(t) for t in five], {k: p.grad.detach().clone() for k, p in dcn.fcn.named_parameters()}))
        dcn.zero_grad(set_to_none=True)
    (f1, g1), (f0, g0) = res
    assert f1[0] > 0 and f1[2] > 0
    for x, y in zip(f1, f0):
        assert abs(x - y) <= 1e-5 * max(1.0, abs(y)), (f1, f0)
    assert rel(g1["resnet34_8s.fc.weight"], g0["resnet34_8s.fc.weight"]) < 1e-4


def _fixture(name):
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", name + ".npz"))
    cfg = dict(LO.DEFAULT_LOSS_CONFIG)
    for k, v in zip(g["cfg_keys"], g["cfg_vals"]):
        cfg[str(k)] = type(cfg[str(k)])(v)
    return g, cfg


@pytest.mark.parametrize("name", ["loss_unit_d4", "loss_unit_d16"])
def test_fused_unit_loss_equals_executed_reference(name):
    g, cfg = _fixture(name)
    H, W = int(g["H"]), int(g["W"])
    D = g["low_a"].shape[1]
    leaves, preds = [], []
    for key in ("low_a", "low_b"):
        low = torch.from_numpy(g[key]).to(DEV).permute(0, 2, 3, 1).reshape(1, -1, D).contiguous().requires_grad_()
        y = torch.empty(1, H * W, D, device=DEV)          # the values are never read on the fused route
        resnet_dilated.attach_lowres(y, low, H, W, unit=True)
        leaves.append(low); preds.append(y)
    pcl = pdc_b200.PixelwiseContrastiveLoss([H, W], dict(cfg))
    pcl.debug = True
    idx = {k: torch.from_numpy(g[k]).to(DEV) for k in IDX_KEYS}
    five = loss_composer.get_loss(pcl, torch.zeros(1, dtype=torch.int64), preds[0], preds[1], *[idx[k] for k in IDX_KEYS])
    five[0].backward()
    np.testing.assert_allclose([float(t) for t in five], g["five"], rtol=1e-5, atol=1e-7)
    assert pcl.debug_data["num_hard_negatives_device"].cpu()[0, 1:4].tolist() == g["counts"].tolist()
    # d(loss)/d(low) = upsample^T(d(loss)/d(res)), the fixture's gradient taken to the low map in float64
    for leaf, key, dkey in ((leaves[0], "low_a", "dA"), (leaves[1], "low_b", "dB")):
        low64 = torch.from_numpy(g[key]).double().requires_grad_()
        UO.upsample(low64, H, W).backward(torch.from_numpy(g[dkey]).double())
        ref = low64.grad.permute(0, 2, 3, 1).reshape(1, -1, D)
        assert rel(leaf.grad, ref) < 1e-5


# --------------------------------------------------------------------------------------------------------------- batch 8
def unit_route(lows, H, W, fused):
    """The low maps [B, h*w, D] as leaves, their bilinear upsample normalised per pixel by torch, as [B, H*W, D] views:
    tagged with the unit flag (fused) or not (the generic gather differentiates through torch's normalisation)."""
    leaves, preds = [], []
    for t in lows:
        leaf = t.clone().to(DEV).requires_grad_()
        B, _, D = leaf.shape
        x = F.interpolate(leaf.view(B, H // 8, W // 8, D).permute(0, 3, 1, 2), size=(H, W), mode="bilinear", align_corners=True)
        y = x / x.norm(dim=1, keepdim=True)
        if fused:
            y = y.detach()
        p = y.view(B, D, H * W).permute(0, 2, 1)
        if fused:
            resnet_dilated.attach_lowres(p, leaf, H, W, unit=True)
        leaves.append(leaf); preds.append(p)
    return leaves, preds


def both_routes(B, D, H, W, run, seed=3):
    g = torch.Generator().manual_seed(seed)
    lows = [0.3 * torch.randn(B, (H // 8) * (W // 8), D, generator=g) for _ in range(2)]
    out = []
    for fused in (True, False):
        leaves, (pa, pb) = unit_route(lows, H, W, fused)
        assert (loss_composer._fused_lowres(pa, pb, W) is not None) == fused
        five = run(pa, pb)
        five[0].backward()
        out.append(([float(t) for t in five], [t.grad for t in leaves]))
    (f1, g1), (f0, g0) = out
    assert f1[0] > 0
    for x, y in zip(f1, f0):
        assert abs(x - y) <= 1e-5 * max(1.0, abs(y)), (f1, f0)
    for a, b in zip(g1, g0):
        assert rel(a, b) < 1e-5
    return f1


CASES = {
    "scaled": dict(M_masked=1.5, M_background=1.2),
    "unscaled": dict(M_masked=1.5, M_background=1.2, scale_by_hard_negatives=False),
    "pixel_weight": dict(M_masked=1.5, M_background=1.2, use_l2_pixel_loss_on_masked_non_matches=True,
                         use_l2_pixel_loss_on_background_non_matches=True, M_pixel=25),
}


@pytest.mark.parametrize("D", [3, 4, 7, 8, 16, 32])
@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("blind", [0, 50], ids=["no_blind", "blind"])
def test_batch8_fused_unit_loss_equals_generic(D, case, blind):
    B, H, W = 8, 64, 96
    data = synthetic.make_pair_batch(B, H, W, 60, 180, 120, blind, seed=5)
    d = {k: (v.to(DEV) if v is not None else None) for k, v in data.items()}
    if not blind:
        d["blind_a"] = d["blind_b"] = loss_composer.empty_tensor().to(DEV)
    cfg = dict(LO.DEFAULT_LOSS_CONFIG, **CASES[case])

    def run(pa, pb):
        pcl = pdc_b200.PixelwiseContrastiveLoss([H, W], dict(cfg))
        return loss_composer.get_loss(pcl, torch.zeros(B, dtype=torch.int64), pa, pb, *[d[k] for k in IDX_KEYS])
    f = both_routes(B, D, H, W, run)
    if blind:
        assert f[4] > 0


@pytest.mark.parametrize("D", [3, 16])
def test_batch8_ragged_lengths(D):
    B, H, W = 8, 64, 96
    g = torch.Generator().manual_seed(9)
    P = H * W
    lists = {}
    for k, n_max in (("matches", 50), ("masked", 150), ("background", 100), ("blind", 40)):
        n = [int(x) for x in torch.randint(1, n_max, (B,), generator=g)]
        lists[k + "_a"] = [torch.randint(0, P, (m,), generator=g) for m in n]
        lists[k + "_b"] = [torch.randint(0, P, (m,), generator=g) for m in n]
    idx, num_valid = {}, {}
    for k in ("matches", "masked", "background", "blind"):
        idx[k + "_a"], num_valid[k] = loss_composer.pad_index_lists(lists[k + "_a"], device=DEV)
        idx[k + "_b"], _ = loss_composer.pad_index_lists(lists[k + "_b"], device=DEV)
    cfg = dict(LO.DEFAULT_LOSS_CONFIG, M_masked=1.5, M_background=1.2)

    def run(pa, pb):
        pcl = pdc_b200.PixelwiseContrastiveLoss([H, W], dict(cfg))
        return loss_composer.get_loss(pcl, torch.zeros(B, dtype=torch.int64), pa, pb, *[idx[k] for k in IDX_KEYS],
                                      num_valid=num_valid)
    both_routes(B, D, H, W, run)


def _training_config():
    return {"training": dict(num_matching_attempts=40, num_non_matches_per_match=4, fraction_masked_non_matches=0.5,
                             fraction_background_non_matches=0.5, sample_matches_only_off_mask=True, domain_randomize=True,
                             use_image_b_mask_inv=True, cross_scene_num_samples=100)}


def _plane_pairs(B, H, W, seed):
    x, K = synthetic.plane_scene_pairs(B, H, W, seed)
    return {k: v.to(DEV) if isinstance(v, torch.Tensor) else v for k, v in x.items()}, K


def test_batch8_mixed_pair_types():
    H, W, D = 64, 96, 4
    tc = _training_config()
    x, K = _plane_pairs(5, H, W, 61)
    within = S.within_scene_batch(x["rgb_a"], x["rgb_b"], x["depth_a"], x["depth_b"], x["mask_a"], x["mask_b"], x["pose_a"],
                                  x["pose_b"], K, tc, generator=torch.Generator(device=DEV).manual_seed(61))
    y, _ = _plane_pairs(3, H, W, 62)
    across = S.across_scene_batch(y["rgb_a"], y["rgb_b"], y["mask_a"], y["mask_b"], tc,
                                  generator=torch.Generator(device=DEV).manual_seed(62))
    batch = S.concat_batches([within, across])
    B = len(batch["match_type"])
    assert B == 8 and (batch["match_type"] == T.DIFFERENT_OBJECT).sum() == 3
    cfg = dict(LO.DEFAULT_LOSS_CONFIG, M_masked=1.5, M_background=1.2)

    def run(pa, pb):
        pcl = pdc_b200.PixelwiseContrastiveLoss([H, W], dict(cfg))
        return loss_composer.get_mixed_loss(pcl, batch["match_type"], pa, pb, *[batch[k] for k in BATCH_KEYS],
                                            num_valid=batch["num_valid"])
    f = both_routes(B, D, H, W, run)
    assert f[4] > 0


# ----------------------------------------------------------------------------------------------- full-resolution cotangent
def test_standalone_unit_upsample_and_zero_descriptor():
    N_, D, h, w, H, W = 3, 5, 8, 12, 64, 96
    g = torch.Generator().manual_seed(4)
    low = torch.randn(N_, D, h, w, generator=g, dtype=torch.float64)
    low[1, :, 0, 0] = 0.0                                  # output pixel (0, 0) of image 1 blends only this cell: NaN
    x = low.float().to(DEV).contiguous()
    y = torch.empty(N_, D, H, W, device=DEV)
    N.check(N.lib.ddn_upsample_bilinear_unit_forward(N.ptr(x), N.ptr(y), N_, D, h, w, H, W, N.stream_ptr()))
    ref = UO.unit_upsample(low.float().double(), H, W)
    yc = y.double().cpu()
    assert bool(torch.isnan(yc[1, :, 0, 0]).all())
    finite = torch.ones(N_, H, W, dtype=torch.bool)
    finite[1, 0, 0] = False
    assert bool(torch.isfinite(yc.permute(0, 2, 3, 1)[finite]).all())
    ok = ((yc - ref).abs() <= unit_bound(low.float().double(), H, W)).permute(0, 2, 3, 1)[finite]
    assert bool(ok.all())
    # adjoint vs float64 autograd (image 1's zero cell left out: its gradient is NaN in both)
    low[1, :, 0, 0] = 0.5
    x = low.float().to(DEV).contiguous()
    dy = torch.randn(N_, D, H, W, generator=g).to(DEV)
    dx = torch.empty_like(x)
    scratch = torch.empty(N_ * D * H * W, device=DEV)
    N.check(N.lib.ddn_upsample_bilinear_unit_backward(N.ptr(x), N.ptr(dy), N.ptr(dx), N.ptr(scratch), N_, D, h, w, H, W,
                                                      N.stream_ptr()))
    l64 = low.float().double().requires_grad_()
    UO.unit_upsample(l64, H, W).backward(dy.double().cpu())
    assert rel(dx, l64.grad) < 1e-6


@pytest.mark.parametrize("backbone", ["Resnet34_8s", "Resnet50_8s"])
def test_triplet_loss_cotangent_through_the_normalisation(backbone):
    D, B, H, W = 3, 2, 64, 96
    data = synthetic.make_pair_batch(B, H, W, 40, 120, 120, 0, seed=17)
    d = {k: (v.to(DEV) if v is not None else None) for k, v in data.items()}
    grads = []
    for kernel in (True, False):
        dcn = network(D, H, W, backbone)
        dcn.train()
        if kernel:
            ya, yb = dcn.forward_pair(d["img_a"], d["img_b"], per_pixel_normalize=True)
        else:
            raw = dcn.fcn(torch.cat([d["img_a"], d["img_b"]], 0), bn_groups=2)
            y = raw / raw.norm(dim=1, keepdim=True)
            ya, yb = y[:B], y[B:]
        pa, pb = dcn.process_network_output(ya, B), dcn.process_network_output(yb, B)
        pcl = pdc_b200.PixelwiseContrastiveLoss(dcn.image_shape, dict(LO.DEFAULT_LOSS_CONFIG))
        loss = sum(pcl.get_triplet_loss(pa[i:i + 1], pb[i:i + 1], d["matches_a"][i], d["matches_b"][i], d["masked_a"][i],
                                        d["masked_b"][i], 0.1) for i in range(B))
        loss.backward()
        grads.append({k: p.grad.detach().clone() for k, p in dcn.fcn.named_parameters()})
    for k in grads[1]:
        assert rel(grads[0][k], grads[1][k]) < 1e-4, k


# ------------------------------------------------------------------------------------------------- parameter gradients
# The machinery of tests/test_gpu_training_size_gradients.py: decisive BatchNorm biases (amp 5), scale_by_hard_negatives off
# (continuous in the descriptors), and each bf16x3 tensor gated at the larger of 1e-3 and 4x its noise floor -- the distance
# from float64 of the same float64 oracle with every ReLU input perturbed by a relative 1e-5 (the larger of two draws).
# STEM_PARAMS sit behind the max-pool's ties: 2e-2.  Both BatchNorm groups (A, B) are normalised separately, as forward_pair does.
AMP, NOISE_EPS, NOISE_SEEDS, FLOOR_FACTOR, GATE = 5.0, 1e-5, (1, 2), 4.0, 1e-3


def _float64_reference(mod, state, D, d, cfg, H, W, noise=None):
    o = mod.seeded_oracle(D=D, seed=0).to(DEV, torch.float64)
    o.load_state_dict(state)
    o.train()
    handles = R34.perturbed_relus(o, *noise) if noise is not None else []
    B = d["img_a"].shape[0]
    ya, yb = o(d["img_a"].double()), o(d["img_b"].double())
    ya, yb = ya / ya.norm(dim=1, keepdim=True), yb / yb.norm(dim=1, keepdim=True)
    pcl = LO.TorchPixelwiseContrastiveLoss([H, W], dict(cfg))
    five = LO.batched_within_scene_loss(pcl, R34.process_network_output(ya, B, D, H, W),
                                        R34.process_network_output(yb, B, D, H, W), d)
    names = [k for k, _ in o.named_parameters()]
    gr = torch.autograd.grad(five[0], [p for _, p in o.named_parameters()])
    out = {k: v.cpu() for k, v in zip(names, gr)}, [float(t) for t in five]
    for h in handles:
        h.remove()
    del o, gr, ya, yb, five
    torch.cuda.empty_cache()
    return out


@pytest.mark.parametrize("backbone,H,W,B", [("Resnet34_8s", 64, 96, 2), ("Resnet50_8s", 64, 96, 2),
                                            ("Resnet34_8s", 480, 640, 2)])
def test_parameter_gradients_through_the_normalisation_vs_float64(backbone, H, W, B):
    D = 3
    mod = R34 if backbone == "Resnet34_8s" else R50
    state = mod.decisive_biases(mod.seeded_oracle(D=D, seed=0), amp=AMP).state_dict()
    data = synthetic.make_pair_batch(B, H, W, 200, 600, 600, 0, seed=23)
    d = {k: (v.to(DEV) if v is not None else None) for k, v in data.items()}
    cfg = dict(LO.DEFAULT_LOSS_CONFIG, scale_by_hard_negatives=False, M_masked=1.5, M_background=1.2)
    g64, f64 = _float64_reference(mod, state, D, d, cfg, H, W)
    noisy = [_float64_reference(mod, state, D, d, cfg, H, W, noise=(NOISE_EPS, s))[0] for s in NOISE_SEEDS]
    floor = {k: max(rel(n[k], g64[k]) for n in noisy) for k in g64}
    dcn = network(D, H, W, backbone)
    dcn.fcn.load_state_dict(state)
    dcn.train()
    ya, yb = dcn.forward_pair(d["img_a"], d["img_b"], per_pixel_normalize=True)
    pa, pb = dcn.process_network_output(ya, B), dcn.process_network_output(yb, B)
    assert loss_composer._fused_lowres(pa, pb, W)[3] is True          # the fused unit loss is under test
    pcl = pdc_b200.PixelwiseContrastiveLoss(dcn.image_shape, dict(cfg))
    blind = loss_composer.empty_tensor().to(DEV)
    five = loss_composer.get_loss(pcl, torch.zeros(B, dtype=torch.int64), pa, pb, d["matches_a"], d["matches_b"],
                                  d["masked_a"], d["masked_b"], d["background_a"], d["background_b"], blind, blind)
    five[0].backward()
    got_five = [float(t) for t in five]
    for a, r in zip(got_five, f64):
        assert abs(a - r) <= 1e-4 * max(1.0, abs(r)), (got_five, f64)
    scale = max(float(v.double().norm()) for v in g64.values())
    worst = 0.0
    for k, p in dcn.fcn.named_parameters():
        r = g64[k]
        if float(r.double().norm()) < 1e-6 * scale:
            assert float(p.grad.double().norm()) < 1e-4 * scale, k
            continue
        e = rel(p.grad, r)
        gate = 2e-2 if k in mod.STEM_PARAMS else max(GATE, FLOOR_FACTOR * floor[k])
        assert e < gate, "%s: rel err %.3e (gate %.1e, noise floor %.1e)" % (k, e, gate, floor[k])
        if k not in mod.STEM_PARAMS:
            worst = max(worst, e)
    print("unit-descriptor parameter gradients [%s %dx%d B=%d]: worst non-stem rel err %.2e" % (backbone, W, H, B, worst))


# ------------------------------------------------------------------------------------------------ sync, launches, repeat
def test_fused_unit_step_no_sync_launches_independent_of_B_and_repeatable():
    D, H, W = 3, 64, 96
    launches = []
    for B in (1, 8):
        dcn = network(D, H, W)
        dcn.train()
        data = synthetic.make_pair_batch(B, H, W, 40, 120, 120, 20, seed=29)
        d = {k: (v.to(DEV) if v is not None else None) for k, v in data.items()}
        pcl = pdc_b200.PixelwiseContrastiveLoss(dcn.image_shape, dict(LO.DEFAULT_LOSS_CONFIG, M_masked=1.5))
        state = {k: v.clone() for k, v in dcn.fcn.state_dict().items()}
        runs = []
        for rep in range(3):                  # rep 0 warms up (first-call uploads); reps 1 and 2 are checked
            dcn.fcn.load_state_dict(state)
            dcn.zero_grad(set_to_none=True)
            torch.cuda.synchronize()
            n0 = N.launch_count()
            torch.cuda.set_sync_debug_mode("error" if rep else "default")
            try:
                ya, yb = dcn.forward_pair(d["img_a"], d["img_b"], per_pixel_normalize=True)
                pa, pb = dcn.process_network_output(ya, B), dcn.process_network_output(yb, B)
                five = loss_composer.get_within_scene_loss(pcl, pa, pb, *[d[k] for k in IDX_KEYS])
                five[0].backward()
            finally:
                torch.cuda.set_sync_debug_mode("default")
            if rep == 0:
                continue
            if rep == 1:
                launches.append(N.launch_count() - n0)
            runs.append(([t.detach().clone() for t in five], ya.detach().clone(),
                         {k: p.grad.detach().clone() for k, p in dcn.fcn.named_parameters()}))
        (f0, y0, g0), (f1, y1, g1) = runs
        assert float(f0[0]) > 0
        assert all(torch.equal(a, b) for a, b in zip(f0, f1)) and torch.equal(y0, y1)
        assert all(torch.equal(g0[k], g1[k]) for k in g0)
    assert launches[0] == launches[1], launches
