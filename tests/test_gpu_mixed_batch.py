"""GPU: batches whose pairs have different SpartanDatasetDataType values (sampling.concat_batches over the three producers,
loss_composer.get_mixed_loss through ddn_pair_type_compose).

* get_mixed_loss equals the mean over pairs of the reference's get_loss evaluated per pair at batch 1 on the unpadded
  lists, for batches mixing within-scene, MULTI_OBJECT, synthetic and DIFFERENT_OBJECT pairs with an empty pair of each
  type, under both scale_by_hard_negatives* flags, both l2-pixel flags and M_masked != M_background (the blind list is
  scored at M_masked for within-scene pairs and at M_background for different-object pairs), on the full-resolution and
  the low-resolution route: five values within 2e-6 relative, gradients within 1e-5 relative;
* a batch of one type gives what get_loss gives, with equal and with different margins (bit-identical five values for the
  within-scene types on one route);
* concat_batches copies every row bit for bit, pads with -1 and refuses a match_type that left the host; no host
  synchronisation, launches independent of B;
* one training step at 640 x 480 on the shoes mix (3 within-scene, 3 different-object, 2 synthetic)."""
import pytest
import torch
import torch.nn.functional as F

import pdc_b200
from pdc_b200 import _native as N
from pdc_b200 import loss_composer
from pdc_b200 import ops
from pdc_b200 import resnet_dilated
from pdc_b200 import sampling as S
from pdc_b200 import synthetic
from pdc_b200.loss_composer import SpartanDatasetDataType as T
from oracle import loss_oracle as LO
from oracle.resnet34_8s_oracle import process_network_output

pytestmark = pytest.mark.gpu
DEV = "cuda"
KEYS = [k % s for k in ("matches_%s", "masked_non_matches_%s", "background_non_matches_%s", "blind_non_matches_%s")
        for s in "ab"]
COLUMN = {k: i // 2 for i, k in enumerate(KEYS)}          # the counts column of each index key
WITHIN = (T.SINGLE_OBJECT_WITHIN_SCENE, T.MULTI_OBJECT, T.SYNTHETIC_MULTI_OBJECT)


def training_config(n_attempts=40, non_matches=4, samples=100):
    return {"training": dict(num_matching_attempts=n_attempts, num_non_matches_per_match=non_matches,
                             fraction_masked_non_matches=0.5, fraction_background_non_matches=0.5,
                             sample_matches_only_off_mask=True, domain_randomize=True, use_image_b_mask_inv=True,
                             cross_scene_num_samples=samples)}


DEFAULT = training_config(10000, 150, 10000)


def plane_pairs(B, H, W, seed, empty=()):
    """pdc_b200.synthetic.plane_scene_pairs with the image tensors on the device."""
    x, K = synthetic.plane_scene_pairs(B, H, W, seed, empty)
    return {k: v.to(DEV) if isinstance(v, torch.Tensor) else v for k, v in x.items()}, K


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def within_part(B, H, W, tc, seed, empty=(), match_type=None):
    x, K = plane_pairs(B, H, W, seed, empty)
    out = S.within_scene_batch(x["rgb_a"], x["rgb_b"], x["depth_a"], x["depth_b"], x["mask_a"], x["mask_b"], x["pose_a"],
                               x["pose_b"], K, tc, generator=gen(seed))
    if match_type is not None:
        out["match_type"] = torch.full_like(out["match_type"], match_type)
    return out


def across_part(B, H, W, tc, seed, empty=()):
    x, _ = plane_pairs(B, H, W, seed, empty)
    return S.across_scene_batch(x["rgb_a"], x["rgb_b"], x["mask_a"], x["mask_b"], tc, generator=gen(seed))


def synthetic_part(B, H, W, tc, seed, empty=()):
    (a, K), (b, _) = plane_pairs(B, H, W, seed, empty), plane_pairs(B, H, W, seed + 1)
    tup = lambda x: (x["rgb_a"], x["rgb_b"], x["depth_a"], x["depth_b"], x["mask_a"], x["mask_b"], x["pose_a"], x["pose_b"])
    return S.synthetic_multi_object_batch(tup(a), tup(b), K, tc, generator=gen(seed))


def mixed_parts(H, W, tc, seed=0):
    """Within-scene 3, MULTI_OBJECT 2, DIFFERENT_OBJECT 3, synthetic 3, the first pair of every part empty."""
    return [within_part(3, H, W, tc, seed + 1, empty=(0,)),
            within_part(2, H, W, tc, seed + 2, empty=(0,), match_type=T.MULTI_OBJECT),
            across_part(3, H, W, tc, seed + 3, empty=(0,)),
            synthetic_part(3, H, W, tc, seed + 4, empty=(0,))]


def rel(x, y):
    return float((x.detach().cpu() - y).norm() / max(float(y.norm()), 1e-30))


class Descriptors(object):
    """Random descriptor images for the device loss and the same values for the CPU reference.  route "full": [B, D, H, W]
    images; route "lowres": [B, h*w, D] low-resolution maps, the device images are their bilinear upsample tagged with the
    map (the loss runs through the upsample), the reference upsamples them with F.interpolate(align_corners=True)."""

    def __init__(self, route, B, D, H, W, seed=2):
        self.route, self.B, self.D, self.H, self.W = route, B, D, H, W
        g = torch.Generator().manual_seed(seed)
        shape = (B, D, H, W) if route == "full" else (B, (H // 8) * (W // 8), D)
        self.x = [0.3 * torch.randn(*shape, generator=g) for _ in range(2)]

    def _nchw(self, t):
        return t.view(self.B, self.H // 8, self.W // 8, self.D).permute(0, 3, 1, 2).contiguous()

    def device(self):
        B, D, H, W = self.B, self.D, self.H, self.W
        self.leaves = [t.to(DEV).requires_grad_() for t in self.x]
        if self.route == "full":
            return [process_network_output(t, B, D, H, W) for t in self.leaves]
        preds = []
        for t in self.leaves:
            y = ops.upsample_bilinear_forward(self._nchw(t.detach()), H, W)
            p = y.view(B, D, H * W).permute(0, 2, 1)
            resnet_dilated.attach_lowres(p, t, H, W)
            preds.append(p)
        return preds

    def reference(self):
        B, D, H, W = self.B, self.D, self.H, self.W
        self.ref_leaves = [t.clone().requires_grad_() for t in self.x]
        if self.route == "full":
            return [process_network_output(t, B, D, H, W) for t in self.ref_leaves]
        return [process_network_output(F.interpolate(self._nchw(t), size=(H, W), mode="bilinear", align_corners=True),
                                       B, D, H, W) for t in self.ref_leaves]


def reference_five(batch, pa, pb, lc, H, W):
    """Mean over the pairs of the reference's get_loss at batch 1 on the unpadded lists; an empty pair adds 0."""
    B = len(batch["match_type"])
    ref = LO.TorchPixelwiseContrastiveLoss([H, W], dict(lc))
    terms = [torch.zeros(()) for _ in range(5)]
    for b in range(B):
        t = int(batch["match_type"][b])
        c = batch["counts"][b].cpu().tolist()
        lists = {k: batch[k][b, :c[COLUMN[k]]].cpu() for k in KEYS}
        if t == T.DIFFERENT_OBJECT:
            if c[3] == 0:
                continue
            o = LO.get_loss(ref, torch.tensor([t]), pa[b:b + 1], pb[b:b + 1], *([None] * 6),
                            lists["blind_non_matches_a"], lists["blind_non_matches_b"])
        else:
            if c[0] == 0:
                assert sum(c) == 0, (b, c)        # only the producers' empty pairs have no matches
                continue
            if c[3] == 0:
                lists["blind_non_matches_a"] = lists["blind_non_matches_b"] = LO.empty_tensor()
            o = LO.get_loss(ref, torch.tensor([t]), pa[b:b + 1], pb[b:b + 1], *[lists[k] for k in KEYS])
        terms = [s + o[i].reshape(()) for i, s in enumerate(terms)]
    return [s / B for s in terms]


def assert_five_close(five, five_r):
    for i in range(5):
        a, r = float(five[i]), float(five_r[i])
        assert abs(a - r) <= 2e-6 * max(1.0, abs(r)), (i, a, r)


# M_masked != M_background in two entries: within-scene pairs score the blind list at M_masked, different-object pairs at
# M_background (the reference's multi-object configurations use M_background 1.0 or 2.0 with M_masked 0.5), and the
# masked and background hinges are told apart
FLAGS = [dict(scale_by_hard_negatives=True, scale_by_hard_negatives_DIFFERENT_OBJECT=True, M_masked=0.5, M_background=2.0),
         dict(scale_by_hard_negatives=False, scale_by_hard_negatives_DIFFERENT_OBJECT=False,
              use_l2_pixel_loss_on_masked_non_matches=True, use_l2_pixel_loss_on_background_non_matches=True, M_pixel=9),
         dict(scale_by_hard_negatives=True, scale_by_hard_negatives_DIFFERENT_OBJECT=False,
              use_l2_pixel_loss_on_masked_non_matches=True, M_pixel=9),
         dict(scale_by_hard_negatives=False, scale_by_hard_negatives_DIFFERENT_OBJECT=True,
              use_l2_pixel_loss_on_background_non_matches=True, M_pixel=9, M_masked=1.2, M_background=0.4)]


@pytest.fixture(scope="module")
def mixed_batch():
    H, W = 24, 32
    batch = S.concat_batches(mixed_parts(H, W, training_config()))
    mt, counts = batch["match_type"].tolist(), batch["counts"].cpu()
    for typ in (T.SINGLE_OBJECT_WITHIN_SCENE, T.MULTI_OBJECT, T.DIFFERENT_OBJECT, T.SYNTHETIC_MULTI_OBJECT):
        rows = [b for b in range(len(mt)) if mt[b] == typ]
        assert any(int(counts[b].sum()) == 0 for b in rows), typ          # an empty pair of every type
        assert any(int(counts[b].sum()) > 0 for b in rows), typ
    return H, W, batch


@pytest.mark.parametrize("route", ["full", "lowres"])
@pytest.mark.parametrize("flags", range(len(FLAGS)))
def test_mixed_loss_equals_per_pair_reference(mixed_batch, route, flags):
    H, W, batch = mixed_batch
    B, D = len(batch["match_type"]), 3
    lc = dict(LO.DEFAULT_LOSS_CONFIG, **FLAGS[flags])
    desc = Descriptors(route, B, D, H, W)
    pa, pb = desc.device()
    pcl = pdc_b200.PixelwiseContrastiveLoss([H, W], dict(lc))
    pcl.debug = True
    five = loss_composer.get_mixed_loss(pcl, batch["match_type"], pa, pb, *[batch[k] for k in KEYS],
                                        num_valid=batch["num_valid"])
    five[0].backward()
    par, pbr = desc.reference()
    five_r = reference_five(batch, par, pbr, lc, H, W)
    assert float(five_r[0]) > 0 and float(five_r[4]) > 0
    five_r[0].backward()
    assert_five_close(five, five_r)
    for g, r in zip(desc.leaves, desc.ref_leaves):
        assert rel(g.grad, r.grad) < 1e-5
    # the blind list is routed by type: term 3 only counts within-scene pairs, term 4 only different-object pairs
    counts = pcl.debug_data["num_hard_negatives_device"].cpu()
    different = batch["match_type"] == T.DIFFERENT_OBJECT
    assert counts.shape == (B, 5)
    assert int(counts[different, :4].abs().sum()) == 0 and int(counts[~different, 4].abs().sum()) == 0
    assert int(counts[different, 4].sum()) > 0


@pytest.mark.parametrize("margins", [(0.5, 0.5), (0.5, 2.0)], ids=["equal_margins", "M_background_2"])
# get_loss scores DIFFERENT_OBJECT from the full-resolution images only, so that type is compared on that route
@pytest.mark.parametrize("route,typ", [(r, t) for r in ("full", "lowres") for t in WITHIN] + [("full", T.DIFFERENT_OBJECT)])
def test_uniform_batch_equals_get_loss(route, typ, margins):
    H, W, D = 24, 32, 3
    tc = training_config()
    if typ == T.DIFFERENT_OBJECT:
        batch = across_part(4, H, W, tc, 31, empty=(1,))
    elif typ == T.SYNTHETIC_MULTI_OBJECT:
        batch = synthetic_part(4, H, W, tc, 31, empty=(1,))
    else:
        batch = within_part(4, H, W, tc, 31, empty=(1,), match_type=typ)
    B = 4
    lc = dict(LO.DEFAULT_LOSS_CONFIG, M_masked=margins[0], M_background=margins[1])
    res = []
    for fn in (loss_composer.get_loss, loss_composer.get_mixed_loss):
        desc = Descriptors(route, B, D, H, W)
        pa, pb = desc.device()
        five = fn(pdc_b200.PixelwiseContrastiveLoss([H, W], dict(lc)), batch["match_type"], pa, pb,
                  *[batch[k] for k in KEYS], num_valid=batch["num_valid"])
        five[0].backward()
        res.append(([f.detach().clone() for f in five], [t.grad for t in desc.leaves]))
    (f0, g0), (f1, g1) = res
    assert float(f0[0]) > 0
    if typ in WITHIN:
        # same sums, same arithmetic: the pair-type compose reproduces the within-scene compose bit for bit
        assert all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(f0, f1)), (f0, f1)
    else:
        assert_five_close(f1, f0)
    for a, b in zip(g1, g0):
        assert rel(a, b.cpu()) < 1e-5


def test_concat_batches_rows_padding_and_counts():
    H, W = 24, 32
    parts = mixed_parts(H, W, training_config(), seed=10)
    batch = S.concat_batches(parts)
    B = sum(len(p["match_type"]) for p in parts)
    assert batch["image_a"].shape == (B, 3, H, W) and batch["counts"].shape == (B, 4)
    assert batch["match_type"].device.type == "cpu" and batch["match_type"].dtype == torch.int64
    r = 0
    for p in parts:
        n = len(p["match_type"])
        for k in ("image_a", "image_b"):
            assert torch.equal(batch[k][r:r + n].view(torch.int32), p[k].view(torch.int32)), k
        for k in KEYS:
            w = p[k].shape[1]
            assert batch[k].shape[1] == max(q[k].shape[1] for q in parts), k
            assert torch.equal(batch[k][r:r + n, :w], p[k]), k
            assert bool((batch[k][r:r + n, w:] == -1).all()), k
        assert torch.equal(batch["counts"][r:r + n], p["counts"]) and torch.equal(batch["empty"][r:r + n], p["empty"])
        assert batch["match_type"][r:r + n].tolist() == p["match_type"].tolist()
        r += n
    for i, k in enumerate(("matches", "masked", "background", "blind")):
        assert torch.equal(batch["num_valid"][k], batch["counts"][:, i]), k
    # a part relabelled with a CUDA match_type is refused with a clear error (get_mixed_loss reads the types on the host)
    parts[1]["match_type"] = parts[1]["match_type"].to(DEV)
    with pytest.raises(ValueError, match="match_type of part 1 is on cuda"):
        S.concat_batches(parts)
    # every row's entries past its count are -1
    for k in KEYS:
        col = torch.arange(batch[k].shape[1], device=DEV)[None, :]
        assert bool((batch[k][col >= batch["counts"][:, COLUMN[k]][:, None]] == -1).all()), k


def test_no_sync_and_launches_independent_of_B():
    H, W, D = 24, 32, 3
    tc = training_config()
    launches = []
    for n_within, n_different in ((1, 1), (5, 3)):
        parts = [within_part(n_within, H, W, tc, 41), across_part(n_different, H, W, tc, 42)]
        B = n_within + n_different
        desc = Descriptors("full", B, D, H, W)
        pa, pb = desc.device()
        pcl = pdc_b200.PixelwiseContrastiveLoss([H, W], dict(LO.DEFAULT_LOSS_CONFIG))
        torch.cuda.synchronize()
        n0 = N.launch_count()
        torch.cuda.set_sync_debug_mode("error")
        try:
            batch = S.concat_batches(parts)
            five = loss_composer.get_mixed_loss(pcl, batch["match_type"], pa, pb, *[batch[k] for k in KEYS],
                                                num_valid=batch["num_valid"])
            five[0].backward()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        launches.append(N.launch_count() - n0)
        assert bool(torch.isfinite(five[0]).all()) and float(five[0]) > 0
    assert launches[0] == launches[1] == 3, launches          # gather, compose, scatter


def test_training_step_shoes_mix_640x480():
    B, H, W, D = 8, 480, 640, 3
    parts = [within_part(3, H, W, DEFAULT, 51), across_part(3, H, W, DEFAULT, 52), synthetic_part(2, H, W, DEFAULT, 53)]
    batch = S.concat_batches(parts)
    assert batch["match_type"].tolist() == [T.SINGLE_OBJECT_WITHIN_SCENE] * 3 + [T.DIFFERENT_OBJECT] * 3 + \
        [T.SYNTHETIC_MULTI_OBJECT] * 2
    dcn = pdc_b200.DenseCorrespondenceNetwork.from_config({"descriptor_dimension": D, "image_width": W, "image_height": H},
                                                          load_stored_params=False)
    pcl = pdc_b200.PixelwiseContrastiveLoss(dcn.image_shape, dict(pdc_b200.DEFAULT_LOSS_CONFIG))
    a, b = dcn.forward_pair(batch["image_a"], batch["image_b"])
    five = loss_composer.get_mixed_loss(pcl, batch["match_type"], dcn.process_network_output(a, B),
                                        dcn.process_network_output(b, B), *[batch[k] for k in KEYS],
                                        num_valid=batch["num_valid"])
    five[0].backward()
    assert bool(torch.isfinite(five[0]).all()) and float(five[0]) > 0
    assert all(bool(torch.isfinite(f).all()) for f in five)
    grads = [p.grad for p in dcn.parameters() if p.grad is not None]
    assert grads and all(bool(torch.isfinite(g).all()) for g in grads)
    assert any(float(g.abs().max()) > 0 for g in grads)
