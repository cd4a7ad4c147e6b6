"""GPU: descriptor statistics (csrc/descriptor_stats.cu) and the batched across-object best match (csrc/match_stats.cu)
via pdc_b200.evaluation, against float64, the executed reference's fixture (tests/golden/descriptor_statistics.npz) and
find_best_matches_cuda.

Gates: min / max and counts exact; means within 1e-6 relative of float64; best-match pixels exact and distances bit-equal
to numpy's float32 arithmetic; strided input, contiguous input and a second run bit-identical."""
import os

import numpy as np
import pytest
import torch

import pdc_b200
from pdc_b200 import _native as N
from pdc_b200 import evaluation as E
from oracle import descriptor_stats_oracle as DO

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "descriptor_statistics.npz")


def _images(n, H, W, D, seed, empty=()):
    g = torch.Generator(device=DEV).manual_seed(seed)
    res = torch.randn(n, D, H, W, device=DEV, generator=g) * 2.0 + torch.linspace(-1, 1, D, device=DEV)[None, :, None, None]
    mask = (torch.rand(n, H, W, device=DEV, generator=g) < 0.3).to(torch.float32)
    for i in empty:
        mask[i] = 0
    return res, mask          # res NCHW, as the network returns it


def _check_f64(out, res_nhwc, mask):
    """-> worst relative mean error; min / max / counts asserted exact against torch / float64."""
    n, D = res_nhwc.shape[0], res_nhwc.shape[-1]
    flat = res_nhwc.reshape(n, -1, D)
    sel = mask.reshape(n, -1) != 0
    assert torch.equal(out["mask_count"], sel.sum(1))
    assert torch.equal(out["min"], flat.min(1)[0]) and torch.equal(out["max"], flat.max(1)[0])
    worst = (out["mean"].double() - flat.double().mean(1)).abs().div(flat.double().mean(1).abs()).max().item()
    for i in range(n):
        if not sel[i].any():
            assert torch.isnan(out["mask_min"][i]).all() and torch.isnan(out["mask_mean"][i]).all()
            continue
        m = flat[i][sel[i]]
        assert torch.equal(out["mask_min"][i], m.min(0)[0]) and torch.equal(out["mask_max"][i], m.max(0)[0])
        e = ((out["mask_mean"][i].double() - m.double().mean(0)).abs() / m.double().mean(0).abs()).max().item()
        worst = max(worst, e)
    return worst


@pytest.mark.parametrize("D", [3, 16])
@pytest.mark.parametrize("mask_dtype", [torch.float32, torch.uint8, torch.bool])
def test_statistics_against_float64_small(D, mask_dtype):
    res, mask = _images(5, 64, 96, D, seed=D, empty=(2,))
    x = res.permute(0, 2, 3, 1)
    out = E.descriptor_statistics(x, mask.to(mask_dtype))
    assert _check_f64(out, x, mask) <= 1e-6
    assert int(out["mask_count"][2]) == 0


def test_statistics_against_float64_full_size():
    res, mask = _images(100, 480, 640, 3, seed=11, empty=(7,))
    x = res.permute(0, 2, 3, 1)
    assert _check_f64(E.descriptor_statistics(x, mask), x, mask) <= 1e-6


@pytest.mark.parametrize("D", [3, 16, 32])
def test_strided_contiguous_and_repeated_runs_are_identical(D):
    res, mask = _images(4, 37, 53, D, seed=100 + D, empty=(1,))
    a = E.descriptor_statistics(res.permute(0, 2, 3, 1), mask)                    # NCHW storage, [N,H,W,D] view
    b = E.descriptor_statistics(res.permute(0, 2, 3, 1).contiguous(), mask)       # NHWC storage
    c = E.descriptor_statistics(res.permute(0, 2, 3, 1), mask)
    for k in a:
        assert torch.equal(a[k].view(torch.int32) if a[k].is_floating_point() else a[k],
                           b[k].view(torch.int32) if b[k].is_floating_point() else b[k]), k
        assert torch.equal(a[k].view(torch.int32) if a[k].is_floating_point() else a[k],
                           c[k].view(torch.int32) if c[k].is_floating_point() else c[k]), k
    # one image as forward_single_image_tensor returns it ([H,W,D] permuted view)
    one = E.descriptor_statistics(res[3].permute(1, 2, 0), mask[3])
    for k in a:
        assert torch.equal(one[k][0], a[k][3]), k
    # a column crop: rows are not W pixels apart, the general addressing
    crop = res.permute(0, 2, 3, 1)[:, :, 2:-3]
    m = mask[:, :, 2:-3].contiguous()
    d = E.descriptor_statistics(crop, m)
    e = E.descriptor_statistics(crop.contiguous(), m)
    for k in d:
        assert torch.equal(d[k], e[k]) or (d[k].is_floating_point() and torch.equal(d[k].view(torch.int32), e[k].view(torch.int32))), k
    assert _check_f64(d, crop, m) <= 1e-6


def test_all_empty_masks():
    res, mask = _images(3, 16, 24, 4, seed=5, empty=(0, 1, 2))
    out = E.descriptor_statistics(res.permute(0, 2, 3, 1), mask)
    assert (out["mask_count"] == 0).all()
    for k in ("mask_min", "mask_max", "mask_mean"):
        assert torch.isnan(out[k]).all()
    assert not torch.isnan(out["mean"]).any()
    with pytest.raises(TypeError):
        E.fold_descriptor_statistics(out)


@pytest.mark.parametrize("D", [3, 16])
def test_fixture_statistics(D):
    g = np.load(GOLDEN)
    res = torch.from_numpy(g["res_d%d" % D]).to(DEV)
    stats = E.fold_descriptor_statistics(E.descriptor_statistics(res, torch.from_numpy(g["mask_d%d" % D]).to(DEV)))
    for key in ("entire_image", "mask_image"):
        for f in ("min", "max"):
            assert np.array_equal(stats[key][f], g["stats_d%d/%s/%s" % (D, key, f)]), (key, f)
        np.testing.assert_allclose(stats[key]["mean"], g["stats_d%d/%s/mean" % (D, key)], rtol=1e-6, atol=1e-7)


def test_statistics_refusals_launch_nothing():
    res, mask = _images(2, 8, 12, 3, seed=1)
    x = res.permute(0, 2, 3, 1)
    before = N.launch_count()
    for args in ((x, mask[:1]), (x, mask[:, :7]), (x, mask.double()), (x.double(), mask), (x.cpu(), mask),
                 (torch.zeros(2, 8, 12, 33, device=DEV), mask), (torch.zeros(2, 8, 12, 0, device=DEV), mask)):
        with pytest.raises(RuntimeError):
            E.descriptor_statistics(*args)
    assert N.launch_count() == before


@pytest.mark.parametrize("D", [3, 16])
def test_best_match_batch_equals_fixture(D):
    g = np.load(GOLDEN)
    ra = torch.from_numpy(g["bm_res_a_d%d" % D]).to(DEV); rb = torch.from_numpy(g["bm_res_b_d%d" % D]).to(DEV)
    uv_a = torch.from_numpy(g["bm_uv_a_d%d" % D]).to(DEV)
    # three pairs in one launch: the fixture's, one with B flipped (other answers), the fixture's again in NCHW storage
    res_a = torch.stack([ra, ra, ra]); res_b = torch.stack([rb, rb.flip(0), rb])
    res_b = res_b.permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1)
    Q = uv_a.shape[0]
    pair = torch.arange(3, device=DEV).repeat_interleave(Q)
    uv, diff, bad = E.best_match_batch(res_a, res_b, uv_a.repeat(3, 1), pair)
    assert int(bad) == 0
    for p in (0, 2):
        assert np.array_equal(uv[p * Q:(p + 1) * Q].cpu().numpy(), g["bm_uv_b_d%d" % D])
        assert diff[p * Q:(p + 1) * Q].cpu().numpy().tobytes() == g["bm_diff_d%d" % D].tobytes()
    flipped = rb.flip(0).cpu().numpy()
    for i, u in enumerate(g["bm_uv_a_d%d" % D]):
        uv_o, d_o = DO.best_match(u, g["bm_res_a_d%d" % D], flipped)
        assert tuple(uv[Q + i].tolist()) == uv_o and diff[Q + i].item() == d_o


def test_best_match_batch_bad_queries():
    res, _ = _images(2, 8, 12, 3, seed=2)
    x = res.permute(0, 2, 3, 1)
    uv_a = torch.tensor([[0, 0], [12, 0], [0, 8], [11, 7], [-1, 3]], device=DEV)
    pair = torch.tensor([0, 0, 1, 2, 1], device=DEV)
    uv, diff, bad = E.best_match_batch(x, x, uv_a, pair)
    assert int(bad) == 4
    assert uv[0].tolist() == [0, 0] and diff[0].item() == 0.0          # a pixel's own descriptor
    assert (uv[1:] == -1).all() and torch.isnan(diff[1:]).all()


@pytest.mark.parametrize("D", [3, 16])
def test_best_match_batch_equals_find_best_matches_cuda_per_pair(D):
    """25 pairs x 100 samples at 640x480: pixels equal find_best_matches_cuda's, distances within its FMA rounding;
    a subset bit-equal to numpy's float32 find_best_match."""
    P, M, H, W = 25, 100, 480, 640
    ra, _ = _images(P, H, W, D, seed=30 + D)
    rb, _ = _images(P, H, W, D, seed=60 + D)
    ra = ra.permute(0, 2, 3, 1); rb = rb.permute(0, 2, 3, 1)
    g = torch.Generator(device=DEV).manual_seed(D)
    flat = torch.randint(0, H * W, (P * M,), device=DEV, generator=g)
    uv_a = torch.stack([flat % W, flat // W], 1)
    pair = torch.arange(P, device=DEV).repeat_interleave(M)
    uv, diff, bad = E.best_match_batch(ra, rb, uv_a, pair)
    uv2, diff2, _ = E.best_match_batch(ra, rb, uv_a, pair)
    assert int(bad) == 0 and torch.equal(uv, uv2) and torch.equal(diff.view(torch.int32), diff2.view(torch.int32))
    same = 0
    for p in range(P):
        sl = slice(p * M, (p + 1) * M)
        ref_uv, ref_diff = pdc_b200.DenseCorrespondenceNetwork.find_best_matches_cuda(uv_a[sl], ra[p], rb[p])
        same += int((uv[sl] == ref_uv).all(1).sum())
        torch.testing.assert_close(diff[sl], ref_diff, rtol=2e-6, atol=1e-6)
    assert same >= P * M - 2                     # an FMA-rounded near-tie may pick another pixel
    host_a, host_b = ra[0].cpu().numpy(), rb[0].cpu().numpy()
    for i in range(0, M, 10):
        uv_o, d_o = DO.best_match(uv_a[i].tolist(), host_a, host_b)
        assert tuple(uv[i].tolist()) == uv_o and diff[i].item() == d_o


def test_across_object_analysis():
    P, H, W, D, M = 4, 48, 64, 8, 50
    ra, mask = _images(P, H, W, D, seed=7, empty=(2,))
    rb, _ = _images(P, H, W, D, seed=8)
    ra = ra.permute(0, 2, 3, 1); rb = rb.permute(0, 2, 3, 1)
    meta = [dict(scene_name_a="sa%d" % i, scene_name_b="sb%d" % i, img_a_idx=i, img_b_idx=10 + i, object_id_a="A",
                 object_id_b="B") for i in range(P)]
    gen = torch.Generator(device=DEV).manual_seed(3)
    out = E.across_object_analysis(ra, rb, mask, meta, num_uv_a_samples=M, generator=gen)
    assert list(out["pair"]) == [0] * M + [1] * M + [3] * M               # the empty mask gives no rows
    assert set(E.DCNEvaluationPandaTemplateAcrossObject.columns) <= set(out)
    assert list(out["img_b_idx"][:M]) == [10] * M and out["scene_name_a"][-1] == "sa3"
    m = mask.cpu().numpy(); a = ra.cpu().numpy(); b = rb.cpu().numpy()
    for r in range(0, len(out["pair"]), 7):
        p, (u, v) = out["pair"][r], out["uv_a"][r]
        assert m[p, v, u] != 0
        uv_o, d_o = DO.best_match((u, v), a[p], b[p])
        assert tuple(out["uv_b"][r]) == uv_o and out["norm_diff_descriptor_best_match"][r] == d_o


@pytest.mark.parametrize("D,normalize", [(3, False), (3, True), (8, True)])
def test_over_images_equals_the_per_image_forward(D, normalize):
    """descriptor_statistics_over_images on a small network equals the reference's route: forward_single_image_tensor
    image by image, statistics and fold in float64 (oracle/descriptor_stats_oracle.py).  With normalize=True the
    network's norm only broadcasts per image for a batch of one; D = 8 with 8 images is the case where a batched forward
    would run without an error and normalise the wrong images."""
    n, H, W = 8, 64, 96
    torch.manual_seed(D)
    dcn = pdc_b200.DenseCorrespondenceNetwork.from_config(
        {"descriptor_dimension": D, "image_width": W, "image_height": H, "normalize": normalize}, load_stored_params=False)
    g = torch.Generator().manual_seed(100 + D)
    imgs = torch.randn(n, 3, H, W, generator=g)
    masks = (torch.rand(n, H, W, generator=g) < 0.4).to(torch.uint8)
    masks[5] = 0                                                    # skipped for both keys
    got = E.descriptor_statistics_over_images(dcn, imgs, masks)
    dcn.eval()
    with torch.no_grad():
        per = [DO.per_image(dcn.forward_single_image_tensor(imgs[i]).cpu().numpy(), masks[i].numpy()) for i in range(n)]
    ref = DO.fold(per, n)
    for key in ("entire_image", "mask_image"):
        assert got[key]["min"] == ref[key]["min"] and got[key]["max"] == ref[key]["max"], key
        scale = max(abs(x) for x in ref[key]["max"] + ref[key]["min"])
        np.testing.assert_allclose(got[key]["mean"], ref[key]["mean"], rtol=1e-6, atol=1e-6 * scale)
