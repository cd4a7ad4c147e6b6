"""GPU: pdc_b200.sampling.synthetic_multi_object_batch (csrc/synthetic_multi_object.cu) against the reference's
get_synthetic_multi_object_within_scene_data.

* images: the merged images (or an early return's image twice) equal the executed reference's
  (tests/golden/synthetic_multi_object_batch.npz) through the normalisation table, bit for bit;
* correspondences of each half against the reference's own: survivors equal up to one, matched pixels within one pixel
  (fp32 FFMA against the CPU's matrix products, as tests/test_gpu_within_scene.py);
* everything downstream (merges, prunes, concatenation, non-matches, counts, padding, each early return) equals
  oracle/synthetic_multi_object_oracle.py fed with ddn_find_pixel_correspondences's correspondences half by half, bit for
  bit, on the golden cases, at 640 x 480 with B = 8 and at tiny shapes;
* repeatability, no host synchronisation, launches independent of B, the generator path;
* get_loss(SYNTHETIC_MULTI_OBJECT, num_valid=...) equals the mean of the per-pair reference losses; one training step at
  640 x 480, B = 8."""
import os

import numpy as np
import pytest
import torch

import pdc_b200
from pdc_b200 import _native as N
from pdc_b200 import loss_composer
from pdc_b200 import sampling as S
from oracle import loss_oracle as LO
from oracle import make_golden_synthetic as MG
from oracle import synthetic_multi_object_oracle as SO
from oracle import within_scene_oracle as WO
from oracle.resnet34_8s_oracle import process_network_output

pytestmark = pytest.mark.gpu
DEV = "cuda"
LUT = torch.from_numpy(WO.normalize_lut())
LISTS = (("matches", "matches_a", "matches_b", 0), ("masked_non_matches", "masked_a", "masked_b", 1),
         ("background_non_matches", "background_a", "background_b", 2))
FIELDS = ("rgb_1", "rgb_2", "depth_1", "depth_2", "mask_1", "mask_2", "pose_1", "pose_2")
DEFAULT = {"training": dict(num_matching_attempts=10000, num_non_matches_per_match=150, fraction_masked_non_matches=0.5,
                            fraction_background_non_matches=0.5, sample_matches_only_off_mask=True, domain_randomize=True,
                            use_image_b_mask_inv=True)}


def training_config(cfg):
    return {"training": dict(num_matching_attempts=cfg["n_attempts"], num_non_matches_per_match=1,
                             fraction_masked_non_matches=cfg["k_masked"], fraction_background_non_matches=cfg["k_background"],
                             sample_matches_only_off_mask=cfg["sample_matches_only_off_mask"], domain_randomize=False,
                             use_image_b_mask_inv=cfg["use_image_b_mask_inv"])}


def normalised(rgb_u8):
    x = torch.as_tensor(rgb_u8).long()
    return torch.stack([LUT[c][x[..., c]] for c in range(3)], dim=-3)


def stack(As, Bs, rands):
    def tup(scenes):
        return tuple(np.stack([s[k] for s in scenes]) if k.startswith("pose") else torch.from_numpy(np.stack([s[k] for s in scenes])).to(DEV)
                     for k in FIELDS)
    return tup(As), tup(Bs), {k: torch.from_numpy(np.stack([r[k] for r in rands])).to(DEV) for k in rands[0]}


def device_uv(s, K, cfg, cand_u, cand_v):
    """The half's correspondences as the device finds them (candidates drawn as the device draws them)."""
    H, W = s["mask_1"].shape
    n = cfg["n_attempts"]
    u, v = torch.from_numpy(cand_u[:n].copy()), torch.from_numpy(cand_v[:n].copy())
    nz = torch.nonzero(torch.from_numpy(s["mask_1"]).reshape(-1)).squeeze(1)
    if cfg["sample_matches_only_off_mask"] and len(nz):
        cand = nz[torch.clamp(torch.floor(u * len(nz)).long(), max=len(nz) - 1)]
    else:
        cand = torch.clamp(torch.floor(v * H).long(), max=H - 1) * W + torch.clamp(torch.floor(u * W).long(), max=W - 1)
    a, _, u2, v2 = S.find_pixel_correspondences(torch.from_numpy(s["depth_1"]).to(DEV), s["pose_1"],
                                                torch.from_numpy(s["depth_2"]).to(DEV), s["pose_2"], cand.to(DEV), K)
    a = a.cpu()
    return a % W, a // W, u2.cpu(), v2.cpu()


def check_against_oracle(out, As, Bs, K, cfg, rands):
    for b, (A, Bsc, rand) in enumerate(zip(As, Bs, rands)):
        uv = tuple(device_uv(s, K, cfg, rand["cand_u"][h], rand["cand_v"][h]) for h, s in enumerate((A, Bsc)))
        o = SO.get_synthetic_data(SO.RESTATED, A, Bsc, K, cfg, rand, uv=uv)
        assert bool(out["empty"][b]) == o["empty"], (b, o["ret"])
        for img in ("a", "b"):
            assert torch.equal(out["image_" + img][b].cpu().view(torch.int32), normalised(o["rgb_" + img]).view(torch.int32)), (b, img)
        counts = out["counts"][b].cpu()
        assert int(counts[3]) == 0 and bool((out["blind_non_matches_a"][b] == -1).all())
        for key, ka, kb, c in LISTS:
            n = len(o[ka])
            assert int(counts[c]) == n, (b, key, int(counts[c]), n)
            for side, k in (("a", ka), ("b", kb)):
                row = out["%s_%s" % (key, side)][b].cpu()
                assert torch.equal(row[:n], torch.from_numpy(o[k])), (b, key, side)
                assert bool((row[n:] == -1).all()), (b, key, side)


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "synthetic_multi_object_batch.npz"))


def golden_groups():
    groups = {}
    for i, (name, _, _, over) in enumerate(MG.CASES):
        groups.setdefault(tuple(sorted(over.items())), []).append(i)
    return list(groups.values())


@pytest.mark.parametrize("group", golden_groups(), ids=lambda g: MG.CASES[g[0]][0])
def test_golden_cases(golden, group):
    cases = [MG.case_inputs(i) for i in group]
    As, Bs, K, cfg, rands = [c[0] for c in cases], [c[1] for c in cases], cases[0][2], cases[0][3], [c[4] for c in cases]
    sa, sb, rand = stack(As, Bs, rands)
    out = S.synthetic_multi_object_batch(sa, sb, K, training_config(cfg), rand=rand)
    for b, i in enumerate(group):
        name = MG.CASES[i][0]
        for img in ("a", "b"):
            ref = normalised(golden["%s/rgb_%s" % (name, img)])
            assert torch.equal(out["image_" + img][b].cpu().view(torch.int32), ref.view(torch.int32)), (name, img)
        assert bool(out["empty"][b]) == bool(golden[name + "/empty"]), name
        # against the reference's own correspondences: survivors equal up to one, matched pixels within one pixel
        n = int(out["counts"][b, 0])
        got = list(zip(out["matches_a"][b, :n].tolist(), out["matches_b"][b, :n].tolist()))
        ref = list(zip(golden[name + "/matches_a"].tolist(), golden[name + "/matches_b"].tolist()))
        assert abs(len(got) - len(ref)) <= 1, (name, len(got), len(ref))
        ga, ra = dict(got), dict(ref)
        for a in set(ga) & set(ra):
            assert abs(ga[a] % MG.W - ra[a] % MG.W) <= 1 and abs(ga[a] // MG.W - ra[a] // MG.W) <= 1, (name, a)
        if got == ref:
            for key, ka, kb, c in LISTS:
                m = int(out["counts"][b, c])
                assert out["%s_a" % key][b, :m].cpu().tolist() == golden["%s/%s" % (name, ka)].tolist(), (name, key)
                assert out["%s_b" % key][b, :m].cpu().tolist() == golden["%s/%s" % (name, kb)].tolist(), (name, key)
    check_against_oracle(out, As, Bs, K, cfg, rands)


def scene(B, H, W, seed):
    """B pairs of two ray-cast tilted-plane scenes each (as tests/test_gpu_ops.py), random RGB, blob masks."""
    K = np.array([[533.6422696034836 * W / 640, 0, 319.4091030774892 * W / 640], [0, 534.7824445233571 * H / 480,
                  236.4374299691866 * H / 480], [0, 0, 1.0]])
    g = np.random.RandomState(seed)

    def pose(rx, ry, t):
        cx, sx, cy, sy = np.cos(rx), np.sin(rx), np.cos(ry), np.sin(ry)
        Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]); Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
        T = np.eye(4); T[:3, :3] = Ry.dot(Rx); T[:3, 3] = t
        return T

    def render(T):
        us, vs = np.meshgrid(np.arange(W), np.arange(H))
        rays = np.linalg.inv(K).dot(np.stack([us.ravel(), vs.ravel(), np.ones(H * W)]))
        nrm, d0 = np.array([-0.1, 0.05, 1.0]), 1.2
        s = (d0 - nrm.dot(T[:3, 3])) / nrm.dot(T[:3, :3].dot(rays))
        return np.round(s * 1000.0).reshape(H, W).astype(np.float32)

    def one():
        p1 = pose(0.02 * g.randn(), 0.02 * g.randn(), [0, 0, 0]); p2 = pose(0.05 * g.randn(), 0.1 * g.randn(), 0.05 * g.randn(3))
        m1 = (g.rand(H, W) > 0.2).astype(np.uint8); m1[: H // 4] = 0; m1[H // 2: H // 2 + 2] = 255
        m2 = (g.rand(H, W) > 0.3).astype(np.uint8); m2[:, : W // 3] = 0; m2[-1, -1] = 2
        return dict(rgb_1=g.randint(0, 256, (H, W, 3)).astype(np.uint8), rgb_2=g.randint(0, 256, (H, W, 3)).astype(np.uint8),
                    depth_1=render(p1), depth_2=render(p2), mask_1=m1, mask_2=m2, pose_1=p1, pose_2=p2)
    return [one() for _ in range(B)], [one() for _ in range(B)], K


def run_scene(B, H, W, tc, seed):
    As, Bs, K = scene(B, H, W, seed)
    rand = S.draw_synthetic_multi_object_rand(B, H, W, tc, generator=torch.Generator(device=DEV).manual_seed(seed))
    rands = [{k: v[b].cpu().numpy() for k, v in rand.items()} for b in range(B)]
    sa, sb, _ = stack(As, Bs, rands)
    return As, Bs, K, rands, (sa, sb), rand, S.synthetic_multi_object_batch(sa, sb, K, tc, rand=rand)


def test_default_config_640x480_batch_of_8():
    B, H, W = 8, 480, 640
    As, Bs, K, rands, (sa, sb), rand, out = run_scene(B, H, W, DEFAULT, 7)
    assert tuple(out["matches_a"].shape) == (B, 20000) and tuple(out["masked_non_matches_a"].shape) == (B, 1500000)
    assert tuple(out["blind_non_matches_a"].shape) == (B, 1)
    assert int(out["counts"][:, 0].max()) > 1000
    check_against_oracle(out, As, Bs, K, S.within_scene_cfg(DEFAULT), rands)
    again = S.synthetic_multi_object_batch(sa, sb, K, DEFAULT, rand=rand)
    for k, v in out.items():
        if isinstance(v, torch.Tensor) and v.is_cuda:
            assert torch.equal(v, again[k]), k


@pytest.mark.parametrize("shape", [(1, 1), (1, 9), (7, 1), (5, 7), (37, 53)])
def test_tiny_and_ragged_shapes(shape):
    H, W = shape
    tc = {"training": dict(DEFAULT["training"], num_matching_attempts=23, num_non_matches_per_match=5,
                           fraction_background_non_matches=0.4)}
    As, Bs, K, rands, _, _, out = run_scene(4, H, W, tc, 11 + H * W)
    check_against_oracle(out, As, Bs, K, S.within_scene_cfg(tc), rands)


def test_no_sync_launch_count_and_generator_path():
    H, W = 48, 64
    tc = {"training": dict(DEFAULT["training"], num_matching_attempts=300, num_non_matches_per_match=6)}
    launches = []
    for B in (1, 8):
        As, Bs, K = scene(B, H, W, 3)
        sa, sb, _ = stack(As, Bs, [{"merge": np.zeros(2)}])
        rand = S.draw_synthetic_multi_object_rand(B, H, W, tc, generator=torch.Generator(device=DEV).manual_seed(5))
        gen = torch.Generator(device=DEV).manual_seed(5)
        torch.cuda.synchronize()
        n0 = N.launch_count()
        torch.cuda.set_sync_debug_mode("error")
        try:
            out = S.synthetic_multi_object_batch(sa, sb, K, tc, rand=rand)
            out_g = S.synthetic_multi_object_batch(sa, sb, K, tc, generator=gen)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        launches.append((N.launch_count() - n0) // 2)
        for k, v in out.items():
            if isinstance(v, torch.Tensor) and v.is_cuda:
                assert torch.equal(v, out_g[k]), k
    assert launches[0] == launches[1] == 15, launches


def test_loss_with_num_valid_equals_per_pair_loss():
    group = golden_groups()[0]
    cases = [MG.case_inputs(i) for i in group]
    As, Bs, K, cfg, rands = [c[0] for c in cases], [c[1] for c in cases], cases[0][2], cases[0][3], [c[4] for c in cases]
    sa, sb, rand = stack(As, Bs, rands)
    out = S.synthetic_multi_object_batch(sa, sb, K, training_config(cfg), rand=rand)
    B, H, W, D = len(group), MG.H, MG.W, 3
    assert bool(out["empty"].any()) and not bool(out["empty"].all())
    gen = torch.Generator().manual_seed(2)
    A = 0.3 * torch.randn(B, D, H, W, generator=gen); Bt = 0.3 * torch.randn(B, D, H, W, generator=gen)
    lc = dict(LO.DEFAULT_LOSS_CONFIG)
    keys = [k % s for k in ("matches_%s", "masked_non_matches_%s", "background_non_matches_%s", "blind_non_matches_%s") for s in "ab"]
    Ag = A.to(DEV).requires_grad_(); Bg = Bt.to(DEV).requires_grad_()
    five = loss_composer.get_loss(pdc_b200.PixelwiseContrastiveLoss([H, W], dict(lc)), out["match_type"],
                                  process_network_output(Ag, B, D, H, W), process_network_output(Bg, B, D, H, W),
                                  *[out[k] for k in keys], num_valid=out["num_valid"])
    five[0].backward()
    Ar = A.clone().requires_grad_(); Br = Bt.clone().requires_grad_()
    par, pbr = process_network_output(Ar, B, D, H, W), process_network_output(Br, B, D, H, W)
    ref = LO.TorchPixelwiseContrastiveLoss([H, W], dict(lc))
    terms = [torch.zeros(()) for _ in range(5)]
    for b in range(B):
        c = out["counts"][b].cpu()
        if int(c[0]) == 0:
            continue
        lists = [out["%s_%s" % (key, s)][b, :int(c[i])].cpu() for key, _, _, i in LISTS for s in ("a", "b")]
        o = LO.get_loss(ref, torch.tensor([LO.SpartanDatasetDataType.SYNTHETIC_MULTI_OBJECT]), par[b:b + 1], pbr[b:b + 1],
                        *lists, LO.empty_tensor(), LO.empty_tensor())
        terms = [t + o[i].reshape(()) for i, t in enumerate(terms)]
    five_r = [t / B for t in terms]
    five_r[0].backward()
    for i in range(5):
        assert abs(float(five[i]) - float(five_r[i])) <= 2e-6 * max(1.0, abs(float(five_r[i]))), (i, float(five[i]), float(five_r[i]))
    rel = lambda x, y: float((x.detach().cpu() - y).norm() / max(float(y.norm()), 1e-30))
    assert rel(Ag.grad, Ar.grad) < 1e-5 and rel(Bg.grad, Br.grad) < 1e-5


def test_training_step_on_a_produced_batch_640x480():
    B, H, W, D = 8, 480, 640, 3
    As, Bs, K = scene(B, H, W, 5)
    sa, sb, _ = stack(As, Bs, [{"merge": np.zeros(2)}])
    out = S.synthetic_multi_object_batch(sa, sb, K, DEFAULT, generator=torch.Generator(device=DEV).manual_seed(3))
    dcn = pdc_b200.DenseCorrespondenceNetwork.from_config({"descriptor_dimension": D, "image_width": W, "image_height": H},
                                                          load_stored_params=False)
    pcl = pdc_b200.PixelwiseContrastiveLoss(dcn.image_shape, dict(pdc_b200.DEFAULT_LOSS_CONFIG))
    keys = [k % s for k in ("matches_%s", "masked_non_matches_%s", "background_non_matches_%s", "blind_non_matches_%s") for s in "ab"]
    a, b = dcn.forward_pair(out["image_a"], out["image_b"])
    five = loss_composer.get_loss(pcl, out["match_type"], dcn.process_network_output(a, B), dcn.process_network_output(b, B),
                                  *[out[k] for k in keys], num_valid=out["num_valid"])
    five[0].backward()
    assert bool(torch.isfinite(five[0]).all()) and float(five[0]) > 0
    grads = [p.grad for p in dcn.parameters() if p.grad is not None]
    assert grads and all(bool(torch.isfinite(g).all()) for g in grads)
