"""GPU: pdc_b200.sampling.within_scene_batch (csrc/within_scene.cu) against the reference's get_within_scene_data.

* images: the augmented, flipped images are the executed reference's (tests/golden/within_scene_batch.npz) pushed through
  the normalisation table, bit for bit;
* correspondences: the batched finder equals ddn_find_pixel_correspondences pair by pair (then flipped), bit for bit;
* everything downstream (flip, all index sets, counts, padding, the empty pair) equals oracle/within_scene_oracle.py fed
  with the device's correspondences, bit for bit; against the reference's own correspondences, the 0.2 % rule of
  tests/test_gpu_ops.py applies (fp32 FFMA vs the CPU's matrix products);
* 640 x 480 at the default training config with B = 8, and tiny / ragged shapes;
* repeatability, no host synchronisation, launches independent of B, the generator path, the random-number ranges;
* the loss on the padded output with num_valid equals the mean of the per-pair losses on the unpadded lists."""
import os

import numpy as np
import pytest
import torch

import pdc_b200
from pdc_b200 import _native as N
from pdc_b200 import loss_composer
from pdc_b200 import sampling as S
from oracle import loss_oracle as LO
from oracle import make_golden_within_scene as MG
from oracle import within_scene_oracle as WO
from oracle.resnet34_8s_oracle import process_network_output

pytestmark = pytest.mark.gpu
DEV = "cuda"
LISTS = (("matches", "matches_a", "matches_b", 0), ("masked_non_matches", "masked_a", "masked_b", 1),
         ("background_non_matches", "background_a", "background_b", 2), ("blind_non_matches", "blind_a", "blind_b", 3))
LUT = torch.from_numpy(WO.normalize_lut())


def training_config(cfg):
    nn = 1
    return {"training": dict(num_matching_attempts=cfg["n_attempts"], num_non_matches_per_match=nn,
                             fraction_masked_non_matches=cfg["k_masked"] / nn, fraction_background_non_matches=cfg["k_background"] / nn,
                             sample_matches_only_off_mask=cfg["sample_matches_only_off_mask"],
                             domain_randomize=cfg["domain_randomize"], use_image_b_mask_inv=cfg["use_image_b_mask_inv"])}


def normalised(rgb_u8):
    """uint8 [..., H, W, 3] -> fp32 [..., 3, H, W] through the table (== ToTensor + Normalize)."""
    x = torch.as_tensor(rgb_u8).long()
    return torch.stack([LUT[c][x[..., c]] for c in range(3)], dim=-3)


def stack_inputs(inputs, rands):
    t = lambda k, dt=None: torch.from_numpy(np.stack([x[k] for x in inputs])).to(DEV)
    r = {k: torch.from_numpy(np.stack([x[k] for x in rands])).to(DEV) for k in rands[0]}
    return (t("rgb_a"), t("rgb_b"), t("depth_a"), t("depth_b"), t("mask_a"), t("mask_b"),
            np.stack([x["pose_a"] for x in inputs]), np.stack([x["pose_b"] for x in inputs]), inputs[0]["K"]), r


def candidates(x, cfg, rand):
    """The finder's candidate pixels (as the device draws them): from mask_a or uniform."""
    H, W = x["mask_a"].shape
    n = cfg["n_attempts"]
    u, v = torch.from_numpy(rand["cand_u"][:n]), torch.from_numpy(rand["cand_v"][:n])
    nz = torch.nonzero(torch.from_numpy(x["mask_a"]).reshape(-1)).squeeze(1)
    if cfg["sample_matches_only_off_mask"] and len(nz):
        return nz[torch.clamp(torch.floor(u * len(nz)).long(), max=len(nz) - 1)]
    return torch.clamp(torch.floor(v * H).long(), max=H - 1) * W + torch.clamp(torch.floor(u * W).long(), max=W - 1)


def check_against_oracle(out, inputs, rands, cfg):
    """Device vs oracle fed with ddn_find_pixel_correspondences's correspondences, pair by pair, bit for bit."""
    for b, (x, rand) in enumerate(zip(inputs, rands)):
        H, W = x["mask_a"].shape
        cand = candidates(x, cfg, rand).to(DEV)
        a, bb, u2, v2 = S.find_pixel_correspondences(torch.from_numpy(x["depth_a"]).to(DEV), x["pose_a"],
                                                     torch.from_numpy(x["depth_b"]).to(DEV), x["pose_b"], cand, x["K"])
        a, u2, v2 = a.cpu(), u2.cpu(), v2.cpu()
        o = WO.get_within_scene_data(WO.RESTATED, x["rgb_a"], x["rgb_b"], x["depth_a"], x["depth_b"], x["mask_a"], x["mask_b"],
                                     x["pose_a"], x["pose_b"], x["K"], cfg, rand, uv=(a % W, a // W, u2, v2))
        assert bool(out["empty"][b]) == o["empty"], b
        for img in ("a", "b"):
            got = out["image_" + img][b].cpu()
            assert torch.equal(got.view(torch.int32), normalised(o["rgb_" + img]).view(torch.int32)), (b, img)
        counts = out["counts"][b].cpu()
        for key, ka, kb, c in LISTS:
            n = len(o[ka])
            assert int(counts[c]) == n, (b, key, int(counts[c]), n)
            for side, k in (("a", ka), ("b", kb)):
                row = out["%s_%s" % (key, side)][b].cpu()
                assert torch.equal(row[:n], torch.from_numpy(o[k])), (b, key, side)
                assert bool((row[n:] == -1).all()), (b, key, side)


def golden_groups():
    groups = {}
    for i, (name, _, _, over) in enumerate(MG.CASES):
        groups.setdefault(tuple(sorted(over.items())), []).append(i)
    return list(groups.values())


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "within_scene_batch.npz"))


@pytest.mark.parametrize("group", golden_groups(), ids=lambda g: MG.CASES[g[0]][0])
def test_golden_cases(golden, group):
    cases = [MG.case_inputs(i) for i in group]
    inputs, cfg, rands = [c[0] for c in cases], cases[0][1], [c[2] for c in cases]
    args, rand = stack_inputs(inputs, rands)
    out = S.within_scene_batch(*args, training_config(cfg), rand=rand)
    for b, i in enumerate(group):
        name = MG.CASES[i][0]
        for img in ("a", "b"):
            ref = normalised(golden["%s/rgb_%s" % (name, img)])
            assert torch.equal(out["image_" + img][b].cpu().view(torch.int32), ref.view(torch.int32)), (name, img)
        assert bool(out["empty"][b]) == bool(golden[name + "/empty"])
        # against the reference's own correspondences: the same candidates survive and a match in B moves by at most one
        # pixel (the planar scene puts sub-pixel positions on integers, where fp32 FFMA and the CPU's matrix products
        # truncate differently); equal matches -> every list equal
        n = int(out["counts"][b, 0])
        got = list(zip(out["matches_a"][b, :n].tolist(), out["matches_b"][b, :n].tolist()))
        ref = list(zip(golden[name + "/matches_a"].tolist(), golden[name + "/matches_b"].tolist()))
        ga, ra = dict(got), dict(ref)
        assert len(set(ga) ^ set(ra)) <= 1, (name, sorted(set(ga) ^ set(ra)))
        for a in set(ga) & set(ra):
            assert abs(ga[a] % MG.W - ra[a] % MG.W) <= 1 and abs(ga[a] // MG.W - ra[a] // MG.W) <= 1, (name, a, ga[a], ra[a])
        if got == ref:
            for key, ka, kb, c in LISTS:
                m = int(out["counts"][b, c])
                assert out["%s_a" % key][b, :m].cpu().tolist() == golden["%s/%s" % (name, ka)].tolist(), (name, key)
                assert out["%s_b" % key][b, :m].cpu().tolist() == golden["%s/%s" % (name, kb)].tolist(), (name, key)
    check_against_oracle(out, inputs, rands, cfg)
    if any(bool(golden[MG.CASES[i][0] + "/empty"]) for i in group):
        b = [bool(golden[MG.CASES[i][0] + "/empty"]) for i in group].index(True)
        assert int(out["counts"][b].abs().sum()) == 0
        assert torch.equal(out["image_a"][b], out["image_b"][b])


def scene(B, H, W, seed):
    """B pairs of a ray-cast tilted plane (as tests/test_gpu_ops.py), random RGB, blob masks (values 1 and some 255)."""
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
    inputs = []
    for b in range(B):
        pa = pose(0.02 * g.randn(), 0.02 * g.randn(), [0, 0, 0]); pb = pose(0.05 * g.randn(), 0.1 * g.randn(), 0.05 * g.randn(3))
        da, db = render(pa), render(pb)
        da[: H // 8, : W // 5] = 0.0
        mask_a = (g.rand(H, W) > 0.1).astype(np.uint8); mask_a[: H // 4] = 0; mask_a[H // 2: H // 2 + 2] = 255
        mask_b = (g.rand(H, W) > 0.2).astype(np.uint8); mask_b[:, : W // 3] = 0
        inputs.append(dict(rgb_a=g.randint(0, 256, (H, W, 3)).astype(np.uint8), rgb_b=g.randint(0, 256, (H, W, 3)).astype(np.uint8),
                           depth_a=da, depth_b=db, mask_a=mask_a, mask_b=mask_b, pose_a=pa, pose_b=pb, K=K))
    return inputs


DEFAULT = {"training": dict(num_matching_attempts=10000, num_non_matches_per_match=150, fraction_masked_non_matches=0.5,
                            fraction_background_non_matches=0.5, sample_matches_only_off_mask=True, domain_randomize=True,
                            use_image_b_mask_inv=True)}


def run_scene(B, H, W, tc, seed):
    inputs = scene(B, H, W, seed)
    gen = torch.Generator(device=DEV).manual_seed(seed)
    rand = S.draw_within_scene_rand(B, H, W, tc, generator=gen)
    rands = [{k: v[b].cpu().numpy() for k, v in rand.items()} for b in range(B)]
    args, _ = stack_inputs(inputs, rands)
    return inputs, rands, args, rand, S.within_scene_batch(*args, tc, rand=rand)


def test_default_config_640x480_batch_of_8():
    B, H, W = 8, 480, 640
    inputs, rands, args, rand, out = run_scene(B, H, W, DEFAULT, 7)
    cfg = S.within_scene_cfg(DEFAULT)
    assert tuple(out["image_a"].shape) == (B, 3, H, W) and tuple(out["matches_a"].shape) == (B, 10000)
    assert tuple(out["masked_non_matches_a"].shape) == (B, 750000) and tuple(out["blind_non_matches_b"].shape) == (B, H * W)
    assert int(out["counts"][:, 0].min()) > 1000 and int(out["counts"][:, 3].min()) > 1000
    check_against_oracle(out, inputs, rands, cfg)
    # repeatability
    again = S.within_scene_batch(*args, DEFAULT, rand=rand)
    for k, v in out.items():
        if isinstance(v, torch.Tensor) and v.is_cuda:
            assert torch.equal(v, again[k]), k


@pytest.mark.parametrize("shape", [(1, 1), (1, 9), (7, 1), (5, 7), (37, 53)])
def test_tiny_and_ragged_shapes(shape):
    H, W = shape
    tc = {"training": dict(DEFAULT["training"], num_matching_attempts=23, num_non_matches_per_match=5,
                           fraction_background_non_matches=0.0)}
    inputs, rands, args, rand, out = run_scene(3, H, W, tc, 11 + H * W)
    assert out["background_non_matches_a"].shape == (3, 0)
    check_against_oracle(out, inputs, rands, S.within_scene_cfg(tc))


def test_no_sync_launch_count_and_generator_path():
    H, W = 48, 64
    tc = {"training": dict(DEFAULT["training"], num_matching_attempts=300, num_non_matches_per_match=6)}
    launches = []
    for B in (1, 8):
        inputs = scene(B, H, W, 3)
        args = (torch.from_numpy(np.stack([x["rgb_a"] for x in inputs])).to(DEV), torch.from_numpy(np.stack([x["rgb_b"] for x in inputs])).to(DEV),
                torch.from_numpy(np.stack([x["depth_a"] for x in inputs])).to(DEV), torch.from_numpy(np.stack([x["depth_b"] for x in inputs])).to(DEV),
                torch.from_numpy(np.stack([x["mask_a"] for x in inputs])).to(DEV), torch.from_numpy(np.stack([x["mask_b"] for x in inputs])).to(DEV),
                np.stack([x["pose_a"] for x in inputs]), np.stack([x["pose_b"] for x in inputs]), inputs[0]["K"])
        rand = S.draw_within_scene_rand(B, H, W, tc, generator=torch.Generator(device=DEV).manual_seed(5))
        gen = torch.Generator(device=DEV).manual_seed(5)
        torch.cuda.synchronize()
        n0 = N.launch_count()
        torch.cuda.set_sync_debug_mode("error")
        try:
            out = S.within_scene_batch(*args, tc, rand=rand)
            out_g = S.within_scene_batch(*args, tc, generator=gen)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        launches.append((N.launch_count() - n0) // 2)
        for k, v in out.items():
            if isinstance(v, torch.Tensor) and v.is_cuda:
                assert torch.equal(v, out_g[k]), k
    assert launches[0] == launches[1] == 16, launches


def test_random_number_ranges_and_masked_pixels_keep_their_rgb():
    B, H, W = 128, 24, 40
    tc = {"training": dict(DEFAULT["training"], num_matching_attempts=50, num_non_matches_per_match=2)}
    rand = S.draw_within_scene_rand(B, H, W, tc, generator=torch.Generator(device=DEV).manual_seed(9))
    dec = rand["params"][:, :, :5].float()
    assert float(dec.max()) == 1.0 and float(dec.min()) == 0.0
    assert bool(((dec.mean(dim=(0, 1)) - 0.5).abs() < 0.08).all()), dec.mean(dim=(0, 1))
    col = rand["params"][:, :, 5:11]
    assert int(col.max()) == 254 and int(col.min()) == 0 and int(rand["params"][:, :, 11:].max()) == 0
    assert int(rand["noise"].max()) == 49 and int(rand["noise"].min()) == 0
    for k in ("cand_u", "masked_v", "blind"):
        assert 0.0 <= float(rand[k].min()) and float(rand[k].max()) < 1.0
    inputs = scene(B, H, W, 4)
    rands = [{k: v[b].cpu().numpy() for k, v in rand.items()} for b in range(B)]
    args, _ = stack_inputs(inputs, rands)
    out = S.within_scene_batch(*args, tc, rand=rand)
    p = rand["params"].cpu()
    for b in range(B):
        for img, key in ((0, "a"), (1, "b")):
            rgb, m = inputs[b]["rgb_" + key], inputs[b]["mask_" + key]
            if p[b, img, 4]:
                rgb, m = rgb[::-1, ::-1], m[::-1, ::-1]
            keep = torch.from_numpy(np.ascontiguousarray(m) == 1)
            ref = normalised(np.ascontiguousarray(rgb))
            got = out["image_" + key][b].cpu()
            assert torch.equal(got[:, keep], ref[:, keep]), (b, key)


def test_loss_with_num_valid_equals_per_pair_loss():
    group = golden_groups()[0]
    cases = [MG.case_inputs(i) for i in group]
    inputs, cfg, rands = [c[0] for c in cases], cases[0][1], [c[2] for c in cases]
    args, rand = stack_inputs(inputs, rands)
    out = S.within_scene_batch(*args, training_config(cfg), rand=rand)
    B, H, W, D = len(group), MG.H, MG.W, 3
    gen = torch.Generator().manual_seed(2)
    A = 0.3 * torch.randn(B, D, H, W, generator=gen); Bt = 0.3 * torch.randn(B, D, H, W, generator=gen)
    lc = dict(LO.DEFAULT_LOSS_CONFIG)
    Ag = A.to(DEV).requires_grad_(); Bg = Bt.to(DEV).requires_grad_()
    five = loss_composer.get_loss(pdc_b200.PixelwiseContrastiveLoss([H, W], dict(lc)), out["match_type"],
                                  process_network_output(Ag, B, D, H, W), process_network_output(Bg, B, D, H, W),
                                  *[out["%s_%s" % (key, s)] for key, _, _, _ in LISTS for s in ("a", "b")], num_valid=out["num_valid"])
    five[0].backward()
    # reference: per-pair losses on the unpadded lists; an empty pair (no matches) contributes 0 and counts in the mean
    Ar = A.clone().requires_grad_(); Br = Bt.clone().requires_grad_()
    par, pbr = process_network_output(Ar, B, D, H, W), process_network_output(Br, B, D, H, W)
    ref = LO.TorchPixelwiseContrastiveLoss([H, W], dict(lc))
    terms = [torch.zeros(()) for _ in range(5)]
    for b in range(B):
        c = out["counts"][b].cpu()
        if int(c[0]) == 0:
            continue
        lists = [out["%s_%s" % (key, s)][b, :int(c[i])].cpu() for key, _, _, i in LISTS for s in ("a", "b")]
        if int(c[3]) == 0:
            lists[6] = lists[7] = LO.empty_tensor()
        o = LO.get_within_scene_loss(ref, par[b:b + 1], pbr[b:b + 1], *lists)
        terms = [t + o[i].reshape(()) for i, t in enumerate(terms)]
    five_r = [t / B for t in terms]
    five_r[0].backward()
    for i in range(5):
        assert abs(float(five[i]) - float(five_r[i])) <= 2e-6 * max(1.0, abs(float(five_r[i]))), (i, float(five[i]), float(five_r[i]))
    rel = lambda x, y: float((x.detach().cpu() - y).norm() / max(float(y.norm()), 1e-30))
    assert rel(Ag.grad, Ar.grad) < 1e-5 and rel(Bg.grad, Br.grad) < 1e-5
