"""GPU: pdc_b200.sampling.across_scene_batch (csrc/across_scene.cu) against the reference's get_across_scene_data.

There is no reprojection on this path, so every output is bit-exact:
* the augmented, flipped images pushed through the normalisation table and the blind lists equal the executed
  reference's (tests/golden/across_scene_batch.npz), and equal oracle/across_scene_oracle.py pair by pair at 640 x 480
  with the default training config and B = 8, and at tiny / ragged shapes;
* empty pairs (mask_a, mask_b or both empty) are image A twice with count 0 and rows of -1;
* repeatability, no host synchronisation, launches independent of B, the generator path;
* get_loss(DIFFERENT_OBJECT) on the output equals the mean of the per-pair reference losses, with and without
  scale_by_hard_negatives_DIFFERENT_OBJECT; SINGLE_OBJECT_ACROSS_SCENE reaches the reference's NameError;
* one training step (forward_pair + get_loss + backward) at 640 x 480, B = 8, on a produced batch."""
import os

import numpy as np
import pytest
import torch

import pdc_b200
from pdc_b200 import _native as N
from pdc_b200 import loss_composer
from pdc_b200 import sampling as S
from pdc_b200.loss_composer import SpartanDatasetDataType as T
from oracle import across_scene_oracle as AO
from oracle import loss_oracle as LO
from oracle import make_golden_across_scene as MG
from oracle import within_scene_oracle as WO
from oracle.resnet34_8s_oracle import process_network_output

pytestmark = pytest.mark.gpu
DEV = "cuda"
LUT = torch.from_numpy(WO.normalize_lut())
EMPTY_KEYS = ("matches", "masked_non_matches", "background_non_matches")
DEFAULT = {"training": dict(cross_scene_num_samples=10000, domain_randomize=True)}


def training_config(cfg):
    return {"training": dict(cross_scene_num_samples=cfg["num_samples"], domain_randomize=cfg["domain_randomize"])}


def normalised(rgb_u8):
    """uint8 [..., H, W, 3] -> fp32 [..., 3, H, W] through the table (== ToTensor + Normalize)."""
    x = torch.as_tensor(rgb_u8).long()
    return torch.stack([LUT[c][x[..., c]] for c in range(3)], dim=-3)


def images(inputs):
    t = lambda k: torch.from_numpy(np.stack([x[k] for x in inputs])).to(DEV)
    return t("rgb_a"), t("rgb_b"), t("mask_a"), t("mask_b")


def stack(inputs, rands):
    return images(inputs), {k: torch.from_numpy(np.stack([r[k] for r in rands])).to(DEV) for k in rands[0]}


def check_against_oracle(out, inputs, rands, cfg):
    """Device vs the restated reference, pair by pair, bit for bit."""
    B = len(inputs)
    for k in EMPTY_KEYS:
        assert out[k + "_a"].shape == (B, 0) and out[k + "_b"].shape == (B, 0)
    n = cfg["num_samples"]
    for b, (x, rand) in enumerate(zip(inputs, rands)):
        o = AO.get_across_scene_data(AO.RESTATED, x["rgb_a"], x["rgb_b"], x["mask_a"], x["mask_b"], cfg, rand)
        assert o["python_left"] == 0 and o["numpy_left"] == 0 and o["torch_left"] == 0
        assert bool(out["empty"][b]) == o["empty"], b
        for img in ("a", "b"):
            got = out["image_" + img][b].cpu()
            assert torch.equal(got.view(torch.int32), normalised(o["rgb_" + img]).view(torch.int32)), (b, img)
        c = out["counts"][b].cpu().tolist()
        assert c == [0, 0, 0, 0 if o["empty"] else n], (b, c)
        for side in ("a", "b"):
            row = out["blind_non_matches_" + side][b].cpu()
            if o["empty"]:
                assert bool((row == -1).all()), (b, side)
            else:
                assert torch.equal(row, torch.from_numpy(o["blind_" + side])), (b, side)
        assert int(out["num_valid"]["blind"][b]) == c[3]


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "across_scene_batch.npz"))


def golden_groups():
    groups = {}
    for i, (name, _, _, over) in enumerate(MG.CASES):
        groups.setdefault(tuple(sorted(over.items())), []).append(i)
    return list(groups.values())


@pytest.mark.parametrize("group", golden_groups(), ids=lambda g: MG.CASES[g[0]][0])
def test_golden_cases(golden, group):
    cases = [MG.case_inputs(i) for i in group]
    inputs, cfg, rands = [c[0] for c in cases], cases[0][1], [c[2] for c in cases]
    args, rand = stack(inputs, rands)
    out = S.across_scene_batch(*args, training_config(cfg), rand=rand)
    for b, i in enumerate(group):
        name = MG.CASES[i][0]
        for img in ("a", "b"):
            ref = normalised(golden["%s/rgb_%s" % (name, img)])
            assert torch.equal(out["image_" + img][b].cpu().view(torch.int32), ref.view(torch.int32)), (name, img)
        empty = bool(golden[name + "/empty"])
        assert bool(out["empty"][b]) == empty, name
        for side in ("a", "b"):
            row = out["blind_non_matches_" + side][b].cpu()
            if empty:
                assert bool((row == -1).all()) and int(out["counts"][b, 3]) == 0, name
            else:
                assert row.tolist() == golden["%s/blind_%s" % (name, side)].tolist(), (name, side)
    check_against_oracle(out, inputs, rands, cfg)


def scene(B, H, W, seed, empty=()):
    """B pairs of random RGB with blob masks (values 1, some 255 and 2); pair b gets an empty mask_a / mask_b / both when
    empty[b] is "a" / "b" / "ab"."""
    g = np.random.RandomState(seed)
    inputs = []
    for b in range(B):
        mask_a = (g.rand(H, W) > 0.3).astype(np.uint8); mask_a[: H // 4] = 0; mask_a[H // 2: H // 2 + 2] = 255
        mask_b = (g.rand(H, W) > 0.6).astype(np.uint8); mask_b[:, : W // 3] = 0; mask_b[-1, -1] = 2
        e = empty[b] if b < len(empty) else ""
        if "a" in e:
            mask_a[:] = 0
        if "b" in e:
            mask_b[:] = 0
        inputs.append(dict(rgb_a=g.randint(0, 256, (H, W, 3)).astype(np.uint8), rgb_b=g.randint(0, 256, (H, W, 3)).astype(np.uint8),
                           mask_a=mask_a, mask_b=mask_b))
    return inputs


def run_scene(B, H, W, tc, seed, empty=()):
    inputs = scene(B, H, W, seed, empty)
    rand = S.draw_across_scene_rand(B, H, W, tc, generator=torch.Generator(device=DEV).manual_seed(seed))
    rands = [{k: v[b].cpu().numpy() for k, v in rand.items()} for b in range(B)]
    args, _ = stack(inputs, rands)
    return inputs, rands, args, rand, S.across_scene_batch(*args, tc, rand=rand)


def test_default_config_640x480_batch_of_8_with_empty_pairs():
    B, H, W = 8, 480, 640
    inputs, rands, args, rand, out = run_scene(B, H, W, DEFAULT, 7, empty=("", "a", "", "b", "", "ab"))
    assert tuple(out["image_a"].shape) == (B, 3, H, W) and tuple(out["blind_non_matches_a"].shape) == (B, 10000)
    assert out["empty"].cpu().tolist() == [False, True, False, True, False, True, False, False]
    check_against_oracle(out, inputs, rands, S.across_scene_cfg(DEFAULT))
    for b in (1, 3, 5):                                        # an empty pair returns the normalised image A twice
        ref = normalised(inputs[b]["rgb_a"]).to(DEV)
        assert torch.equal(out["image_a"][b], ref) and torch.equal(out["image_b"][b], ref)
    again = S.across_scene_batch(*args, DEFAULT, rand=rand)
    for k, v in out.items():
        if isinstance(v, torch.Tensor) and v.is_cuda:
            assert torch.equal(v, again[k]), k


@pytest.mark.parametrize("shape", [(1, 1), (1, 9), (7, 1), (5, 7), (37, 53)])
def test_tiny_and_ragged_shapes(shape):
    H, W = shape
    tc = {"training": dict(DEFAULT["training"], cross_scene_num_samples=29)}
    inputs, rands, args, rand, out = run_scene(4, H, W, tc, 11 + H * W, empty=("", "", "b"))
    check_against_oracle(out, inputs, rands, S.across_scene_cfg(tc))


def test_no_sync_launch_count_and_generator_path():
    H, W = 48, 64
    tc = {"training": dict(DEFAULT["training"], cross_scene_num_samples=300)}
    launches = []
    for B in (1, 8):
        inputs = scene(B, H, W, 3, empty=("", "a"))
        args = images(inputs)
        rand = S.draw_across_scene_rand(B, H, W, tc, generator=torch.Generator(device=DEV).manual_seed(5))
        gen = torch.Generator(device=DEV).manual_seed(5)
        torch.cuda.synchronize()
        n0 = N.launch_count()
        torch.cuda.set_sync_debug_mode("error")
        try:
            out = S.across_scene_batch(*args, tc, rand=rand)
            out_g = S.across_scene_batch(*args, tc, generator=gen, match_type=T.SINGLE_OBJECT_ACROSS_SCENE)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        launches.append((N.launch_count() - n0) // 2)
        for k, v in out.items():
            if isinstance(v, torch.Tensor) and v.is_cuda:
                assert torch.equal(v, out_g[k]), k
        assert out["match_type"].tolist() == [T.DIFFERENT_OBJECT] * B
        assert out_g["match_type"].tolist() == [T.SINGLE_OBJECT_ACROSS_SCENE] * B
    assert launches[0] == launches[1] == 5, launches


def test_random_number_layout():
    B, H, W = 16, 12, 20
    tc = {"training": dict(DEFAULT["training"], cross_scene_num_samples=77)}
    rand = S.draw_across_scene_rand(B, H, W, tc, generator=torch.Generator(device=DEV).manual_seed(9))
    assert rand["params"].shape == (B, 2, 16) and rand["noise"].shape == (B, 2, 2, H, W, 3)
    assert rand["blind_a"].shape == rand["blind_b"].shape == (B, 77) and rand["blind_a"].dtype == torch.float32
    assert not torch.equal(rand["blind_a"], rand["blind_b"])
    for k in ("blind_a", "blind_b"):
        assert 0.0 <= float(rand[k].min()) and float(rand[k].max()) < 1.0
    assert int(rand["params"][:, :, 5:11].max()) <= 254 and int(rand["params"][:, :, 11:].max()) == 0
    assert int(rand["params"][:, :, :5].max()) <= 1 and int(rand["noise"].max()) <= 49


@pytest.mark.parametrize("scale_by_hard", [True, False])
def test_different_object_loss_equals_per_pair_reference(scale_by_hard):
    B, H, W, D = 6, 24, 32, 3
    tc = {"training": dict(DEFAULT["training"], cross_scene_num_samples=200)}
    _, _, _, _, out = run_scene(B, H, W, tc, 21, empty=("", "b", "", "", "a"))
    gen = torch.Generator().manual_seed(2)
    A = 0.2 * torch.randn(B, D, H, W, generator=gen); Bt = 0.2 * torch.randn(B, D, H, W, generator=gen)
    lc = dict(LO.DEFAULT_LOSS_CONFIG, scale_by_hard_negatives_DIFFERENT_OBJECT=scale_by_hard)
    Ag = A.to(DEV).requires_grad_(); Bg = Bt.to(DEV).requires_grad_()
    keys = [k % s for k in ("matches_%s", "masked_non_matches_%s", "background_non_matches_%s", "blind_non_matches_%s")
            for s in "ab"]
    five = loss_composer.get_loss(pdc_b200.PixelwiseContrastiveLoss([H, W], dict(lc)), out["match_type"],
                                  process_network_output(Ag, B, D, H, W), process_network_output(Bg, B, D, H, W),
                                  *[out[k] for k in keys], num_valid=out["num_valid"])
    five[0].backward()
    # reference: per-pair losses on the unpadded lists (batch size 1); an empty pair contributes 0 and counts in the mean
    Ar = A.clone().requires_grad_(); Br = Bt.clone().requires_grad_()
    par, pbr = process_network_output(Ar, B, D, H, W), process_network_output(Br, B, D, H, W)
    ref = LO.TorchPixelwiseContrastiveLoss([H, W], dict(lc))
    terms = [torch.zeros(()) for _ in range(5)]
    for b in range(B):
        n = int(out["counts"][b, 3])
        if n == 0:
            continue
        o = LO.get_loss(ref, torch.tensor([T.DIFFERENT_OBJECT]), par[b:b + 1], pbr[b:b + 1], None, None, None, None, None, None,
                        out["blind_non_matches_a"][b, :n].cpu(), out["blind_non_matches_b"][b, :n].cpu())
        terms = [t + o[i].reshape(()) for i, t in enumerate(terms)]
    five_r = [t / B for t in terms]
    assert float(five_r[0]) > 0
    five_r[0].backward()
    for i in range(5):
        assert abs(float(five[i]) - float(five_r[i])) <= 2e-6 * max(1.0, abs(float(five_r[i]))), (i, float(five[i]), float(five_r[i]))
    rel = lambda x, y: float((x.detach().cpu() - y).norm() / max(float(y.norm()), 1e-30))
    assert rel(Ag.grad, Ar.grad) < 1e-5 and rel(Bg.grad, Br.grad) < 1e-5


def test_single_object_across_scene_reaches_the_reference_name_error():
    B, H, W, D = 2, 16, 24, 3
    tc = {"training": dict(DEFAULT["training"], cross_scene_num_samples=50)}
    inputs = scene(B, H, W, 4)
    args = images(inputs)
    out = S.across_scene_batch(*args, tc, generator=torch.Generator(device=DEV).manual_seed(1),
                               match_type=T.SINGLE_OBJECT_ACROSS_SCENE)
    pred = torch.zeros(B, H * W, D, device=DEV)
    keys = [k % s for k in ("matches_%s", "masked_non_matches_%s", "background_non_matches_%s", "blind_non_matches_%s")
            for s in "ab"]
    with pytest.raises(NameError, match="pcl"):
        loss_composer.get_loss(pdc_b200.PixelwiseContrastiveLoss([H, W], dict(LO.DEFAULT_LOSS_CONFIG)), out["match_type"],
                               pred, pred, *[out[k] for k in keys], num_valid=out["num_valid"])


def test_training_step_on_a_produced_batch_640x480():
    B, H, W, D = 8, 480, 640, 3
    inputs = scene(B, H, W, 5, empty=("", "", "a"))
    args = images(inputs)
    out = S.across_scene_batch(*args, DEFAULT, generator=torch.Generator(device=DEV).manual_seed(3))
    dcn = pdc_b200.DenseCorrespondenceNetwork.from_config({"descriptor_dimension": D, "image_width": W, "image_height": H},
                                                          load_stored_params=False)
    pcl = pdc_b200.PixelwiseContrastiveLoss(dcn.image_shape, dict(pdc_b200.DEFAULT_LOSS_CONFIG))
    keys = [k % s for k in ("matches_%s", "masked_non_matches_%s", "background_non_matches_%s", "blind_non_matches_%s")
            for s in "ab"]
    a, b = dcn.forward_pair(out["image_a"], out["image_b"])
    five = loss_composer.get_loss(pcl, out["match_type"], dcn.process_network_output(a, B), dcn.process_network_output(b, B),
                                  *[out[k] for k in keys], num_valid=out["num_valid"])
    five[0].backward()
    assert bool(torch.isfinite(five[0]).all()) and float(five[0]) > 0
    grads = [p.grad for p in dcn.parameters() if p.grad is not None]
    assert grads and all(bool(torch.isfinite(g).all()) for g in grads)
    assert any(float(g.abs().max()) > 0 for g in grads)
