"""Pins the oracle against the real reference and writes tests/golden/*.npz.

Needs a checkout of the reference (PDC_REFERENCE_ROOT=<dir>):   python oracle/make_golden.py [reference_checks]

For every backbone case the REAL reference module (loaded unmodified by oracle/ref_loader.py)
and the oracle restatement are run on the same seeded weights and inputs and must agree
bit-for-bit (forward, running statistics, parameter gradients); the reference's outputs are what
is stored.  For the loss the reference's OWN source is executed (oracle/build_ref.py: the Python-2 files with a short
list of line-anchored py2->py3 patches, written to the git-ignored oracle/_ref/): its outputs and autograd gradients
are what is stored, and the torch restatement must equal them bit-for-bit and the numpy one to 1e-6.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "pytorch-dense-correspondence_b200"))

from oracle import loss_oracle as LO            # noqa: E402
from oracle import build_ref                    # noqa: E402
from oracle import ref_loader                   # noqa: E402
from oracle.resnet34_8s_oracle import seeded_oracle, process_network_output  # noqa: E402
import synthetic                                # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
torch.set_num_threads(os.cpu_count())


def bit_equal(a, b, what):
    assert a.shape == b.shape, what
    assert torch.equal(a, b), "%s: oracle != reference (max abs diff %g)" % (what, (a - b).abs().max().item())


def backbone_case(name, D, B, H, W, seed_data):
    oracle = seeded_oracle(D=D, seed=0)
    ref = ref_loader.reference_resnet34_8s(D, oracle.state_dict())
    assert list(ref.state_dict().keys()) == list(oracle.state_dict().keys())
    g = torch.Generator().manual_seed(seed_data)
    x = torch.randn(B, 3, H, W, generator=g)
    out = {}
    ref.train(); oracle.train()
    y_ref = ref(x); y_or = oracle(x)
    bit_equal(y_ref, y_or, name + " train fwd")
    for k in ("resnet34_8s.bn1.running_mean", "resnet34_8s.bn1.running_var",
              "resnet34_8s.layer4.2.bn2.running_mean", "resnet34_8s.layer4.2.bn2.running_var",
              "resnet34_8s.layer3.0.downsample.1.running_var"):
        bit_equal(ref.state_dict()[k], oracle.state_dict()[k], name + " " + k)
        out["rs:" + k] = ref.state_dict()[k].numpy().copy()
    # a backward through a fixed random cotangent
    cot = torch.randn(y_ref.shape, generator=g)
    (y_ref * cot).sum().backward(); (y_or * cot).sum().backward()
    gr = dict(ref.named_parameters()); go = dict(oracle.named_parameters())
    for k in gr:
        bit_equal(gr[k].grad, go[k].grad, name + " grad " + k)
    out["x_seed"] = np.int64(seed_data)
    out["y_train"] = y_ref.detach().numpy() if H * W <= 96 * 96 else y_ref.detach()[:, :, ::16, ::16].numpy()
    for k in ("resnet34_8s.conv1.weight", "resnet34_8s.bn1.weight", "resnet34_8s.bn1.bias",
              "resnet34_8s.layer1.0.conv1.weight", "resnet34_8s.layer2.0.downsample.0.weight",
              "resnet34_8s.layer2.0.conv1.weight", "resnet34_8s.layer3.0.bn1.weight",
              "resnet34_8s.layer4.2.bn2.bias", "resnet34_8s.fc.weight", "resnet34_8s.fc.bias"):
        out["grad:" + k] = gr[k].grad.numpy().copy()
    out["gradnorm:all"] = np.array([gr[k].grad.double().norm().item() for k in gr])
    ref.eval(); oracle.eval()
    with torch.no_grad():
        ye_ref = ref(x); ye_or = oracle(x)
    bit_equal(ye_ref, ye_or, name + " eval fwd")
    out["y_eval"] = ye_ref.numpy() if H * W <= 96 * 96 else ye_ref[:, :, ::16, ::16].numpy()
    np.savez_compressed(os.path.join(GOLD, name + ".npz"), **out)
    print("wrote", name, {k: v.shape for k, v in out.items() if hasattr(v, "shape") and v.ndim})


def loss_case(name, D, H, W, Nm, k_masked, k_bg, n_blind, cfg_over, seed):
    cfg = dict(LO.DEFAULT_LOSS_CONFIG); cfg.update(cfg_over)
    g = torch.Generator().manual_seed(seed)
    P = H * W
    # descriptors with the scale the network produces (|.| ~ 0.19, SURVEY 8d) so both hinge branches fire
    A = (0.25 * torch.randn(1, D, H, W, generator=g)).requires_grad_()
    Bt = (0.25 * torch.randn(1, D, H, W, generator=g)).requires_grad_()
    pa = process_network_output(A, 1, D, H, W); pb = process_network_output(Bt, 1, D, H, W)
    ma = torch.randint(0, P, (Nm,), generator=g); mb = torch.randint(0, P, (Nm,), generator=g)
    na_m = ma.repeat_interleave(k_masked); nb_m = torch.randint(0, P, (Nm * k_masked,), generator=g)
    na_b = ma.repeat_interleave(k_bg); nb_b = torch.randint(0, P, (Nm * k_bg,), generator=g)
    if n_blind:
        xa = torch.randint(0, P, (n_blind,), generator=g); xb = torch.randint(0, P, (n_blind,), generator=g)
    else:
        xa = xb = LO.empty_tensor()
    # the executed reference (oracle/_ref) produces the stored values ...
    ref = build_ref.load()
    mt = torch.tensor([ref.dataset.SpartanDatasetDataType.SINGLE_OBJECT_WITHIN_SCENE])
    five = ref.composer.get_loss(ref.pcl.PixelwiseContrastiveLoss([H, W], dict(cfg)), mt, pa, pb, ma, mb, na_m, nb_m, na_b, nb_b, xa, xb)
    five[0].reshape(()).backward()
    # ... and the torch restatement must reproduce them bit-for-bit (same ops, same order)
    A2 = A.detach().clone().requires_grad_(); B2 = Bt.detach().clone().requires_grad_()
    five_o = LO.get_loss(LO.TorchPixelwiseContrastiveLoss([H, W], dict(cfg)), mt, process_network_output(A2, 1, D, H, W),
                         process_network_output(B2, 1, D, H, W), ma, mb, na_m, nb_m, na_b, nb_b, xa, xb)
    five_o[0].reshape(()).backward()
    assert [float(t) for t in five_o] == [float(t) for t in five], name
    assert torch.equal(A2.grad, A.grad) and torch.equal(B2.grad, Bt.grad), name
    idx = dict(matches_a=ma.numpy(), matches_b=mb.numpy(), masked_a=na_m.numpy(), masked_b=nb_m.numpy(),
               background_a=na_b.numpy(), background_b=nb_b.numpy(),
               blind_a=xa.numpy(), blind_b=xb.numpy())
    An = A.detach().numpy()[0].reshape(D, P).T; Bn = Bt.detach().numpy()[0].reshape(D, P).T
    five_np, counts = LO.np_within_scene_loss(An, Bn, idx, cfg, W)
    for t, n_ in zip(five, five_np):
        assert abs(float(t) - n_) <= 1e-6 * max(1.0, abs(n_)), (name, float(t), n_)
    out = dict(idx)
    out.update(A=A.detach().numpy(), B=Bt.detach().numpy(), five=np.array([float(t) for t in five]),
               counts=np.array(counts), dA=A.grad.numpy(), dB=Bt.grad.numpy(),
               cfg_keys=np.array(sorted(cfg_over.keys())), cfg_vals=np.array([float(cfg_over[k]) for k in sorted(cfg_over)]))
    np.savez_compressed(os.path.join(GOLD, name + ".npz"), **out)
    print("wrote", name, "five", out["five"], "counts", counts)


def train_step_case(name, D, B, H, W, Nm, Nn, seed):
    """fwd(A), fwd(B), within-scene loss (mean over pairs), backward -- reference backbone + the loss restatement (which the
    loss cases above and tests/test_oracle_ref_cpu.py pin bit-for-bit to the executed reference loss)."""
    oracle = seeded_oracle(D=D, seed=0)
    ref = ref_loader.reference_resnet34_8s(D, oracle.state_dict())
    ref.train()
    data = synthetic.make_pair_batch(B, H, W, Nm, Nn, Nn, 0, seed=seed)
    pcl = LO.TorchPixelwiseContrastiveLoss([H, W], dict(LO.DEFAULT_LOSS_CONFIG))
    ya = ref(data["img_a"]); yb = ref(data["img_b"])
    pa = process_network_output(ya, B, D, H, W); pb = process_network_output(yb, B, D, H, W)
    five = LO.batched_within_scene_loss(pcl, pa, pb, data)
    five[0].backward()
    gr = dict(ref.named_parameters())
    out = dict(five=np.array([float(t) for t in five]), seed=np.int64(seed),
               gradnorm=np.array([gr[k].grad.double().norm().item() for k in gr]))
    for k in ("resnet34_8s.conv1.weight", "resnet34_8s.fc.weight", "resnet34_8s.fc.bias",
              "resnet34_8s.layer4.0.downsample.1.weight", "resnet34_8s.layer1.2.bn2.bias"):
        out["grad:" + k] = gr[k].grad.numpy().copy()
    out["rs:resnet34_8s.bn1.running_mean"] = ref.state_dict()["resnet34_8s.bn1.running_mean"].numpy().copy()
    np.savez_compressed(os.path.join(GOLD, name + ".npz"), **out)
    print("wrote", name, "five", out["five"])


def _same(a, b, what):
    assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b), what


def reference_checks():
    """tests/golden/reference_checks.npz: the executed reference's results on every case of oracle/ref_cases.py (and the
    backbone modules on a small input), each required here to equal the restatement's bit-for-bit."""
    from oracle import ref_cases as RC
    ref = build_ref.load()
    out = {}
    # loss: every method, every composer branch
    r = RC.every_loss_method(ref.pcl.PixelwiseContrastiveLoss)
    o = RC.every_loss_method(LO.TorchPixelwiseContrastiveLoss)
    assert sorted(r) == sorted(o)
    for k in r:
        _same(o[k], r[k], k)
        out["method/" + k] = r[k]
    r = RC.composer_branches(ref.pcl.PixelwiseContrastiveLoss, ref.composer.get_loss, ref.dataset.SpartanDataset.empty_tensor)
    o = RC.composer_branches(LO.TorchPixelwiseContrastiveLoss, LO.get_loss, LO.empty_tensor)
    assert sorted(r) == sorted(o)
    for k in r:
        _same(o[k], r[k], k)
        out["composer/" + k] = r[k]
    for k in dir(ref.dataset.SpartanDatasetDataType):
        if k.isupper():
            out["datatype/" + k] = np.array(getattr(ref.dataset.SpartanDatasetDataType, k))
    # the non-match sampler: create_non_correspondences draws torch.rand(n) (mask branch) or torch.rand(2, n) (no mask), then two
    # more draws for the no-op perturbation -- it is given the uniforms the restatement takes as arguments
    H, W, k, ma, ru, rv, masks = RC.sampler_inputs()
    uv_a = (ma % W, ma // W)
    uv_b = ((ma % W).float(), (ma // W).float())
    n = len(ma) * k
    real_rand = ref.finder.torch.rand
    for i, m in enumerate(masks):
        calls = []

        def fake_rand(*shape):
            calls.append(shape)
            if len(calls) == 1:
                return ru.clone() if shape == (n,) else torch.stack((ru, rv)).clone()
            return torch.zeros(*shape)
        ref.finder.torch.rand = fake_rand
        try:
            uv_b_non = ref.finder.create_non_correspondences(uv_b, (H, W), num_non_matches_per_match=k, img_b_mask=m)
        finally:
            ref.finder.torch.rand = real_rand
        SD = ref.dataset.SpartanDataset
        uv_a_long, uv_b_long = SD.create_non_matches(None, uv_a, uv_b_non, k)
        na_r = SD.flatten_uv_tensor(uv_a_long, W).squeeze(1); nb_r = SD.flatten_uv_tensor(uv_b_long, W).squeeze(1)
        na_o, nb_o = LO.create_non_correspondences_flat(ma, (H, W), k, m, ru, rv)
        assert torch.equal(na_o, na_r) and torch.equal(nb_o, nb_r)
        out["sampler/%d/a" % i], out["sampler/%d/b" % i] = na_r.numpy(), nb_r.numpy()
    # the reprojection match finder: it first draws (and discards) rand(2, n) for unmasked candidates, then rand(n)
    da, pa, db, pb, mask, ru, K, n = RC.reprojection_scene()
    ref.finder.torch.rand = lambda *s: ru.clone() if s == (n,) else torch.zeros(*s)
    try:
        uv_a_r, uv_b_r = ref.finder.batch_find_pixel_correspondences(da, pa, db, pb, num_attempts=n, img_a_mask=mask, K=K)
    finally:
        ref.finder.torch.rand = real_rand
    for i, t in enumerate(uv_a_r + uv_b_r):
        out["reprojection/%d" % i] = t.numpy()
    # the backbone modules, train and eval, and the dilation bookkeeping the modern torchvision API gets differently
    D = 8
    oracle = seeded_oracle(D=D, seed=0)
    refnet = ref_loader.reference_resnet34_8s(D, oracle.state_dict())
    out["backbone/keys"] = np.array(list(refnet.state_dict().keys()))
    x = torch.randn(1, 3, 40, 56, generator=torch.Generator().manual_seed(2))
    for mode in ("train", "eval"):
        getattr(refnet, mode)(); getattr(oracle, mode)()
        with torch.no_grad():
            y = refnet(x)
            bit_equal(y, oracle(x), "backbone " + mode)
        out["backbone/" + mode] = y.numpy()
    r = refnet.resnet34_8s
    out["backbone/geometry"] = np.array([r.layer3[0].conv1.dilation[0], r.layer3[0].conv1.padding[0], r.layer4[0].conv1.dilation[0],
                                         r.layer4[0].downsample[0].stride[0], r.layer2[0].conv1.stride[0],
                                         r.layer2[0].downsample[0].stride[0]])
    np.savez_compressed(os.path.join(GOLD, "reference_checks.npz"), **out)
    print("wrote reference_checks", len(out), "arrays")


if __name__ == "__main__":
    assert ref_loader.reference_available() and build_ref.reference_available(), "set PDC_REFERENCE_ROOT to a checkout of the reference"
    build_ref.build()
    os.makedirs(GOLD, exist_ok=True)
    if sys.argv[1:] == ["reference_checks"]:      # only the cross-check file (the other goldens stay as they are)
        reference_checks()
        sys.exit(0)
    backbone_case("backbone_small_d3", D=3, B=2, H=64, W=96, seed_data=11)
    backbone_case("backbone_small_d16", D=16, B=1, H=48, W=64, seed_data=12)
    backbone_case("backbone_full_d3", D=3, B=1, H=480, W=640, seed_data=13)
    loss_case("loss_default_d3", 3, 48, 64, 50, 3, 2, 0, {}, 21)
    loss_case("loss_pixelw_blind_d8", 8, 48, 64, 40, 4, 4, 37,
              {"use_l2_pixel_loss_on_masked_non_matches": True, "use_l2_pixel_loss_on_background_non_matches": True,
               "M_pixel": 25, "M_masked": 0.7, "M_background": 0.4, "non_match_loss_weight": 2.0}, 22)
    loss_case("loss_noscale_d16", 16, 48, 64, 64, 2, 1, 5, {"scale_by_hard_negatives": False, "M_masked": 1.5,
                                                             "M_background": 1.2}, 23)
    train_step_case("train_step_small_d3", D=3, B=2, H=64, W=96, Nm=40, Nn=120, seed=31)
    reference_checks()
