"""GPU: Resnet34_8s forward / backward and the whole training step through the reference-facing Python API
against the CPU oracle (and the golden vectors written from the real reference).

Gates (BASELINE.json north_star): descriptors within 1e-3 relative fp32, scalar loss within 1e-4."""
import os

import numpy as np
import pytest
import torch

import pdc_b200
from pdc_b200 import loss_composer, synthetic, _native as N
from oracle import loss_oracle as LO
from oracle.resnet34_8s_oracle import decisive_biases, gate_param_grads, rel, seeded_oracle, process_network_output

pytestmark = pytest.mark.gpu
DEV = "cuda"
PRECISIONS = ["fp32"] + (["bf16x3"] if os.environ.get("DDN_TEST_TC", "1") == "1" else [])


def relmax(a, b):
    a = a.double().cpu(); b = b.double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def make_net(D, precision="fp32", oracle=None):
    oracle = oracle or seeded_oracle(D=D, seed=0)
    prec = {"fp32": N.PRECISION_FP32_SIMT, "bf16x3": N.PRECISION_BF16X3, "bf16": N.PRECISION_BF16}[precision]
    net = pdc_b200.Resnet34_8s(num_classes=D, precision=prec)
    net.load_state_dict(oracle.state_dict())
    return net.cuda(), oracle


def cuda_oracle_grads(D, x, cot):
    """PyTorch's own CUDA fp32 (cuDNN, TF32 off) run of the oracle: its distance from the CPU oracle is the noise
    floor of this network's gradients (ReLU / max-pool decisions flip on 1-ulp differences and train-mode BN amplifies
    them), so gradient gates are expressed relative to it instead of as an absolute number."""
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    o = seeded_oracle(D).train().cuda()
    y = o(x.to(DEV))
    (y * cot.to(DEV)).sum().backward()
    return {k: p.grad.detach().cpu() for k, p in o.named_parameters()}


def check_param_grads(net, ref_grads, floor_grads, factor=3.0, strict=2e-3, label="", precision="fp32"):
    """ref_grads: CPU-oracle (or golden) gradients; floor_grads: the cuDNN fp32 run of the same step.
    bf16x3 carries ~2^-17 per operand instead of 2^-24: its forward error is 5e-5..8e-5 (gate 1e-3), which the
    cancellation-heavy per-channel sums (BN beta/gamma gradients) amplify to ~1e-2 even where fp32 runs agree to
    1e-3, and the chaotic tensors land at up to ~5.2x the fp32 noise floor (measured on H100: layer1.2.bn2.bias of the
    train-step golden, whose ReLU decisions flip with the operand split; see DESIGN.md)."""
    if precision != "fp32":
        factor, strict = max(factor, 6.0), max(strict, 2e-2)
    worst = 0.0
    num = den = 0.0
    scale = max(float(r.double().norm()) for r in ref_grads.values())
    for k, p in net.named_parameters():
        if k not in ref_grads:
            continue
        r = ref_grads[k]
        if float(r.double().norm()) < 1e-5 * scale:
            # e.g. fc.bias under the contrastive loss: d/dA and d/dB cancel exactly in exact arithmetic, what is left is
            # rounding noise in every implementation -> only require it to stay negligible
            assert float(p.grad.double().norm()) < 1e-4 * scale, k
            continue
        e = rel(p.grad, r)
        floor = rel(floor_grads[k], r) if floor_grads is not None and k in floor_grads else 0.0
        assert e <= max(strict, factor * floor), "%s %s: rel err %.3e vs noise floor %.3e" % (label, k, e, floor)
        worst = max(worst, e)
        num += float((p.grad.double().cpu() - r.double()).norm() ** 2); den += float(r.double().norm() ** 2)
    return worst, (num / den) ** 0.5


WELL_CONDITIONED = ("resnet34_8s.fc.weight", "resnet34_8s.fc.bias")


def tc_or_skip(precision):
    if precision != "fp32" and N.lib.ddn_resnet34_8s_workspace_bytes(1, 64, 64, 3, 1, N.PRECISION_BF16X3) == 0:
        pytest.skip("tensor-core path not in this build")


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name,D,B,H,W", [("backbone_small_d3", 3, 2, 64, 96), ("backbone_small_d16", 16, 1, 48, 64)])
def test_backbone_small_vs_golden(golden_dir, precision, name, D, B, H, W):
    tc_or_skip(precision)
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    net, _ = make_net(D, precision)
    gen = torch.Generator().manual_seed(int(g["x_seed"]))
    x = torch.randn(B, 3, H, W, generator=gen)
    cot = torch.randn(B, D, H, W, generator=gen)
    net.train()
    y = net(x.to(DEV))
    assert y.shape == (B, D, H, W) and y.is_contiguous()
    tol = 1e-3
    assert rel(y, torch.tensor(g["y_train"])) < tol and relmax(y, torch.tensor(g["y_train"])) < tol
    sd = net.state_dict()
    for k in g.files:
        if k.startswith("rs:"):
            assert rel(sd[k[3:]], torch.tensor(g[k])) < 1e-3, k
    assert int(sd["resnet34_8s.bn1.num_batches_tracked"]) == 1
    (y * cot.to(DEV)).sum().backward()
    params = dict(net.named_parameters())
    golden_grads = {k[5:]: torch.tensor(g[k]) for k in g.files if k.startswith("grad:")}
    floor = cuda_oracle_grads(D, x, cot)
    check_param_grads(net, golden_grads, floor, label=name, precision=precision)
    for k in WELL_CONDITIONED:          # the last layer sees no ReLU/BN chaos: tight absolute gate
        assert rel(params[k].grad, golden_grads[k]) < (1e-4 if precision == "fp32" else 1e-3), k
    norms = np.array([float(p.grad.double().norm()) for _, p in net.named_parameters()])
    np.testing.assert_allclose(norms, g["gradnorm:all"], rtol=3e-2)
    net.eval()
    with torch.no_grad():
        ye = net(x.to(DEV))
    assert rel(ye, torch.tensor(g["y_eval"])) < tol
    assert int(net.state_dict()["resnet34_8s.bn1.num_batches_tracked"]) == 1     # eval does not count


@pytest.mark.parametrize("precision", PRECISIONS)
def test_backbone_full_size_vs_golden_and_oracle(golden_dir, precision):
    """640x480, D=3: the golden sub-sampled descriptors (from the real reference) and the full oracle output."""
    tc_or_skip(precision)
    g = np.load(os.path.join(golden_dir, "backbone_full_d3.npz"))
    net, oracle = make_net(3, precision)
    gen = torch.Generator().manual_seed(int(g["x_seed"]))
    x = torch.randn(1, 3, 480, 640, generator=gen)
    cot = torch.randn(1, 3, 480, 640, generator=gen)
    net.train(); oracle.train()
    y = net(x.to(DEV))
    assert rel(y[:, :, ::16, ::16], torch.tensor(g["y_train"])) < 1e-3
    y_or = oracle(x)
    assert rel(y, y_or.detach()) < 1e-3 and relmax(y, y_or.detach()) < 1e-3
    (y * cot.to(DEV)).sum().backward()
    params = dict(net.named_parameters())
    (y_or * cot).sum().backward()
    oracle_grads = {k: p.grad for k, p in oracle.named_parameters()}
    floor = cuda_oracle_grads(3, x, cot)
    worst, agg = check_param_grads(net, oracle_grads, floor, label="full", precision=precision)
    print("full-size gradients: worst per-tensor rel err %.2e, aggregate %.2e" % (worst, agg))
    for k in g.files:                   # and the committed sub-set written from the real reference
        if k.startswith("grad:"):
            assert rel(oracle_grads[k[5:]], torch.tensor(g[k])) < 1e-4, k
    for k in WELL_CONDITIONED:
        assert rel(params[k].grad, oracle_grads[k]) < (1e-4 if precision == "fp32" else 1e-3), k
    norms = np.array([float(p.grad.double().norm()) for _, p in net.named_parameters()])
    np.testing.assert_allclose(norms, g["gradnorm:all"], rtol=3e-2)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_train_step_small_vs_golden(golden_dir, precision):
    """fwd(A), fwd(B), loss_composer.get_loss, backward -- exactly the calls of training.py:329-345 -- on a
    batch of 2 pairs; golden written from the real reference backbone + restated loss."""
    tc_or_skip(precision)
    g = np.load(os.path.join(golden_dir, "train_step_small_d3.npz"))
    D, B, H, W = 3, 2, 64, 96
    cfg = {"descriptor_dimension": D, "image_width": W, "image_height": H}
    dcn = pdc_b200.DenseCorrespondenceNetwork.from_config(cfg, load_stored_params=False)
    assert dcn.training and next(dcn.parameters()).is_cuda
    dcn.fcn.precision = {"fp32": 0, "bf16x3": 1}[precision]
    dcn.fcn.load_state_dict(seeded_oracle(D).state_dict())
    data = synthetic.make_pair_batch(B, H, W, 40, 120, 120, 0, seed=int(g["seed"]))
    d = {k: (v.to(DEV) if v is not None else None) for k, v in data.items()}
    pcl = pdc_b200.PixelwiseContrastiveLoss(image_shape=dcn.image_shape, config=dict(LO.DEFAULT_LOSS_CONFIG))
    opt = torch.optim.Adam(dcn.parameters(), lr=1e-4, weight_decay=1e-4)
    opt.zero_grad()
    pa = dcn.process_network_output(dcn.forward(d["img_a"]), B)
    pb = dcn.process_network_output(dcn.forward(d["img_b"]), B)
    blind = loss_composer.empty_tensor().to(DEV)
    five = loss_composer.get_loss(pcl, torch.tensor([0, 0]), pa, pb, d["matches_a"], d["matches_b"], d["masked_a"],
                                  d["masked_b"], d["background_a"], d["background_b"], blind, blind)
    got = np.array([float(t) for t in five])
    np.testing.assert_allclose(got, g["five"], rtol=1e-4, atol=1e-7)
    five[0].backward()
    params = dict(dcn.fcn.named_parameters())
    # noise floor for this step: the oracle on CUDA (cuDNN fp32) with the restated loss
    torch.backends.cudnn.allow_tf32 = False
    o = seeded_oracle(D).train().cuda()
    pcl_o = LO.TorchPixelwiseContrastiveLoss([H, W], dict(LO.DEFAULT_LOSS_CONFIG))
    ya, yb = o(d["img_a"]), o(d["img_b"])
    five_o = LO.batched_within_scene_loss(pcl_o, process_network_output(ya, B, D, H, W),
                                          process_network_output(yb, B, D, H, W), d)
    five_o[0].backward()
    floor = {k: p.grad.detach().cpu() for k, p in o.named_parameters()}
    golden_grads = {k[5:]: torch.tensor(g[k]) for k in g.files if k.startswith("grad:")}
    check_param_grads(dcn.fcn, golden_grads, floor, strict=5e-3, label="train_step", precision=precision)
    assert rel(params["resnet34_8s.fc.weight"].grad, golden_grads["resnet34_8s.fc.weight"]) < (2e-4 if precision == "fp32" else 2e-3)
    assert rel(dcn.state_dict()["_fcn.resnet34_8s.bn1.running_mean"], torch.tensor(g["rs:resnet34_8s.bn1.running_mean"])) < 1e-3
    before = dcn.fcn.flat_parameters.clone()
    opt.step()                                      # Adam updates the views == the flat array the kernels read
    assert float((dcn.fcn.flat_parameters - before).abs().max()) > 0
    assert int(dcn.state_dict()["_fcn.resnet34_8s.bn1.num_batches_tracked"]) == 2


def test_single_image_inference_and_state_dict_roundtrip(tmp_path):
    D = 3
    net, oracle = make_net(D)
    dcn = pdc_b200.DenseCorrespondenceNetwork(net, D, image_width=96, image_height=64)
    dcn.eval(); oracle.eval()
    x = torch.randn(3, 64, 96, generator=torch.Generator().manual_seed(4))
    res = dcn.forward_single_image_tensor(x)
    assert res.shape == (64, 96, D)
    with torch.no_grad():
        ref = oracle(x.unsqueeze(0))[0].permute(1, 2, 0)
    assert rel(res, ref) < 1e-3
    uv, diff, nd = dcn.find_best_match((10, 20), res.detach().cpu().numpy(), res.detach().cpu().numpy())
    assert uv == (10, 20) and diff == 0.0 and nd.shape == (64, 96)
    f = tmp_path / "000001.pth"
    torch.save(dcn.state_dict(), f)
    assert all(k.startswith("_fcn.resnet34_8s.") for k in dcn.state_dict())
    cfg = {"descriptor_dimension": D, "image_width": 96, "image_height": 64}
    import yaml
    (tmp_path / "training.yaml").write_text(yaml.safe_dump({"dense_correspondence_network": cfg}))
    dcn2 = pdc_b200.DenseCorrespondenceNetwork.from_model_folder(str(tmp_path))
    dcn2.eval()
    assert rel(dcn2.forward_single_image_tensor(x), res) < 1e-3          # default arithmetic: bf16x3 on the tensor cores
    dcn2.fcn.precision = N.PRECISION_FP32_SIMT
    assert torch.equal(dcn2.forward_single_image_tensor(x), res)
    # a reference-style checkpoint (keys without the _fcn. prefix) loads through the fallback of net.py:429-433
    torch.save(oracle.state_dict(), tmp_path / "000002.pth")
    dcn3 = pdc_b200.DenseCorrespondenceNetwork.from_model_folder(str(tmp_path), iteration=2)
    dcn3.eval()
    dcn3.fcn.precision = N.PRECISION_FP32_SIMT
    assert torch.equal(dcn3.forward_single_image_tensor(x), res)


def test_contract_errors_on_gpu():
    net, _ = make_net(3)
    with pytest.raises(RuntimeError):
        net(torch.zeros(1, 3, 60, 80, device=DEV))                  # not multiples of 8
    with pytest.raises(RuntimeError):
        net(torch.zeros(1, 3, 64, 64, device=DEV, dtype=torch.float16))
    with pytest.raises(RuntimeError):
        net(torch.zeros(1, 4, 64, 64, device=DEV))
    with pytest.raises(NotImplementedError):
        net(torch.zeros(1, 3, 64, 64, device=DEV), feature_alignment=True)
    with pytest.raises(RuntimeError):
        net(torch.zeros(3, 3, 64, 64, device=DEV), bn_groups=2)     # groups must divide the batch
    net.eval()
    with torch.no_grad():
        y = net(torch.zeros(1, 3, 64, 64, device=DEV))
    assert not y.requires_grad                                       # inference: folded BatchNorm, nothing kept
    for p in net.parameters():
        p.requires_grad_(False)
    y = net(torch.zeros(1, 3, 64, 64, device=DEV))
    assert not y.requires_grad                                       # all parameters frozen: nothing to differentiate


def test_fused_adam_matches_torch_adam():
    """ddn_adam_step vs torch.optim.Adam(lr=1e-4, weight_decay=1e-4) (training.py:133-145) over 3 steps with a decaying lr."""
    D = 3
    net_a, _ = make_net(D)
    net_b, _ = make_net(D)
    ref = torch.optim.Adam(net_a.parameters(), lr=1e-4, weight_decay=1e-4)
    ours = pdc_b200.FusedAdam(net_b, lr=1e-4, weight_decay=1e-4)
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(1, 3, 64, 96, generator=gen).to(DEV); cot = torch.randn(1, D, 64, 96, generator=gen).to(DEV)
    for it in range(3):
        for opt, net in ((ref, net_a), (ours, net_b)):
            opt.zero_grad()
            (net(x) * cot).sum().backward()
            opt.param_groups[0]["lr"] = 1e-4 * (0.9 ** it)
        # identical gradients by construction: copy so that only the optimizer arithmetic is compared
        net_b.flat_gradient.copy_(net_a.flat_gradient)
        ref.step(); ours.step()
        a, b = net_a.flat_parameters, net_b.flat_parameters
        assert float((a - b).abs().max()) <= 2e-7 + 1e-6 * float(a.abs().max()), it
    # checkpoints are exchanged in torch.optim.Adam's own format (training.py:509-511 writes NNNNNN.pth.opt)
    sd, ref_sd = ours.state_dict(), ref.state_dict()
    assert len(sd["state"]) == len(ref_sd["state"]) == len(list(net_b.parameters()))
    for i in (0, 7, len(sd["state"]) - 1):
        assert float(sd["state"][i]["step"]) == 3.0 and sd["state"][i]["exp_avg"].shape == ref_sd["state"][i]["exp_avg"].shape
        for k in ("exp_avg", "exp_avg_sq"):
            a, b = sd["state"][i][k], ref_sd["state"][i][k]
            assert float((a - b).abs().max()) <= 1e-3 * float(b.abs().max()) + 1e-20, (i, k)
    resumed = pdc_b200.FusedAdam(net_b, lr=1.0)
    resumed.load_state_dict(ref_sd)
    assert resumed.step_count == 3 and resumed.param_groups[0]["lr"] == ref.param_groups[0]["lr"]


def test_weight_pack_cache_follows_parameter_updates():
    """The tensor-core weight packs are cached across calls; any parameter write (optimizer, load_state_dict, FusedAdam,
    a second module reusing freed addresses) must invalidate them."""
    D = 3
    x = torch.randn(1, 3, 64, 96, generator=torch.Generator().manual_seed(8)).to(DEV)
    net, oracle = make_net(D, "bf16x3")
    net.eval(); oracle.eval()
    with torch.no_grad():
        y0 = net(x).clone()
        assert rel(y0, oracle(x.cpu())) < 1e-3
        assert torch.equal(net(x), y0)                       # cached packs, same result
        for p in net.parameters():                           # in-place update through the views (what optimizers do)
            p.mul_(1.01)
        for p in oracle.parameters():
            p.mul_(1.01)
        y1 = net(x)
        assert rel(y1, oracle(x.cpu())) < 1e-3 and not torch.equal(y1, y0)
    del net
    net2, oracle2 = make_net(D, "bf16x3")                    # new module, very likely the same device addresses
    net2.eval(); oracle2.eval()
    with torch.no_grad():
        assert rel(net2(x), oracle2(x.cpu())) < 1e-3
    opt = pdc_b200.FusedAdam(net2, lr=1e-2)
    net2.train()
    (net2(x) ** 2).sum().backward()
    opt.step()                                               # raw-pointer write
    net2.eval()
    with torch.no_grad():
        ya = net2(x)
        net2.precision = N.PRECISION_FP32_SIMT               # the fp32 path never uses the cache: must agree
        yb = net2(x)
    assert rel(ya, yb) < 1e-3


# ----------------------------------------------------------------------------------------------------
# Whole-network gradients on decisive BatchNorm biases (oracle.resnet34_8s_oracle.decisive_biases): every ReLU decision is the
# same in every arithmetic, so every parameter gradient is a well-conditioned function of weights and inputs and is gated per
# tensor against float64.  DECISIVE_AMP: the bias magnitude at these sizes (tests/test_oracle_cpu.py checks its ReLU margin).
DECISIVE_AMP = 8.0


def _double_copy(oracle):
    ref64 = seeded_oracle(D=oracle.resnet34_8s.fc.out_channels, seed=0).double()
    ref64.load_state_dict({k: v.double() if v.is_floating_point() else v for k, v in oracle.state_dict().items()})
    return ref64


def _well_conditioned_case(precision, mode, D, B, H, W, seed):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 3, H, W, generator=gen)
    cot = torch.randn(B, D, H, W, generator=gen)
    oracle = decisive_biases(seeded_oracle(D=D, seed=0), amp=DECISIVE_AMP)
    if mode == "eval":      # frozen statistics that actually normalise: one pass with momentum 1 copies the batch statistics
        bns = [m for m in oracle.modules() if isinstance(m, torch.nn.BatchNorm2d)]
        for m in bns:
            m.momentum = 1.0
        oracle.train()
        with torch.no_grad():
            oracle(x)
        for m in bns:
            m.momentum = 0.1
    net, _ = make_net(D, precision, oracle)
    ref64 = _double_copy(oracle)
    for m in (oracle, net, ref64):
        m.train(mode == "train")
    y = net(x.to(DEV))
    y64 = ref64(x.double())
    assert rel(y, y64.detach()) < (2e-5 if precision == "fp32" else 1e-3)
    (y * cot.to(DEV)).sum().backward()
    (y64 * cot.double()).sum().backward()
    y32 = oracle(x); (y32 * cot).sum().backward()      # the fp32 CPU oracle's own distance from fp64: the conditioning certificate
    g64 = {k: p.grad for k, p in ref64.named_parameters()}
    scale = max(float(v.norm()) for v in g64.values())
    cert = max(rel(p.grad, g64[k]) for k, p in oracle.named_parameters() if float(g64[k].norm()) >= 1e-6 * scale)
    assert cert < 1e-4, "gradients should be well conditioned here (fp32 oracle vs fp64: %.2e)" % cert
    worst, _ = gate_param_grads({k: p.grad for k, p in net.named_parameters()}, g64, 2e-4 if precision == "fp32" else 1e-3,
                                    "%s %s-mode" % (precision, mode))
    return worst, cert, net, oracle, y, cot


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("mode", ["train", "eval"])
@pytest.mark.parametrize("D,B,H,W", [(3, 2, 64, 96), (8, 1, 120, 160)])
def test_whole_network_gradients_well_conditioned(precision, mode, D, B, H, W):
    """EVERY parameter gradient of the whole chain (conv fwd / dgrad / wgrad incl. the stride-2 and 1x1 convs, BatchNorm
    backward with batch statistics, residual adds, max-pool, fc, upsample) gated TIGHTLY per tensor against the oracle in fp64.
    The usual obstacle -- ReLU / max-pool decisions that flip on 1-ulp differences give this randomly initialised network a
    1e-2 gradient noise floor even between PyTorch's own CPU and CUDA runs -- is removed by making the ReLU decisions
    decisive (oracle.resnet34_8s_oracle.decisive_biases), NOT by loosening the gate; the fp32 CPU oracle's own distance from
    fp64 is asserted as the conditioning certificate (< 1e-4).  train: batch statistics (the training path).  eval: frozen
    running statistics -- the reference backpropagates through an eval()-mode network via autograd, here DDN_MODE_EVAL_SAVE."""
    tc_or_skip(precision)
    worst, cert, net, oracle, y, cot = _well_conditioned_case(precision, mode, D, B, H, W, seed=77)
    print("well-conditioned whole-net gradients [%s, %s-mode BN, D=%d]: worst per-tensor rel err %.2e (fp32 CPU oracle vs fp64: %.1e)"
          % (precision, mode, D, worst, cert))
    sd = net.state_dict(); so = oracle.state_dict()
    if mode == "eval":      # running statistics untouched by an eval-mode forward + backward
        assert torch.equal(sd["resnet34_8s.bn1.running_mean"].cpu(), so["resnet34_8s.bn1.running_mean"])
    else:
        assert rel(sd["resnet34_8s.layer4.2.bn2.running_var"], so["resnet34_8s.layer4.2.bn2.running_var"]) < 1e-4
    with pytest.raises(RuntimeError):          # a second backward through the same graph is refused with a clear message
        (y * cot.to(DEV)).sum().backward()


@pytest.mark.parametrize("precision", PRECISIONS)
def test_forward_pair_gradients_well_conditioned(precision):
    """bn_groups = 2: forward_pair(A, B) on decisive biases against two float64 oracle calls (A, then B), backward of
    (ya*ca + yb*cb).sum().  Every parameter gradient per tensor, the descriptors of both groups and every running statistic
    after the A-then-B update.  B is drawn with a different mean and scale than A, so a kernel that normalises, masks or
    back-propagates one group with the other group's statistics moves the result far beyond the gates."""
    tc_or_skip(precision)
    torch.cuda.reset_peak_memory_stats()
    D, B, H, W = 3, 2, 64, 96
    gen = torch.Generator().manual_seed(78)
    xa = torch.randn(B, 3, H, W, generator=gen); xb = 0.5 + 1.5 * torch.randn(B, 3, H, W, generator=gen)
    ca = torch.randn(B, D, H, W, generator=gen); cb = torch.randn(B, D, H, W, generator=gen)
    oracle = decisive_biases(seeded_oracle(D=D, seed=0), amp=DECISIVE_AMP)
    dcn = pdc_b200.DenseCorrespondenceNetwork.from_config({"descriptor_dimension": D, "image_width": W, "image_height": H},
                                                          load_stored_params=False)
    dcn.fcn.precision = {"fp32": N.PRECISION_FP32_SIMT, "bf16x3": N.PRECISION_BF16X3}[precision]
    dcn.fcn.load_state_dict(oracle.state_dict())
    dcn.train()
    ya, yb = dcn.forward_pair(xa.to(DEV), xb.to(DEV))
    ((ya * ca.to(DEV)).sum() + (yb * cb.to(DEV)).sum()).backward()
    refs = []
    for ref in (_double_copy(oracle), oracle):          # float64: the reference; fp32: the conditioning certificate
        dt = next(ref.parameters()).dtype
        ref.train()
        ya_r, yb_r = ref(xa.to(dt)), ref(xb.to(dt))
        ((ya_r * ca.to(dt)).sum() + (yb_r * cb.to(dt)).sum()).backward()
        refs.append((ya_r.detach(), yb_r.detach(), {k: p.grad for k, p in ref.named_parameters()}, ref.state_dict()))
    (ya64, yb64, g64, s64), (_, _, g32, _) = refs
    scale = max(float(v.norm()) for v in g64.values())
    cert = max(rel(g32[k], g64[k]) for k in g64 if float(g64[k].norm()) >= 1e-6 * scale)
    assert cert < 1e-4, "gradients should be well conditioned here (fp32 oracle vs fp64: %.2e)" % cert
    tol = 2e-5 if precision == "fp32" else 1e-3
    assert rel(ya, ya64) < tol and rel(yb, yb64) < tol
    worst, worst_stem = gate_param_grads({k: p.grad for k, p in dcn.fcn.named_parameters()}, g64,
                                             2e-4 if precision == "fp32" else 1e-3, "forward_pair %s" % precision)
    sd = dcn.fcn.state_dict()
    worst_rs = 0.0
    for k, v in s64.items():
        if "running" in k:
            e = rel(sd[k], v)
            assert e < 1e-4, "%s: rel err %.3e" % (k, e)
            worst_rs = max(worst_rs, e)
        elif "tracked" in k:
            assert int(sd[k]) == 2, k
    print("forward_pair whole-net gradients [%s]: worst per-tensor rel err %.2e (stem %.2e), running statistics %.2e "
          "(fp32 CPU oracle vs fp64: %.1e); peak device memory %.2f GB"
          % (precision, worst, worst_stem, worst_rs, cert, torch.cuda.max_memory_allocated() / 1e9))


@pytest.mark.parametrize("precision", PRECISIONS)
def test_forward_pair_equals_two_forward_calls(precision):
    """forward_pair(A, B) == (forward(A), forward(B)): per-group BatchNorm statistics, running statistics updated A-then-B,
    and one backward producing the sum of the two calls' gradients."""
    tc_or_skip(precision)
    D, B, H, W = 3, 2, 64, 96
    cfg = {"descriptor_dimension": D, "image_width": W, "image_height": H}
    oracle = seeded_oracle(D=D, seed=0)
    gen = torch.Generator().manual_seed(5)
    xa = torch.randn(B, 3, H, W, generator=gen).to(DEV); xb = (0.5 + 1.5 * torch.randn(B, 3, H, W, generator=gen)).to(DEV)
    ca = torch.randn(B, D, H, W, generator=gen).to(DEV); cb = torch.randn(B, D, H, W, generator=gen).to(DEV)
    outs = []
    for pair in (False, True):
        dcn = pdc_b200.DenseCorrespondenceNetwork.from_config(cfg, load_stored_params=False)
        dcn.fcn.precision = {"fp32": N.PRECISION_FP32_SIMT, "bf16x3": N.PRECISION_BF16X3}[precision]
        dcn.fcn.load_state_dict(oracle.state_dict())
        dcn.train()
        if pair:
            ya, yb = dcn.forward_pair(xa, xb)
        else:
            ya, yb = dcn.forward(xa), dcn.forward(xb)
        ((ya * ca).sum() + (yb * cb).sum()).backward()
        outs.append((ya.detach(), yb.detach(), {k: p.grad.detach().clone() for k, p in dcn.fcn.named_parameters()},
                     {k: v.detach().clone() for k, v in dcn.fcn.state_dict().items() if "running" in k or "tracked" in k}))
    (ya0, yb0, g0, s0), (ya1, yb1, g1, s1) = outs
    tol = 1e-5 if precision == "fp32" else 2e-4
    assert rel(ya1, ya0) < tol and rel(yb1, yb0) < tol
    for k in s0:
        if "tracked" in k:
            assert int(s0[k]) == int(s1[k]) == 2, k
        else:
            assert rel(s1[k], s0[k]) < 1e-5, k
    # gradients: the same function evaluated with different tile shapes / summation orders; compare against the two-call
    # run relative to the train-mode noise floor (see check_param_grads) -- and tightly on the well-conditioned last layer
    for k in ("resnet34_8s.fc.weight",):
        assert rel(g1[k], g0[k]) < (1e-4 if precision == "fp32" else 1e-3), k
    num = sum(float((g1[k].double() - g0[k].double()).norm() ** 2) for k in g0)
    den = sum(float(g0[k].double().norm() ** 2) for k in g0)
    assert (num / den) ** 0.5 < (2e-2 if precision == "fp32" else 5e-2)


def test_bench_configuration_parity():
    """The configuration bench.py times (configs[1]: 8 pairs, D=3, 640x480, 1000 matches + 1000 + 1000 non-matches per pair,
    train-mode BN, fwd A + fwd B + get_loss + backward, bf16x3) against the CPU oracle on the same inputs:
    descriptors 1e-3 (north_star), loss 1e-4 (north_star), fc gradients 1e-3 -- through both the two-call API and forward_pair."""
    tc_or_skip("bf16x3")
    D, B, H, W = 3, 8, 480, 640
    oracle = seeded_oracle(D=D, seed=0).train()
    data = synthetic.make_pair_batch(B, H, W, 1000, 1000, 1000, 0, seed=1)
    pcl_o = LO.TorchPixelwiseContrastiveLoss([H, W], dict(LO.DEFAULT_LOSS_CONFIG))
    ya_o, yb_o = oracle(data["img_a"]), oracle(data["img_b"])
    five_o = LO.batched_within_scene_loss(pcl_o, process_network_output(ya_o, B, D, H, W), process_network_output(yb_o, B, D, H, W), data)
    five_o[0].backward()
    go = {k: p.grad for k, p in oracle.named_parameters()}
    d = {k: (v.to(DEV) if v is not None else None) for k, v in data.items()}
    blind = loss_composer.empty_tensor().to(DEV)
    for pair in (False, True):
        dcn = pdc_b200.DenseCorrespondenceNetwork.from_config({"descriptor_dimension": D, "image_width": W, "image_height": H},
                                                              load_stored_params=False)
        dcn.fcn.precision = N.PRECISION_BF16X3
        dcn.fcn.load_state_dict(seeded_oracle(D=D, seed=0).state_dict())
        dcn.train()
        pcl = pdc_b200.PixelwiseContrastiveLoss(dcn.image_shape, dict(LO.DEFAULT_LOSS_CONFIG))
        if pair:
            a, b = dcn.forward_pair(d["img_a"], d["img_b"])
        else:
            a, b = dcn.forward(d["img_a"]), dcn.forward(d["img_b"])
        five = loss_composer.get_loss(pcl, torch.zeros(B, dtype=torch.int64), dcn.process_network_output(a, B),
                                      dcn.process_network_output(b, B), d["matches_a"], d["matches_b"], d["masked_a"], d["masked_b"],
                                      d["background_a"], d["background_b"], blind, blind)
        five[0].backward()
        e_a, e_b = rel(a.detach(), ya_o.detach()), rel(b.detach(), yb_o.detach())
        e_loss = abs(float(five[0]) - float(five_o[0])) / abs(float(five_o[0]))
        params = dict(dcn.fcn.named_parameters())
        e_fc = rel(params["resnet34_8s.fc.weight"].grad, go["resnet34_8s.fc.weight"])
        print("bench-config parity [%s]: descriptors %.2e / %.2e, loss %.2e (%.6f vs %.6f), fc.weight grad %.2e"
              % ("forward_pair" if pair else "two calls", e_a, e_b, e_loss, float(five[0]), float(five_o[0]), e_fc))
        assert e_a < 1e-3 and e_b < 1e-3 and e_loss < 1e-4 and e_fc < 1e-3
        for i in range(1, 5):
            assert abs(float(five[i]) - float(five_o[i])) <= 1e-4 * max(1.0, abs(float(five_o[i])))
        del dcn, a, b, five
        torch.cuda.empty_cache()


@pytest.mark.parametrize("D", [8, 16])
def test_full_size_forward_other_descriptor_dimensions(D):
    """640x480 forwards at the descriptor dimensions of configs[2] (D=16) and configs[4] (D=8), train and eval mode."""
    tc_or_skip("bf16x3")
    net, oracle = make_net(D, "bf16x3")
    x = torch.randn(1, 3, 480, 640, generator=torch.Generator().manual_seed(40 + D))
    net.train(); oracle.train()
    y = net(x.to(DEV)); y_o = oracle(x)
    assert rel(y, y_o.detach()) < 1e-3 and relmax(y, y_o.detach()) < 1e-3
    net.eval(); oracle.eval()
    with torch.no_grad():
        ye = net(x.to(DEV)); ye_o = oracle(x)
    assert rel(ye, ye_o) < 1e-3 and relmax(ye, ye_o) < 1e-3


def test_step_with_fused_upsample_loss_equals_generic_path():
    """forward_pair + get_loss + backward with the loss fused into the upsample (the network's own outputs) vs the generic
    full-resolution gather (copies of them, which carry no low-resolution map): same loss, same parameter gradients (fc
    tightly; all within the train-mode noise floor)."""
    tc_or_skip("bf16x3")
    D, B, H, W = 3, 2, 64, 96
    data = synthetic.make_pair_batch(B, H, W, 40, 120, 120, 0, seed=31)
    d = {k: (v.to(DEV) if v is not None else None) for k, v in data.items()}
    blind = loss_composer.empty_tensor().to(DEV)
    outs = {}
    for fused in (True, False):
        dcn = pdc_b200.DenseCorrespondenceNetwork.from_config({"descriptor_dimension": D, "image_width": W, "image_height": H},
                                                              load_stored_params=False)
        dcn.fcn.load_state_dict(seeded_oracle(D=D, seed=0).state_dict())
        dcn.train()
        pcl = pdc_b200.PixelwiseContrastiveLoss(dcn.image_shape, dict(LO.DEFAULT_LOSS_CONFIG))
        a, b = dcn.forward_pair(d["img_a"], d["img_b"])
        pa, pb = dcn.process_network_output(a, B), dcn.process_network_output(b, B)
        assert (pdc_b200.resnet_dilated.lowres_of(pa) is not None)
        if not fused:
            pa, pb = pa.clone(), pb.clone()
            assert pdc_b200.resnet_dilated.lowres_of(pa) is None and pdc_b200.resnet_dilated.lowres_of(pb) is None
        five = loss_composer.get_loss(pcl, torch.zeros(B, dtype=torch.int64), pa, pb, d["matches_a"], d["matches_b"], d["masked_a"],
                                      d["masked_b"], d["background_a"], d["background_b"], blind, blind)
        five[0].backward()
        outs[fused] = ([float(t) for t in five], {k: p.grad.detach().clone() for k, p in dcn.fcn.named_parameters()})
    (f1, g1), (f0, g0) = outs[True], outs[False]
    for x, y in zip(f1, f0):
        assert abs(x - y) <= 2e-6 * max(1.0, abs(y))
    assert rel(g1["resnet34_8s.fc.weight"], g0["resnet34_8s.fc.weight"]) < 1e-4
    num = sum(float((g1[k].double() - g0[k].double()).norm() ** 2) for k in g0); den = sum(float(g0[k].double().norm() ** 2) for k in g0)
    assert (num / den) ** 0.5 < 1e-3


def test_weight_pack_cache_cannot_go_stale():
    """A parameter write that autograd's version counters do not see (``p.data.mul_``) must still reach the packed bf16
    weights the convolutions read: the library fingerprints the parameter array on the device at every forward."""
    tc_or_skip("bf16x3")
    net, oracle = make_net(3, "bf16x3")
    net.train()
    x = torch.randn(1, 3, 64, 96, generator=torch.Generator().manual_seed(3)).to(DEV)
    y0 = net(x).detach().clone()
    p = dict(net.named_parameters())["resnet34_8s.layer3.1.conv2.weight"]
    v0 = p._version
    p.data.add_(0.05 * torch.randn(p.shape, generator=torch.Generator().manual_seed(9)).to(DEV))   # (not a rescaling: train-mode BN would undo it)
    assert p._version == v0                     # invisible to the version counter: a version-keyed cache would miss this
    y1 = net(x).detach().clone()
    fresh = pdc_b200.Resnet34_8s(num_classes=3, precision=N.PRECISION_BF16X3).cuda()
    sd = {k: v.clone() for k, v in net.state_dict().items()}
    fresh.load_state_dict(oracle.state_dict())          # pristine running statistics, like `net` had before its forwards
    with torch.no_grad():
        dict(fresh.named_parameters())["resnet34_8s.layer3.1.conv2.weight"].copy_(sd["resnet34_8s.layer3.1.conv2.weight"])
    fresh.train()
    y_ref = fresh(x).detach()
    assert rel(y1, y_ref) < 1e-6, "stale packed weights in use"
    assert rel(y1, y0) > 1e-3
