"""GPU: every parameter gradient of the pair-batched training step at the size bench.py times -- 640x480, train-mode BatchNorm
in two groups (forward_pair), the fused-upsample loss -- gated per tensor against the same network in float64 on the GPU.

The BatchNorm biases come from oracle.resnet34_8s_oracle.decisive_biases, which makes the gradient a well-conditioned function
of weights and inputs as far as this size allows (see the comment above the test); the same oracle in fp32 (cuDNN, TF32 off)
is the conditioning certificate: every non-stem tensor of it has to lie within 1e-4 of float64 before the product gates mean
anything.  Two arms share one reference forward:
  cot        backward of (ya*ca + yb*cb).sum() -- reaches every kernel of the backward through the full-resolution cotangent;
  loss       get_loss through the loss fused with the upsample (the low-resolution gradient, launch_add_lowres_nhwc), against
             oracle.loss_oracle on the float64 descriptors.  scale_by_hard_negatives=False: that branch is continuous in the
             descriptors, whereas the 1/#hard-negatives scale jumps when one distance crosses the margin.
The references are computed first and kept on the host, so the float64 activations are freed before the product runs."""
import time

import pytest
import torch

import pdc_b200
from pdc_b200 import loss_composer, synthetic, resnet_dilated, _native as N
from oracle import loss_oracle as LO
from oracle.resnet34_8s_oracle import (STEM_PARAMS, decisive_biases, gate_param_grads, perturbed_relus, rel, seeded_oracle,
                                      process_network_output)

pytestmark = pytest.mark.gpu
DEV = "cuda"
H, W = 480, 640
ARMS = ("cot", "loss")


def relmax(a, b):
    a = a.double().cpu(); b = b.double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


@pytest.fixture
def exact_fp32_cudnn():
    """The fp32 certificate must be fp32: TF32 off for cuDNN and cuBLAS, restored afterwards."""
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def _loss_config():
    cfg = dict(LO.DEFAULT_LOSS_CONFIG)
    cfg["scale_by_hard_negatives"] = False
    return cfg


def _reference(state, dtype, D, d, ca, cb, noise=None):
    """Oracle in `dtype` on the GPU: forward(A), forward(B), then both arms' gradients from that one forward.  noise = (eps,
    seed): every ReLU input perturbed by a relative eps (perturbed_relus).  Everything it returns is on the host."""
    B = d["img_a"].shape[0]
    o = seeded_oracle(D=D, seed=0).to(DEV, dtype)
    o.load_state_dict(state)
    o.train()
    if noise is not None:
        perturbed_relus(o, *noise)
    params = [p for _, p in o.named_parameters()]
    names = [k for k, _ in o.named_parameters()]
    ya, yb = o(d["img_a"].to(dtype)), o(d["img_b"].to(dtype))
    g_cot = torch.autograd.grad((ya * ca.to(dtype)).sum() + (yb * cb.to(dtype)).sum(), params, retain_graph=True)
    pcl = LO.TorchPixelwiseContrastiveLoss([H, W], _loss_config())
    five = LO.batched_within_scene_loss(pcl, process_network_output(ya, B, D, H, W), process_network_output(yb, B, D, H, W), d)
    g_loss = torch.autograd.grad(five[0], params)
    out = {"ya": ya.detach().cpu(), "yb": yb.detach().cpu(), "five": [float(t.detach()) for t in five],
           "cot": {k: g.cpu() for k, g in zip(names, g_cot)}, "loss": {k: g.cpu() for k, g in zip(names, g_loss)},
           "running": {k: v.cpu() for k, v in o.state_dict().items() if "running" in k}}
    del o, params, ya, yb, five, g_cot, g_loss
    torch.cuda.empty_cache()
    return out


def _product(state, precision, D, d, ca, cb, arm):
    B = d["img_a"].shape[0]
    dcn = pdc_b200.DenseCorrespondenceNetwork.from_config({"descriptor_dimension": D, "image_width": W, "image_height": H},
                                                          load_stored_params=False)
    dcn.fcn.precision = {"fp32": N.PRECISION_FP32_SIMT, "bf16x3": N.PRECISION_BF16X3}[precision]
    dcn.fcn.load_state_dict(state)
    dcn.train()
    ya, yb = dcn.forward_pair(d["img_a"], d["img_b"])
    five = None
    if arm == "cot":
        ((ya * ca).sum() + (yb * cb).sum()).backward()
    else:
        pa, pb = dcn.process_network_output(ya, B), dcn.process_network_output(yb, B)
        assert resnet_dilated.lowres_of(pa) is not None and resnet_dilated.lowres_of(pb) is not None   # the fused loss is under test
        pcl = pdc_b200.PixelwiseContrastiveLoss(dcn.image_shape, _loss_config())
        blind = loss_composer.empty_tensor().to(DEV)
        five = loss_composer.get_loss(pcl, torch.zeros(B, dtype=torch.int64), pa, pb, d["matches_a"], d["matches_b"],
                                      d["masked_a"], d["masked_b"], d["background_a"], d["background_b"], blind, blind)
        five[0].backward()
        five = [float(t.detach()) for t in five]
    out = {"ya": ya.detach().cpu(), "yb": yb.detach().cpu(), "five": five,
           "grads": {k: p.grad.detach().cpu() for k, p in dcn.fcn.named_parameters()},
           "running": {k: v.detach().cpu() for k, v in dcn.fcn.state_dict().items() if "running" in k or "tracked" in k}}
    del dcn, ya, yb
    torch.cuda.empty_cache()
    return out


def _certificate(g32, g64):
    scale = max(float(v.double().norm()) for v in g64.values())
    return max(rel(g32[k], g64[k]) for k in g64 if k not in STEM_PARAMS and float(g64[k].double().norm()) >= 1e-6 * scale)


# At 640x480 decisive_biases cannot keep every ReLU input away from zero: the zero-padded borders of the convolutions turn the
# constant offsets of the identity chain into normalised outliers of up to |xhat| ~ 27, and amp >= 16, which would clear them,
# leaves the fp32 oracle 2.2e-4 from float64.  AMP = 5 is the one amp for every case here (of 5, 6 and 8 the only one whose
# certificate holds at 8+8: 6.2e-5; amp 6 gives 3.9e-3, amp 8 1.3e-4).  At amp 5 a few ReLU inputs lie within the bf16x3
# forward error of zero, and each one that flips moves the BatchNorm bias gradients of layer1..layer3, heavily cancelling sums,
# by ~1e-3.  Which ones flip depends on the summation order, so a fixed gate would pass or fail by luck.  The bf16x3 gradients
# are therefore gated at the larger of 1e-3 and FLOOR_FACTOR x the noise floor: the distance from float64 of the same oracle,
# in float64, with every ReLU input perturbed by a relative NOISE_EPS (perturbed_relus; the larger of two draws).  That level is
# certified by float64 alone.  Measured on an H100 80GB HBM3 at 700 W, 8+8 cotangent arm:
#   - the two noise draws put 7.8e-3 and 4.1e-3 into layer2.2.bn1.bias, and the bf16x3 product 4.1e-3;
#   - 80 of the 107 non-stem tensors have a floor above 1e-3 / FLOOR_FACTOR, and the product stays within 0.9x the floor;
#   - the fp32 CUDA-core product (a different kernel family, with ~100x rarer flips) stays at 5.8e-5 on the same
#     configuration, under a plain 2e-4 gate with no floor.
AMP = 5.0
NOISE_EPS, NOISE_SEEDS, FLOOR_FACTOR = 1e-5, (1, 2), 4.0


@pytest.mark.parametrize("precision,D,B,gate", [
    ("bf16x3", 3, 8, 1e-3),     # the benchmarked configuration: 8+8 images, D = 3
    ("fp32", 3, 8, 2e-4),       # the fp32 CUDA-core instrument on the same configuration
    ("bf16x3", 16, 2, 1e-3),    # a wider descriptor, 2+2 images
])
def test_training_step_gradients_vs_float64(exact_fp32_cudnn, precision, D, B, gate):
    if precision != "fp32" and N.lib.ddn_resnet34_8s_workspace_bytes(1, 64, 64, 3, 1, N.PRECISION_BF16X3) == 0:
        pytest.skip("tensor-core path not in this build")
    t0 = time.perf_counter()
    torch.cuda.reset_peak_memory_stats()
    data = synthetic.make_pair_batch(B, H, W, 1000, 1000, 1000, 0, seed=1)
    d = {k: (v.to(DEV) if v is not None else None) for k, v in data.items()}
    gen = torch.Generator().manual_seed(11)
    ca = torch.randn(B, D, H, W, generator=gen).to(DEV); cb = torch.randn(B, D, H, W, generator=gen).to(DEV)
    state = decisive_biases(seeded_oracle(D=D, seed=0), amp=AMP).state_dict()
    r64 = _reference(state, torch.float64, D, d, ca, cb)
    r32 = _reference(state, torch.float32, D, d, ca, cb)
    cert = {arm: _certificate(r32[arm], r64[arm]) for arm in ARMS}
    assert max(cert.values()) < 1e-4, "gradients should be well conditioned here (fp32 oracle vs fp64: %s)" % cert
    del r32
    floor = None
    if precision != "fp32":
        noisy = [_reference(state, torch.float64, D, d, ca, cb, noise=(NOISE_EPS, s)) for s in NOISE_SEEDS]
        floor = {arm: {k: max(rel(n[arm][k], r64[arm][k]) for n in noisy) for k in r64[arm]} for arm in ARMS}
        del noisy
    report = []
    for arm in ARMS:
        p = _product(state, precision, D, d, ca, cb, arm)
        # descriptors of both groups, and the running statistics after the A-then-B update
        for y, y64 in ((p["ya"], r64["ya"]), (p["yb"], r64["yb"])):
            assert rel(y, y64) < 2e-4 and relmax(y, y64) < 2e-4, (rel(y, y64), relmax(y, y64))
        worst_rs = 0.0
        for k, v in r64["running"].items():
            e = rel(p["running"][k], v)
            assert e < 1e-4, "%s: rel err %.3e" % (k, e)
            worst_rs = max(worst_rs, e)
        assert all(int(v) == 2 for k, v in p["running"].items() if "tracked" in k)
        if arm == "loss":
            for got, ref in zip(p["five"], r64["five"]):
                assert abs(got - ref) <= 1e-4 * max(1.0, abs(ref)), (p["five"], r64["five"])
        fl = floor[arm] if floor is not None else None
        worst, worst_stem = gate_param_grads(p["grads"], r64[arm], gate, arm + " arm", floor=fl, floor_factor=FLOOR_FACTOR)
        scale = max(float(v.double().norm()) for v in r64[arm].values())
        on_floor = [k for k in fl if k not in STEM_PARAMS and FLOOR_FACTOR * fl[k] > gate
                    and float(r64[arm][k].double().norm()) >= 1e-6 * scale] if fl is not None else []
        ratio = max((rel(p["grads"][k], r64[arm][k]) / fl[k] for k in on_floor), default=0.0)
        report.append("%s arm %.2e (stem %.2e; %d tensors gated on the noise floor, worst error/floor %.1f; certificate %.1e)"
                      % (arm, worst, worst_stem, len(on_floor), ratio, cert[arm]))
        del p
    torch.cuda.synchronize()
    print("training-size gradients [%s, D=%d, %d+%d images of %dx%d, amp %g]: worst per-tensor rel err %s; running statistics "
          "%.2e; %.0f s, peak device memory %.1f GB"
          % (precision, D, B, B, W, H, AMP, "; ".join(report), worst_rs, time.perf_counter() - t0,
             torch.cuda.max_memory_allocated() / 1e9))
