"""GPU: Resnet50_8s (Bottleneck [3, 4, 6, 3], 2048-channel trunk).

- every convolution shape the Bottleneck network adds, one operator at a time at its 640x480 bench size (16 images),
  tensor cores against the fp32 CUDA-core instrument;
- descriptors against the float64 oracle (small size and 640x480, train and eval), whole-network gradients against float64
  on the decisive construction (train, eval with gradients, forward_pair with two BatchNorm groups);
- consistency: forward_pair == two forwards, fused-upsample loss == generic loss, folded inference == eval with saved
  activations, bit-identical repeated training steps; D = 32 at 640x480 (the widest fc head); FusedAdam and the weight-pack
  cache on the new module."""
import os
import time

import numpy as np
import pytest
import torch

import pdc_b200
from pdc_b200 import loss_composer, ops, synthetic, _native as N
from oracle import loss_oracle as LO
from oracle.resnet50_8s_oracle import STEM_PARAMS, calibrated_state, decisive_biases, rel, seeded_oracle

pytestmark = pytest.mark.gpu
DEV = "cuda"
PREC = {"fp32": N.PRECISION_FP32_SIMT, "bf16x3": N.PRECISION_BF16X3, "bf16": N.PRECISION_BF16}
CONV_TOL = {"bf16x3": 2e-5, "bf16": 8e-3}

NEW_SHAPES = [
    # N, H, W, Cin, Cout, k, stride, pad, dil
    (16, 120, 160, 64, 64, 1, 1, 0, 1),       # layer1.0.conv1
    (16, 120, 160, 256, 64, 1, 1, 0, 1),      # layer1.1.conv1
    (16, 120, 160, 64, 256, 1, 1, 0, 1),      # layer1 conv3, layer1.0.downsample
    (16, 120, 160, 128, 128, 3, 2, 1, 1),     # layer2.0.conv2: stride-2 3x3 with Cin = 128 (128-wide wgrad tile, stride 2)
    (16, 120, 160, 256, 512, 1, 2, 0, 1),     # layer2.0.downsample: 1x1 stride 2
    (16, 60, 80, 512, 128, 1, 1, 0, 1),       # layer2 conv1
    (16, 60, 80, 128, 512, 1, 1, 0, 1),       # layer2 conv3
    (16, 60, 80, 512, 256, 1, 1, 0, 1),       # layer3.0.conv1
    (16, 60, 80, 256, 1024, 1, 1, 0, 1),      # layer3 conv3
    (16, 60, 80, 1024, 256, 1, 1, 0, 1),      # layer3 conv1
    (16, 60, 80, 512, 1024, 1, 1, 0, 1),      # layer3.0.downsample
    (16, 60, 80, 1024, 512, 1, 1, 0, 1),      # layer4.0.conv1
    (16, 60, 80, 512, 2048, 1, 1, 0, 1),      # layer4 conv3
    (16, 60, 80, 2048, 512, 1, 1, 0, 1),      # layer4 conv1
    (16, 60, 80, 1024, 2048, 1, 1, 0, 1),     # layer4.0.downsample
]


def _operands(case):
    n, h, w, cin, cout, k, s, p, d = case
    g = torch.Generator(device=DEV).manual_seed(sum(case))
    x = torch.randn(n, h, w, cin, generator=g, device=DEV)
    wt = torch.randn(cout, cin, k, k, generator=g, device=DEV) * (2.0 / (k * k * cin)) ** 0.5
    ho = (h + 2 * p - d * (k - 1) - 1) // s + 1
    wo = (w + 2 * p - d * (k - 1) - 1) // s + 1
    dy = torch.randn(n, ho, wo, cout, generator=g, device=DEV)
    return x, wt, dy


@pytest.mark.parametrize("case", NEW_SHAPES, ids=lambda c: "%dx%d_%d-%d_k%d_s%d" % (c[1], c[2], c[3], c[4], c[5], c[6]))
def test_new_conv_shapes_vs_fp32_instrument(case):
    t0 = time.perf_counter()
    n, h, w, cin, cout, k, s, p, d = case
    x, wt, dy = _operands(case)
    y32 = ops.conv2d_forward(x, wt, s, p, d, precision=N.PRECISION_FP32_SIMT)
    dx32, dw32 = ops.conv2d_backward(x, wt, dy, s, p, d, precision=N.PRECISION_FP32_SIMT)
    errs = []
    for name in ("bf16x3", "bf16"):
        y = ops.conv2d_forward(x, wt, s, p, d, precision=PREC[name])
        dx, dw = ops.conv2d_backward(x, wt, dy, s, p, d, precision=PREC[name])
        e = (rel(y, y32), rel(dx, dx32), rel(dw, dw32))
        assert max(e) < CONV_TOL[name], (name, e)
        errs.append(e)
        if name == "bf16x3":       # deterministic: a second call is bit-identical
            y2 = ops.conv2d_forward(x, wt, s, p, d, precision=PREC[name])
            dx2, dw2 = ops.conv2d_backward(x, wt, dy, s, p, d, precision=PREC[name])
            assert torch.equal(y, y2) and torch.equal(dx, dx2) and torch.equal(dw, dw2)
    torch.cuda.synchronize()
    print("conv %s: bf16x3 (fwd, dgrad, wgrad) %s, bf16 %s, %.1f s" % (case, ["%.1e" % v for v in errs[0]],
                                                                     ["%.1e" % v for v in errs[1]], time.perf_counter() - t0))


def _net(D, state, precision):
    m = pdc_b200.Resnet50_8s(num_classes=D).cuda()
    m.precision = PREC[precision]
    m.load_state_dict(state)
    return m


def _oracle64(D, state):
    o = seeded_oracle(D).to(DEV, torch.float64)
    o.load_state_dict(state)
    return o


@pytest.fixture
def exact_fp32_cudnn():
    """The fp32 certificates must be fp32: TF32 off for cuDNN and cuBLAS, restored afterwards."""
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


# Conditioning.  At the default init, train-mode BatchNorm over 2 images amplifies per-operation rounding ~500x: the fp32
# instrument lands 5e-5 from float64 and bf16x3 0.9e-3 to 1.2e-3, so a 1e-3 gate would pass or fail by luck.  The parity tests
# therefore run the decisive construction (decisive_biases).  Eval mode also needs running statistics that normalise: with the
# initial (0, 1) the smallest ReLU input is 8e-6 from zero, so eval cases run on statistics calibrated over the test batch
# (calibrated_state).  On the gradient tests' input (seed 9) the smallest float64 ReLU input is 0.035 from zero in train mode
# and 0.0207 in eval mode (asserted by test_resnet50_8s_cpu.py::test_decisive_bias_certificate_64x96); every gradient case
# also asserts its own certificate, the fp32 oracle within 1e-4 of float64.
def _decisive(D):
    return decisive_biases(seeded_oracle(D)).state_dict()


DESC_GATE = {"bf16x3": 1e-3, "fp32": 2e-5}


@pytest.mark.parametrize("H,W,B", [(64, 96, 2), (480, 640, 2)])
@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
def test_descriptors_vs_float64(H, W, B, precision):
    t0 = time.perf_counter()
    torch.cuda.reset_peak_memory_stats()
    D = 3
    state = _decisive(D)
    x = torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(7)).to(DEV)
    state_eval = calibrated_state(state, D, x.double())
    o = _oracle64(D, state)
    with torch.no_grad():
        y64_train = o.train()(x.double())
        rs64 = {k: v.clone() for k, v in o.state_dict().items() if "running" in k}
        o.load_state_dict(state_eval)
        y64_eval = o.eval()(x.double())
    del o
    m = _net(D, state, precision)
    with torch.no_grad():
        y_train = m.train()(x)
        sd = {k: v.clone() for k, v in m.state_dict().items()}
        m.load_state_dict(state_eval)
        y_eval = m.eval()(x)
    e = (rel(y_train, y64_train), rel(y_eval, y64_eval))
    assert max(e) < DESC_GATE[precision], e
    for k, v in rs64.items():
        assert rel(sd[k], v) < 1e-4, k
    torch.cuda.synchronize()
    print("descriptors [%s, %dx%d, B=%d]: train %.2e, eval %.2e; %.1f s, peak %.1f GB"
          % (precision, W, H, B, e[0], e[1], time.perf_counter() - t0, torch.cuda.max_memory_allocated() / 1e9))


@pytest.mark.parametrize("name,B,H,W", [("resnet50_8s_small_d3", 2, 64, 96), ("resnet50_8s_full_d3", 1, 480, 640)])
@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
def test_descriptors_vs_golden(golden_dir, name, B, H, W, precision):
    """Against the outputs of the real reference Resnet50_8s (oracle/make_golden_resnet50.py): train-mode descriptors and
    running statistics, then eval-mode descriptors on the stored calibrated running statistics."""
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    state = _decisive(3)
    x = torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(int(g["x_seed"]))).to(DEV)
    sub = (lambda t: t) if H * W <= 96 * 96 else (lambda t: t[:, :, ::16, ::16])
    m = _net(3, state, precision)
    with torch.no_grad():
        y = m.train()(x)
        sd = m.state_dict()
        for k in g.files:
            if k.startswith("rs:"):
                assert rel(sd[k[3:]], torch.tensor(g[k])) < 1e-4, k
        m.load_state_dict({k: (torch.tensor(g["cal:" + k]) if "running" in k else v) for k, v in state.items()})
        ye = m.eval()(x)
    e = (rel(sub(y), torch.tensor(g["y_train"])), rel(sub(ye), torch.tensor(g["y_eval"])))
    assert max(e) < DESC_GATE[precision], e
    print("golden %s [%s]: train %.2e, eval %.2e" % (name, precision, e[0], e[1]))


def _grads(state, D, x, cot, train, groups, dtype):
    """The oracle in `dtype` on the GPU: descriptors, parameter gradients and (train) the running statistics after the
    forward; groups = 2 runs the two halves of the batch as two forward calls (A, then B), like the reference's step."""
    o = seeded_oracle(D).to(DEV, dtype)
    o.load_state_dict(state)
    o.train(train)
    if groups == 2:
        B = x.shape[0] // 2
        y = torch.cat([o(x[:B].to(dtype)), o(x[B:].to(dtype))], 0)
    else:
        y = o(x.to(dtype))
    (y * cot.to(dtype)).sum().backward()
    running = {k: v.detach().clone() for k, v in o.state_dict().items() if "running" in k}
    return y.detach(), {k: p.grad.detach().clone() for k, p in o.named_parameters()}, running


# A plain per-tensor gate on the decisive construction: 1e-3 for bf16x3, as for Resnet34_8s (DESIGN section 2), 2e-4 for the
# fp32 instrument; STEM_PARAMS sit behind the 3x3/2 max-pool, whose ties cannot be made decisive: 2e-2.  Tensors that vanish
# in float64 must stay negligible in the product.  Pair mode feeds a shifted and rescaled image B, so that the two BatchNorm
# groups have different statistics, and checks every running statistic after the A-then-B update.
@pytest.mark.parametrize("mode", ["train", "eval_save", "pair"])
@pytest.mark.parametrize("precision,gate", [("bf16x3", 1e-3), ("fp32", 2e-4)])
def test_gradients_vs_float64_decisive(exact_fp32_cudnn, mode, precision, gate):
    D, B, H, W = 3, 2, 64, 96
    state = _decisive(D)
    gen = torch.Generator().manual_seed(9)
    x = torch.randn(B, 3, H, W, generator=gen).to(DEV)
    cot = torch.randn(B, D, H, W, generator=gen).to(DEV)
    if mode == "eval_save":
        state = calibrated_state(state, D, x.double())
    if mode == "pair":
        x = torch.cat([x[:1], 1.5 * x[1:] + 0.3], 0)
    train, groups = mode != "eval_save", 2 if mode == "pair" else 1
    y64, g64, rs64 = _grads(state, D, x, cot, train, groups, torch.float64)
    _, g32, _ = _grads(state, D, x, cot, train, groups, torch.float32)
    scale = max(float(v.norm()) for v in g64.values())
    live = [k for k in g64 if float(g64[k].norm()) >= 1e-6 * scale]
    cert = max(rel(g32[k], g64[k]) for k in live if k not in STEM_PARAMS)
    assert cert < 1e-4, "gradients should be well conditioned here (fp32 oracle vs float64: %.2e)" % cert
    m = _net(D, state, precision)
    m.train(train)
    if mode == "pair":
        dcn = pdc_b200.DenseCorrespondenceNetwork(m, D, image_width=W, image_height=H)
        ya, yb = dcn.forward_pair(x[:1], x[1:])
        y = torch.cat([ya, yb], 0)
    else:
        y = m(x)
    (y * cot).sum().backward()
    assert rel(y, y64) < DESC_GATE[precision]
    if train:
        sd = m.state_dict()
        for k, v in rs64.items():
            assert rel(sd[k], v) < 1e-4, k
    got = {k: p.grad for k, p in m.named_parameters()}
    worst = worst_stem = 0.0
    for k, r in g64.items():
        if k not in live:
            assert float(got[k].norm()) < 1e-4 * scale, "%s should vanish" % k
            continue
        e = rel(got[k], r)
        g = 2e-2 if k in STEM_PARAMS else gate
        assert e < g, "%s: rel err %.3e (gate %.0e)" % (k, e, g)
        if k in STEM_PARAMS:
            worst_stem = max(worst_stem, e)
        else:
            worst = max(worst, e)
    print("gradients [%s, %s]: worst per-tensor rel err %.2e (stem %.2e); certificate %.1e"
          % (precision, mode, worst, worst_stem, cert))


def _step_state(D):
    return seeded_oracle(D).state_dict()


def test_forward_pair_equals_two_forwards_and_fused_loss_equals_generic():
    D, B, H, W = 3, 2, 480, 640
    state = _step_state(D)
    data = synthetic.make_pair_batch(B, H, W, 500, 500, 500, 0, seed=3)
    d = {k: (v.to(DEV) if v is not None else None) for k, v in data.items()}
    m = _net(D, state, "bf16x3").train()
    dcn = pdc_b200.DenseCorrespondenceNetwork(m, D, image_width=W, image_height=H)
    pa, pb = dcn.forward_pair(d["img_a"], d["img_b"])
    m.load_state_dict(state)
    fa = dcn.forward(d["img_a"]); fb = dcn.forward(d["img_b"])
    assert rel(pa, fa) < 1e-6 and rel(pb, fb) < 1e-6
    pcl = pdc_b200.PixelwiseContrastiveLoss(dcn.image_shape, dict(LO.DEFAULT_LOSS_CONFIG))
    blind = loss_composer.empty_tensor().cuda()
    args = (d["matches_a"], d["matches_b"], d["masked_a"], d["masked_b"], d["background_a"], d["background_b"], blind, blind)
    fused = loss_composer.get_loss(pcl, torch.tensor([0]), dcn.process_network_output(pa, B), dcn.process_network_output(pb, B), *args)
    ca, cb = pa.detach().clone(), pb.detach().clone()      # untagged copies: the generic gather
    generic = loss_composer.get_loss(pcl, torch.tensor([0]), dcn.process_network_output(ca, B), dcn.process_network_output(cb, B), *args)
    for a, b in zip(fused, generic):
        assert abs(float(a) - float(b)) <= 1e-5 * max(1.0, abs(float(b)))


def test_folded_inference_equals_eval_save():
    D, B, H, W = 3, 2, 480, 640
    m = _net(D, _step_state(D), "bf16x3").eval()
    x = torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(4)).to(DEV)
    with torch.no_grad():
        y_fold = m(x)
    xs = x.clone().requires_grad_(True)       # a gradient is wanted: running statistics, activations kept, no folding
    y_save = m(xs)
    assert rel(y_fold, y_save.detach()) < 1e-5


def test_two_training_steps_bit_identical():
    D, B, H, W = 3, 4, 480, 640
    state = _step_state(D)
    data = synthetic.make_pair_batch(B, H, W, 500, 500, 500, 0, seed=8)
    d = {k: (v.to(DEV) if v is not None else None) for k, v in data.items()}
    outs = []
    for _ in range(2):
        m = _net(D, state, "bf16x3").train()
        dcn = pdc_b200.DenseCorrespondenceNetwork(m, D, image_width=W, image_height=H)
        pcl = pdc_b200.PixelwiseContrastiveLoss(dcn.image_shape, dict(LO.DEFAULT_LOSS_CONFIG))
        a, b = dcn.forward_pair(d["img_a"], d["img_b"])
        blind = loss_composer.empty_tensor().cuda()
        five = loss_composer.get_loss(pcl, torch.tensor([0]), dcn.process_network_output(a, B), dcn.process_network_output(b, B),
                                      d["matches_a"], d["matches_b"], d["masked_a"], d["masked_b"], d["background_a"],
                                      d["background_b"], blind, blind)
        five[0].backward()
        outs.append((five[0].detach().clone(), a.detach().clone(), m.flat_gradient.clone(),
                     {k: v.clone() for k, v in m.state_dict().items()}))
    (l1, a1, g1, s1), (l2, a2, g2, s2) = outs
    assert torch.equal(l1, l2) and torch.equal(a1, a2) and torch.equal(g1, g2)
    assert all(torch.equal(s1[k], s2[k]) for k in s1)


def test_d32_at_640x480_widest_head(exact_fp32_cudnn):
    """D = 32: the C = 2048 fc kernels at their largest ([32][2048] weights, chunked), forward and backward, against float64.
    The decisive construction is not certified at 640x480, so the feature gradient the fc hands back (seen through
    layer4.2.conv3's weight gradient) carries its own certificate: the fp32 oracle within 1e-4 of float64 there."""
    D, B, H, W = 32, 2, 480, 640
    state = _decisive(D)
    gen = torch.Generator().manual_seed(12)
    x = torch.randn(B, 3, H, W, generator=gen).to(DEV)
    cot = torch.randn(B, D, H, W, generator=gen).to(DEV)
    k4 = "resnet50_8s.layer4.2.conv3.weight"
    y64, g64, _ = _grads(state, D, x, cot, True, 1, torch.float64)
    _, g32, _ = _grads(state, D, x, cot, True, 1, torch.float32)
    cert = rel(g32[k4], g64[k4])
    assert cert < 1e-4, cert
    g64 = {k: g64[k] for k in ("resnet50_8s.fc.weight", "resnet50_8s.fc.bias", k4)}
    del g32
    m = _net(D, state, "bf16x3").train()
    y = m(x)
    (y * cot).sum().backward()
    got = dict(m.named_parameters())
    e = (rel(y, y64), rel(got["resnet50_8s.fc.weight"].grad, g64["resnet50_8s.fc.weight"]),
         rel(got["resnet50_8s.fc.bias"].grad, g64["resnet50_8s.fc.bias"]))
    assert max(e) < 1e-3, e
    # the feature gradient the fc hands to layer4: reaches every conv3 of layer4 through its weight gradient
    e4 = rel(got[k4].grad, g64[k4])
    assert e4 < 1e-3, e4
    print("D=32 head: descriptors %.2e, fc.weight grad %.2e, fc.bias grad %.2e, layer4.2.conv3 grad %.2e" % (e + (e4,)))


def test_fused_adam_and_weight_cache():
    D, B, H, W = 3, 2, 64, 96
    state = _step_state(D)
    x = torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(2)).to(DEV)
    m = _net(D, state, "bf16x3").train()
    ref = _net(D, state, "bf16x3").train()
    opt = pdc_b200.FusedAdam(m, lr=1e-3, weight_decay=1e-4)
    topt = torch.optim.Adam(ref.parameters(), lr=1e-3, weight_decay=1e-4)
    for it in range(3):
        for net, o in ((ref, topt), (m, opt)):
            o.zero_grad()
            net(x).square().mean().backward()
        # identical gradients by construction: copy so that only the optimizer arithmetic is compared
        m.flat_gradient.copy_(ref.flat_gradient)
        topt.step(); opt.step()
        a, b = ref.flat_parameters, m.flat_parameters
        assert float((a - b).abs().max()) <= 2e-7 + 1e-6 * float(a.abs().max()), it
    # the weight-pack cache cannot go stale: a write through .data is seen by the next forward
    ref.load_state_dict(m.state_dict())
    m.eval(); ref.eval()
    with torch.no_grad():
        y0 = m(x)
        w_m = getattr(m.resnet50_8s.layer4, "2").conv3.weight
        w_m.data.mul_(0.5)
        getattr(ref.resnet50_8s.layer4, "2").conv3.weight.data.copy_(w_m.data)
        y1, y1r = m(x), ref(x)
    assert not torch.equal(y0, y1)
    assert torch.equal(y1, y1r)


# ---- the fused epilogues at the 1024 / 2048-channel shapes, one operator at a time (bf16x3, two BatchNorm groups), each
# against float64 in two ways: the whole op, and the epilogue alone recomputed in float64 from what the kernel wrote
FUSED_SHAPES = [
    (16, 60, 80, 512, 2048, 1, 1, 0, 1),      # layer4 conv3: forward statistics over 2048 channels
    (16, 60, 80, 1024, 2048, 1, 1, 0, 1),     # layer4.0.downsample
    (16, 60, 80, 2048, 512, 1, 1, 0, 1),      # layer4 conv1: its data gradient carries the column sums of 2048 channels
    (16, 60, 80, 256, 1024, 1, 1, 0, 1),      # layer3 conv3
    (16, 60, 80, 1024, 256, 1, 1, 0, 1),      # layer3 conv1 (data gradient: 1024 channels)
]
G = 2


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _conv64(x, w, s, p, d):
    return torch.nn.functional.conv2d(_nchw(x).double(), w.double(), stride=s, padding=p, dilation=d).permute(0, 2, 3, 1)


def _group_stats(t, eps=1e-5):
    n = t.shape[0]
    v = t.double().reshape(G, -1, t.shape[-1])
    mean = v.mean(1)
    var = v.var(1, unbiased=False)
    return mean, 1.0 / torch.sqrt(var + eps), v.var(1, unbiased=True), n


@pytest.mark.parametrize("case", FUSED_SHAPES, ids=lambda c: "%dx%d_%d-%d" % (c[1], c[2], c[3], c[4]))
def test_fused_epilogues_wide_channels(case):
    n, h, w, cin, cout, k, s, p, d = case
    x, wt, dy = _operands(case)
    gen = torch.Generator(device=DEV).manual_seed(5)
    # training forward: raw + per-group statistics + running statistics (A then B)
    rm = torch.zeros(cout, device=DEV); rv = torch.ones(cout, device=DEV)
    raw, mean, invstd = ops.conv2d_bn_stats_forward(x, wt, s, p, d, bn_groups=G, running_mean=rm, running_var=rv)
    raw64 = _conv64(x, wt, s, p, d)
    assert rel(raw, raw64) < 2e-5
    m64, is64, uv64, _ = _group_stats(raw)                       # (b): from what the kernel wrote
    assert rel(mean, m64) < 2e-6 and rel(invstd, is64) < 2e-6
    rm64 = torch.zeros(cout, dtype=torch.float64, device=DEV); rv64 = torch.ones(cout, dtype=torch.float64, device=DEV)
    for g in range(G):
        rm64 = 0.9 * rm64 + 0.1 * m64[g]; rv64 = 0.9 * rv64 + 0.1 * uv64[g]
    assert rel(rm, rm64) < 2e-6 and rel(rv, rv64) < 2e-6
    ma, isa, _, _ = _group_stats(raw64)                          # (a): the whole op
    assert rel(mean, ma) < 2e-5 and rel(invstd, isa) < 2e-5
    # inference forward with eval BatchNorm, an addend and the ReLU folded in
    gamma = 1 + 0.1 * torch.randn(cout, generator=gen, device=DEV); beta = 0.5 * torch.randn(cout, generator=gen, device=DEV)
    rmean = 0.1 * torch.randn(cout, generator=gen, device=DEV); rvar = 0.5 + torch.rand(cout, generator=gen, device=DEV)
    add = torch.randn(raw.shape, generator=gen, device=DEV)
    y, _, _ = ops.conv2d_folded_forward(x, wt, gamma, beta, rmean, rvar, s, p, d, addend=add, relu=True)
    sc = gamma.double() / torch.sqrt(rvar.double() + 1e-5)
    y64 = torch.relu(raw64 * sc + (beta.double() - rmean.double() * sc) + add.double())
    assert rel(y, y64) < 2e-5
    # data gradient + the column sums of the BatchNorm backward that consumes it (ReLU mask recomputed from raw_in)
    raw_in = torch.randn(n, h, w, cin, generator=gen, device=DEV)
    mi, isi = (t.float() for t in _group_stats(raw_in)[:2])
    gi = 1 + 0.1 * torch.randn(cin, generator=gen, device=DEV); bi = 0.5 * torch.randn(cin, generator=gen, device=DEV)
    dx, dgamma, dbeta, sums = ops.conv2d_backward_data_bn_stats(wt, dy, raw_in, mi, isi, gi, bi, s, p, d)
    dx64 = torch.nn.grad.conv2d_input(_nchw(raw_in).shape, wt.double(), _nchw(dy).double(), stride=s, padding=p,
                                      dilation=d).permute(0, 2, 3, 1)
    assert rel(dx, dx64) < 2e-5
    xr = raw_in.reshape(G, -1, cin)
    xhat = (xr.double() - mi.double()[:, None]) * isi.double()[:, None]
    # the kernel's fmaf(raw - mean, gamma * invstd, beta) > 0: the fp32 operands, their product exact in float64
    mask = ((xr - mi[:, None]).double() * (gi * isi)[:, None].double() + bi.double()) > 0
    gg = dx.reshape(G, -1, cin).double() * mask
    s0, s1 = gg.sum(1), (gg * xhat).sum(1)
    assert rel(sums[:, 0], s0) < 2e-6 and rel(sums[:, 1], s1) < 2e-6
    assert rel(dbeta, s0.sum(0)) < 2e-6 and rel(dgamma, s1.sum(0)) < 2e-6
    # a second call is bit-identical
    dx2, dgamma2, dbeta2, sums2 = ops.conv2d_backward_data_bn_stats(wt, dy, raw_in, mi, isi, gi, bi, s, p, d)
    assert torch.equal(dx, dx2) and torch.equal(sums, sums2) and torch.equal(dgamma, dgamma2)
