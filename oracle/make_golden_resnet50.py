"""Pins oracle/resnet50_8s_oracle.py against the real reference Resnet50_8s and writes tests/golden/resnet50_8s_*.npz.

Needs a checkout of the reference (PDC_REFERENCE_ROOT=<dir>):   python oracle/make_golden_resnet50.py

The REAL reference module (oracle/ref_loader_resnet50.py) and the oracle run on the same weights and inputs and must agree
bit for bit: train-mode forward, running statistics, every parameter gradient (small case), and the eval-mode forward.  The
reference's outputs are what is stored.  The weights are the decisive construction (decisive_biases, amp 6, seed 5) on the
seeded oracle: at the default init a train-mode Resnet50_8s amplifies rounding ~500x, which would make the stored outputs
useless as a 1e-3 gate for the tensor-core product.  Eval mode runs on calibrated running statistics (one train-mode forward
over the same batch with momentum 1), stored as cal:<key>, for the same reason: the initial (0, 1) leaves a ReLU input 8e-6
from zero.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_loader_resnet50 as RL             # noqa: E402
from oracle.resnet50_8s_oracle import decisive_biases, seeded_oracle  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
torch.set_num_threads(os.cpu_count())
P = "resnet50_8s."
RUNNING = (P + "bn1.running_mean", P + "bn1.running_var", P + "layer1.0.downsample.1.running_var",
           P + "layer2.0.bn2.running_mean", P + "layer4.2.bn3.running_mean", P + "layer4.2.bn3.running_var")
GRADS = (P + "conv1.weight", P + "bn1.bias", P + "layer1.0.conv1.weight", P + "layer1.0.downsample.0.weight",
         P + "layer2.0.conv2.weight", P + "layer2.0.bn2.bias", P + "layer3.0.bn2.weight", P + "layer4.0.downsample.1.weight",
         P + "layer4.2.bn3.bias", P + "fc.weight", P + "fc.bias")


def bit_equal(a, b, what):
    assert a.shape == b.shape, what
    assert torch.equal(a, b), "%s: oracle != reference (max abs diff %g)" % (what, (a - b).abs().max().item())


def decisive_state(D):
    return decisive_biases(seeded_oracle(D=D, seed=0)).state_dict()


def case(name, D, B, H, W, seed_data, backward):
    state = decisive_state(D)
    oracle = seeded_oracle(D=D, seed=0)
    oracle.load_state_dict(state)
    ref = RL.reference_resnet50_8s(D, state)
    assert list(ref.state_dict().keys()) == list(oracle.state_dict().keys())
    g = torch.Generator().manual_seed(seed_data)
    x = torch.randn(B, 3, H, W, generator=g)
    sub = (lambda t: t) if H * W <= 96 * 96 else (lambda t: t[:, :, ::16, ::16])
    out = {"x_seed": np.int64(seed_data)}
    ref.train(); oracle.train()
    y_ref = ref(x); y_or = oracle(x)
    bit_equal(y_ref, y_or, name + " train fwd")
    out["y_train"] = sub(y_ref.detach()).numpy().copy()
    for k in RUNNING:
        bit_equal(ref.state_dict()[k], oracle.state_dict()[k], name + " " + k)
        out["rs:" + k] = ref.state_dict()[k].numpy().copy()
    if backward:                 # a backward through a fixed random cotangent drawn after x
        cot = torch.randn(y_ref.shape, generator=g)
        (y_ref * cot).sum().backward(); (y_or * cot).sum().backward()
        gr = dict(ref.named_parameters()); go = dict(oracle.named_parameters())
        for k in gr:
            bit_equal(gr[k].grad, go[k].grad, name + " grad " + k)
        for k in GRADS:
            out["grad:" + k] = gr[k].grad.numpy().copy()
        out["gradnorm:all"] = np.array([gr[k].grad.double().norm().item() for k in gr])
    # eval on running statistics calibrated over this batch
    for net in (ref, oracle):
        net.load_state_dict(state)
        for m in net.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.momentum = 1.0
        net.train()
        with torch.no_grad():
            net(x)
        net.eval()
    for k, v in ref.state_dict().items():
        if "running" in k:
            bit_equal(v, oracle.state_dict()[k], name + " calibrated " + k)
            out["cal:" + k] = v.numpy().copy()
    with torch.no_grad():
        ye_ref = ref(x); ye_or = oracle(x)
    bit_equal(ye_ref, ye_or, name + " eval fwd")
    out["y_eval"] = sub(ye_ref).numpy().copy()
    np.savez_compressed(os.path.join(GOLD, name + ".npz"), **out)
    print("wrote", name, os.path.getsize(os.path.join(GOLD, name + ".npz")), "bytes")


if __name__ == "__main__":
    assert RL.reference_available(), "set PDC_REFERENCE_ROOT to a checkout of the reference"
    os.makedirs(GOLD, exist_ok=True)
    case("resnet50_8s_small_d3", D=3, B=2, H=64, W=96, seed_data=11, backward=True)
    case("resnet50_8s_full_d3", D=3, B=1, H=480, W=640, seed_data=13, backward=False)
