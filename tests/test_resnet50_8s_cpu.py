"""CPU: the Resnet50_8s parameter layout, argument checking before any launch, the oracle against the outputs of the real
reference module (tests/golden/resnet50_8s_*.npz, oracle/make_golden_resnet50.py), and the decisive-bias certificate."""
import os

import numpy as np
import pytest
import torch

import pdc_b200
from pdc_b200 import _native as N
from oracle.resnet50_8s_oracle import decisive_biases, relu_margins, seeded_oracle, calibrated_state

A50 = N.ARCH_RESNET50_8S


@pytest.mark.parametrize("D", [3, 32])
def test_tables_are_reference_state_dict(D):
    o = seeded_oracle(D)
    learn = [(k, tuple(p.shape)) for k, p in o.named_parameters()]
    tab = N.param_table(D, A50)
    assert len(tab) == 161 and len(learn) == 161
    assert [("resnet50_8s." + n, s) for n, s, _, _ in tab] == learn
    offs = [o_ for _, _, o_, _ in tab]
    assert offs == sorted(offs) and all(o_ % 4 == 0 for o_ in offs)          # ordered, 16-byte aligned
    for (_, _, o1, n1), (_, _, o2, _) in zip(tab, tab[1:]):
        assert o1 + n1 <= o2
    assert N.lib.ddn_net_param_count(A50, D) >= offs[-1] + tab[-1][3]
    sd = o.state_dict()
    btab = N.buffer_table(A50)
    assert len(btab) == 106 == sum(1 for k in sd if "running" in k)
    for name, shape, _, _ in btab:
        assert tuple(sd["resnet50_8s." + name].shape) == shape
    assert len(sd) == 320
    # the largest weight, layer4.0.conv2 (3x3 512 -> 512), fits the tensor-core weight staging of 9 x 512 x 512 elements
    assert max(n for name, _, _, n in tab if name.endswith("weight") and not name.startswith("fc")) <= 9 * 512 * 512
    n_conv = sum(n for name, s, _, n in tab if len(s) == 4 and not name.startswith("fc"))
    assert round(n_conv / 1e6, 2) == 23.45


def test_module_aliases_flat_array_and_round_trips_state_dict():
    o = seeded_oracle(3)
    m = pdc_b200.Resnet50_8s(num_classes=3)
    sd = m.state_dict()
    assert list(sd) == list(o.state_dict())
    base = m._flat.data_ptr()
    for (_, _, off, _), p in zip(m._ptab, m.parameters()):
        assert p.data_ptr() == base + 4 * off
    m.load_state_dict(o.state_dict())
    for k, v in o.state_dict().items():
        assert torch.equal(m.state_dict()[k], v), k


def test_get_fcn_accepts_resnet50_and_refuses_others():
    cfg = {"descriptor_dimension": 3, "image_width": 96, "image_height": 64,
           "backbone": {"model_class": "Resnet", "resnet_name": "Resnet50_8s"}}
    fcn = pdc_b200.DenseCorrespondenceNetwork.get_fcn(cfg)
    assert isinstance(fcn, pdc_b200.Resnet50_8s) and fcn.num_classes == 3
    for name in ("Resnet101_8s", "Resnet18_8s", "Resnet50_16s", "math"):
        with pytest.raises(ValueError):
            pdc_b200.DenseCorrespondenceNetwork.get_fcn(dict(cfg, backbone={"model_class": "Resnet", "resnet_name": name}))


def test_queries_and_refusals_before_any_launch():
    for mode in (0, 1, 2):
        for prec in (0, 1, 2):
            assert N.lib.ddn_net_workspace_bytes(A50, 16, 480, 640, 3, mode, prec) > 0
    w34 = N.lib.ddn_net_workspace_bytes(N.ARCH_RESNET34_8S, 2, 480, 640, 3, 1, 1)
    assert w34 == N.lib.ddn_resnet34_8s_workspace_bytes(2, 480, 640, 3, 1, 1)
    assert N.lib.ddn_net_workspace_bytes(A50, 2, 480, 640, 3, 1, 1) > 2 * w34          # 3x the activations
    assert N.lib.ddn_net_workspace_bytes(A50, 1, 481, 640, 3, 1, 0) == 0
    assert N.lib.ddn_net_workspace_bytes(A50, 1, 480, 640, 33, 1, 0) == 0
    for bad in (-1, 2, 101):
        assert N.lib.ddn_net_workspace_bytes(bad, 1, 480, 640, 3, 1, 1) == 0
        assert N.lib.ddn_net_param_count(bad, 3) == N.lib.ddn_net_buffer_count(bad) == -1
        assert N.lib.ddn_net_param_table(bad, 3, None, 0) == N.lib.ddn_net_buffer_table(bad, None, 0) == -1
        assert N.lib.ddn_net_grad_buckets(bad, 3, None, 0) == -1
        assert N.lib.ddn_net_weight_cache_bytes(bad, 3) == 0
        assert N.lib.ddn_net_forward(bad, None, None, None, None, None, 0, 1, 480, 640, 3, 1, 1, 0.1, 1e-5, 1, None, None) == -1
    assert N.lib.ddn_net_forward(A50, None, None, None, None, None, 0, 1, 480, 640, 3, 1, 1, 0.1, 1e-5, 1, None, None) == -1
    assert N.lib.ddn_net_backward(A50, None, None, None, None, None, 0, 1, 480, 640, 3, 1, 1, 1e-5, 1, N.NO_BUCKET_CALLBACK,
                                  None, None) == -1
    assert N.lib.ddn_net_weight_cache_bytes(A50, 3) >= 8 * N.lib.ddn_net_param_count(A50, 3)


def test_grad_buckets_cover_the_parameters_in_completion_order():
    tab = N.param_table(3, A50)
    first = {n.split(".")[0]: o for n, _, o, _ in reversed(tab)}
    b = N.grad_buckets(3, A50)
    assert len(b) == 4
    assert [o for o, _ in b] == [first["layer4"], first["layer3"], first["layer2"], 0]
    assert b[0][0] + b[0][1] == N.lib.ddn_net_param_count(A50, 3)
    for (o1, _), (o2, n2) in zip(b, b[1:]):
        assert o2 + n2 == o1
    # Resnet34_8s keeps its buckets
    assert N.grad_buckets(3) == N.grad_buckets(3, N.ARCH_RESNET34_8S)


def test_decisive_bias_certificate_64x96():
    """On the inputs the GPU gradient tests use (seed 9, 2 images of 64x96), every float64 ReLU input of the decisive
    construction keeps a margin of at least 0.03 from zero in train mode (measured 0.035), and at least 0.02 in eval mode on
    running statistics calibrated over the same batch (measured 0.0207): the ReLU masks are the same in any arithmetic whose
    forward error is below that, so those tests gate a well-conditioned function."""
    x = torch.randn(2, 3, 64, 96, generator=torch.Generator().manual_seed(9)).double()
    o = decisive_biases(seeded_oracle(3)).double()
    state = {k: v.clone() for k, v in o.state_dict().items()}
    m = relu_margins(o.train(), x)
    assert len(m) == 49                      # stem + 16 blocks x 3
    assert min(lo for lo, _ in m) > 0.03
    o.load_state_dict(calibrated_state(state, 3, x))
    assert min(lo for lo, _ in relu_margins(o.eval(), x)) > 0.02


@pytest.mark.parametrize("name,B,H,W,backward", [("resnet50_8s_small_d3", 2, 64, 96, True), ("resnet50_8s_full_d3", 1, 480, 640, False)])
def test_oracle_matches_golden(golden_dir, name, B, H, W, backward):
    """The oracle (fp32, CPU) against the outputs the real reference Resnet50_8s stored (bit-equal where they were written)."""
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    state = decisive_biases(seeded_oracle(3)).state_dict()
    o = seeded_oracle(3)
    o.load_state_dict(state)
    gen = torch.Generator().manual_seed(int(g["x_seed"]))
    x = torch.randn(B, 3, H, W, generator=gen)
    sub = (lambda t: t) if backward else (lambda t: t[:, :, ::16, ::16])
    y = o.train()(x)
    np.testing.assert_allclose(sub(y.detach()).numpy(), g["y_train"], rtol=1e-4, atol=1e-5)
    sd = o.state_dict()
    for k in g.files:
        if k.startswith("rs:"):
            np.testing.assert_allclose(sd[k[3:]].numpy(), g[k], rtol=1e-4, atol=1e-6, err_msg=k)
    if backward:
        cot = torch.randn(y.shape, generator=gen)
        (y * cot).sum().backward()
        gr = dict(o.named_parameters())
        for k in g.files:
            if k.startswith("grad:"):
                np.testing.assert_allclose(gr[k[5:]].grad.numpy(), g[k], rtol=1e-3, atol=1e-6 * float(np.abs(g[k]).max()), err_msg=k)
        np.testing.assert_allclose([gr[k].grad.double().norm().item() for k in gr], g["gradnorm:all"], rtol=1e-3)
    o.load_state_dict({k: (torch.tensor(g["cal:" + k]) if "running" in k else v) for k, v in state.items()})
    with torch.no_grad():
        ye = o.eval()(x)
    np.testing.assert_allclose(sub(ye).numpy(), g["y_eval"], rtol=1e-4, atol=1e-5)
