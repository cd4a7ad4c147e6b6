"""CPU: the pieces of test_gpu_conv_exact.py that need no GPU -- the split-operand certificate, the float64 models against a
float32 convolution of integer data, and the coverage of the kernel paths by its case list at 132 SMs (an H100 SXM)."""
import pytest
import torch
import torch.nn.functional as F

import conv_exact_common as C


@pytest.mark.parametrize("density", [1.0, 0.5, 0.1])
def test_split_operands_are_on_the_grid(density):
    g = torch.Generator().manual_seed(7)
    x, h, l = C.draw((64, 257), "split", density, g, "cpu")
    C.certify_operand((x, h, l))
    assert set(h.unique().tolist()) <= {-1.0, 0.0, 1.0}
    steps = (l * 2 ** 10).abs()
    assert torch.equal(steps, steps.round()) and float(steps.max()) == 3.0
    assert torch.equal(l.sign(), h.sign() * (steps > 0))         # lo points away from zero, or is zero
    assert torch.equal(l[h == 0], torch.zeros_like(l[h == 0]))
    x, h, l = C.draw((64, 257), "integer", density, g, "cpu")
    C.certify_operand((x, h, l))
    assert set(x.unique().tolist()) <= {-2.0, -1.0, 0.0, 1.0, 2.0} and not l.any()


def test_lo_toward_zero_would_leave_the_grid():
    """why the split operands put lo on the far side: 1 - 3 * 2^-10 rounds to the bf16 value 1 - 2^-8"""
    x = torch.tensor([1 - 3 * 2.0 ** -10])
    hi, lo = C.split_bf16(x)
    assert float(hi) == 1 - 2.0 ** -8 and float(hi) != 1.0
    with pytest.raises(AssertionError):
        C.certify_operand((x, torch.ones(1), torch.tensor([-3 * 2.0 ** -10])))


def test_certificate_refuses_a_sum_past_2_22_steps():
    a = (torch.full((1, 1, 1, 4096), 2.0), torch.full((1, 1, 1, 4096), 2.0), torch.zeros(1, 1, 1, 4096))
    b = (torch.full((1, 4096, 1, 1), 2.0 ** 10), torch.full((1, 4096, 1, 1), 2.0 ** 10), torch.zeros(1, 4096, 1, 1))
    with pytest.raises(AssertionError, match="certificate"):
        C.Model(C.conv_fwd_fn(1, 0, 1), a, b, "integer")


SMALL = [
    # N, H, W, Cin, Cout, k, stride, pad, dil
    (2, 9, 11, 8, 12, 3, 1, 1, 1),
    (1, 12, 10, 4, 6, 3, 1, 2, 2),
    (2, 10, 12, 6, 8, 3, 2, 1, 1),
    (2, 10, 8, 8, 4, 1, 2, 0, 1),
]


@pytest.mark.parametrize("shape", SMALL, ids=[str(s) for s in SMALL])
def test_models_equal_a_float32_conv_of_integer_data(shape):
    n, h, w, cin, cout, k, s, p, d = shape
    g = torch.Generator().manual_seed(sum(shape))
    x = C.draw((n, h, w, cin), "integer", 1.0, g, "cpu")
    wt = C.draw((cout, cin, k, k), "integer", 1.0, g, "cpu")
    y32 = F.conv2d(C.nchw(x[0]), wt[0], None, s, p, d)
    ho, wo = y32.shape[2:]
    dy = C.draw((n, ho, wo, cout), "integer", 1.0, g, "cpu")
    fwd = C.Model(C.conv_fwd_fn(s, p, d), x, wt, "integer")
    assert torch.equal(fwd.of("bf16x3"), C.nhwc(y32)) and torch.equal(fwd.of("bf16"), C.nhwc(y32))
    xr = C.nchw(x[0]).clone().requires_grad_(True)
    wr = wt[0].clone().requires_grad_(True)
    F.conv2d(xr, wr, None, s, p, d).backward(C.nchw(dy[0]))
    dgrad = C.Model(C.conv_dgrad_fn((n, h, w, cin), s, p, d), dy, wt, "integer")
    wgrad = C.Model(C.conv_wgrad_fn((cout, cin, k, k), s, p, d), dy, x, "integer")
    assert torch.equal(dgrad.of("bf16x3"), C.nhwc(xr.grad))
    assert torch.equal(wgrad.of("bf16x3"), wr.grad)


def test_split_model_is_three_products():
    """bf16x3 = h*h + h*l + l*h (no l*l), bf16 = h*h, on a 1x1 conv small enough to sum by hand"""
    g = torch.Generator().manual_seed(3)
    x = C.draw((1, 2, 3, 16), "split", 0.7, g, "cpu")
    wt = C.draw((5, 16, 1, 1), "split", 0.7, g, "cpu")
    m = C.Model(C.conv_fwd_fn(1, 0, 1), x, wt, "split")
    xh, xl = x[1].double(), x[2].double()
    wh, wl = wt[1].double()[:, :, 0, 0], wt[2].double()[:, :, 0, 0]
    hh = torch.einsum("nhwc,oc->nhwo", xh, wh)
    x3 = hh + torch.einsum("nhwc,oc->nhwo", xh, wl) + torch.einsum("nhwc,oc->nhwo", xl, wh)
    assert torch.equal(m.of("bf16"), hh.float()) and torch.equal(m.of("bf16x3"), x3.float())
    assert not torch.equal(x3, torch.einsum("nhwc,oc->nhwo", xh + xl, wh + wl))   # the lo*lo term is really left out


def test_case_list_reaches_every_path_at_132_sms():
    seen, missed = C.coverage(132)
    assert not missed, missed
    assert C.REQUIRED <= seen, sorted(C.REQUIRED - seen)


def test_mirror_matches_the_documented_plans_at_132_sms():
    """a few plans the case list is built around, restated by hand"""
    w = C.worker_sms(132, 0)
    l4 = C.plans(C.BY_LABEL["layer4"], w)
    assert l4["fwd"]["kernel"] == "conv_tc_kernel<128>" and l4["fwd"]["num_kb"] == 72
    assert l4["fwd"]["full_items"] == 2400 - 24 and l4["fwd"]["tail_split"] == 4       # 2400 items, rem 24 -> 32-channel pieces
    l3 = C.plans(C.BY_LABEL["layer3"], w)
    assert l3["fwd"]["num_kb"] == 36 and l3["fwd"]["full_items"] == 1200 - 12 and l3["fwd"]["tail_split"] == 4
    assert C.reserved_for(C.BY_LABEL["tail64"], 132) > 0
    assert C.plans(C.BY_LABEL["wide_out"], w)["fwd"]["n_co"] == 16
    assert C.worker_sms(132, 130) == 8 and C.worker_sms(132, 8) == 124
    # the locator names the tail piece of the last item's channels
    loc = C.locate_conv(l4["fwd"], 15, 59, 79, 511)
    assert "tail piece" in loc and "channels 480..511" in loc
    halo = C.plans(C.BY_LABEL["halo_bench"], w)
    assert halo["wgrad"]["kernel"] == "wgrad64_halo_kernel" and halo["wgrad"]["n_tiles"] == 16 * 15 * 10
