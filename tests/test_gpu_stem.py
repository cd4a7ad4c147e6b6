"""GPU: the stem's forward tail and its whole backward, one operator at a time, against float64.

The stem is conv1 7x7/2 -> bn1 -> ReLU -> max-pool 3x3/2 pad 1.  conv1's forward and bn1's statistics are tested in
test_gpu_fused_epilogues.py (STEM_PARTIAL, STEM_BENCH).  This file covers what follows, through the C ABI entries that run
the network's own code (`ddn_stem_pool_forward`: `stem_bn_relu_pool_kernel`; `ddn_stem_backward`: engine.cu's
`stem_backward`, which `net_backward` calls too):

- pool forward: y against float64 within the rounding bound of the kernel's three fp32 operations, the bf16 planes
  bit-exact against the split of the kernel's own y, argmax exact in every window whose top two differ by more than 1e-5
  of the channel's std, all-zero windows on their first in-bounds element, and planted exact ties (padded borders
  included) on the first maximum, as torch;
- pool / ReLU backward (`stem_pool_relu_bwd_kernel`) fed the kernel's own argmax: relative 1e-6 per element;
- bn1's backward (C = 64, no ReLU, training and eval): dgamma / dbeta |d| / sum|terms| <= 1e-6, dx relative Frobenius 1e-5,
  the dx planes bit-exact;
- conv1's weight gradient (`tc_stem_wgrad` + the kind-1 `tc_unpack_wgrads` entry; the SIMT instrument's NHWC4 path) against
  float64 `conv2d_weight` at the conv gates, with SMs reserved at the bench shape, and bit-identical on a second call;
- the composed stem backward at the bench shape, starting from the stem's forward kernels.

Every gate's worst value is printed at the end of the module (run with -s).  On one H100 80GB HBM3 at 700 W the 55 tests
take about 5 s (16 s with the interpreter's start).  The bench-shape cases hold a few float64 copies of raw [16,240,320,64]
(629 MB each).
"""
import functools

import pytest
import torch
import torch.nn.functional as F

from pdc_b200 import ops, _native as N

pytestmark = pytest.mark.gpu
DEV = "cuda"
PREC = {"bf16x3": N.PRECISION_BF16X3, "bf16": N.PRECISION_BF16, "fp32": N.PRECISION_FP32_SIMT}
# the conv gates of the other tensor-core tests, except bf16x3: in training mode bn1's backward leaves dx with zero mean per
# channel and group, so conv1's weight gradient is a sum of 1.2 M terms of both signs at the bench shape (cancellation kappa
# ~ 400, against 9 in eval mode) accumulated in fp32 over ~28 k pixels per chunk; it lands at 3.5e-5 there (DESIGN.md §2)
WGRAD_TOL = {"bf16x3": 5e-5, "bf16": 8e-3, "fp32": 5e-6}
POOL_BWD_TOL = 1e-6        # |d g| / sum of |dy| scattered to that element
SUMS_TOL = 1e-6            # |d dgamma|, |d dbeta| over the sum of the magnitudes of their terms
DX_TOL = 1e-5              # bn1's dx, relative Frobenius
BN_PARAM_TOL = 1e-5        # composed chain: bn1.weight / bn1.bias gradients, relative Frobenius
DECISIVE = 1e-5            # a window's argmax is compared where its top two differ by more than this x the channel's std
U = 2.0 ** -24
EPS = 1e-5

# label, N, H, W (image; conv1's output raw is Hc x Wc = (H-1)//2+1 x (W-1)//2+1)
SMALL = ("small", 2, 64, 96)
PARTIAL = ("partial", 4, 488, 648)     # raw 244x324: partial 64-column patch tiles, W1 % 16 = 4
BENCH = ("bench", 16, 480, 640)        # what forward_pair runs at 8 pairs
ODD = ("odd", 2, 50, 74)               # raw 25x37: the last pool windows hang over the bottom and right edges
CASES = [SMALL, PARTIAL, BENCH, ODD]

WORST = {}                 # gate -> worst value seen in this session (DESIGN.md §2 records them)


def gate(name, err, tol):
    WORST[name] = max(WORST.get(name, 0.0), err)
    assert err <= tol, "%s: %.3e > %.1e" % (name, err, tol)


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    for k in sorted(WORST):
        print("stem gate %-46s worst %.3e" % (k, WORST[k]))


def rel(a, b):
    a = a.double(); b = b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def nchw(t):
    return t.permute(0, 3, 1, 2)


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def raw_hw(case):
    _, _, h, w = case
    return (h - 1) // 2 + 1, (w - 1) // 2 + 1


def pool_hw(hc, wc):
    return (hc - 1) // 2 + 1, (wc - 1) // 2 + 1


def groups(case):
    return [1, 2] if case[1] % 2 == 0 else [1]


def per_image(t, G, n):
    """[G, C] -> [N, 1, 1, C]: the row of each image's BatchNorm group"""
    return t.repeat_interleave(n // G, dim=0)[:, None, None, :]


def group_rows(t, G):
    return t.reshape(G, -1, t.shape[-1])


# ------------------------------------------------------------------------------------------------ operands
@functools.lru_cache(maxsize=1)
def operands(case, G):
    """raw with per-channel offsets and scales, group 1 shifted and scaled so that its statistics are clearly not group 0's;
    the float64 statistics per group (rounded to fp32, as the forward hands them on); gamma of both signs; beta near 0 and
    below it, so that many windows are all zero after the ReLU; frozen statistics for eval mode; the image x (nonzero at
    every border) and dy_pool (nonzero mean, so that the batch terms of bn1's backward matter)"""
    _, n, h, w = case
    hc, wc = raw_hw(case)
    hp, wp = pool_hw(hc, wc)
    g = torch.Generator(device=DEV).manual_seed(n * 1000 + h + w + G)
    raw = torch.randn(n, hc, wc, 64, generator=g, device=DEV) * (torch.rand(64, generator=g, device=DEV) + 0.5) \
        + torch.randn(64, generator=g, device=DEV)
    raw[n // 2:] = raw[n // 2:] * 1.7 + 0.8 if G == 2 else raw[n // 2:]
    r = group_rows(raw.double(), G)
    mu, var = r.mean(1), r.var(1, unbiased=False)
    mean = mu.float().contiguous()
    invstd = (1.0 / (var + EPS).sqrt()).float().contiguous()
    gamma = (torch.rand(64, generator=g, device=DEV) + 0.5) * torch.randn(64, generator=g, device=DEV).sign()
    beta = torch.randn(64, generator=g, device=DEV) * 0.8 - 0.3
    rm = torch.randn(64, generator=g, device=DEV) * 0.3
    rv = torch.rand(64, generator=g, device=DEV) + 0.5
    frozen_mean = rm.expand(G, 64).contiguous()
    frozen_invstd = (1.0 / (rv.double() + EPS).sqrt()).float().expand(G, 64).contiguous()
    x = torch.randn(n, 3, h, w, generator=g, device=DEV) + 0.2
    dy_pool = torch.randn(n, hp, wp, 64, generator=g, device=DEV) + 0.3
    return raw, mean, invstd, gamma, beta, frozen_mean, frozen_invstd, x, dy_pool


def bn_terms(raw, mean, invstd, gamma, beta, G):
    """float64 t = (raw - mean) * invstd * gamma and the BatchNorm output t + beta, from the fp32 inputs the kernel reads"""
    n = raw.shape[0]
    t = (raw.double() - per_image(mean, G, n).double()) * per_image(invstd, G, n).double() * gamma.double()
    return t, t + beta.double()


def windows(v_nhwc, fill):
    """[N,H,W,C] -> [N,C,9,Hp*Wp]: the 3x3/2 pad-1 pool windows, padding = fill, position r*3+s"""
    n, h, w, c = v_nhwc.shape
    p = F.pad(nchw(v_nhwc), (1, 1, 1, 1), value=fill)
    return F.unfold(p, 3, stride=2).reshape(n, c, 9, -1)


def from_windows(t, hp, wp):
    """[N,C,Hp*Wp] -> [N,Hp,Wp,C]"""
    n, c, _ = t.shape
    return t.reshape(n, c, hp, wp).permute(0, 2, 3, 1)


def first_inbounds(hp, wp):
    """window-local index of the first in-bounds element of every window [Hp, Wp, 1]"""
    r0 = (torch.arange(hp, device=DEV) == 0).long()
    s0 = (torch.arange(wp, device=DEV) == 0).long()
    return (r0[:, None] * 3 + s0[None, :])[:, :, None]


def scatter_to_argmax(v, argmax, hc, wc):
    """float64 sum of v [N,Hp,Wp,C] into the element each window's argmax names: [N,Hc,Wc,C]; asserts that nothing lands on
    the padding"""
    n, hp, wp, c = v.shape
    out = torch.zeros(n, 2 * hp + 1, 2 * wp + 1, c, dtype=torch.float64, device=DEV)
    a = argmax.long()
    for r in range(3):
        for s in range(3):
            out[:, r:r + 2 * hp:2, s:s + 2 * wp:2, :] += torch.where(a == r * 3 + s, v, torch.zeros_like(v))
    inner = out[:, 1:hc + 1, 1:wc + 1, :].clone()
    out[:, 1:hc + 1, 1:wc + 1, :] = 0
    assert float(out.abs().max()) == 0.0, "an argmax points at the padding"
    return inner


# ------------------------------------------------------------------------------------------------ pool forward
def check_pool_forward(case, G):
    raw, mean, invstd, gamma, beta = operands(case, G)[:5]
    n = raw.shape[0]
    hc, wc = raw_hw(case)
    hp, wp = pool_hw(hc, wc)
    y, y_hi, y_lo, argmax = ops.stem_pool_forward(raw, mean, invstd, gamma, beta, want_y=True, want_planes=True)
    t, lin = bn_terms(raw, mean, invstd, gamma, beta, G)
    relu = lin.clamp_min(0)
    # y: the kernel's fmaf((raw - mean)_f32, (gamma*invstd)_f32, beta) rounds three times: |d| <= u (2|t| + |lin|) per element,
    # and the max of a window is within the largest bound of its elements
    bound = windows(U * (2.001 * t.abs() + lin.abs()) + 1e-38, 0.0).amax(2)
    ref_w = windows(relu, float("-inf"))
    ref = from_windows(ref_w.amax(2), hp, wp)
    ref_mp = nhwc(F.max_pool2d(nchw(relu).contiguous(), 3, 2, 1))
    assert torch.equal(ref, ref_mp)
    gate("pool y / rounding bound", float(((y.double() - ref).abs() / from_windows(bound, hp, wp)).max()), 1.0)
    # planes: the round-to-nearest split of the kernel's own y
    hi_ref = y.to(torch.bfloat16)
    assert torch.equal(y_hi.view(torch.int16), hi_ref.view(torch.int16))
    assert torch.equal(y_lo.view(torch.int16), (y - hi_ref.float()).to(torch.bfloat16).view(torch.int16))
    y2, hi2, lo2, am2 = ops.stem_pool_forward(raw, mean, invstd, gamma, beta, want_y=False, want_planes=True, want_lo=False)
    assert y2 is None and lo2 is None and torch.equal(hi2.view(torch.int16), y_hi.view(torch.int16)) and torch.equal(am2, argmax)
    # argmax in decisive windows: the first maximum of float64 torch, both from max_pool2d's indices and from the windows
    top2 = ref_w.topk(2, dim=2).values
    std = gamma.double().abs()[None, :, None]
    decisive = from_windows((top2[:, :, 0] - top2[:, :, 1]) > DECISIVE * std, hp, wp)
    ref_k = from_windows(ref_w.argmax(2), hp, wp)
    _, idx = F.max_pool2d(nchw(relu).contiguous(), 3, 2, 1, return_indices=True)
    idx = nhwc(idx)
    hh = 2 * torch.arange(hp, device=DEV)[:, None, None] - 1 + ref_k // 3
    ww = 2 * torch.arange(wp, device=DEV)[None, :, None] - 1 + ref_k % 3
    assert torch.equal(torch.where(decisive, hh * wc + ww, 0), torch.where(decisive, idx, 0))
    am = argmax.long()
    assert torch.equal(torch.where(decisive, am, 0), torch.where(decisive, ref_k, 0))
    assert int(decisive.sum()) > 0.2 * decisive.numel()
    # windows whose every element is below zero by more than the rounding bound: all zero, argmax on the first in-bounds element
    neg = from_windows(windows(lin + U * (2.001 * t.abs() + lin.abs()), float("-inf")).amax(2) < 0, hp, wp)
    assert int(neg.sum()) > 0.02 * neg.numel()
    first = first_inbounds(hp, wp).expand(n, hp, wp, 64)
    assert torch.equal(torch.where(neg, am, 0), torch.where(neg, first, 0))
    assert float(torch.where(neg, y, torch.zeros_like(y)).abs().max()) == 0.0
    return y, argmax


@pytest.mark.parametrize("case,G", [pytest.param(c, G, id="%s-G%d" % (c[0], G)) for c in CASES for G in groups(c)])
def test_pool_forward(case, G):
    check_pool_forward(case, G)


@pytest.mark.parametrize("case", [SMALL, ODD, PARTIAL], ids=lambda c: c[0])
def test_pool_forward_exact_ties(case):
    """mean 0, invstd 1, gamma 1, beta 0: the BatchNorm is exact, so y = maxpool(relu(raw)) bit for bit; raw on a grid of 7
    integers plants exact ties inside windows, at the padded borders and in all-zero windows.  Every tie resolves to the first
    maximum in row-major order, as torch's max_pool2d does."""
    _, n, _, _ = case
    hc, wc = raw_hw(case)
    hp, wp = pool_hw(hc, wc)
    g = torch.Generator(device=DEV).manual_seed(hc * wc)
    raw = torch.randint(-3, 4, (n, hc, wc, 64), generator=g, device=DEV).float()
    raw[:, :, -1, ::2] = 3.0          # ties along the right and bottom edges, whose windows hang over the border
    raw[:, -1, :, 1::2] = 3.0
    raw[:, 0, 0, :] = 2.0
    z = torch.zeros(1, 64, device=DEV)
    one = torch.ones(64, device=DEV)
    y, _, _, argmax = ops.stem_pool_forward(raw, z, z + 1, one, torch.zeros(64, device=DEV))
    relu = raw.clamp_min(0)
    ref, idx = F.max_pool2d(nchw(relu.double()).contiguous(), 3, 2, 1, return_indices=True)
    assert torch.equal(y, nhwc(ref).float())
    ref_w = windows(relu.double(), float("-inf"))
    ref_k = from_windows(ref_w.argmax(2), hp, wp)          # torch.argmax: the first maximal value
    ties = from_windows((ref_w == ref_w.amax(2, keepdim=True)).sum(2) > 1, hp, wp)
    assert int(ties.sum()) > 0.3 * ties.numel()
    assert torch.equal(argmax.long(), ref_k)
    hh = 2 * torch.arange(hp, device=DEV)[:, None, None] - 1 + ref_k // 3
    ww = 2 * torch.arange(wp, device=DEV)[None, :, None] - 1 + ref_k % 3
    assert torch.equal(hh * wc + ww, nhwc(idx))


# ------------------------------------------------------------------------------------------------ backward, piece by piece
def backward_params():
    out = []
    for case in CASES:
        for G in groups(case):
            for prec in PREC:
                if prec == "fp32" and case not in (SMALL, PARTIAL):
                    continue
                for mode in ("train", "eval"):
                    out.append(pytest.param(case, G, prec, mode, id="%s-G%d-%s-%s" % (case[0], G, prec, mode)))
    return out


@functools.lru_cache(maxsize=1)
def kernel_argmax(case, G):
    raw, mean, invstd, gamma, beta = operands(case, G)[:5]
    return ops.stem_pool_forward(raw, mean, invstd, gamma, beta)[3]


def run_backward(case, G, prec, mode):
    raw, mean, invstd, gamma, beta, fmean, finvstd, x, dy_pool = operands(case, G)
    training = mode == "train"
    m, s = (mean, invstd) if training else (fmean, finvstd)
    return ops.stem_backward(x, raw, m, s, gamma, beta, kernel_argmax(case, G), dy_pool, training=training, want_g=True,
                             want_dx=True, want_planes=prec != "fp32", precision=PREC[prec])


def wgrad_ref(x, dx):
    return torch.nn.grad.conv2d_weight(x.double(), (64, 3, 7, 7), nchw(dx.double()), 2, 3)


def check_wgrad(name, dw, x, dx, tol):
    """relative Frobenius error against float64; also records the cancellation kappa = |W(|x|, |dx|)| / |W(x, dx)| and the
    error over |W(|x|, |dx|)|, which does not depend on it"""
    ref = wgrad_ref(x, dx)
    mag = wgrad_ref(x.abs(), dx.abs())
    e = rel(dw, ref)
    WORST["kappa " + name] = max(WORST.get("kappa " + name, 0.0), float(mag.norm() / ref.norm()))
    WORST["over magnitude " + name] = max(WORST.get("over magnitude " + name, 0.0), e * float(ref.norm() / mag.norm()))
    gate(name, e, tol)


def bn_backward_ref(g, raw, mean, invstd, gamma, G, training):
    """float64 bn1 backward of g: (dx, dgamma, dbeta, magnitude bounds of dgamma / dbeta)"""
    n = raw.shape[0]
    g = g.double()
    xhat = (raw.double() - per_image(mean, G, n).double()) * per_image(invstd, G, n).double()
    sg, sgx = group_rows(g, G).sum(1), group_rows(g * xhat, G).sum(1)              # [G, 64]
    bg, bgx = group_rows(g.abs(), G).sum(1).sum(0), group_rows((g * xhat).abs(), G).sum(1).sum(0)
    k1 = per_image(invstd, G, n).double() * gamma.double()
    if training:
        mg = g.numel() // (64 * G)
        dx = k1 * (g - per_image(sg, G, n) / mg - xhat * per_image(sgx, G, n) / mg)
    else:
        dx = k1 * g
    return dx, sgx.sum(0), sg.sum(0), bgx, bg


@pytest.mark.parametrize("case,G,prec,mode", backward_params())
def test_backward_pieces(case, G, prec, mode):
    raw, mean, invstd, gamma, beta, fmean, finvstd, x, dy_pool = operands(case, G)
    training = mode == "train"
    m, s = (mean, invstd) if training else (fmean, finvstd)
    hc, wc = raw_hw(case)
    argmax = kernel_argmax(case, G)
    dw, dgamma, dbeta, g, dx, dx_hi, dx_lo = run_backward(case, G, prec, mode)
    # pool / ReLU backward: scatter to the kernel's argmax, masked by the float64 BatchNorm output (elements within 1e-6 std
    # of zero are left out of the comparison)
    _, lin = bn_terms(raw, m, s, gamma, beta, G)
    std = gamma.double().abs()
    g_ref = scatter_to_argmax(dy_pool.double(), argmax, hc, wc) * (lin > 0)
    scale = scatter_to_argmax(dy_pool.double().abs(), argmax, hc, wc)
    keep = lin.abs() > 1e-6 * std
    gate("pool/relu backward", float(((g.double() - g_ref).abs() * keep / (scale + 1e-30)).max()), POOL_BWD_TOL)
    # bn1 backward of the kernel's own g (what the BatchNorm kernels read)
    dx_ref, dg_ref, db_ref, bg, bb = bn_backward_ref(g, raw, m, s, gamma, G, training)
    gate("bn dgamma |d|/sum|terms|", float(((dgamma.double() - dg_ref).abs() / (bg + 1e-30)).max()), SUMS_TOL)
    gate("bn dbeta |d|/sum|terms|", float(((dbeta.double() - db_ref).abs() / (bb + 1e-30)).max()), SUMS_TOL)
    gate("bn dx rel (%s)" % mode, rel(dx, dx_ref), DX_TOL)
    if prec != "fp32":                  # the planes the weight gradient reads: the round-to-nearest split of dx
        hi_ref = dx.to(torch.bfloat16)
        assert torch.equal(dx_hi.view(torch.int16), hi_ref.view(torch.int16))
        if prec == "bf16x3":
            assert torch.equal(dx_lo.view(torch.int16), (dx - hi_ref.float()).to(torch.bfloat16).view(torch.int16))
    # conv1 weight gradient of the kernel's own dx against float64
    check_wgrad("conv1 wgrad rel %s %s" % (prec, mode), dw, x, dx, WGRAD_TOL[prec])
    if case is BENCH and mode == "train":
        again = run_backward(case, G, prec, mode)
        for a, b in zip((dw, dgamma, dbeta, g, dx), again[:5]):
            assert torch.equal(a, b)


def wgrad_chunks(tiles, total_kb, workers):
    """conv_tc.cu tc_wgrad_chunks"""
    even = tiles * total_kb / workers
    best, best_span = 1, float("inf")
    for s in range(1, max(1, total_kb // 4) + 1):
        span = -(-s * tiles // workers) * -(-total_kb // s)
        if span <= 1.02 * even:
            return s
        if span < best_span:
            best, best_span = s, span
    return best


@pytest.mark.parametrize("prec", ["bf16x3", "bf16"])
def test_wgrad_with_reserved_sms(prec):
    """Fewer persistent workers: tc_wgrad_chunks picks another chunk count S for the stem's 3 tiles; same gate."""
    case, G = BENCH, 2
    _, n, _, _ = case
    hc, wc = raw_hw(case)
    total_kb = n * -(-hc // 4) * -(-wc // 16)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    s0 = wgrad_chunks(3, total_kb, sms)
    r = next(r for r in range(8, 65) if wgrad_chunks(3, total_kb, sms - r) != s0)
    assert N.lib.ddn_set_reserved_sms(r) == 0
    try:
        dw, _, _, _, dx, _, _ = run_backward(case, G, prec, "train")
    finally:
        assert N.lib.ddn_set_reserved_sms(0) == 0
    print("stem wgrad: S = %d on %d SMs, %d with %d reserved" % (s0, sms, wgrad_chunks(3, total_kb, sms - r), r))
    check_wgrad("conv1 wgrad rel %s (reserved SMs)" % prec, dw, operands(case, G)[7], dx, WGRAD_TOL[prec])


# ------------------------------------------------------------------------------------------------ composed, bench shape
@pytest.mark.parametrize("prec", ["bf16x3", "bf16"])
def test_composed_stem_backward(prec):
    """conv2d_bn_stats_forward (the stem) -> ddn_stem_pool_forward -> ddn_stem_backward against a float64 chain that starts
    from the forward kernels' raw and statistics (their error is gated in test_gpu_fused_epilogues.py) and routes the pool
    gradient through the kernel's argmax: the op-level counterpart of the whole-network 2e-2 stem gate."""
    _, n, h, w = BENCH
    G = 2
    g = torch.Generator(device=DEV).manual_seed(7)
    x = torch.randn(n, 3, h, w, generator=g, device=DEV) + 0.2
    wt = torch.randn(64, 3, 7, 7, generator=g, device=DEV) * (2.0 / 147) ** 0.5
    gamma = (torch.rand(64, generator=g, device=DEV) + 0.5) * torch.randn(64, generator=g, device=DEV).sign()
    beta = torch.randn(64, generator=g, device=DEV) * 0.5
    raw, mean, invstd = ops.conv2d_bn_stats_forward(x, wt, 2, 3, 1, bn_groups=G, precision=PREC[prec])
    _, y_hi, _, argmax = ops.stem_pool_forward(raw, mean, invstd, gamma, beta, want_y=False, want_planes=True,
                                               want_lo=prec == "bf16x3")
    hc, wc = raw.shape[1:3]
    dy_pool = torch.randn(*y_hi.shape, generator=g, device=DEV) + 0.3
    dw, dgamma, dbeta, _, _, _, _ = ops.stem_backward(x, raw, mean, invstd, gamma, beta, argmax, dy_pool, precision=PREC[prec])
    _, lin = bn_terms(raw, mean, invstd, gamma, beta, G)
    g64 = scatter_to_argmax(dy_pool.double(), argmax, hc, wc) * (lin > 0)
    dx64, dg64, db64, _, _ = bn_backward_ref(g64, raw, mean, invstd, gamma, G, True)
    check_wgrad("composed conv1.weight rel " + prec, dw, x, dx64, WGRAD_TOL[prec])
    gate("composed bn1.weight rel", rel(dgamma, dg64), BN_PARAM_TOL)
    gate("composed bn1.bias rel", rel(dbeta, db64), BN_PARAM_TOL)
