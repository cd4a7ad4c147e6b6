"""GPU: the fused epilogues of the tensor-core convolutions, one operator at a time, against float64.

Every tensor-core conv of a training step ends in one of three epilogues (conv_tc.cu `conv_epilogue_rows`, in
`conv_tc_kernel` and `conv64_halo_kernel`): the training forward's BatchNorm statistics, the inference forward's folded
eval-mode BatchNorm, and the data gradient's BatchNorm-backward column sums.  Each case is checked two ways:

(a) the whole fused op against a float64 torch reference on the GPU, at the conv gates of test_conv2d_tcgen05
    (relative Frobenius 2e-5 for bf16x3, 8e-3 for bf16);
(b) the epilogue alone: its reductions and conversions against float64 computed from the tensor the kernel itself wrote,
    which removes the bf16 GEMM error, so these gates are tight and the same for both precisions.

Each case names the kernel path it exercises.  The tail-piece cases reserve SMs so that the host cuts the last wave into
64- or 32-channel pieces (the split rule of `tc_conv_planes`, reproduced here from the SM count).

On one H100 80GB HBM3 at 700 W the file runs in about 6 s with a peak of 4.3 GB of device memory (torch allocator).
"""
import functools

import pytest
import torch
import torch.nn.functional as F

from pdc_b200 import ops, _native as N

pytestmark = pytest.mark.gpu
DEV = "cuda"
PREC = {"bf16x3": N.PRECISION_BF16X3, "bf16": N.PRECISION_BF16}
GEMM_TOL = {"bf16x3": 2e-5, "bf16": 8e-3}
# (b) gates: per channel and BatchNorm group
MEAN_TOL = 1e-6        # |d mean| / std
INVSTD_TOL = 2e-6      # relative
RUNNING_TOL = 2e-6     # running mean (in units of the running std) and running var (relative)
SUMS_TOL = 1e-6        # |d sum| / sum of magnitudes
MOMENTUM, EPS = 0.1, 1e-5


WORST = {}             # gate -> worst value seen in this session (DESIGN.md §2 records them)


def gate(name, err, tol):
    WORST[name] = max(WORST.get(name, 0.0), err)
    assert err <= tol, "%s: %.3e > %.1e" % (name, err, tol)


def rel(a, b):
    a = a.double(); b = b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def nchw(t):
    return t.permute(0, 3, 1, 2)


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def is_stem(case):
    return case[5] == 3


def out_hw(case):
    _, _, n, h, w, cin, cout, k, s, p, d = case
    return (h + 2 * p - d * (k - 1) - 1) // s + 1, (w + 2 * p - d * (k - 1) - 1) // s + 1


# label, path, N, H, W, Cin, Cout, k, stride, pad, dil
HALO_SMALL = ("halo_small", "conv64_halo_kernel, 2 images of 3x2 tiles", 2, 24, 32, 64, 64, 3, 1, 1, 1)
HALO_BENCH = ("halo_bench", "conv64_halo_kernel at layer1's bench size, 2400 tiles", 16, 120, 160, 64, 64, 3, 1, 1, 1)
STRADDLE = ("straddle", "conv_tc_kernel<128>, 3 sub-tiles per image: tile 1 holds image 0 and image 1", 2, 12, 16, 128, 128, 3, 1, 1, 1)
PARTIAL = ("partial", "conv_tc_kernel<128>, sub-tiles cut in both dimensions (13x9 of 16x16)", 2, 13, 9, 256, 256, 3, 1, 2, 2)
PARTIAL_ODD = ("partial_odd", "conv_tc_kernel<128>, odd n_sub: the last tile's second sub-tile is invalid", 3, 11, 9, 256, 256, 3, 1, 2, 2)
LAYER4 = ("layer4", "conv_tc_kernel<128>, layer4 3x3 dil 4 at bench size", 16, 60, 80, 512, 512, 3, 1, 4, 4)
S2_3X3 = ("s2_3x3", "conv_tc_kernel<128> forward through TMA strides; dgrad: zero insertion, conv_tc_kernel<64>", 4, 120, 160, 64, 128, 3, 2, 1, 1)
S2_1X1 = ("s2_1x1", "1x1 stride 2 (layer2.0.downsample)", 4, 120, 160, 64, 128, 1, 2, 0, 1)
BN64 = ("bn64", "conv_tc_kernel<64> (64 -> 64 dil 2, not the halo kernel)", 2, 24, 32, 64, 64, 3, 1, 2, 2)
STEM_PARTIAL = ("stem_partial", "stem patch GEMM, 244x324 output: partial sub-tiles", 4, 488, 648, 3, 64, 7, 2, 3, 1)
STEM_BENCH = ("stem_bench", "stem patch GEMM at bench size", 16, 480, 640, 3, 64, 7, 2, 3, 1)


def groups(case):
    return [1, 2] if case[2] % 2 == 0 else [1]


def params(cases):
    out = []
    for case in cases:
        for G in groups(case):
            for prec in PREC:
                out.append(pytest.param(case, G, prec, id="%s-G%s-%s" % (case[0], G, prec)))
    return out


def gen(case, salt):
    return torch.Generator(device=DEV).manual_seed(sum(case[2:]) * 7 + salt)


def weights(case, g):
    _, _, _, _, _, cin, cout, k, _, _, _ = case
    return torch.randn(cout, cin, k, k, generator=g, device=DEV) * (2.0 / (k * k * cin)) ** 0.5


def group_rows(t, G):
    """[N, ...] -> [G, N/G * ..., C] (channels last)"""
    return t.reshape(G, -1, t.shape[-1])


# ------------------------------------------------------------------------------------------------ training forward
@functools.lru_cache(maxsize=1)
def fwd_operands(case):
    _, _, n, h, w, cin, cout, k, s, p, d = case
    g = gen(case, 1)
    if is_stem(case):
        x = torch.randn(n, 3, h, w, generator=g, device=DEV) + 0.2          # NCHW: the network's input layout
        x64 = x.double()
    else:
        x = torch.randn(n, h, w, cin, generator=g, device=DEV) + 0.2
        x64 = nchw(x.double())
    wt = weights(case, g)
    raw64 = nhwc(F.conv2d(x64, wt.double(), None, s, p, d))
    rm0 = torch.randn(cout, generator=g, device=DEV) * 0.2
    rv0 = torch.rand(cout, generator=g, device=DEV) + 0.5
    return x, wt, raw64, rm0, rv0


def batch_stats(raw, G):
    r = group_rows(raw.double(), G)
    mu = r.mean(1)
    var = r.var(1, unbiased=False)
    return mu, var, r.shape[1]


def running_ref(rm0, rv0, mu, var, cnt):
    rm, rv = rm0.double(), rv0.double()
    for gi in range(mu.shape[0]):       # group 0 first, then group 1 (forward(A), then forward(B))
        rm = (1 - MOMENTUM) * rm + MOMENTUM * mu[gi]
        rv = (1 - MOMENTUM) * rv + MOMENTUM * var[gi] * cnt / (cnt - 1)
    return rm, rv


def run_fwd(case, G, prec):
    _, _, _, _, _, _, _, _, s, p, d = case
    x, wt, _, rm0, rv0 = fwd_operands(case)
    rm, rv = rm0.clone(), rv0.clone()
    raw, mean, invstd = ops.conv2d_bn_stats_forward(x, wt, s, p, d, bn_groups=G, running_mean=rm, running_var=rv,
                                                    momentum=MOMENTUM, eps=EPS, precision=PREC[prec])
    return raw, mean, invstd, rm, rv


def check_fwd(case, G, prec):
    raw, mean, invstd, rm, rv = run_fwd(case, G, prec)
    _, _, raw64, rm0, rv0 = fwd_operands(case)
    # (a) the fused op against float64
    assert raw.shape == raw64.shape
    tol = GEMM_TOL[prec]
    gate("fwd raw (a) " + prec, rel(raw, raw64), tol)
    mu64, var64, _ = batch_stats(raw64, G)
    std64 = var64.sqrt()
    gate("fwd mean (a) " + prec, float(((mean.double() - mu64).abs() / std64).max()), tol)
    gate("fwd invstd (a) " + prec, float((invstd.double() * (var64 + EPS).sqrt() - 1).abs().max()), tol)
    # (b) the epilogue's statistics of the raw output the kernel itself wrote
    mu, var, cnt = batch_stats(raw, G)
    std = var.sqrt()
    e_mean = float(((mean.double() - mu).abs() / std).max())
    e_inv = float((invstd.double() * (var + EPS).sqrt() - 1).abs().max())
    rm_ref, rv_ref = running_ref(rm0, rv0, mu, var, cnt)
    e_rm = float(((rm.double() - rm_ref).abs() / rv_ref.sqrt()).max())
    e_rv = float(((rv.double() - rv_ref).abs() / rv_ref).max())
    gate("fwd mean (b)", e_mean, MEAN_TOL)
    gate("fwd invstd (b)", e_inv, INVSTD_TOL)
    gate("fwd running mean (b)", e_rm, RUNNING_TOL)
    gate("fwd running var (b)", e_rv, RUNNING_TOL)
    return raw, mean, invstd, rm, rv


FWD_CASES = [HALO_SMALL, HALO_BENCH, STRADDLE, PARTIAL, PARTIAL_ODD, LAYER4, S2_3X3, S2_1X1, BN64, STEM_PARTIAL, STEM_BENCH]


@pytest.mark.parametrize("case,G,prec", params(FWD_CASES))
def test_forward_bn_stats(case, G, prec):
    out = check_fwd(case, G, prec)
    if case is LAYER4 and G == 2 and prec == "bf16x3":       # one training-size case: bit-identical on a second call
        again = run_fwd(case, G, prec)
        for a, b in zip(out, again):
            assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------ inference forward (folded)
@functools.lru_cache(maxsize=1)
def fold_operands(case):
    _, _, n, h, w, cin, cout, k, s, p, d = case
    g = gen(case, 2)
    x = torch.randn(n, h, w, cin, generator=g, device=DEV)
    wt = weights(case, g)
    gamma = torch.rand(cout, generator=g, device=DEV) + 0.5
    beta = torch.randn(cout, generator=g, device=DEV) * 0.5
    rm = torch.randn(cout, generator=g, device=DEV) * 0.2
    rv = torch.rand(cout, generator=g, device=DEV) * 1.5 + 0.5
    ho, wo = out_hw(case)
    addend = torch.randn(n, ho, wo, cout, generator=g, device=DEV)
    conv64 = nhwc(F.conv2d(nchw(x.double()), wt.double(), None, s, p, d))
    scale = gamma.double() / (rv.double() + EPS).sqrt()
    shift = beta.double() - rm.double() * scale
    return x, wt, gamma, beta, rm, rv, addend, conv64 * scale + shift


def check_folded(case, prec, addend, relu, outputs):
    """outputs: "y+planes", "planes" (as act1 in the network) or "y"."""
    _, _, _, _, _, _, _, _, s, p, d = case
    x, wt, gamma, beta, rm, rv, add, lin64 = fold_operands(case)
    add = add if addend else None
    call = functools.partial(ops.conv2d_folded_forward, x, wt, gamma, beta, rm, rv, s, p, d, addend=add, relu=relu, eps=EPS,
                             precision=PREC[prec])
    ref = lin64 + add.double() if addend else lin64
    ref = ref.clamp_min(0) if relu else ref
    y, y_hi, y_lo = call(want_y=True, want_planes=True)
    # (a) against float64
    gate("folded y (a) " + prec, rel(y, ref), GEMM_TOL[prec])
    # (b) the planes are the round-to-nearest split of the kernel's own fp32 output, bit for bit
    hi_ref = y.to(torch.bfloat16)
    assert torch.equal(y_hi.view(torch.int16), hi_ref.view(torch.int16))
    if prec == "bf16x3":
        lo_ref = (y - hi_ref.float()).to(torch.bfloat16)
        assert torch.equal(y_lo.view(torch.int16), lo_ref.view(torch.int16))
    else:
        sentinel = torch.full_like(y_hi, -7.0)
        _, _, lo = call(want_y=False, want_planes=True, y_lo=sentinel.clone())
        assert torch.equal(lo.view(torch.int16), sentinel.view(torch.int16))        # single-pass bf16 writes no lo plane
    if outputs in ("planes", "y+planes"):
        _, hi2, lo2 = call(want_y=False, want_planes=True)
        assert torch.equal(hi2.view(torch.int16), y_hi.view(torch.int16))
        if prec == "bf16x3":
            assert torch.equal(lo2.view(torch.int16), y_lo.view(torch.int16))
    if outputs == "y":
        y2, none_hi, _ = call(want_y=True, want_planes=False)
        assert none_hi is None and torch.equal(y2, y)
    return y, y_hi, y_lo


FOLD_CASES = [
    # case, addend, relu, outputs
    (HALO_SMALL, True, True, "y+planes"),
    (HALO_BENCH, True, True, "y+planes"),
    (PARTIAL, False, True, "planes"),
    (S2_3X3, True, True, "y+planes"),
    (S2_1X1, False, False, "y"),              # the downsample branch of the folded network: bn_d(conv_d(x)), fp32
]


@pytest.mark.parametrize("prec", list(PREC))
@pytest.mark.parametrize("case,addend,relu,outputs", FOLD_CASES, ids=[c[0][0] for c in FOLD_CASES])
def test_folded_forward(case, addend, relu, outputs, prec):
    out = check_folded(case, prec, addend, relu, outputs)
    if case is HALO_BENCH and prec == "bf16x3":
        again = check_folded(case, prec, addend, relu, outputs)
        for a, b in zip(out, again):
            assert torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a.view(torch.int16),
                               b.view(torch.int32) if b.dtype == torch.float32 else b.view(torch.int16))


# ------------------------------------------------------------------------------------------------ data gradient + column sums
@functools.lru_cache(maxsize=1)
def dgrad_operands(case, G):
    _, _, n, h, w, cin, cout, k, s, p, d = case
    g = gen(case, 3 + G)
    wt = weights(case, g)
    ho, wo = out_hw(case)
    dy = torch.randn(n, ho, wo, cout, generator=g, device=DEV)
    addend = torch.randn(n, h, w, cin, generator=g, device=DEV)
    # the consuming BatchNorm: raw with per-channel offsets, its per-group statistics, affine parameters
    raw = torch.randn(n, h, w, cin, generator=g, device=DEV) * (torch.rand(cin, generator=g, device=DEV) + 0.5) \
        + torch.randn(cin, generator=g, device=DEV)
    mu, var, _ = batch_stats(raw, G)
    mean = mu.float().contiguous(); invstd = (1.0 / (var + EPS).sqrt()).float().contiguous()
    gamma = torch.rand(cin, generator=g, device=DEV) + 0.5
    beta = torch.randn(cin, generator=g, device=DEV) * 0.5
    # the bf16 hi plane of a block output y = relu(bn(raw) + residual): zeros, positives, a few tiny values
    y = (torch.randn(n, h, w, cin, generator=g, device=DEV)).clamp_min(0)
    y[..., ::7] *= 1e-30
    y_hi = y.to(torch.bfloat16)
    dx64 = nhwc(torch.nn.grad.conv2d_input((n, cin, h, w), wt.double(), nchw(dy.double()), s, p, d))
    return wt, dy, addend, raw, mean, invstd, gamma, beta, y_hi, dx64


def per_image(t, G, n):
    """[G, C] -> [N, 1, 1, C]: the row of each image's BatchNorm group"""
    return t.repeat_interleave(n // G, dim=0)[:, None, None, :]


def recomputed_mask(raw, mean, invstd, gamma, beta, G):
    """the kernel's test fmaf((raw - mu)_f32, (gamma * invstd)_f32, beta) > 0, reproduced exactly: the product of two fp32
    values is exact in float64 and rounding keeps the sign of the sum"""
    n = raw.shape[0]
    t = raw - per_image(mean, G, n)                        # fp32 subtraction, as in the kernel
    scl = gamma[None, :] * invstd                          # fp32 product, as in the kernel
    return (t.double() * per_image(scl, G, n).double() + beta.double()) > 0


def run_dgrad(case, G, prec, mask, addend):
    _, _, _, _, _, _, _, _, s, p, d = case
    wt, dy, add, raw, mean, invstd, gamma, beta, y_hi, _ = dgrad_operands(case, G)
    return ops.conv2d_backward_data_bn_stats(wt, dy, raw, mean, invstd, gamma, beta, s, p, d, addend=add if addend else None,
                                             y_hi=y_hi if mask == "y_hi" else None, precision=PREC[prec])


def column_sums(gx, xhat, G):
    return torch.stack([group_rows(gx, G).sum(1), group_rows(gx * xhat, G).sum(1)], 1)     # [G, 2, C]


def check_dgrad(case, G, prec, mask, addend):
    n = case[2]
    wt, dy, add, raw, mean, invstd, gamma, beta, y_hi, dx64 = dgrad_operands(case, G)
    dx, dgamma, dbeta, sums = run_dgrad(case, G, prec, mask, addend)
    m = (y_hi.float() > 0) if mask == "y_hi" else recomputed_mask(raw, mean, invstd, gamma, beta, G)
    xhat = (raw.double() - per_image(mean, G, n).double()) * per_image(invstd, G, n).double()
    ref_dx = dx64 + add.double() if addend else dx64
    # (a) against float64: the gradient, and the sums of the float64 gradient under the same mask
    gate("dgrad dx (a) " + prec, rel(dx, ref_dx), GEMM_TOL[prec])
    g64 = ref_dx * m
    # the GEMM error scales with the terms, not with dx + addend, which can cancel
    bound = column_sums((dx64.abs() + add.double().abs() if addend else dx64.abs()) * m, xhat.abs(), G)
    gate("dgrad sums (a) " + prec, float(((sums.double() - column_sums(g64, xhat, G)).abs() / bound).max()), GEMM_TOL[prec])
    # (b) the epilogue's sums of the gradient the kernel itself wrote
    gk = dx.double() * m
    ref = column_sums(gk, xhat, G)
    bound = column_sums(gk.abs(), xhat.abs(), G)
    e_sums = float(((sums.double() - ref).abs() / bound).max())
    e_db = float(((dbeta.double() - ref[:, 0].sum(0)).abs() / bound[:, 0].sum(0)).max())
    e_dg = float(((dgamma.double() - ref[:, 1].sum(0)).abs() / bound[:, 1].sum(0)).max())
    gate("dgrad sums (b)", e_sums, SUMS_TOL)
    gate("dgrad dbeta (b)", e_db, SUMS_TOL)
    gate("dgrad dgamma (b)", e_dg, SUMS_TOL)
    return dx, dgamma, dbeta, sums


DGRAD_CASES = [
    # case, mask, addend
    (HALO_SMALL, "recompute", True),
    (HALO_BENCH, "recompute", False),
    (STRADDLE, "recompute", False),
    (STRADDLE, "y_hi", True),
    (PARTIAL, "recompute", True),
    (PARTIAL_ODD, "y_hi", False),
    (LAYER4, "y_hi", True),                    # as in the network: bn2's mask from the block output's plane + the residual gradient
    (S2_3X3, "recompute", True),
    (S2_1X1, "y_hi", False),
    (BN64, "recompute", True),
]


def dgrad_params():
    out = []
    for case, mask, addend in DGRAD_CASES:
        for G in groups(case):
            for prec in PREC:
                out.append(pytest.param(case, mask, addend, G, prec, id="%s-%s-G%d-%s" % (case[0], mask, G, prec)))
    return out


@pytest.mark.parametrize("case,mask,addend,G,prec", dgrad_params())
def test_backward_data_bn_stats(case, mask, addend, G, prec):
    out = check_dgrad(case, G, prec, mask, addend)
    if case is LAYER4 and G == 2 and prec == "bf16x3":
        again = run_dgrad(case, G, prec, mask, addend)
        for a, b in zip(out, again):
            assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------ tail pieces
def tail_split(tiles, block_n, workers):
    """tc_conv_planes: the tiles of the last, partial wave are cut along N into `split` pieces"""
    rem = tiles % workers
    split = 1
    if rem:
        while split * 2 <= 8 and block_n // (split * 2) >= 32 and rem * split * 2 <= workers:
            split *= 2
    return split


def reserved_for(tiles, block_n, want):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for r in range(0, 65):
        workers = 8 if r >= sms - 8 else sms - r          # engine.cu tc_worker_sms
        if tail_split(tiles, block_n, workers) == want:
            return r
    return None


def conv_tiles(n, ho, wo, gout):
    n_sub = n * -(-ho // 4) * -(-wo // 16)
    block_n = 128 if gout % 128 == 0 else 64
    return -(-n_sub // 2) * (gout // block_n), block_n


TAIL_CASES = [
    # case, expected piece width (BLOCK_N / split)
    (("tail64_bn128", "conv_tc_kernel<128>, tail pieces of 64 channels", 2, 48, 64, 128, 128, 3, 1, 1, 1), 64),
    (("tail32_bn128", "conv_tc_kernel<128>, tail pieces of 32 channels", 2, 16, 32, 128, 128, 3, 1, 1, 1), 32),
    (("tail32_bn64", "conv_tc_kernel<64>, tail pieces of 32 channels", 2, 16, 32, 64, 64, 3, 1, 2, 2), 32),
]


@pytest.mark.parametrize("prec", list(PREC))
@pytest.mark.parametrize("case,width", TAIL_CASES, ids=[c[0][0] for c in TAIL_CASES])
def test_tail_pieces(case, width, prec):
    _, _, n, h, w, cin, cout, k, s, p, d = case
    ho, wo = out_hw(case)
    plans = []
    for what, (tiles, block_n) in (("forward", conv_tiles(n, ho, wo, cout)), ("dgrad", conv_tiles(n, h, w, cin))):
        r = reserved_for(tiles, block_n, block_n // width)
        assert r is not None, "no reserved-SM count gives %d-channel pieces for %s" % (width, what)
        plans.append((what, r))
    try:
        for what, r in plans:
            assert N.lib.ddn_set_reserved_sms(r) == 0
            for G in groups(case):
                if what == "forward":
                    check_fwd(case, G, prec)
                else:
                    check_dgrad(case, G, prec, "recompute", True)
                    check_dgrad(case, G, prec, "y_hi", False)
            if what == "forward":
                check_folded(case, prec, True, True, "y+planes")
    finally:
        assert N.lib.ddn_set_reserved_sms(0) == 0
