"""GPU: every tensor-core convolution path element by element, bit-exact against float64 on exact-arithmetic operands.

The other conv tests gate a relative Frobenius norm over the whole tensor (2e-5 bf16x3, 8e-3 bf16).  A bug local to one
work item -- a dropped k-block, a skipped cross term, an unwritten element that happens to hold the right value from the
previous call, a store past the tensor's edge -- can hide under that norm.  Here the operands are built so that every
product is exact and every partial sum is exact in fp32 (conv_exact_common.py: integer and split data, and a certificate
asserted per case), so each output element of each precision and kernel path must be bit-equal to a float64 model.

The test owns every buffer and calls the C ABI directly:
- every output is a view into a larger buffer whose guard bands (>= one output image or 1 MiB) hold a fixed bit pattern and
  must come back bit-identical; the output itself is NaN before the call;
- every input sits inside a NaN-filled buffer, so a read past its end turns an output into NaN;
- the workspace is 0xFF bytes (NaN as fp32, bf16 and fp64);
- every case sets the reserved-SM count explicitly, so the dispatch mirror knows the worker count, and a mismatch is
  reported as the count of wrong elements and the first coordinates mapped to sub-tile, work item, channel piece and
  k-block range (or halo tile / weight-gradient chunk).

On one H100 80GB HBM3 at 700 W the file's runtime and peak device memory are recorded in DESIGN.md §2.
"""
import functools
import zlib

import pytest
import torch

from pdc_b200 import _native as N

import conv_exact_common as C

pytestmark = pytest.mark.gpu
DEV = "cuda"
PREC = {"bf16x3": N.PRECISION_BF16X3, "bf16": N.PRECISION_BF16, "fp32": N.PRECISION_FP32_SIMT}
GUARD = 0x5A5AA5A5                      # guard-band bit pattern
NAN = 0x7FC00000
MIB = 1 << 20
MOMENTUM, EPS = 0.1, 1e-5


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def gen(case, what):
    return torch.Generator(device=DEV).manual_seed(zlib.crc32(("%s/%s" % (case["label"], what)).encode()))


# ------------------------------------------------------------------------------------------------ buffers the test owns
def _aligned(n_elems, dtype, fill):
    """a flat buffer of n_elems (+ slack) whose returned offset is 1024-byte aligned"""
    esz = torch.empty(0, dtype=dtype).element_size()
    buf = torch.full((n_elems + 1024 // esz,), fill, dtype=dtype, device=DEV)
    off = ((-buf.data_ptr()) % 1024) // esz
    return buf, off


def _guard_elems(image_elems):
    g = max(image_elems, MIB // 4)
    return -(-g // 256) * 256          # whole KiB: keeps the output 1024-byte aligned


class Out:
    """an fp32 output view, NaN, between two guard bands of GUARD"""

    def __init__(self, shape, image_elems):
        self.shape, self.n = tuple(shape), 1
        for s in shape:
            self.n *= s
        self.g = _guard_elems(image_elems)
        self.buf, off = _aligned(2 * self.g + self.n, torch.int32, GUARD)
        self.lo, self.hi = off + self.g, off + self.g + self.n
        self.buf[self.lo:self.hi] = NAN
        self.t = self.buf[self.lo:self.hi].view(torch.float32).view(self.shape)

    def guards_intact(self):
        return bool((self.buf[:self.lo] == GUARD).all()) and bool((self.buf[self.hi:] == GUARD).all())


def inp(t):
    """a copy of t inside a NaN-filled buffer (1 MiB of NaN on both sides), 1024-byte aligned"""
    t = t.contiguous()
    g = MIB // 4
    buf, off = _aligned(2 * g + t.numel(), torch.float32, float("nan"))
    v = buf[off + g:off + g + t.numel()].view(t.shape)
    v.copy_(t)
    v._keep = buf
    return v


def workspace(nbytes):
    buf, off = _aligned(max(int(nbytes), 256), torch.uint8, 255)
    return buf[off:off + max(int(nbytes), 256)]


def out_hw(shape):
    _, h, w, _, _, k, s, p, d = shape
    return (h + 2 * p - d * (k - 1) - 1) // s + 1, (w + 2 * p - d * (k - 1) - 1) // s + 1


@pytest.fixture
def reserved(request):
    """sets the case's reserved-SM count (the dispatch mirror picks it) and restores 0"""
    case = request.node.callspec.params["case"]
    r = C.reserved_for(case, sms())
    assert N.lib.ddn_set_reserved_sms(r) == 0
    try:
        yield C.plans(case, C.worker_sms(sms(), r))
    finally:
        assert N.lib.ddn_set_reserved_sms(0) == 0


def check(what, out, ref, locate):
    """out: Out; ref: fp32 model.  Guards bit-identical, no NaN, every element equal to the model."""
    assert out.guards_intact(), "%s: a guard band next to the output was written" % what
    got = out.t
    bad = (got != ref) | torch.isnan(got)
    nbad = int(bad.sum())
    if nbad:
        lines = []
        for idx in bad.nonzero()[:6].tolist():
            lines.append("  %s: got %r, want %r -- %s" % (tuple(idx), float(got[tuple(idx)]), float(ref[tuple(idx)]), locate(*idx)))
        pytest.fail("%s: %d of %d elements differ from the exact model (%d NaN)\n%s"
                    % (what, nbad, got.numel(), int(torch.isnan(got).sum()), "\n".join(lines)))


def params(cases, precs, groups=False):
    out = []
    for case in cases:
        for kind in ("integer", "split"):
            for prec in precs:
                if prec == "fp32" and kind == "split":
                    continue                     # the fp32 product of split data has a lo*lo term on a 2^-20 grid
                gs = ([1, 2] if case["shape"][0] % 2 == 0 else [1]) if groups else [None]
                for G in gs:
                    label = "%s-%s-%s" % (case["label"], kind, prec) + ("" if G is None else "-G%d" % G)
                    out.append(pytest.param(case, kind, prec, G, id=label))
    return out


# ------------------------------------------------------------------------------------------------ operands and models
@functools.lru_cache(maxsize=1)
def fwd_data(label, kind):
    case = C.BY_LABEL[label]
    n, h, w, cin, cout, k, s, p, d = case["shape"]
    g = gen(case, "fwd/" + kind)
    dens = 1.0 if kind == "integer" else C.density_for(k * k * cin)
    x = C.draw((n, 3, h, w) if case["stem"] else (n, h, w, cin), kind, dens, g, DEV)
    wt = C.draw((cout, cin, k, k), kind, dens, g, DEV)
    for op in (x, wt):
        C.certify_operand(op)
    if case["stem"]:
        f = lambda a, b: C.nhwc(torch.nn.functional.conv2d(a, b, None, s, p, d))
    else:
        f = C.conv_fwd_fn(s, p, d)
    with torch.backends.cudnn.flags(enabled=False):
        model = C.Model(f, x, wt, kind)
    return x[0], wt[0], model


@functools.lru_cache(maxsize=1)
def bwd_data(label, kind):
    """x, w, dy of ddn_conv2d_backward, with the models of dx (dy x w) and dw (dy x x)"""
    case = C.BY_LABEL[label]
    n, h, w, cin, cout, k, s, p, d = case["shape"]
    ho, wo = out_hw(case["shape"])
    g = gen(case, "bwd/" + kind)
    if kind == "integer":
        d_dy = d_x = d_w = 1.0
    else:
        k_w, k_d = n * ho * wo, k * k * cout
        d_dy = C.density_for(k_w)
        d_x = C.density_for(k_w, d_dy)
        d_w = C.density_for(k_d, d_dy)
    x = C.draw((n, h, w, cin), kind, d_x, g, DEV)
    wt = C.draw((cout, cin, k, k), kind, d_w, g, DEV)
    dy = C.draw((n, ho, wo, cout), kind, d_dy, g, DEV)
    for op in (x, wt, dy):
        C.certify_operand(op)
    with torch.backends.cudnn.flags(enabled=False):
        m_dx = C.Model(C.conv_dgrad_fn((n, h, w, cin), s, p, d), dy, wt, kind)
        m_dw = C.Model(C.conv_wgrad_fn((cout, cin, k, k), s, p, d), dy, x, kind)
    return x[0], wt[0], dy[0], m_dx, m_dw


@functools.lru_cache(maxsize=1)
def dgrad_bn_data(label, kind):
    """w, dy and an integer addend of ddn_conv2d_backward_data_bn_stats, with the model of dx = dgrad + addend"""
    case = C.BY_LABEL[label]
    n, h, w, cin, cout, k, s, p, d = case["shape"]
    ho, wo = out_hw(case["shape"])
    g = gen(case, "dgrad_bn/" + kind)
    dens = 1.0 if kind == "integer" else C.density_for(k * k * cout)
    wt = C.draw((cout, cin, k, k), kind, dens, g, DEV)
    dy = C.draw((n, ho, wo, cout), kind, dens, g, DEV)
    for op in (wt, dy):
        C.certify_operand(op)
    addend = torch.randint(-2, 3, (n, h, w, cin), generator=g, device=DEV).float()
    raw = torch.randn(n, h, w, cin, generator=g, device=DEV)
    with torch.backends.cudnn.flags(enabled=False):
        model = C.Model(C.conv_dgrad_fn((n, h, w, cin), s, p, d), dy, wt, kind, extra=addend)
    return wt[0], dy[0], addend, raw, model


def conv_locator(pl):
    return lambda n, h, w, ch: C.locate_conv(pl, n, h, w, ch)


# ------------------------------------------------------------------------------------------------ ddn_conv2d_forward
@pytest.mark.parametrize("case,kind,prec,G", params(C.CONV_CASES, ["bf16x3", "bf16", "fp32"]))
def test_forward(case, kind, prec, G, reserved):
    n, h, w, cin, cout, k, s, p, d = case["shape"]
    ho, wo = out_hw(case["shape"])
    x, wt, model = fwd_data(case["label"], kind)
    xi, wi = inp(x), inp(wt)
    y = Out((n, ho, wo, cout), ho * wo * cout)
    nb = N.lib.ddn_conv2d_workspace_bytes(n, h, w, cin, cout, k, s, p, d, PREC[prec])
    ws = workspace(nb)
    N.check(N.lib.ddn_conv2d_forward(N.ptr(xi), N.ptr(wi), N.ptr(y.t), n, h, w, cin, cout, k, s, p, d, PREC[prec],
                                     N.ptr(ws), ws.numel(), N.stream_ptr()))
    torch.cuda.synchronize()
    check("forward y", y, model.of(prec), conv_locator(reserved["fwd"]))


# ------------------------------------------------------------------------------------------------ ddn_conv2d_backward
@pytest.mark.parametrize("case,kind,prec,G", params(C.CONV_CASES, ["bf16x3", "bf16", "fp32"]))
def test_backward(case, kind, prec, G, reserved):
    n, h, w, cin, cout, k, s, p, d = case["shape"]
    x, wt, dy, m_dx, m_dw = bwd_data(case["label"], kind)
    xi, wi, dyi = inp(x), inp(wt), inp(dy)
    dx = Out((n, h, w, cin), h * w * cin)
    dw = Out((cout, cin, k, k), 0)
    nb = N.lib.ddn_conv2d_workspace_bytes(n, h, w, cin, cout, k, s, p, d, PREC[prec])
    ws = workspace(nb)
    N.check(N.lib.ddn_conv2d_backward(N.ptr(xi), N.ptr(wi), N.ptr(dyi), N.ptr(dx.t), N.ptr(dw.t), n, h, w, cin, cout, k, s, p, d,
                                      PREC[prec], N.ptr(ws), ws.numel(), N.stream_ptr()))
    torch.cuda.synchronize()
    check("data gradient dx", dx, m_dx.of(prec), conv_locator(reserved["dgrad"]))
    check("weight gradient dw", dw, m_dw.of(prec), lambda co, ci, r, s_: C.locate_wgrad(reserved["wgrad"], co, ci, r, s_))


# the fused entries take maps of at least 8x8 (check_fused): every case but `tiny`
FUSED_CASES = [k for k in C.CASES if k["shape"][1] >= 8 and k["shape"][2] >= 8]


# ------------------------------------------------------------------------------------------------ ddn_conv2d_bn_stats_forward
def run_bn_stats_forward(case, x, wt, G, prec):
    n, h, w, cin, cout, k, s, p, d = case["shape"]
    ho, wo = out_hw(case["shape"])
    xi, wi = inp(x), inp(wt)
    raw = Out((n, ho, wo, cout), ho * wo * cout)
    mean = torch.empty(G, cout, device=DEV)
    invstd = torch.empty(G, cout, device=DEV)
    ws = workspace(N.lib.ddn_conv2d_fused_workspace_bytes(n, h, w, cin, cout, k, s, p, d, PREC[prec]))
    N.check(N.lib.ddn_conv2d_bn_stats_forward(N.ptr(xi), N.ptr(wi), N.ptr(raw.t), N.ptr(mean), N.ptr(invstd), None, None,
                                              n, h, w, cin, cout, k, s, p, d, G, MOMENTUM, EPS, PREC[prec],
                                              N.ptr(ws), ws.numel(), N.stream_ptr()))
    torch.cuda.synchronize()
    return raw


@pytest.mark.parametrize("case,kind,prec,G", params(FUSED_CASES, ["bf16x3", "bf16"], groups=True))
def test_bn_stats_forward_raw(case, kind, prec, G, reserved):
    x, wt, model = fwd_data(case["label"], kind)
    raw = run_bn_stats_forward(case, x, wt, G, prec)
    check("bn_stats forward raw", raw, model.of(prec), conv_locator(reserved["fwd"]))


# ------------------------------------------------------------------------------------------------ ddn_conv2d_backward_data_bn_stats
@pytest.mark.parametrize("case,kind,prec,G", params([k for k in FUSED_CASES if not k["stem"]], ["bf16x3", "bf16"], groups=True))
def test_backward_data_bn_stats_dx(case, kind, prec, G, reserved):
    n, h, w, cin, cout, k, s, p, d = case["shape"]
    wt, dy, addend, raw, model = dgrad_bn_data(case["label"], kind)
    wi, dyi, addi, rawi = inp(wt), inp(dy), inp(addend), inp(raw)
    mean = torch.zeros(G, cin, device=DEV)
    invstd = torch.ones(G, cin, device=DEV)
    gamma = torch.ones(cin, device=DEV)
    beta = torch.zeros(cin, device=DEV)
    dx = Out((n, h, w, cin), h * w * cin)
    dgamma, dbeta = torch.empty(cin, device=DEV), torch.empty(cin, device=DEV)
    sums = torch.empty(G, 2, cin, device=DEV)
    ws = workspace(N.lib.ddn_conv2d_fused_workspace_bytes(n, h, w, cin, cout, k, s, p, d, PREC[prec]))
    N.check(N.lib.ddn_conv2d_backward_data_bn_stats(N.ptr(wi), N.ptr(dyi), N.ptr(addi), N.ptr(rawi), N.ptr(mean), N.ptr(invstd),
                                                    N.ptr(gamma), N.ptr(beta), None, N.ptr(dx.t), N.ptr(dgamma), N.ptr(dbeta),
                                                    N.ptr(sums), n, h, w, cin, cout, k, s, p, d, G, PREC[prec],
                                                    N.ptr(ws), ws.numel(), N.stream_ptr()))
    torch.cuda.synchronize()
    check("data gradient + addend dx", dx, model.of(prec), conv_locator(reserved["dgrad"]))


# ------------------------------------------------------------------------------------------------ stem weight gradient
# eval mode with gamma = invstd = 1, mean = beta = 0 and a positive integer raw: d raw = scatter(dy_pool) through the pool's
# argmax, an integer tensor; dw_conv1 is then the float64 weight gradient of that over the image
STEM_WGRAD_CASES = [("odd", 2, 50, 74), ("partial", 4, 488, 648)]


def stem_wgrad_params():
    out = []
    for case in STEM_WGRAD_CASES:
        for kind in ("integer", "split"):
            for prec in ("bf16x3", "bf16", "fp32"):
                if prec == "fp32" and kind == "split":
                    continue
                out.append(pytest.param(case, kind, prec, id="%s-%s-%s" % (case[0], kind, prec)))
    return out


@functools.lru_cache(maxsize=1)
def stem_wgrad_data(case, kind):
    label, n, h, w = case
    hc, wc = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    hp, wp = (hc - 1) // 2 + 1, (wc - 1) // 2 + 1
    g = torch.Generator(device=DEV).manual_seed(zlib.crc32(("stem/%s/%s" % (label, kind)).encode()))
    k_w = n * hc * wc                              # pixels of the weight-gradient sum
    dy_dens = 0.3
    x = C.draw((n, 3, h, w), kind, 1.0 if kind == "integer" else C.density_for(k_w, dy_dens, cap=1.0, target=1024), g, DEV)
    C.certify_operand(x)
    raw = torch.randint(1, 5, (n, hc, wc, 64), generator=g, device=DEV).float()
    dy_pool = torch.randint(-2, 3, (n, hp, wp, 64), generator=g, device=DEV).float() \
        * (torch.rand(n, hp, wp, 64, generator=g, device=DEV) < dy_dens).float()
    return x, raw, dy_pool


def stem_scatter(dy_pool, argmax, hc, wc):
    """float64 d raw: every pooled gradient added to its window's argmax position (r*3+s of the 3x3/2 pad-1 window)"""
    n, hp, wp, c = dy_pool.shape
    a = argmax.long()
    ph = torch.arange(hp, device=DEV)[None, :, None, None]
    pw = torch.arange(wp, device=DEV)[None, None, :, None]
    rr, ss = 2 * ph - 1 + a // 3, 2 * pw - 1 + a % 3
    assert bool(((rr >= 0) & (rr < hc) & (ss >= 0) & (ss < wc)).all()), "argmax outside the map"
    nn_ = torch.arange(n, device=DEV)[:, None, None, None].expand_as(a)
    cc = torch.arange(c, device=DEV)[None, None, None, :].expand_as(a)
    flat = ((nn_ * hc + rr) * wc + ss) * c + cc
    g = torch.zeros(n * hc * wc * c, dtype=torch.float64, device=DEV)
    g.index_add_(0, flat.reshape(-1), dy_pool.double().reshape(-1))
    return g.view(n, hc, wc, c)


@pytest.mark.parametrize("case,kind,prec", stem_wgrad_params())
def test_stem_weight_gradient(case, kind, prec):
    _, n, h, w = case
    hc, wc = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    hp, wp = (hc - 1) // 2 + 1, (wc - 1) // 2 + 1
    x, raw, dy_pool = stem_wgrad_data(case, kind)
    mean, invstd = torch.zeros(1, 64, device=DEV), torch.ones(1, 64, device=DEV)
    gamma, beta = torch.ones(64, device=DEV), torch.zeros(64, device=DEV)
    argmax = torch.empty(n, hp, wp, 64, dtype=torch.uint8, device=DEV)
    y = torch.empty(n, hp, wp, 64, device=DEV)
    assert N.lib.ddn_set_reserved_sms(0) == 0
    N.check(N.lib.ddn_stem_pool_forward(N.ptr(raw), N.ptr(mean), N.ptr(invstd), N.ptr(gamma), N.ptr(beta), N.ptr(y), None, None,
                                        N.ptr(argmax), n, hc, wc, 1, N.stream_ptr()))
    g64 = stem_scatter(dy_pool, argmax, hc, wc)
    gparts = (g64.float(), g64.float(), torch.zeros_like(g64, dtype=torch.float32))
    C.certify_operand(gparts)                      # d raw is integer: its bf16 split is (g, 0)
    with torch.backends.cudnn.flags(enabled=False):
        model = C.Model(C.conv_wgrad_fn((64, 3, 7, 7), 2, 3, 1, x_is_nchw=True), gparts, x, kind)
    xi, rawi, dyi = inp(x[0]), inp(raw), inp(dy_pool)
    g_out = Out((n, hc, wc, 64), hc * wc * 64)
    dw = Out((64, 3, 7, 7), 0)
    dgamma, dbeta = torch.empty(64, device=DEV), torch.empty(64, device=DEV)
    nb = N.lib.ddn_stem_workspace_bytes(n, h, w, PREC[prec])
    ws = workspace(nb)
    N.check(N.lib.ddn_stem_backward(N.ptr(xi), N.ptr(rawi), N.ptr(mean), N.ptr(invstd), N.ptr(gamma), N.ptr(beta), N.ptr(argmax),
                                    N.ptr(dyi), N.ptr(g_out.t), None, None, None, N.ptr(dgamma), N.ptr(dbeta), N.ptr(dw.t),
                                    n, h, w, 1, 0, PREC[prec], N.ptr(ws), ws.numel(), N.stream_ptr()))
    torch.cuda.synchronize()
    check("stem g_out", g_out, g64.float(), lambda *i: "stem_pool_relu_bwd")
    pl = C.wgrad_plan(n, hc, wc, 192, 64, 1, 1, 1, C.worker_sms(sms(), 0))
    check("stem dw_conv1", dw, model.of(prec),
          lambda co, c_, r, s_: "patch column %d: %s" % ((r * 7 + s_) * 3 + c_, C.locate_wgrad(pl, co, (r * 7 + s_) * 3 + c_, 0, 0)))


# ------------------------------------------------------------------------------------------------ coverage of the case list
def test_case_list_reaches_every_path_at_this_sm_count():
    seen, missed = C.coverage(sms())
    assert not missed, "cases that do not reach the path they claim at %d SMs: %s" % (sms(), missed)
    assert C.REQUIRED <= seen, "paths no case reaches at %d SMs: %s" % (sms(), sorted(C.REQUIRED - seen))
