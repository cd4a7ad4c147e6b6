"""GPU: the fc head (head.cu) and the BatchNorm kernels at the widths of the Resnet50_8s trunk, one operator at a time,
against float64.

fc (`ddn_fc_forward` / `ddn_fc_backward`: `fc_forward_kernel<DM>`, `fc_dgrad_kernel<DM>`, `fc_wgrad_kernel<DM, NQ>` and
`fc_part_reduce_kernel`) is checked two ways:

(a) exact arithmetic: small integers for w, bias and dlow, features on a 2^-8 grid (integer hi plane + small integers x 2^-8
    in the lo plane), every |partial sum| below 2^24 grid steps (asserted).  Every fp32 result is then exact whatever the
    summation order, so low, low_nhwc, dfeat, dw and dbias must be bit-equal to float64.  Outputs and the `part` workspace
    are NaN before the call: an element left unwritten, or an unwritten partial that is read, fails.
(b) random values, per element: |got - ref| <= k u sum|terms| with u = 2^-24 and k the longest rounding chain of the kernel
    (`fc_chains`, derived from head.cu).  The float64 reference of the plane paths is hi.float() + lo.float() (or hi alone):
    the values the kernel reads.

The cases cover every DM bin and its masked interior (D = 1 ... 32, both NQ), C = 512, 1024 and 2048, the three feature
sources (fp32, bf16 hi + lo, bf16 hi alone), one pixel per image, fewer pixels than one slot and one forward tile, weight-
gradient slots that cross image boundaries and end on an odd pixel pair (N = 3, Mimg = 77), and the bench geometry
16 x 60x80 at both trunk widths, where a second call must be bit-identical.

BatchNorm (`ddn_batchnorm_forward` / `_backward`) runs at C = 1024, 2048 and 4096 (column sums cut into 1024-channel slices,
backward apply tables above 48 KB of shared memory), train and eval, with and without ReLU and residual, against float64
at the gates of test_gpu_ops.py::test_batchnorm_forward_backward.  Every channel has its own mean and scale, so a slice
that reads another slice's columns is a gross error.

On one H100 80GB HBM3 at 700 W the file runs in about 12 s with a peak of 16.4 GB of device memory (torch allocator).
"""
import pytest
import torch
import torch.nn.functional as F

from pdc_b200 import ops, _native as N

gpu = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
FC_CHUNK = 512                 # head.cu: channels staged per forward / data-gradient block
WARP_LEVELS = 5                # warp_sum: 32 lanes
MOMENTUM, EPS = 0.1, 1e-5

WORST = {}                     # gate -> worst value seen in this session (DESIGN.md §2 records them)


def gate(name, err, tol):
    WORST[name] = max(WORST.get(name, 0.0), err)
    assert err <= tol, "%s: %.3e > %.1e" % (name, err, tol)


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    for name in sorted(WORST):
        print("worst %-40s %.3e" % (name, WORST[name]))


def rel(a, b):
    a = a.double(); b = b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


# ------------------------------------------------------------------------------------------------ fc slot geometry
def fc_slots(C):
    """head.cu fc_slots: (max_slots, min_pixels) of the weight gradient's pixel slots"""
    return (512, 16) if C <= 512 else (64, 1)


def slot_layout(n, mimg, C):
    """launch_fc_backward: pixels per slot and the [p0, p1) range of every slot"""
    total = n * mimg
    max_slots, min_pixels = fc_slots(C)
    pps = max(min_pixels, -(-total // max_slots))
    return pps, [(p0, min(total, p0 + pps)) for p0 in range(0, total, pps)]


def row_counts(p0, p1):
    """fc_wgrad_kernel: row rr of a slot takes the pixels p0 + rr, p0 + rr + 4, ... in pairs"""
    return [len(range(p0 + rr, p1, 4)) for rr in range(4)]


def crosses_image(slots, mimg):
    return any(p0 // mimg != (p1 - 1) // mimg for p0, p1 in slots)


def odd_tail(slots):
    return any(c % 2 for p0, p1 in slots for c in row_counts(p0, p1))


def short_slot(slots):
    return any(p1 - p0 < 4 for p0, p1 in slots)


SMALL_GEOMS = [
    # label, N, Mimg
    ("mimg1", 3, 1),           # one pixel per image: every slot shorter than 4 pixels
    ("tiny", 2, 7),            # 14 pixels: less than one 16-pixel slot and one 32-pixel forward tile
    ("ragged", 3, 77),         # slots that cross image boundaries and end on an odd pixel pair
]
BENCH_GEOM = ("bench", 16, 60 * 80)


@pytest.mark.parametrize("C", [512, 1024, 2048])
def test_fc_slot_geometry(C):
    """the geometries of the fc cases produce the slot layouts they are meant to exercise"""
    pps, slots = slot_layout(3, 1, C)
    assert short_slot(slots) and all(p1 - p0 < 4 for p0, p1 in slots)
    pps, slots = slot_layout(2, 7, C)
    assert 2 * 7 < 16 and 2 * 7 < 32 and short_slot(slots) == (C > 512)
    pps, slots = slot_layout(3, 77, C)
    assert crosses_image(slots, 77) and odd_tail(slots)
    if C == 512:
        assert (pps, len(slots)) == (16, 15) and slots[-1] == (224, 231)        # 7-pixel last slot: rows of 2, 2, 2, 1
        assert crosses_image(slot_layout(2, 7, C)[1], 7) and odd_tail(slot_layout(2, 7, C)[1])
    else:
        assert (pps, len(slots)) == (4, 58) and short_slot(slots)               # 1 pixel per row; the last slot has 3
    pps, slots = slot_layout(16, 60 * 80, C)
    assert (pps, len(slots)) == ((150, 512) if C == 512 else (1200, 64))
    if C == 512:
        assert row_counts(*slots[0]) == [38, 38, 37, 37]                         # odd pairs at the bench size too


# ------------------------------------------------------------------------------------------------ fc operands and reference
def fc_chains(C, D, pps):
    """Longest chain of fp32 roundings any single term passes through, per output (Higham: |err| <= gamma_L sum|terms|,
    gamma_L = L u / (1 - L u) < (L + 1) u here, which also covers the fp64 slot reduce, about 512 x 2^-53):
      low:   per lane 4 quads x 4 nested FMAs per chunk (FC_CHUNK/4 quads over 32 lanes) + 5 warp_sum levels
             + (chunks - 1) chunk adds + the bias add
      dfeat: D FMAs
      dw:    ceil(pps/4) FMAs of one pixel row + 3 row folds + the fp32 rounding of the fp64 slot sum
      dbias: per pixel pair (ga + gb) and its add, ceil(pps/8) pairs + 1, + 3 row folds + the fp32 rounding"""
    chains = {
        "low": 4 * (FC_CHUNK // 4 // 32) + WARP_LEVELS + (C // FC_CHUNK - 1) + 1,
        "dfeat": D,
        "dw": -(-pps // 4) + 3 + 1,
        "dbias": -(-pps // 8) + 1 + 3 + 1,
    }
    return {k: v + 1 for k, v in chains.items()}


SOURCES = ["fp32", "bf16x3", "bf16"]    # fp32 features (the instrument), hi + lo planes, hi plane alone


def fc_operands(kind, n, mimg, C, D, source, seed):
    """-> (feat or hi plane [N, Mimg, C], lo plane or None, w [D, C], bias [D], dlow [N, D, Mimg], values the kernel reads [P, C])"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    P = n * mimg
    if kind == "exact":
        hi = torch.randint(-4, 5, (P, C), generator=g, device=DEV).float()
        lo = torch.randint(-8, 9, (P, C), generator=g, device=DEV).float() * 2.0 ** -8
        w = torch.randint(-3, 4, (D, C), generator=g, device=DEV).float()
        bias = torch.randint(-3, 4, (D,), generator=g, device=DEV).float()
        dlow = torch.randint(-3, 4, (n, D, mimg), generator=g, device=DEV).float()
        if P > 4096:       # sparse cotangent: the weight-gradient sums stay below 2^24 grid steps
            dlow *= torch.rand(n, D, mimg, generator=g, device=DEV) < 1.0 / 32
        hi_b, lo_b = hi.to(torch.bfloat16), lo.to(torch.bfloat16)
        assert torch.equal(hi_b.float(), hi) and torch.equal(lo_b.float(), lo)
    else:
        x = torch.randn(P, C, generator=g, device=DEV)
        w = torch.randn(D, C, generator=g, device=DEV) * C ** -0.5
        bias = torch.randn(D, generator=g, device=DEV)
        dlow = torch.randn(n, D, mimg, generator=g, device=DEV)
        if source == "fp32":
            return x.view(n, mimg, C), None, w, bias, dlow, x
        hi_b = x.to(torch.bfloat16)
        lo_b = (x - hi_b.float()).to(torch.bfloat16)
    if source == "fp32":
        val = hi_b.float() + lo_b.float()
        return val.view(n, mimg, C), None, w, bias, dlow, val
    if source == "bf16x3":
        return hi_b.view(n, mimg, C), lo_b.view(n, mimg, C), w, bias, dlow, hi_b.float() + lo_b.float()
    return hi_b.view(n, mimg, C), None, w, bias, dlow, hi_b.float()


def fc_reference(val, w, bias, dlow):
    """float64 results and sum|terms| per output element, all as [P, D] / [P, C] / [D, C] / [D]"""
    n, D, mimg = dlow.shape
    v = val.double(); va = v.abs()
    w64 = w.double(); wa = w64.abs()
    g = dlow.double().permute(0, 2, 1).reshape(n * mimg, D); ga = g.abs()
    return {
        "low": (v @ w64.T + bias.double(), va @ wa.T + bias.double().abs()),
        "dfeat": (g @ w64, ga @ wa),
        "dw": (g.T @ v, ga.T @ va),
        "dbias": (g.sum(0), ga.sum(0)),
    }


def run_fc(feat, lo, w, bias, dlow):
    """forward and backward with every output and the workspace NaN beforehand"""
    n, mimg, C = feat.shape
    D = w.shape[0]
    nan = float("nan")
    low, low_nhwc = ops.fc_forward(feat, w, bias, feat_lo=lo, low=torch.full((n, D, mimg), nan, device=DEV),
                                   low_nhwc=torch.full((n * mimg, D), nan, device=DEV))
    ws = torch.full((N.lib.ddn_fc_workspace_bytes(C, D) // 4,), nan, device=DEV)
    dfeat, dw, dbias = ops.fc_backward(dlow, feat, w, feat_lo=lo, dfeat=torch.full((n * mimg, C), nan, device=DEV),
                                       dw=torch.full((D, C), nan, device=DEV), dbias=torch.full((D,), nan, device=DEV), workspace=ws)
    return {"low": low, "low_nhwc": low_nhwc, "dfeat": dfeat, "dw": dw, "dbias": dbias}


def as_ref_layout(name, t, n, mimg):
    """kernel output -> the [P, D] / [P, C] / [D, C] / [D] layout of fc_reference"""
    if name == "low":
        return t.permute(0, 2, 1).reshape(n * mimg, -1)
    return t


def check_fc(kind, n, mimg, C, D, source, seed):
    feat, lo, w, bias, dlow, val = fc_operands(kind, n, mimg, C, D, source, seed)
    out = run_fc(feat, lo, w, bias, dlow)
    ref = fc_reference(val, w, bias, dlow)
    # the NHWC copy is the planar map, transposed
    assert torch.equal(out["low_nhwc"], as_ref_layout("low", out["low"], n, mimg))
    pps = slot_layout(n, mimg, C)[0]
    chains = fc_chains(C, D, pps)
    for name in ("low", "dfeat", "dw", "dbias"):
        got = as_ref_layout(name, out[name], n, mimg).double()
        r, terms = ref[name]
        if kind == "exact":
            assert float((terms * 256).max()) < 2 ** 24, "operands too large for exact fp32 sums"
            bad = int((got != r).sum())          # NaN != anything
            assert bad == 0, "%s: %d of %d elements differ from float64" % (name, bad, r.numel())
        else:
            err = (got - r).abs()
            bound = chains[name] * U * terms
            ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, float("inf"), 0.0))
            gate("fc %s, |err| / (k u sum|terms|)" % name, float(ratio.max()), 1.0)
    return out


def small_params():
    out = []
    for label, n, mimg in SMALL_GEOMS:
        for C in (512, 1024, 2048):
            for D in (1, 3, 4, 5, 8, 9, 16, 17, 31, 32):
                for source in SOURCES:
                    for kind in ("exact", "random"):
                        out.append(pytest.param(kind, n, mimg, C, D, source, id="%s-%s-C%d-D%d-%s" % (kind, label, C, D, source)))
    return out


@gpu
@pytest.mark.parametrize("kind,n,mimg,C,D,source", small_params())
def test_fc_small(kind, n, mimg, C, D, source):
    check_fc(kind, n, mimg, C, D, source, seed=1000 * D + C + mimg + SOURCES.index(source))


def bench_params():
    _, n, mimg = BENCH_GEOM
    return [pytest.param(kind, n, mimg, C, D, source, id="%s-bench-C%d-D%d-%s" % (kind, C, D, source))
            for kind in ("exact", "random") for C in (512, 2048) for D in (3, 32) for source in SOURCES]


@gpu
@pytest.mark.parametrize("kind,n,mimg,C,D,source", bench_params())
def test_fc_bench_geometry(kind, n, mimg, C, D, source):
    """16 x 60x80: 512 slots of 150 pixels at C = 512, 64 of 1200 at C = 2048; a second call is bit-identical"""
    out = check_fc(kind, n, mimg, C, D, source, seed=7 * D + C)
    feat, lo, w, bias, dlow, _ = fc_operands(kind, n, mimg, C, D, source, seed=7 * D + C)
    again = run_fc(feat, lo, w, bias, dlow)
    for name in out:
        assert torch.equal(out[name].view(torch.int32), again[name].view(torch.int32)), name


# ------------------------------------------------------------------------------------------------ BatchNorm at C >= 1024
BN_ROWS = [
    # C, M
    (1024, 5), (2048, 5), (4096, 5),            # fewer rows than one wave of column-sum blocks: 2 blocks of 4 and 1 rows
    (1024, 9999), (2048, 9999), (4096, 9999),   # odd M: the last block ends on the single-row tail of the two-row loop
    (2048, 16 * 60 * 80),                       # layer4 of Resnet50_8s at the bench size
]


def bn_operands(C, M, residual):
    g = torch.Generator(device=DEV).manual_seed(C + M)
    c = torch.arange(C, device=DEV, dtype=torch.float32)
    scale = 1.0 + (c % 5) * 0.25                 # every channel its own scale and mean
    offset = (2.0 * c / C - 1.0) * 0.5
    x = torch.randn(M, C, generator=g, device=DEV) * scale + offset
    gamma = torch.rand(C, generator=g, device=DEV) + 0.5
    beta = torch.randn(C, generator=g, device=DEV)
    res = torch.randn(M, C, generator=g, device=DEV) if residual else None
    rm0 = offset + 0.1 * torch.randn(C, generator=g, device=DEV)
    rv0 = scale ** 2 * (0.8 + 0.4 * torch.rand(C, generator=g, device=DEV))
    dy = torch.randn(M, C, generator=g, device=DEV)
    return x, gamma, beta, res, rm0, rv0, dy


def bn_params():
    out = []
    for C, M in BN_ROWS:
        for training in (True, False):
            for relu, residual in ((False, False), (True, False), (False, True), (True, True)):
                out.append(pytest.param(C, M, training, relu, residual,
                                        id="C%d-M%d-%s%s%s" % (C, M, "train" if training else "eval", "-relu" if relu else "",
                                                               "-res" if residual else "")))
    return out


@gpu
@pytest.mark.parametrize("C,M,training,relu,residual", bn_params())
def test_wide_batchnorm(C, M, training, relu, residual):
    x, gamma, beta, res, rm0, rv0, dy = bn_operands(C, M, residual)
    rm, rv = rm0.clone(), rv0.clone()
    y, mean, invstd = ops.batchnorm_forward(x, gamma, beta, res, relu=relu, training=training, running_mean=rm, running_var=rv,
                                            momentum=MOMENTUM, eps=EPS)
    x64 = x.double().requires_grad_()
    g64 = gamma.double().requires_grad_(); b64 = beta.double().requires_grad_()
    r64 = res.double().requires_grad_() if residual else None
    rm64, rv64 = rm0.double(), rv0.double()
    lin = F.batch_norm(x64, rm64, rv64, g64, b64, training, MOMENTUM, EPS)     # updates rm64 / rv64 in train mode
    if residual:
        lin = lin + r64
    ref = lin.clamp_min(0) if relu else lin
    gate("bn y", rel(y, ref.detach()), 2e-6)
    if not training:
        gate("bn eval mean, invstd", max(rel(mean, rm0), rel(invstd, 1.0 / (rv0.double() + EPS).sqrt())), 2e-6)
        assert torch.equal(rm, rm0) and torch.equal(rv, rv0)
        return
    xd = x.double()
    gate("bn mean, invstd", max(rel(mean, xd.mean(0)), rel(invstd, 1.0 / (xd.var(0, unbiased=False) + EPS).sqrt())), 2e-6)
    gate("bn running mean, var", max(rel(rm, rm64), rel(rv, rv64)), 1e-6)       # momentum 0.1, unbiased variance
    dx, dgamma, dbeta, dres = ops.batchnorm_backward(dy, x, y, gamma, mean, invstd, relu=relu, need_residual_grad=residual)
    # the ReLU mask is the kernel's own (y > 0): an fp32 y within an ulp of zero would otherwise flip one gradient element
    (lin * (y > 0) if relu else lin).backward(dy.double())
    gate("bn dx", rel(dx, x64.grad), 1e-5)
    gate("bn dgamma, dbeta", max(rel(dgamma, g64.grad), rel(dbeta, b64.grad)), 1e-5)
    if residual:
        gate("bn d residual", rel(dres, r64.grad), 1e-6)
