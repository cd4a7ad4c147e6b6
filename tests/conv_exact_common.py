"""Shared by test_gpu_conv_exact.py and test_conv_exact_cpu.py: exact-arithmetic operands, their certificate, the float64
models of what each conv kernel path computes, and a Python restatement of the host rules that pick the kernel path.

Operands (`draw`):
  integer  every value in {-2..2}; hi = x, lo = 0.  Serves all three precisions.
  split    x = h + sign(h) * m * 2^-10 with h in {-1, 0, +1}, m in {0..3}: hi = bf16_rn(x) = h, lo = bf16_rn(x - hi) =
           sign(h) * m * 2^-10 exactly.  The lo part points away from zero: toward zero, 1 - 3 * 2^-10 would round to the
           bf16 value 1 - 2^-8 and leave the grid.
Models: bf16x3 = sum(h_a h_b + h_a l_b + l_a h_b) (the three products of mma_k16 / mma_k16_x; no lo*lo term), bf16 =
sum(h_a h_b).  Every term lies on a grid (1 for integer data, 2^-10 for split data); while the sum of |terms| of every
output stays <= 2^22 grid steps, every partial sum the kernel can form -- in any order, with any accumulator split -- is
exact in fp32 with two bits to spare, so the kernel's result must be bit-equal to the model.
"""
import math

import torch
import torch.nn.functional as F

GRID = {"integer": 1.0, "split": 2.0 ** -10}
CERT_STEPS = 2.0 ** 22          # sum of |terms| per output element, in grid steps
SUB_H, SUB_W = 4, 16            # conv_tc_kernel sub-tile (one TMA box, 64 MMA rows)
HALO_TH, HALO_TW = 8, 16        # conv64_halo_kernel / wgrad64_halo_kernel tile


# ------------------------------------------------------------------------------------------------ operands and certificate
def draw(shape, kind, density, gen, device):
    """-> (x, hi, lo), float32: x is what the library receives, (hi, lo) the split it must make of it"""
    def keep():
        return (torch.rand(shape, generator=gen, device=device) < density).float()
    if kind == "integer":
        x = torch.randint(-2, 3, shape, generator=gen, device=device).float()
        if density < 1:
            x = x * keep()
        return x, x.clone(), torch.zeros_like(x)
    h = (torch.randint(0, 2, shape, generator=gen, device=device) * 2 - 1).float() * keep()
    m = torch.randint(0, 4, shape, generator=gen, device=device).float()
    lo = h * m * 2.0 ** -10
    return h + lo, h, lo


def split_bf16(x):
    """the library's split (split_bf16_kernel, pack_weights_tc_kernel, ...): hi = bf16_rn(x), lo = bf16_rn(x - hi)"""
    hi = x.to(torch.bfloat16).float()
    return hi, (x - hi).to(torch.bfloat16).float()


def certify_operand(op):
    x, h, l = op
    hi, lo = split_bf16(x)
    assert torch.equal(hi, h), "operand off the grid: bf16_rn(x) != h"
    assert torch.equal(lo, l), "operand off the grid: bf16_rn(x - hi) != lo"
    assert torch.equal(hi + lo, x), "hi + lo != x"


def density_for(k_len, other=None, cap=0.5, target=2048.0):
    """nonzero density of a split operand for sums of length k_len (the other operand's density `other`, or the same)"""
    if other is None:
        return min(cap, math.sqrt(target / k_len))
    return min(cap, target / (k_len * other))


class Model:
    """float64 models of one bilinear op f(a, b) on exact operands, and the certificate of its fp32 exactness"""

    def __init__(self, f, a, b, kind, extra=None):
        ha, la, hb, lb = a[1].double(), a[2].double(), b[1].double(), b[2].double()
        hh = f(ha, hb)
        cross = f(ha, lb) + f(la, hb) if kind == "split" else None
        bound = f(ha.abs() + la.abs(), hb.abs() + lb.abs())
        if extra is not None:                # an addend the epilogue adds (integer)
            hh = hh + extra.double()
            bound = bound + extra.double().abs()
        self.max_steps = float(bound.max()) / GRID[kind]
        assert self.max_steps <= CERT_STEPS, "certificate: sum of |terms| reaches %.0f grid steps > 2^22" % self.max_steps
        del bound
        self.bf16 = hh
        self.bf16x3 = hh + cross if cross is not None else hh
        for m in (self.bf16, self.bf16x3):
            assert torch.equal(m.float().double(), m), "model not exact in fp32"

    def of(self, prec):
        return (self.bf16 if prec == "bf16" else self.bf16x3).float()


def nchw(t):
    return t.permute(0, 3, 1, 2).contiguous()


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def conv_fwd_fn(s, p, d):
    """x [N,H,W,Cin], w [Cout,Cin,k,k] -> y [N,Ho,Wo,Cout]"""
    return lambda x, w: nhwc(F.conv2d(nchw(x), w, None, s, p, d))


def conv_dgrad_fn(in_shape_nhwc, s, p, d):
    """dy [N,Ho,Wo,Cout], w -> dx [N,H,W,Cin]"""
    n, h, w_, c = in_shape_nhwc
    return lambda dy, w: nhwc(torch.nn.grad.conv2d_input((n, c, h, w_), w, nchw(dy), s, p, d))


def conv_wgrad_fn(w_shape, s, p, d, x_is_nchw=False):
    """dy [N,Ho,Wo,Cout], x [N,H,W,Cin] (or NCHW) -> dw [Cout,Cin,k,k]"""
    return lambda dy, x: torch.nn.grad.conv2d_weight(x if x_is_nchw else nchw(x), w_shape, nchw(dy), s, p, d)


# ------------------------------------------------------------------------------------------------ dispatch mirror
def ceil_div(a, b):
    return -(-a // b)


def worker_sms(sms, reserved):
    """engine.cu tc_worker_sms"""
    return 8 if reserved >= sms - 8 else sms - reserved


def conv_plan(N, Ho, Wo, gin, gout, k, stride, dil, workers):
    """tc_conv_planes: the kernel and work decomposition of one forward / data-gradient conv with OUTPUT size Ho x Wo,
    gin input and gout output channels"""
    if k == 3 and gin == 64 and gout == 64 and stride == 1 and dil == 1 and Ho % HALO_TH == 0 and Wo % HALO_TW == 0:
        tiles_h, tiles_w = Ho // HALO_TH, Wo // HALO_TW
        n_tiles = N * tiles_h * tiles_w
        return dict(kernel="conv64_halo_kernel", N=N, Ho=Ho, Wo=Wo, tiles_h=tiles_h, tiles_w=tiles_w, n_tiles=n_tiles,
                    grid=min(n_tiles, workers), stride=stride)
    block_n = 128 if gout % 128 == 0 else 64
    tiles_h, tiles_w = ceil_div(Ho, SUB_H), ceil_div(Wo, SUB_W)
    n_sub = N * tiles_h * tiles_w
    n_co = gout // block_n
    tiles = ceil_div(n_sub, 2) * n_co
    rem = tiles % workers
    split = 1
    if rem:
        while split * 2 <= 8 and block_n // (split * 2) >= 32 and rem * split * 2 <= workers:
            split *= 2
    full, total = tiles - rem, tiles - rem + rem * split
    if split == 1:
        full, total = tiles, tiles
    return dict(kernel="conv_tc_kernel<%d>" % block_n, N=N, Ho=Ho, Wo=Wo, block_n=block_n, tiles_h=tiles_h, tiles_w=tiles_w,
                n_sub=n_sub, n_co=n_co, full_items=full, tail_split=split, total_items=total, grid=min(total, workers),
                num_kb=k * k * (gin // 64), stride=stride)


def wgrad_chunks(tiles, total_kb, workers):
    """conv_tc.cu tc_wgrad_chunks"""
    even = tiles * total_kb / workers
    best, best_span = 1, 1e300
    for s in range(1, max(1, total_kb // 4) + 1):
        span = float(ceil_div(s * tiles, workers)) * float(ceil_div(total_kb, s))
        if span <= 1.02 * even:
            return s
        if span < best_span:
            best, best_span = s, span
    return best


def wgrad_plan(N, H, W, Cin, Cout, k, stride, dil, workers):
    """tc_wgrad_planes (H, W: input size)"""
    if k == 3 and Cin == 64 and Cout == 64 and stride == 1 and dil == 1 and H % HALO_TH == 0 and W % HALO_TW == 0:
        n_tiles = N * (H // HALO_TH) * (W // HALO_TW)
        return dict(kernel="wgrad64_halo_kernel", n_tiles=n_tiles, grid=min(n_tiles, workers), k=k, stride=stride)
    bn = 128 if Cin % 128 == 0 else 64
    Ho, Wo = H // stride, W // stride
    tiles_h, tiles_w = ceil_div(Ho, SUB_H), ceil_div(Wo, SUB_W)
    total_kb = N * tiles_h * tiles_w
    n_co, n_ci = ceil_div(Cout, 128), Cin // bn
    n_tiles = n_co * n_ci * k * k
    chunks = wgrad_chunks(n_tiles, total_kb, workers)
    return dict(kernel="wgrad_tc_kernel<%d>" % bn, bn=bn, total_kb=total_kb, n_co=n_co, n_ci=n_ci, n_tiles=n_tiles,
                chunks=chunks, grid=min(chunks * n_tiles, workers), k=k, stride=stride)


def plans(case, workers):
    """-> {"fwd": conv plan, "dgrad": conv plan (None for the stem), "wgrad": wgrad plan} of one case"""
    n, h, w, cin, cout, k, s, p, d = case["shape"]
    if case.get("stem"):
        h1, w1 = (h - 1) // 2 + 1, (w - 1) // 2 + 1
        return {"fwd": conv_plan(n, h1, w1, 192, 64, 1, 1, 1, workers), "dgrad": None,
                "wgrad": wgrad_plan(n, h1, w1, 192, 64, 1, 1, 1, workers)}
    # a stride-2 data gradient is a stride-1 conv (dil 1) over zero-inserted planes of the input's size
    dg = conv_plan(n, h, w, cout, cin, k, 1, d if s == 1 else 1, workers)
    dg["zero_insert"] = s == 2
    return {"fwd": conv_plan(n, h // s, w // s, cin, cout, k, s, d, workers), "dgrad": dg,
            "wgrad": wgrad_plan(n, h, w, cin, cout, k, s, d, workers)}


def conv_features(pl, direction):
    f = {"%s:%s" % (direction, pl["kernel"])}
    if pl["kernel"] == "conv64_halo_kernel":
        return f
    per = pl["tiles_h"] * pl["tiles_w"]
    if per % 2 == 1 and pl["N"] >= 2:
        f.add("item straddles two images")
    if pl["Ho"] % SUB_H and pl["Wo"] % SUB_W:
        f.add("sub-tiles cut in H and W")
    if pl["n_sub"] % 2:
        f.add("odd n_sub: invalid second sub-tile")
    if pl["Ho"] < SUB_H and pl["Wo"] < SUB_W:
        f.add("map smaller than one sub-tile")
    if pl["tail_split"] > 1:
        f.add("%d-channel tail pieces" % (pl["block_n"] // pl["tail_split"]))
    if pl["num_kb"] == 1:
        f.add("num_kb = 1")
    if pl["num_kb"] == 32:
        f.add("num_kb = 32")
    if pl["n_co"] == 16:
        f.add("16 channel slices")
    if direction == "fwd" and pl["stride"] == 2:
        f.add("forward stride 2 (TMA element strides)")
    if pl.get("zero_insert") and pl["block_n"] == 64 and pl["tail_split"] == 2:
        f.add("zero-inserted dgrad on conv_tc_kernel<64>, 32-channel pieces")
    return f


def wgrad_features(pl):
    f = {"wgrad:%s" % pl["kernel"]}
    if pl["kernel"].startswith("wgrad_tc"):
        f.add("wgrad S = 1" if pl["chunks"] == 1 else "wgrad S > 1")
        if pl["stride"] == 2:
            f.add("wgrad stride 2")
    return f


def case_features(case, sms):
    pl = plans(case, worker_sms(sms, reserved_for(case, sms)))
    f = conv_features(pl["fwd"], "fwd") | wgrad_features(pl["wgrad"])
    if pl["dgrad"] is not None:
        f |= conv_features(pl["dgrad"], "dgrad")
    return f


def reserved_for(case, sms):
    """the reserved-SM count a case runs at: 0, or the first count whose plan cuts the tail into the case's piece width"""
    want = case.get("pieces")
    if want is None:
        return 0
    direction, width = want
    for r in range(0, 65):
        pl = plans(case, worker_sms(sms, r))[direction]
        if pl["kernel"].startswith("conv_tc") and pl["tail_split"] > 1 and pl["block_n"] // pl["tail_split"] == width:
            return r
    raise AssertionError("no reserved-SM count gives %s %d-channel pieces for %s at %d SMs" % (direction, width, case["label"], sms))


def c(label, shape, claims, pieces=None, stem=False):
    return dict(label=label, shape=shape, claims=set(claims), pieces=pieces, stem=stem)


# label, (N, H, W, Cin, Cout, k, stride, pad, dil), the paths it must reach
CASES = [
    c("halo_small", (2, 24, 32, 64, 64, 3, 1, 1, 1), ["fwd:conv64_halo_kernel", "dgrad:conv64_halo_kernel", "wgrad:wgrad64_halo_kernel"]),
    c("halo_bench", (16, 120, 160, 64, 64, 3, 1, 1, 1), ["fwd:conv64_halo_kernel", "dgrad:conv64_halo_kernel", "wgrad:wgrad64_halo_kernel"]),
    c("bn64_dil2", (2, 24, 32, 64, 64, 3, 1, 2, 2), ["fwd:conv_tc_kernel<64>", "dgrad:conv_tc_kernel<64>", "wgrad:wgrad_tc_kernel<64>"]),
    c("straddle", (2, 12, 16, 128, 128, 3, 1, 1, 1), ["fwd:conv_tc_kernel<128>", "item straddles two images"]),
    c("partial", (2, 13, 9, 256, 256, 3, 1, 2, 2), ["sub-tiles cut in H and W"]),
    c("partial_odd", (3, 11, 9, 256, 256, 3, 1, 2, 2), ["odd n_sub: invalid second sub-tile"]),
    c("tiny", (1, 3, 5, 512, 512, 3, 1, 4, 4), ["map smaller than one sub-tile"]),
    c("layer3", (16, 60, 80, 256, 256, 3, 1, 2, 2), ["fwd:conv_tc_kernel<128>", "wgrad:wgrad_tc_kernel<128>", "32-channel tail pieces"],
      pieces=("fwd", 32)),
    c("layer4", (16, 60, 80, 512, 512, 3, 1, 4, 4), ["fwd:conv_tc_kernel<128>", "32-channel tail pieces", "wgrad S > 1"],
      pieces=("fwd", 32)),
    c("tail64", (16, 60, 80, 512, 512, 3, 1, 4, 4), ["64-channel tail pieces"], pieces=("fwd", 64)),
    c("s2_3x3", (16, 120, 160, 64, 128, 3, 2, 1, 1), ["forward stride 2 (TMA element strides)", "wgrad stride 2",
                                                      "zero-inserted dgrad on conv_tc_kernel<64>, 32-channel pieces"],
      pieces=("dgrad", 32)),
    c("s2_1x1", (16, 120, 160, 256, 512, 1, 2, 0, 1), ["forward stride 2 (TMA element strides)", "wgrad stride 2"]),
    c("one_kblock", (16, 120, 160, 64, 256, 1, 1, 0, 1), ["num_kb = 1"]),
    c("wide_in", (16, 60, 80, 2048, 512, 1, 1, 0, 1), ["num_kb = 32"]),
    c("wide_out", (16, 60, 80, 512, 2048, 1, 1, 0, 1), ["16 channel slices"]),
    c("stem_partial", (4, 488, 648, 3, 64, 7, 2, 3, 1), ["fwd:conv_tc_kernel<64>", "wgrad:wgrad_tc_kernel<64>"], stem=True),
    c("stem_bench", (16, 480, 640, 3, 64, 7, 2, 3, 1), ["fwd:conv_tc_kernel<64>"], stem=True),
]
CONV_CASES = [k for k in CASES if not k["stem"]]
STEM_CASES = [k for k in CASES if k["stem"]]
BY_LABEL = {k["label"]: k for k in CASES}

REQUIRED = {
    "fwd:conv64_halo_kernel", "dgrad:conv64_halo_kernel", "wgrad:wgrad64_halo_kernel",
    "fwd:conv_tc_kernel<64>", "dgrad:conv_tc_kernel<64>", "wgrad:wgrad_tc_kernel<64>",
    "fwd:conv_tc_kernel<128>", "dgrad:conv_tc_kernel<128>", "wgrad:wgrad_tc_kernel<128>",
    "item straddles two images", "sub-tiles cut in H and W", "odd n_sub: invalid second sub-tile", "map smaller than one sub-tile",
    "32-channel tail pieces", "64-channel tail pieces", "forward stride 2 (TMA element strides)",
    "zero-inserted dgrad on conv_tc_kernel<64>, 32-channel pieces", "num_kb = 1", "num_kb = 32", "16 channel slices",
    "wgrad stride 2", "wgrad S = 1", "wgrad S > 1",
}


def coverage(sms):
    """-> (features reached by the case list, per-case claims not reached)"""
    seen, missed = set(), {}
    for case in CASES:
        f = case_features(case, sms)
        seen |= f
        if not case["claims"] <= f:
            missed[case["label"]] = sorted(case["claims"] - f)
    return seen, missed


# ------------------------------------------------------------------------------------------------ failure report
def locate_conv(pl, n, h, w, ch):
    """where output element (n, h, w, ch) of a forward / data-gradient conv is computed"""
    if pl["kernel"] == "conv64_halo_kernel":
        t = (n * pl["tiles_h"] + h // HALO_TH) * pl["tiles_w"] + w // HALO_TW
        return "halo tile %d (h0 %d, w0 %d, warpgroup %d) on CTA %d, its tile %d" % (
            t, h // HALO_TH * HALO_TH, w // HALO_TW * HALO_TW, (w % HALO_TW) // 8, t % pl["grid"], t // pl["grid"])
    st = (n * pl["tiles_h"] + h // SUB_H) * pl["tiles_w"] + w // SUB_W
    sp, wg = st // 2, st % 2
    bn, split = pl["block_n"], pl["tail_split"]
    tile = sp * pl["n_co"] + ch // bn
    if tile < pl["full_items"]:
        idx, width, co0 = tile, bn, ch // bn * bn
    else:
        width = bn // split
        piece = (ch % bn) // width
        idx = pl["full_items"] + (tile - pl["full_items"]) * split + piece
        co0 = ch // bn * bn + piece * width
    return "sub-tile %d (h0 %d, w0 %d, warpgroup %d), item %d on CTA %d, channels %d..%d (%s), k-blocks 0..%d" % (
        st, h // SUB_H * SUB_H, w // SUB_W * SUB_W, wg, idx, idx % pl["grid"], co0, co0 + width - 1,
        "full tile" if width == bn else "tail piece", pl["num_kb"] - 1)


def locate_wgrad(pl, co, ci, r, s):
    """where weight-gradient element dw[co, ci, r, s] is accumulated"""
    tap = r * pl["k"] + s
    if pl["kernel"] == "wgrad64_halo_kernel":
        return "tap %d (warpgroup %d), summed over %d halo tiles by %d CTAs" % (tap, r, pl["n_tiles"], pl["grid"])
    tile = co // 128 + pl["n_co"] * (ci // pl["bn"] + pl["n_ci"] * tap)
    items = ["item %d (CTA %d, k-blocks %d..%d)" % (cc * pl["n_tiles"] + tile, (cc * pl["n_tiles"] + tile) % pl["grid"],
                                                     cc * pl["total_kb"] // pl["chunks"], (cc + 1) * pl["total_kb"] // pl["chunks"] - 1)
             for cc in range(min(pl["chunks"], 3))]
    return "tap %d, tile %d (co0 %d, ci0 %d, warpgroup %d), %d chunk(s): %s%s" % (
        tap, tile, co // 128 * 128, ci // pl["bn"] * pl["bn"], (co % 128) // 64, pl["chunks"], ", ".join(items),
        ", ..." if pl["chunks"] > 3 else "")
