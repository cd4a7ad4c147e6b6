"""Thin functional wrappers over the single-operator C-ABI entry points (used by the unit tests and as
building blocks).  NHWC fp32 CUDA tensors in, NHWC fp32 CUDA tensors out; no autograd here."""
import torch

from . import _native as N


def _ws(nbytes, device):
    return torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=device)


def conv2d_forward(x_nhwc, w_oihw, stride=1, pad=0, dil=1, precision=N.PRECISION_FP32_SIMT):
    N.require_cuda_f32(x_nhwc, "x"); N.require_cuda_f32(w_oihw, "w")
    n, h, w, cin = x_nhwc.shape
    cout, cin2, k, k2 = w_oihw.shape
    assert cin == cin2 and k == k2
    ho = (h + 2 * pad - dil * (k - 1) - 1) // stride + 1
    wo = (w + 2 * pad - dil * (k - 1) - 1) // stride + 1
    y = torch.empty(n, ho, wo, cout, dtype=torch.float32, device=x_nhwc.device)
    nb = N.lib.ddn_conv2d_workspace_bytes(n, h, w, cin, cout, k, stride, pad, dil, precision)
    ws = _ws(nb, x_nhwc.device)
    N.check(N.lib.ddn_conv2d_forward(N.ptr(x_nhwc), N.ptr(w_oihw), N.ptr(y), n, h, w, cin, cout, k, stride, pad, dil,
                                     precision, N.ptr(ws), ws.numel(), N.stream_ptr()))
    return y


def conv2d_backward(x_nhwc, w_oihw, dy_nhwc, stride=1, pad=0, dil=1, need_dx=True, precision=N.PRECISION_FP32_SIMT):
    N.require_cuda_f32(x_nhwc, "x"); N.require_cuda_f32(w_oihw, "w"); N.require_cuda_f32(dy_nhwc, "dy")
    n, h, w, cin = x_nhwc.shape
    cout, _, k, _ = w_oihw.shape
    dx = torch.empty_like(x_nhwc) if need_dx else None
    dw = torch.empty_like(w_oihw)
    nb = N.lib.ddn_conv2d_workspace_bytes(n, h, w, cin, cout, k, stride, pad, dil, precision)
    ws = _ws(nb, x_nhwc.device)
    N.check(N.lib.ddn_conv2d_backward(N.ptr(x_nhwc), N.ptr(w_oihw), N.ptr(dy_nhwc), N.ptr(dx), N.ptr(dw),
                                      n, h, w, cin, cout, k, stride, pad, dil, precision, N.ptr(ws), ws.numel(),
                                      N.stream_ptr()))
    return dx, dw


def _out_hw(h, w, k, stride, pad, dil):
    return (h + 2 * pad - dil * (k - 1) - 1) // stride + 1, (w + 2 * pad - dil * (k - 1) - 1) // stride + 1


def _fused_ws(n, h, w, cin, cout, k, stride, pad, dil, precision, device):
    nb = N.lib.ddn_conv2d_fused_workspace_bytes(n, h, w, cin, cout, k, stride, pad, dil, precision)
    return _ws(nb, device)


def conv2d_bn_stats_forward(x, w_oihw, stride=1, pad=0, dil=1, bn_groups=1, running_mean=None, running_var=None,
                            momentum=0.1, eps=1e-5, precision=N.PRECISION_BF16X3):
    """Tensor-core conv + the batch statistics of its output per BatchNorm group (training-forward epilogue).
    x is NHWC, or NCHW [N,3,H,W] for the stem (Cin 3, 7x7, stride 2, pad 3).  running_mean / running_var are updated in place.
    -> (raw [N,Ho,Wo,Cout], mean [G,Cout], invstd [G,Cout])"""
    N.require_cuda_f32(x, "x"); N.require_cuda_f32(w_oihw, "w")
    cout, cin, k, _ = w_oihw.shape
    if cin == 3 and k == 7:
        n, _, h, w = x.shape
    else:
        n, h, w, cin2 = x.shape
        assert cin2 == cin
    ho, wo = _out_hw(h, w, k, stride, pad, dil)
    raw = torch.empty(n, ho, wo, cout, dtype=torch.float32, device=x.device)
    mean = torch.empty(bn_groups, cout, dtype=torch.float32, device=x.device)
    invstd = torch.empty_like(mean)
    ws = _fused_ws(n, h, w, cin, cout, k, stride, pad, dil, precision, x.device)
    N.check(N.lib.ddn_conv2d_bn_stats_forward(N.ptr(x), N.ptr(w_oihw), N.ptr(raw), N.ptr(mean), N.ptr(invstd), N.ptr(running_mean),
                                              N.ptr(running_var), n, h, w, cin, cout, k, stride, pad, dil, bn_groups, momentum, eps,
                                              precision, N.ptr(ws), ws.numel(), N.stream_ptr()))
    return raw, mean, invstd


def conv2d_folded_forward(x, w_oihw, gamma, beta, running_mean, running_var, stride=1, pad=0, dil=1, addend=None, relu=True,
                          eps=1e-5, want_y=True, want_planes=False, y_lo=None, precision=N.PRECISION_BF16X3):
    """Tensor-core conv with eval-mode BatchNorm, addend and ReLU folded into its epilogue (inference).
    want_planes: also (or, with want_y=False, only) the bf16 operand planes of y.  y_lo: optional caller tensor for the lo plane.
    -> (y fp32 or None, y_hi bf16 or None, y_lo bf16 or None)"""
    N.require_cuda_f32(x, "x"); N.require_cuda_f32(w_oihw, "w")
    n, h, w, cin = x.shape
    cout, _, k, _ = w_oihw.shape
    ho, wo = _out_hw(h, w, k, stride, pad, dil)
    y = torch.empty(n, ho, wo, cout, dtype=torch.float32, device=x.device) if want_y else None
    y_hi = torch.empty(n, ho, wo, cout, dtype=torch.bfloat16, device=x.device) if want_planes else None
    if want_planes and y_lo is None:
        y_lo = torch.empty_like(y_hi)
    ws = _fused_ws(n, h, w, cin, cout, k, stride, pad, dil, precision, x.device)
    N.check(N.lib.ddn_conv2d_folded_forward(N.ptr(x), N.ptr(w_oihw), N.ptr(gamma), N.ptr(beta), N.ptr(running_mean), N.ptr(running_var),
                                            N.ptr(addend), N.ptr(y), N.ptr(y_hi), N.ptr(y_lo), n, h, w, cin, cout, k, stride, pad, dil,
                                            int(relu), eps, precision, N.ptr(ws), ws.numel(), N.stream_ptr()))
    return y, y_hi, y_lo


def conv2d_backward_data_bn_stats(w_oihw, dy, raw, mean, invstd, gamma, beta, stride=1, pad=0, dil=1, addend=None, y_hi=None,
                                  precision=N.PRECISION_BF16X3):
    """Tensor-core data gradient dx = conv2d_input(dy, w) + addend, with the column sums of the BatchNorm backward that consumes
    dx (raw [N,H,W,Cin], mean / invstd [G,Cin]; ReLU mask from the bf16 plane y_hi, or recomputed from raw when y_hi is None).
    -> (dx, dgamma [Cin], dbeta [Cin], sums [G,2,Cin])"""
    N.require_cuda_f32(w_oihw, "w"); N.require_cuda_f32(dy, "dy"); N.require_cuda_f32(raw, "raw")
    n, h, w, cin = raw.shape
    cout, _, k, _ = w_oihw.shape
    G = mean.shape[0]
    dx = torch.empty_like(raw)
    dgamma = torch.empty(cin, dtype=torch.float32, device=raw.device)
    dbeta = torch.empty_like(dgamma)
    sums = torch.empty(G, 2, cin, dtype=torch.float32, device=raw.device)
    ws = _fused_ws(n, h, w, cin, cout, k, stride, pad, dil, precision, raw.device)
    N.check(N.lib.ddn_conv2d_backward_data_bn_stats(N.ptr(w_oihw), N.ptr(dy), N.ptr(addend), N.ptr(raw), N.ptr(mean), N.ptr(invstd),
                                                    N.ptr(gamma), N.ptr(beta), N.ptr(y_hi), N.ptr(dx), N.ptr(dgamma), N.ptr(dbeta),
                                                    N.ptr(sums), n, h, w, cin, cout, k, stride, pad, dil, G, precision, N.ptr(ws),
                                                    ws.numel(), N.stream_ptr()))
    return dx, dgamma, dbeta, sums


def stem_pool_forward(raw, mean, invstd, gamma, beta, want_y=True, want_planes=False, want_lo=True):
    """The stem's bn1 -> ReLU -> max-pool 3x3/2 on conv1's output raw [N,Hc,Wc,64]; mean / invstd [G,64] per BatchNorm group.
    -> (y [N,Hp,Wp,64] fp32 or None, y_hi bf16 or None, y_lo bf16 or None, argmax uint8 [N,Hp,Wp,64])"""
    N.require_cuda_f32(raw, "raw")
    n, hc, wc, c = raw.shape
    assert c == 64
    hp, wp = (hc - 1) // 2 + 1, (wc - 1) // 2 + 1
    y = torch.empty(n, hp, wp, 64, dtype=torch.float32, device=raw.device) if want_y else None
    y_hi = torch.empty(n, hp, wp, 64, dtype=torch.bfloat16, device=raw.device) if want_planes else None
    y_lo = torch.empty_like(y_hi) if want_planes and want_lo else None
    argmax = torch.empty(n, hp, wp, 64, dtype=torch.uint8, device=raw.device)
    N.check(N.lib.ddn_stem_pool_forward(N.ptr(raw), N.ptr(mean), N.ptr(invstd), N.ptr(gamma), N.ptr(beta), N.ptr(y), N.ptr(y_hi),
                                        N.ptr(y_lo), N.ptr(argmax), n, hc, wc, mean.shape[0], N.stream_ptr()))
    return y, y_hi, y_lo, argmax


def stem_backward(x, raw, mean, invstd, gamma, beta, argmax, dy_pool, training=True, want_g=False, want_dx=False,
                  want_planes=False, precision=N.PRECISION_BF16X3):
    """The network's stem backward (pool / ReLU -> bn1 -> conv1 weight gradient) for the NCHW image x [N,3,H,W].
    want_planes (tensor cores): also the bf16 planes of d raw that the weight gradient reads (lo: BF16X3 only).
    -> (dw_conv1 [64,3,7,7], dgamma [64], dbeta [64], g or None, dx_bn or None, dx_hi or None, dx_lo or None), [N,Hc,Wc,64] each"""
    for t, name in ((x, "x"), (raw, "raw"), (dy_pool, "dy_pool")):
        N.require_cuda_f32(t, name)
    n, _, h, w = x.shape
    dw = torch.empty(64, 3, 7, 7, dtype=torch.float32, device=x.device)
    dgamma = torch.empty(64, dtype=torch.float32, device=x.device)
    dbeta = torch.empty_like(dgamma)
    g = torch.empty_like(raw) if want_g else None
    dx = torch.empty_like(raw) if want_dx else None
    dx_hi = torch.empty(raw.shape, dtype=torch.bfloat16, device=x.device) if want_planes else None
    dx_lo = torch.empty_like(dx_hi) if want_planes and precision == N.PRECISION_BF16X3 else None
    ws = _ws(N.lib.ddn_stem_workspace_bytes(n, h, w, precision), x.device)
    N.check(N.lib.ddn_stem_backward(N.ptr(x), N.ptr(raw), N.ptr(mean), N.ptr(invstd), N.ptr(gamma), N.ptr(beta), N.ptr(argmax),
                                    N.ptr(dy_pool), N.ptr(g), N.ptr(dx), N.ptr(dx_hi), N.ptr(dx_lo), N.ptr(dgamma), N.ptr(dbeta),
                                    N.ptr(dw), n, h, w, mean.shape[0], int(training), precision, N.ptr(ws), ws.numel(),
                                    N.stream_ptr()))
    return dw, dgamma, dbeta, g, dx, dx_hi, dx_lo


def batchnorm_forward(x, gamma, beta, residual=None, relu=False, training=True, running_mean=None, running_var=None,
                      momentum=0.1, eps=1e-5):
    """x [..., C] channels-last.  -> (y, save_mean, save_invstd)"""
    N.require_cuda_f32(x, "x")
    C = x.shape[-1]
    M = x.numel() // C
    y = torch.empty_like(x)
    mean = torch.empty(C, dtype=torch.float32, device=x.device)
    invstd = torch.empty(C, dtype=torch.float32, device=x.device)
    nb = N.lib.ddn_batchnorm_workspace_bytes(M, C)
    ws = _ws(nb, x.device)
    N.check(N.lib.ddn_batchnorm_forward(N.ptr(x), N.ptr(gamma), N.ptr(beta), N.ptr(residual), N.ptr(y), N.ptr(mean),
                                        N.ptr(invstd), N.ptr(running_mean), N.ptr(running_var), M, C, int(relu),
                                        int(training), momentum, eps, N.ptr(ws), ws.numel(), N.stream_ptr()))
    return y, mean, invstd


def batchnorm_backward(dy, x, y, gamma, mean, invstd, relu=False, need_residual_grad=False):
    N.require_cuda_f32(dy, "dy")
    C = x.shape[-1]
    M = x.numel() // C
    dx = torch.empty_like(x)
    dgamma = torch.empty(C, dtype=torch.float32, device=x.device)
    dbeta = torch.empty(C, dtype=torch.float32, device=x.device)
    dres = torch.empty_like(x) if need_residual_grad else None
    ws = _ws(N.lib.ddn_batchnorm_workspace_bytes(M, C), x.device)
    N.check(N.lib.ddn_batchnorm_backward(N.ptr(dy), N.ptr(x), N.ptr(y), N.ptr(gamma), N.ptr(mean), N.ptr(invstd),
                                         N.ptr(dx), N.ptr(dgamma), N.ptr(dbeta), N.ptr(dres), M, C, int(relu),
                                         N.ptr(ws), ws.numel(), N.stream_ptr()))
    return dx, dgamma, dbeta, dres


def upsample_bilinear_forward(x, H, W):
    """x [N,C,h,w] -> [N,C,H,W], align_corners=True."""
    N.require_cuda_f32(x, "x")
    n, c, h, w = x.shape
    y = torch.empty(n, c, H, W, dtype=torch.float32, device=x.device)
    N.check(N.lib.ddn_upsample_bilinear_forward(N.ptr(x), N.ptr(y), n * c, h, w, H, W, N.stream_ptr()))
    return y


def upsample_bilinear_backward(dy, h, w):
    N.require_cuda_f32(dy, "dy")
    n, c, H, W = dy.shape
    dx = torch.empty(n, c, h, w, dtype=torch.float32, device=dy.device)
    N.check(N.lib.ddn_upsample_bilinear_backward(N.ptr(dy), N.ptr(dx), n * c, h, w, H, W, N.stream_ptr()))
    return dx


def _fc_features(feat, feat_lo):
    """feat [N, ..., C]: fp32, or the bf16 hi plane (with its lo plane feat_lo, or alone) -> (fp32, hi, lo, N, Mimg, C)"""
    if not isinstance(feat, torch.Tensor) or not feat.is_cuda or not feat.is_contiguous():
        raise RuntimeError("feat must be a contiguous CUDA tensor: this path has no CPU fallback")
    n, c = feat.shape[0], feat.shape[-1]
    if feat.dtype == torch.bfloat16:
        if feat_lo is not None and (feat_lo.dtype != torch.bfloat16 or feat_lo.shape != feat.shape or not feat_lo.is_contiguous()):
            raise RuntimeError("feat_lo must be a contiguous bf16 plane of feat's shape")
        return None, feat, feat_lo, n, feat.numel() // (n * c), c
    N.require_cuda_f32(feat, "feat")
    if feat_lo is not None:
        raise RuntimeError("feat_lo goes with a bf16 hi plane, not with fp32 features")
    return feat, None, None, n, feat.numel() // (n * c), c


def fc_forward(feat, w, bias, feat_lo=None, low=None, low_nhwc=None):
    """The scoring 1x1 conv + bias.  feat [N, ..., C] channels-last (fp32, or bf16 planes feat = hi + feat_lo), w [D, C], bias [D].
    low [N, D, Mimg] is allocated when None; low_nhwc [N, Mimg, D] is written only when given.  -> (low, low_nhwc)"""
    f32, hi, lo, n, mimg, c = _fc_features(feat, feat_lo)
    N.require_cuda_f32(w, "w"); N.require_cuda_f32(bias, "bias")
    d = w.shape[0]
    if low is None:
        low = torch.empty(n, d, mimg, dtype=torch.float32, device=feat.device)
    N.check(N.lib.ddn_fc_forward(N.ptr(f32), N.ptr(hi), N.ptr(lo), N.ptr(w), N.ptr(bias), N.ptr(low), N.ptr(low_nhwc), mimg, n, c, d,
                                 N.stream_ptr()))
    return low, low_nhwc


def fc_backward(dlow, feat, w, feat_lo=None, dfeat=None, dw=None, dbias=None, workspace=None):
    """dlow [N, D, Mimg] -> (dfeat [N*Mimg, C], dw [D, C], dbias [D]); outputs and the workspace are allocated when None."""
    f32, hi, lo, n, mimg, c = _fc_features(feat, feat_lo)
    N.require_cuda_f32(dlow, "dlow"); N.require_cuda_f32(w, "w")
    d = w.shape[0]
    dfeat = torch.empty(n * mimg, c, dtype=torch.float32, device=feat.device) if dfeat is None else dfeat
    dw = torch.empty_like(w) if dw is None else dw
    dbias = torch.empty(d, dtype=torch.float32, device=feat.device) if dbias is None else dbias
    ws = _ws(N.lib.ddn_fc_workspace_bytes(c, d), feat.device) if workspace is None else workspace
    N.check(N.lib.ddn_fc_backward(N.ptr(dlow), N.ptr(f32), N.ptr(hi), N.ptr(lo), N.ptr(w), N.ptr(dfeat), N.ptr(dw), N.ptr(dbias),
                                  mimg, n, c, d, N.ptr(ws), ws.numel() * ws.element_size(), N.stream_ptr()))
    return dfeat, dw, dbias


def scale_inplace(t, scale):
    N.require_cuda_f32(t, "t")
    N.check(N.lib.ddn_scale_inplace(N.ptr(t), t.numel(), float(scale), N.stream_ptr()))
    return t
