"""CPU: libddn_b200.so loads without a GPU, exports every function include/ddn_b200.h declares, describes the
parameter layout of the reference state dict, and rejects contract violations before touching the device."""
import ctypes
import os
import re

import pytest
import torch

import pdc_b200
from pdc_b200 import _native as N
from oracle.resnet34_8s_oracle import seeded_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_functions():
    text = open(os.path.join(ROOT, "include", "ddn_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(ddn_[a-z0-9_]+)\s*\(", text)))


def test_header_symbols_exported_and_bound():
    names = _declared_functions()
    assert len(names) >= 20
    lib = ctypes.CDLL(N.LIB_PATH)
    for n in names:
        assert hasattr(lib, n), "declared in ddn_b200.h but not exported: " + n
    assert set(names) == set(N.EXPORTED_SYMBOLS), set(names) ^ set(N.EXPORTED_SYMBOLS)
    assert N.lib.ddn_abi_version() == 3


@pytest.mark.parametrize("D", [3, 8, 16])
def test_param_table_is_reference_state_dict(D):
    sd = seeded_oracle(D).state_dict()
    learn = [(k, tuple(v.shape)) for k, v in seeded_oracle(D).named_parameters()]
    tab = N.param_table(D)
    assert [("resnet34_8s." + n, s) for n, s, _, _ in tab] == learn
    assert len(tab) == 110
    # offsets: in order, non-overlapping, 16-byte aligned
    end = 0
    for _, s, off, n in tab:
        assert off >= end and off % 4 == 0
        end = off + n
    assert N.lib.ddn_resnet34_8s_param_count(D) >= end
    assert sum(n for _, _, _, n in tab) == sum(v.numel() for k, v in seeded_oracle(D).named_parameters())
    btab = N.buffer_table()
    assert len(btab) == 72
    for name, shape, _, _ in btab:
        assert tuple(sd["resnet34_8s." + name].shape) == shape
    m = pdc_b200.Resnet34_8s(num_classes=D)
    assert list(m.state_dict().keys()) == list(sd.keys()) and len(sd) == 218
    m.load_state_dict(sd)
    for k, v in m.state_dict().items():
        assert torch.equal(v, sd[k]), k
    # every parameter aliases the flat array at the advertised offset
    for (name, shape, off, n), p in zip(tab, m._params):
        assert p.data_ptr() == m._flat.data_ptr() + 4 * off


def test_workspace_and_argument_checks():
    wb = N.lib.ddn_resnet34_8s_workspace_bytes(1, 480, 640, 3, 1, N.PRECISION_FP32_SIMT)
    assert 3e8 < wb < 2e9
    assert N.lib.ddn_resnet34_8s_workspace_bytes(2, 480, 640, 3, 1, 0) > 1.9 * wb - 5e7
    assert N.lib.ddn_resnet34_8s_workspace_bytes(1, 481, 640, 3, 1, 0) == 0          # H not a multiple of 8
    assert N.lib.ddn_resnet34_8s_workspace_bytes(1, 480, 640, 33, 1, 0) == 0         # D out of range
    assert b"multiple" in N.lib.ddn_last_error() or b"dimension" in N.lib.ddn_last_error()
    # null pointers / bad sizes are refused with DDN_EINVAL and never reach a kernel launch
    before = N.launch_count()
    assert N.lib.ddn_resnet34_8s_forward(None, None, None, None, None, 0, 1, 480, 640, 3, 1, 1, 0.1, 1e-5, 0, None, None) == -1
    assert N.lib.ddn_contrastive_terms_forward(None, None, 0, 0, 0, 1, 10, 3, 4, None, 0, None, None, None) == -1
    assert N.lib.ddn_upsample_bilinear_forward(None, None, 1, 1, 1, 1, 1, None) == -1
    assert N.lib.ddn_conv2d_workspace_bytes(1, 60, 80, 64, 64, 3, 1, 1, 1, 0) >= 3 * 9 * 64 * 64 * 4
    assert N.lib.ddn_batchnorm_workspace_bytes(4800, 6) == 0 and N.lib.ddn_batchnorm_workspace_bytes(4800, 512) > 0
    assert N.launch_count() == before
    # the fused-epilogue conv entries: every refusal happens before the first launch (fake, never dereferenced pointers)
    fake = ctypes.c_void_p(1 << 40)
    big = 1 << 40
    X3 = N.PRECISION_BF16X3
    assert N.lib.ddn_conv2d_fused_workspace_bytes(2, 24, 32, 64, 64, 3, 1, 1, 1, X3) > 0
    assert N.lib.ddn_conv2d_fused_workspace_bytes(2, 24, 32, 64, 64, 3, 1, 1, 1, N.PRECISION_FP32_SIMT) == 0

    def stats(n=2, h=24, w=32, cin=64, cout=64, k=3, s=1, p=1, d=1, G=1, prec=X3, x=fake):
        return N.lib.ddn_conv2d_bn_stats_forward(x, fake, fake, fake, fake, None, None, n, h, w, cin, cout, k, s, p, d, G, 0.1, 1e-5,
                                                 prec, fake, big, None)

    def folded(n=2, h=24, w=32, cin=64, cout=64, k=3, s=1, p=1, d=1, prec=X3, y=fake, y_hi=None, y_lo=None, x=fake):
        return N.lib.ddn_conv2d_folded_forward(x, fake, fake, fake, fake, fake, None, y, y_hi, y_lo, n, h, w, cin, cout, k, s, p, d, 1,
                                               1e-5, prec, fake, big, None)

    def dgrad(n=2, h=24, w=32, cin=64, cout=64, k=3, s=1, p=1, d=1, G=1, prec=X3, dy=fake, y_hi=None, gamma=fake):
        return N.lib.ddn_conv2d_backward_data_bn_stats(fake, dy, None, fake, fake, fake, gamma, fake, y_hi, fake, fake, fake, fake,
                                                       n, h, w, cin, cout, k, s, p, d, G, prec, fake, big, None)

    for call in (stats, dgrad):
        assert call(G=3) == -1                                       # G = 3
        assert call(n=3, G=2) == -1                                  # N % G != 0
    assert stats(x=None) == -1 and folded(x=None) == -1 and dgrad(dy=None) == -1              # null pointers
    assert folded(y=None) == -1                                      # no output at all
    assert folded(y_lo=fake) == -1                                   # a lo plane without its hi plane
    assert dgrad(gamma=None) == -1                                   # recomputed mask without gamma
    for call in (stats, folded, dgrad):
        assert call(prec=N.PRECISION_FP32_SIMT) == -3                # no fused epilogues on the CUDA cores
        assert call(prec=7) == -1
        assert call(cin=48) == -3                                    # unsupported shape
        assert call(k=5, p=2) == -3
    assert stats(n=3, h=64, w=96, cin=3, k=7, s=2, p=3, G=2) == -1  # stem: G does not divide N
    assert folded(cin=3, k=7, s=2, p=3) == -3 and dgrad(cin=3, k=7, s=2, p=3) == -3
    assert N.lib.ddn_conv2d_bn_stats_forward(fake, fake, fake, fake, fake, None, None, 2, 24, 32, 64, 64, 3, 1, 1, 1, 1, 0.1, 1e-5,
                                             X3, fake, 1024, None) == -1             # workspace too small
    assert N.launch_count() == before
    # SM reservation for a concurrent collective: a host-side setting with a range check (INTEGRATION.md A, data parallel)
    assert N.lib.ddn_set_reserved_sms(8) == 0 and N.lib.ddn_set_reserved_sms(0) == 0
    assert N.lib.ddn_set_reserved_sms(-1) == -1 and N.lib.ddn_set_reserved_sms(1000) == -1
    with pytest.raises(N.DdnError):
        N.check(-1)


def test_fc_entries_refuse_before_any_launch():
    """ddn_fc_forward / ddn_fc_backward check every argument before the first launch (fake, never dereferenced pointers:
    each call below fails one check)."""
    fake = ctypes.c_void_p(1 << 40)                 # 16-byte aligned
    assert N.lib.ddn_fc_workspace_bytes(512, 3) == 4 * 512 * (3 * 512 + 3)      # 512 slots for the 512-channel trunk
    assert N.lib.ddn_fc_workspace_bytes(1024, 32) == 4 * 64 * (32 * 1024 + 32)  # 64 for wider ones
    assert N.lib.ddn_fc_workspace_bytes(2048, 1) == 4 * 64 * (2048 + 1)
    for C, D in ((640, 3), (256, 3), (0, 3), (512, 0), (512, 33)):
        assert N.lib.ddn_fc_workspace_bytes(C, D) == 0
    ws_bytes = N.lib.ddn_fc_workspace_bytes(512, 3)

    def fwd(feat=fake, hi=None, lo=None, w=fake, low=fake, mimg=77, n=3, C=512, D=3):
        return N.lib.ddn_fc_forward(feat, hi, lo, w, fake, low, fake, mimg, n, C, D, None)

    def bwd(feat=fake, hi=None, lo=None, w=fake, dfeat=fake, mimg=77, n=3, C=512, D=3, ws=fake, nbytes=ws_bytes):
        return N.lib.ddn_fc_backward(fake, feat, hi, lo, w, dfeat, fake, fake, mimg, n, C, D, ws, nbytes, None)

    def off(nbytes):
        return ctypes.c_void_p((1 << 40) + nbytes)

    before = N.launch_count()
    for call in (fwd, bwd):
        for C in (640, 256):
            assert call(C=C) == -1 and b"multiple of 512" in N.lib.ddn_last_error()
        for D in (0, 33):
            assert call(D=D) == -1 and b"1<=D<=32" in N.lib.ddn_last_error()
        assert call(feat=None) == -1 and b"exactly one feature source" in N.lib.ddn_last_error()     # no source
        assert call(hi=fake) == -1 and b"exactly one feature source" in N.lib.ddn_last_error()       # fp32 and planes
        assert call(lo=fake) == -1 and b"feat_lo" in N.lib.ddn_last_error()                          # lo without hi
        assert call(feat=None, lo=fake) == -1                                                        # lo alone
        assert call(n=0) == -1 and call(mimg=0) == -1
        assert call(w=None) == -1
        assert call(feat=off(8)) == -1 and b"16-byte" in N.lib.ddn_last_error()
        assert call(feat=None, hi=off(8)) == -1 and b"16-byte" in N.lib.ddn_last_error()
        assert call(feat=None, hi=fake, lo=off(4)) == -1 and b"16-byte" in N.lib.ddn_last_error()
    assert fwd(low=None) == -1
    assert bwd(dfeat=off(4)) == -1 and b"dfeat" in N.lib.ddn_last_error()
    assert bwd(nbytes=ws_bytes - 4) == -1 and b"workspace" in N.lib.ddn_last_error()
    assert bwd(ws=off(2)) == -1 and b"workspace" in N.lib.ddn_last_error()
    assert bwd(ws=None) == -1
    assert N.launch_count() == before


def test_stem_entries_refuse_before_any_launch():
    """ddn_stem_pool_forward / ddn_stem_backward check every argument before the first launch (fake, never dereferenced
    pointers: each call below fails one check)."""
    fake = ctypes.c_void_p(1 << 40)
    X3, SIMT = N.PRECISION_BF16X3, N.PRECISION_FP32_SIMT
    ws_x3 = N.lib.ddn_stem_workspace_bytes(2, 64, 96, X3)
    ws_simt = N.lib.ddn_stem_workspace_bytes(2, 64, 96, SIMT)
    m1 = 2 * 32 * 48
    assert ws_x3 >= m1 * 64 * (4 + 4 + 2 + 2) + m1 * 192 * 4 + 64 * 192 * 8      # g, dx, dx planes, patch planes, fp64 dW
    assert ws_simt >= m1 * 64 * 8 + 2 * 64 * 96 * 4 * 4                          # g, dx, the NHWC4 image
    assert N.lib.ddn_stem_workspace_bytes(2, 64, 96, N.PRECISION_BF16) > 0
    for n, h, w, prec in ((0, 64, 96, X3), (2, 0, 96, X3), (2, 64, 0, X3), (2, 64, 96, 3), (2, 64, 96, -1)):
        assert N.lib.ddn_stem_workspace_bytes(n, h, w, prec) == 0

    def pool(raw=fake, mean=fake, y=fake, y_hi=None, y_lo=None, argmax=fake, n=2, hc=32, wc=48, G=1):
        return N.lib.ddn_stem_pool_forward(raw, mean, fake, fake, fake, y, y_hi, y_lo, argmax, n, hc, wc, G, None)

    def bwd(x=fake, argmax=fake, dy=fake, dw=fake, dgamma=fake, n=2, h=64, w=96, G=1, prec=X3, ws=fake, nbytes=None):
        nbytes = N.lib.ddn_stem_workspace_bytes(n, h, w, prec) if nbytes is None else nbytes
        return N.lib.ddn_stem_backward(x, fake, fake, fake, fake, fake, argmax, dy, None, None, None, None, dgamma, fake, dw,
                                       n, h, w, G, 1, prec, ws, nbytes, None)

    before = N.launch_count()
    assert pool(raw=None) == -1 and pool(mean=None) == -1 and pool(argmax=None) == -1     # null inputs / argmax
    assert pool(y=None) == -1 and b"output" in N.lib.ddn_last_error()                      # no output at all
    assert pool(y_lo=fake) == -1 and b"y_lo" in N.lib.ddn_last_error()                     # a lo plane without its hi plane
    for kw in (dict(n=0), dict(hc=0), dict(wc=0)):
        assert pool(**kw) == -1
    for kw in (dict(G=3), dict(G=0), dict(n=3, G=2)):
        assert pool(**kw) == -1 and b"bn_groups" in N.lib.ddn_last_error()
    for kw in (dict(x=None), dict(argmax=None), dict(dy=None), dict(dw=None), dict(dgamma=None)):
        assert bwd(**kw) == -1 and b"null" in N.lib.ddn_last_error()
    for prec in (-1, 3):
        assert bwd(prec=prec, nbytes=1 << 40) == -1 and b"precision" in N.lib.ddn_last_error()
    for kw in (dict(n=0), dict(h=0), dict(w=0)):
        assert bwd(nbytes=1 << 40, **kw) == -1 and b"sizes" in N.lib.ddn_last_error()
    for kw in (dict(G=3), dict(G=0), dict(n=3, G=2)):
        assert bwd(**kw) == -1 and b"bn_groups" in N.lib.ddn_last_error()
    assert bwd(n=70000, G=1, nbytes=1 << 62) == -1 and b"launch grid" in N.lib.ddn_last_error()
    for prec, nbytes in ((X3, ws_x3), (SIMT, ws_simt)):
        assert bwd(prec=prec, nbytes=nbytes - 1) == -2 and b"workspace" in N.lib.ddn_last_error()
    assert bwd(ws=None) == -1 and b"workspace" in N.lib.ddn_last_error()
    assert bwd(ws=ctypes.c_void_p((1 << 40) + 128)) == -1 and b"256-byte" in N.lib.ddn_last_error()
    assert N.launch_count() == before


def test_batchnorm_workspace_covers_every_supported_width():
    """the standalone BatchNorm entries take the channel counts the kernels take, the network's 2048 included"""
    for C in (4, 64, 512, 1024, 2048, 4096):
        assert N.lib.ddn_batchnorm_workspace_bytes(4800, C) > 0, C
    for C in (6, 1536, 8192, 0):
        assert N.lib.ddn_batchnorm_workspace_bytes(4800, C) == 0, C


def test_product_refuses_cpu_tensors():
    m = pdc_b200.Resnet34_8s(num_classes=3)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.zeros(1, 3, 64, 64))
    pcl = pdc_b200.PixelwiseContrastiveLoss([8, 8], {"M_pixel": 50})
    with pytest.raises(RuntimeError, match="CUDA"):
        pcl.match_loss(torch.zeros(1, 64, 3), torch.zeros(1, 64, 3), torch.tensor([1]), torch.tensor([2]))
    with pytest.raises(ValueError):
        pdc_b200.DenseCorrespondenceNetwork.get_fcn({"backbone": {"model_class": "Resnet", "resnet_name": "Resnet101_8s"},
                                                     "descriptor_dimension": 3})
    with pytest.raises(ValueError):
        pdc_b200.DenseCorrespondenceNetwork.get_fcn({"backbone": {"model_class": "Foo"}, "descriptor_dimension": 3})


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "pytorch-dense-correspondence_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in text and "from oracle" not in text and "oracle/" not in text, f
