"""Resnet34_8s and Resnet50_8s -- drop-ins for the backbone classes the reference builds with
``getattr(resnet_dilated, config["backbone"]["resnet_name"])(num_classes=D)``
(dense_correspondence/network/dense_correspondence_network.py:373-375;
originals: external/pytorch-segmentation-detection/pytorch_segmentation_detection/models/resnet_dilated.py:283-322 and
:399-435 on top of .../vision/torchvision/models/resnet.py:112-265 -- BasicBlock [3, 4, 6, 3] and Bottleneck [3, 4, 6, 3]).
The description below says Resnet34_8s; Resnet50_8s is the same module over its own parameter tables (``resnet50_8s.*``, 320
state-dict keys).

Same constructor, same ``forward(x, feature_alignment=False)``, same 218 state-dict keys
(``resnet34_8s.conv1.weight`` ... ``resnet34_8s.fc.bias``), same train()/eval() BatchNorm semantics --
but the module holds no torch.nn layers: all learnable tensors are views into one flat fp32 array
and the whole forward / backward runs inside libddn_b200.so (hand-written sm_90a kernels) through
one autograd.Function.  CUDA only; there is no CPU path.

Differences from the reference constructor, on purpose: no ImageNet download (``pretrained=True`` at
resnet_dilated.py:292-295 needs the network); weights start from the reference's own initialisers
(He-normal convs resnet.py:174-180, fc ~ N(0, 0.01) resnet_dilated.py:305-308) and are normally
overwritten by ``load_state_dict``.
"""
import math
import os

import torch
import torch.nn as nn

from . import _native as N

_BN_MOMENTUM = 0.1   # nn.BatchNorm2d defaults, resnet.py:46
_BN_EPS = 1e-5

_cache_nonce = [0]
_default_precision = [N.PRECISION_BF16X3]     # fp32-equivalent results on the tensor cores


def set_default_precision(p):
    """'bf16x3' (wgmma, operands split hi+lo: fp32-equivalent results, the default) or 'bf16' (wgmma single pass: fast,
    fails the 1e-3 descriptor gate).  There is ONE execution path -- the tensor cores; the fp32 CUDA-core kernels that the
    library also contains are a parity instrument of the test-suite, not a backend, and are refused unless
    DDN_TEST_FP32_SIMT=1 is set (tests/conftest.py sets it)."""
    _default_precision[0] = {"fp32": N.PRECISION_FP32_SIMT, "bf16x3": N.PRECISION_BF16X3, "bf16": N.PRECISION_BF16}[p]


def _check_precision(prec):
    if prec == N.PRECISION_FP32_SIMT and os.environ.get("DDN_TEST_FP32_SIMT") != "1":
        raise RuntimeError("the fp32 CUDA-core convolutions are a parity instrument of the test-suite, not a selectable backend "
                           "(set DDN_TEST_FP32_SIMT=1 to use them); the product path is precision 'bf16x3' on the tensor cores")


def attach_lowres(y, low, H, W, unit=False):
    """Tags a descriptor image with the low-resolution map it is the bilinear upsample of.  loss_composer looks for the tag and,
    when both images of a pair carry it, evaluates the loss through the 4 low-resolution cells of every sampled pixel
    (csrc/loss_lowres.cu) instead of gathering from the full-resolution tensor.  The tag records the tensor's version so that an
    in-place modification of the image silently falls back to the generic path.  ``unit=True``: the image is the upsample
    with every pixel's descriptor normalised to unit length (the reference's ``normalize`` option, per pixel); the fused loss
    then normalises each blended descriptor the same way.  -> tag ``(low, H, W, version, unit)``."""
    y._ddn_lowres = (low, int(H), int(W), y._version, bool(unit))


def lowres_of(t):
    """The tag ``attach_lowres`` left on ``t``, or None when there is none or ``t`` was modified in place since."""
    tag = getattr(t, "_ddn_lowres", None)
    if tag is None or t._version != tag[3]:
        return None
    return tag


class _Holder(nn.Module):
    """A name-space node of the reference module tree (it owns parameters/buffers, never computes)."""

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("backbone sub-modules are parameter holders; call the top-level module")


class _Backbone(torch.autograd.Function):
    """forward / backward of the whole backbone as ONE autograd node over the C ABI.

    Parameter gradients are written by the library into one flat array and, by default, attached / accumulated into
    ``p.grad`` by this function itself (every ``p.grad`` is a view of ``Resnet34_8s.flat_gradient``: the data-parallel
    all-reduce and the fused optimizer see one buffer, and the second backward of a step is one flat add instead of 110
    AccumulateGrad kernels).  Consequences, on purpose: ``torch.autograd.grad`` w.r.t. the parameters returns None for
    them -- unless a parameter carries a hook, in which case the real per-tensor gradients are returned to autograd so
    that hooks and AccumulateGrad behave normally (the slow path).  Parameters with ``requires_grad=False`` get no gradient.
    """

    @staticmethod
    def forward(ctx, x, owner, groups, unit, *params):
        N.require_cuda_f32(x, "input image batch")
        if x.dim() != 4 or x.shape[1] != 3:
            raise RuntimeError("expected input of shape [N,3,H,W], got %s" % (tuple(x.shape),))
        B, _, H, W = x.shape
        if groups not in (1, 2) or B % groups:
            raise RuntimeError("bn_groups must be 1 or 2 and divide the batch size (got %d for a batch of %d)" % (groups, B))
        D = owner.num_classes
        flat, bufs = owner._ensure_flat(x.device)
        keep = any(ctx.needs_input_grad)    # grad mode is off inside Function.forward; this is the signal
        # train(): batch statistics.  eval(): running statistics -- folded into the convs when nothing is differentiated,
        # kept un-folded with the activations saved when a gradient is wanted (the reference can backpropagate through an
        # eval()-mode network: frozen BatchNorm statistics)
        mode = N.MODE_TRAIN if owner.training else (N.MODE_EVAL_SAVE if keep else N.MODE_INFER)
        prec = owner.precision
        _check_precision(prec)
        owner._register_weight_cache(flat, prec)
        arch = owner._ARCH
        flags = N.NET_UNIT_DESCRIPTORS if unit else 0
        ws_bytes = N.lib.ddn_net_workspace_bytes_v2(arch, B, H, W, D, mode, prec, flags)
        if ws_bytes == 0:
            raise N.DdnError("bad shape for %s: %s" % (type(owner).__name__, N.lib.ddn_last_error().decode()))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device)
        y = torch.empty(B, D, H, W, dtype=torch.float32, device=x.device)
        # the low-resolution map y is the bilinear upsample of, [B, H/8*W/8, D]: second output, so that a loss fused with the
        # upsample (contrastive_ops.within_scene_loss on tensors carrying `_ddn_lowres`) can differentiate through it directly
        low = torch.empty(B, (H // 8) * (W // 8), D, dtype=torch.float32, device=x.device)
        N.check(N.lib.ddn_net_forward_v2(arch, N.ptr(x), N.ptr(flat), N.ptr(bufs), N.ptr(y), N.ptr(ws), ws_bytes,
                                         B, H, W, D, mode, groups, _BN_MOMENTUM, _BN_EPS, prec, N.ptr(low), flags, N.stream_ptr()))
        ctx.set_materialize_grads(False)
        if owner.training:
            torch._foreach_add_(owner._nbt, groups)
        if keep:
            ctx.owner, ctx.ws, ctx.shape, ctx.prec, ctx.mode, ctx.groups = owner, ws, (B, H, W, D), prec, mode, groups
            ctx.flags = flags
            ctx.param_version = owner._flat_version
        ctx.keep = keep
        return y, low

    @staticmethod
    def backward(ctx, dy, dlow):
        if dy is None and dlow is None:
            return (None, None, None, None) + (None,) * len(ctx.owner._params) if ctx.keep else None
        if not ctx.keep:
            raise RuntimeError("backbone backward: nothing required a gradient in the forward; no activations were saved")
        if ctx.ws is None:
            raise RuntimeError("backbone: trying to backward through the backbone a second time; its saved activations "
                               "(one caller-owned workspace) were released by the first backward -- retain_graph is not supported")
        owner = ctx.owner
        B, H, W, D = ctx.shape
        if owner._flat_version != ctx.param_version:
            raise RuntimeError("parameters were re-allocated between forward and backward")
        ref = dy if dy is not None else dlow
        if dy is not None:
            dy = dy.contiguous()
            N.require_cuda_f32(dy, "descriptor cotangent")
        if dlow is not None:
            dlow = dlow.contiguous()
            N.require_cuda_f32(dlow, "low-resolution descriptor cotangent")
        flat, _ = owner._ensure_flat(ref.device)
        owner._register_weight_cache(flat, ctx.prec)
        grads = torch.empty_like(flat)
        hook = owner._bucket_hook        # data_parallel.GradientAllReducer: all-reduce each bucket while the backward still runs
        cb = N.NO_BUCKET_CALLBACK
        if hook is not None:
            if owner._pad_index is not None:     # the padding words travel through the all-reduce: define them
                grads.index_fill_(0, owner._pad_index_on(grads.device), 0.0)
            sc = hook.cotangent_scale()          # the mean over ranks, folded into the (linear) backward
            dy = dy * sc if dy is not None else None
            dlow = dlow * sc if dlow is not None else None

            def _on_bucket(_user, bucket, offset, numel, _g=grads, _h=hook):
                _h.__call_bucket__(_g, int(bucket), int(offset), int(numel))
            cb = N.GRAD_BUCKET_FN(_on_bucket)
        N.check(N.lib.ddn_net_backward_v2(owner._ARCH, N.ptr(dy), N.ptr(dlow), N.ptr(flat), N.ptr(grads), N.ptr(ctx.ws),
                                          ctx.ws.numel(), B, H, W, D, ctx.mode, ctx.groups, _BN_EPS, ctx.prec, ctx.flags, cb, None,
                                          N.stream_ptr()))
        ctx.ws = None
        if hook is not None:
            hook.finish(grads)
        ps = owner._params
        if hook is None and owner._pad_index is not None:   # alignment padding between tensors: keep it zero (it is all-reduced / stepped too)
            grads.index_fill_(0, owner._pad_index_on(grads.device), 0.0)
        wants = ctx.needs_input_grad[4:]
        for p, want, (_, _, o, n) in zip(ps, wants, owner._ptab):
            if not want:
                grads[o:o + n].zero_()      # frozen parameter: no gradient, and nothing for a flat optimizer / all-reduce to see
        if any(p._backward_hooks or getattr(p, "_post_accumulate_grad_hooks", None) for p in ps):
            # slow path: hand the per-tensor gradients to autograd (hooks, AccumulateGrad, autograd.grad all work)
            return (None, None, None, None) + tuple(grads[o:o + n].view(s) if want else None
                                              for want, (_, s, o, n) in zip(wants, owner._ptab))
        fg = owner._flat_grad
        fresh = fg is None or fg.device != grads.device
        if not fresh:
            base = fg.data_ptr()
            for p, want, (_, _, o, _) in zip(ps, wants, owner._ptab):
                if want and (p.grad is None or p.grad.data_ptr() != base + 4 * o):
                    fresh = True
                    break
        if fresh:                      # first backward since zero_grad(set_to_none=True) (or a partial one: start over)
            owner._flat_grad = grads
            for p, want, (_, s, o, n) in zip(ps, wants, owner._ptab):
                if want:
                    p.grad = grads[o:o + n].view(s)
        else:
            fg.add_(grads)
        return (None, None, None, None) + (None,) * len(ps)


class _DilatedResnet(nn.Module):
    """The flat-array backbone; subclasses name the architecture (``_ARCH``) and the reference's root attribute (``_ROOT``)."""
    _ARCH = None
    _ROOT = None

    def _pad_index_on(self, device):
        t = self._pad_index_dev.get(device)
        if t is None:
            t = self._pad_index_dev[device] = self._pad_index.to(device)
        return t

    def __init__(self, num_classes=1000, precision=None):
        super().__init__()
        if not (1 <= num_classes <= 32):
            raise ValueError("this build supports descriptor dimensions 1..32 (got %d)" % num_classes)
        self.num_classes = num_classes
        self.precision = _default_precision[0] if precision is None else precision
        self._ptab = N.param_table(num_classes, self._ARCH)
        self._btab = N.buffer_table(self._ARCH)
        n_params = int(N.lib.ddn_net_param_count(self._ARCH, num_classes))
        n_bufs = int(N.lib.ddn_net_buffer_count(self._ARCH))
        self._flat = torch.zeros(n_params, dtype=torch.float32)
        self._flat_bufs = torch.zeros(n_bufs, dtype=torch.float32)
        self._flat_version = 0
        self._flat_grad = None
        pads = []
        for (_, _, off, n) in self._ptab:
            pads += list(range(off + n, (off + n + 3) // 4 * 4))
        self._pad_index = torch.tensor(pads, dtype=torch.long) if pads else None
        self._pad_index_dev = {}      # device -> resident copy (a pageable .to(device) inside backward would stall the host on the stream)
        self._wcache = None
        self._wcache_nonce = 0
        self._bucket_hook = None      # data_parallel.GradientAllReducer: called per finished gradient bucket during backward
        self._params = []
        self._nbt = []
        root = _Holder()
        setattr(self, self._ROOT, root)
        buf_by_name = {name: (shape, off, n) for name, shape, off, n in self._btab}
        for name, shape, off, n in self._ptab:
            path = name.split(".")
            node = root
            for part in path[:-1]:
                if not hasattr(node, part):
                    node.add_module(part, _Holder())
                node = getattr(node, part)
            p = nn.Parameter(self._flat[off:off + n].view(shape))
            node.register_parameter(path[-1], p)
            self._params.append(p)
            prefix = ".".join(path[:-1])
            if path[-1] == "bias" and (prefix + ".running_mean") in buf_by_name:   # a BatchNorm: add its buffers
                for bname in ("running_mean", "running_var"):
                    s, o, m = buf_by_name[prefix + "." + bname]
                    node.register_buffer(bname, self._flat_bufs[o:o + m].view(s))
                node.register_buffer("num_batches_tracked", torch.tensor(0, dtype=torch.long))
                self._nbt.append(node.num_batches_tracked)
        self._holders_with_buffers = [m for m in root.modules() if "running_mean" in m._buffers]
        self.reset_parameters()

    # ---- initialisation (resnet.py:174-180, resnet_dilated.py:305-308)
    def reset_parameters(self):
        with torch.no_grad():
            for (name, shape, _, _), p in zip(self._ptab, self._params):
                if name.startswith("fc."):
                    p.normal_(0, 0.01) if name == "fc.weight" else p.zero_()
                elif len(shape) == 4:
                    p.normal_(0, math.sqrt(2.0 / (shape[2] * shape[3] * shape[0])))
                elif name.endswith(".weight"):
                    p.fill_(1.0)
                else:
                    p.zero_()
            for m in self._holders_with_buffers:
                m.running_mean.zero_()
                m.running_var.fill_(1.0)
                m.num_batches_tracked.zero_()

    # ---- flat storage management
    def _is_flat(self, device):
        if self._flat.device != device or self._flat_bufs.device != device:
            return False
        base, bbase = self._flat.data_ptr(), self._flat_bufs.data_ptr()
        for (_, _, off, _), p in zip(self._ptab, self._params):
            if p.data_ptr() != base + 4 * off or p.dtype != torch.float32:
                return False
        for m in self._holders_with_buffers:
            if m.running_mean.device != device:
                return False
        for (name, _, off, _) in self._btab:
            node = getattr(self, self._ROOT)
            parts = name.split(".")
            for part in parts[:-1]:
                node = getattr(node, part)
            if node._buffers[parts[-1]].data_ptr() != bbase + 4 * off:
                return False
        return True

    def _ensure_flat(self, device):
        """(Re)packs parameters and BN statistics into the two flat arrays the C ABI takes; a no-op
        unless something (.cuda(), .to(), p.data = ...) re-allocated them."""
        if self._is_flat(device):
            return self._flat, self._flat_bufs
        with torch.no_grad():
            flat = torch.zeros(self._flat.numel(), dtype=torch.float32, device=device)
            for (_, shape, off, n), p in zip(self._ptab, self._params):
                flat[off:off + n].copy_(p.detach().reshape(-1).to(device=device, dtype=torch.float32))
                p.data = flat[off:off + n].view(shape)
            bufs = torch.zeros(self._flat_bufs.numel(), dtype=torch.float32, device=device)
            for (name, shape, off, n) in self._btab:
                node = getattr(self, self._ROOT)
                parts = name.split(".")
                for part in parts[:-1]:
                    node = getattr(node, part)
                old = node._buffers[parts[-1]]
                bufs[off:off + n].copy_(old.detach().reshape(-1).to(device=device, dtype=torch.float32))
                node._buffers[parts[-1]] = bufs[off:off + n].view(shape)
            self._nbt = []
            for m in self._holders_with_buffers:
                m._buffers["num_batches_tracked"] = m._buffers["num_batches_tracked"].to(device)
                self._nbt.append(m._buffers["num_batches_tracked"])
            self._flat, self._flat_bufs = flat, bufs
            self._flat_version += 1
        return self._flat, self._flat_bufs

    def _apply(self, fn, *args, **kwargs):
        out = super()._apply(fn, *args, **kwargs)
        dev = self._params[0].device
        if dev.type == "cuda":
            self._ensure_flat(dev)
        else:
            self._flat = self._flat.to(dev)   # CPU copy only serves state_dict round trips
        return out

    def _register_weight_cache(self, flat, prec):
        """Gives the library a buffer for the packed bf16 weights of every conv.  Nothing here tracks parameter changes: the
        library fingerprints the flat parameter array ON THE DEVICE at the start of every forward and re-packs when (and only
        when) it changed, so writes through ``.data``, raw pointers, optimizers or NCCL can never leave stale packs in use."""
        if prec == N.PRECISION_FP32_SIMT:
            return
        if self._wcache is None or self._wcache.device != flat.device:
            self._wcache = torch.empty(N.lib.ddn_net_weight_cache_bytes(self._ARCH, self.num_classes), dtype=torch.uint8,
                                       device=flat.device)
            _cache_nonce[0] += 1           # a fresh buffer may reuse the address of a dead one: never look "unchanged"
            self._wcache_nonce = _cache_nonce[0]
        N.check(N.lib.ddn_resnet34_8s_set_weight_cache(N.ptr(self._wcache), self._wcache.numel(), N.ptr(flat),
                                                       (self._wcache_nonce << 20) + self._flat_version, prec))

    def mark_parameters_changed(self):
        """Kept for existing callers: a no-op now (parameter changes are detected on the device)."""

    @property
    def flat_gradient(self):
        """The flat fp32 array all ``p.grad`` alias after a backward (None before the first one / after zero_grad)."""
        if self._flat_grad is None or self._params[0].grad is None:
            return None
        return self._flat_grad

    @property
    def flat_parameters(self):
        """The single fp32 array every parameter aliases (valid after the module is on its device)."""
        return self._ensure_flat(self._params[0].device)[0]

    def forward(self, x, feature_alignment=False, bn_groups=1, per_pixel_normalize=False):
        """``bn_groups=2``: the batch is two consecutive groups (image-A batch, image-B batch), each normalised by its own
        batch statistics -- the two forward calls of a reference training step in one launch sequence.
        ``per_pixel_normalize=True``: every pixel's descriptor is divided by its L2 norm inside the upsample kernel, image by
        image (what the reference's ``normalize`` option computes for a batch of one); a zero descriptor gives NaN, as
        ``x / ||x||`` does.  The output is tagged so that a fused loss normalises the same way."""
        if feature_alignment:
            raise NotImplementedError("feature_alignment=True is not on the dense-descriptor hot path "
                                      "(resnet_dilated.py:314 is never taken by the reference)")
        unit = bool(per_pixel_normalize)
        y, low = _Backbone.apply(x, self, bn_groups, unit, *self._params)
        attach_lowres(y, low, x.shape[2], x.shape[3], unit=unit)
        return y


class Resnet34_8s(_DilatedResnet):
    """resnet_dilated.py:283-322: ResNet(BasicBlock, [3, 4, 6, 3]), output stride 8, fc = Conv2d(512, D, 1)."""
    _ARCH = N.ARCH_RESNET34_8S
    _ROOT = "resnet34_8s"


class Resnet50_8s(_DilatedResnet):
    """resnet_dilated.py:399-435: ResNet(Bottleneck, [3, 4, 6, 3]), output stride 8, fc = Conv2d(2048, D, 1)."""
    _ARCH = N.ARCH_RESNET50_8S
    _ROOT = "resnet50_8s"
