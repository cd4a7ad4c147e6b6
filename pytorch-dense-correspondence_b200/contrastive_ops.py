"""autograd.Function wrappers over the loss kernels of libddn_b200.so (csrc/loss.cu).

``contrastive_terms``  -- generic: per (pair, term) fp64 sums + int64 hard-negative counts, differentiable
                          in the two descriptor images (used by every PixelwiseContrastiveLoss method).
``within_scene_loss``  -- fused loss_composer.get_within_scene_loss: one gather/reduce launch, one compose
                          launch, no host synchronisation; backward is one scatter launch.
``pair_type_loss``     -- the same gather and scatter for a batch whose pairs have different SpartanDatasetDataType
                          values (loss_composer.get_mixed_loss); the compose gives each pair its own type's loss.
Descriptor images are consumed as the strided ``[B, P, D]`` views ``process_network_output`` makes.
"""
import ctypes

import torch

from . import _native as N


class Term(object):
    """One list of index pairs scored one way (see ddn_loss_term in include/ddn_b200.h)."""
    __slots__ = ("idx_a", "idx_b", "kind", "margin", "gt_b", "m_pixel", "lengths", "gt_lengths")

    def __init__(self, idx_a, idx_b, kind, margin=0.0, gt_b=None, m_pixel=0.0, lengths=None, gt_lengths=None):
        self.idx_a, self.idx_b, self.kind, self.margin, self.gt_b, self.m_pixel = idx_a, idx_b, kind, margin, gt_b, m_pixel
        self.lengths, self.gt_lengths = lengths, gt_lengths      # ragged batches: [B] int64 true counts (rows padded with -1)


def _as_pred(pred, name):
    if not isinstance(pred, torch.Tensor) or not pred.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor: the loss has no CPU fallback" % name)
    if pred.dtype != torch.float32:
        raise RuntimeError("%s must be float32" % name)
    if pred.dim() == 2:
        pred = pred.unsqueeze(0)
    if pred.dim() != 3:
        raise RuntimeError("%s must have shape [B, W*H, D]" % name)
    return pred


def _as_index(idx, B, name):
    if not isinstance(idx, torch.Tensor) or not idx.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor" % name)
    if idx.dtype != torch.int64:
        raise RuntimeError("%s must be int64 (torch.LongTensor), got %s" % (name, idx.dtype))
    if idx.dim() == 1:          # one index list shared by every pair of the batch (e.g. the [-1] sentinel)
        idx = idx.unsqueeze(0).expand(B, -1)
    if idx.dim() != 2 or idx.shape[0] != B:
        raise RuntimeError("%s must have shape [n] or [B, n] with B=%d, got %s" % (name, B, tuple(idx.shape)))
    return idx.contiguous()


def _as_lengths(t, B, name):
    if t is None:
        return None
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.int64 or t.shape != (B,):
        raise RuntimeError("%s must be a CUDA int64 tensor of shape [%d]" % (name, B))
    return t.contiguous()


def _strides(pa, pb):
    if pa.shape != pb.shape or pa.stride() != pb.stride():
        pb = pb.contiguous() if pa.is_contiguous() else pb
        if pa.shape != pb.shape or pa.stride() != pb.stride():
            raise RuntimeError("image_a_pred and image_b_pred must share shape and strides")
    return pb


def _build_terms(terms, B):
    arr = (N.LossTerm * len(terms))()
    keep = []
    for i, t in enumerate(terms):
        ia = _as_index(t.idx_a, B, "index tensor a of term %d" % i)
        ib = _as_index(t.idx_b, B, "index tensor b of term %d" % i)
        if ia.shape != ib.shape:
            raise RuntimeError("term %d: a/b index tensors differ in length" % i)
        keep += [ia, ib]
        arr[i].idx_a, arr[i].idx_b = ia.data_ptr(), ib.data_ptr()
        arr[i].n = ia.shape[1]
        arr[i].kind = t.kind
        arr[i].margin = float(t.margin)
        arr[i].flags = 0
        if t.gt_b is not None:
            gt = _as_index(t.gt_b, B, "matches_b of term %d" % i)
            keep.append(gt)
            arr[i].gt_b, arr[i].n_gt = gt.data_ptr(), gt.shape[1]
            arr[i].flags = N.TERM_PIXEL_WEIGHT
            arr[i].m_pixel = float(t.m_pixel)
            gl = _as_lengths(t.gt_lengths, B, "gt_lengths of term %d" % i)
            if gl is not None:
                keep.append(gl)
                arr[i].len_gt = gl.data_ptr()
        ln = _as_lengths(t.lengths, B, "lengths of term %d" % i)
        if ln is not None:
            keep.append(ln)
            arr[i].len = ln.data_ptr()
    return arr, keep


class _Terms(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred_a, pred_b, image_width, terms):
        B, P, D = pred_a.shape
        arr, keep = _build_terms(terms, B)
        sums = torch.empty(B, len(terms), dtype=torch.float64, device=pred_a.device)
        counts = torch.empty(B, len(terms), dtype=torch.int64, device=pred_a.device)
        sb, sp, sc = pred_a.stride()
        N.check(N.lib.ddn_contrastive_terms_forward(N.ptr(pred_a), N.ptr(pred_b), sb, sp, sc, B, P, D, image_width,
                                                    arr, len(terms), N.ptr(sums), N.ptr(counts), N.stream_ptr()))
        ctx.save_for_backward(pred_a, pred_b)
        ctx.arr, ctx.keep, ctx.image_width = arr, keep, image_width
        ctx.mark_non_differentiable(counts)
        return sums, counts

    @staticmethod
    def backward(ctx, dsums, _dcounts):
        pred_a, pred_b = ctx.saved_tensors
        B, P, D = pred_a.shape
        coef = dsums.to(torch.float32).contiguous()
        da = torch.empty_strided(pred_a.shape, pred_a.stride(), dtype=torch.float32, device=pred_a.device).zero_()
        db = torch.empty_strided(pred_a.shape, pred_a.stride(), dtype=torch.float32, device=pred_a.device).zero_()
        sb, sp, sc = pred_a.stride()
        N.check(N.lib.ddn_contrastive_terms_backward(N.ptr(pred_a), N.ptr(pred_b), sb, sp, sc, B, P, D, ctx.image_width,
                                                     ctx.arr, len(ctx.arr), N.ptr(coef), None, N.ptr(da), N.ptr(db),
                                                     N.stream_ptr()))
        return da, db, None, None


def contrastive_terms(pred_a, pred_b, image_width, terms):
    """-> (sums [B,T] float64, counts [B,T] int64); differentiable w.r.t. pred_a / pred_b."""
    pred_a = _as_pred(pred_a, "image_a_pred")
    pred_b = _strides(pred_a, _as_pred(pred_b, "image_b_pred"))
    return _Terms.apply(pred_a, pred_b, int(image_width), list(terms))


def _within_scene_compose(sums, counts, cfg, five, coef, st):
    B, T = sums.shape
    N.check(N.lib.ddn_within_scene_compose(N.ptr(sums), N.ptr(counts), B, T, ctypes.byref(cfg), N.ptr(five), N.ptr(coef), st))


def _pair_type_compose(sums, counts, cfg, five, coef, st):
    B, T = sums.shape
    N.check(N.lib.ddn_pair_type_compose(N.ptr(sums), N.ptr(counts), B, T, ctypes.byref(cfg), N.ptr(cfg._pair_type),
                                        N.ptr(five), N.ptr(coef), st))


def _fused_outputs(ctx, counts, five):
    loss = five[0:1]
    rest = five[1:].clone()
    ctx.mark_non_differentiable(rest, counts)
    return loss, rest, counts


def _gather_compose(ctx, pred_a, pred_b, image_width, terms, cfg, compose):
    """Forward of the fused losses from the full-resolution images: one gather launch, one ``compose`` launch."""
    B, P, D = pred_a.shape
    T = len(terms)
    arr, keep = _build_terms(terms, B)
    dev = pred_a.device
    sums = torch.empty(B, T, dtype=torch.float64, device=dev)
    counts = torch.empty(B, T, dtype=torch.int64, device=dev)
    five = torch.empty(5, dtype=torch.float32, device=dev)
    coef = torch.empty(B, T, dtype=torch.float32, device=dev)
    sb, sp, sc = pred_a.stride()
    st = N.stream_ptr()
    N.check(N.lib.ddn_contrastive_terms_forward(N.ptr(pred_a), N.ptr(pred_b), sb, sp, sc, B, P, D, image_width,
                                                arr, T, N.ptr(sums), N.ptr(counts), st))
    compose(sums, counts, cfg, five, coef, st)
    ctx.save_for_backward(pred_a, pred_b, coef)
    ctx.arr, ctx.keep, ctx.image_width = arr, keep, image_width
    return _fused_outputs(ctx, counts, five)


def _gather_compose_lowres(ctx, low_a, low_b, geom, terms, cfg, compose, unit):
    """Forward of the fused losses through the bilinear upsample: one gather launch, one ``compose`` launch.  ``unit``: the
    blended descriptors are normalised to unit length first (DDN_LOWRES_UNIT)."""
    B, _, D = low_a.shape
    h, w, H, W = geom
    T = len(terms)
    arr, keep = _build_terms(terms, B)
    dev = low_a.device
    sums = torch.empty(B, T, dtype=torch.float64, device=dev)
    counts = torch.empty(B, T, dtype=torch.int64, device=dev)
    five = torch.empty(5, dtype=torch.float32, device=dev)
    coef = torch.empty(B, T, dtype=torch.float32, device=dev)
    st = N.stream_ptr()
    flags = N.LOWRES_UNIT if unit else 0
    N.check(N.lib.ddn_contrastive_terms_forward_lowres_v2(N.ptr(low_a), N.ptr(low_b), B, h, w, H, W, D, arr, T,
                                                          N.ptr(sums), N.ptr(counts), flags, st))
    compose(sums, counts, cfg, five, coef, st)
    ctx.save_for_backward(low_a, low_b, coef)
    ctx.arr, ctx.keep, ctx.geom, ctx.flags = arr, keep, geom, flags
    return _fused_outputs(ctx, counts, five)


class _WithinScene(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred_a, pred_b, image_width, terms, cfg):
        return _gather_compose(ctx, pred_a, pred_b, image_width, terms, cfg, _within_scene_compose)

    @staticmethod
    def backward(ctx, dloss, _drest, _dcounts):
        pred_a, pred_b, coef = ctx.saved_tensors
        B, P, D = pred_a.shape
        da = torch.empty_strided(pred_a.shape, pred_a.stride(), dtype=torch.float32, device=pred_a.device).zero_()
        db = torch.empty_strided(pred_a.shape, pred_a.stride(), dtype=torch.float32, device=pred_a.device).zero_()
        up = dloss.to(torch.float32).contiguous()
        sb, sp, sc = pred_a.stride()
        N.check(N.lib.ddn_contrastive_terms_backward(N.ptr(pred_a), N.ptr(pred_b), sb, sp, sc, B, P, D, ctx.image_width,
                                                     ctx.arr, len(ctx.arr), N.ptr(coef), N.ptr(up), N.ptr(da), N.ptr(db),
                                                     N.stream_ptr()))
        return da, db, None, None, None


class _PairTypes(_WithinScene):
    """The same gather and scatter as ``_WithinScene``; the compose gives every pair its own type's loss
    (ddn_pair_type_compose)."""

    @staticmethod
    def forward(ctx, pred_a, pred_b, image_width, terms, cfg):
        return _gather_compose(ctx, pred_a, pred_b, image_width, terms, cfg, _pair_type_compose)


class _WithinSceneLowres(torch.autograd.Function):
    """within_scene_loss fused with the bilinear upsample: the descriptors are blended from the low-resolution maps
    ``low_a`` / ``low_b`` [B, h*w, D] (csrc/loss_lowres.cu); the gradient is scattered into d(low) -- the full-resolution
    descriptor images and their gradients are never read or written.  ``unit``: every blended descriptor is normalised to
    unit length (the images are unit-descriptor outputs of the network)."""

    @staticmethod
    def forward(ctx, low_a, low_b, geom, terms, cfg, unit=False):
        return _gather_compose_lowres(ctx, low_a, low_b, geom, terms, cfg, _within_scene_compose, unit)

    @staticmethod
    def backward(ctx, dloss, _drest, _dcounts):
        low_a, low_b, coef = ctx.saved_tensors
        B, _, D = low_a.shape
        h, w, H, W = ctx.geom
        da = torch.zeros_like(low_a)
        db = torch.zeros_like(low_b)
        up = dloss.to(torch.float32).contiguous()
        scratch = torch.empty(2 * low_a.numel(), dtype=torch.float64, device=low_a.device)    # the fp64 scatter accumulator
        N.check(N.lib.ddn_contrastive_terms_backward_lowres_v2(N.ptr(low_a), N.ptr(low_b), B, h, w, H, W, D, ctx.arr,
                                                               len(ctx.arr), N.ptr(coef), N.ptr(up), N.ptr(da), N.ptr(db),
                                                               N.ptr(scratch), ctx.flags, N.stream_ptr()))
        return da, db, None, None, None, None


class _PairTypesLowres(_WithinSceneLowres):
    """``_PairTypes`` through the bilinear upsample (the gather and scatter of ``_WithinSceneLowres``)."""

    @staticmethod
    def forward(ctx, low_a, low_b, geom, terms, cfg, unit=False):
        return _gather_compose_lowres(ctx, low_a, low_b, geom, terms, cfg, _pair_type_compose, unit)


def _unpack_lowres(lowres):
    """(low_a, low_b, geom) or (low_a, low_b, geom, unit) -> (low_a, low_b, geom, unit)"""
    low_a, low_b, geom = lowres[:3]
    return low_a, low_b, geom, bool(lowres[3]) if len(lowres) > 3 else False


def within_scene_loss(pred_a, pred_b, image_width, terms, match_loss_weight, non_match_loss_weight,
                      scale_by_hard_negatives, has_blind, lengths=None, lowres=None):
    """terms = [match, masked, background(, blind)].  -> (loss [1], (match, masked, background, blind) [4], counts [B,T]).
    Mean over the B pairs; only ``loss`` carries gradient (the other four are logging values,
    dense_correspondence/training/training.py:369-411)."""
    pred_a = _as_pred(pred_a, "image_a_pred")
    pred_b = _strides(pred_a, _as_pred(pred_b, "image_b_pred"))
    B = pred_a.shape[0]
    n = [_as_index(t.idx_a, B, "indices").shape[1] for t in terms]
    cfg = N.WithinSceneCfg(float(match_loss_weight), float(non_match_loss_weight), int(bool(scale_by_hard_negatives)),
                           int(bool(has_blind)), n[0], n[1], n[2], n[3] if has_blind else 0)
    keep = []
    if lengths is not None:      # ragged batch: per-pair true counts, (matches, masked, background[, blind])
        for field, t in zip(("len_match", "len_masked", "len_background", "len_blind"), lengths):
            t = _as_lengths(t, B, field)
            if t is not None:
                keep.append(t)
                setattr(cfg, field, t.data_ptr())
    cfg._keep = keep
    if lowres is not None:        # (low_a, low_b, (h, w, H, W)[, unit]): both images are bilinear upsamples of these maps
        low_a, low_b, geom, unit = _unpack_lowres(lowres)
        return _WithinSceneLowres.apply(low_a.contiguous(), low_b.contiguous(), geom, list(terms), cfg, unit)
    return _WithinScene.apply(pred_a, pred_b, int(image_width), list(terms), cfg)


def pair_type_loss(pred_a, pred_b, image_width, terms, pair_type, match_loss_weight, non_match_loss_weight,
                   scale_by_hard_negatives, scale_by_hard_negatives_different_object, lengths, lowres=None):
    """terms = [match, masked, background, blind@M_masked, blind@M_background], the two blind terms over the same index
    tensors with their lengths routed by pair type; pair_type: [B] int32 CUDA SpartanDatasetDataType values; lengths =
    (matches, masked, background, blind) [B] int64 CUDA true counts (blind unrouted).  -> as ``within_scene_loss``: every
    pair scored by its own type's formula, mean over the B pairs; only ``loss`` carries gradient."""
    pred_a = _as_pred(pred_a, "image_a_pred")
    pred_b = _strides(pred_a, _as_pred(pred_b, "image_b_pred"))
    B = pred_a.shape[0]
    if len(terms) != 5:
        raise RuntimeError("pair_type_loss takes 5 terms (got %d)" % len(terms))
    if not isinstance(pair_type, torch.Tensor) or not pair_type.is_cuda or pair_type.dtype != torch.int32 \
            or pair_type.shape != (B,):
        raise RuntimeError("pair_type must be a CUDA int32 tensor of shape [%d]" % B)
    n = [_as_index(t.idx_a, B, "indices").shape[1] for t in terms]
    cfg = N.PairTypeComposeCfg(float(match_loss_weight), float(non_match_loss_weight), int(bool(scale_by_hard_negatives)),
                               int(bool(scale_by_hard_negatives_different_object)), n[0], n[1], n[2], n[3])
    keep = [pair_type]
    for field, t in zip(("len_match", "len_masked", "len_background", "len_blind"), lengths):
        t = _as_lengths(t, B, field)
        if t is None:
            raise RuntimeError("pair_type_loss needs every per-pair count (%s is missing)" % field)
        keep.append(t)
        setattr(cfg, field, t.data_ptr())
    cfg._keep, cfg._pair_type = keep, pair_type.contiguous()
    if lowres is not None:
        low_a, low_b, geom, unit = _unpack_lowres(lowres)
        return _PairTypesLowres.apply(low_a.contiguous(), low_b.contiguous(), geom, list(terms), cfg, unit)
    return _PairTypes.apply(pred_a, pred_b, int(image_width), list(terms), cfg)
