"""Device-side non-match sampling (SURVEY.md 8f row 2): the index tensors ``loss_composer.get_loss`` consumes, produced on
the GPU instead of by the CPU dataset workers (correspondence_finder.create_non_correspondences +
SpartanDataset.create_non_matches + flatten_uv_tensor; see csrc/sampling.cu for the line references)."""
import numpy as np
import torch

from . import _native as N


def sample_non_matches(matches_a, img_b_mask, image_shape, num_non_matches_per_match, generator=None, rand=None):
    """matches_a: int64 [Nm] flat indices (CUDA).  img_b_mask: float32 [H, W] CUDA tensor (nonzero = selectable) or None.
    -> (non_matches_a [Nm*k], non_matches_b [Nm*k]) int64 CUDA flat pixel indices, k = num_non_matches_per_match.
    ``rand`` (optional) = (rand_u, rand_v) float32 [Nm*k] uniform numbers to use instead of drawing them."""
    H, W = image_shape
    if not matches_a.is_cuda or matches_a.dtype != torch.int64:
        raise RuntimeError("matches_a must be an int64 CUDA tensor")
    dev = matches_a.device
    n = matches_a.numel() * int(num_non_matches_per_match)
    if rand is None:
        rand_u = torch.rand(n, device=dev, generator=generator)
        rand_v = torch.rand(n, device=dev, generator=generator)
    else:
        rand_u, rand_v = rand
        N.require_cuda_f32(rand_u, "rand_u"); N.require_cuda_f32(rand_v, "rand_v")
    if img_b_mask is not None:
        N.require_cuda_f32(img_b_mask, "img_b_mask")
        if tuple(img_b_mask.shape) != (H, W):
            raise RuntimeError("mask must have shape [H, W]")
    out_a = torch.empty(n, dtype=torch.int64, device=dev)
    out_b = torch.empty(n, dtype=torch.int64, device=dev)
    nb = N.lib.ddn_sample_non_matches_scratch_bytes(H, W)
    scratch = torch.empty(nb, dtype=torch.uint8, device=dev)
    N.check(N.lib.ddn_sample_non_matches(N.ptr(img_b_mask), H, W, N.ptr(rand_u), N.ptr(rand_v), n, N.ptr(matches_a.contiguous()),
                                         int(num_non_matches_per_match), N.ptr(out_a), N.ptr(out_b), N.ptr(scratch), nb,
                                         N.stream_ptr()))
    return out_a, out_b


def find_pixel_correspondences(depth_a, pose_a, depth_b, pose_b, candidates_a, K):
    """Device-side ``batch_find_pixel_correspondences`` (correspondence_finder.py:409-619) for candidate pixels that were
    already drawn in image A (e.g. with ``sample_non_matches(..., img_a_mask, ...)[1]``).
    depth_a / depth_b: float32 [H, W] CUDA depth images in millimetres; pose_a / pose_b: 4x4 camera-to-world (numpy or
    nested lists); K: 3x3 intrinsics; candidates_a: int64 [n] CUDA flat pixels.
    -> (matches_a [m], matches_b [m]) int64 flat pixels and (u2, v2) float32 sub-pixel positions; m is read back once."""
    import ctypes
    import numpy as np
    N.require_cuda_f32(depth_a, "depth_a"); N.require_cuda_f32(depth_b, "depth_b")
    H, W = depth_a.shape
    n = candidates_a.numel()
    dev = depth_a.device
    Kd = np.ascontiguousarray(np.asarray(K, dtype=np.float64).reshape(9))
    Pa = np.ascontiguousarray(np.asarray(pose_a, dtype=np.float64).reshape(16))
    Pb = np.ascontiguousarray(np.asarray(pose_b, dtype=np.float64).reshape(16))
    out_a = torch.empty(n, dtype=torch.int64, device=dev); out_b = torch.empty(n, dtype=torch.int64, device=dev)
    u2 = torch.empty(n, dtype=torch.float32, device=dev); v2 = torch.empty(n, dtype=torch.float32, device=dev)
    count = torch.zeros(1, dtype=torch.int64, device=dev)
    nb = N.lib.ddn_find_pixel_correspondences_scratch_bytes(n)
    scratch = torch.empty(nb, dtype=torch.uint8, device=dev)
    vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    N.check(N.lib.ddn_find_pixel_correspondences(N.ptr(depth_a), N.ptr(depth_b), H, W, N.ptr(candidates_a.contiguous()), n,
                                                 vp(Kd), vp(Pa), vp(Pb), N.ptr(out_a), N.ptr(out_b), N.ptr(u2), N.ptr(v2),
                                                 N.ptr(count), N.ptr(scratch), nb, N.stream_ptr()))
    m = int(count.item())
    return out_a[:m], out_b[:m], u2[:m], v2[:m]


# ----------------------------------------------------------------------------- within-scene training batches
# DEFAULT_IMAGE_MEAN / DEFAULT_IMAGE_STD_DEV (modules/dense_correspondence_manipulation/utils/constants.py:18-19): the
# Normalize of SpartanDataset.rgb_image_to_tensor
IMAGE_MEAN = (0.5573105812072754, 0.37420374155044556, 0.37020164728164673)
IMAGE_STD = (0.24336038529872894, 0.2987397611141205, 0.31875079870224)

_RAND_KEYS = ("cand_u", "cand_v", "masked_u", "masked_v", "background_u", "background_v", "blind")


def within_scene_cfg(training_config):
    """The ``training`` section of a training config -> the sampling sizes of SpartanDataset
    (dense_correspondence_dataset_masked.py:538-551): k = int(fraction * num_non_matches_per_match)."""
    t = training_config["training"]
    nn = t["num_non_matches_per_match"]
    return dict(n_attempts=int(t["num_matching_attempts"]), k_masked=int(t["fraction_masked_non_matches"] * nn),
                k_background=int(t["fraction_background_non_matches"] * nn),
                sample_matches_only_off_mask=bool(t["sample_matches_only_off_mask"]),
                domain_randomize=bool(t["domain_randomize"]), use_image_b_mask_inv=bool(t["use_image_b_mask_inv"]))


def _rand_shapes(B, H, W, c):
    n = c["n_attempts"]
    return {"cand_u": (B, n), "cand_v": (B, n), "masked_u": (B, n * c["k_masked"]), "masked_v": (B, n * c["k_masked"]),
            "background_u": (B, n * c["k_background"]), "background_v": (B, n * c["k_background"]), "blind": (B, H * W)}


def _rand_device(generator, device):
    return torch.device(device) if device is not None else (generator.device if generator is not None else torch.device("cuda"))


def _draw_augment_rand(B, H, W, generator, dev):
    """``params`` and ``noise`` of the background randomisation and flip (the layout of draw_within_scene_rand)."""
    params = torch.zeros(B, 2, N.WS_PARAM_BYTES, dtype=torch.uint8, device=dev)
    params[:, :, :N.WS_RGB1] = torch.randint(0, 2, (B, 2, N.WS_RGB1), dtype=torch.uint8, device=dev, generator=generator)
    params[:, :, N.WS_RGB1:N.WS_RGB2 + 3] = torch.randint(0, 255, (B, 2, 6), dtype=torch.uint8, device=dev, generator=generator)
    return {"params": params,
            "noise": torch.randint(0, 50, (B, 2, 2, H, W, 3), dtype=torch.uint8, device=dev, generator=generator)}


def draw_within_scene_rand(B, H, W, training_config, generator=None, device=None):
    """Every random number ``within_scene_batch`` consumes for B pairs of H x W images, drawn on the device.
    -> dict: ``params`` uint8 [B, 2, 16] (image A, B: randomise / gradient / vertical / noise / flip decisions in {0, 1} at
    bytes 0-4, colours rgb1 at 5-7 and rgb2 at 8-10 in 0..254, the reference's uint8(U * 255)), ``noise`` uint8
    [B, 2, 2, H, W, 3] in 0..49 (uint8(U * 50)), and the uniform fp32 arrays ``cand_u/v`` [B, n_attempts],
    ``masked_u/v`` [B, n_attempts * k_masked], ``background_u/v`` [B, n_attempts * k_background], ``blind`` [B, H * W]."""
    c = within_scene_cfg(training_config)
    dev = _rand_device(generator, device)
    out = _draw_augment_rand(B, H, W, generator, dev)
    shapes = _rand_shapes(B, H, W, c)
    sizes = [shapes[k][0] * shapes[k][1] for k in _RAND_KEYS]
    flat = torch.rand(sum(sizes), device=dev, generator=generator)
    for k, part in zip(_RAND_KEYS, torch.split(flat, sizes)):
        out[k] = part.view(shapes[k])
    return out


def _require(t, name, dtype, shape):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor: this path has no CPU fallback" % name)
    if t.dtype != dtype:
        raise RuntimeError("%s must be %s (got %s)" % (name, dtype, t.dtype))
    if tuple(t.shape) != tuple(shape):
        raise RuntimeError("%s must have shape %s (got %s)" % (name, tuple(shape), tuple(t.shape)))
    return t.contiguous()


def within_scene_batch(rgb_a, rgb_b, depth_a, depth_b, mask_a, mask_b, pose_a, pose_b, K, training_config, generator=None,
                       rand=None):
    """SpartanDataset.get_within_scene_data (dataset/spartan_dataset_masked.py:646-769, SINGLE_OBJECT_WITHIN_SCENE) for B
    image pairs on the device, in one call that never synchronises with the host.

    rgb_*: uint8 [B, H, W, 3]; mask_*: uint8 [B, H, W] (nonzero = object, any value); depth_*: float32 [B, H, W] in
    millimetres; all CUDA.  pose_*: [B, 4, 4] camera-to-world (host, numpy or CPU tensor); K: 3x3 intrinsics.
    ``training_config``: a config with the reference's ``training`` section.  The random numbers are ``rand`` (as returned
    by ``draw_within_scene_rand``) or are drawn from ``generator``.
    -> dict: ``image_a`` / ``image_b`` float32 [B, 3, H, W] (augmented, flipped, normalised); ``matches_a/b``,
    ``masked_non_matches_a/b``, ``background_non_matches_a/b``, ``blind_non_matches_a/b`` int64 [B, cap] padded with -1;
    ``num_valid`` (the ``get_loss`` argument); ``counts`` int64 [B, 4]; ``empty`` bool [B] (the reference's
    return_empty_data: mask_a empty while sampling on it); ``match_type`` (CPU, SINGLE_OBJECT_WITHIN_SCENE per pair)."""
    import ctypes
    import numpy as np
    from .loss_composer import SpartanDatasetDataType
    if training_config.get("training", {}).get("debug", False):
        raise NotImplementedError("within_scene_batch: debug=True (plotting) is not supported")
    c = within_scene_cfg(training_config)
    if not isinstance(rgb_a, torch.Tensor) or rgb_a.dim() != 4:
        raise RuntimeError("rgb_a must be a uint8 CUDA tensor [B, H, W, 3]")
    B, H, W = rgb_a.shape[:3]
    if not 1 <= B <= N.WS_MAX_PAIRS:
        raise RuntimeError("within_scene_batch takes 1 to %d pairs per call (got %d)" % (N.WS_MAX_PAIRS, B))
    dev = rgb_a.device
    rgb_a = _require(rgb_a, "rgb_a", torch.uint8, (B, H, W, 3)); rgb_b = _require(rgb_b, "rgb_b", torch.uint8, (B, H, W, 3))
    mask_a = _require(mask_a, "mask_a", torch.uint8, (B, H, W)); mask_b = _require(mask_b, "mask_b", torch.uint8, (B, H, W))
    depth_a = _require(depth_a, "depth_a", torch.float32, (B, H, W)); depth_b = _require(depth_b, "depth_b", torch.float32, (B, H, W))
    Kd = np.ascontiguousarray(np.asarray(K, dtype=np.float64).reshape(9))
    Pa = np.ascontiguousarray(np.asarray(pose_a, dtype=np.float64))
    Pb = np.ascontiguousarray(np.asarray(pose_b, dtype=np.float64))
    if Pa.shape != (B, 4, 4) or Pb.shape != (B, 4, 4):
        raise RuntimeError("pose_a / pose_b must have shape [B, 4, 4]")
    if rand is None:
        rand = draw_within_scene_rand(B, H, W, training_config, generator=generator, device=dev)
    shapes = dict(_rand_shapes(B, H, W, c), params=(B, 2, N.WS_PARAM_BYTES), noise=(B, 2, 2, H, W, 3))
    rand = {k: _require(rand[k], "rand[%r]" % k, torch.uint8 if k in ("params", "noise") else torch.float32, shapes[k])
            for k in shapes}
    n, cap_m, cap_b = c["n_attempts"], shapes["masked_u"][1], shapes["background_u"][1]
    i64 = dict(dtype=torch.int64, device=dev)
    out = {"image_a": torch.empty(B, 3, H, W, device=dev), "image_b": torch.empty(B, 3, H, W, device=dev),
           "matches_a": torch.empty(B, n, **i64), "matches_b": torch.empty(B, n, **i64),
           "masked_non_matches_a": torch.empty(B, cap_m, **i64), "masked_non_matches_b": torch.empty(B, cap_m, **i64),
           "background_non_matches_a": torch.empty(B, cap_b, **i64), "background_non_matches_b": torch.empty(B, cap_b, **i64),
           "blind_non_matches_a": torch.empty(B, H * W, **i64), "blind_non_matches_b": torch.empty(B, H * W, **i64),
           "counts": torch.empty(B, 4, **i64), "empty": torch.empty(B, dtype=torch.bool, device=dev)}
    cfg = N.WsBatchCfg(B, H, W, int(c["sample_matches_only_off_mask"]), int(c["domain_randomize"]),
                       int(c["use_image_b_mask_inv"]), n, c["k_masked"], c["k_background"],
                       (ctypes.c_float * 3)(*IMAGE_MEAN), (ctypes.c_float * 3)(*IMAGE_STD))
    r = N.WsBatchRand(*[rand[k].data_ptr() or None for k in ("params", "noise") + _RAND_KEYS])
    o = N.WsBatchOut(*[out[k].data_ptr() or None for k in (
        "image_a", "image_b", "matches_a", "matches_b", "masked_non_matches_a", "masked_non_matches_b",
        "background_non_matches_a", "background_non_matches_b", "blind_non_matches_a", "blind_non_matches_b", "counts", "empty")])
    nb = N.lib.ddn_within_scene_batch_scratch_bytes(ctypes.byref(cfg))
    if nb == 0:
        raise RuntimeError("within_scene_batch: configuration refused (%s, B=%d, H=%d, W=%d)" % (c, B, H, W))
    scratch = torch.empty(nb, dtype=torch.uint8, device=dev)
    vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    N.check(N.lib.ddn_within_scene_batch(ctypes.byref(cfg), N.ptr(rgb_a), N.ptr(rgb_b), N.ptr(mask_a), N.ptr(mask_b),
                                         N.ptr(depth_a), N.ptr(depth_b), vp(Kd), vp(Pa), vp(Pb), ctypes.byref(r),
                                         ctypes.byref(o), N.ptr(scratch), nb, N.stream_ptr()))
    cnt = out["counts"].t().contiguous()
    out["num_valid"] = {"matches": cnt[0], "masked": cnt[1], "background": cnt[2], "blind": cnt[3]}
    out["match_type"] = torch.full((B,), SpartanDatasetDataType.SINGLE_OBJECT_WITHIN_SCENE, dtype=torch.int64)
    return out


# ----------------------------------------------------------------------------- across-scene training batches
def across_scene_cfg(training_config):
    """The ``training`` section of a training config -> the sizes of SpartanDataset.get_across_scene_data:
    ``num_samples`` = cross_scene_num_samples (dense_correspondence_dataset_masked.py:549) and domain_randomize."""
    t = training_config["training"]
    return dict(num_samples=int(t["cross_scene_num_samples"]), domain_randomize=bool(t["domain_randomize"]))


def draw_across_scene_rand(B, H, W, training_config, generator=None, device=None):
    """Every random number ``across_scene_batch`` consumes for B pairs of H x W images, drawn on the device.
    -> dict: ``params`` uint8 [B, 2, 16] and ``noise`` uint8 [B, 2, 2, H, W, 3] (as ``draw_within_scene_rand``), and the
    uniform fp32 ``blind_a`` / ``blind_b`` [B, cross_scene_num_samples] (the draws over mask_a and mask_b)."""
    n = across_scene_cfg(training_config)["num_samples"]
    dev = _rand_device(generator, device)
    out = _draw_augment_rand(B, H, W, generator, dev)
    flat = torch.rand(2 * B * n, device=dev, generator=generator)
    out["blind_a"], out["blind_b"] = flat[:B * n].view(B, n), flat[B * n:].view(B, n)
    return out


def across_scene_batch(rgb_a, rgb_b, mask_a, mask_b, training_config, generator=None, rand=None, match_type=None):
    """SpartanDataset.get_across_scene_data (dataset/spartan_dataset_masked.py:1056-1141) for B image pairs on the device,
    in one call that never synchronises with the host: the producer of DIFFERENT_OBJECT (get_different_object_data) and
    SINGLE_OBJECT_ACROSS_SCENE (get_single_object_across_scene_data) pairs, which differ only in ``match_type``.

    rgb_*: uint8 [B, H, W, 3]; mask_*: uint8 [B, H, W] (nonzero = object, any value); all CUDA.  The reference's depth
    and poses only feed its debug plots and are not inputs.  ``training_config``: a config with the reference's
    ``training`` section (cross_scene_num_samples, domain_randomize).  The random numbers are ``rand`` (as returned by
    ``draw_across_scene_rand``) or are drawn from ``generator``.  ``match_type``: DIFFERENT_OBJECT (default) or
    SINGLE_OBJECT_ACROSS_SCENE.
    -> the keys of ``within_scene_batch``: ``image_a`` / ``image_b`` float32 [B, 3, H, W]; ``blind_non_matches_a/b`` int64
    [B, cross_scene_num_samples]; ``matches_a/b``, ``masked_non_matches_a/b``, ``background_non_matches_a/b`` int64 [B, 0];
    ``counts`` int64 [B, 4] (blind count in column 3); ``num_valid``; ``empty`` bool [B] (the reference's
    return_empty_data: mask_a or mask_b empty; that pair's blind rows are -1 and both images are the normalised image A);
    ``match_type`` (CPU)."""
    import ctypes
    from .loss_composer import SpartanDatasetDataType as T
    if match_type is None:
        match_type = T.DIFFERENT_OBJECT
    if match_type not in (T.DIFFERENT_OBJECT, T.SINGLE_OBJECT_ACROSS_SCENE):
        raise ValueError("across_scene_batch: match_type must be DIFFERENT_OBJECT or SINGLE_OBJECT_ACROSS_SCENE (got %r)"
                         % (match_type,))
    if training_config.get("training", {}).get("debug", False):
        raise NotImplementedError("across_scene_batch: debug=True (plotting) is not supported")
    c = across_scene_cfg(training_config)
    if not isinstance(rgb_a, torch.Tensor) or rgb_a.dim() != 4:
        raise RuntimeError("rgb_a must be a uint8 CUDA tensor [B, H, W, 3]")
    B, H, W = rgb_a.shape[:3]
    if not 1 <= B <= N.AS_MAX_PAIRS:
        raise RuntimeError("across_scene_batch takes 1 to %d pairs per call (got %d)" % (N.AS_MAX_PAIRS, B))
    dev = rgb_a.device
    rgb_a = _require(rgb_a, "rgb_a", torch.uint8, (B, H, W, 3)); rgb_b = _require(rgb_b, "rgb_b", torch.uint8, (B, H, W, 3))
    mask_a = _require(mask_a, "mask_a", torch.uint8, (B, H, W)); mask_b = _require(mask_b, "mask_b", torch.uint8, (B, H, W))
    if rand is None:
        rand = draw_across_scene_rand(B, H, W, training_config, generator=generator, device=dev)
    n = c["num_samples"]
    shapes = dict(params=(B, 2, N.WS_PARAM_BYTES), noise=(B, 2, 2, H, W, 3), blind_a=(B, n), blind_b=(B, n))
    rand = {k: _require(rand[k], "rand[%r]" % k, torch.uint8 if k in ("params", "noise") else torch.float32, shapes[k])
            for k in shapes}
    i64 = dict(dtype=torch.int64, device=dev)
    none = torch.empty(B, 0, **i64)
    out = {"image_a": torch.empty(B, 3, H, W, device=dev), "image_b": torch.empty(B, 3, H, W, device=dev),
           "matches_a": none, "matches_b": none.clone(), "masked_non_matches_a": none.clone(),
           "masked_non_matches_b": none.clone(), "background_non_matches_a": none.clone(),
           "background_non_matches_b": none.clone(),
           "blind_non_matches_a": torch.empty(B, n, **i64), "blind_non_matches_b": torch.empty(B, n, **i64),
           "counts": torch.empty(B, 4, **i64), "empty": torch.empty(B, dtype=torch.bool, device=dev)}
    cfg = N.AsBatchCfg(B, H, W, int(c["domain_randomize"]), n, (ctypes.c_float * 3)(*IMAGE_MEAN), (ctypes.c_float * 3)(*IMAGE_STD))
    r = N.AsBatchRand(*[rand[k].data_ptr() for k in ("params", "noise", "blind_a", "blind_b")])
    o = N.AsBatchOut(*[out[k].data_ptr() for k in ("image_a", "image_b", "blind_non_matches_a", "blind_non_matches_b",
                                                   "counts", "empty")])
    nb = N.lib.ddn_across_scene_batch_scratch_bytes(ctypes.byref(cfg))
    if nb == 0:
        raise RuntimeError("across_scene_batch: configuration refused (%s, B=%d, H=%d, W=%d)" % (c, B, H, W))
    scratch = torch.empty(nb, dtype=torch.uint8, device=dev)
    N.check(N.lib.ddn_across_scene_batch(ctypes.byref(cfg), N.ptr(rgb_a), N.ptr(rgb_b), N.ptr(mask_a), N.ptr(mask_b),
                                         ctypes.byref(r), ctypes.byref(o), N.ptr(scratch), nb, N.stream_ptr()))
    cnt = out["counts"].t().contiguous()
    out["num_valid"] = {"matches": cnt[0], "masked": cnt[1], "background": cnt[2], "blind": cnt[3]}
    out["match_type"] = torch.full((B,), int(match_type), dtype=torch.int64)
    return out


# ----------------------------------------------------------------------------- mixed pair-type batches
# The order in which SpartanDataset lists the types it draws from (dense_correspondence_dataset_masked.py:557-586)
DATA_TYPE_ORDER = ("SINGLE_OBJECT_WITHIN_SCENE", "SINGLE_OBJECT_ACROSS_SCENE", "DIFFERENT_OBJECT", "MULTI_OBJECT",
                   "SYNTHETIC_MULTI_OBJECT")
INDEX_KEYS = ("matches_a", "matches_b", "masked_non_matches_a", "masked_non_matches_b", "background_non_matches_a",
              "background_non_matches_b", "blind_non_matches_a", "blind_non_matches_b")


def draw_data_types(B, training_config, generator=None):
    """One SpartanDatasetDataType per pair, drawn as SpartanDataset draws one per sample (_get_data_load_type,
    dense_correspondence_dataset_masked.py:557-586 and np.random.choice): the types of
    ``training.data_type_probabilities`` with p > 0, in the reference's order, probabilities normalised, each pair drawn
    independently (uniform u, first type whose cumulative probability exceeds u).  ``generator``: a CPU torch.Generator,
    so a seed gives the same types on every machine.  -> CPU int64 [B]."""
    from .loss_composer import SpartanDatasetDataType
    probs = training_config.get("training", {}).get("data_type_probabilities")
    if probs is None:
        raise ValueError("training_config has no training.data_type_probabilities")
    if isinstance(B, bool) or not isinstance(B, int) or B < 1:
        raise ValueError("B must be a positive int (got %r)" % (B,))
    if generator is not None and generator.device.type != "cpu":
        raise ValueError("draw_data_types draws with a CPU torch.Generator (got one on %s)" % generator.device)
    types, p = [], []
    for name in DATA_TYPE_ORDER:
        if name not in probs:
            raise ValueError("data_type_probabilities has no %s" % name)
        v = float(probs[name])
        if not v >= 0.0 or v == float("inf"):
            raise ValueError("data_type_probabilities[%s] must be finite and >= 0 (got %r)" % (name, probs[name]))
        if v > 0:
            types.append(getattr(SpartanDatasetDataType, name))
            p.append(v)
    if not p:
        raise ValueError("every data_type_probabilities entry is 0")
    cdf = torch.tensor(p, dtype=torch.float64).cumsum(0)
    cdf /= cdf[-1].clone()
    u = torch.rand(B, dtype=torch.float64, generator=generator)
    idx = torch.searchsorted(cdf, u, right=True).clamp_(max=len(p) - 1)
    return torch.tensor(types, dtype=torch.int64)[idx]


def concat_batches(parts):
    """One batch from several producer outputs (``within_scene_batch``, ``across_scene_batch``,
    ``synthetic_multi_object_batch``, any ``match_type`` relabelling kept), pairs in part order: the images concatenated,
    each index key padded with -1 to the widest part then concatenated, ``counts``, ``empty`` and ``match_type``
    concatenated and ``num_valid`` rebuilt from ``counts``.  Pair order does not change the loss or the BatchNorm
    statistics, so no shuffle is needed.  Everything stays on the device without a host synchronisation; the number of
    launches depends on the number of parts, not on B."""
    if not parts:
        raise ValueError("concat_batches needs at least one part")
    shape = tuple(parts[0]["image_a"].shape[1:])
    match_types = []
    for i, p in enumerate(parts):
        if tuple(p["image_a"].shape[1:]) != shape or tuple(p["image_b"].shape[1:]) != shape:
            raise ValueError("concat_batches: every part must have images of shape [B, %s]" % ", ".join(map(str, shape)))
        mt = torch.as_tensor(p["match_type"])
        if mt.device.type != "cpu":      # the types are checked and read on the host (get_mixed_loss), without a sync
            raise ValueError("concat_batches: match_type of part %d is on %s; keep it the CPU tensor the producers return "
                             "(relabel with torch.full_like(out[\"match_type\"], t))" % (i, mt.device))
        if tuple(mt.shape) != (p["image_a"].shape[0],):
            raise ValueError("concat_batches: match_type of part %d must have shape [%d] (got %s)"
                             % (i, p["image_a"].shape[0], tuple(mt.shape)))
        match_types.append(mt.to(torch.int64))
    rows = [p["image_a"].shape[0] for p in parts]
    dev = parts[0]["image_a"].device
    out = {"image_a": torch.cat([p["image_a"] for p in parts]), "image_b": torch.cat([p["image_b"] for p in parts])}
    for k in INDEX_KEYS:
        width = max(p[k].shape[1] for p in parts)
        t = torch.empty(sum(rows), width, dtype=torch.int64, device=dev)
        r = 0
        for p, n in zip(parts, rows):
            w = p[k].shape[1]
            t[r:r + n, :w].copy_(p[k])
            if w < width:
                t[r:r + n, w:].fill_(-1)
            r += n
        out[k] = t
    out["counts"] = torch.cat([p["counts"] for p in parts])
    out["empty"] = torch.cat([p["empty"] for p in parts])
    out["match_type"] = torch.cat(match_types)
    cnt = out["counts"].t().contiguous()
    out["num_valid"] = {"matches": cnt[0], "masked": cnt[1], "background": cnt[2], "blind": cnt[3]}
    return out


# ----------------------------------------------------------------------------- synthetic multi-object training batches
_SMO_RAND_KEYS = ("cand_u", "cand_v", "masked_u", "masked_v", "background_u", "background_v")


def _smo_rand_shapes(B, c):
    n = c["n_attempts"]
    return {"cand_u": (B, 2, n), "cand_v": (B, 2, n), "masked_u": (B, 2 * n * c["k_masked"]),
            "masked_v": (B, 2 * n * c["k_masked"]), "background_u": (B, 2 * n * c["k_background"]),
            "background_v": (B, 2 * n * c["k_background"])}


def draw_synthetic_multi_object_rand(B, H, W, training_config, generator=None, device=None):
    """Every random number ``synthetic_multi_object_batch`` consumes for B pairs, drawn on the device.
    -> dict: ``merge`` uint8 [B, 2] in {0, 1} (1: merge 1 / merge 2 puts scene B in the foreground, the reference's
    ``random.random() < 0.5``), and the uniform fp32 ``cand_u/v`` [B, 2 (scene A, scene B), n_attempts],
    ``masked_u/v`` [B, 2 * n_attempts * k_masked], ``background_u/v`` [B, 2 * n_attempts * k_background].  H and W are
    accepted for symmetry with the other producers; no number depends on them."""
    c = within_scene_cfg(training_config)
    dev = _rand_device(generator, device)
    out = {"merge": torch.randint(0, 2, (B, 2), dtype=torch.uint8, device=dev, generator=generator)}
    shapes = _smo_rand_shapes(B, c)
    sizes = [int(np.prod(shapes[k])) for k in _SMO_RAND_KEYS]
    flat = torch.rand(sum(sizes), device=dev, generator=generator)
    for k, part in zip(_SMO_RAND_KEYS, torch.split(flat, sizes)):
        out[k] = part.view(shapes[k])
    return out


def synthetic_multi_object_batch(scene_a, scene_b, K, training_config, generator=None, rand=None):
    """SpartanDataset.get_synthetic_multi_object_within_scene_data (dataset/spartan_dataset_masked.py:890-1053,
    SYNTHETIC_MULTI_OBJECT) for B pairs on the device, in one call that never synchronises with the host.

    scene_a, scene_b: 8-tuples ``(rgb_1, rgb_2, depth_1, depth_2, mask_1, mask_2, pose_1, pose_2)`` in
    ``within_scene_batch``'s argument order: rgb uint8 [B, H, W, 3], depth float32 [B, H, W] (millimetres), mask uint8
    [B, H, W] (CUDA); poses [B, 4, 4] camera-to-world on the host.  K: 3x3 intrinsics, shared by both scenes.  The random
    numbers are ``rand`` (as returned by ``draw_synthetic_multi_object_rand``) or are drawn from ``generator``.
    -> the keys of ``within_scene_batch``: ``image_a`` / ``image_b`` float32 [B, 3, H, W] (merged images 1 and 2);
    ``matches_a/b`` [B, 2 * n_attempts], ``masked_non_matches_a/b`` [B, 2 * n_attempts * k_masked],
    ``background_non_matches_a/b`` [B, 2 * n_attempts * k_background], ``blind_non_matches_a/b`` [B, 1] (always -1: the
    reference returns empty_tensor()), int64 padded with -1; ``counts`` int64 [B, 4]; ``num_valid``; ``empty`` bool [B]
    (one of the reference's four early returns); ``match_type`` (CPU, SYNTHETIC_MULTI_OBJECT).  At most 64 pairs per call:
    each pair's two reprojection matrix sets travel as kernel parameters."""
    import ctypes
    from .loss_composer import SpartanDatasetDataType
    if training_config.get("training", {}).get("debug", False):
        raise NotImplementedError("synthetic_multi_object_batch: debug=True (plotting) is not supported")
    c = within_scene_cfg(training_config)
    if len(scene_a) != 8 or len(scene_b) != 8:
        raise RuntimeError("scene_a / scene_b must be (rgb_1, rgb_2, depth_1, depth_2, mask_1, mask_2, pose_1, pose_2)")
    if not isinstance(scene_a[0], torch.Tensor) or scene_a[0].dim() != 4:
        raise RuntimeError("rgb_1 must be a uint8 CUDA tensor [B, H, W, 3]")
    B, H, W = scene_a[0].shape[:3]
    if not 1 <= B <= N.SMO_MAX_PAIRS:
        raise RuntimeError("synthetic_multi_object_batch takes 1 to %d pairs per call (got %d)" % (N.SMO_MAX_PAIRS, B))
    dev = scene_a[0].device
    spec = (("rgb_1", torch.uint8, (B, H, W, 3)), ("rgb_2", torch.uint8, (B, H, W, 3)), ("depth_1", torch.float32, (B, H, W)),
            ("depth_2", torch.float32, (B, H, W)), ("mask_1", torch.uint8, (B, H, W)), ("mask_2", torch.uint8, (B, H, W)))
    stacked = {}
    for i, (name, dt, shape) in enumerate(spec):
        a = _require(scene_a[i], "scene_a." + name, dt, shape); b = _require(scene_b[i], "scene_b." + name, dt, shape)
        stacked[name] = torch.stack((a, b), dim=1)              # [B, 2 (scene A, scene B), ...]
    poses = {}
    for i, name in ((6, "pose_1"), (7, "pose_2")):
        pa = np.asarray(scene_a[i], dtype=np.float64); pb = np.asarray(scene_b[i], dtype=np.float64)
        if pa.shape != (B, 4, 4) or pb.shape != (B, 4, 4):
            raise RuntimeError("%s must have shape [B, 4, 4]" % name)
        poses[name] = np.ascontiguousarray(np.stack((pa, pb), axis=1))
    Kd = np.ascontiguousarray(np.asarray(K, dtype=np.float64).reshape(9))
    if rand is None:
        rand = draw_synthetic_multi_object_rand(B, H, W, training_config, generator=generator, device=dev)
    shapes = dict(_smo_rand_shapes(B, c), merge=(B, 2))
    rand = {k: _require(rand[k], "rand[%r]" % k, torch.uint8 if k == "merge" else torch.float32, shapes[k]) for k in shapes}
    n = c["n_attempts"]
    cap_m, cap_b = shapes["masked_u"][1], shapes["background_u"][1]
    i64 = dict(dtype=torch.int64, device=dev)
    out = {"image_a": torch.empty(B, 3, H, W, device=dev), "image_b": torch.empty(B, 3, H, W, device=dev),
           "matches_a": torch.empty(B, 2 * n, **i64), "matches_b": torch.empty(B, 2 * n, **i64),
           "masked_non_matches_a": torch.empty(B, cap_m, **i64), "masked_non_matches_b": torch.empty(B, cap_m, **i64),
           "background_non_matches_a": torch.empty(B, cap_b, **i64), "background_non_matches_b": torch.empty(B, cap_b, **i64),
           "blind_non_matches_a": torch.empty(B, 1, **i64), "blind_non_matches_b": torch.empty(B, 1, **i64),
           "counts": torch.empty(B, 4, **i64), "empty": torch.empty(B, dtype=torch.bool, device=dev)}
    cfg = N.SmoBatchCfg(B, H, W, int(c["sample_matches_only_off_mask"]), int(c["use_image_b_mask_inv"]), n, c["k_masked"],
                        c["k_background"], (ctypes.c_float * 3)(*IMAGE_MEAN), (ctypes.c_float * 3)(*IMAGE_STD))
    r = N.SmoBatchRand(*[rand[k].data_ptr() or None for k in ("merge",) + _SMO_RAND_KEYS])
    o = N.SmoBatchOut(*[out[k].data_ptr() or None for k in (
        "image_a", "image_b", "matches_a", "matches_b", "masked_non_matches_a", "masked_non_matches_b",
        "background_non_matches_a", "background_non_matches_b", "blind_non_matches_a", "blind_non_matches_b", "counts", "empty")])
    nb = N.lib.ddn_synthetic_multi_object_batch_scratch_bytes(ctypes.byref(cfg))
    if nb == 0:
        raise RuntimeError("synthetic_multi_object_batch: configuration refused (%s, B=%d, H=%d, W=%d)" % (c, B, H, W))
    scratch = torch.empty(nb, dtype=torch.uint8, device=dev)
    vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    N.check(N.lib.ddn_synthetic_multi_object_batch(
        ctypes.byref(cfg), N.ptr(stacked["rgb_1"]), N.ptr(stacked["rgb_2"]), N.ptr(stacked["mask_1"]), N.ptr(stacked["mask_2"]),
        N.ptr(stacked["depth_1"]), N.ptr(stacked["depth_2"]), vp(Kd), vp(poses["pose_1"]), vp(poses["pose_2"]),
        ctypes.byref(r), ctypes.byref(o), N.ptr(scratch), nb, N.stream_ptr()))
    cnt = out["counts"].t().contiguous()
    out["num_valid"] = {"matches": cnt[0], "masked": cnt[1], "background": cnt[2], "blind": cnt[3]}
    out["match_type"] = torch.full((B,), SpartanDatasetDataType.SYNTHETIC_MULTI_OBJECT, dtype=torch.int64)
    return out
