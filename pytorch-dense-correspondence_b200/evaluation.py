"""Per-match evaluation statistics on the device (SURVEY.md 8f row 4): the columns that
``DenseCorrespondenceEvaluation.compute_descriptor_match_statistics`` (dense_correspondence/evaluation/evaluation.py:1006-1178)
records for each ground-truth match, for many matches over many image pairs in one launch (csrc/match_stats.cu).

``match_statistics`` is the batched entry point (CUDA tensors in, a dict of CUDA tensors out, no host synchronisation).
``DenseCorrespondenceEvaluation`` keeps the reference's signatures for the per-match call and its helpers, and
``quantitative_analysis_on_pair`` is the dataset-free body of ``single_same_scene_image_pair_quantitative_analysis``
(evaluation.py:862-958).

Two further steps of ``run_evaluation_on_network`` (evaluation.py:2308-2410) that need no dataset stack:
``descriptor_statistics`` / ``descriptor_statistics_over_images`` / ``save_descriptor_statistics`` compute and write
descriptor_statistics.yaml (``compute_descriptor_statistics_on_dataset``, :2157-2305; csrc/descriptor_stats.cu), which
``DenseCorrespondenceNetwork.descriptor_image_stats`` reads back; ``best_match_batch`` / ``across_object_analysis`` are
the across-object analysis (``evaluate_network_across_objects``, :305-338, 784-858, 977-1004) in one best-match launch.

Reference quirks that are kept: the depth at uv_a is never checked for validity (evaluation.py:1103); ``compute_3d_position``
is called with (u, v) although its docstring says (row, column) (:1112-1115, :1185); an empty mask_b divides by an integer
zero (:1086), which the batched call reports as a NaN fraction and ``compute_descriptor_match_statistics`` as
``ZeroDivisionError``.  The threshold ``norm_diff_descriptor_ground_truth`` is nd(uv_b) computed like every other pixel's
distance; the reference takes it from np.linalg.norm (a BLAS dot, :1070), which can differ from it in the last bits.
"""
import ctypes

import numpy as np
import torch

from . import _native as N

DEPTH_IM_SCALE = 1000.0

# DCNEvaluationPandaTemplate.columns (evaluation.py:37-61)
COLUMNS = ['scene_name', 'scene_name_a', 'scene_name_b', 'object_id_a', 'object_id_b', 'img_a_idx', 'img_b_idx', 'is_valid',
           'is_valid_masked', 'norm_diff_descriptor_ground_truth', 'norm_diff_descriptor', 'norm_diff_descriptor_masked',
           'norm_diff_ground_truth_3d', 'norm_diff_pred_3d', 'norm_diff_pred_3d_masked', 'pixel_match_error_l2',
           'pixel_match_error_l2_masked', 'pixel_match_error_l1', 'fraction_pixels_closer_than_ground_truth',
           'fraction_pixels_closer_than_ground_truth_masked', 'average_l2_distance_for_false_positives',
           'average_l2_distance_for_false_positives_masked', 'keypoint_name']

# column order of the three output blocks of ddn_match_statistics (DDN_MS_* in include/ddn_b200.h)
F32_COLUMNS = ['norm_diff_descriptor_ground_truth', 'norm_diff_descriptor']
F64_COLUMNS = ['norm_diff_descriptor_masked', 'norm_diff_ground_truth_3d', 'norm_diff_pred_3d', 'norm_diff_pred_3d_masked',
               'pixel_match_error_l2', 'pixel_match_error_l2_masked', 'pixel_match_error_l1',
               'fraction_pixels_closer_than_ground_truth', 'fraction_pixels_closer_than_ground_truth_masked',
               'average_l2_distance_for_false_positives', 'average_l2_distance_for_false_positives_masked']
I64_COLUMNS = ['is_valid', 'is_valid_masked', 'u_pred', 'v_pred', 'u_pred_masked', 'v_pred_masked',
               'num_pixels_closer_than_ground_truth', 'num_pixels_closer_than_ground_truth_masked', 'num_pixels_in_masked_image']
MAX_D = 32


def _batched(t, name, ndim, device=None):
    """[N, ...] (or a single image without the N axis) -> CUDA tensor with the N axis."""
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor: this path has no CPU fallback" % name)
    if t.dim() == ndim - 1:
        t = t.unsqueeze(0)
    if t.dim() != ndim:
        raise RuntimeError("%s must have %d dimensions (got shape %s)" % (name, ndim, tuple(t.shape)))
    if device is not None and t.device != device:
        raise RuntimeError("%s is on %s, the descriptors on %s" % (name, t.device, device))
    return t


def _index(t, name, shape_tail, device):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor" % name)
    if t.dtype != torch.int64:
        raise RuntimeError("%s must be int64 (got %s)" % (name, t.dtype))
    if t.dim() != 1 + len(shape_tail) or tuple(t.shape[1:]) != shape_tail:
        raise RuntimeError("%s must have shape [Q%s] (got %s)" % (name, "".join(", %d" % s for s in shape_tail), tuple(t.shape)))
    if t.device != device:
        raise RuntimeError("%s is on %s, the descriptors on %s" % (name, t.device, device))
    return t.contiguous()


def _host_f64(x, shape, name):
    a = np.ascontiguousarray(np.asarray(x.cpu() if isinstance(x, torch.Tensor) else x, dtype=np.float64))
    if a.shape != shape:
        a = a.reshape(shape) if a.size == int(np.prod(shape)) else None
    if a is None:
        raise RuntimeError("%s must hold %s float64 values" % (name, shape))
    return a


def match_statistics(res_a, res_b, uv_a, uv_b, pair, mask_b, depth_a, depth_b, poses_a, poses_b, K):
    """The statistics of compute_descriptor_match_statistics for Q matches over N image pairs, in one launch.

    res_a, res_b  [N,H,W,D] (or [H,W,D]) float32 CUDA descriptor images, any strides (forward_single_image_tensor's view).
    uv_a, uv_b    [Q,2] int64 CUDA (u, v) pixels; uv_b already clipped and rounded (clip_pixel_to_image_size_and_round).
    pair          [Q] int64 CUDA: the image pair of each match.  Keeping one pair's matches together is fastest.
    mask_b        [N,H,W] CUDA (1 on the object), depth_a / depth_b [N,H,W] CUDA in millimetres (any real dtype).
    poses_a/b     [N,4,4] camera-to-world (host arrays), K the 3x3 intrinsics (host); inv(K) is taken with numpy as the
                  reference does.
    -> {column: [Q] CUDA tensor} with the reference's column names (float32 / float64 as the reference computes them,
    is_valid* bool) plus the extra integer columns of I64_COLUMNS and "bad_queries" (int64 [1]: queries whose pair or
    pixel indices were out of range; their rows are NaN / -1).  Nothing is read back to the host."""
    if not isinstance(res_a, torch.Tensor) or not isinstance(res_b, torch.Tensor):
        raise RuntimeError("res_a and res_b must be CUDA tensors")
    N.require_cuda_f32(res_a, "res_a", contiguous=False); N.require_cuda_f32(res_b, "res_b", contiguous=False)
    res_a = _batched(res_a, "res_a", 4); res_b = _batched(res_b, "res_b", 4, device=res_a.device)
    dev = res_a.device
    n, H, W, D = res_b.shape
    if tuple(res_a.shape) != (n, H, W, D):
        raise RuntimeError("res_a %s and res_b %s must have the same shape" % (tuple(res_a.shape), tuple(res_b.shape)))
    if not 1 <= D <= MAX_D:
        raise RuntimeError("descriptor dimension %d outside 1..%d" % (D, MAX_D))
    maps = []
    for t, name in ((mask_b, "mask_b"), (depth_a, "depth_a"), (depth_b, "depth_b")):
        t = _batched(t, name, 3, device=dev)
        if tuple(t.shape) != (n, H, W):
            raise RuntimeError("%s must have shape %s (got %s)" % (name, (n, H, W), tuple(t.shape)))
        maps.append(t.to(torch.float32).contiguous())
    uv_a = _index(uv_a, "uv_a", (2,), dev); uv_b = _index(uv_b, "uv_b", (2,), dev); pair = _index(pair, "pair", (), dev)
    Q = uv_a.shape[0]
    if uv_b.shape[0] != Q or pair.shape[0] != Q:
        raise RuntimeError("uv_a, uv_b and pair must have the same length")
    Kinv = np.ascontiguousarray(np.linalg.inv(_host_f64(K, (3, 3), "K")))
    Pa = _host_f64(poses_a, (n, 4, 4), "poses_a"); Pb = _host_f64(poses_b, (n, 4, 4), "poses_b")
    f32 = torch.empty(Q, len(F32_COLUMNS), dtype=torch.float32, device=dev)
    f64 = torch.empty(Q, len(F64_COLUMNS), dtype=torch.float64, device=dev)
    i64 = torch.empty(Q, len(I64_COLUMNS), dtype=torch.int64, device=dev)
    bad = torch.empty(1, dtype=torch.int64, device=dev)
    nb = N.lib.ddn_match_statistics_scratch_bytes(n, H, W, Q)
    if nb == 0:
        raise N.DdnError(N.lib.ddn_last_error().decode())
    scratch = torch.empty(nb, dtype=torch.uint8, device=dev)
    hp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    sa = np.array(res_a.stride(), dtype=np.int64); sb = np.array(res_b.stride(), dtype=np.int64)
    N.check(N.lib.ddn_match_statistics(N.ptr(res_a), hp(sa), N.ptr(res_b), hp(sb), n, H, W, D, N.ptr(pair), N.ptr(uv_a), N.ptr(uv_b),
                                       Q, N.ptr(maps[0]), N.ptr(maps[1]), N.ptr(maps[2]), hp(Kinv), hp(Pa), hp(Pb), N.ptr(f32),
                                       N.ptr(f64), N.ptr(i64), N.ptr(bad), N.ptr(scratch), nb, N.stream_ptr()))
    out = {k: f32[:, i] for i, k in enumerate(F32_COLUMNS)}
    out.update({k: f64[:, i] for i, k in enumerate(F64_COLUMNS)})
    out.update({k: i64[:, i] for i, k in enumerate(I64_COLUMNS)})
    out["is_valid"] = out["is_valid"] == 1
    out["is_valid_masked"] = out["is_valid_masked"] == 1
    out["bad_queries"] = bad
    return out


class PandaDataFrameWrapper(object):
    """evaluation/utils.py:13-38: one pandas row whose columns are fixed at construction."""

    def __init__(self, columns):
        import pandas as pd
        data = [np.nan] * len(columns)
        self._columns = columns
        self._df = pd.DataFrame(data=[data], columns=columns)

    def set_value(self, key, value):
        if key not in self._columns:
            raise KeyError("%s is not in the index" % (key))
        self._df[key] = value

    def get_value(self, key):
        return self._df[key]

    @property
    def dataframe(self):
        return self._df


class DCNEvaluationPandaTemplate(PandaDataFrameWrapper):
    columns = COLUMNS

    def __init__(self):
        PandaDataFrameWrapper.__init__(self, DCNEvaluationPandaTemplate.columns)


def _descriptors(res):
    if isinstance(res, torch.Tensor):
        return res if res.is_cuda else res.cuda()
    return torch.from_numpy(np.ascontiguousarray(res, dtype=np.float32)).cuda()


class DenseCorrespondenceEvaluation(object):
    """The per-match statistics of the reference's DenseCorrespondenceEvaluation (evaluation.py), computed on the device."""

    @staticmethod
    def clip_pixel_to_image_size_and_round(uv, image_width, image_height):
        """evaluation.py:603-607 (Python 3 round: halves go to the even neighbour)."""
        u = min(int(round(uv[0])), image_width - 1)
        v = min(int(round(uv[1])), image_height - 1)
        return (u, v)

    @staticmethod
    def is_depth_valid(depth):
        """evaluation.py:960-972; depth in metres."""
        MAX_DEPTH = 10.0
        return ((depth > 0) and (depth < MAX_DEPTH))

    @staticmethod
    def compute_3d_position(uv, depth, camera_intrinsics_matrix, camera_to_world):
        """evaluation.py:1180-1200 with pinhole_projection_image_to_world (correspondence_finder.py:123-144): uv is (u, v)
        as the reference passes it, although its docstring says (row, column)."""
        u_v_1 = np.array([uv[0], uv[1], 1])
        pos_in_camera_frame = depth * np.linalg.inv(camera_intrinsics_matrix).dot(u_v_1)
        return np.dot(camera_to_world, np.append(pos_in_camera_frame, 1))[:3]

    @staticmethod
    def compute_descriptor_match_statistics(depth_a, depth_b, mask_a, mask_b, uv_a, uv_b, pose_a, pose_b,
                                            res_a, res_b, camera_matrix, params=None,
                                            rgb_a=None, rgb_b=None, debug=False):
        """evaluation.py:1006-1178 for one match, on the device.  res_a / res_b [H,W,D]: numpy arrays or CUDA tensors;
        depth_* in millimetres, mask_b 1 on the object.  -> DCNEvaluationPandaTemplate.  Reads the row back to the host."""
        if debug:
            raise NotImplementedError("debug=True plots the match; plotting is not part of this package")
        ra, rb = _descriptors(res_a), _descriptors(res_b)
        H, W = rb.shape[0], rb.shape[1]
        for name, (u, v) in (("uv_a", uv_a), ("uv_b", uv_b)):
            if not (0 <= int(u) < W and 0 <= int(v) < H):
                raise IndexError("%s = %s lies outside the %dx%d image" % (name, (u, v), W, H))
        dev = rb.device
        mb = torch.as_tensor(np.asarray(mask_b)).to(dev)
        if int(torch.count_nonzero(mb)) == 0:
            raise ZeroDivisionError("mask_b is empty: the masked fraction divides by zero (evaluation.py:1086)")
        da = torch.as_tensor(np.asarray(depth_a, dtype=np.float32)).to(dev)
        db = torch.as_tensor(np.asarray(depth_b, dtype=np.float32)).to(dev)
        q = lambda uv: torch.tensor([[int(uv[0]), int(uv[1])]], dtype=torch.int64, device=dev)
        out = match_statistics(ra, rb, q(uv_a), q(uv_b), torch.zeros(1, dtype=torch.int64, device=dev), mb, da, db,
                               np.asarray(pose_a)[None], np.asarray(pose_b)[None], camera_matrix)
        t = DCNEvaluationPandaTemplate()
        for k in F32_COLUMNS:
            t.set_value(k, np.float32(out[k].item()))
        for k in F64_COLUMNS:
            t.set_value(k, float(out[k].item()))
        t.set_value('is_valid', bool(out['is_valid'].item()))
        t.set_value('is_valid_masked', bool(out['is_valid_masked'].item()))
        return t


def quantitative_analysis_on_pair(dcn, rgb_a, rgb_b, depth_a, depth_b, mask_a, mask_b, pose_a, pose_b, K, num_matches=100,
                                  generator=None, num_attempts=20):
    """The dataset-free body of single_same_scene_image_pair_quantitative_analysis (evaluation.py:862-958) on the device.

    rgb_a / rgb_b [3,H,W] normalised image tensors (dataset.rgb_image_to_tensor's output); depth_* [H,W] in millimetres;
    mask_* [H,W] (1 on the object); pose_* 4x4 camera-to-world; K 3x3; generator: a CUDA torch.Generator or None.  Runs the eval-mode forward of both images, draws
    `num_attempts` candidate pixels from mask_a (batch_find_pixel_correspondences' default is 20), finds their matches
    with the reprojection finder, keeps `num_matches` of them drawn without replacement and computes their statistics.
    The reference draws with Python's `random.sample`, which cannot be reproduced here: the chosen matches differ, each
    row's values do not.
    -> dict of host numpy arrays: the statistics columns, I64_COLUMNS, and "uv_a" / "uv_b" [M,2] of the chosen matches;
    None when no match survives (the reference returns None too)."""
    from . import sampling
    H, W = dcn.image_shape
    with torch.no_grad():
        res_a = dcn.forward_single_image_tensor(rgb_a)
        res_b = dcn.forward_single_image_tensor(rgb_b)
    dev = res_a.device
    f = lambda x: torch.as_tensor(np.asarray(x.cpu() if isinstance(x, torch.Tensor) else x, dtype=np.float32)).to(dev)
    da, db, ma, mb = f(depth_a), f(depth_b), f(mask_a), f(mask_b)
    dummy = torch.zeros(1, dtype=torch.int64, device=dev)
    _, cand = sampling.sample_non_matches(dummy, ma, (H, W), num_attempts, generator=generator)
    matches_a, _, u2, v2 = sampling.find_pixel_correspondences(da, pose_a, db, pose_b, cand, K)
    m = matches_a.numel()
    if m == 0:
        return None
    pick = torch.randperm(m, generator=generator, device=dev)[:min(num_matches, m)]
    uv_a = torch.stack([matches_a[pick] % W, matches_a[pick] // W], 1)
    # clip_pixel_to_image_size_and_round on the device: torch.round is Python 3's round (halves to even)
    uv_b = torch.stack([torch.round(u2[pick]).long().clamp(max=W - 1), torch.round(v2[pick]).long().clamp(max=H - 1)], 1)
    out = match_statistics(res_a, res_b, uv_a, uv_b, torch.zeros(len(pick), dtype=torch.int64, device=dev), mb, da, db,
                           np.asarray(pose_a)[None], np.asarray(pose_b)[None], K)
    rows = {k: v.cpu().numpy() for k, v in out.items() if k != "bad_queries"}
    rows["uv_a"] = uv_a.cpu().numpy(); rows["uv_b"] = uv_b.cpu().numpy()
    return rows


# ---------------------------------------------------------------------------------------------------------------------
# Descriptor statistics (compute_descriptor_statistics_on_dataset, evaluation.py:2157-2305; csrc/descriptor_stats.cu)

STAT_KEYS = ['min', 'max', 'mean', 'mask_min', 'mask_max', 'mask_mean']      # row order of ddn_descriptor_statistics


def descriptor_statistics(res, mask):
    """Per-image, per-channel descriptor statistics of N images in one launch (compute_descriptor_statistics,
    evaluation.py:2177-2219).

    res   [N,H,W,D] (or [H,W,D]) float32 CUDA, any strides: pass the network's NCHW output as ``res.permute(0, 2, 3, 1)``
          and forward_single_image_tensor's [H,W,D] view as it is; neither is copied.  1 <= D <= 32.
    mask  [N,H,W] (or [H,W]) CUDA float32, uint8 or bool; nonzero = object.
    -> {'min', 'max', 'mean', 'mask_min', 'mask_max', 'mask_mean': [N,D] float32, 'mask_count': [N] int64} CUDA tensors,
    without a host synchronisation.  Whole-image statistics use every pixel, mask statistics the nonzero mask pixels; an
    image with an empty mask has mask_count 0 and NaN mask statistics.  min / max are torch.min / torch.max exactly;
    means are fp64 sums rounded once to float32 (torch's float32 mean may differ from them in the last bits)."""
    if not isinstance(res, torch.Tensor) or not res.is_cuda:
        raise RuntimeError("res must be a CUDA tensor: this path has no CPU fallback")
    N.require_cuda_f32(res, "res", contiguous=False)
    res = _batched(res, "res", 4)
    n, H, W, D = res.shape
    if not 1 <= D <= MAX_D:
        raise RuntimeError("descriptor dimension %d outside 1..%d" % (D, MAX_D))
    mask = _batched(mask, "mask", 3, device=res.device)
    if tuple(mask.shape) != (n, H, W):
        raise RuntimeError("mask must have shape %s (got %s)" % ((n, H, W), tuple(mask.shape)))
    if mask.dtype == torch.bool:
        mask = mask.view(torch.uint8)
    if mask.dtype not in (torch.float32, torch.uint8):
        raise RuntimeError("mask must be float32, uint8 or bool (got %s)" % mask.dtype)
    mask = mask.contiguous()
    dev = res.device
    stats = torch.empty(n, len(STAT_KEYS), D, dtype=torch.float32, device=dev)
    count = torch.empty(n, dtype=torch.int64, device=dev)
    nb = N.lib.ddn_descriptor_statistics_scratch_bytes(n, H, W, D)
    if nb == 0:
        raise N.DdnError(N.lib.ddn_last_error().decode())
    scratch = torch.empty(nb, dtype=torch.uint8, device=dev)
    strides = np.array(res.stride(), dtype=np.int64)
    N.check(N.lib.ddn_descriptor_statistics(N.ptr(res), strides.ctypes.data_as(ctypes.c_void_p), n, H, W, D, N.ptr(mask),
                                            0 if mask.dtype == torch.float32 else 1, N.ptr(stats), N.ptr(count), N.ptr(scratch),
                                            nb, N.stream_ptr()))
    out = {k: stats[:, i] for i, k in enumerate(STAT_KEYS)}
    out['mask_count'] = count
    return out


def fold_descriptor_statistics(per_image, num_images=None):
    """update_stats and the final loop of compute_descriptor_statistics_on_dataset (evaluation.py:2237-2292) over
    per-image statistics ({key: [N,D]} and 'mask_count' [N], as descriptor_statistics returns them; tensors or arrays).

    Reference quirks kept: an image whose mask is empty is skipped for both keys (:2279-2282); the mean is the float32 sum
    of the kept images' means times 1/num_images (num_images defaults to N, the images asked for, even when some were
    skipped; :2290); if every image was skipped the reference fails with a TypeError (None * float), and so does this.
    -> {'entire_image': {'mean', 'max', 'min': [D] lists}, 'mask_image': {...}}, the schema of descriptor_statistics.yaml."""
    host = {k: (v.cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)) for k, v in per_image.items()}
    n = host['mask_count'].shape[0]
    num_images = n if num_images is None else int(num_images)
    stats = {'entire_image': {'mean': None, 'max': None, 'min': None}, 'mask_image': {'mean': None, 'max': None, 'min': None}}
    for i in range(n):
        if host['mask_count'][i] == 0:
            continue
        for key, prefix in (('entire_image', ''), ('mask_image', 'mask_')):
            d = stats[key]
            mn, mx, mean = (np.asarray(host[prefix + s][i], dtype=np.float32) for s in ('min', 'max', 'mean'))
            # torch.min / torch.max of two tensors, like np.minimum / np.maximum, propagate NaN
            d['min'] = mn.copy() if d['min'] is None else np.minimum(d['min'], mn)
            d['max'] = mx.copy() if d['max'] is None else np.maximum(d['max'], mx)
            d['mean'] = mean.copy() if d['mean'] is None else d['mean'] + mean          # float32 += float32
    for key, val in stats.items():
        if val['mean'] is None:
            raise TypeError("every mask was empty: compute_descriptor_statistics_on_dataset fails here too "
                            "(1.0/num_images * None, evaluation.py:2290)")
        val['mean'] = np.float32(1.0 / num_images) * val['mean']       # a float32 tensor times a Python float
        for field in val:
            val[field] = [float(x) for x in val[field]]
    return stats


def descriptor_statistics_over_images(dcn, rgbs, masks):
    """The dataset-free body of compute_descriptor_statistics_on_dataset (evaluation.py:2157-2305): the eval-mode forward
    of every image, ONE statistics launch over all of them, and the reference's fold.

    Each image is forwarded on its own, as the reference's forward_single_image_tensor does (net.py:265-299): with
    normalize=True the network divides by a norm that only broadcasts per image for a batch of one (net.py:256-259), so
    a batched forward would normalise the wrong images.  Everything runs on the device that holds dcn's parameters.

    rgbs   [N,3,H,W] normalised image tensor, or a sequence of [3,H,W] ones (dataset.rgb_image_to_tensor's output)
    masks  [N,H,W] (or a sequence of [H,W]) masks, 1 on the object; tensors or arrays
    -> the reference's {'entire_image': {...}, 'mask_image': {...}} dict of lists (fold_descriptor_statistics)."""
    imgs = rgbs if isinstance(rgbs, torch.Tensor) else torch.stack([torch.as_tensor(x) for x in rgbs])
    if isinstance(masks, torch.Tensor):
        mk = masks
    else:
        mk = torch.stack([m if isinstance(m, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(m)) for m in masks])
    n = imgs.shape[0]
    if imgs.dim() != 4 or imgs.shape[1] != 3 or mk.dim() != 3 or mk.shape[0] != n:
        raise ValueError("rgbs must be [N,3,H,W] and masks [N,H,W] (got %s and %s)" % (tuple(imgs.shape), tuple(mk.shape)))
    if mk.dtype not in (torch.float32, torch.uint8, torch.bool):
        mk = mk.to(torch.float32)
    dev = next(dcn.parameters()).device
    if dev.type != "cuda":
        raise RuntimeError("dcn must be on a CUDA device: this path has no CPU fallback")
    dcn.eval()
    H, W = imgs.shape[2], imgs.shape[3]
    with torch.cuda.device(dev), torch.no_grad():
        res = torch.empty(n, dcn.descriptor_dimension, H, W, dtype=torch.float32, device=dev)
        for i in range(n):
            x = imgs[i:i + 1].detach().to(device=dev, dtype=torch.float32).contiguous()
            res[i:i + 1] = dcn.forward(x)
        per_image = descriptor_statistics(res.permute(0, 2, 3, 1), mk.to(dev))
    return fold_descriptor_statistics(per_image, n)


def save_descriptor_statistics(stats, filename):
    """utils.saveToYaml (dense_correspondence_manipulation/utils/utils.py:29-44), as compute_descriptor_statistics_on_dataset
    writes descriptor_statistics.yaml into the network's parameter folder."""
    import yaml
    with open(filename, 'w') as outfile:
        yaml.dump(stats, outfile, default_flow_style=False)


# ---------------------------------------------------------------------------------------------------------------------
# Across-object analysis (evaluate_network_across_objects, evaluation.py:305-338, 784-858, 977-1004)

class DCNEvaluationPandaTemplateAcrossObject(PandaDataFrameWrapper):
    """evaluation.py:66-76."""
    columns = ['scene_name_a', 'scene_name_b', 'img_a_idx', 'img_b_idx', 'object_id_a', 'object_id_b',
               'norm_diff_descriptor_best_match']

    def __init__(self):
        PandaDataFrameWrapper.__init__(self, DCNEvaluationPandaTemplateAcrossObject.columns)


def best_match_batch(res_a, res_b, uv_a, pair):
    """find_best_match (net.py:488-525) for Q query pixels over N image pairs in one launch (csrc/match_stats.cu).

    res_a, res_b  [N,H,W,D] (or [H,W,D]) float32 CUDA, any strides; uv_a [Q,2] int64 CUDA (u, v) pixels of image A;
    pair [Q] int64 CUDA, the image pair of each query (keeping one pair's queries together is fastest).
    -> (best_uv [Q,2] int64, best_diff [Q] float32, bad_queries [1] int64) CUDA tensors, no host synchronisation.
    best_diff is find_best_match's best_match_diff bit for bit (numpy's float32 arithmetic on a contiguous array); ties go
    to the first pixel in row-major order.  Queries out of range get (-1, -1), NaN and are counted in bad_queries."""
    if not isinstance(res_a, torch.Tensor) or not isinstance(res_b, torch.Tensor):
        raise RuntimeError("res_a and res_b must be CUDA tensors")
    N.require_cuda_f32(res_a, "res_a", contiguous=False); N.require_cuda_f32(res_b, "res_b", contiguous=False)
    res_a = _batched(res_a, "res_a", 4); res_b = _batched(res_b, "res_b", 4, device=res_a.device)
    dev = res_a.device
    n, H, W, D = res_b.shape
    if tuple(res_a.shape) != (n, H, W, D):
        raise RuntimeError("res_a %s and res_b %s must have the same shape" % (tuple(res_a.shape), tuple(res_b.shape)))
    if not 1 <= D <= MAX_D:
        raise RuntimeError("descriptor dimension %d outside 1..%d" % (D, MAX_D))
    uv_a = _index(uv_a, "uv_a", (2,), dev); pair = _index(pair, "pair", (), dev)
    Q = uv_a.shape[0]
    if pair.shape[0] != Q:
        raise RuntimeError("uv_a and pair must have the same length")
    uv = torch.empty(Q, 2, dtype=torch.int64, device=dev)
    diff = torch.empty(Q, dtype=torch.float32, device=dev)
    bad = torch.empty(1, dtype=torch.int64, device=dev)
    nb = N.lib.ddn_best_match_batch_scratch_bytes(Q)
    if nb == 0:
        raise N.DdnError(N.lib.ddn_last_error().decode())
    scratch = torch.empty(nb, dtype=torch.uint8, device=dev)
    hp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    sa = np.array(res_a.stride(), dtype=np.int64); sb = np.array(res_b.stride(), dtype=np.int64)
    N.check(N.lib.ddn_best_match_batch(N.ptr(res_a), hp(sa), N.ptr(res_b), hp(sb), n, H, W, D, N.ptr(pair), N.ptr(uv_a), Q,
                                       N.ptr(uv), N.ptr(diff), N.ptr(bad), N.ptr(scratch), nb, N.stream_ptr()))
    return uv, diff, bad


def across_object_analysis(res_a, res_b, mask_a, pair=None, num_uv_a_samples=100, generator=None):
    """single_across_object_image_pair_quantitative_analysis (evaluation.py:784-858) for a batch of N image pairs, from
    descriptor images the device already holds: ``num_uv_a_samples`` pixels are drawn from each mask_a on the device (the
    route quantitative_analysis_on_pair takes) and every one's best match in res_b is found in ONE launch.

    res_a, res_b  [N,H,W,D] (or [H,W,D]) float32 CUDA descriptor images of object A and object B, any strides
    mask_a        [N,H,W] (or [H,W]) masks of object A, 1 on the object
    pair          None, or N dicts holding the template's other columns (scene_name_a, scene_name_b, img_a_idx,
                  img_b_idx, object_id_a, object_id_b); a missing key leaves its column NaN
    generator     a CUDA torch.Generator or None
    -> dict of host numpy arrays, one row per sample: the columns of DCNEvaluationPandaTemplateAcrossObject,
    "uv_a" / "uv_b" [R,2] (u, v) and "pair" [R].  A pair with an empty mask_a gives no rows (the reference returns an empty
    list).  The reference draws with random.sample (without replacement, and it raises when the mask has fewer than
    num_uv_a_samples pixels); this draws uniformly with replacement, so the sampled pixels differ, each row's value for
    its uv_a does not."""
    from . import sampling
    if not isinstance(res_a, torch.Tensor) or not res_a.is_cuda:
        raise RuntimeError("res_a must be a CUDA tensor: this path has no CPU fallback")
    ra = _batched(res_a, "res_a", 4)
    n, H, W, _ = ra.shape
    dev = ra.device
    ma = mask_a if isinstance(mask_a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(mask_a))
    ma = _batched(ma.to(dev), "mask_a", 3).to(torch.float32).contiguous()
    if tuple(ma.shape) != (n, H, W):
        raise RuntimeError("mask_a must have shape %s (got %s)" % ((n, H, W), tuple(ma.shape)))
    if pair is not None and len(pair) != n:
        raise ValueError("pair must hold one dict per image pair (%d, got %d)" % (n, len(pair)))
    k = int(num_uv_a_samples)
    counts = torch.count_nonzero(ma.view(n, -1), dim=1).cpu().numpy()
    keep = [i for i in range(n) if counts[i] > 0]
    cols = {c: np.array([], dtype=object if c != 'norm_diff_descriptor_best_match' else np.float32)
            for c in DCNEvaluationPandaTemplateAcrossObject.columns}
    if not keep or k <= 0:
        cols.update(uv_a=np.zeros((0, 2), np.int64), uv_b=np.zeros((0, 2), np.int64), pair=np.zeros(0, np.int64))
        return cols
    dummy = torch.zeros(1, dtype=torch.int64, device=dev)
    flat = torch.cat([sampling.sample_non_matches(dummy, ma[i], (H, W), k, generator=generator)[1] for i in keep])
    pidx = torch.tensor(keep, dtype=torch.int64, device=dev).repeat_interleave(k)
    uv_a = torch.stack([flat % W, flat // W], 1)
    uv_b, diff, _ = best_match_batch(ra, res_b, uv_a, pidx)
    rows = pidx.cpu().numpy()
    out = {'norm_diff_descriptor_best_match': diff.cpu().numpy(), 'uv_a': uv_a.cpu().numpy(), 'uv_b': uv_b.cpu().numpy(),
           'pair': rows}
    for c in DCNEvaluationPandaTemplateAcrossObject.columns[:-1]:
        out[c] = np.array([(pair[i].get(c, np.nan) if pair is not None else np.nan) for i in rows], dtype=object)
    return out
