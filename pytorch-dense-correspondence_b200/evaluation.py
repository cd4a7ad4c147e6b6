"""Per-match evaluation statistics on the device (SURVEY.md 8f row 4): the columns that
``DenseCorrespondenceEvaluation.compute_descriptor_match_statistics`` (dense_correspondence/evaluation/evaluation.py:1006-1178)
records for each ground-truth match, for many matches over many image pairs in one launch (csrc/match_stats.cu).

``match_statistics`` is the batched entry point (CUDA tensors in, a dict of CUDA tensors out, no host synchronisation).
``DenseCorrespondenceEvaluation`` keeps the reference's signatures for the per-match call and its helpers, and
``quantitative_analysis_on_pair`` is the dataset-free body of ``single_same_scene_image_pair_quantitative_analysis``
(evaluation.py:862-958).

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
