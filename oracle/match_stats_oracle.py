"""Float64 / numpy restatement of the per-match evaluation statistics, for many queries at once.

TEST INFRASTRUCTURE.  Restates DenseCorrespondenceEvaluation.compute_descriptor_match_statistics
(dense_correspondence/evaluation/evaluation.py:1006-1178) with find_best_match (network/dense_correspondence_network.py:488-525),
compute_3d_position (evaluation.py:1180-1200) and pinhole_projection_image_to_world (correspondence_finder.py:123-144), with
the same numpy expressions, so that on the fixture cases it is bit-equal to the executed reference (tests/golden/
match_statistics.npz, oracle/make_golden_eval.py).  Two differences are selectable:
  threshold="reference"  norm_diff_descriptor_ground_truth = np.linalg.norm(des_a - des_b)   (evaluation.py:1070)
  threshold="device"     ... = nd(uv_b), the distance map's own value (what csrc/match_stats.cu computes)
and res_a / res_b are made contiguous first: the reference's descriptor images reached numpy through PyTorch 1.1's .cpu(),
which returned a contiguous copy, so its np.sum(..., axis=2) ran numpy's pairwise order over the descriptor axis.
"""
import numpy as np

DEPTH_IM_SCALE = 1000.0
F32 = ("norm_diff_descriptor_ground_truth", "norm_diff_descriptor")
F64 = ("norm_diff_descriptor_masked", "norm_diff_ground_truth_3d", "norm_diff_pred_3d", "norm_diff_pred_3d_masked",
       "pixel_match_error_l2", "pixel_match_error_l2_masked", "pixel_match_error_l1", "fraction_pixels_closer_than_ground_truth",
       "fraction_pixels_closer_than_ground_truth_masked", "average_l2_distance_for_false_positives",
       "average_l2_distance_for_false_positives_masked")
INTS = ("u_pred", "v_pred", "u_pred_masked", "v_pred_masked", "num_pixels_closer_than_ground_truth",
        "num_pixels_closer_than_ground_truth_masked", "num_pixels_in_masked_image")
BOOLS = ("is_valid", "is_valid_masked")


def pairwise_sum_last_axis(a):
    """numpy's float32 pairwise summation of a contiguous last axis of length D <= 128, restated with elementwise float32
    adds: D < 8 a sequential sum from 0; otherwise 8 running partials r[j] += a[i+j], ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)),
    then the remaining D % 8 elements in sequence."""
    a = np.asarray(a, dtype=np.float32)
    D = a.shape[-1]
    if D < 8:
        s = np.zeros(a.shape[:-1], np.float32)
        for i in range(D):
            s = s + a[..., i]
        return s
    r = [a[..., j].copy() for j in range(8)]
    full = D - D % 8
    for i in range(8, full, 8):
        for j in range(8):
            r[j] = r[j] + a[..., i + j]
    s = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
    for i in range(full, D):
        s = s + a[..., i]
    return s


def is_depth_valid(depth):
    return ((depth > 0) and (depth < 10.0))


def compute_3d_position(uv, depth, K, camera_to_world):
    u_v_1 = np.array([uv[0], uv[1], 1])
    pos = depth * np.linalg.inv(K).dot(u_v_1)
    return np.dot(camera_to_world, np.append(pos, 1))[:3]


def one_match(depth_a, depth_b, mask_b, uv_a, uv_b, pose_a, pose_b, res_a, res_b, K, threshold="reference", empty_mask_nan=False):
    """One query, the reference's statements in order.  -> dict.  An empty mask_b raises ZeroDivisionError as the reference
    does, or gives a NaN masked fraction with empty_mask_nan=True."""
    res_a = np.ascontiguousarray(res_a); res_b = np.ascontiguousarray(res_b)
    # the dataset's types: a uint8 mask (so the masked map is float64) and integer depths (float64 after / DEPTH_IM_SCALE)
    mask_b = np.asarray(mask_b).astype(np.uint8)
    depth_a = np.asarray(depth_a, dtype=np.float64); depth_b = np.asarray(depth_b, dtype=np.float64)
    d = res_a[uv_a[1], uv_a[0]]
    norm_diffs = np.sqrt(np.sum(np.square(res_b - d), axis=2))
    idx = np.unravel_index(np.argmin(norm_diffs), norm_diffs.shape)
    uv_p = (idx[1], idx[0])
    masked = norm_diffs + (1 - mask_b) * 1e6
    idx_m = np.unravel_index(np.argmin(masked), masked.shape)
    uv_pm = (idx_m[1], idx_m[0])
    o = {"norm_diff_descriptor": norm_diffs[idx], "norm_diff_descriptor_masked": masked[idx_m],
         "u_pred": uv_p[0], "v_pred": uv_p[1], "u_pred_masked": uv_pm[0], "v_pred_masked": uv_pm[1]}
    o["pixel_match_error_l2"] = np.linalg.norm((np.array(uv_b) - np.array(uv_p)), ord=2)
    o["pixel_match_error_l2_masked"] = np.linalg.norm((np.array(uv_b) - np.array(uv_pm)), ord=2)
    o["pixel_match_error_l1"] = np.linalg.norm((np.array(uv_b) - np.array(uv_p)), ord=1)
    if threshold == "reference":
        t = np.linalg.norm(d - res_b[uv_b[1], uv_b[0], :])
    else:
        t = norm_diffs[uv_b[1], uv_b[0]]
    o["norm_diff_descriptor_ground_truth"] = t
    v_i, u_i = np.where(norm_diffs < t)
    v_m, u_m = np.where(masked < t)
    o["num_pixels_closer_than_ground_truth"] = len(u_i)
    o["num_pixels_closer_than_ground_truth_masked"] = len(u_m)
    o["num_pixels_in_masked_image"] = len(np.nonzero(mask_b)[0])
    o["fraction_pixels_closer_than_ground_truth"] = len(u_i) * 1.0 / (res_a.shape[0] * res_a.shape[1])
    if empty_mask_nan and o["num_pixels_in_masked_image"] == 0:
        o["fraction_pixels_closer_than_ground_truth_masked"] = np.nan
    else:
        o["fraction_pixels_closer_than_ground_truth_masked"] = len(u_m) * 1.0 / o["num_pixels_in_masked_image"]
    o["average_l2_distance_for_false_positives"] = 0.0 if len(u_i) == 0 else \
        np.average(np.sqrt((u_i - uv_b[0]) ** 2 + (v_i - uv_b[1]) ** 2))
    o["average_l2_distance_for_false_positives_masked"] = 0.0 if len(u_m) == 0 else \
        np.average(np.sqrt((u_m - uv_b[0]) ** 2 + (v_m - uv_b[1]) ** 2))
    za = depth_a[uv_a[1], uv_a[0]] / DEPTH_IM_SCALE
    zb = depth_b[uv_b[1], uv_b[0]] / DEPTH_IM_SCALE
    zp = depth_b[uv_p[1], uv_p[0]] / DEPTH_IM_SCALE
    zpm = depth_b[uv_pm[1], uv_pm[0]] / DEPTH_IM_SCALE
    pa = compute_3d_position(uv_a, za, K, pose_a)
    pb = compute_3d_position(uv_b, zb, K, pose_b)
    pp = compute_3d_position(uv_p, zp, K, pose_b)
    ppm = compute_3d_position(uv_pm, zpm, K, pose_b)
    o["is_valid"] = is_depth_valid(zp)
    o["is_valid_masked"] = is_depth_valid(zpm)
    o["norm_diff_ground_truth_3d"] = np.linalg.norm(pb - pa) if is_depth_valid(zb) else np.nan
    o["norm_diff_pred_3d"] = np.linalg.norm(pb - pp) if (is_depth_valid(zb) and o["is_valid"]) else np.nan
    o["norm_diff_pred_3d_masked"] = np.linalg.norm(pb - ppm) if (is_depth_valid(zb) and o["is_valid_masked"]) else np.nan
    return o


def match_statistics(res_a, res_b, uv_a, uv_b, pair, mask_b, depth_a, depth_b, poses_a, poses_b, K, threshold="device"):
    """Batched: res_* [N,H,W,D], uv_* [Q,2], pair [Q], mask_b / depth_* [N,H,W], poses_* [N,4,4].  An empty mask gives a NaN
    masked fraction (the batched convention).  -> {column: [Q] array} (float32 / float64 / int64 / bool as the reference)."""
    out = {k: [] for k in F32 + F64 + INTS + BOOLS}
    for i in range(len(pair)):
        n = int(pair[i])
        ua = (int(uv_a[i][0]), int(uv_a[i][1])); ub = (int(uv_b[i][0]), int(uv_b[i][1]))
        o = one_match(depth_a[n], depth_b[n], np.asarray(mask_b[n]), ua, ub, poses_a[n], poses_b[n], res_a[n], res_b[n], K,
                      threshold, empty_mask_nan=True)
        for k in out:
            out[k].append(o[k])
    res = {k: np.array(out[k], dtype=np.float32) for k in F32}
    res.update({k: np.array(out[k], dtype=np.float64) for k in F64})
    res.update({k: np.array(out[k], dtype=np.int64) for k in INTS})
    res.update({k: np.array(out[k], dtype=bool) for k in BOOLS})
    return res
