"""Float64 restatement of the reference's descriptor statistics (compute_descriptor_statistics_on_dataset,
dense_correspondence/evaluation/evaluation.py:2157-2305) and of find_best_match's best match
(dense_correspondence/network/dense_correspondence_network.py:488-525).

per_image(res, mask)  the nested compute_descriptor_statistics (:2177-2219) for one [H,W,D] image in float64 numpy:
                      min / max / mean over every pixel and over the nonzero mask pixels; None for the mask part
                      of an empty mask, as the reference returns (None, None).
fold(images, num_images)  update_stats (:2237-2263) and the final loop (:2289-2292): images whose mask is empty are
                      skipped for both keys, mean = sum of the kept images' means times 1/num_images.
best_match(uv_a, res_a, res_b)  np.argmin of sqrt(sum((res_b - res_a[v, u])^2)) in float32 on a contiguous array.
"""
import numpy as np


def per_image(res, mask):
    """res [H,W,D], mask [H,W] -> ((min, max, mean), (mask_min, mask_max, mask_mean) or None), float64 [D] arrays."""
    flat = np.asarray(res, dtype=np.float64).reshape(-1, res.shape[-1])
    whole = (flat.min(0), flat.max(0), flat.mean(0))
    sel = np.asarray(mask).reshape(-1) != 0
    if not sel.any():
        return whole, None
    m = flat[sel]
    return whole, (m.min(0), m.max(0), m.mean(0))


def fold(images, num_images):
    """images: [(whole, masked)] as per_image returns them -> the reference's dict of lists."""
    stats = {'entire_image': {'mean': None, 'max': None, 'min': None}, 'mask_image': {'mean': None, 'max': None, 'min': None}}
    for whole, masked in images:
        if masked is None:
            continue
        for key, (mn, mx, mean) in (('entire_image', whole), ('mask_image', masked)):
            d = stats[key]
            d['min'] = mn if d['min'] is None else np.minimum(d['min'], mn)
            d['max'] = mx if d['max'] is None else np.maximum(d['max'], mx)
            d['mean'] = mean if d['mean'] is None else d['mean'] + mean
    for val in stats.values():
        val['mean'] = 1.0 / num_images * val['mean']
        for field in val:
            val[field] = [float(x) for x in val[field]]
    return stats


def best_match(uv_a, res_a, res_b):
    """-> ((u, v), distance as float32) of find_best_match on contiguous float32 arrays."""
    d = np.ascontiguousarray(res_a, dtype=np.float32)[uv_a[1], uv_a[0]]
    nd = np.sqrt(np.sum(np.square(np.ascontiguousarray(res_b, dtype=np.float32) - d), axis=2))
    i = int(np.argmin(nd))
    v, u = np.unravel_index(i, nd.shape)
    return (int(u), int(v)), nd[v, u]
