"""Writes tests/golden/match_statistics.npz: inputs and the EXECUTED reference's per-match evaluation statistics.

TEST INFRASTRUCTURE (needs the reference: PDC_REFERENCE_ROOT, oracle/build_ref_eval.py).  The scene is a 64x96 crop of the ray-cast
plane of oracle/ref_cases.reprojection_scene (principal point moved with the crop), with a depth hole in each image and the
occluder of view B.  Descriptors are small integers ("exact grid"), so every square and every sum is exact in float32 and
numpy's pairwise sum, a sequential sum and the BLAS dot of np.linalg.norm all agree.  Two descriptor sets: D = 3 (sequential
order) and D = 9 (pairwise order).  Three masks per set (pairs 0, 1, 2 of the batch): the object mask, a full mask and an
empty one (the reference raises ZeroDivisionError there, which is recorded).  The queries include a ground truth outside
the mask, an invalid depth at uv_b and at the prediction, uv_b on the last row and column after clipping, and tied minima.

    PDC_REFERENCE_ROOT=<reference checkout> python oracle/make_golden_eval.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import build_ref, build_ref_eval, ref_cases  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "match_statistics.npz")
H, W = 64, 96
R0, C0 = 40, 50          # crop origin in the 120x160 scene
COLUMNS = ("is_valid", "is_valid_masked", "norm_diff_descriptor_ground_truth", "norm_diff_descriptor",
           "norm_diff_descriptor_masked", "norm_diff_ground_truth_3d", "norm_diff_pred_3d", "norm_diff_pred_3d_masked",
           "pixel_match_error_l2", "pixel_match_error_l2_masked", "pixel_match_error_l1", "fraction_pixels_closer_than_ground_truth",
           "fraction_pixels_closer_than_ground_truth_masked", "average_l2_distance_for_false_positives",
           "average_l2_distance_for_false_positives_masked")


def inputs():
    """-> dict of the fixture's inputs (descriptors as int8, depths uint16, masks uint8)."""
    da, pa, db, pb, mask, _, K, _ = ref_cases.reprojection_scene()
    da = da[R0:R0 + H, C0:C0 + W].copy(); db = db[R0:R0 + H, C0:C0 + W].copy()
    da[5:12, 70:80] = 0                          # a hole in A (uv_a depth is never checked)
    db[50:60, 0:10] = 0                          # a hole in B: invalid depth at uv_b / at the prediction
    Kc = K.copy(); Kc[0, 2] -= C0; Kc[1, 2] -= R0
    masks = np.zeros((3, H, W), np.uint8)
    masks[0, 8:56, 12:84] = 1                    # the object
    masks[1] = 1                                 # full
    rng = np.random.default_rng(2024)
    out = dict(K=Kc, pose_a=pa, pose_b=pb, depth_a=da, depth_b=db, mask_b=masks)
    for D, lim in ((3, 3), (9, 1)):
        ra = rng.integers(-lim, lim + 1, size=(H, W, D)).astype(np.int8)
        rb = rng.integers(-lim, lim + 1, size=(H, W, D)).astype(np.int8)
        nq = 24
        uv_a = np.stack([rng.integers(0, W, nq), rng.integers(0, H, nq)], 1)
        uv_b_raw = np.stack([rng.integers(0, W, nq) + rng.uniform(-0.45, 0.45, nq),
                             rng.integers(0, H, nq) + rng.uniform(-0.45, 0.45, nq)], 1)
        uv_b_raw[0] = (W - 0.4, H - 0.3)         # rounds past the last column / row: clipped to (W-1, H-1)
        uv_b_raw[1] = (4.2, 54.1)                # inside B's hole: invalid depth at uv_b
        uv_b_raw[2] = (90.0, 2.0)                # outside the object mask
        # query 3: its descriptor also at (3, 52) (in B's hole, the first pixel with nd = 0) -> invalid depth at the prediction
        rb[52, 3] = ra[uv_a[3][1], uv_a[3][0]]
        # query 4: its descriptor at two pixels in row 20 (and perhaps elsewhere): tied minima, the first one wins
        rb[20, 30] = rb[20, 60] = ra[uv_a[4][1], uv_a[4][0]]
        out["res_a_d%d" % D] = ra; out["res_b_d%d" % D] = rb
        out["uv_a_d%d" % D] = uv_a; out["uv_b_raw_d%d" % D] = uv_b_raw
    return out


def run_reference(inp):
    ev = build_ref_eval.load()
    DCE = ev.DenseCorrespondenceEvaluation
    res = {}
    for D in (3, 9):
        ra = inp["res_a_d%d" % D].astype(np.float32); rb = inp["res_b_d%d" % D].astype(np.float32)
        uv_b = np.array([DCE.clip_pixel_to_image_size_and_round(tuple(x), W, H) for x in inp["uv_b_raw_d%d" % D]])
        res["uv_b_d%d" % D] = uv_b
        for n in range(3):
            cols = {c: [] for c in COLUMNS}
            raised = []
            for i in range(len(uv_b)):
                ua = (int(inp["uv_a_d%d" % D][i][0]), int(inp["uv_a_d%d" % D][i][1])); ub = (int(uv_b[i][0]), int(uv_b[i][1]))
                try:
                    t = DCE.compute_descriptor_match_statistics(inp["depth_a"], inp["depth_b"], None, inp["mask_b"][n], ua, ub,
                                                                inp["pose_a"], inp["pose_b"], ra, rb, inp["K"])
                    df = t.dataframe
                    for c in COLUMNS:
                        cols[c].append(df[c].values[0])
                    raised.append("")
                except ZeroDivisionError as e:
                    raised.append(type(e).__name__)
                    for c in COLUMNS:
                        cols[c].append(np.nan)
            for c in COLUMNS:
                res["out_d%d_p%d/%s" % (D, n, c)] = np.array(cols[c], dtype=np.float32 if c in COLUMNS[2:4] else np.float64)
            res["out_d%d_p%d/raised" % (D, n)] = np.array(raised)
    return res


def main():
    if not build_ref.reference_available():
        raise SystemExit("set PDC_REFERENCE_ROOT to a checkout of the reference")
    build_ref_eval.build()
    inp = inputs()
    out = dict(inp)
    out.update(run_reference(inp))
    np.savez_compressed(OUT, **out)
    print("wrote %s (%.1f KB)" % (OUT, os.path.getsize(OUT) / 1024.0))


if __name__ == "__main__":
    main()
