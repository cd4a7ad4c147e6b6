"""Writes tests/golden/within_scene_batch.npz: what the EXECUTED reference's get_within_scene_data path computes for a set
of within-scene pairs with scripted random numbers.

TEST INFRASTRUCTURE (needs PDC_REFERENCE_ROOT; see oracle/build_ref_augment.py).  The scene is a 32 x 48 crop of
oracle/ref_cases.reprojection_scene() (its intrinsics shifted with the crop).  CASES covers background randomisation on
and off, solid and gradient backgrounds, vertical and horizontal gradients, noise on and off, each flip, a mask holding
255 and 2, an empty mask_a (return_empty_data), empty and full mask_b, sample_matches_only_off_mask = False,
use_image_b_mask_inv = False and domain_randomize = False.  The augmented images are stored as uint8 (normalisation is
a per-(channel, value) function, checked on all 256 values in tests/test_within_scene_cpu.py).

    PDC_REFERENCE_ROOT=... python oracle/make_golden_within_scene.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_cases  # noqa: E402
from oracle import within_scene_oracle as WO  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "within_scene_batch.npz")
Y0, X0, H, W = 40, 50, 32, 48
CFG = dict(n_attempts=200, k_masked=3, k_background=2, sample_matches_only_off_mask=True, domain_randomize=True,
           use_image_b_mask_inv=True)
# (name, decisions of A and B: (randomise, gradient, vertical, noise, flip), mask kind, cfg overrides)
CASES = [
    ("solid_flip_b", ((1, 0, 0, 0, 0), (1, 0, 0, 0, 1)), "object", {}),
    ("gradient_vertical_noise_flip_a", ((1, 1, 1, 1, 1), (1, 1, 1, 0, 0)), "object", {}),
    ("gradient_horizontal_noise_flip_both", ((1, 1, 0, 1, 1), (1, 1, 0, 1, 1)), "object", {}),
    ("no_randomise_a_mask_255", ((0, 1, 1, 1, 0), (1, 1, 0, 0, 1)), "values", {}),
    ("solid_noise", ((1, 0, 1, 1, 0), (1, 0, 0, 1, 0)), "object", {}),
    ("empty_mask_a", ((1, 1, 1, 1, 1), (1, 1, 1, 1, 1)), "empty_a", {}),
    ("empty_mask_b", ((1, 1, 0, 1, 1), (1, 0, 0, 1, 0)), "empty_b", {}),
    ("full_mask_b", ((1, 0, 0, 1, 1), (1, 1, 1, 1, 1)), "full_b", {}),
    ("off_mask_false", ((1, 1, 1, 0, 1), (0, 0, 0, 0, 1)), "object", {"sample_matches_only_off_mask": False}),
    ("mask_inv_false", ((1, 0, 0, 0, 1), (1, 1, 0, 1, 0)), "object", {"use_image_b_mask_inv": False}),
    ("domain_randomize_false", ((1, 1, 1, 1, 1), (1, 1, 1, 1, 1)), "object", {"domain_randomize": False}),
]


def scene():
    da, pa, db, pb, _, _, K, _ = ref_cases.reprojection_scene()
    K = K.copy(); K[0, 2] -= X0; K[1, 2] -= Y0
    crop = lambda d: np.ascontiguousarray(d[Y0:Y0 + H, X0:X0 + W]).astype(np.float32)
    return crop(da), pa, crop(db), pb, K


def case_inputs(i):
    """-> inputs, cfg and random numbers of case i (seeded, numpy)."""
    name, dec, kind, over = CASES[i]
    cfg = dict(CFG); cfg.update(over)
    g = np.random.RandomState(100 + i)
    da, pa, db, pb, K = scene()
    rgb_a = g.randint(0, 256, (H, W, 3)).astype(np.uint8); rgb_b = g.randint(0, 256, (H, W, 3)).astype(np.uint8)
    mask_a = np.zeros((H, W), np.uint8); mask_a[4:28, 6:40] = 1
    mask_b = np.zeros((H, W), np.uint8); mask_b[8:30, 3:35] = 1; mask_b[12:16, 10:20] = 0
    if kind == "values":
        mask_a[10:14, 10:30] = 255; mask_b[20:24, 5:15] = 255; mask_a[5, 7] = 2; mask_b[9, 4] = 2
    elif kind == "empty_a":
        mask_a[:] = 0
    elif kind == "empty_b":
        mask_b[:] = 0
    elif kind == "full_b":
        mask_b[:] = 1
    n, P = cfg["n_attempts"], H * W
    params = np.zeros((2, 16), np.uint8)
    params[:, :5] = np.asarray(dec, np.uint8); params[:, 5:11] = g.randint(0, 255, (2, 6))
    u = lambda m: g.random_sample(m).astype(np.float32)
    rand = dict(params=params, noise=g.randint(0, 50, (2, 2, H, W, 3)).astype(np.uint8), cand_u=u(n), cand_v=u(n),
                masked_u=u(n * cfg["k_masked"]), masked_v=u(n * cfg["k_masked"]),
                background_u=u(n * cfg["k_background"]), background_v=u(n * cfg["k_background"]), blind=u(P))
    return dict(rgb_a=rgb_a, rgb_b=rgb_b, depth_a=da, depth_b=db, mask_a=mask_a, mask_b=mask_b, pose_a=pa, pose_b=pb, K=K), cfg, rand


def run_case(fns, i):
    x, cfg, rand = case_inputs(i)
    return WO.get_within_scene_data(fns, x["rgb_a"], x["rgb_b"], x["depth_a"], x["depth_b"], x["mask_a"], x["mask_b"],
                                    x["pose_a"], x["pose_b"], x["K"], cfg, rand)


KEYS = ("rgb_a", "rgb_b", "matches_a", "matches_b", "masked_a", "masked_b", "background_a", "background_b", "blind_a", "blind_b")


def main():
    from oracle import build_ref_augment
    fns = WO.executed_reference(build_ref_augment.load())
    out = {}
    for i, (name, _, _, _) in enumerate(CASES):
        r = run_case(fns, i)
        assert r["empty"] or (r["python_left"] == 0 and r["numpy_left"] == 0), (name, r)
        out["%s/empty" % name] = np.array(r["empty"])
        for k in KEYS:
            out["%s/%s" % (name, k)] = r[k].astype(np.uint8 if k.startswith("rgb") else np.int32)
        print("%-40s empty=%d matches=%d masked=%d background=%d blind=%d" % (
            name, r["empty"], len(r["matches_a"]), len(r["masked_a"]), len(r["background_a"]), len(r["blind_a"])))
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
