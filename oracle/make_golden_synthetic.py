"""Writes tests/golden/synthetic_multi_object_batch.npz: what the EXECUTED reference's
get_synthetic_multi_object_within_scene_data path computes for a set of pairs with scripted random numbers.

TEST INFRASTRUCTURE (needs PDC_REFERENCE_ROOT; see oracle/build_ref_augment.py).  Both scenes are the 32 x 48 crop of
oracle/ref_cases.reprojection_scene() that oracle/make_golden_within_scene.py uses, seen from the same two views, each
with its own colours and masks (both halves share K, as the reference's scenes do).  CASES covers both foreground
choices in each merge, pruning that removes some matches and all of them (an occlusion return after merge 1 and after
merge 2), masks holding 255 and 2 (the wrapping merged mask 2), empty mask_a1 and mask_b1,
sample_matches_only_off_mask = False and use_image_b_mask_inv = False.

    PDC_REFERENCE_ROOT=... python oracle/make_golden_synthetic.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import make_golden_within_scene as MW  # noqa: E402
from oracle import synthetic_multi_object_oracle as SO  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "synthetic_multi_object_batch.npz")
H, W = MW.H, MW.W
CFG = dict(n_attempts=200, k_masked=3, k_background=2, sample_matches_only_off_mask=True, domain_randomize=False,
           use_image_b_mask_inv=True)
# (name, merge decisions (1 = scene B in the foreground), mask kind, cfg overrides)
CASES = [
    ("fg_b_fg_b", (1, 1), "object", {}),
    ("fg_a_fg_b", (0, 1), "object", {}),
    ("fg_b_fg_a", (1, 0), "object", {}),
    ("fg_a_fg_a_mask_255_wrap", (0, 0), "values", {}),
    ("occluded_after_merge_1", (1, 0), "full_b1", {}),
    ("occluded_after_merge_2", (0, 0), "full_a2", {}),
    ("empty_mask_a1", (1, 1), "empty_a1", {}),
    ("empty_mask_b1", (0, 1), "empty_b1", {}),
    ("off_mask_false", (1, 0), "object", {"sample_matches_only_off_mask": False}),
    ("mask_inv_false", (0, 1), "object", {"use_image_b_mask_inv": False}),
]


def case_inputs(i):
    """-> scene_a, scene_b (dicts), K, cfg and random numbers of case i (seeded, numpy)."""
    name, merge, kind, over = CASES[i]
    cfg = dict(CFG); cfg.update(over)
    g = np.random.RandomState(500 + i)
    da, pa, db, pb, K = MW.scene()
    rgb = lambda: g.randint(0, 256, (H, W, 3)).astype(np.uint8)
    rect = lambda y0, y1, x0, x1: (lambda m: (m.__setitem__((slice(y0, y1), slice(x0, x1)), 1), m)[1])(np.zeros((H, W), np.uint8))
    A = dict(rgb_1=rgb(), rgb_2=rgb(), depth_1=da, depth_2=db, mask_1=rect(4, 28, 6, 40), mask_2=rect(8, 30, 3, 35),
             pose_1=pa, pose_2=pb)
    # scene B: the same views, with other colours and objects
    B = dict(rgb_1=rgb(), rgb_2=rgb(), depth_1=da, depth_2=db, mask_1=rect(0, 14, 20, 48), mask_2=rect(16, 32, 0, 24),
             pose_1=pa, pose_2=pb)
    if kind == "values":
        A["mask_2"][8:30, 3:35] = 255; B["mask_2"][20:24, 10:30] = 2; A["mask_1"][5, 7] = 255
    elif kind == "full_b1":
        B["mask_1"][:] = 1
    elif kind == "full_a2":
        A["mask_2"][:] = 1
    elif kind == "empty_a1":
        A["mask_1"][:] = 0
    elif kind == "empty_b1":
        B["mask_1"][:] = 0
    n = cfg["n_attempts"]
    u = lambda *shape: g.random_sample(shape).astype(np.float32)
    rand = dict(merge=np.asarray(merge, np.uint8), cand_u=u(2, n), cand_v=u(2, n), masked_u=u(2 * n * cfg["k_masked"]),
                masked_v=u(2 * n * cfg["k_masked"]), background_u=u(2 * n * cfg["k_background"]),
                background_v=u(2 * n * cfg["k_background"]))
    return A, B, K, cfg, rand


def run_case(fns, i, uv=None):
    A, B, K, cfg, rand = case_inputs(i)
    return SO.get_synthetic_data(fns, A, B, K, cfg, rand, uv=uv)


KEYS = ("rgb_a", "rgb_b", "matches_a", "matches_b", "masked_a", "masked_b", "background_a", "background_b")


def main():
    from oracle import build_ref_augment
    fns = SO.executed_reference(build_ref_augment.load())
    out = {}
    for i, (name, _, _, _) in enumerate(CASES):
        r = run_case(fns, i)
        assert r["empty"] or (r["python_left"] == 0 and r["torch_left"] == 0), (name, r)
        out["%s/empty" % name] = np.array(r["empty"])
        out["%s/ret" % name] = np.array(r["ret"])
        for k in KEYS:
            out["%s/%s" % (name, k)] = r[k].astype(np.uint8 if k.startswith("rgb") else np.int32)
        print("%-28s ret=%-10s matches=%d masked=%d background=%d" % (
            name, r["ret"], len(r["matches_a"]), len(r["masked_a"]), len(r["background_a"])))
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
