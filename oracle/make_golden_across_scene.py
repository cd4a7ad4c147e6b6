"""Writes tests/golden/across_scene_batch.npz: what the EXECUTED reference's get_across_scene_data path computes for a set
of across-scene pairs with scripted random numbers.

TEST INFRASTRUCTURE (needs PDC_REFERENCE_ROOT; see oracle/build_ref_augment.py).  The images are 32 x 48 of seeded uniform
random RGB with rectangular masks: this path reads no depth or pose, so no scene geometry is involved.
CASES covers background randomisation on and off, solid and gradient backgrounds, vertical and horizontal gradients,
noise on and off, each flip and both, a mask holding 255 and 2, an empty mask_a, an empty mask_b, both empty (each the
return_empty_data), a single-pixel mask and domain_randomize = False with and without flips.  The augmented images are
stored as uint8 (normalisation is a per-(channel, value) function, checked on all 256 values in
tests/test_within_scene_cpu.py).

    PDC_REFERENCE_ROOT=... python oracle/make_golden_across_scene.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import across_scene_oracle as AO  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "across_scene_batch.npz")
H, W = 32, 48
CFG = dict(num_samples=500, domain_randomize=True)
# (name, decisions of A and B: (randomise, gradient, vertical, noise, flip), mask kind, cfg overrides)
CASES = [
    ("solid_flip_b", ((1, 0, 0, 0, 0), (1, 0, 0, 0, 1)), "object", {}),
    ("gradient_vertical_noise_flip_a", ((1, 1, 1, 1, 1), (1, 1, 1, 0, 0)), "object", {}),
    ("gradient_horizontal_noise_flip_both", ((1, 1, 0, 1, 1), (1, 1, 0, 1, 1)), "object", {}),
    ("no_randomise_a_mask_255", ((0, 1, 1, 1, 0), (1, 1, 0, 0, 1)), "values", {}),
    ("solid_noise_no_flip", ((1, 0, 1, 1, 0), (1, 0, 0, 1, 0)), "object", {}),
    ("single_pixel_masks", ((1, 1, 0, 0, 1), (1, 0, 0, 1, 1)), "single", {}),
    ("empty_mask_a", ((1, 1, 1, 1, 1), (1, 1, 1, 1, 1)), "empty_a", {}),
    ("empty_mask_b", ((1, 1, 0, 1, 1), (1, 0, 0, 1, 0)), "empty_b", {}),
    ("empty_both", ((1, 0, 0, 1, 1), (1, 1, 1, 1, 1)), "empty_both", {}),
    ("domain_randomize_false_flip_both", ((1, 1, 1, 1, 1), (1, 1, 1, 1, 1)), "object", {"domain_randomize": False}),
    ("domain_randomize_false_no_flip", ((1, 1, 1, 1, 0), (1, 1, 1, 1, 0)), "values", {"domain_randomize": False}),
]


def case_inputs(i):
    """-> inputs, cfg and random numbers of case i (seeded, numpy)."""
    name, dec, kind, over = CASES[i]
    cfg = dict(CFG); cfg.update(over)
    g = np.random.RandomState(300 + i)
    rgb_a = g.randint(0, 256, (H, W, 3)).astype(np.uint8); rgb_b = g.randint(0, 256, (H, W, 3)).astype(np.uint8)
    mask_a = np.zeros((H, W), np.uint8); mask_a[4:28, 6:40] = 1; mask_a[10:12, 8:30] = 0
    mask_b = np.zeros((H, W), np.uint8); mask_b[8:30, 3:35] = 1; mask_b[12:16, 10:20] = 0
    if kind == "values":
        mask_a[10:14, 10:30] = 255; mask_b[20:24, 5:15] = 255; mask_a[5, 7] = 2; mask_b[9, 4] = 2
    elif kind == "single":
        mask_a[:] = 0; mask_a[3, 5] = 1; mask_b[:] = 0; mask_b[30, 41] = 7
    elif kind == "empty_a":
        mask_a[:] = 0
    elif kind == "empty_b":
        mask_b[:] = 0
    elif kind == "empty_both":
        mask_a[:] = 0; mask_b[:] = 0
    n = cfg["num_samples"]
    params = np.zeros((2, 16), np.uint8)
    params[:, :5] = np.asarray(dec, np.uint8); params[:, 5:11] = g.randint(0, 255, (2, 6))
    u = lambda m: g.random_sample(m).astype(np.float32)
    rand = dict(params=params, noise=g.randint(0, 50, (2, 2, H, W, 3)).astype(np.uint8), blind_a=u(n), blind_b=u(n))
    return dict(rgb_a=rgb_a, rgb_b=rgb_b, mask_a=mask_a, mask_b=mask_b), cfg, rand


def run_case(fns, i):
    x, cfg, rand = case_inputs(i)
    return AO.get_across_scene_data(fns, x["rgb_a"], x["rgb_b"], x["mask_a"], x["mask_b"], cfg, rand)


KEYS = ("rgb_a", "rgb_b", "blind_a", "blind_b")


def main():
    from oracle import build_ref_augment
    fns = AO.executed_reference(build_ref_augment.load())
    out = {}
    for i, (name, _, _, _) in enumerate(CASES):
        r = run_case(fns, i)
        assert r["python_left"] == 0 and r["numpy_left"] == 0 and r["torch_left"] == 0, (name, r)
        out["%s/empty" % name] = np.array(r["empty"])
        for k in KEYS:
            out["%s/%s" % (name, k)] = r[k].astype(np.uint8 if k.startswith("rgb") else np.int32)
        print("%-40s empty=%d blind=%d" % (name, r["empty"], len(r["blind_a"])))
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
