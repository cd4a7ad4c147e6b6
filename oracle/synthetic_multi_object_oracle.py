"""Restatement of SpartanDataset.get_synthetic_multi_object_within_scene_data
(dense_correspondence/dataset/spartan_dataset_masked.py:890-1053, SYNTHETIC_MULTI_OBJECT, debug off) for one pair, with
its random numbers given.

TEST INFRASTRUCTURE, in the pattern of oracle/within_scene_oracle.py.  ``get_synthetic_data(fns, ...)`` restates the method
body (each half is get_within_scene_data up to its for_synthetic_multi_object return, :646-658) and calls the functions it
uses through ``fns``:
  * ``RESTATED`` (this module): the finder restatements of within_scene_oracle and independent restatements of
    merge_images_with_occlusions, prune_matches_if_occluded and merge_matches (correspondence_augmentation.py:217-347);
  * ``executed_reference(oracle/build_ref_augment.load())``: the EXECUTED reference; oracle/make_golden_synthetic.py runs
    it to write tests/golden/synthetic_multi_object_batch.npz, and tests/test_synthetic_multi_object_cpu.py requires
    RESTATED to reproduce that bit for bit.
``scripted(rand, ...)`` returns the pair's numbers (the layout of pdc_b200.sampling.draw_synthetic_multi_object_rand) in the
method's call order: the finder's draws of scene A, then of scene B; the two merge decisions (random.random); the masked and
the background non-match draws.
"""
import contextlib
import random
import types

import numpy as np
import torch
from PIL import Image

from oracle import within_scene_oracle as WO


@contextlib.contextmanager
def scripted(rand, candidates_from_mask):
    """rand: one pair's numbers (numpy): merge [2] uint8, cand_u / cand_v [2, n], masked_u/v, background_u/v."""
    def uniform_pair(u, v):
        def f(*size):
            if len(size) == 2:
                return torch.stack((torch.from_numpy(u[:size[1]].copy()), torch.from_numpy(v[:size[1]].copy())))
            return torch.from_numpy(u[:size[0]].copy())
        return f
    zeros = lambda *size: torch.zeros(*size)
    per_half = 2 if candidates_from_mask else 1
    tq = WO._Queue([uniform_pair(rand["cand_u"][0], rand["cand_v"][0])] * per_half +
                   [uniform_pair(rand["cand_u"][1], rand["cand_v"][1])] * per_half +
                   [uniform_pair(rand["masked_u"], rand["masked_v"]), zeros,
                    uniform_pair(rand["background_u"], rand["background_v"]), zeros])
    pq = WO._Queue([0.25 if d else 0.75 for d in rand["merge"]])     # random.random() < 0.5: scene B in the foreground

    def t_rand(*size, **kw):
        if len(size) == 1 and isinstance(size[0], (tuple, list, torch.Size)):
            size = tuple(size[0])
        return tq.pop()(*size)

    saved = (random.random, torch.rand)
    random.random, torch.rand = (lambda: pq.pop()), t_rand
    try:
        yield types.SimpleNamespace(python=pq, torch=tq)
    finally:
        random.random, torch.rand = saved


# ----------------------------------------------------------------------------- correspondence_augmentation.py:217-347
def _prune_matches_if_occluded(foreground_mask_numpy, background_matches_pair):
    (ua, va), (ub, vb) = background_matches_pair
    keep = [i for i in range(len(ua)) if foreground_mask_numpy[int(va[i]), int(ua[i])] == 0]
    if not keep:
        return (None, None)
    k = torch.LongTensor(keep)
    return (ua[k], va[k]), (ub[k], vb[k])


def _merge_images_with_occlusions(image_a, image_b, mask_a, mask_b, matches_pair_a, matches_pair_b):
    fg_is_b = random.random() < 0.5
    if fg_is_b:
        bg_img, bg_mask, bg_pair, fg_img, fg_mask, fg_pair = image_a, mask_a, matches_pair_a, image_b, mask_b, matches_pair_b
    else:
        bg_img, bg_mask, bg_pair, fg_img, fg_mask, fg_pair = image_b, mask_b, matches_pair_b, image_a, mask_a, matches_pair_a
    fm = np.asarray(fg_mask)
    m3 = np.repeat(fm[:, :, None], 3, axis=2).astype(np.uint8)
    merged = np.asarray(fg_img) * m3 + (np.uint8(1) - m3) * np.asarray(bg_img)
    bg_pair = _prune_matches_if_occluded(fm, bg_pair)
    a_pair, b_pair = (bg_pair, fg_pair) if fg_is_b else (fg_pair, bg_pair)
    merged_mask = (fm + np.asarray(bg_mask)).clip(0, 1)
    return Image.fromarray(merged.astype(np.uint8)), merged_mask, a_pair[0], a_pair[1], b_pair[0], b_pair[1]


def _merge_matches(matches_one, matches_two):
    return torch.cat((matches_one[0], matches_two[0])), torch.cat((matches_one[1], matches_two[1]))


RESTATED = types.SimpleNamespace(
    batch_find_pixel_correspondences=WO.RESTATED.batch_find_pixel_correspondences,
    create_non_correspondences=WO.RESTATED.create_non_correspondences,
    merge_images_with_occlusions=_merge_images_with_occlusions,
    prune_matches_if_occluded=_prune_matches_if_occluded,
    merge_matches=_merge_matches)


def executed_reference(ref):
    """The same namespace over the executed reference (ref = oracle/build_ref_augment.load())."""
    return types.SimpleNamespace(
        batch_find_pixel_correspondences=lambda *a, **kw: ref.finder.batch_find_pixel_correspondences(*a, **kw),
        create_non_correspondences=ref.finder.create_non_correspondences,
        merge_images_with_occlusions=ref.aug.merge_images_with_occlusions,
        prune_matches_if_occluded=ref.aug.prune_matches_if_occluded,
        merge_matches=ref.aug.merge_matches)


# ----------------------------------------------------------------------------- spartan_dataset_masked.py:890-1053
def get_synthetic_data(fns, scene_a, scene_b, K, cfg, rand, uv=None):
    """One pair.  scene_*: dicts rgb_1, rgb_2 uint8 [H, W, 3], depth_1, depth_2 [H, W] millimetres, mask_1, mask_2 uint8
    [H, W], pose_1, pose_2 4x4; K 3x3; cfg as pdc_b200.sampling.within_scene_cfg; rand: the pair's numbers.  ``uv`` =
    ((u1, v1, u2, v2) of scene A, (...) of scene B) replaces the finder's results (its candidates are still drawn).
    -> dict: uint8 images ``rgb_a`` / ``rgb_b`` (merged 1, merged 2, or the early return's image twice), int64 lists
    matches_a/b, masked_a/b, background_a/b, ``empty`` and ``ret`` (which return: "merged", "a1", "b1", "occluded_1",
    "occluded_2")."""
    H, W = scene_a["mask_1"].shape
    none = np.zeros(0, dtype=np.int64)

    def early(img, ret):
        return dict(rgb_a=img.copy(), rgb_b=img.copy(), empty=True, ret=ret, matches_a=none, matches_b=none, masked_a=none,
                    masked_b=none, background_a=none, background_b=none)

    with scripted(rand, cfg["sample_matches_only_off_mask"]) as script:
        def half(s, h):
            uv1, uv2 = fns.batch_find_pixel_correspondences(s["depth_1"], s["pose_1"], s["depth_2"], s["pose_2"], img_a_mask=(
                s["mask_1"] if cfg["sample_matches_only_off_mask"] else None), num_attempts=cfg["n_attempts"], K=K)
            if uv is not None and uv1 is not None:
                uv1, uv2 = (uv[h][0], uv[h][1]), (uv[h][2], uv[h][3])
            return uv1, uv2
        uv_a1, uv_a2 = half(scene_a, 0)
        if uv_a1 is None:
            return early(scene_a["rgb_1"], "a1")
        uv_b1, uv_b2 = half(scene_b, 1)
        if uv_b1 is None:
            return early(scene_b["rgb_1"], "b1")
        L = lambda uv: (uv[0].long(), uv[1].long())
        uv_a1, uv_a2, uv_b1, uv_b2 = L(uv_a1), L(uv_a2), L(uv_b1), L(uv_b2)
        img = lambda s, k: Image.fromarray(s[k])
        merged_rgb_1, _, uv_a1, uv_a2, uv_b1, uv_b2 = fns.merge_images_with_occlusions(
            img(scene_a, "rgb_1"), img(scene_b, "rgb_1"), img(scene_a, "mask_1"), img(scene_b, "mask_1"), (uv_a1, uv_a2),
            (uv_b1, uv_b2))
        if uv_a1 is None or uv_a2 is None or uv_b1 is None or uv_b2 is None:
            return early(scene_b["rgb_1"], "occluded_1")
        merged_rgb_2, merged_mask_2, uv_a2, uv_a1, uv_b2, uv_b1 = fns.merge_images_with_occlusions(
            img(scene_a, "rgb_2"), img(scene_b, "rgb_2"), img(scene_a, "mask_2"), img(scene_b, "mask_2"), (uv_a2, uv_a1),
            (uv_b2, uv_b1))
        if uv_a1 is None or uv_a2 is None or uv_b1 is None or uv_b2 is None:
            return early(scene_b["rgb_1"], "occluded_2")
        matches_1 = fns.merge_matches(uv_a1, uv_b1)
        matches_2 = fns.merge_matches(uv_a2, uv_b2)
        matches_2 = (matches_2[0].float(), matches_2[1].float())
        mask_t = torch.from_numpy(np.asarray(merged_mask_2).copy()).type(torch.FloatTensor)
        masked = fns.create_non_correspondences(matches_2, (H, W), num_non_matches_per_match=cfg["k_masked"], img_b_mask=mask_t)
        inv = 1 - mask_t if cfg["use_image_b_mask_inv"] else None
        background = fns.create_non_correspondences(matches_2, (H, W), num_non_matches_per_match=cfg["k_background"],
                                                    img_b_mask=inv)
        ma_long, mb_long = WO._create_non_matches(matches_1, masked, cfg["k_masked"])
        ba_long, bb_long = WO._create_non_matches(matches_1, background, cfg["k_background"])
        host = lambda t: t.reshape(-1).numpy().astype(np.int64)
        return dict(rgb_a=np.asarray(merged_rgb_1).copy(), rgb_b=np.asarray(merged_rgb_2).copy(), empty=False, ret="merged",
                    matches_a=host(WO._flatten(matches_1, W)), matches_b=host(WO._flatten(matches_2, W)),
                    masked_a=host(WO._flatten(ma_long, W)), masked_b=host(WO._flatten(mb_long, W)),
                    background_a=host(WO._flatten(ba_long, W)), background_b=host(WO._flatten(bb_long, W)),
                    python_left=len(script.python.items), torch_left=len(script.torch.items))
