"""Restatement of SpartanDataset.get_within_scene_data (dense_correspondence/dataset/spartan_dataset_masked.py:646-769,
SINGLE_OBJECT_WITHIN_SCENE, debug off) for one pair, with its random numbers given.

TEST INFRASTRUCTURE.  ``get_within_scene_data(fns, ...)`` restates the method body and calls the functions it calls
through ``fns``:
  * ``RESTATED`` (this module): independent restatements of correspondence_augmentation.py:19-214 and of the finder's
    sampling functions; they need nothing outside the repository, and the tests run them;
  * oracle/build_ref_augment.load(): the EXECUTED reference; oracle/make_golden_within_scene.py runs it to write
    tests/golden/within_scene_batch.npz, and tests/test_within_scene_cpu.py requires RESTATED to reproduce that bit for bit.
Both draw their random numbers from ``scripted(rand)``, which replaces random.random, numpy.random.uniform and torch.rand
by functions returning the pair's numbers (the layout of pdc_b200.sampling.draw_within_scene_rand) in call order.
"""
import contextlib
import random
import types

import numpy as np
import torch
from PIL import Image

from oracle import loss_oracle as LO

IMAGE_MEAN = (0.5573105812072754, 0.37420374155044556, 0.37020164728164673)     # constants.py:18-19
IMAGE_STD = (0.24336038529872894, 0.2987397611141205, 0.31875079870224)
RGB1, RGB2, FLIP = 5, 8, 4


def normalize_lut():
    """ToTensor + Normalize of every uint8 value: fp32 [3, 256] = ((x / 255) - mean_c) / std_c, IEEE fp32 division."""
    x = np.arange(256, dtype=np.float32) / np.float32(255)
    mean = np.asarray(IMAGE_MEAN, dtype=np.float32)[:, None]; std = np.asarray(IMAGE_STD, dtype=np.float32)[:, None]
    return ((x[None, :] - mean) / std).astype(np.float32)


# ----------------------------------------------------------------------------- scripted random numbers
class _Queue(object):
    def __init__(self, items):
        self.items = list(items)

    def pop(self):
        if not self.items:
            raise RuntimeError("the reference drew more random numbers than the script holds")
        return self.items.pop(0)


def _decision(d):
    return 0.75 if d else 0.25          # every decision is `random.random() < 0.5` -> not taken / `uniform() > 0.5` -> taken


@contextlib.contextmanager
def scripted(rand, H, W, domain_randomize, candidates_from_mask):
    """rand: one pair's numbers (numpy): params [2, 16] uint8, noise [2, 2, H, W, 3] uint8, cand_u/v, masked_u/v,
    background_u/v, blind fp32.  Colours c are returned as (c + 0.5) / 255 (uint8(U * 255) = c), noise n as (n + 0.5) / 50."""
    py, npu = [], []
    for img in range(2 if domain_randomize else 0):
        p = rand["params"][img]
        py.append(_decision(p[0]))
        if not p[0]:
            continue
        py.append(_decision(p[1]))
        npu.append((p[RGB1:RGB1 + 3].astype(np.float64) + 0.5) / 255)
        if p[1]:
            npu.append((p[RGB2:RGB2 + 3].astype(np.float64) + 0.5) / 255)
            npu.append(_decision(p[2]))
        py.append(_decision(p[3]))
        if p[3]:
            for k in range(2):
                npu.append((rand["noise"][img, k].astype(np.float64) + 0.5) / 50)
    py += [_decision(rand["params"][0][FLIP]), _decision(rand["params"][1][FLIP])]

    def uniform_pair(u, v):
        def f(*size):
            if len(size) == 2:          # pytorch_rand_select_pixel: torch.rand(2, n)
                return torch.stack((torch.from_numpy(u[:size[1]].copy()), torch.from_numpy(v[:size[1]].copy())))
            return torch.from_numpy(u[:size[0]].copy())
        return f
    zeros = lambda *size: torch.zeros(*size)          # the finder's no-op perturbation draw (correspondence_finder.py:363)
    # batch_find_pixel_correspondences always draws torch.rand(2, n) first (:460-461) and, sampling on the mask, then
    # torch.rand(n) (:473): both get the candidate numbers, only the one used matters
    tq = _Queue([uniform_pair(rand["cand_u"], rand["cand_v"])] * (2 if candidates_from_mask else 1) +
                [uniform_pair(rand["masked_u"], rand["masked_v"]), zeros,
                 uniform_pair(rand["background_u"], rand["background_v"]), zeros, uniform_pair(rand["blind"], rand["blind"])])
    pq, nq = _Queue(py), _Queue(npu)

    def np_uniform(size=None):
        v = nq.pop()
        assert (np.shape(v) == ()) == (size is None) and (size is None or tuple(np.shape(v)) == tuple(np.atleast_1d(size)))
        return v

    def t_rand(*size, **kw):
        if len(size) == 1 and isinstance(size[0], (tuple, list, torch.Size)):
            size = tuple(size[0])
        return tq.pop()(*size)

    saved = (random.random, np.random.uniform, torch.rand)
    random.random, np.random.uniform, torch.rand = (lambda: pq.pop()), np_uniform, t_rand
    state = types.SimpleNamespace(python=pq, numpy=nq, torch=tq)
    try:
        yield state
    finally:
        random.random, np.random.uniform, torch.rand = saved


# ----------------------------------------------------------------------------- restated reference functions
def _random_image(shape):                       # correspondence_augmentation.py:125-146, 148-214
    def rgb():
        return np.array(np.random.uniform(size=3) * 255, dtype=np.uint8)
    if random.random() < 0.5:
        img = np.ones(shape, dtype=np.uint8) * rgb()
    else:
        rgb1 = np.ones(shape, dtype=np.uint8) * rgb(); rgb2 = np.ones(shape, dtype=np.uint8) * rgb()
        vertical = bool(np.random.uniform() > 0.5)
        h, w = shape[0], shape[1]
        p = np.tile(np.linspace(0, 1, h)[:, None], (1, w)) if vertical else np.tile(np.linspace(0, 1, w), (h, 1))
        img = np.zeros_like(rgb1)
        for c in range(3):
            img[:, :, c] = rgb2[:, :, c] * p + rgb1[:, :, c] * (1.0 - p)
    if random.random() < 0.5:
        return img
    n1 = np.array(np.random.uniform(size=shape) * 50, dtype=np.uint8)
    n2 = np.array(np.random.uniform(size=shape) * 50, dtype=np.uint8)
    return img + n1 - n2


def _random_domain_randomize_background(image_rgb, image_mask):     # :86-123
    if random.random() < 0.5:
        return image_rgb
    rgb = np.asarray(image_rgb); m = np.repeat(np.asarray(image_mask)[:, :, None], 3, axis=2).astype(np.uint8)
    out = rgb * m + (np.uint8(1) - m) * _random_image(rgb.shape)
    return Image.fromarray(out.astype(np.uint8))


def _random_image_and_indices_mutation(images, uv):                 # :19-84: a 180-degree rotation, half of the time
    if random.random() < 0.5:
        return images, uv
    rotated = [Image.fromarray(np.ascontiguousarray(np.asarray(im)[::-1, ::-1])) for im in images]
    h, w = np.asarray(images[-1]).shape[:2]
    return rotated, ((w - 1) - uv[0], (h - 1) - uv[1])


def _random_sample_from_masked_image_torch(img_mask, num_samples):  # correspondence_finder.py:92-121
    H, W = img_mask.shape
    nz = torch.nonzero(img_mask.reshape(-1))
    if len(nz) == 0:
        return None, None
    flat = torch.index_select(nz, 0, torch.floor(torch.rand(num_samples) * len(nz)).long()).squeeze(1)
    return flat % W, flat // W


def _batch_find_pixel_correspondences(img_a_depth, img_a_pose, img_b_depth, img_b_pose, num_attempts=20, img_a_mask=None, K=None):
    """correspondence_finder.py:409-619 (candidates drawn first, then oracle/loss_oracle's restatement; the uniform draw
    happens even when the candidates come from the mask, as in the reference); every pruning stage
    that leaves nothing returns empty tensors, as the reference does on torch >= 1.0 (nonzero() keeps 2 dimensions)."""
    H, W = img_a_depth.shape
    r = torch.rand(2, num_attempts)
    if img_a_mask is None:
        u, v = torch.floor(r[0] * W).long(), torch.floor(r[1] * H).long()
    else:
        u, v = _random_sample_from_masked_image_torch(torch.from_numpy(img_a_mask).float(), num_attempts)
        if u is None:
            return None, None
    uv_a, uv_b = LO.batch_find_pixel_correspondences(img_a_depth.astype(np.float32), img_a_pose, img_b_depth.astype(np.float32),
                                                     img_b_pose, v * W + u, K)
    if uv_a is None:
        return (torch.zeros(0, dtype=torch.int64),) * 2, (torch.zeros(0),) * 2
    return uv_a, uv_b


def _create_non_correspondences(uv_b_matches, img_b_shape, num_non_matches_per_match=100, img_b_mask=None):   # :276-405
    H, W = img_b_shape
    n = len(uv_b_matches[0]) * num_non_matches_per_match
    nz = torch.nonzero(img_b_mask.reshape(-1)) if img_b_mask is not None else torch.zeros(0, 1, dtype=torch.int64)
    if len(nz) == 0:
        r = torch.rand(2, n)
        u, v = torch.floor(r[0] * W).long(), torch.floor(r[1] * H).long()
    else:
        flat = torch.index_select(nz, 0, torch.floor(torch.rand(n) * len(nz)).long()).squeeze(1)
        u, v = flat % W, flat // W
    torch.rand(n)                           # the "too close" perturbation: drawn, multiplied by zero
    m, k = len(uv_b_matches[0]), num_non_matches_per_match
    return u.float().view(m, k), v.float().view(m, k)


RESTATED = types.SimpleNamespace(
    random_domain_randomize_background=_random_domain_randomize_background,
    random_image_and_indices_mutation=_random_image_and_indices_mutation,
    batch_find_pixel_correspondences=_batch_find_pixel_correspondences,
    create_non_correspondences=_create_non_correspondences,
    random_sample_from_masked_image_torch=_random_sample_from_masked_image_torch)


def executed_reference(ref):
    """The same namespace over the executed reference (ref = oracle/build_ref_augment.load())."""
    return types.SimpleNamespace(
        random_domain_randomize_background=ref.aug.random_domain_randomize_background,
        random_image_and_indices_mutation=ref.aug.random_image_and_indices_mutation,
        batch_find_pixel_correspondences=lambda *a, **kw: ref.finder.batch_find_pixel_correspondences(*a, **kw),
        create_non_correspondences=ref.finder.create_non_correspondences,
        random_sample_from_masked_image_torch=ref.finder.random_sample_from_masked_image_torch)


# ----------------------------------------------------------------------------- spartan_dataset_masked.py:646-769
def _flatten(uv, W):                            # flatten_uv_tensor (:1255-1264)
    return uv[1].long() * W + uv[0].long()


def _create_non_matches(uv_a, uv_b_non_matches, k):      # :841-858
    uv_a_long = (torch.t(uv_a[0].repeat(k, 1)).contiguous().view(-1, 1), torch.t(uv_a[1].repeat(k, 1)).contiguous().view(-1, 1))
    return uv_a_long, (uv_b_non_matches[0].reshape(-1, 1), uv_b_non_matches[1].reshape(-1, 1))


def get_within_scene_data(fns, rgb_a, rgb_b, depth_a, depth_b, mask_a, mask_b, pose_a, pose_b, K, cfg, rand, uv=None):
    """One pair.  rgb_* uint8 [H, W, 3], mask_* uint8 [H, W], depth_* [H, W] millimetres, pose_* 4x4, K 3x3; cfg as
    pdc_b200.sampling.within_scene_cfg; rand: the pair's numbers.  ``uv`` = (u_a, v_a, u2, v2) replaces the finder's
    result (its candidates are still drawn).  -> dict: uint8 images ``rgb_a`` / ``rgb_b`` [H, W, 3] (as
    rgb_image_to_tensor receives them), int64 lists matches_a/b, masked_a/b, background_a/b, blind_a/b (blind empty when
    the reference returns its [-1] sentinel), ``empty`` (return_empty_data)."""
    H, W = mask_a.shape
    with scripted(rand, H, W, cfg["domain_randomize"], cfg["sample_matches_only_off_mask"]) as script:
        uv_a, uv_b = fns.batch_find_pixel_correspondences(depth_a, pose_a, depth_b, pose_b, img_a_mask=(
            mask_a if cfg["sample_matches_only_off_mask"] else None), num_attempts=cfg["n_attempts"], K=K)
        if uv is not None and uv_a is not None:
            uv_a, uv_b = (uv[0], uv[1]), (uv[2], uv[3])
        none = np.zeros(0, dtype=np.int64)
        if uv_a is None:
            return dict(rgb_a=rgb_a.copy(), rgb_b=rgb_a.copy(), empty=True, matches_a=none, matches_b=none, masked_a=none,
                        masked_b=none, background_a=none, background_b=none, blind_a=none, blind_b=none)
        image_a_rgb, image_b_rgb = Image.fromarray(rgb_a), Image.fromarray(rgb_b)
        image_a_mask, image_b_mask = Image.fromarray(mask_a), Image.fromarray(mask_b)
        if cfg["domain_randomize"]:
            image_a_rgb = fns.random_domain_randomize_background(image_a_rgb, image_a_mask)
            image_b_rgb = fns.random_domain_randomize_background(image_b_rgb, image_b_mask)
        [image_a_rgb, image_a_mask], uv_a = fns.random_image_and_indices_mutation([image_a_rgb, image_a_mask], uv_a)
        [image_b_rgb, image_b_mask], uv_b = fns.random_image_and_indices_mutation([image_b_rgb, image_b_mask], uv_b)

        image_b_mask_torch = torch.from_numpy(np.asarray(image_b_mask).copy()).type(torch.FloatTensor)
        uv_b_masked = fns.create_non_correspondences(uv_b, (H, W), num_non_matches_per_match=cfg["k_masked"],
                                                     img_b_mask=image_b_mask_torch)
        mask_inv = 1 - image_b_mask_torch if cfg["use_image_b_mask_inv"] else None
        uv_b_background = fns.create_non_correspondences(uv_b, (H, W), num_non_matches_per_match=cfg["k_background"],
                                                         img_b_mask=mask_inv)
        matches_a, matches_b = _flatten(uv_a, W), _flatten(uv_b, W)
        ma_long, mb_long = _create_non_matches(uv_a, uv_b_masked, cfg["k_masked"])
        ba_long, bb_long = _create_non_matches(uv_a, uv_b_background, cfg["k_background"])

        matched = torch.zeros(W * H).long()                     # mask_image_from_uv_flat_tensor (:1267-1282)
        matched[matches_a] = 1
        mask_a_flat = torch.from_numpy(np.asarray(image_a_mask).copy()).long().view(-1)
        blind_a = (mask_a_flat - matched).nonzero()
        blind_b = None
        if len(blind_a) > 0:
            blind_a = blind_a.squeeze(1)
            blind_uv_b = fns.random_sample_from_masked_image_torch(image_b_mask_torch, blind_a.size()[0])
            if blind_uv_b[0] is not None and len(blind_uv_b[0]) > 0:
                blind_b = blind_uv_b[1] * W + blind_uv_b[0]
        if blind_b is None:
            blind_a = blind_b = torch.zeros(0, dtype=torch.int64)
        host = lambda t: t.reshape(-1).numpy().astype(np.int64)
        return dict(rgb_a=np.asarray(image_a_rgb).copy(), rgb_b=np.asarray(image_b_rgb).copy(), empty=False,
                    matches_a=host(matches_a), matches_b=host(matches_b),
                    masked_a=host(_flatten(ma_long, W)), masked_b=host(_flatten(mb_long, W)),
                    background_a=host(_flatten(ba_long, W)), background_b=host(_flatten(bb_long, W)),
                    blind_a=host(blind_a), blind_b=host(blind_b), python_left=len(script.python.items),
                    numpy_left=len(script.numpy.items))
