"""Restatement of SpartanDataset.get_across_scene_data (dense_correspondence/dataset/spartan_dataset_masked.py:1056-1141,
debug off) for one pair, with its random numbers given: the producer of DIFFERENT_OBJECT (get_different_object_data,
:874-888) and SINGLE_OBJECT_ACROSS_SCENE (get_single_object_across_scene_data, :860-872) pairs.

TEST INFRASTRUCTURE, in the pattern of oracle/within_scene_oracle.py.  ``get_across_scene_data(fns, ...)`` restates the
method body and calls the functions it calls through ``fns``:
  * ``RESTATED`` (this module): the independent restatements of within_scene_oracle (correspondence_augmentation.py:19-214,
    correspondence_finder.py:92-121), with the sampler taking the numpy mask the method passes it;
  * ``executed_reference(oracle/build_ref_augment.load())``: the EXECUTED reference; oracle/make_golden_across_scene.py
    runs it to write tests/golden/across_scene_batch.npz, and tests/test_across_scene_cpu.py requires RESTATED to
    reproduce that bit for bit.
Both draw their random numbers from ``scripted(rand, ...)``, which replaces random.random, numpy.random.uniform and
torch.rand by functions returning the pair's numbers (the layout of pdc_b200.sampling.draw_across_scene_rand) in the
method's call order: torch.rand(n) for mask_a, then for mask_b (each only when that mask has a nonzero pixel); then, for
a pair that is not empty, the python / numpy decisions of the background randomisation of A then B, and the two flips.
"""
import contextlib
import random
import types

import numpy as np
import torch
from PIL import Image

from oracle import within_scene_oracle as WO


@contextlib.contextmanager
def scripted(rand, domain_randomize, mask_a_nonempty, mask_b_nonempty):
    """rand: one pair's numbers (numpy): params [2, 16] uint8, noise [2, 2, H, W, 3] uint8, blind_a / blind_b fp32 [n].
    Colours c are returned as (c + 0.5) / 255 (uint8(U * 255) = c), noise n as (n + 0.5) / 50, decisions d as 0.75 / 0.25."""
    py, npu = [], []
    if mask_a_nonempty and mask_b_nonempty:
        for img in range(2 if domain_randomize else 0):
            p = rand["params"][img]
            py.append(WO._decision(p[0]))
            if not p[0]:
                continue
            py.append(WO._decision(p[1]))
            npu.append((p[WO.RGB1:WO.RGB1 + 3].astype(np.float64) + 0.5) / 255)
            if p[1]:
                npu.append((p[WO.RGB2:WO.RGB2 + 3].astype(np.float64) + 0.5) / 255)
                npu.append(WO._decision(p[2]))
            py.append(WO._decision(p[3]))
            if p[3]:
                for k in range(2):
                    npu.append((rand["noise"][img, k].astype(np.float64) + 0.5) / 50)
        py += [WO._decision(rand["params"][0][WO.FLIP]), WO._decision(rand["params"][1][WO.FLIP])]
    draws = [rand[k] for k, nonempty in (("blind_a", mask_a_nonempty), ("blind_b", mask_b_nonempty)) if nonempty]
    pq, nq, tq = WO._Queue(py), WO._Queue(npu), WO._Queue(draws)

    def np_uniform(size=None):
        v = nq.pop()
        assert (np.shape(v) == ()) == (size is None) and (size is None or tuple(np.shape(v)) == tuple(np.atleast_1d(size)))
        return v

    def t_rand(*size, **kw):
        if len(size) == 1 and isinstance(size[0], (tuple, list, torch.Size)):
            size = tuple(size[0])
        u = tq.pop()
        assert len(size) == 1 and size[0] == len(u), size
        return torch.from_numpy(np.asarray(u, dtype=np.float32).copy())

    saved = (random.random, np.random.uniform, torch.rand)
    random.random, np.random.uniform, torch.rand = (lambda: pq.pop()), np_uniform, t_rand
    state = types.SimpleNamespace(python=pq, numpy=nq, torch=tq)
    try:
        yield state
    finally:
        random.random, np.random.uniform, torch.rand = saved


def _random_sample_from_masked_image_torch(img_mask, num_samples):      # correspondence_finder.py:92-121
    if isinstance(img_mask, np.ndarray):
        img_mask = torch.from_numpy(np.array(img_mask)).float()
    return WO._random_sample_from_masked_image_torch(img_mask, num_samples)


RESTATED = types.SimpleNamespace(
    random_domain_randomize_background=WO.RESTATED.random_domain_randomize_background,
    random_image_and_indices_mutation=WO.RESTATED.random_image_and_indices_mutation,
    random_sample_from_masked_image_torch=_random_sample_from_masked_image_torch)


def executed_reference(ref):
    """The same namespace over the executed reference (ref = oracle/build_ref_augment.load())."""
    return types.SimpleNamespace(
        random_domain_randomize_background=ref.aug.random_domain_randomize_background,
        random_image_and_indices_mutation=ref.aug.random_image_and_indices_mutation,
        random_sample_from_masked_image_torch=ref.finder.random_sample_from_masked_image_torch)


# ----------------------------------------------------------------------------- spartan_dataset_masked.py:1056-1141
def get_across_scene_data(fns, rgb_a, rgb_b, mask_a, mask_b, cfg, rand):
    """One pair.  rgb_* uint8 [H, W, 3], mask_* uint8 [H, W]; cfg as pdc_b200.sampling.across_scene_cfg; rand: the pair's
    numbers.  -> dict: uint8 images ``rgb_a`` / ``rgb_b`` [H, W, 3] (as rgb_image_to_tensor receives them), int64 lists
    ``blind_a`` / ``blind_b`` (empty for return_empty_data), ``empty``, and the scripted numbers left unconsumed."""
    with scripted(rand, cfg["domain_randomize"], bool(mask_a.any()), bool(mask_b.any())) as script:
        image_a_rgb, image_b_rgb = Image.fromarray(rgb_a), Image.fromarray(rgb_b)
        image_a_mask, image_b_mask = Image.fromarray(mask_a), Image.fromarray(mask_b)
        num_samples = cfg["num_samples"]
        blind_uv_a = fns.random_sample_from_masked_image_torch(np.asarray(image_a_mask), num_samples)
        blind_uv_b = fns.random_sample_from_masked_image_torch(np.asarray(image_b_mask), num_samples)
        left = lambda: dict(python_left=len(script.python.items), numpy_left=len(script.numpy.items),
                            torch_left=len(script.torch.items))
        if blind_uv_a[0] is None or blind_uv_b[0] is None:         # return_empty_data with image A twice
            none = np.zeros(0, dtype=np.int64)
            return dict(rgb_a=rgb_a.copy(), rgb_b=rgb_a.copy(), empty=True, blind_a=none, blind_b=none, **left())
        if cfg["domain_randomize"]:
            image_a_rgb = fns.random_domain_randomize_background(image_a_rgb, image_a_mask)
            image_b_rgb = fns.random_domain_randomize_background(image_b_rgb, image_b_mask)
        [image_a_rgb, image_a_mask], blind_uv_a = fns.random_image_and_indices_mutation([image_a_rgb, image_a_mask], blind_uv_a)
        [image_b_rgb, image_b_mask], blind_uv_b = fns.random_image_and_indices_mutation([image_b_rgb, image_b_mask], blind_uv_b)
        W = mask_b.shape[1]
        host = lambda t: t.reshape(-1).numpy().astype(np.int64)
        return dict(rgb_a=np.asarray(image_a_rgb).copy(), rgb_b=np.asarray(image_b_rgb).copy(), empty=False,
                    blind_a=host(WO._flatten(blind_uv_a, W)), blind_b=host(WO._flatten(blind_uv_b, W)), **left())
