"""CPU: the within-scene batch producer's oracle, normalisation and C ABI refusals.

* oracle/within_scene_oracle.py's restatement reproduces, bit for bit, what the executed reference computed for every case
  of oracle/make_golden_within_scene.py (stored in tests/golden/within_scene_batch.npz);
* the normalisation table ((x / 255) - mean) / std equals torchvision's ToTensor + Normalize on all 256 values;
* ddn_within_scene_batch refuses every malformed argument with -1 before launching anything.
(The device results against the same goldens: tests/test_gpu_within_scene.py.)"""
import ctypes
import os

import numpy as np
import pytest
import torch

import pdc_b200  # noqa: F401
from pdc_b200 import _native as N
from pdc_b200 import sampling as S
from oracle import make_golden_within_scene as MG
from oracle import within_scene_oracle as WO


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "within_scene_batch.npz"))


@pytest.mark.parametrize("case", [c[0] for c in MG.CASES])
def test_restatement_equals_executed_reference(golden, case):
    r = MG.run_case(WO.RESTATED, [c[0] for c in MG.CASES].index(case))
    assert bool(golden[case + "/empty"]) == r["empty"]
    if not r["empty"]:
        assert r["python_left"] == 0 and r["numpy_left"] == 0          # every scripted decision was drawn
    for k in MG.KEYS:
        np.testing.assert_array_equal(r[k], golden["%s/%s" % (case, k)].astype(r[k].dtype), err_msg=k)


def test_golden_covers_the_cases(golden):
    g = lambda c, k: golden["%s/%s" % (c, k)]
    assert bool(g("empty_mask_a", "empty")) and np.array_equal(g("empty_mask_a", "rgb_a"), g("empty_mask_a", "rgb_b"))
    assert len(g("empty_mask_b", "blind_a")) == 0 and len(g("empty_mask_b", "masked_a")) > 0
    x, _, _ = MG.case_inputs(3)
    assert (x["mask_a"] == 255).any() and (x["mask_b"] == 255).any()
    for c, _, _, _ in MG.CASES:
        if not bool(g(c, "empty")):
            assert len(g(c, "matches_a")) > 0 and len(g(c, "blind_a")) > 0 or c == "empty_mask_b"


def test_normalisation_table_equals_torchvision():
    T = pytest.importorskip("torchvision.transforms")
    from PIL import Image
    img = np.stack([np.arange(256, dtype=np.uint8)] * 3, axis=1).reshape(16, 16, 3)
    ref = T.Compose([T.ToTensor(), T.Normalize(list(S.IMAGE_MEAN), list(S.IMAGE_STD))])(Image.fromarray(img)).numpy()
    lut = WO.normalize_lut()
    ours = np.stack([lut[c][img[:, :, c]] for c in range(3)])
    assert ours.dtype == np.float32 and np.array_equal(ours.view(np.uint32), ref.view(np.uint32))
    assert S.IMAGE_MEAN == WO.IMAGE_MEAN and S.IMAGE_STD == WO.IMAGE_STD


def _cfg(**kw):
    c = dict(B=2, H=32, W=48, sample_matches_only_off_mask=1, domain_randomize=1, use_image_b_mask_inv=1, n_attempts=200,
             k_masked=3, k_background=2, mean=(ctypes.c_float * 3)(0.5, 0.4, 0.4), std=(ctypes.c_float * 3)(0.2, 0.3, 0.3))
    c.update(kw)
    return N.WsBatchCfg(**c)


def test_within_scene_batch_refusals_launch_nothing():
    fake = 1 << 40
    big = 1 << 40
    K = (ctypes.c_double * 9)(100.0, 0, 20, 0, 100.0, 15, 0, 0, 1)
    poses = (ctypes.c_double * (16 * 200))(*([1.0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 1.0] * 200))
    singular = (ctypes.c_double * 9)()
    rand_keys = [f for f, _ in N.WsBatchRand._fields_]
    out_keys = [f for f, _ in N.WsBatchOut._fields_]

    def call(cfg=None, ins=fake, K=K, pa=poses, rand=None, out=None, scratch=fake, scratch_bytes=big, rnull=None, onull=None):
        cfg = cfg if cfg is not None else _cfg()
        r = N.WsBatchRand(**{k: (None if k == rnull else fake) for k in rand_keys}) if rand is None else rand
        o = N.WsBatchOut(**{k: (None if k == onull else fake) for k in out_keys}) if out is None else out
        return N.lib.ddn_within_scene_batch(ctypes.byref(cfg) if cfg is not False else None, fake, fake, ins, fake, fake, fake,
                                            K, pa, poses, ctypes.byref(r), ctypes.byref(o), scratch, scratch_bytes, None)

    before = N.launch_count()
    assert N.lib.ddn_within_scene_batch_scratch_bytes(ctypes.byref(_cfg())) > 0
    bad_cfgs = [_cfg(B=0), _cfg(B=N.WS_MAX_PAIRS + 1), _cfg(H=0), _cfg(W=-3), _cfg(H=1 << 15, W=1 << 15), _cfg(n_attempts=0),
                _cfg(n_attempts=1 << 30), _cfg(k_masked=-1), _cfg(k_background=-1), _cfg(k_masked=1 << 25),
                _cfg(sample_matches_only_off_mask=2), _cfg(domain_randomize=-1), _cfg(use_image_b_mask_inv=5),
                _cfg(std=(ctypes.c_float * 3)(0.2, 0.0, 0.3)), _cfg(mean=(ctypes.c_float * 3)(float("nan"), 0, 0))]
    for c in bad_cfgs:
        assert N.lib.ddn_within_scene_batch_scratch_bytes(ctypes.byref(c)) == 0
        assert call(cfg=c) == -1
    assert N.lib.ddn_within_scene_batch_scratch_bytes(None) == 0
    assert call(cfg=False) == -1
    for kw in [dict(ins=None), dict(K=None), dict(pa=None), dict(K=singular), dict(scratch=None), dict(scratch_bytes=16)] + \
              [dict(rnull=k) for k in rand_keys] + [dict(onull=k) for k in out_keys]:
        assert call(**kw) == -1, kw
    assert N.launch_count() == before


def test_python_wrapper_refusals():
    B, H, W = 1, 8, 16
    cfg = {"training": dict(num_matching_attempts=10, num_non_matches_per_match=4, fraction_masked_non_matches=0.5,
                            fraction_background_non_matches=0.5, sample_matches_only_off_mask=True, domain_randomize=True,
                            use_image_b_mask_inv=True)}
    rgb = torch.zeros(B, H, W, 3, dtype=torch.uint8); m = torch.zeros(B, H, W, dtype=torch.uint8); d = torch.zeros(B, H, W)
    pose = np.eye(4)[None]
    with pytest.raises(RuntimeError, match="CUDA"):
        S.within_scene_batch(rgb, rgb, d, d, m, m, pose, pose, np.eye(3), cfg)
    with pytest.raises(NotImplementedError):
        S.within_scene_batch(rgb, rgb, d, d, m, m, pose, pose, np.eye(3), {"training": dict(cfg["training"], debug=True)})
    assert S.within_scene_cfg(cfg) == dict(n_attempts=10, k_masked=2, k_background=2, sample_matches_only_off_mask=True,
                                           domain_randomize=True, use_image_b_mask_inv=True)
