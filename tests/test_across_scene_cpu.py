"""CPU: the across-scene batch producer's oracle, configuration and C ABI refusals.

* oracle/across_scene_oracle.py's restatement reproduces, bit for bit, what the executed reference computed for every case
  of oracle/make_golden_across_scene.py (stored in tests/golden/across_scene_batch.npz), consuming every scripted number;
* ddn_across_scene_batch refuses every malformed argument with -1 before launching anything;
* the Python wrapper refuses CPU tensors, debug=True and a match type that is not an across-scene type.
(The device results against the same goldens: tests/test_gpu_across_scene.py.)"""
import ctypes
import os

import numpy as np
import pytest
import torch

import pdc_b200  # noqa: F401
from pdc_b200 import _native as N
from pdc_b200 import sampling as S
from pdc_b200.loss_composer import SpartanDatasetDataType as T
from oracle import across_scene_oracle as AO
from oracle import make_golden_across_scene as MG

NAMES = [c[0] for c in MG.CASES]


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "across_scene_batch.npz"))


@pytest.mark.parametrize("case", NAMES)
def test_restatement_equals_executed_reference(golden, case):
    r = MG.run_case(AO.RESTATED, NAMES.index(case))
    assert bool(golden[case + "/empty"]) == r["empty"]
    assert r["python_left"] == 0 and r["numpy_left"] == 0 and r["torch_left"] == 0     # every scripted number was drawn
    for k in MG.KEYS:
        np.testing.assert_array_equal(r[k], golden["%s/%s" % (case, k)].astype(r[k].dtype), err_msg=k)


def test_golden_covers_the_cases(golden):
    g = lambda c, k: golden["%s/%s" % (c, k)]
    for c in ("empty_mask_a", "empty_mask_b", "empty_both"):
        assert bool(g(c, "empty")) and len(g(c, "blind_a")) == 0 and np.array_equal(g(c, "rgb_a"), g(c, "rgb_b"))
        x, _, _ = MG.case_inputs(NAMES.index(c))
        assert np.array_equal(g(c, "rgb_a"), x["rgb_a"])            # un-augmented image A
    for i, (c, dec, _, over) in enumerate(MG.CASES):
        if bool(g(c, "empty")):
            continue
        x, cfg, _ = MG.case_inputs(i)
        assert len(g(c, "blind_a")) == len(g(c, "blind_b")) == cfg["num_samples"]
        # every blind pixel lies on its (possibly flipped) mask
        for side, d in (("a", dec[0]), ("b", dec[1])):
            m = x["mask_" + side].reshape(-1)
            p = g(c, "blind_" + side).astype(np.int64)
            assert (m[(m.size - 1 - p) if d[4] else p] != 0).all(), (c, side)
    x, _, _ = MG.case_inputs(NAMES.index("no_randomise_a_mask_255"))
    assert (x["mask_a"] == 255).any() and (x["mask_b"] == 2).any()
    assert len(set(g("single_pixel_masks", "blind_b").tolist())) == 1


def _cfg(**kw):
    c = dict(B=2, H=32, W=48, domain_randomize=1, num_samples=500, mean=(ctypes.c_float * 3)(0.5, 0.4, 0.4),
             std=(ctypes.c_float * 3)(0.2, 0.3, 0.3))
    c.update(kw)
    return N.AsBatchCfg(**c)


def test_across_scene_batch_refusals_launch_nothing():
    fake = 1 << 40
    big = 1 << 40
    rand_keys = [f for f, _ in N.AsBatchRand._fields_]
    out_keys = [f for f, _ in N.AsBatchOut._fields_]

    def call(cfg=None, rgb_a=fake, rgb_b=fake, mask_a=fake, mask_b=fake, scratch=fake, scratch_bytes=big, rnull=None,
             onull=None, rand=True, out=True):
        cfg = cfg if cfg is not None else _cfg()
        r = N.AsBatchRand(**{k: (None if k == rnull else fake) for k in rand_keys})
        o = N.AsBatchOut(**{k: (None if k == onull else fake) for k in out_keys})
        return N.lib.ddn_across_scene_batch(ctypes.byref(cfg) if cfg is not False else None, rgb_a, rgb_b, mask_a, mask_b,
                                            ctypes.byref(r) if rand else None, ctypes.byref(o) if out else None,
                                            scratch, scratch_bytes, None)

    before = N.launch_count()
    assert N.lib.ddn_across_scene_batch_scratch_bytes(ctypes.byref(_cfg())) > 0
    assert N.lib.ddn_across_scene_batch_scratch_bytes(ctypes.byref(_cfg(B=N.AS_MAX_PAIRS, H=4, W=4))) > 0
    bad_cfgs = [_cfg(B=0), _cfg(B=N.AS_MAX_PAIRS + 1), _cfg(H=0), _cfg(W=-3), _cfg(H=1 << 15, W=1 << 15),
                _cfg(num_samples=0), _cfg(num_samples=-5), _cfg(num_samples=1 << 30), _cfg(domain_randomize=2),
                _cfg(domain_randomize=-1), _cfg(std=(ctypes.c_float * 3)(0.2, 0.0, 0.3)),
                _cfg(std=(ctypes.c_float * 3)(0.2, float("nan"), 0.3)), _cfg(mean=(ctypes.c_float * 3)(float("nan"), 0, 0))]
    for c in bad_cfgs:
        assert N.lib.ddn_across_scene_batch_scratch_bytes(ctypes.byref(c)) == 0
        assert call(cfg=c) == -1
    assert N.lib.ddn_across_scene_batch_scratch_bytes(None) == 0
    assert call(cfg=False) == -1
    need = N.lib.ddn_across_scene_batch_scratch_bytes(ctypes.byref(_cfg()))
    for kw in [dict(rgb_a=None), dict(rgb_b=None), dict(mask_a=None), dict(mask_b=None), dict(rand=False), dict(out=False),
               dict(scratch=None), dict(scratch_bytes=16), dict(scratch_bytes=need - 1)] + \
              [dict(rnull=k) for k in rand_keys] + [dict(onull=k) for k in out_keys]:
        assert call(**kw) == -1, kw
    assert N.launch_count() == before


TC = {"training": dict(cross_scene_num_samples=40, domain_randomize=True)}


def test_python_wrapper_refusals_and_cfg():
    B, H, W = 1, 8, 16
    rgb = torch.zeros(B, H, W, 3, dtype=torch.uint8); m = torch.zeros(B, H, W, dtype=torch.uint8)
    with pytest.raises(RuntimeError, match="CUDA"):
        S.across_scene_batch(rgb, rgb, m, m, TC)
    with pytest.raises(NotImplementedError):
        S.across_scene_batch(rgb, rgb, m, m, {"training": dict(TC["training"], debug=True)})
    for mt in (T.SINGLE_OBJECT_WITHIN_SCENE, T.MULTI_OBJECT, T.SYNTHETIC_MULTI_OBJECT, 7):
        with pytest.raises(ValueError, match="match_type"):
            S.across_scene_batch(rgb, rgb, m, m, TC, match_type=mt)
    with pytest.raises(RuntimeError, match="pairs per call"):
        S.across_scene_batch(torch.zeros(0, H, W, 3, dtype=torch.uint8), rgb, m, m, TC)
    assert S.across_scene_cfg(TC) == dict(num_samples=40, domain_randomize=True)
    full = {"training": dict(cross_scene_num_samples=10000, domain_randomize=False, num_matching_attempts=10000)}
    assert S.across_scene_cfg(full) == dict(num_samples=10000, domain_randomize=False)
