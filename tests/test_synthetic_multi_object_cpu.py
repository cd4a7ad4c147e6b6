"""CPU: the synthetic multi-object batch producer's oracle and C ABI refusals.

* oracle/synthetic_multi_object_oracle.py's restatement (merges, occlusion pruning, merge_matches, non-matches) reproduces,
  bit for bit, what the executed reference computed for every case of oracle/make_golden_synthetic.py
  (tests/golden/synthetic_multi_object_batch.npz), including which of the four early returns a pair takes;
* ddn_synthetic_multi_object_batch refuses every malformed argument with -1 before launching anything;
* the Python wrapper refuses CPU tensors and debug=True.
(The device results: tests/test_gpu_synthetic_multi_object.py.)"""
import ctypes
import os

import numpy as np
import pytest
import torch

import pdc_b200  # noqa: F401
from pdc_b200 import _native as N
from pdc_b200 import sampling as S
from oracle import make_golden_synthetic as MG
from oracle import synthetic_multi_object_oracle as SO

NAMES = [c[0] for c in MG.CASES]


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "synthetic_multi_object_batch.npz"))


@pytest.mark.parametrize("case", NAMES)
def test_restatement_equals_executed_reference(golden, case):
    r = MG.run_case(SO.RESTATED, NAMES.index(case))
    assert bool(golden[case + "/empty"]) == r["empty"] and str(golden[case + "/ret"]) == r["ret"]
    if not r["empty"]:
        assert r["python_left"] == 0 and r["torch_left"] == 0
    for k in MG.KEYS:
        np.testing.assert_array_equal(r[k], golden["%s/%s" % (case, k)].astype(r[k].dtype), err_msg=k)


def test_golden_covers_the_cases(golden):
    rets = {c: str(golden[c + "/ret"]) for c in NAMES}
    assert rets["empty_mask_a1"] == "a1" and rets["empty_mask_b1"] == "b1"
    assert rets["occluded_after_merge_1"] == "occluded_1" and rets["occluded_after_merge_2"] == "occluded_2"
    merged = [c for c in NAMES if rets[c] == "merged"]
    assert {MG.CASES[NAMES.index(c)][1] for c in merged} == {(0, 0), (0, 1), (1, 0), (1, 1)}
    A, B, _, _, _ = MG.case_inputs(NAMES.index("fg_a_fg_a_mask_255_wrap"))
    assert ((A["mask_2"].astype(int) + B["mask_2"]) == 256).any()          # the uint8 sum wraps to 0
    # pruning removes some matches: fewer than the two halves' reprojection survivors
    for c in merged:
        assert 0 < len(golden[c + "/matches_a"]) < 2 * MG.CFG["n_attempts"]


def _cfg(**kw):
    c = dict(B=2, H=32, W=48, sample_matches_only_off_mask=1, use_image_b_mask_inv=1, n_attempts=200, k_masked=3,
             k_background=2, mean=(ctypes.c_float * 3)(0.5, 0.4, 0.4), std=(ctypes.c_float * 3)(0.2, 0.3, 0.3))
    c.update(kw)
    return N.SmoBatchCfg(**c)


def test_synthetic_batch_refusals_launch_nothing():
    fake = 1 << 40
    K = (ctypes.c_double * 9)(100.0, 0, 20, 0, 100.0, 15, 0, 0, 1)
    poses = (ctypes.c_double * (16 * 2 * 64))(*([1.0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 1.0] * 128))
    singular = (ctypes.c_double * 9)()
    rand_keys = [f for f, _ in N.SmoBatchRand._fields_]
    out_keys = [f for f, _ in N.SmoBatchOut._fields_]

    def call(cfg=None, ins=fake, K=K, pa=poses, scratch=fake, scratch_bytes=1 << 40, rnull=None, onull=None):
        cfg = cfg if cfg is not None else _cfg()
        r = N.SmoBatchRand(**{k: (None if k == rnull else fake) for k in rand_keys})
        o = N.SmoBatchOut(**{k: (None if k == onull else fake) for k in out_keys})
        return N.lib.ddn_synthetic_multi_object_batch(ctypes.byref(cfg) if cfg is not False else None, fake, fake, ins, fake,
                                                      fake, fake, K, pa, poses, ctypes.byref(r), ctypes.byref(o), scratch,
                                                      scratch_bytes, None)

    before = N.launch_count()
    assert N.SMO_MAX_PAIRS == N.WS_MAX_PAIRS // 2 == 64
    assert N.lib.ddn_synthetic_multi_object_batch_scratch_bytes(ctypes.byref(_cfg(B=64))) > 0
    bad = [_cfg(B=0), _cfg(B=N.SMO_MAX_PAIRS + 1), _cfg(H=0), _cfg(W=-3), _cfg(H=1 << 15, W=1 << 15), _cfg(n_attempts=0),
           _cfg(n_attempts=1 << 29), _cfg(k_masked=-1), _cfg(k_background=-1), _cfg(k_masked=1 << 25),
           _cfg(sample_matches_only_off_mask=2), _cfg(use_image_b_mask_inv=-1),
           _cfg(std=(ctypes.c_float * 3)(0.2, 0.0, 0.3)), _cfg(mean=(ctypes.c_float * 3)(float("nan"), 0, 0))]
    for c in bad:
        assert N.lib.ddn_synthetic_multi_object_batch_scratch_bytes(ctypes.byref(c)) == 0
        assert call(cfg=c) == -1
    assert N.lib.ddn_synthetic_multi_object_batch_scratch_bytes(None) == 0
    assert call(cfg=False) == -1
    need = N.lib.ddn_synthetic_multi_object_batch_scratch_bytes(ctypes.byref(_cfg()))
    for kw in [dict(ins=None), dict(K=None), dict(pa=None), dict(K=singular), dict(scratch=None), dict(scratch_bytes=need - 1)] + \
              [dict(rnull=k) for k in rand_keys] + [dict(onull=k) for k in out_keys]:
        assert call(**kw) == -1, kw
    assert N.launch_count() == before


def test_python_wrapper_refusals():
    B, H, W = 1, 8, 16
    cfg = {"training": dict(num_matching_attempts=10, num_non_matches_per_match=4, fraction_masked_non_matches=0.5,
                            fraction_background_non_matches=0.5, sample_matches_only_off_mask=True, domain_randomize=False,
                            use_image_b_mask_inv=True)}
    rgb = torch.zeros(B, H, W, 3, dtype=torch.uint8); m = torch.zeros(B, H, W, dtype=torch.uint8); d = torch.zeros(B, H, W)
    pose = np.eye(4)[None]
    scene = (rgb, rgb, d, d, m, m, pose, pose)
    with pytest.raises(RuntimeError, match="CUDA"):
        S.synthetic_multi_object_batch(scene, scene, np.eye(3), cfg)
    with pytest.raises(NotImplementedError):
        S.synthetic_multi_object_batch(scene, scene, np.eye(3), {"training": dict(cfg["training"], debug=True)})
    with pytest.raises(RuntimeError, match="pairs per call"):
        big = (torch.zeros(65, H, W, 3, dtype=torch.uint8),) + scene[1:]
        S.synthetic_multi_object_batch(big, scene, np.eye(3), cfg)
