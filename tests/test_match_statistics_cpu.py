"""CPU: the per-match evaluation statistics (csrc/match_stats.cu, pdc_b200.evaluation) -- the summation order the kernel
restates, the float64 oracle against the executed reference's fixture, and every refusal before a launch."""
import ctypes
import importlib
import os
import sys

import numpy as np
import pytest
import torch

import pdc_b200
from pdc_b200 import _native as N
from pdc_b200 import evaluation as E
from oracle import match_stats_oracle as MO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "match_statistics.npz")


@pytest.mark.parametrize("D", list(range(1, 33)))
def test_pairwise_order_is_numpys_sum(D):
    """The order csrc/match_stats.cu uses (MO.pairwise_sum_last_axis) is bit-equal to np.sum(..., axis=2) on a contiguous
    [H,W,D] float32 array, i.e. to find_best_match's norm_diffs on the reference's contiguous host copy."""
    rng = np.random.default_rng(D)
    res_b = rng.standard_normal((37, 53, D)).astype(np.float32) * np.float32(3.0)
    q = rng.standard_normal(D).astype(np.float32)
    sq = np.square(res_b - q)
    assert np.array_equal(np.sum(sq, axis=2), MO.pairwise_sum_last_axis(sq))


def _golden():
    return np.load(GOLDEN)


@pytest.mark.parametrize("D", [3, 9])
def test_oracle_matches_executed_reference(D):
    g = _golden()
    ra = g["res_a_d%d" % D].astype(np.float32); rb = g["res_b_d%d" % D].astype(np.float32)
    uv_a = g["uv_a_d%d" % D]; uv_b = g["uv_b_d%d" % D]
    for n in range(3):
        raised = g["out_d%d_p%d/raised" % (D, n)]
        for i in range(len(uv_a)):
            args = (g["depth_a"], g["depth_b"], g["mask_b"][n], tuple(uv_a[i]), tuple(uv_b[i]), g["pose_a"], g["pose_b"], ra, rb, g["K"])
            if raised[i]:
                with pytest.raises(ZeroDivisionError):
                    MO.one_match(*args)
                continue
            o = MO.one_match(*args, threshold="reference")
            for c in E.F32_COLUMNS + E.F64_COLUMNS + ["is_valid", "is_valid_masked"]:
                ref = g["out_d%d_p%d/%s" % (D, n, c)][i]
                got = np.array(o[c], dtype=ref.dtype)
                assert np.array_equal(got, ref, equal_nan=True), (D, n, i, c, got, ref)
            # on exact-grid descriptors the device's threshold is the reference's
            assert MO.one_match(*args, threshold="device")["norm_diff_descriptor_ground_truth"] == o["norm_diff_descriptor_ground_truth"]


def test_golden_covers_the_edge_cases():
    g = _golden()
    for D in (3, 9):
        uv_b = g["uv_b_d%d" % D]
        assert tuple(uv_b[0]) == (95, 63)                                              # clipped to the last column / row
        assert np.isnan(g["out_d%d_p0/norm_diff_ground_truth_3d" % D][1])             # invalid depth at uv_b
        assert g["mask_b"][0][uv_b[2][1], uv_b[2][0]] == 0                             # ground truth outside the mask
        assert (g["out_d%d_p2/raised" % D] == "ZeroDivisionError").all()              # empty mask
        assert g["mask_b"][1].all()                                                    # full mask
    assert (g["out_d9_p0/is_valid"] == 0).any()                                        # invalid depth at the prediction


def test_match_statistics_refusals_launch_nothing():
    fake = ctypes.c_void_p(1 << 40)
    big = 1 << 40
    good = (ctypes.c_int64 * 4)(64 * 96 * 3, 96 * 3, 3, 1)
    kinv = (ctypes.c_double * 9)(); poses = (ctypes.c_double * 32)()

    def call(N_=1, H=64, W=96, D=3, Q=10, sa=good, sb=good, res_a=fake, pair=fake, K=kinv, pa=poses, scratch_bytes=big, bad=fake):
        return N.lib.ddn_match_statistics(res_a, sa, fake, sb, N_, H, W, D, pair, fake, fake, Q, fake, fake, fake, K, pa, poses,
                                          fake, fake, fake, bad, fake, scratch_bytes, None)

    before = N.launch_count()
    assert N.lib.ddn_match_statistics_scratch_bytes(1, 64, 96, 10) > 0
    assert N.lib.ddn_match_statistics_scratch_bytes(0, 64, 96, 10) == 0
    assert N.lib.ddn_match_statistics_scratch_bytes(1, 1 << 16, 1 << 15, 10) == 0      # H*W >= 2^31
    assert N.lib.ddn_match_statistics_scratch_bytes(1, 64, 96, 0) == 0
    for kw in (dict(res_a=None), dict(pair=None), dict(K=None), dict(pa=None), dict(bad=None), dict(sa=None),
               dict(D=0), dict(D=33), dict(N_=0), dict(N_=70000), dict(Q=0), dict(Q=1 << 23), dict(H=0), dict(W=-1),
               dict(H=1 << 16, W=1 << 15), dict(sa=(ctypes.c_int64 * 4)(-1, 1, 1, 1)), dict(sb=(ctypes.c_int64 * 4)(1 << 41, 1, 1, 1)),
               dict(scratch_bytes=16)):
        assert call(**kw) == -1, kw
    assert N.launch_count() == before


def test_python_wrapper_refuses_cpu_tensors():
    """(wrong dtypes and shapes of CUDA tensors: tests/test_gpu_match_statistics.py)"""
    H, W, D = 8, 12, 3
    cpu = torch.zeros(H, W, D)
    pose = np.eye(4)[None]
    with pytest.raises(RuntimeError, match="CUDA"):
        E.match_statistics(cpu, cpu, torch.zeros(1, 2, dtype=torch.int64), torch.zeros(1, 2, dtype=torch.int64),
                           torch.zeros(1, dtype=torch.int64), torch.ones(H, W), torch.ones(H, W), torch.ones(H, W), pose, pose, np.eye(3))
    with pytest.raises(RuntimeError, match="CUDA"):
        E.match_statistics(cpu.double(), cpu.double(), None, None, None, None, None, None, pose, pose, np.eye(3))
    with pytest.raises(NotImplementedError):
        E.DenseCorrespondenceEvaluation.compute_descriptor_match_statistics(None, None, None, None, (0, 0), (0, 0), None, None,
                                                                            None, None, None, debug=True)


def test_reference_helpers():
    DCE = E.DenseCorrespondenceEvaluation
    assert DCE.clip_pixel_to_image_size_and_round((95.6, 10.4), 96, 64) == (95, 10)
    assert DCE.clip_pixel_to_image_size_and_round((2.5, 63.9), 96, 64) == (2, 63)
    assert DCE.is_depth_valid(0.5) and not DCE.is_depth_valid(0.0) and not DCE.is_depth_valid(10.0)
    g = _golden()
    for uv, z in (((3, 7), 1.234), ((95, 0), 0.0)):
        assert np.array_equal(DCE.compute_3d_position(uv, z, g["K"], g["pose_b"]), MO.compute_3d_position(uv, z, g["K"], g["pose_b"]))


def test_compat_import_path_resolves():
    compat = os.path.join(ROOT, "pytorch-dense-correspondence_b200", "compat")
    saved = {k: v for k, v in sys.modules.items() if k.split(".")[0] == "dense_correspondence"}
    for k in saved:
        del sys.modules[k]
    sys.path.insert(0, compat)
    try:
        mod = importlib.import_module("dense_correspondence.evaluation.evaluation")
        assert mod.DenseCorrespondenceEvaluation is pdc_b200.DenseCorrespondenceEvaluation
        assert mod.match_statistics is pdc_b200.match_statistics
    finally:
        sys.path.remove(compat)
        for k in [k for k in sys.modules if k.split(".")[0] == "dense_correspondence"]:
            del sys.modules[k]
        sys.modules.update(saved)
