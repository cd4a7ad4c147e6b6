"""CPU: descriptor statistics and the across-object best match (csrc/descriptor_stats.cu, csrc/match_stats.cu,
pdc_b200.evaluation) -- the float64 oracle against the executed reference's fixture, the reference's fold quirks, the
descriptor_statistics.yaml round trip through descriptor_image_stats, and every refusal before a launch."""
import ctypes
import importlib
import os
import sys

import numpy as np
import pytest
import torch
import yaml

import pdc_b200
from pdc_b200 import _native as N
from pdc_b200 import evaluation as E
from oracle import descriptor_stats_oracle as DO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "descriptor_statistics.npz")
KEYS = ("entire_image", "mask_image")
FIELDS = ("min", "max", "mean")


def _golden():
    return np.load(GOLDEN)


def _reference(g, D):
    return {k: {f: g["stats_d%d/%s/%s" % (D, k, f)] for f in FIELDS} for k in KEYS}


def _torch_per_image(res, masks):
    """compute_descriptor_statistics (evaluation.py:2177-2219) in torch float32, image by image, as the reference
    computes it -> the per-image dict descriptor_statistics returns."""
    n, D = res.shape[0], res.shape[-1]
    out = {k: np.full((n, D), np.nan, np.float32) for k in E.STAT_KEYS}
    out["mask_count"] = np.zeros(n, np.int64)
    for i in range(n):
        flat = torch.from_numpy(res[i]).contiguous().view(-1, D)
        out["min"][i] = flat.min(0)[0].numpy(); out["max"][i] = flat.max(0)[0].numpy(); out["mean"][i] = flat.mean(0).numpy()
        idx = torch.nonzero(torch.from_numpy(masks[i].reshape(-1).astype(np.float32))).squeeze(1)
        out["mask_count"][i] = idx.numel()
        if idx.numel():
            m = flat.index_select(0, idx)
            out["mask_min"][i] = m.min(0)[0].numpy(); out["mask_max"][i] = m.max(0)[0].numpy()
            out["mask_mean"][i] = m.mean(0).numpy()
    return out


@pytest.mark.parametrize("D", [3, 16])
def test_float64_oracle_matches_executed_reference(D):
    g = _golden()
    res, masks = g["res_d%d" % D], g["mask_d%d" % D]
    assert (masks.reshape(len(masks), -1).sum(1) == 0).sum() == 1            # one image is skipped
    got = DO.fold([DO.per_image(r, m) for r, m in zip(res, masks)], len(res))
    ref = _reference(g, D)
    for k in KEYS:
        assert np.array_equal(got[k]["min"], ref[k]["min"]) and np.array_equal(got[k]["max"], ref[k]["max"]), k
        # the reference's means are float32 torch means; the oracle's are float64
        np.testing.assert_allclose(got[k]["mean"], ref[k]["mean"], rtol=1e-6, atol=1e-7)


@pytest.mark.parametrize("D", [3, 16])
def test_fold_is_the_references_bit_for_bit(D):
    """fold_descriptor_statistics on the reference's own per-image float32 statistics gives the fixture exactly: the
    skipped image, the float32 running sum and the 1/num_images factor are the reference's."""
    g = _golden()
    got = E.fold_descriptor_statistics(_torch_per_image(g["res_d%d" % D], g["mask_d%d" % D]))
    ref = _reference(g, D)
    for k in KEYS:
        for f in FIELDS:
            assert isinstance(got[k][f], list) and all(type(x) is float for x in got[k][f])
            assert np.array_equal(np.array(got[k][f]), ref[k][f]), (k, f)


def test_fold_quirks():
    D = 2
    per = {k: np.zeros((3, D), np.float32) for k in E.STAT_KEYS}
    per["min"][:] = [[0, 0], [-9, -9], [1, 1]]          # image 1 holds the global minimum but its mask is empty
    per["max"][:] = [[1, 1], [9, 9], [2, 2]]
    per["mean"][:] = [[1, 2], [100, 100], [3, 4]]
    per["mask_min"][:] = [[0.5, 0.5], [np.nan, np.nan], [1.5, 1.5]]
    per["mask_max"][:] = [[0.7, 0.7], [np.nan, np.nan], [1.7, 1.7]]
    per["mask_mean"][:] = [[0.6, 0.6], [np.nan, np.nan], [1.6, 1.6]]
    per["mask_count"] = np.array([4, 0, 5])
    s = E.fold_descriptor_statistics(per)
    assert s["entire_image"]["min"] == [0.0, 0.0] and s["entire_image"]["max"] == [2.0, 2.0]      # skipped for both keys
    assert s["mask_image"]["min"] == [0.5, 0.5] and s["mask_image"]["max"] == [float(np.float32(1.7))] * 2
    third = np.float32(1.0 / 3)
    assert s["entire_image"]["mean"] == [float(third * np.float32(4)), float(third * np.float32(6))]   # / 3, not / 2
    assert s["mask_image"]["mean"] == [float(third * (np.float32(0.6) + np.float32(1.6)))] * 2
    assert E.fold_descriptor_statistics(per, num_images=10)["entire_image"]["mean"][0] == float(np.float32(0.1) * np.float32(4))
    per["mask_count"] = np.zeros(3, np.int64)
    with pytest.raises(TypeError):
        E.fold_descriptor_statistics(per)


def test_yaml_round_trip_through_descriptor_image_stats(tmp_path):
    g = _golden()
    stats = E.fold_descriptor_statistics(_torch_per_image(g["res_d3"], g["mask_d3"]))
    E.save_descriptor_statistics(stats, str(tmp_path / "descriptor_statistics.yaml"))
    dcn = pdc_b200.DenseCorrespondenceNetwork(None, 3)
    dcn.config = {"path_to_network_params_folder": str(tmp_path)}
    loaded = dcn.descriptor_image_stats
    assert loaded == stats
    assert set(loaded) == set(KEYS) and all(set(loaded[k]) == set(FIELDS) for k in KEYS)
    assert dcn.descriptor_image_stats is loaded                  # loaded once, as net.py:148 does
    # the reference's reader (utils.getDictFromYamlFilename: yaml.load with the C loader) reads the same values
    loader = getattr(yaml, "CLoader", yaml.FullLoader)
    with open(str(tmp_path / "descriptor_statistics.yaml")) as f:
        assert yaml.load(f, Loader=loader) == stats
    with pytest.raises(ValueError):
        pdc_b200.DenseCorrespondenceNetwork(None, 3).descriptor_image_stats         # no parameter folder configured


@pytest.mark.parametrize("D", [3, 16])
def test_best_match_oracle_matches_executed_reference(D):
    g = _golden()
    ra, rb = g["bm_res_a_d%d" % D], g["bm_res_b_d%d" % D]
    for i, uv in enumerate(g["bm_uv_a_d%d" % D]):
        uv_b, diff = DO.best_match(uv, ra, rb)
        assert uv_b == tuple(g["bm_uv_b_d%d" % D][i]) and np.float32(diff).tobytes() == g["bm_diff_d%d" % D][i].tobytes()
    assert tuple(g["bm_uv_b_d%d" % D][0]) == (15, 3) and g["bm_diff_d%d" % D][0] == 0        # tie at 0: the first pixel
    assert tuple(g["bm_uv_b_d%d" % D][1]) == (7, 5)                                          # tie above 0: the first pixel


def test_descriptor_statistics_refusals_launch_nothing():
    fake = ctypes.c_void_p(1 << 40)
    good = (ctypes.c_int64 * 4)(64 * 96 * 3, 96 * 3, 3, 1)

    def call(N_=2, H=64, W=96, D=3, s=good, res=fake, mask=fake, dtype=0, out=fake, count=fake, scratch=fake, nbytes=1 << 40):
        return N.lib.ddn_descriptor_statistics(res, s, N_, H, W, D, mask, dtype, out, count, scratch, nbytes, None)

    before = N.launch_count()
    assert N.lib.ddn_descriptor_statistics_scratch_bytes(2, 64, 96, 3) > 0
    for bad in ((0, 64, 96, 3), (1, 0, 96, 3), (1, 64, 96, 0), (1, 64, 96, 33), (1, 1 << 16, 1 << 15, 3), (70000, 4, 4, 3)):
        assert N.lib.ddn_descriptor_statistics_scratch_bytes(*bad) == 0, bad
    for kw in (dict(res=None), dict(mask=None), dict(out=None), dict(count=None), dict(scratch=None), dict(s=None),
               dict(D=0), dict(D=33), dict(N_=0), dict(N_=70000), dict(H=0), dict(W=-1), dict(H=1 << 16, W=1 << 15),
               dict(dtype=2), dict(s=(ctypes.c_int64 * 4)(-1, 1, 1, 1)), dict(s=(ctypes.c_int64 * 4)(1 << 41, 1, 1, 1)),
               dict(s=(ctypes.c_int64 * 4)(1 << 39, 1 << 39, 1, 1)), dict(nbytes=16)):
        assert call(**kw) == -1, kw
    assert N.launch_count() == before


def test_best_match_batch_refusals_launch_nothing():
    fake = ctypes.c_void_p(1 << 40)
    good = (ctypes.c_int64 * 4)(64 * 96 * 3, 96 * 3, 3, 1)

    def call(N_=1, H=64, W=96, D=3, Q=10, sa=good, sb=good, res_a=fake, pair=fake, uv=fake, bad=fake, nbytes=1 << 40):
        return N.lib.ddn_best_match_batch(res_a, sa, fake, sb, N_, H, W, D, pair, fake, Q, uv, fake, bad, fake, nbytes, None)

    before = N.launch_count()
    assert N.lib.ddn_best_match_batch_scratch_bytes(10) > 0
    assert N.lib.ddn_best_match_batch_scratch_bytes(0) == 0
    assert N.lib.ddn_best_match_batch_scratch_bytes(65535 * 8 + 1) == 0
    for kw in (dict(res_a=None), dict(pair=None), dict(uv=None), dict(bad=None), dict(sa=None), dict(D=0), dict(D=33),
               dict(N_=0), dict(Q=0), dict(Q=65535 * 8 + 1), dict(H=0), dict(W=-1), dict(H=1 << 16, W=1 << 15),
               dict(sa=(ctypes.c_int64 * 4)(-1, 1, 1, 1)), dict(sb=(ctypes.c_int64 * 4)(1 << 41, 1, 1, 1)), dict(nbytes=16)):
        assert call(**kw) == -1, kw
    assert N.launch_count() == before


def test_python_wrappers_refuse_cpu_tensors():
    """(wrong shapes and dtypes of CUDA tensors: tests/test_gpu_descriptor_statistics.py)"""
    res = torch.zeros(2, 8, 12, 3)
    mask = torch.ones(2, 8, 12)
    with pytest.raises(RuntimeError, match="CUDA"):
        E.descriptor_statistics(res, mask)
    with pytest.raises(RuntimeError, match="CUDA"):
        E.best_match_batch(res, res, torch.zeros(1, 2, dtype=torch.int64), torch.zeros(1, dtype=torch.int64))
    with pytest.raises(RuntimeError, match="CUDA"):
        E.across_object_analysis(res, res, mask)
    with pytest.raises(ValueError):
        E.descriptor_statistics_over_images(None, torch.zeros(2, 3, 8, 12), torch.ones(3, 8, 12))


def test_compat_import_path_resolves():
    compat = os.path.join(ROOT, "pytorch-dense-correspondence_b200", "compat")
    saved = {k: v for k, v in sys.modules.items() if k.split(".")[0] == "dense_correspondence"}
    for k in saved:
        del sys.modules[k]
    sys.path.insert(0, compat)
    try:
        mod = importlib.import_module("dense_correspondence.evaluation.evaluation")
        assert mod.descriptor_statistics is pdc_b200.descriptor_statistics
        assert mod.across_object_analysis is pdc_b200.across_object_analysis
        assert mod.DCNEvaluationPandaTemplateAcrossObject.columns[-1] == "norm_diff_descriptor_best_match"
    finally:
        sys.path.remove(compat)
        for k in [k for k in sys.modules if k.split(".")[0] == "dense_correspondence"]:
            del sys.modules[k]
        sys.modules.update(saved)
