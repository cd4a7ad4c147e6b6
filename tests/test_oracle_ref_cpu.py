"""CPU: the oracle restatements are pinned against what the EXECUTED reference source computed (oracle/make_golden.py runs
the reference's own files -- oracle/build_ref.py: documented line-anchored py2->py3 patches -- on the cases of
oracle/ref_cases.py and stores the results in tests/golden/reference_checks.npz and tests/golden/loss_*.npz):

  * loss: values, hard-negative counts and autograd gradients of PixelwiseContrastiveLoss.* and loss_composer.*
    (dense_correspondence/loss_functions/pixelwise_contrastive_loss.py:35-411, loss_composer.py:7-218)
  * non-match sampler: create_non_correspondences + create_non_matches + flatten_uv_tensor
    (correspondence_tools/correspondence_finder.py:276-405, dataset/spartan_dataset_masked.py:841-858,1255-1264)
  * reprojection match finder: batch_find_pixel_correspondences (correspondence_finder.py:409-619)

The generator requires the restatement to equal the reference bit-for-bit; here integer results must match exactly and
floating-point ones to ~1 ulp, because a different CPU can reorder a vectorised fp32 reduction."""
import os

import numpy as np
import pytest
import torch

from oracle import loss_oracle as LO
from oracle import ref_cases as RC
from oracle.resnet34_8s_oracle import process_network_output


@pytest.fixture(scope="module")
def stored(golden_dir):
    return np.load(os.path.join(golden_dir, "reference_checks.npz"))


def assert_same_result(got, want, what, rtol=1e-6, atol=1e-7):
    assert got.shape == want.shape, what
    if np.issubdtype(want.dtype, np.floating):
        assert got.dtype == want.dtype, what
        np.testing.assert_allclose(got, want, rtol=rtol, atol=atol, err_msg=what)
    else:
        assert np.array_equal(got, want), what


def _golden_case(golden_dir, name):
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    cfg = dict(LO.DEFAULT_LOSS_CONFIG)
    for k, v in zip(g["cfg_keys"], g["cfg_vals"]):
        k = str(k)
        cfg[k] = bool(v) if isinstance(LO.DEFAULT_LOSS_CONFIG[k], bool) else float(v)
    idx = {k: torch.tensor(g[k]) for k in ("matches_a", "matches_b", "masked_a", "masked_b", "background_a", "background_b",
                                           "blind_a", "blind_b")}
    return g, cfg, idx


def _run(pcl, get_loss, A, B, idx, match_type=0):
    A = A.clone().requires_grad_(); B = B.clone().requires_grad_()
    _, D, H, W = A.shape
    pa = process_network_output(A, 1, D, H, W); pb = process_network_output(B, 1, D, H, W)
    five = get_loss(pcl, torch.tensor([match_type]), pa, pb, idx["matches_a"], idx["matches_b"], idx["masked_a"], idx["masked_b"],
                    idx["background_a"], idx["background_b"], idx["blind_a"], idx["blind_b"])
    five[0].reshape(()).backward()
    return [float(t) for t in five], A.grad, B.grad


@pytest.mark.parametrize("name", ["loss_default_d3", "loss_pixelw_blind_d8", "loss_noscale_d16"])
def test_composed_loss_restatement_equals_executed_reference(golden_dir, name):
    # the committed goldens ARE the executed reference's outputs (oracle/make_golden.py writes them from it)
    g, cfg, idx = _golden_case(golden_dir, name)
    A, B = torch.tensor(g["A"]), torch.tensor(g["B"])
    _, D, H, W = A.shape
    five_o, dA_o, dB_o = _run(LO.TorchPixelwiseContrastiveLoss([H, W], dict(cfg)), LO.get_loss, A, B, idx)
    np.testing.assert_allclose(five_o, g["five"], rtol=1e-6, atol=1e-8)
    np.testing.assert_allclose(dA_o.numpy(), g["dA"], rtol=1e-5, atol=1e-8)
    np.testing.assert_allclose(dB_o.numpy(), g["dB"], rtol=1e-5, atol=1e-8)


def test_every_loss_method_equals_executed_reference(stored):
    got = RC.every_loss_method(LO.TorchPixelwiseContrastiveLoss)
    want = {k[len("method/"):]: stored[k] for k in stored.files if k.startswith("method/")}
    assert sorted(got) == sorted(want)
    for k in want:
        assert_same_result(got[k], want[k], k)


def test_composer_branches_equal_executed_reference(stored):
    """every configuration x match type, the blind sentinel [-1] (not entered), max(h, 1), and the reference's own
    NameError (across-scene) / ValueError (unknown type)."""
    got = RC.composer_branches(LO.TorchPixelwiseContrastiveLoss, LO.get_loss, LO.empty_tensor)
    want = {k[len("composer/"):]: stored[k] for k in stored.files if k.startswith("composer/")}
    assert sorted(got) == sorted(want)
    for k in want:
        assert_same_result(got[k], want[k], k)
    assert float(got["sentinel/five"][4]) == 0.0
    assert str(want["raises/across_scene"]) in ("NameError", "UnboundLocalError") and str(want["raises/unknown"]) == "ValueError"
    T = LO.SpartanDatasetDataType
    types = [k for k in stored.files if k.startswith("datatype/")]
    assert types and all(getattr(T, k[len("datatype/"):]) == int(stored[k]) for k in types)


def test_non_match_sampler_restatement_equals_executed_reference(stored):
    """The reference sampler was given the same uniform numbers the restatement takes as arguments."""
    H, W, k, ma, ru, rv, masks = RC.sampler_inputs()
    for i, m in enumerate(masks):
        na_o, nb_o = LO.create_non_correspondences_flat(ma, (H, W), k, m, ru, rv)
        assert_same_result(na_o.numpy(), stored["sampler/%d/a" % i], "sampler %d a" % i)
        assert_same_result(nb_o.numpy(), stored["sampler/%d/b" % i], "sampler %d b" % i)
        if i == 0:
            assert bool((m.view(-1)[nb_o] == 1).all())


def test_reprojection_restatement_equals_executed_reference(stored):
    da, pa, db, pb, mask, ru, K, n = RC.reprojection_scene()
    # the candidates random_sample_from_masked_image_torch drew (correspondence_finder.py:92-121)
    nz = torch.nonzero(torch.from_numpy(mask).view(-1))
    cand = torch.index_select(nz, 0, torch.floor(ru * len(nz)).long()).squeeze(1)
    uv_a_o, uv_b_o = LO.batch_find_pixel_correspondences(da, pa, db, pb, cand, K)
    assert len(stored["reprojection/0"]) > 0.3 * n and len(stored["reprojection/0"]) < n      # some pruned by every rule
    for i, t in enumerate(uv_a_o + uv_b_o):
        assert_same_result(t.numpy(), stored["reprojection/%d" % i], "reprojection %d" % i)
