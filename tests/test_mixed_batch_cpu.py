"""CPU: mixed pair-type batches -- the refusals of ddn_pair_type_compose (before any launch), sampling.draw_data_types
(the reference's per-sample type rule), the host-side checks of loss_composer.get_mixed_loss, which raise before
anything touches CUDA, and sampling.concat_batches' refusal of a match_type that is not on the host."""
import ctypes

import numpy as np
import pytest
import torch

import pdc_b200
from pdc_b200 import _native as N
from pdc_b200 import loss_composer
from pdc_b200 import sampling as S
from pdc_b200.loss_composer import SpartanDatasetDataType as T
from oracle import loss_oracle as LO

PROBS = dict(SINGLE_OBJECT_WITHIN_SCENE=0.0, SINGLE_OBJECT_ACROSS_SCENE=0.0, DIFFERENT_OBJECT=0.0, MULTI_OBJECT=0.0,
             SYNTHETIC_MULTI_OBJECT=0.0)


def config(**p):
    return {"training": {"data_type_probabilities": dict(PROBS, **p)}}


def test_compose_refusals_launch_nothing():
    fake = ctypes.c_void_p(1 << 40)       # never dereferenced: every refusal happens on the host
    cfg = N.PairTypeComposeCfg(1.0, 1.0, 1, 1, 10, 20, 20, 30)
    before = N.launch_count()
    f = N.lib.ddn_pair_type_compose
    assert f(None, fake, 2, 5, ctypes.byref(cfg), fake, fake, fake, None) == -1
    assert f(fake, None, 2, 5, ctypes.byref(cfg), fake, fake, fake, None) == -1
    assert f(fake, fake, 2, 5, None, fake, fake, fake, None) == -1
    assert f(fake, fake, 2, 5, ctypes.byref(cfg), None, fake, fake, None) == -1
    assert f(fake, fake, 2, 5, ctypes.byref(cfg), fake, None, fake, None) == -1
    assert f(fake, fake, 2, 5, ctypes.byref(cfg), fake, fake, None, None) == -1
    assert b"null" in N.lib.ddn_last_error()
    for n_terms in (3, 4, 6):
        assert f(fake, fake, 2, n_terms, ctypes.byref(cfg), fake, fake, fake, None) == -1
    for B in (0, -1):
        assert f(fake, fake, B, 5, ctypes.byref(cfg), fake, fake, fake, None) == -1
    assert b"5 terms" in N.lib.ddn_last_error()
    assert N.launch_count() == before


def test_draw_data_types_order_and_zero_probabilities():
    g = torch.Generator().manual_seed(0)
    t = S.draw_data_types(2000, config(SYNTHETIC_MULTI_OBJECT=1.0, SINGLE_OBJECT_WITHIN_SCENE=1.0, DIFFERENT_OBJECT=1.0), g)
    assert t.dtype == torch.int64 and t.device.type == "cpu" and t.shape == (2000,)
    assert set(t.tolist()) == {T.SINGLE_OBJECT_WITHIN_SCENE, T.DIFFERENT_OBJECT, T.SYNTHETIC_MULTI_OBJECT}
    # the types are listed in the reference's order and picked by the first cumulative probability above u
    u = torch.rand(2000, dtype=torch.float64, generator=torch.Generator().manual_seed(0))
    cdf = np.cumsum([1.0, 1.0, 1.0])
    ref = np.array([T.SINGLE_OBJECT_WITHIN_SCENE, T.DIFFERENT_OBJECT, T.SYNTHETIC_MULTI_OBJECT])[
        np.minimum(np.searchsorted(cdf / cdf[-1], u.numpy(), side="right"), 2)]
    assert t.tolist() == ref.tolist()
    assert set(S.draw_data_types(500, config(MULTI_OBJECT=0.2), g).tolist()) == {T.MULTI_OBJECT}


def test_draw_data_types_normalises_the_probabilities():
    n = 100000
    t = S.draw_data_types(n, config(SINGLE_OBJECT_WITHIN_SCENE=1.0, DIFFERENT_OBJECT=3.0), torch.Generator().manual_seed(4))
    for typ, p in ((T.SINGLE_OBJECT_WITHIN_SCENE, 0.25), (T.DIFFERENT_OBJECT, 0.75)):
        frac = float((t == typ).double().mean())
        assert abs(frac - p) <= 3 * (p * (1 - p) / n) ** 0.5, (typ, frac)
    shoes = S.draw_data_types(n, config(SINGLE_OBJECT_WITHIN_SCENE=1 / 3.0, DIFFERENT_OBJECT=1 / 3.0,
                                        SYNTHETIC_MULTI_OBJECT=1 / 3.0), torch.Generator().manual_seed(5))
    for typ in (T.SINGLE_OBJECT_WITHIN_SCENE, T.DIFFERENT_OBJECT, T.SYNTHETIC_MULTI_OBJECT):
        assert abs(float((shoes == typ).double().mean()) - 1 / 3.0) <= 3 * (2 / 9.0 / n) ** 0.5


def test_draw_data_types_is_deterministic_under_a_seed():
    tc = config(SINGLE_OBJECT_WITHIN_SCENE=0.75, DIFFERENT_OBJECT=0.25)
    a = S.draw_data_types(64, tc, torch.Generator().manual_seed(123))
    b = S.draw_data_types(64, tc, torch.Generator().manual_seed(123))
    c = S.draw_data_types(64, tc, torch.Generator().manual_seed(124))
    assert torch.equal(a, b) and not torch.equal(a, c)


@pytest.mark.parametrize("tc", [
    config(),                                                          # every probability 0
    config(SINGLE_OBJECT_WITHIN_SCENE=1.0, DIFFERENT_OBJECT=-0.5),     # negative
    config(SINGLE_OBJECT_WITHIN_SCENE=float("nan")),
    {"training": {"data_type_probabilities": {k: 1.0 for k in list(PROBS)[:4]}}},   # a missing key
    {"training": {}},
], ids=["all_zero", "negative", "nan", "missing_key", "no_section"])
def test_draw_data_types_refusals(tc):
    with pytest.raises(ValueError):
        S.draw_data_types(4, tc)


def test_draw_data_types_refuses_bad_sizes():
    tc = config(SINGLE_OBJECT_WITHIN_SCENE=1.0)
    for B in (0, -2, 2.0, True):
        with pytest.raises(ValueError):
            S.draw_data_types(B, tc)


def _mixed_loss(match_type):
    e = loss_composer.empty_tensor()
    pcl = pdc_b200.PixelwiseContrastiveLoss([4, 6], dict(LO.DEFAULT_LOSS_CONFIG))
    return loss_composer.get_mixed_loss(pcl, match_type, None, None, e, e, e, e, e, e, e, e, num_valid=None)


@pytest.mark.parametrize("match_type", [[0, 7], [5], [-1, 0], [0, 2, 3, 4, 9]])
def test_get_mixed_loss_refuses_unknown_types_on_the_host(match_type):
    with pytest.raises(ValueError, match="Should only have above scenes"):
        _mixed_loss(torch.tensor(match_type))


@pytest.mark.parametrize("match_type", [[1], [0, 1, 2], [2, 2, 1]])
def test_get_mixed_loss_single_object_across_scene_reaches_the_reference_name_error(match_type):
    with pytest.raises(NameError, match="name 'pcl' is not defined"):
        _mixed_loss(torch.tensor(match_type))


def test_get_mixed_loss_refuses_bad_match_type_and_missing_counts():
    for mt in (torch.tensor([[0, 2]]), torch.tensor([0.0, 2.0]), torch.tensor([], dtype=torch.int64)):
        with pytest.raises(ValueError):
            _mixed_loss(mt)
    with pytest.raises(ValueError, match="num_valid"):
        _mixed_loss(torch.tensor([0, 2]))          # valid types, but no per-pair counts


def _cpu_part(B, match_type):
    i64 = dict(dtype=torch.int64)
    part = {"image_a": torch.zeros(B, 3, 4, 6), "image_b": torch.zeros(B, 3, 4, 6), "counts": torch.zeros(B, 4, **i64),
            "empty": torch.zeros(B, dtype=torch.bool), "match_type": match_type}
    part.update({k: torch.full((B, 2), -1, **i64) for k in S.INDEX_KEYS})
    return part


def test_concat_batches_refuses_a_match_type_off_the_host():
    good = _cpu_part(2, torch.full((2,), T.SINGLE_OBJECT_WITHIN_SCENE, dtype=torch.int64))
    # a relabelled part whose types left the host: refused where the mistake is made, before anything is copied
    # (a "meta" tensor stands in for a CUDA one on a machine without a GPU)
    moved = _cpu_part(3, torch.full((3,), T.DIFFERENT_OBJECT, dtype=torch.int64, device="meta"))
    with pytest.raises(ValueError, match="match_type of part 1 is on meta"):
        S.concat_batches([good, moved])
    with pytest.raises(ValueError, match="match_type of part 1 must have shape"):
        S.concat_batches([good, _cpu_part(3, torch.zeros(2, dtype=torch.int64))])
    out = S.concat_batches([good, _cpu_part(3, torch.full((3,), T.DIFFERENT_OBJECT))])
    assert out["match_type"].tolist() == [T.SINGLE_OBJECT_WITHIN_SCENE] * 2 + [T.DIFFERENT_OBJECT] * 3
