"""GPU: device-resident training frames (pdc_b200.frames.FrameStore, csrc/frames.cu ddn_frames_gather).

* the gather equals torch indexing of the store bit for bit (rgb[idx], depth[idx].float(), mask[idx]) for the device and
  the pinned-host store, at B = 1, 8 and 128, at 640x480 and at 37x53 (rows that are not a multiple of 16 bytes);
* out-of-range indices and B above the limit are refused before any launch;
* every producer fed by FrameStore.batch gives the outputs, every key, of the same producer fed by hand-stacked frames;
* the shoes mix (3 within-scene + 3 different-object + 2 synthetic) is built without a host synchronisation, and two runs
  with the same seeds give the same batch;
* a training step fed by the store gives the loss terms and flat gradient of the step fed by hand-stacked frames."""
import ctypes

import numpy as np
import pytest
import torch

import pdc_b200
from pdc_b200 import _native as N
from pdc_b200 import frames as FR
from pdc_b200 import loss_composer
from pdc_b200 import sampling as S
from pdc_b200 import synthetic
from pdc_b200.loss_composer import SpartanDatasetDataType as T

pytestmark = pytest.mark.gpu
DEV = "cuda"
KEYS = S.INDEX_KEYS


def training_config(n_attempts=40, non_matches=4, samples=100):
    return {"training": dict(num_matching_attempts=n_attempts, num_non_matches_per_match=non_matches,
                             fraction_masked_non_matches=0.5, fraction_background_non_matches=0.5,
                             sample_matches_only_off_mask=True, domain_randomize=True, use_image_b_mask_inv=True,
                             cross_scene_num_samples=samples)}


def depth_f32(depth):
    """The uint16 store as float32, converted on the host (torch's CUDA kernels barely support uint16)."""
    return torch.from_numpy(depth.cpu().numpy().astype(np.float32))


def random_store(F, H, W, storage, seed=0):
    g = torch.Generator().manual_seed(seed)
    scene = {"rgb": torch.randint(0, 256, (F, H, W, 3), dtype=torch.uint8, generator=g),
             "depth": torch.randint(0, 65536, (F, H, W), dtype=torch.int32, generator=g).to(torch.uint16),
             "mask": torch.randint(0, 256, (F, H, W), dtype=torch.uint8, generator=g),
             "poses": np.tile(np.eye(4), (F, 1, 1)), "object_id": "o"}
    return FR.FrameStore.from_arrays({"s": scene}, np.eye(3), storage=storage)


@pytest.fixture(scope="module")
def stores():
    out = {}
    for H, W in ((480, 640), (37, 53)):
        for storage in ("cuda", "pinned"):
            out[(H, W, storage)] = random_store(48, H, W, storage, seed=H)
    return out


@pytest.mark.parametrize("storage", ["cuda", "pinned"])
@pytest.mark.parametrize("shape", [(480, 640), (37, 53)])
@pytest.mark.parametrize("B", [1, 8, 128])
def test_gather_equals_torch_indexing(stores, storage, shape, B):
    st = stores[(*shape, storage)]
    assert st.rgb.is_cuda == (storage == "cuda") and (storage == "cuda" or st.rgb.is_pinned())
    rng = np.random.default_rng(B)
    ia, ib = rng.integers(0, st.num_frames, B), rng.integers(0, st.num_frames, B)
    ia[0], ib[-1] = 0, st.num_frames - 1
    rgb, dep, mask = st.gather(ia, ib)
    ref_rgb, ref_dep, ref_mask = st.rgb.to(DEV), depth_f32(st.depth).to(DEV), st.mask.to(DEV)
    for side, idx in ((0, ia), (1, ib)):
        i = torch.as_tensor(idx, device=DEV)
        assert torch.equal(rgb[side], ref_rgb[i])
        assert dep[side].dtype == torch.float32 and torch.equal(dep[side], ref_dep[i])
        assert torch.equal(mask[side], ref_mask[i])
    rgb2, dep2, mask2 = st.gather(ia, ib, depth=False)
    assert dep2 is None and torch.equal(rgb2[0], rgb[0]) and torch.equal(mask2[1], mask[1])


def test_gather_refusals_before_any_launch(stores):
    st = stores[(37, 53, "cuda")]
    torch.cuda.synchronize()
    n0 = N.launch_count()
    for ia, ib in (([0, st.num_frames], [0, 1]), ([-1], [0]), ([0], [st.num_frames + 5])):
        with pytest.raises(ValueError, match="frame indices"):
            st.gather(ia, ib)
    with pytest.raises(ValueError, match="1 to 128"):
        st.gather(np.zeros(129, dtype=np.int64), np.zeros(129, dtype=np.int64))
    # the C entry point itself refuses the same, before its launch
    F, (H, W) = st.num_frames, st.image_shape
    out = torch.empty(2, 129, H, W, 3, dtype=torch.uint8, device=DEV)
    m = torch.empty(2, 129, H, W, dtype=torch.uint8, device=DEV)
    for B, bad in ((2, F), (2, -3), (129, 0), (0, 0)):
        idx = (ctypes.c_int32 * 129)(*([0] * 129))
        idx[min(1, max(B - 1, 0))] = bad
        with pytest.raises(N.DdnError):
            N.check(N.lib.ddn_frames_gather(N.ptr(st.rgb), N.ptr(st.depth), N.ptr(st.mask), F, H, W, idx, idx, B,
                                            N.ptr(out[0]), N.ptr(out[1]), None, None, N.ptr(m[0]), N.ptr(m[1]), N.stream_ptr()))
    assert N.launch_count() == n0


# ------------------------------------------------------------------------------------------------ dataset-fed batches
H, W = 64, 96


@pytest.fixture(scope="module")
def store(tmp_path_factory):
    from scipy.spatial.transform import Rotation
    rot = lambda k: tuple(Rotation.from_euler("xyz", [0.05 * k, -0.08 * k, 0.02 * k]).as_quat()[[3, 0, 1, 2]])
    poses = lambda n, step: [(3 * i + 1, rot(i), (step * i, 0.02 * i, 0.01 * i)) for i in range(n)]
    scenes = {"a0": poses(5, 0.15), "a1": poses(4, 0.25), "b0": poses(5, 0.3), "b1": poses(3, 0.12),
              "m0": poses(4, 0.3), "stuck": [(0, (1.0, 0, 0, 0), (0, 0, 0)), (1, (0, 0, 0, 1.0), (0.05, 0, 0))]}
    root = str(tmp_path_factory.mktemp("logs"))
    synthetic.write_reference_scenes(root, scenes, H, W, seed=5)
    cfg = {"logs_root_path": root,
           "single_object_scenes_config_files": [{"object_id": "x", "train": ["a0", "a1"], "test": []},
                                                 {"object_id": "y", "train": ["b0", "b1", "stuck"], "test": []}],
           "multi_object_scenes_config_files": [{"train": ["m0"], "test": []}]}
    return FR.FrameStore.from_dataset_config(cfg, storage="cuda")


def hand_part(st, t, frames, empty, tc, g):
    """The producer of type t fed by frames stacked with torch indexing of the store, drawing from generator g."""
    pick = lambda col: (st.rgb[torch.as_tensor(frames[:, col], device=DEV)],
                        depth_f32(st.depth)[torch.as_tensor(frames[:, col])].to(DEV),
                        st.mask[torch.as_tensor(frames[:, col], device=DEV)], st.poses[frames[:, col]])
    if t in (T.SINGLE_OBJECT_ACROSS_SCENE, T.DIFFERENT_OBJECT):
        a, b = pick(0), pick(1)
        return S.across_scene_batch(a[0], b[0], a[2], b[2], tc, generator=g, match_type=t)
    a, b = pick(0), pick(1)
    if t == T.SYNTHETIC_MULTI_OBJECT:
        c, d = pick(2), pick(3)
        out = S.synthetic_multi_object_batch((a[0], b[0], a[1], b[1], a[2], b[2], a[3], b[3]),
                                             (c[0], d[0], c[1], d[1], c[2], d[2], c[3], d[3]), st.K, tc, generator=g)
    else:
        out = S.within_scene_batch(a[0], b[0], a[1], b[1], a[2], b[2], a[3], b[3], st.K, tc, generator=g)
        out["match_type"] = torch.full_like(out["match_type"], t)
    n_ok = int((~empty).sum())
    for k in KEYS:
        out[k][n_ok:] = -1
    out["counts"][n_ok:] = 0
    out["empty"][n_ok:] = True
    return out


def assert_same(x, y):
    for k in ("image_a", "image_b", "counts", "empty") + tuple(KEYS):
        assert torch.equal(x[k], y[k]), k
    assert torch.equal(x["match_type"], y["match_type"])
    for k in ("matches", "masked", "background", "blind"):
        assert torch.equal(x["num_valid"][k], y["num_valid"][k]), k


@pytest.mark.parametrize("t", [T.SINGLE_OBJECT_WITHIN_SCENE, T.SINGLE_OBJECT_ACROSS_SCENE, T.DIFFERENT_OBJECT, T.MULTI_OBJECT,
                               T.SYNTHETIC_MULTI_OBJECT])
def test_each_producer_fed_by_the_store_equals_hand_stacked(store, t):
    tc = training_config()
    types = torch.full((12,), int(t), dtype=torch.int64)
    out = store.batch(types, tc, generator=torch.Generator(device=DEV).manual_seed(7), rng=np.random.default_rng(3))
    sel = store.select(types, np.random.default_rng(3))
    ref = S.concat_batches([hand_part(store, int(t), sel.frames, sel.empty, tc, torch.Generator(device=DEV).manual_seed(7))])
    assert_same(out, ref)
    assert out["metadata"] == sel.metadata and len(out["metadata"]) == 12
    # a pair without an image b is empty; the synthetic producer also empties pairs by its own early returns
    empty = out["empty"].cpu()
    assert bool(empty[torch.as_tensor(sel.empty)].all())
    if t != T.SYNTHETIC_MULTI_OBJECT:
        assert torch.equal(empty, torch.as_tensor(sel.empty))             # no fixture mask is empty


def test_batch_above_a_producer_limit_is_split(store):
    tc = training_config(n_attempts=8, non_matches=2, samples=20)
    types = torch.tensor([T.DIFFERENT_OBJECT] * 130 + [T.SYNTHETIC_MULTI_OBJECT] * 70, dtype=torch.int64)
    out = store.batch(types, tc, generator=torch.Generator(device=DEV).manual_seed(1), rng=np.random.default_rng(1))
    assert out["image_a"].shape == (200, 3, H, W) and out["match_type"].tolist() == types.tolist()
    assert len(out["metadata"]) == 200


SHOES = [T.SINGLE_OBJECT_WITHIN_SCENE] * 3 + [T.DIFFERENT_OBJECT] * 3 + [T.SYNTHETIC_MULTI_OBJECT] * 2


def test_shoes_mix_without_sync_and_repeatable(store):
    tc = training_config()
    types = torch.tensor(SHOES, dtype=torch.int64)
    runs = []
    for _ in range(2):
        g, rng = torch.Generator(device=DEV).manual_seed(21), np.random.default_rng(22)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            runs.append(store.batch(types, tc, generator=g, rng=rng))
        finally:
            torch.cuda.set_sync_debug_mode("default")
    assert runs[0]["match_type"].tolist() == SHOES
    assert_same(runs[0], runs[1])
    assert runs[0]["metadata"] == runs[1]["metadata"]


def test_training_step_fed_by_the_store_equals_hand_stacked(store):
    D, B = 3, 8
    tc = training_config()
    types = torch.tensor(SHOES, dtype=torch.int64)
    out = store.batch(types, tc, generator=torch.Generator(device=DEV).manual_seed(31), rng=np.random.default_rng(32))
    sel = store.select(types, np.random.default_rng(32))
    g = torch.Generator(device=DEV).manual_seed(31)            # batch() hands one generator to the producers in turn
    parts = [hand_part(store, int(t), sel.frames[sel.types == t], sel.empty[sel.types == t], tc, g)
             for t in np.unique(sel.types)]
    ref = S.concat_batches(parts)
    assert_same(out, ref)
    res = []
    dcn0 = None
    for batch in (out, ref):
        dcn = pdc_b200.DenseCorrespondenceNetwork.from_config({"descriptor_dimension": D, "image_width": W, "image_height": H},
                                                              load_stored_params=False)
        if dcn0 is None:
            dcn0 = {k: v.clone() for k, v in dcn.fcn.state_dict().items()}
        dcn.fcn.load_state_dict(dcn0)
        pcl = pdc_b200.PixelwiseContrastiveLoss(dcn.image_shape, dict(pdc_b200.DEFAULT_LOSS_CONFIG))
        a, b = dcn.forward_pair(batch["image_a"], batch["image_b"])
        five = loss_composer.get_mixed_loss(pcl, batch["match_type"], dcn.process_network_output(a, B),
                                            dcn.process_network_output(b, B), *[batch[k] for k in KEYS],
                                            num_valid=batch["num_valid"])
        five[0].backward()
        flat = torch.cat([p.grad.reshape(-1) for p in dcn.parameters() if p.grad is not None])
        res.append(([f.detach().clone() for f in five], flat))
    assert bool(torch.isfinite(res[0][0][0]).all()) and float(res[0][0][0]) > 0
    for x, y in zip(res[0][0], res[1][0]):
        assert torch.equal(x, y)
    assert torch.equal(res[0][1], res[1][1])

