"""CPU: pdc_b200.frames.FrameStore without a GPU -- decoding, host tables, train/test lists, refusals before allocation, and
pair selection against oracle/frames_oracle.py (a one-draw-at-a-time restatement of SpartanDataset's selection)."""
import os

import numpy as np
import pytest
import torch
from PIL import Image
from scipy.spatial.transform import Rotation

import pdc_b200
from pdc_b200 import frames as FR
from pdc_b200 import synthetic
from oracle import frames_oracle as FO

T = pdc_b200.SpartanDatasetDataType
H, W = 64, 96
R90 = (np.cos(np.pi / 4), 0.0, 0.0, np.sin(np.pi / 4))     # 90 degrees about z, (w, x, y, z)
I4 = (1.0, 0.0, 0.0, 0.0)


def scene_poses():
    """Non-contiguous image indices.  obj_a_0: frames 0-2 lie within 0.2 m of each other, 7 and 9 far away, so some draws
    of image b fail; obj_b_1: every frame at one position, each turned 90 degrees from the last: no frame qualifies."""
    rot = lambda k: tuple(Rotation.from_euler("xyz", [0.1 * k, -0.05 * k, 0.02]).as_quat()[[3, 0, 1, 2]])
    return {
        "obj_a_0": [(0, I4, (0, 0, 0)), (1, rot(1), (0.05, 0, 0)), (2, rot(2), (0.1, 0.05, 0)), (7, rot(3), (0.6, 0, 0)),
                    (9, rot(4), (0.5, 0.4, 0.1))],
        "obj_a_1": [(3, rot(1), (0, 0, 0)), (4, rot(2), (0.3, 0, 0)), (8, rot(3), (0, 0.3, 0))],
        "obj_b_0": [(0, rot(2), (0, 0, 0)), (5, I4, (0.25, 0, 0)), (6, rot(1), (0.1, 0.1, 0)), (11, rot(3), (0.0, 0.0, 0.3))],
        "obj_b_1": [(1, I4, (0.1, 0.1, 0.1)), (2, R90, (0.1, 0.1, 0.1)), (4, I4, (0.1, 0.1, 0.1))],
        "multi_0": [(0, I4, (0, 0, 0)), (2, rot(1), (0.4, 0, 0)), (3, rot(2), (0, 0, 0.1))],
    }


SINGLE = [{"object_id": "shoe_a", "train": ["obj_a_0", "obj_a_1"], "test": ["obj_a_1"], "evaluation_labeled_data_path": []},
          {"object_id": "shoe_b", "train": ["obj_b_0", "obj_b_1"], "test": ["obj_b_0"], "evaluation_labeled_data_path": []}]
MULTI = [{"train": ["multi_0"], "test": [], "evaluation_labeled_data_path": []}]


@pytest.fixture(scope="module")
def dataset(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("logs"))
    K = synthetic.write_reference_scenes(root, scene_poses(), H, W, seed=3)
    cfg = {"logs_root_path": root, "single_object_scenes_config_files": SINGLE, "multi_object_scenes_config_files": MULTI}
    return root, cfg, K


def test_host_store_is_the_decoded_files(dataset):
    root, cfg, K = dataset
    st = FR.FrameStore.from_dataset_config(cfg, storage="host", threads=3)
    poses = scene_poses()
    order = ["obj_a_0", "obj_a_1", "obj_b_0", "obj_b_1", "multi_0"]
    assert st.scene_names == order and st.image_shape == (H, W) and st.num_frames == sum(len(poses[s]) for s in order)
    assert st.rgb.dtype == torch.uint8 and st.depth.dtype == torch.uint16 and st.mask.dtype == torch.uint8
    assert np.array_equal(st.K, K)
    f = 0
    for s_id, s in enumerate(order):
        assert st.scene_start[s_id] == f
        for idx, q, t in sorted(poses[s]):
            d = os.path.join(root, s, "processed")
            rgb = np.asarray(Image.open(os.path.join(d, "images", "%06d_rgb.png" % idx)).convert("RGB"))
            depth = np.asarray(Image.open(os.path.join(d, "rendered_images", "%06d_depth.png" % idx)))
            mask = np.asarray(Image.open(os.path.join(d, "image_masks", "%06d_mask.png" % idx)))
            assert depth.dtype == np.uint16
            assert np.array_equal(st.rgb[f].numpy(), rgb)
            assert np.array_equal(st.depth[f].numpy(), depth)
            assert np.array_equal(st.mask[f].numpy(), mask)
            assert st.image_index[f] == idx
            ref = np.eye(4)
            ref[:3, :3] = Rotation.from_quat([q[1], q[2], q[3], q[0]]).as_matrix()
            ref[:3, 3] = t
            np.testing.assert_allclose(st.poses[f], ref, atol=1e-12)
            f += 1
    assert st.scene_start[-1] == f


def test_modes_pick_the_configured_scene_lists(dataset):
    _, cfg, _ = dataset
    tr = FR.FrameStore.from_dataset_config(cfg, mode="train", storage="host")
    te = FR.FrameStore.from_dataset_config(cfg, mode="test", storage="host")
    assert tr.objects == te.objects == {"shoe_a": {"train": ["obj_a_0", "obj_a_1"], "test": ["obj_a_1"]},
                                        "shoe_b": {"train": ["obj_b_0", "obj_b_1"], "test": ["obj_b_0"]}}
    assert te.scene_names == ["obj_a_1", "obj_b_0"] and te.multi_object == {"train": ["multi_0"], "test": []}
    sel = te.select(torch.zeros(32, dtype=torch.int64), np.random.default_rng(0))
    assert {m["scene_name"] for m in sel.metadata} <= {"obj_a_1", "obj_b_0"}
    with pytest.raises(ValueError, match="MULTI_OBJECT"):
        te.select(torch.full((2,), T.MULTI_OBJECT, dtype=torch.int64))


def test_sub_configs_by_file_name(dataset, tmp_path):
    import yaml
    root, _, _ = dataset
    for kind, items in (("single_object", SINGLE), ("multi_object", MULTI)):
        os.makedirs(tmp_path / kind)
        for i, c in enumerate(items):
            (tmp_path / kind / ("%d.yaml" % i)).write_text(yaml.safe_dump(c))
    cfg = {"logs_root_path": os.path.basename(root), "single_object_scenes_config_files": ["0.yaml", "1.yaml"],
           "multi_object_scenes_config_files": ["0.yaml"]}
    st = FR.FrameStore.from_dataset_config(cfg, storage="host", config_dir=str(tmp_path), data_dir=os.path.dirname(root))
    assert st.scene_names == ["obj_a_0", "obj_a_1", "obj_b_0", "obj_b_1", "multi_0"]


@pytest.fixture
def no_allocation(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("allocated before refusing")
    monkeypatch.setattr(FR.FrameStore, "_allocate", staticmethod(refuse))


def _copy(root, tmp_path):
    import shutil
    dst = str(tmp_path / "logs")
    shutil.copytree(root, dst)
    return dst


def _cfg(root):
    return {"logs_root_path": root, "single_object_scenes_config_files": SINGLE, "multi_object_scenes_config_files": MULTI}


def test_missing_file_refused_before_allocation(dataset, tmp_path, no_allocation):
    root = _copy(dataset[0], tmp_path)
    path = os.path.join(root, "obj_b_0", "processed", "image_masks", "000006_mask.png")
    os.remove(path)
    with pytest.raises(ValueError, match="000006_mask.png"):
        FR.FrameStore.from_dataset_config(_cfg(root), storage="host")


def test_mismatched_K_refused_before_allocation(dataset, tmp_path, no_allocation):
    import yaml
    root = _copy(dataset[0], tmp_path)
    p = os.path.join(root, "obj_a_1", "processed", "images", "camera_info.yaml")
    c = yaml.safe_load(open(p))
    c["camera_matrix"]["data"][0] += 1.0
    open(p, "w").write(yaml.safe_dump(c))
    with pytest.raises(ValueError, match="obj_a_1"):
        FR.FrameStore.from_dataset_config(_cfg(root), storage="host")


def test_mismatched_size_refused_before_allocation(dataset, tmp_path, no_allocation):
    root = _copy(dataset[0], tmp_path)
    p = os.path.join(root, "multi_0", "processed", "rendered_images", "000002_depth.png")
    Image.fromarray(np.zeros((H, W + 1), dtype=np.uint16)).save(p)
    with pytest.raises(ValueError, match="multi_0"):
        FR.FrameStore.from_dataset_config(_cfg(root), storage="host")


def test_byte_budget_refused_before_allocation(dataset, monkeypatch):
    calls = []
    real = FR.FrameStore._allocate
    monkeypatch.setattr(FR.FrameStore, "_allocate", staticmethod(lambda *a: calls.append(a) or real(*a)))
    F = 18
    with pytest.raises(ValueError, match="byte_budget"):
        FR.FrameStore.from_dataset_config(dataset[1], storage="host", byte_budget=F * H * W * 6 - 1)
    FR.FrameStore.from_dataset_config(dataset[1], storage="host", byte_budget=F * H * W * 6)
    assert len(calls) == 2      # the refusal happens inside the size check, ahead of the first tensor


def _oracle_tables(st, mode):
    pose_data = {s: {} for s in st.scene_names}
    for s_id, s in enumerate(st.scene_names):
        for f in range(st.scene_start[s_id], st.scene_start[s_id + 1]):
            pose_data[s][int(st.image_index[f])] = st.poses[f]
    return {"single": {c["object_id"]: {"train": c["train"], "test": c["test"]} for c in SINGLE},
            "multi": {"train": MULTI[0]["train"], "test": MULTI[0]["test"]}, "pose_data": pose_data, "mode": mode}


@pytest.mark.parametrize("t", [T.SINGLE_OBJECT_WITHIN_SCENE, T.SINGLE_OBJECT_ACROSS_SCENE, T.DIFFERENT_OBJECT, T.MULTI_OBJECT,
                               T.SYNTHETIC_MULTI_OBJECT, "mixed"])
def test_selection_equals_the_reference_restatement(dataset, t):
    st = FR.FrameStore.from_dataset_config(dataset[1], storage="host")
    ds = _oracle_tables(st, "train")
    B = 400
    rng = np.random.default_rng(11)
    types = torch.as_tensor(rng.integers(0, 5, B) if t == "mixed" else np.full(B, int(t)), dtype=torch.int64)
    u = rng.random((B, FR.NUM_UNIFORMS))
    sel = st.select_from_uniforms(types, u)
    assert sorted(sel.order.tolist()) == list(range(B))
    assert np.all(np.diff(sel.types) >= 0)
    n_empty = 0
    for i in range(B):
        p = int(sel.order[i])
        tt = int(types[p])
        ref = FO.select(ds, tt, u[p])
        m = sel.metadata[i]
        assert m["type"] == tt == sel.types[i]
        empty = ref["images_a"][1] is None or (ref["images_b"] is not None and tt == T.SYNTHETIC_MULTI_OBJECT
                                                and ref["images_b"][1] is None)
        if tt in (T.SINGLE_OBJECT_ACROSS_SCENE, T.DIFFERENT_OBJECT):
            empty = False
            assert (m["scene_name_a"], m["scene_name_b"]) == (ref["scene_a"], ref["scene_b"])
            assert (m["image_a_idx"], m["image_b_idx"]) == (ref["images_a"][0], ref["images_b"][0])
            assert m["scene_name_a"] != m["scene_name_b"]
        elif tt == T.SYNTHETIC_MULTI_OBJECT:
            assert (m["scene_name_a"], m["scene_name_b"]) == (ref["scene_a"], ref["scene_b"])
            assert (m["image_a1_idx"], m["image_a2_idx"] if ref["images_a"][1] is not None else None) == ref["images_a"]
            assert m["image_a_idx"] == ref["images_b"][0]
            if ref["images_a"][1] is not None:
                assert m["image_b_idx"] == ref["images_b"][1]
        else:
            assert m["scene_name"] == ref["scene_a"]
            assert (m["image_a_idx"], m["image_b_idx"]) == ref["images_a"]
        assert bool(sel.empty[i]) == empty
        n_empty += empty
        # the frames are the images named in the metadata
        s = st.scene_names.index(ref["scene_a"])
        assert st.image_index[sel.frames[i, 0]] == ref["images_a"][0] and st.scene_start[s] <= sel.frames[i, 0] < st.scene_start[s + 1]
        if empty:
            assert (sel.frames[i, 1] == sel.frames[i, 0]) or tt == T.SYNTHETIC_MULTI_OBJECT
    if t in (T.SINGLE_OBJECT_WITHIN_SCENE, T.SYNTHETIC_MULTI_OBJECT, "mixed"):
        assert n_empty > 0                                  # obj_b_1 never has an image b
    # within a type, the pairs with an image b come first
    for tt in np.unique(sel.types):
        e = sel.empty[sel.types == tt]
        assert not np.any(e[:-1] & ~e[1:])


def test_no_frame_qualifies_in_a_scene_of_90_degree_turns(dataset):
    st = FR.FrameStore.from_dataset_config(dataset[1], storage="host")
    s = st.scene_names.index("obj_b_1")
    p = st.poses[st.scene_start[s]:st.scene_start[s + 1]]
    # the reference's angle test compares radians with 20 (degrees meant).  Its formula, 2 arccos(2 <q, r>^2 - 1), gives
    # a 90 degree turn as pi; no angle reaches 20, so the turn never qualifies
    assert abs(FO.compute_angle_between_poses(p[0], p[1]) - np.pi) < 1e-9
    sel = st.select(torch.zeros(300, dtype=torch.int64), np.random.default_rng(2))
    hit = [i for i, m in enumerate(sel.metadata) if m["scene_name"] == "obj_b_1"]
    assert hit and all(sel.empty[i] and sel.metadata[i]["image_b_idx"] is None for i in hit)
    # every other scene has a frame more than 0.2 m away from each of its frames
    assert not any(sel.empty[i] for i, m in enumerate(sel.metadata) if m["scene_name"] != "obj_b_1")


def test_selection_refusals(dataset):
    st = FR.FrameStore.from_dataset_config(dataset[1], mode="test", storage="host")
    with pytest.raises(ValueError, match="only one"):
        st.select(torch.full((4,), T.SINGLE_OBJECT_ACROSS_SCENE, dtype=torch.int64))
    with pytest.raises(ValueError, match="shape"):
        st.select_from_uniforms(torch.zeros(3, dtype=torch.int64), np.zeros((3, 5)))


def test_host_store_is_not_gathered(dataset):
    st = FR.FrameStore.from_dataset_config(dataset[1], storage="host")
    with pytest.raises(ValueError, match="pageable"):
        st.gather([0], [1])
