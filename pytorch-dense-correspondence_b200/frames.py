"""Device-resident training frames: every frame of a dataset decoded once, kept in device (or pinned host) memory, pairs
drawn on the host by SpartanDataset's rules, and each step's frames gathered by one kernel launch (csrc/frames.cu) into
the inputs of the batch producers (``sampling.within_scene_batch`` / ``across_scene_batch`` /
``synthetic_multi_object_batch``).

Line references are to the reference's dense_correspondence/dataset/spartan_dataset_masked.py unless stated otherwise.
"""
import ctypes
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import _native as N
from . import sampling
from .loss_composer import SpartanDatasetDataType as T

# the reference's layout (get_image_filename, :357-389; get_pose_data, :328-342; get_camera_intrinsics, :391-406)
RGB_FILE = os.path.join("processed", "images", "%06d_rgb.png")
DEPTH_FILE = os.path.join("processed", "rendered_images", "%06d_depth.png")
MASK_FILE = os.path.join("processed", "image_masks", "%06d_mask.png")
POSE_FILE = os.path.join("processed", "images", "pose_data.yaml")
CAMERA_FILE = os.path.join("processed", "images", "camera_info.yaml")

# get_img_idx_with_different_pose(threshold=0.2, angle_threshold=20, num_attempts=50) as get_within_scene_data calls it
# (:633; dense_correspondence_dataset_masked.py:260-287)
NUM_ATTEMPTS = 50
DISTANCE_THRESHOLD = 0.2

# The uniform numbers one pair's selection reads, whatever its type (unused slots are drawn and ignored, so pair i always
# reads row i):
#   U_OBJ, U_OBJ + 1   the object (random.choice), or two different objects (np.random.choice(n, 2, replace=False))
#   U_SCENE_A          scene A (random.choice over the object's scenes, or the multi-object scenes)
#   U_SCENE_B, +1      scene B: a scene of the second object, or two different scenes of the same object
#   U_HALF1            image a of scene A, then NUM_ATTEMPTS draws of image b
#   U_HALF2            the same for scene B (synthetic multi-object pairs); image b of an across-scene pair
# A choice among n items with uniform u is item min(floor(u n), n - 1); two different items from (u, v) are
# i = choice(u, n) and j = choice(v, n - 1), j += 1 if j >= i.
U_OBJ, U_SCENE_A, U_SCENE_B, U_HALF1 = 0, 2, 3, 5
U_HALF2 = U_HALF1 + 1 + NUM_ATTEMPTS
NUM_UNIFORMS = U_HALF2 + 1 + NUM_ATTEMPTS


def _choice(u, n):
    return np.minimum((np.asarray(u) * n).astype(np.int64), n - 1)


def _two_different(u, v, n):
    i = _choice(u, n)
    j = _choice(v, n - 1)
    return i, j + (j >= i)


def _yaml(path):
    import yaml
    loader = getattr(yaml, "CSafeLoader", yaml.SafeLoader)
    with open(path) as f:
        return yaml.load(f, Loader=loader)


def pose_from_dict(d):
    """utils.homogenous_transform_from_dict: camera_to_world {translation: {x, y, z}, quaternion (or orientation /
    rotation): {w, x, y, z}} -> float64 [4, 4], via transformations.quaternion_matrix."""
    quat = None
    for name in ("orientation", "rotation", "quaternion"):       # the last key present wins, as in getQuaternionFromDict
        if name in d:
            quat = d[name]
    if quat is None:
        raise ValueError("pose has none of orientation / rotation / quaternion")
    q = np.array([quat["w"], quat["x"], quat["y"], quat["z"]], dtype=np.float64)
    n = np.dot(q, q)
    M = np.identity(4)
    if n >= np.finfo(float).eps * 4.0:
        q *= np.sqrt(2.0 / n)
        q = np.outer(q, q)
        M = np.array([[1.0 - q[2, 2] - q[3, 3], q[1, 2] - q[3, 0], q[1, 3] + q[2, 0], 0.0],
                      [q[1, 2] + q[3, 0], 1.0 - q[1, 1] - q[3, 3], q[2, 3] - q[1, 0], 0.0],
                      [q[1, 3] - q[2, 0], q[2, 3] + q[1, 0], 1.0 - q[1, 1] - q[2, 2], 0.0],
                      [0.0, 0.0, 0.0, 1.0]])
    t = d["translation"]
    M[0:3, 3] = [t["x"], t["y"], t["z"]]
    return M


def camera_matrix(camera_info):
    """CameraIntrinsics.from_yaml_file (modules/dense_correspondence_manipulation/utils/utils.py:414-426) -> K [3, 3]."""
    data = camera_info["camera_matrix"]["data"]
    return np.array([[data[0], 0, data[2]], [0, data[4], data[5]], [0, 0, 1]], dtype=np.float64)


def decode_rgb(path):
    from PIL import Image
    return np.asarray(Image.open(path).convert("RGB"))          # get_rgb_image


def decode_depth(path):
    """The raw 16-bit values (millimetres) of get_depth_image's PIL image."""
    from PIL import Image
    a = np.asarray(Image.open(path))
    if a.dtype != np.uint16:
        if a.dtype.kind not in "iu" or a.size and (a.min() < 0 or a.max() > 65535):
            raise ValueError("%s: depth must hold 16-bit unsigned values (got %s)" % (path, a.dtype))
        a = a.astype(np.uint16)
    return a


def decode_mask(path):
    from PIL import Image
    return np.asarray(Image.open(path)).astype(np.uint8, copy=False)     # get_mask_image


class Selection:
    """The frames of one batch, in batch order: pairs grouped by type (ascending SpartanDatasetDataType), and within a
    type the pairs with an image b first.  ``types`` int64 [B]; ``frames`` int64 [B, 4]: store frames a, b (scene A)
    and, for SYNTHETIC_MULTI_OBJECT, a, b of scene B (else -1); a pair with no image b has b = a; ``empty`` bool [B]:
    no image b was found (the reference's return_empty_data); ``order`` int64 [B]: the position of each pair in the
    ``types`` the selection was drawn for; ``metadata``: one dict per pair, the reference's ``metadata``."""

    def __init__(self, types, frames, empty, order, metadata):
        self.types, self.frames, self.empty, self.order, self.metadata = types, frames, empty, order, metadata


class FrameStore:
    """Every frame of a dataset, decoded once: ``rgb`` uint8 [F, H, W, 3], ``depth`` uint16 [F, H, W] (millimetres),
    ``mask`` uint8 [F, H, W], contiguous, on a CUDA device (``storage="cuda"``) or in pinned host memory
    (``storage="pinned"``, read by the gather kernel over the host link; ``"host"``: pageable memory, which the kernel
    cannot read, for inspection without a GPU), and host tables: ``poses`` float64
    [F, 4, 4] (camera to world), ``K`` [3, 3] (one for every scene), ``scene_names``, ``scene_start`` int64 [S + 1]
    (scene s holds frames scene_start[s]:scene_start[s + 1]), ``image_index`` int64 [F] (the pose_data.yaml key of each
    frame), ``objects`` {object_id: {"train": [scene names], "test": [...]}}, ``multi_object`` {"train": [...],
    "test": [...]} and ``mode``.  Only the scenes of ``mode`` are loaded.  Each rank of a data-parallel run builds its
    own store: F * H * W * 6 bytes per rank."""

    def __init__(self, rgb, depth, mask, poses, K, scene_names, scene_start, image_index, objects, multi_object, mode):
        self.rgb, self.depth, self.mask = rgb, depth, mask
        self.poses, self.K = poses, K
        self.scene_names, self.scene_start, self.image_index = list(scene_names), scene_start, image_index
        self.objects, self.multi_object, self.mode = objects, multi_object, mode
        self._scene_id = {s: i for i, s in enumerate(self.scene_names)}
        self._object_ids = [o for o in objects if objects[o][mode]]
        self._object_scenes = [np.array([self._scene_id[s] for s in objects[o][mode]], dtype=np.int64) for o in self._object_ids]
        self._multi_scenes = np.array([self._scene_id[s] for s in multi_object[mode]], dtype=np.int64)
        self._sorted_objects = sorted(objects)

    # ------------------------------------------------------------------------------------------------ construction
    @property
    def num_frames(self):
        return int(self.rgb.shape[0])

    @property
    def image_shape(self):
        return tuple(self.rgb.shape[1:3])

    @staticmethod
    def _allocate(F, H, W, storage, byte_budget, device):
        nbytes = F * H * W * 6
        if byte_budget is not None and nbytes > byte_budget:
            raise ValueError("FrameStore: %d frames of %dx%d take %d bytes, more than byte_budget=%d" % (F, W, H, nbytes, byte_budget))
        if storage == "cuda":
            kw = dict(device=torch.device("cuda") if device is None else torch.device(device))
        elif storage == "pinned":
            kw = dict(pin_memory=True)
        elif storage == "host":             # pageable: for inspection; the gather kernel cannot read it
            kw = {}
        else:
            raise ValueError("storage must be 'cuda', 'pinned' or 'host' (got %r)" % (storage,))
        return (torch.empty(F, H, W, 3, dtype=torch.uint8, **kw), torch.empty(F, H, W, dtype=torch.uint16, **kw),
                torch.empty(F, H, W, dtype=torch.uint8, **kw))

    @classmethod
    def from_dataset_config(cls, config, mode="train", storage="cuda", byte_budget=None, threads=None, config_dir=None,
                            data_dir=None, device=None):
        """The composite dataset config SpartanDataset takes (``logs_root_path``, ``single_object_scenes_config_files``,
        ``multi_object_scenes_config_files``), parsed as in _setup_scene_data (:154-210).  Each entry of the two lists is
        either the parsed sub-config (a dict) or a file name under ``config_dir``/single_object or
        ``config_dir``/multi_object.  A relative ``logs_root_path`` is taken under ``data_dir`` (default: the
        DC_DATA_DIR environment variable).  Every file is checked, and the store's size is known, before anything is
        allocated; then every frame is decoded exactly once in a pool of ``threads`` threads (default: one per CPU)."""
        if mode not in ("train", "test"):
            raise ValueError("mode should be one of [test, train]")
        root = config["logs_root_path"]
        if not os.path.isabs(root):
            data_dir = data_dir if data_dir is not None else os.environ.get("DC_DATA_DIR")
            if data_dir is None:
                raise ValueError("logs_root_path %r is relative: pass data_dir or set DC_DATA_DIR" % root)
            root = os.path.join(data_dir, root)

        def sub(entry, kind):
            if isinstance(entry, dict):
                return entry
            if config_dir is None:
                raise ValueError("%s config %r is a file name: pass config_dir" % (kind, entry))
            path = os.path.join(config_dir, kind, entry)
            if not os.path.isfile(path):
                raise ValueError("%s config file %s does not exist" % (kind, path))
            return _yaml(path)

        objects = {}
        for entry in config.get("single_object_scenes_config_files") or []:
            c = sub(entry, "single_object")
            o = objects.setdefault(c["object_id"], {"train": [], "test": []})   # merge_single_object_configs (:1217-1256)
            o["train"] += list(c["train"]); o["test"] += list(c["test"])
        multi = {"train": [], "test": []}
        for entry in config.get("multi_object_scenes_config_files") or []:
            c = sub(entry, "multi_object")
            multi["train"] += list(c["train"]); multi["test"] += list(c["test"])
        scene_names = []
        for s in [s for o in objects.values() for s in o[mode]] + multi[mode]:
            if s not in scene_names:
                scene_names.append(s)

        # every table, file and size before any allocation
        K, K_scene, poses, image_index, files, starts, shape = None, None, [], [], [], [0], None
        for s in scene_names:
            d = os.path.join(root, s)
            for f in (POSE_FILE, CAMERA_FILE):
                if not os.path.isfile(os.path.join(d, f)):
                    raise ValueError("scene %s: missing %s" % (s, os.path.join(d, f)))
            k = camera_matrix(_yaml(os.path.join(d, CAMERA_FILE)))
            if K is None:
                K, K_scene = k, s
            elif not np.array_equal(k, K):
                raise ValueError("scene %s: camera matrix %s differs from scene %s's %s (a batch takes one K)"
                                 % (s, k.tolist(), K_scene, K.tolist()))
            pose_data = _yaml(os.path.join(d, POSE_FILE))
            idx = sorted(int(i) for i in pose_data)
            if not idx:
                raise ValueError("scene %s: pose_data.yaml lists no frames" % s)
            for i in idx:
                poses.append(pose_from_dict(pose_data[i]["camera_to_world"]))
                image_index.append(i)
                files.append(tuple(os.path.join(d, f % i) for f in (RGB_FILE, DEPTH_FILE, MASK_FILE)))
            starts.append(len(files))
        if not files:
            raise ValueError("the %s split of this dataset has no scenes" % mode)

        def probe(paths):
            from PIL import Image
            sizes = []
            for p in paths:
                if not os.path.isfile(p):
                    return p, None
                with Image.open(p) as im:
                    sizes.append(im.size)
            return paths[0], sizes

        threads = threads or os.cpu_count() or 1
        with ThreadPoolExecutor(threads) as pool:
            for path, sizes in pool.map(probe, files):
                if sizes is None:
                    raise ValueError("missing file %s" % path)
                if shape is None:
                    shape, shape_file = sizes[0], path
                for sz in sizes:
                    if sz != shape:
                        raise ValueError("frame %s is %dx%d, but %s is %dx%d (every frame must have one size)"
                                         % (path, sz[0], sz[1], shape_file, shape[0], shape[1]))
        W, H = shape
        F = len(files)
        rgb, depth, mask = cls._allocate(F, H, W, storage, byte_budget, device)

        def decode(i):
            r, dp, m = files[i]
            return decode_rgb(r), decode_depth(dp), decode_mask(m)

        chunk = 64
        with ThreadPoolExecutor(threads) as pool:
            for c0 in range(0, F, chunk):
                c1 = min(F, c0 + chunk)
                out = list(pool.map(decode, range(c0, c1)))
                rgb[c0:c1].copy_(torch.from_numpy(np.stack([o[0] for o in out])))
                depth[c0:c1].copy_(torch.from_numpy(np.stack([o[1] for o in out])))
                mask[c0:c1].copy_(torch.from_numpy(np.stack([o[2] for o in out])))
        return cls(rgb, depth, mask, np.stack(poses), K, scene_names, np.array(starts, dtype=np.int64),
                   np.array(image_index, dtype=np.int64), objects, multi, mode)

    @classmethod
    def from_arrays(cls, scenes, K, storage="cuda", mode="train", byte_budget=None, device=None):
        """A store from frames already in memory.  ``scenes``: {scene name: {"rgb": uint8 [n, H, W, 3], "depth": uint16
        [n, H, W] (millimetres), "mask": uint8 [n, H, W], "poses": [n, 4, 4] camera to world, and "object_id": str for a
        single-object scene or "multi_object": True; optional "image_index" ([n] ints, default 0..n-1) and "split"
        ("train" (default) or "test")}}; K: 3x3, shared by every scene."""
        if mode not in ("train", "test"):
            raise ValueError("mode should be one of [test, train]")
        objects, multi, names, shape, F = {}, {"train": [], "test": []}, [], None, 0
        for name, s in scenes.items():
            split = s.get("split", "train")
            if split not in ("train", "test"):
                raise ValueError("scene %s: split must be 'train' or 'test'" % name)
            if s.get("multi_object", False):
                multi[split].append(name)
            elif "object_id" in s:
                objects.setdefault(s["object_id"], {"train": [], "test": []})[split].append(name)
            else:
                raise ValueError("scene %s has neither object_id nor multi_object" % name)
            if split != mode:
                continue
            n, H, W = np.asarray(s["depth"]).shape if not isinstance(s["depth"], torch.Tensor) else tuple(s["depth"].shape)
            for k, dt, shp in (("rgb", np.uint8, (n, H, W, 3)), ("depth", np.uint16, (n, H, W)), ("mask", np.uint8, (n, H, W)),
                               ("poses", None, (n, 4, 4))):
                a = s[k]
                if tuple(a.shape) != shp or (dt is not None and np.dtype(str(a.dtype).replace("torch.", "")) != dt):
                    raise ValueError("scene %s: %s must be %s %s (got %s %s)" % (name, k, np.dtype(dt).name if dt else "float",
                                                                              shp, a.dtype, tuple(a.shape)))
            if shape is None:
                shape, shape_scene = (H, W), name
            elif (H, W) != shape:
                raise ValueError("scene %s has %dx%d frames, scene %s %dx%d" % (name, W, H, shape_scene, shape[1], shape[0]))
            names.append(name)
            F += n
        if not names:
            raise ValueError("no scene in the %s split" % mode)
        H, W = shape
        rgb, depth, mask = cls._allocate(F, H, W, storage, byte_budget, device)
        starts, poses, image_index = [0], [], []
        for name in names:
            s = scenes[name]
            n = s["rgb"].shape[0]
            f0 = starts[-1]
            for dst, k in ((rgb, "rgb"), (depth, "depth"), (mask, "mask")):
                dst[f0:f0 + n].copy_(torch.as_tensor(np.asarray(s[k]) if not isinstance(s[k], torch.Tensor) else s[k]))
            poses.append(np.asarray(s["poses"], dtype=np.float64))
            image_index.append(np.asarray(s.get("image_index", np.arange(n)), dtype=np.int64))
            starts.append(f0 + n)
        return cls(rgb, depth, mask, np.concatenate(poses), np.asarray(K, dtype=np.float64).reshape(3, 3), names,
                   np.array(starts, dtype=np.int64), np.concatenate(image_index), objects, multi, mode)

    # ------------------------------------------------------------------------------------------------ selection
    def _image_b(self, scene, a, u):
        """get_img_idx_with_different_pose (dense_correspondence_dataset_masked.py:260-287), vectorised over pairs:
        attempt k draws image _choice(u[:, k]) of the scene and takes it if its camera lies more than 0.2 m from image
        a's.  The reference also accepts an angle above angle_threshold=20, but compute_angle_between_poses returns
        radians (utils.py:261-275, at most 2 pi), so that test never fires and is left out.  -> (b, found); b = a where
        no attempt qualified."""
        start, n = self.scene_start[scene], self.scene_start[scene + 1] - self.scene_start[scene]
        cand = start[:, None] + _choice(u, n[:, None])                                       # [B, attempts]
        dist = np.linalg.norm(self.poses[cand, 0:3, 3] - self.poses[a, 0:3, 3][:, None, :], axis=2)
        ok = dist > DISTANCE_THRESHOLD
        found = ok.any(axis=1)
        b = np.where(found, cand[np.arange(len(a)), ok.argmax(axis=1)], a)
        return b, found

    def _half(self, scene, u):
        """get_within_scene_data's image a (:627) and image b (:633) in ``scene`` [B]; u: [B, 1 + NUM_ATTEMPTS]."""
        a = self.scene_start[scene] + _choice(u[:, 0], self.scene_start[scene + 1] - self.scene_start[scene])
        b, found = self._image_b(scene, a, u[:, 1:])
        return a, b, found

    def _object_scene(self, obj, u):
        return np.array([self._object_scenes[o][_choice(x, len(self._object_scenes[o]))] for o, x in zip(obj, u)], dtype=np.int64)

    def _need_objects(self, k, what):
        if len(self._object_ids) < k:
            raise ValueError("%s pairs need %d single-object %s in the %s split (have %d)"
                             % (what, k, "object" if k == 1 else "objects", self.mode, len(self._object_ids)))

    def select_from_uniforms(self, types, u):
        """The frames of the pairs of ``types`` (CPU int64 [B], as ``sampling.draw_data_types`` returns) by the reference's
        rules, reading the uniform numbers ``u`` float64 [B, NUM_UNIFORMS] (layout: U_* above).  -> Selection."""
        types = np.asarray(torch.as_tensor(types).cpu(), dtype=np.int64).reshape(-1)
        u = np.asarray(u, dtype=np.float64)
        B = len(types)
        if u.shape != (B, NUM_UNIFORMS):
            raise ValueError("u must have shape [%d, %d]" % (B, NUM_UNIFORMS))
        frames = np.full((B, 4), -1, dtype=np.int64)
        found = np.ones(B, dtype=bool)
        obj_a = np.full(B, -1, dtype=np.int64); obj_b = obj_a.copy()
        scene_a = obj_a.copy(); scene_b = obj_a.copy()
        h1 = slice(U_HALF1, U_HALF1 + 1 + NUM_ATTEMPTS); h2 = slice(U_HALF2, U_HALF2 + 1 + NUM_ATTEMPTS)
        for t in np.unique(types):
            r = np.nonzero(types == t)[0]
            v = u[r]
            if t == T.SINGLE_OBJECT_WITHIN_SCENE:             # get_single_object_within_scene_data (:543-559)
                self._need_objects(1, "SINGLE_OBJECT_WITHIN_SCENE")
                obj_a[r] = _choice(v[:, U_OBJ], len(self._object_ids))
                scene_a[r] = self._object_scene(obj_a[r], v[:, U_SCENE_A])
            elif t == T.MULTI_OBJECT:                         # get_multi_object_within_scene_data (:561-575)
                if len(self._multi_scenes) == 0:
                    raise ValueError("MULTI_OBJECT pairs need multi-object scenes in the %s split" % self.mode)
                scene_a[r] = self._multi_scenes[_choice(v[:, U_SCENE_A], len(self._multi_scenes))]
            elif t == T.SINGLE_OBJECT_ACROSS_SCENE:           # get_single_object_across_scene_data (:860-872)
                self._need_objects(1, "SINGLE_OBJECT_ACROSS_SCENE")
                obj_a[r] = obj_b[r] = _choice(v[:, U_OBJ], len(self._object_ids))
                scene_a[r] = self._object_scene(obj_a[r], v[:, U_SCENE_A])
                for i, o, x, y in zip(r, obj_a[r], v[:, U_SCENE_B], v[:, U_SCENE_B + 1]):
                    sc = self._object_scenes[o]                # get_different_scene_for_object (:453-474)
                    if len(sc) == 1:
                        raise ValueError("object %s has only one %s scene: SINGLE_OBJECT_ACROSS_SCENE needs two"
                                         % (self._object_ids[o], self.mode))
                    p, q = _two_different(x, y, len(sc))
                    scene_b[i] = sc[p] if sc[p] != scene_a[i] else sc[q]
            elif t in (T.DIFFERENT_OBJECT, T.SYNTHETIC_MULTI_OBJECT):   # :874-888, :890-905
                self._need_objects(2, "DIFFERENT_OBJECT" if t == T.DIFFERENT_OBJECT else "SYNTHETIC_MULTI_OBJECT")
                obj_a[r], obj_b[r] = _two_different(v[:, U_OBJ], v[:, U_OBJ + 1], len(self._object_ids))
                scene_a[r] = self._object_scene(obj_a[r], v[:, U_SCENE_A])
                scene_b[r] = self._object_scene(obj_b[r], v[:, U_SCENE_B])
            else:
                raise ValueError("unknown pair type %d" % t)
            if t in (T.SINGLE_OBJECT_ACROSS_SCENE, T.DIFFERENT_OBJECT):  # get_across_scene_data (:1077-1084): no pose test
                for col, sc, x in ((0, scene_a[r], v[:, U_HALF1]), (1, scene_b[r], v[:, U_HALF2])):
                    frames[r, col] = self.scene_start[sc] + _choice(x, self.scene_start[sc + 1] - self.scene_start[sc])
            else:                                             # get_within_scene_data (:627-639), once per scene
                frames[r, 0], frames[r, 1], found[r] = self._half(scene_a[r], v[:, h1])
                if t == T.SYNTHETIC_MULTI_OBJECT:
                    frames[r, 2], frames[r, 3], f2 = self._half(scene_b[r], v[:, h2])
                    found[r] &= f2
        order = np.lexsort((np.arange(B), ~found, types))      # by type, pairs with an image b first, else draw order
        meta = [self._metadata(types[i], obj_a[i], obj_b[i], scene_a[i], scene_b[i], frames[i], found[i]) for i in order]
        return Selection(types[order], frames[order], ~found[order], order, meta)

    def select(self, types, rng=None):
        """``select_from_uniforms`` with uniforms drawn from ``rng`` (a numpy.random.Generator; default: a fresh one).
        This cannot reproduce the stream of Python's ``random`` the reference draws from, and does not try to."""
        rng = np.random.default_rng() if rng is None else rng
        B = len(np.asarray(torch.as_tensor(types)).reshape(-1))
        return self.select_from_uniforms(types, rng.random((B, NUM_UNIFORMS)))

    def _metadata(self, t, oa, ob, sa, sb, fr, found):
        """The reference's ``metadata`` dict for one pair; image_b_idx is None where no image b was found.  For a
        SYNTHETIC_MULTI_OBJECT pair the reference's second get_within_scene_data overwrites image_a_idx / image_b_idx with
        scene B's; scene A's are kept here as image_a1_idx / image_a2_idx."""
        idx = lambda f: int(self.image_index[f])
        m = {"type": int(t)}
        if t == T.SINGLE_OBJECT_WITHIN_SCENE:
            oid = self._object_ids[oa]
            m.update(object_id=oid, object_id_int=self._sorted_objects.index(oid), scene_name=self.scene_names[sa])
        elif t == T.MULTI_OBJECT:
            m.update(scene_name=self.scene_names[sa])
        elif t == T.SINGLE_OBJECT_ACROSS_SCENE:
            m.update(object_id=self._object_ids[oa], scene_name_a=self.scene_names[sa], scene_name_b=self.scene_names[sb])
        else:
            m.update(object_id_a=self._object_ids[oa], scene_name_a=self.scene_names[sa], object_id_b=self._object_ids[ob],
                     scene_name_b=self.scene_names[sb])
        if t == T.SYNTHETIC_MULTI_OBJECT:
            m.update(image_a1_idx=idx(fr[0]), image_a2_idx=idx(fr[1]), image_a_idx=idx(fr[2]), image_b_idx=idx(fr[3]))
        else:
            m.update(image_a_idx=idx(fr[0]), image_b_idx=idx(fr[1]))
        if not found:
            m["image_b_idx"] = None
        return m

    # ------------------------------------------------------------------------------------------------ gather
    def gather(self, idx_a, idx_b, depth=True):
        """Frames idx_a[b] and idx_b[b] (host ints, 1 to 128 pairs) in the producers' layout, in one launch on the current
        stream: -> (rgb_a, rgb_b) uint8 [B, H, W, 3], (depth_a, depth_b) float32 [B, H, W] millimetres (None if not
        ``depth``), (mask_a, mask_b) uint8 [B, H, W], on the store's device (a pinned store: the current device)."""
        ia = np.ascontiguousarray(np.asarray(idx_a, dtype=np.int64).reshape(-1))
        ib = np.ascontiguousarray(np.asarray(idx_b, dtype=np.int64).reshape(-1))
        B = len(ia)
        if len(ib) != B:
            raise ValueError("idx_a and idx_b must have the same length")
        if not 1 <= B <= N.FRAMES_MAX_PAIRS:
            raise ValueError("gather takes 1 to %d pairs per call (got %d)" % (N.FRAMES_MAX_PAIRS, B))
        if not (self.rgb.is_cuda or self.rgb.is_pinned()):
            raise ValueError("gather reads a 'cuda' or 'pinned' store, not a pageable 'host' one")
        F = self.num_frames
        if ia.min() < 0 or ib.min() < 0 or ia.max() >= F or ib.max() >= F:
            raise ValueError("frame indices must lie in [0, %d)" % F)
        H, W = self.image_shape
        dev = self.rgb.device if self.rgb.is_cuda else torch.device("cuda", torch.cuda.current_device())
        rgb = torch.empty(2, B, H, W, 3, dtype=torch.uint8, device=dev)
        mask = torch.empty(2, B, H, W, dtype=torch.uint8, device=dev)
        dep = torch.empty(2, B, H, W, dtype=torch.float32, device=dev) if depth else None
        ia32, ib32 = ia.astype(np.int32), ib.astype(np.int32)
        vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
        with torch.cuda.device(dev):
            N.check(N.lib.ddn_frames_gather(N.ptr(self.rgb), N.ptr(self.depth), N.ptr(self.mask), F, H, W, vp(ia32), vp(ib32),
                                            B, N.ptr(rgb[0]), N.ptr(rgb[1]), N.ptr(dep[0]) if depth else None,
                                            N.ptr(dep[1]) if depth else None, N.ptr(mask[0]), N.ptr(mask[1]), N.stream_ptr()))
        return (rgb[0], rgb[1]), ((dep[0], dep[1]) if depth else None), (mask[0], mask[1])

    # ------------------------------------------------------------------------------------------------ batches
    def batch(self, types, training_config, generator=None, rng=None):
        """One training batch for ``types`` (CPU int64 [B], ``sampling.draw_data_types``'s output): frames selected by
        ``select(types, rng)``, one gather launch per producer input group, the matching producer per type present
        (``generator``: their CUDA torch.Generator) and ``sampling.concat_batches``.  -> the keys ``get_loss`` /
        ``get_mixed_loss`` consume (as ``concat_batches`` returns them) plus ``metadata`` (one reference metadata dict per
        pair).  Pairs come grouped by type; ``out["metadata"]`` follows the batch order.  A pair for which no image b was
        found is ``empty`` (the reference's return_empty_data): its counts are 0 and its index rows -1, and image A
        stands in for image B.  Batches above a producer's per-call limit are split across calls.  Nothing here
        synchronises with the device."""
        sel = self.select(types, rng)
        parts = []
        for t in np.unique(sel.types):
            r = np.nonzero(sel.types == t)[0]
            step = N.SMO_MAX_PAIRS if t == T.SYNTHETIC_MULTI_OBJECT else N.FRAMES_MAX_PAIRS
            for c0 in range(r[0], r[-1] + 1, step):
                rows = np.arange(c0, min(c0 + step, r[-1] + 1))
                parts.append(self._part(int(t), sel.frames[rows], sel.empty[rows], training_config, generator))
        out = sampling.concat_batches(parts)
        out["metadata"] = sel.metadata
        return out

    def _part(self, t, frames, empty, training_config, generator):
        K = self.K
        if t in (T.SINGLE_OBJECT_ACROSS_SCENE, T.DIFFERENT_OBJECT):
            rgb, _, mask = self.gather(frames[:, 0], frames[:, 1], depth=False)
            return sampling.across_scene_batch(rgb[0], rgb[1], mask[0], mask[1], training_config, generator=generator,
                                               match_type=t)
        rgb, dep, mask = self.gather(frames[:, 0], frames[:, 1])
        pa, pb = self.poses[frames[:, 0]], self.poses[frames[:, 1]]
        if t == T.SYNTHETIC_MULTI_OBJECT:
            rgb2, dep2, mask2 = self.gather(frames[:, 2], frames[:, 3])
            out = sampling.synthetic_multi_object_batch(
                (rgb[0], rgb[1], dep[0], dep[1], mask[0], mask[1], pa, pb),
                (rgb2[0], rgb2[1], dep2[0], dep2[1], mask2[0], mask2[1], self.poses[frames[:, 2]], self.poses[frames[:, 3]]),
                K, training_config, generator=generator)
        else:
            out = sampling.within_scene_batch(rgb[0], rgb[1], dep[0], dep[1], mask[0], mask[1], pa, pb, K, training_config,
                                              generator=generator)
            out["match_type"] = torch.full_like(out["match_type"], t)       # MULTI_OBJECT: same producer, multi-object scene
        n_ok = int((~empty).sum())                                          # the empty pairs are the last rows
        if n_ok < len(empty):
            for k in sampling.INDEX_KEYS:
                out[k][n_ok:] = -1
            out["counts"][n_ok:] = 0
            out["empty"][n_ok:] = True
        return out
