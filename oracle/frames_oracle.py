"""Restatement of SpartanDataset's pair selection (dense_correspondence/dataset/spartan_dataset_masked.py, and
dense_correspondence_dataset_masked.py for get_img_idx_with_different_pose) for one pair, with its uniform numbers given.

TEST INFRASTRUCTURE: tests/test_frames_cpu.py requires pdc_b200.frames.FrameStore.select_from_uniforms to pick the same
scenes and images.  The methods are restated one by one, in the reference's control flow (one draw at a time, the angle
test included), so they share nothing with the vectorised library code but the uniform layout:

    row[0], row[1]   the object draws           row[2]           scene A
    row[3], row[4]   scene B draws              row[5]           image a of scene A, row[6:56] its image-b attempts
    row[56]          image a of scene B (image b of an across-scene pair), row[57:107] its image-b attempts

``random.choice(seq)`` with uniform u is seq[min(floor(u * len), len - 1)]; ``np.random.choice(arange(n), 2,
replace=False)`` with (u, v) is (i, j) with i = choice(u, n), j = choice(v, n - 1) + (that >= i).  Python 2's
``pose_data.keys()`` has no defined order; the restatement uses the keys sorted.

``ds`` holds the dataset's tables as SpartanDataset holds them: ``single`` {object_id: {"train": [...], "test": [...]}}
(_single_object_scene_dict, in config order), ``multi`` {"train": [...], "test": [...]}, ``pose_data`` {scene:
{image index: 4x4 camera_to_world}} and ``mode``.
"""
import numpy as np

THRESHOLD, ANGLE_THRESHOLD, NUM_ATTEMPTS = 0.2, 20, 50


def _choice(seq, u):
    return seq[min(int(u * len(seq)), len(seq) - 1)]


def _choice2(n, u, v):
    i = min(int(u * n), n - 1)
    j = min(int(v * (n - 1)), n - 2)
    return i, j + (j >= i)


def quaternion_from_matrix(M):
    """transformations.quaternion_from_matrix(isprecise=False) (utils/transformations.py:1281-1355): the eigenvector of
    the largest eigenvalue of the symmetric K, [w, x, y, z] with w >= 0."""
    m00, m01, m02 = M[0, 0], M[0, 1], M[0, 2]
    m10, m11, m12 = M[1, 0], M[1, 1], M[1, 2]
    m20, m21, m22 = M[2, 0], M[2, 1], M[2, 2]
    K = np.array([[m00 - m11 - m22, 0.0, 0.0, 0.0],
                  [m01 + m10, m11 - m00 - m22, 0.0, 0.0],
                  [m02 + m20, m12 + m21, m22 - m00 - m11, 0.0],
                  [m21 - m12, m02 - m20, m10 - m01, m00 + m11 + m22]]) / 3.0
    w, V = np.linalg.eigh(K)
    q = V[[3, 0, 1, 2], np.argmax(w)]
    return -q if q[0] < 0.0 else q


def compute_angle_between_poses(pose_a, pose_b):
    """utils.py:243-275: radians."""
    q, r = quaternion_from_matrix(pose_a), quaternion_from_matrix(pose_b)
    return 2 * np.arccos(2 * np.dot(q, r) ** 2 - 1)


class Pair:
    def __init__(self, ds, row):
        self.ds, self.row = ds, row

    def get_random_image_index(self, scene_name, u):                      # :408-420
        return _choice(sorted(self.ds["pose_data"][scene_name]), u)

    def get_img_idx_with_different_pose(self, scene_name, pose_a, us):     # dense_correspondence_dataset_masked.py:260-287
        counter = 0
        while counter < NUM_ATTEMPTS:
            img_idx = self.get_random_image_index(scene_name, us[counter])
            pose = self.ds["pose_data"][scene_name][img_idx]
            diff = np.linalg.norm(pose_a[0:3, 3] - pose[0:3, 3])
            angle_diff = compute_angle_between_poses(pose_a, pose)           # radians against 20: never fires
            if (diff > THRESHOLD) or (angle_diff > ANGLE_THRESHOLD):
                return img_idx
            counter += 1
        return None

    def within_scene(self, scene_name, start):                            # get_within_scene_data :627-639
        a = self.get_random_image_index(scene_name, self.row[start])
        b = self.get_img_idx_with_different_pose(scene_name, self.ds["pose_data"][scene_name][a],
                                                 self.row[start + 1:start + 1 + NUM_ATTEMPTS])
        return a, b

    def objects(self):
        return list(self.ds["single"].keys())

    def scenes(self, object_id):
        return self.ds["single"][object_id][self.ds["mode"]]

    def two_different_object_ids(self):                                   # :476-494
        ids = self.objects()
        i, j = _choice2(len(ids), self.row[0], self.row[1])
        return ids[i], ids[j]


def select(ds, t, row):
    """One pair of type t (SpartanDatasetDataType value) -> dict(scene_a, scene_b, images_a, images_b): images_* are
    (image a, image b) of each scene, image b None when no frame qualified."""
    p = Pair(ds, row)
    if t == 0:                                                            # get_single_object_within_scene_data :543-559
        object_id = _choice(p.objects(), row[0])
        scene = _choice(p.scenes(object_id), row[2])
        return dict(scene_a=scene, scene_b=None, images_a=p.within_scene(scene, 5), images_b=None)
    if t == 3:                                                            # get_multi_object_within_scene_data :561-575
        scene = _choice(ds["multi"][ds["mode"]], row[2])
        return dict(scene_a=scene, scene_b=None, images_a=p.within_scene(scene, 5), images_b=None)
    if t in (1, 2):
        if t == 1:                                                        # get_single_object_across_scene_data :860-872
            object_id = _choice(p.objects(), row[0])
            scene_a = _choice(p.scenes(object_id), row[2])
            scene_list = p.scenes(object_id)                              # get_different_scene_for_object :453-474
            scene_b = None
            for idx in _choice2(len(scene_list), row[3], row[4]):
                if scene_list[idx] != scene_a:
                    scene_b = scene_list[idx]
                    break
        else:                                                             # get_different_object_data :874-888
            oa, ob = p.two_different_object_ids()
            scene_a, scene_b = _choice(p.scenes(oa), row[2]), _choice(p.scenes(ob), row[3])
        # get_across_scene_data :1077-1084
        return dict(scene_a=scene_a, scene_b=scene_b, images_a=(p.get_random_image_index(scene_a, row[5]), None),
                    images_b=(p.get_random_image_index(scene_b, row[56]), None))
    oa, ob = p.two_different_object_ids()                                 # get_synthetic_multi_object_within_scene_data
    scene_a, scene_b = _choice(p.scenes(oa), row[2]), _choice(p.scenes(ob), row[3])      # :890-905
    return dict(scene_a=scene_a, scene_b=scene_b, images_a=p.within_scene(scene_a, 5), images_b=p.within_scene(scene_b, 56))
