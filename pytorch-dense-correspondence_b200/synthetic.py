"""Seeded synthetic inputs shaped like what SpartanDataset.__getitem__ hands the training loop
(dense_correspondence/dataset/spartan_dataset_masked.py:111-151, :841-858): mean/std-normalised
RGB images and flat pixel indices n = u + W*v (doc/coordinate_conventions.md), with
``non_matches_a`` being every match repeated k times consecutively (spartan_dataset_masked.py:853-854).

Pure CPU torch with an explicit generator, so the same call reproduces the same tensors in the
build container and on the GPU box (SURVEY.md section 8d).  ``plane_scene_pairs`` gives the raw inputs of the device
batch producers in ``sampling`` (uint8 RGB, masks, depth in millimetres, camera poses) for a ray-cast plane.
"""
import numpy as np
import torch


def make_pair_batch(B, H=480, W=640, num_matches=1000, num_masked=1000, num_background=1000,
                    num_blind=0, seed=1):
    """Returns a dict of CPU tensors:
    img_a/img_b [B,3,H,W] fp32; matches_a/b [B,Nm]; masked_a/b [B,Nn_m]; background_a/b [B,Nn_b];
    blind_a/b [B,Nn_x] or None -- all int64 flat indices in [0, H*W)."""
    g = torch.Generator().manual_seed(seed)
    P = H * W
    out = {
        "img_a": torch.randn(B, 3, H, W, generator=g),
        "img_b": torch.randn(B, 3, H, W, generator=g),
        "matches_a": torch.randint(0, P, (B, num_matches), generator=g),
        "matches_b": torch.randint(0, P, (B, num_matches), generator=g),
    }

    def non_matches(n):
        if n == 0:
            return None, None
        k = max(n // num_matches, 1)
        a = out["matches_a"].repeat_interleave(k, dim=1)[:, :n]
        if a.shape[1] < n:  # n not a multiple of Nm: pad with fresh samples
            a = torch.cat([a, torch.randint(0, P, (B, n - a.shape[1]), generator=g)], 1)
        b = torch.randint(0, P, (B, n), generator=g)
        return a.contiguous(), b

    out["masked_a"], out["masked_b"] = non_matches(num_masked)
    out["background_a"], out["background_b"] = non_matches(num_background)
    out["blind_a"], out["blind_b"] = non_matches(num_blind)
    return out


def plane_scene_pairs(B, H, W, seed, empty=()):
    """B image pairs of a ray-cast tilted plane seen from two nearby camera poses, with random RGB and blob masks: the
    inputs of ``sampling.within_scene_batch`` / ``across_scene_batch`` / ``synthetic_multi_object_batch`` (one scene).
    mask_a of the pairs whose index is in ``empty`` is all zero (every producer's return_empty_data).
    -> (dict of CPU tensors ``rgb_a/b`` uint8 [B, H, W, 3], ``depth_a/b`` float32 [B, H, W] (millimetres), ``mask_a/b``
    uint8 [B, H, W], and numpy ``pose_a/b`` [B, 4, 4] camera-to-world; K, the 3x3 intrinsics scaled from 640x480)."""
    K = np.array([[533.6422696034836 * W / 640, 0, 319.4091030774892 * W / 640], [0, 534.7824445233571 * H / 480,
                  236.4374299691866 * H / 480], [0, 0, 1.0]])
    g = np.random.RandomState(seed)

    def pose(rx, ry, t):
        cx, sx, cy, sy = np.cos(rx), np.sin(rx), np.cos(ry), np.sin(ry)
        Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]); Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
        T4 = np.eye(4); T4[:3, :3] = Ry.dot(Rx); T4[:3, 3] = t
        return T4

    us, vs = np.meshgrid(np.arange(W), np.arange(H))
    rays = np.linalg.inv(K).dot(np.stack([us.ravel(), vs.ravel(), np.ones(H * W)]))

    def render(T4):
        nrm, d0 = np.array([-0.1, 0.05, 1.0]), 1.2
        s = (d0 - nrm.dot(T4[:3, 3])) / nrm.dot(T4[:3, :3].dot(rays))
        return np.round(s * 1000.0).reshape(H, W).astype(np.float32)

    x = {k: [] for k in ("rgb_a", "rgb_b", "depth_a", "depth_b", "mask_a", "mask_b", "pose_a", "pose_b")}
    for b in range(B):
        pa = pose(0.02 * g.randn(), 0.02 * g.randn(), [0, 0, 0]); pb = pose(0.05 * g.randn(), 0.1 * g.randn(), 0.05 * g.randn(3))
        mask_a = (g.rand(H, W) > 0.1).astype(np.uint8); mask_a[: H // 4] = 0
        mask_b = (g.rand(H, W) > 0.2).astype(np.uint8); mask_b[:, : W // 3] = 0
        if b in empty:
            mask_a[:] = 0
        for k, v in (("rgb_a", g.randint(0, 256, (H, W, 3))), ("rgb_b", g.randint(0, 256, (H, W, 3))),
                     ("depth_a", render(pa)), ("depth_b", render(pb)), ("mask_a", mask_a), ("mask_b", mask_b),
                     ("pose_a", pa), ("pose_b", pb)):
            x[k].append(v)
    dt = dict(rgb_a=torch.uint8, rgb_b=torch.uint8, depth_a=torch.float32, depth_b=torch.float32, mask_a=torch.uint8,
              mask_b=torch.uint8)
    return {k: torch.from_numpy(np.stack(v)).to(dt[k]) if k in dt else np.stack(v) for k, v in x.items()}, K


def write_reference_scenes(root, scenes, H, W, seed=0, object_fraction=0.3):
    """Write scenes in the reference's on-disk layout (SpartanDataset.get_image_filename / get_pose_data /
    get_camera_intrinsics): ``root/<scene>/processed/images/%06d_rgb.png``, ``rendered_images/%06d_depth.png`` (16-bit
    millimetres), ``image_masks/%06d_mask.png``, ``images/pose_data.yaml`` and ``images/camera_info.yaml``.
    ``scenes``: {name: [(image index, quaternion (w, x, y, z), translation (x, y, z)), ...]}.  Each image is a ray-cast
    tilted plane seen from its pose, with a smooth random RGB texture and a rectangular object mask covering about
    ``object_fraction`` of it.  -> K, the 3x3 intrinsics written (scaled from 640x480)."""
    import os
    import yaml
    from PIL import Image
    from .frames import pose_from_dict
    K = np.array([[533.6422696034836 * W / 640, 0, 319.4091030774892 * W / 640], [0, 534.7824445233571 * H / 480,
                  236.4374299691866 * H / 480], [0, 0, 1.0]])
    g = np.random.RandomState(seed)
    us, vs = np.meshgrid(np.arange(W), np.arange(H))
    rays = np.linalg.inv(K).dot(np.stack([us.ravel(), vs.ravel(), np.ones(H * W)]))
    ramp = (np.stack([us / max(W - 1, 1), vs / max(H - 1, 1), (us + vs) / max(W + H - 2, 1)], axis=2) * 160).astype(np.int64)
    side = np.sqrt(object_fraction)
    for name, frames in scenes.items():
        d = os.path.join(root, name, "processed")
        for sub in ("images", "rendered_images", "image_masks"):
            os.makedirs(os.path.join(d, sub), exist_ok=True)
        pose_data = {}
        for idx, q, t in frames:
            cam = {"quaternion": dict(zip("wxyz", map(float, q))), "translation": dict(zip("xyz", map(float, t)))}
            pose_data[int(idx)] = {"camera_to_world": cam, "rgb_image_filename": "%06d_rgb.png" % idx,
                                   "depth_image_filename": "%06d_depth.png" % idx}
            T4 = pose_from_dict(cam)
            nrm, d0 = np.array([-0.1, 0.05, 1.0]), 1.2 + float(T4[2, 3])
            s = (d0 - nrm.dot(T4[:3, 3])) / nrm.dot(T4[:3, :3].dot(rays))
            depth = np.clip(np.round(s * 1000.0), 0, 65535).reshape(H, W).astype(np.uint16)
            rgb = np.clip(ramp + g.randint(0, 64, (1, 1, 3)) + g.randint(0, 32, (H, W, 3)), 0, 255).astype(np.uint8)
            mask = np.zeros((H, W), dtype=np.uint8)
            h, w = max(1, int(H * side)), max(1, int(W * side))
            y0, x0 = g.randint(0, H - h + 1), g.randint(0, W - w + 1)
            mask[y0:y0 + h, x0:x0 + w] = 1
            Image.fromarray(rgb).save(os.path.join(d, "images", "%06d_rgb.png" % idx))
            Image.fromarray(depth).save(os.path.join(d, "rendered_images", "%06d_depth.png" % idx))
            Image.fromarray(mask).save(os.path.join(d, "image_masks", "%06d_mask.png" % idx))
        with open(os.path.join(d, "images", "pose_data.yaml"), "w") as f:
            yaml.safe_dump(pose_data, f, default_flow_style=False)
        with open(os.path.join(d, "images", "camera_info.yaml"), "w") as f:
            yaml.safe_dump({"camera_matrix": {"cols": 3, "rows": 3, "data": [float(v) for v in K.ravel()]},
                            "image_width": W, "image_height": H}, f, default_flow_style=False)
    return K
