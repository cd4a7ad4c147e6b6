"""Device-resident training frames (pdc_b200.frames.FrameStore) against decoding PNGs in DataLoader workers.

Writes synthetic scenes in the reference's on-disk layout (pdc_b200.synthetic.write_reference_scenes: 640x480 PNGs) into
a temporary directory, then reports
  (a) store build time per frame (decode once + copy), for the device and the pinned-host store;
  (b) ddn_frames_gather alone for 8 pairs with depth (CUDA events over many launches) and as bandwidth (bytes read +
      written over kernel time), for both stores;
  (c) full training steps on the shoes mix (3 within-scene + 3 DIFFERENT_OBJECT + 2 SYNTHETIC_MULTI_OBJECT, 8 pairs,
      D = 3, the reference's default training config):
        store   FrameStore.batch -> forward_pair -> get_mixed_loss -> backward -> FusedAdam
        loader  INTEGRATION.md's DataLoader loop: --workers processes decode each step's PNGs (the same selections), the
                main process copies them to the device and calls the producers, then the same step.
      Each arm's pairs/s (host clock around --iters steps ending in a device synchronise) and host CPU seconds per step
      (resource.getrusage, this process plus its reaped children, i.e. the workers), alternated for --reps rounds.

    python scripts/bench_frames.py [--frames-per-scene 16] [--workers 4] [--reps 3] [--iters 20]

GPU name, SM clock, max SM clock and power limit (nvidia-smi, query only) are printed with the numbers."""
import argparse
import json
import os
import resource
import shutil
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import pdc_b200  # noqa: E402
from pdc_b200 import frames as FR  # noqa: E402
from pdc_b200 import loss_composer  # noqa: E402
from pdc_b200 import sampling as S  # noqa: E402
from pdc_b200 import synthetic  # noqa: E402
from bench_producer import gpu_info  # noqa: E402

H, W, D = 480, 640, 3
T = loss_composer.SpartanDatasetDataType
SHOES = [T.SINGLE_OBJECT_WITHIN_SCENE] * 3 + [T.DIFFERENT_OBJECT] * 3 + [T.SYNTHETIC_MULTI_OBJECT] * 2
DEFAULT = {"training": dict(num_matching_attempts=10000, num_non_matches_per_match=150, fraction_masked_non_matches=0.5,
                            fraction_background_non_matches=0.5, sample_matches_only_off_mask=True, domain_randomize=True,
                            use_image_b_mask_inv=True, cross_scene_num_samples=10000)}


def write_dataset(root, n):
    g = np.random.RandomState(0)
    scenes = {}
    for s in ("a0", "a1", "b0", "b1"):
        frames = []
        for i in range(n):
            r = g.randn(3) * 0.05
            q = np.array([1.0, r[0], r[1], r[2]]); q /= np.linalg.norm(q)
            frames.append((i, tuple(q), tuple(g.randn(3) * 0.25)))
        scenes[s] = frames
    synthetic.write_reference_scenes(root, scenes, H, W, seed=1)
    return {"logs_root_path": root,
            "single_object_scenes_config_files": [{"object_id": "x", "train": ["a0", "a1"], "test": []},
                                                  {"object_id": "y", "train": ["b0", "b1"], "test": []}],
            "multi_object_scenes_config_files": []}


def cpu_seconds():
    s, c = resource.getrusage(resource.RUSAGE_SELF), resource.getrusage(resource.RUSAGE_CHILDREN)
    return s.ru_utime + s.ru_stime + c.ru_utime + c.ru_stime


class StepFrames(torch.utils.data.Dataset):
    """One item = one step's frames decoded from PNG (what a DataLoader worker does for INTEGRATION.md's loop)."""

    def __init__(self, store, root, selections):
        self.files = []
        for sel in selections:
            fr = []
            for row in sel.frames:
                fr.append([self._paths(store, root, f) if f >= 0 else None for f in row])
            self.files.append(fr)

    @staticmethod
    def _paths(store, root, f):
        s = int(np.searchsorted(store.scene_start, f, side="right") - 1)
        d = os.path.join(root, store.scene_names[s])
        i = int(store.image_index[f])
        return [os.path.join(d, p % i) for p in (FR.RGB_FILE, FR.DEPTH_FILE, FR.MASK_FILE)]

    def __len__(self):
        return len(self.files)

    def __getitem__(self, k):
        out = []
        for row in self.files[k]:
            out.append([None if p is None else (torch.from_numpy(np.array(FR.decode_rgb(p[0]))),
                                                torch.from_numpy(FR.decode_depth(p[1]).astype(np.float32)),
                                                torch.from_numpy(np.array(FR.decode_mask(p[2])))) for p in row])
        return out


def loader_batch(item, sel, store, gen, dev):
    parts = []
    for t in np.unique(sel.types):
        rows = np.nonzero(sel.types == t)[0]
        col = lambda c, j: torch.stack([item[r][c][j] for r in rows]).to(dev, non_blocking=True)
        pose = lambda c: store.poses[sel.frames[rows, c]]
        if t == T.DIFFERENT_OBJECT:
            parts.append(S.across_scene_batch(col(0, 0), col(1, 0), col(0, 2), col(1, 2), DEFAULT, generator=gen))
        elif t == T.SINGLE_OBJECT_WITHIN_SCENE:
            parts.append(S.within_scene_batch(col(0, 0), col(1, 0), col(0, 1), col(1, 1), col(0, 2), col(1, 2), pose(0), pose(1),
                                              store.K, DEFAULT, generator=gen))
        else:
            tup = lambda a, b: (col(a, 0), col(b, 0), col(a, 1), col(b, 1), col(a, 2), col(b, 2), pose(a), pose(b))
            parts.append(S.synthetic_multi_object_batch(tup(0, 1), tup(2, 3), store.K, DEFAULT, generator=gen))
    return S.concat_batches(parts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames-per-scene", type=int, default=16)
    ap.add_argument("--workers", type=int, default=4)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    rows = {"gpu": gpu_info(), "B": 8, "H": H, "W": W, "D": D, "workers": args.workers, "host_cpus": os.cpu_count()}
    tmp = tempfile.mkdtemp(prefix="bench_frames_")
    cfg = write_dataset(tmp, args.frames_per_scene)

    # (a) store build
    stores = {}
    for storage in ("cuda", "pinned"):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        stores[storage] = FR.FrameStore.from_dataset_config(cfg, storage=storage)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        rows["build_ms_per_frame_" + storage] = 1e3 * dt / stores[storage].num_frames
    store = stores["cuda"]
    rows["frames"] = store.num_frames

    # (b) the gather launch alone, 8 pairs with depth
    B, P = 8, H * W
    rng = np.random.default_rng(0)
    ia, ib = rng.integers(0, store.num_frames, B), rng.integers(0, store.num_frames, B)
    nbytes = 2 * B * P * ((3 + 2 + 1) + (3 + 4 + 1))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for storage, st in stores.items():
        for _ in range(5):
            st.gather(ia, ib)
        torch.cuda.synchronize()
        n = 200
        e0.record()
        for _ in range(n):
            st.gather(ia, ib)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / n
        rows["gather_us_" + storage] = 1e3 * ms
        rows["gather_GBps_" + storage] = nbytes / (ms * 1e-3) / 1e9
        rows["gather_read_GBps_" + storage] = 2 * B * P * 6 / (ms * 1e-3) / 1e9    # the store side (the host link if pinned)
    rows["gather_bytes"] = nbytes

    # (c) full training steps, store-fed against DataLoader-fed, alternated
    dcn = pdc_b200.DenseCorrespondenceNetwork.from_config({"descriptor_dimension": D, "image_width": W, "image_height": H},
                                                          load_stored_params=False)
    pcl = pdc_b200.PixelwiseContrastiveLoss(dcn.image_shape, dict(pdc_b200.DEFAULT_LOSS_CONFIG))
    opt = pdc_b200.FusedAdam(dcn, lr=1e-4)
    gen = torch.Generator(device=dev).manual_seed(0)
    types = torch.tensor(SHOES, dtype=torch.int64)

    def train(batch):
        a, b = dcn.forward_pair(batch["image_a"], batch["image_b"])
        five = loss_composer.get_mixed_loss(pcl, batch["match_type"], dcn.process_network_output(a, B),
                                            dcn.process_network_output(b, B), *[batch[k] for k in S.INDEX_KEYS],
                                            num_valid=batch["num_valid"])
        opt.zero_grad()
        five[0].backward()
        opt.step()

    sel_rng = np.random.default_rng(1)

    def store_round(iters):
        for _ in range(iters):
            train(store.batch(types, DEFAULT, generator=gen, rng=sel_rng))

    def loader_round(iters):
        sels = [store.select(types, sel_rng) for _ in range(iters)]
        dl = torch.utils.data.DataLoader(StepFrames(store, tmp, sels), batch_size=None, num_workers=args.workers,
                                         pin_memory=True, prefetch_factor=2)
        it = iter(dl)
        for sel, item in zip(sels, it):
            train(loader_batch(item, sel, store, gen, dev))
        del it, dl                                          # join the workers, so their CPU time is counted

    arms = {"store": store_round, "loader": loader_round}
    for fn in arms.values():
        fn(3)
    torch.cuda.synchronize()
    res = {k: {"pairs_per_s": [], "cpu_s_per_step": []} for k in arms}
    for _ in range(args.reps):
        for name, fn in arms.items():
            torch.cuda.synchronize()
            c0, t0 = cpu_seconds(), time.perf_counter()
            fn(args.iters)
            torch.cuda.synchronize()
            t1, c1 = time.perf_counter(), cpu_seconds()
            res[name]["pairs_per_s"].append(B * args.iters / (t1 - t0))
            res[name]["cpu_s_per_step"].append((c1 - c0) / args.iters)
    for name, r in res.items():
        for k, v in r.items():
            rows["%s_%s" % (name, k)] = {"median": statistics.median(v), "min": min(v), "max": max(v)}
    rows["gpu_after_timing"] = gpu_info()
    shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps(rows))


if __name__ == "__main__":
    main()
