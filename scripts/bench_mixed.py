"""Mixed pair-type training steps: 8 pairs of 640x480, D = 3, Resnet34_8s, the reference's default training config
(training.yaml: 10000 matching attempts, 75 + 75 non-matches per match, cross_scene_num_samples 10000).

Arms, each timed as producers + concat_batches + forward_pair + loss + backward:
  within         8 within-scene pairs, get_loss (no concat: the one-type path)
  within_mixed   the same 8 pairs through concat_batches + get_mixed_loss (what the pair-type path adds to a uniform step)
  hats           6 within-scene + 2 DIFFERENT_OBJECT, get_mixed_loss
  shoes          3 within-scene + 3 DIFFERENT_OBJECT + 2 SYNTHETIC_MULTI_OBJECT, get_mixed_loss

    python scripts/bench_mixed.py [--reps 7] [--iters 10]

Every arm is warmed up, then the arms alternate in one process, `--reps` rounds of `--iters` steps each timed with CUDA
events; the JSON line gives each arm's per-round ms per step (median, min, max), its library launches per step and the
time of concat_batches alone.  A separate torch.profiler pass (3 steps per arm, after the timed rounds) gives per-kernel
device times: the loss gather / scatter (4 terms under get_loss, 5 under get_mixed_loss), the compose kernels and the
copies of concat_batches.  GPU name, SM clock, max SM clock and power limit (nvidia-smi, query only) are printed with the
numbers, before and after."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import torch  # noqa: E402

import pdc_b200  # noqa: E402
from pdc_b200 import _native as N  # noqa: E402
from pdc_b200 import loss_composer  # noqa: E402
from pdc_b200 import sampling as S  # noqa: E402
from pdc_b200.synthetic import plane_scene_pairs  # noqa: E402
from bench_producer import gpu_info  # noqa: E402

H, W, D = 480, 640, 3
DEFAULT = {"training": dict(num_matching_attempts=10000, num_non_matches_per_match=150, fraction_masked_non_matches=0.5,
                            fraction_background_non_matches=0.5, sample_matches_only_off_mask=True, domain_randomize=True,
                            use_image_b_mask_inv=True, cross_scene_num_samples=10000)}


def plane_pairs(B, seed, dev):
    x, K = plane_scene_pairs(B, H, W, seed)
    return {k: v.to(dev) if isinstance(v, torch.Tensor) else v for k, v in x.items()}, K


class Producers(object):
    """Inputs for up to 8 pairs of each type, made once; each call draws fresh random numbers on the device."""

    def __init__(self, dev):
        self.gen = torch.Generator(device=dev).manual_seed(0)
        self.x, self.K = plane_pairs(8, 1, dev)
        self.y, _ = plane_pairs(8, 2, dev)

    def _rows(self, x, n):
        return {k: v[:n] for k, v in x.items()}

    def within(self, n):
        x = self._rows(self.x, n)
        return S.within_scene_batch(x["rgb_a"], x["rgb_b"], x["depth_a"], x["depth_b"], x["mask_a"], x["mask_b"],
                                    x["pose_a"], x["pose_b"], self.K, DEFAULT, generator=self.gen)

    def different(self, n):
        x = self._rows(self.y, n)
        return S.across_scene_batch(x["rgb_a"], x["rgb_b"], x["mask_a"], x["mask_b"], DEFAULT, generator=self.gen)

    def synthetic(self, n):
        tup = lambda x: (x["rgb_a"], x["rgb_b"], x["depth_a"], x["depth_b"], x["mask_a"], x["mask_b"], x["pose_a"], x["pose_b"])
        return S.synthetic_multi_object_batch(tup(self._rows(self.x, n)), tup(self._rows(self.y, n)), self.K, DEFAULT,
                                              generator=self.gen)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    rows = {"gpu": gpu_info(), "B": 8, "H": H, "W": W, "D": D}
    prod = Producers(dev)
    dcn = pdc_b200.DenseCorrespondenceNetwork.from_config({"descriptor_dimension": D, "image_width": W, "image_height": H},
                                                          load_stored_params=False)
    pcl = pdc_b200.PixelwiseContrastiveLoss(dcn.image_shape, dict(pdc_b200.DEFAULT_LOSS_CONFIG))

    def step(batch, loss_fn):
        B = batch["image_a"].shape[0]
        a, b = dcn.forward_pair(batch["image_a"], batch["image_b"])
        five = loss_fn(pcl, batch["match_type"], dcn.process_network_output(a, B), dcn.process_network_output(b, B),
                       *[batch[k] for k in S.INDEX_KEYS], num_valid=batch["num_valid"])
        five[0].backward()

    mixes = {"within_mixed": lambda: [prod.within(8)],
             "hats": lambda: [prod.within(6), prod.different(2)],
             "shoes": lambda: [prod.within(3), prod.different(3), prod.synthetic(2)]}
    arms = {"within": lambda: step(prod.within(8), loss_composer.get_loss)}
    for name, parts in mixes.items():
        arms[name] = (lambda parts: lambda: step(S.concat_batches(parts()), loss_composer.get_mixed_loss))(parts)

    for fn in arms.values():                                     # warm-up: every shape the timed rounds use
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    for name, fn in arms.items():
        n0 = N.launch_count()
        fn()
        rows[name + "_launches_per_step"] = N.launch_count() - n0
    times = {name: [] for name in arms}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.reps):
        for name, fn in arms.items():
            torch.cuda.synchronize()
            e0.record()
            for _ in range(args.iters):
                fn()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / args.iters)
    for name, t in times.items():
        rows[name + "_ms"] = {"median": statistics.median(t), "min": min(t), "max": max(t), "rounds": t}

    # concat_batches alone on ready parts
    for name in ("hats", "shoes"):
        parts = mixes[name]()
        for _ in range(3):
            S.concat_batches(parts)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(20):
            S.concat_batches(parts)
        e1.record()
        torch.cuda.synchronize()
        rows[name + "_concat_ms"] = e0.elapsed_time(e1) / 20
    rows["gpu_after_timing"] = gpu_info()

    # per-kernel device times, in a run of their own
    from torch.profiler import ProfilerActivity, profile
    keep = ("loss", "compose", "Cat", "copy", "fill", "where", "Fill")
    prof_rows = {}
    for name, fn in arms.items():
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
        k = {}
        for e in prof.key_averages():
            t = getattr(e, "self_device_time_total", 0) or getattr(e, "self_cuda_time_total", 0)
            if t > 0 and any(s in e.key for s in keep):
                k[e.key[:110]] = {"us_per_step": t / 3.0, "launches_per_step": e.count / 3.0}
        prof_rows[name] = k
    rows["profile"] = prof_rows
    print(json.dumps(rows))


if __name__ == "__main__":
    main()
