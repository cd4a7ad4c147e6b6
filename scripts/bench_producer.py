"""Within-scene batch producer: B = 8 pairs at 640x480, the reference's default training config (training.yaml:16-22).

Rows (one JSON object on stdout; needs a GPU):
  producer_ms          draw_within_scene_rand + within_scene_batch per batch (CUDA events, warm-up, >= 20 iterations)
  producer_call_ms     within_scene_batch alone, random numbers drawn beforehand
  launches_per_call    library kernel launches of one within_scene_batch call
  step_ms / step_with_producer_ms
                       forward_pair + get_loss(num_valid) + backward (Resnet34_8s, D = 3) on a batch produced beforehand,
                       and the same step preceded by the producer
  reference_cpu_ms_per_pair
                       the reference's own functions (oracle/_ref, built by oracle/build_ref_augment.py) for one pair on one
                       host thread with the same random numbers; "not available" when oracle/_ref is missing.  PNG decoding
                       is not included on either side.
GPU name, SM clock and power limit (nvidia-smi, query only) and os.cpu_count() are printed with the numbers."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import pdc_b200  # noqa: E402
from pdc_b200 import _native as N  # noqa: E402
from pdc_b200 import loss_composer  # noqa: E402
from pdc_b200 import sampling as S  # noqa: E402

B, H, W, D = 8, 480, 640, 3
ITERS, WARM = int(os.environ.get("PRODUCER_ITERS", "20")), 3
DEV = torch.device("cuda", 0)
TC = {"training": dict(num_matching_attempts=10000, num_non_matches_per_match=150, fraction_masked_non_matches=0.5,
                       fraction_background_non_matches=0.5, sample_matches_only_off_mask=True, domain_randomize=True,
                       use_image_b_mask_inv=True)}


def gpu_info():
    try:
        q = "name,clocks.sm,clocks.max.sm,power.limit"
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as e:             # the numbers are still device-timed; only the label is missing
        return "nvidia-smi unavailable (%s); %s" % (e, torch.cuda.get_device_name(0))


def timed(fn):
    for _ in range(WARM):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(ITERS):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / ITERS


def inputs():
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_gpu_within_scene import scene
    xs = scene(B, H, W, 1)
    t = lambda k: torch.from_numpy(np.stack([x[k] for x in xs])).to(DEV)
    return xs, (t("rgb_a"), t("rgb_b"), t("depth_a"), t("depth_b"), t("mask_a"), t("mask_b"),
                np.stack([x["pose_a"] for x in xs]), np.stack([x["pose_b"] for x in xs]), xs[0]["K"])


def reference_cpu(xs, rand):
    from oracle import build_ref_augment
    from oracle import within_scene_oracle as WO
    if not build_ref_augment.built():
        return "not available"
    fns = WO.executed_reference(build_ref_augment.load())
    cfg = S.within_scene_cfg(TC)
    torch.set_num_threads(1)
    r = {k: v[0].cpu().numpy() for k, v in rand.items()}
    x = xs[0]
    t0 = time.perf_counter()
    WO.get_within_scene_data(fns, x["rgb_a"], x["rgb_b"], x["depth_a"], x["depth_b"], x["mask_a"], x["mask_b"], x["pose_a"],
                             x["pose_b"], x["K"], cfg, r)
    return 1e3 * (time.perf_counter() - t0)


def main():
    xs, args = inputs()
    gen = torch.Generator(device=DEV).manual_seed(0)
    rand = S.draw_within_scene_rand(B, H, W, TC, generator=gen)
    rows = {"gpu": gpu_info(), "B": B, "H": H, "W": W, "iters": ITERS, "cpu_count": os.cpu_count()}
    rows["producer_ms"] = timed(lambda: S.within_scene_batch(*args, TC, generator=gen))
    rows["producer_call_ms"] = timed(lambda: S.within_scene_batch(*args, TC, rand=rand))
    n0 = N.launch_count()
    out = S.within_scene_batch(*args, TC, rand=rand)
    rows["launches_per_call"] = N.launch_count() - n0
    rows["mean_counts"] = [float(c) for c in out["counts"].double().mean(0).cpu()]

    dcn = pdc_b200.DenseCorrespondenceNetwork.from_config({"descriptor_dimension": D, "image_width": W, "image_height": H},
                                                          load_stored_params=False)
    pcl = pdc_b200.PixelwiseContrastiveLoss(dcn.image_shape, dict(pdc_b200.DEFAULT_LOSS_CONFIG))
    keys = [k % s for k in ("matches_%s", "masked_non_matches_%s", "background_non_matches_%s", "blind_non_matches_%s") for s in "ab"]

    def step(o):
        a, b = dcn.forward_pair(o["image_a"], o["image_b"])
        five = loss_composer.get_loss(pcl, o["match_type"], dcn.process_network_output(a, B), dcn.process_network_output(b, B),
                                      *[o[k] for k in keys], num_valid=o["num_valid"])
        five[0].backward()

    rows["step_ms"] = timed(lambda: step(out))
    rows["step_with_producer_ms"] = timed(lambda: step(S.within_scene_batch(*args, TC, generator=gen)))
    rows["reference_cpu_ms_per_pair"] = reference_cpu(xs, rand)
    rows["gpu_after"] = gpu_info()
    print(json.dumps(rows))


if __name__ == "__main__":
    main()
