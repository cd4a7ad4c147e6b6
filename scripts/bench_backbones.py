"""Resnet34_8s against Resnet50_8s in one process, on the same batches: 8 image pairs of 640x480, D = 3, bf16x3.

Per backbone:
  - training step: forward_pair + get_loss (fused-upsample loss) + backward, image pairs per second;
  - forward only at batch 16, train-mode and eval-mode BatchNorm (eval: no gradient, BatchNorm folded into the convs), images/s;
  - ddn_profile_* per-class device times of one training step (a separate pass, so the per-launch events do not perturb the
    step time);
  - peak device memory of the training step.
Times come from CUDA events around work that ends in a synchronise.  The card's name and power limit are read in the same
process (nvidia-smi query).  Prints one JSON object; needs a GPU.

    python scripts/bench_backbones.py [--steps 20] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import pdc_b200  # noqa: E402
from pdc_b200 import loss_composer, synthetic, _native as N  # noqa: E402

PAIRS, D, H, W = 8, 3, 480, 640


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:          # the measurement still stands; say what is missing
        out = "unavailable (%s)" % e
    return {"gpu": name, "power_limit_and_max_sm_clock": out}


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def measure(cls, d, x16, steps, warmup):
    torch.manual_seed(0)
    fcn = cls(num_classes=D).cuda()
    dcn = pdc_b200.DenseCorrespondenceNetwork(fcn, D, image_width=W, image_height=H)
    pcl = pdc_b200.PixelwiseContrastiveLoss(dcn.image_shape, dict(pdc_b200.DEFAULT_LOSS_CONFIG))
    blind = loss_composer.empty_tensor().cuda()

    def step():
        fcn.zero_grad(set_to_none=True)
        a, b = dcn.forward_pair(d["img_a"], d["img_b"])
        five = loss_composer.get_loss(pcl, torch.tensor([0]), dcn.process_network_output(a, PAIRS), dcn.process_network_output(b, PAIRS),
                                      d["matches_a"], d["matches_b"], d["masked_a"], d["masked_b"], d["background_a"],
                                      d["background_b"], blind, blind)
        five[0].backward()
        return five[0]

    fcn.train()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    ms_step = timed(step, steps, warmup)
    peak = torch.cuda.max_memory_allocated()
    loss = float(step())
    N.lib.ddn_profile_reset(); N.lib.ddn_profile_enable(1)
    for _ in range(steps):
        step()
    torch.cuda.synchronize()
    N.lib.ddn_profile_enable(0)
    prof = {k: {"ms_per_step": v["ms"] / steps, "launches_per_step": v["launches"] // steps} for k, v in N.profile_read().items()}
    fwd = {}
    for mode in ("train", "eval"):
        fcn.train(mode == "train")
        with torch.no_grad():
            ms = timed(lambda: fcn(x16), steps, warmup)
        fwd[mode] = {"ms_per_forward": ms, "imgs_per_s": x16.shape[0] / (ms * 1e-3)}
    out = {"pairs_per_s": PAIRS / (ms_step * 1e-3), "ms_per_step": ms_step, "loss": loss, "finite": bool(torch.isfinite(torch.tensor(loss))),
           "peak_device_memory_GB": peak / 1e9, "forward_batch16": fwd, "profile_ms_per_step": prof}
    del fcn, dcn
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_backbones.py measures on the GPU and has no CPU mode"
    data = synthetic.make_pair_batch(PAIRS, H, W, 1000, 1000, 1000, 0, seed=1)
    d = {k: (v.cuda() if v is not None else None) for k, v in data.items()}
    x16 = torch.cat([d["img_a"], d["img_b"]], 0)
    res = {"workload": "%d pairs of %dx%d, D=%d, bf16x3; forward-only at batch %d" % (PAIRS, W, H, D, x16.shape[0]), "card": card()}
    for cls in (pdc_b200.Resnet34_8s, pdc_b200.Resnet50_8s):
        res[cls.__name__] = measure(cls, d, x16, args.steps, args.warmup)
        print(cls.__name__, json.dumps(res[cls.__name__]), file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
