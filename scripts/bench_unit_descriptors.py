"""Training steps with unit-length descriptors (the reference's ``normalize: True``): 640x480, Resnet34_8s, the reference's
default loss config, D = 3 and D = 4 (the normalize_descriptors experiment's setting).

Arms, each timed as forward_pair + get_loss + backward on a fixed synthetic batch (synthetic.make_pair_batch: 1000 matches,
75000 masked and 75000 background non-matches per pair, as training.yaml samples them):
  unit      8 pairs, forward_pair(..., per_pixel_normalize=True): the upsample writes unit descriptors and the loss fused
            with the upsample normalises every sampled descriptor (DDN_NET_UNIT_DESCRIPTORS, DDN_LOWRES_UNIT)
  plain     the same 8 pairs on a network without normalize: the unnormalised step
  batch1    what a normalize network could train before: one pair per step, forward + forward + the reference's
            normalisation expression in torch and the generic full-resolution loss (reported per pair)

    python scripts/bench_unit_descriptors.py [--reps 5] [--iters 10]

Every arm is warmed up, then the arms alternate in one process, `--reps` rounds of `--iters` steps each timed with CUDA
events; the JSON line gives each arm's per-round ms per step (median, min, max) and its library launches per step.  GPU
name, SM clock, max SM clock and power limit (nvidia-smi, query only) are printed with the numbers, before and after."""
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
from pdc_b200 import loss_composer, synthetic  # noqa: E402
from bench_producer import gpu_info  # noqa: E402

H, W, B = 480, 640, 8
IDX = ("matches_a", "matches_b", "masked_a", "masked_b", "background_a", "background_b")


def network(D, normalize):
    return pdc_b200.DenseCorrespondenceNetwork.from_config(
        {"descriptor_dimension": D, "image_width": W, "image_height": H, "normalize": normalize}, load_stored_params=False)


def arms_for(D, dev):
    data = synthetic.make_pair_batch(B, H, W, 1000, 75000, 75000, 0, seed=1)
    d = {k: (v.to(dev) if v is not None else None) for k, v in data.items()}
    blind = loss_composer.empty_tensor().to(dev)
    unit_net, plain_net = network(D, True), network(D, False)
    plain_net.fcn.load_state_dict(unit_net.fcn.state_dict())
    pcl = pdc_b200.PixelwiseContrastiveLoss(unit_net.image_shape, dict(pdc_b200.DEFAULT_LOSS_CONFIG))

    def step(net, **kw):
        a, b = net.forward_pair(d["img_a"], d["img_b"], **kw)
        pa, pb = net.process_network_output(a, B), net.process_network_output(b, B)
        five = loss_composer.get_loss(pcl, torch.zeros(B, dtype=torch.int64), pa, pb, *[d[k] for k in IDX], blind, blind)
        five[0].backward()

    def batch1():
        # the reference's own route at N == 1: two forward calls, res / norm in torch, the full-resolution loss
        ya = unit_net.fcn(d["img_a"][:1]); yb = unit_net.fcn(d["img_b"][:1])
        ya = ya / torch.norm(ya, 2, 1); yb = yb / torch.norm(yb, 2, 1)
        pa, pb = unit_net.process_network_output(ya, 1), unit_net.process_network_output(yb, 1)
        five = loss_composer.get_loss(pcl, torch.zeros(1, dtype=torch.int64), pa, pb, *[d[k][:1] for k in IDX], blind, blind)
        five[0].backward()

    return {"unit": lambda: step(unit_net, per_pixel_normalize=True), "plain": lambda: step(plain_net), "batch1": batch1}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    rows = {"gpu": gpu_info(), "B": B, "H": H, "W": W}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for D in (3, 4):
        arms = arms_for(D, dev)
        for fn in arms.values():                                 # warm-up: every shape the timed rounds use
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        for name, fn in arms.items():
            n0 = N.launch_count()
            fn()
            rows["D%d_%s_launches_per_step" % (D, name)] = N.launch_count() - n0
        times = {name: [] for name in arms}
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
            rows["D%d_%s_ms" % (D, name)] = {"median": statistics.median(t), "min": min(t), "max": max(t), "rounds": t}
        u, p, one = (statistics.median(times[k]) for k in ("unit", "plain", "batch1"))
        rows["D%d_unit_over_plain" % D] = u / p
        rows["D%d_ms_per_pair" % D] = {"unit": u / B, "plain": p / B, "batch1": one}
        del arms
        torch.cuda.empty_cache()
    rows["gpu_after_timing"] = gpu_info()
    print(json.dumps(rows))


if __name__ == "__main__":
    main()
