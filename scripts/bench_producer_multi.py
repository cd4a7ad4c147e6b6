"""Across-scene (DIFFERENT_OBJECT / SINGLE_OBJECT_ACROSS_SCENE) and synthetic multi-object batch producers: B = 8 pairs at
640x480, the reference's default training config (training.yaml: cross_scene_num_samples 10000, domain_randomize on,
10000 matching attempts, 75 + 75 non-matches per match).  Synthetic rows carry the prefix ``synthetic_``.

    python scripts/bench_producer_multi.py                   # device rows (needs a GPU)
    python scripts/bench_producer_multi.py --reference-cpu   # the reference's CPU producer (host only, needs oracle/_ref)

Device rows (one JSON object on stdout):
  producer_ms          draw_across_scene_rand + across_scene_batch per batch (CUDA events, warm-up, >= 20 iterations)
  producer_call_ms     across_scene_batch alone, random numbers drawn beforehand
  launches_per_call    library kernel launches of one across_scene_batch call
  step_ms / step_with_producer_ms
                       forward_pair + get_loss(DIFFERENT_OBJECT) + backward (Resnet34_8s, D = 3) on a batch produced
                       beforehand, and the same step preceded by the producer
GPU name, SM clock and power limit (nvidia-smi, query only) are printed with the numbers.
--reference-cpu: the reference's own functions (oracle/_ref, built by oracle/build_ref_augment.py) through
oracle/across_scene_oracle.py and oracle/synthetic_multi_object_oracle.py for one pair on one host thread with the same
random numbers, median of 5; PNG decoding is not included on either side."""
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import pdc_b200  # noqa: E402
from pdc_b200 import _native as N  # noqa: E402
from pdc_b200 import loss_composer  # noqa: E402
from pdc_b200 import sampling as S  # noqa: E402
from bench_producer import gpu_info, timed  # noqa: E402

B, H, W, D = 8, 480, 640, 3
TC = {"training": dict(cross_scene_num_samples=10000, domain_randomize=True, num_matching_attempts=10000,
                       num_non_matches_per_match=150, fraction_masked_non_matches=0.5, fraction_background_non_matches=0.5,
                       sample_matches_only_off_mask=True, use_image_b_mask_inv=True)}


def synthetic_inputs():
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_gpu_synthetic_multi_object import scene
    return scene(B, H, W, 1)


def inputs():
    g = np.random.RandomState(1)
    xs = []
    for _ in range(B):
        mask_a = (g.rand(H, W) > 0.3).astype(np.uint8); mask_a[: H // 4] = 0
        mask_b = (g.rand(H, W) > 0.6).astype(np.uint8); mask_b[:, : W // 3] = 0
        xs.append(dict(rgb_a=g.randint(0, 256, (H, W, 3)).astype(np.uint8), rgb_b=g.randint(0, 256, (H, W, 3)).astype(np.uint8),
                       mask_a=mask_a, mask_b=mask_b))
    return xs


def reference_cpu():
    from oracle import across_scene_oracle as AO
    from oracle import build_ref_augment
    if not build_ref_augment.built():
        return {"reference_cpu_ms_per_pair": "not available (oracle/_ref missing)"}
    fns = AO.executed_reference(build_ref_augment.load())
    torch.set_num_threads(1)
    x = inputs()[0]
    g = np.random.RandomState(2)
    n = S.across_scene_cfg(TC)["num_samples"]
    times = []
    for flip in (0, 1, 0, 1, 1):
        params = np.zeros((2, 16), np.uint8)
        params[:, :5] = (1, 1, 0, 1, flip); params[:, 5:11] = g.randint(0, 255, (2, 6))
        r = dict(params=params, noise=g.randint(0, 50, (2, 2, H, W, 3)).astype(np.uint8),
                 blind_a=g.random_sample(n).astype(np.float32), blind_b=g.random_sample(n).astype(np.float32))
        t0 = time.perf_counter()
        AO.get_across_scene_data(fns, x["rgb_a"], x["rgb_b"], x["mask_a"], x["mask_b"], S.across_scene_cfg(TC), r)
        times.append(1e3 * (time.perf_counter() - t0))
    rows = {"reference_cpu_ms_per_pair": statistics.median(times), "reference_cpu_ms_all": times,
            "cpu_count": os.cpu_count(), "randomise": "gradient + noise on both images"}
    from oracle import synthetic_multi_object_oracle as SO
    fns = SO.executed_reference(build_ref_augment.load())
    As, Bs, K = synthetic_inputs()
    c = S.within_scene_cfg(TC)
    times, rets = [], []
    for i, merge in enumerate(((1, 1), (0, 1), (1, 0), (0, 0), (1, 1))):
        u = lambda *shape: g.random_sample(shape).astype(np.float32)
        n = c["n_attempts"]
        r = dict(merge=np.asarray(merge, np.uint8), cand_u=u(2, n), cand_v=u(2, n), masked_u=u(2 * n * c["k_masked"]),
                 masked_v=u(2 * n * c["k_masked"]), background_u=u(2 * n * c["k_background"]),
                 background_v=u(2 * n * c["k_background"]))
        t0 = time.perf_counter()
        o = SO.get_synthetic_data(fns, As[i], Bs[i], K, c, r)
        times.append(1e3 * (time.perf_counter() - t0)); rets.append((o["ret"], len(o["matches_a"])))
    rows.update(synthetic_reference_cpu_ms_per_pair=statistics.median(times), synthetic_reference_cpu_ms_all=times,
                synthetic_returns=rets)
    return rows


def main():
    if "--reference-cpu" in sys.argv:
        print(json.dumps(reference_cpu()))
        return
    dev = torch.device("cuda", 0)
    xs = inputs()
    t = lambda k: torch.from_numpy(np.stack([x[k] for x in xs])).to(dev)
    args = (t("rgb_a"), t("rgb_b"), t("mask_a"), t("mask_b"))
    gen = torch.Generator(device=dev).manual_seed(0)
    rand = S.draw_across_scene_rand(B, H, W, TC, generator=gen)
    rows = {"gpu": gpu_info(), "B": B, "H": H, "W": W, "cross_scene_num_samples": 10000}
    rows["producer_ms"] = timed(lambda: S.across_scene_batch(*args, TC, generator=gen))
    rows["producer_call_ms"] = timed(lambda: S.across_scene_batch(*args, TC, rand=rand))
    n0 = N.launch_count()
    out = S.across_scene_batch(*args, TC, rand=rand)
    rows["launches_per_call"] = N.launch_count() - n0

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
    rows["step_with_producer_ms"] = timed(lambda: step(S.across_scene_batch(*args, TC, generator=gen)))
    As, Bs, K = synthetic_inputs()
    st = lambda scenes: tuple(np.stack([x[k] for x in scenes]) if k.startswith("pose") else
                              torch.from_numpy(np.stack([x[k] for x in scenes])).to(dev)
                              for k in ("rgb_1", "rgb_2", "depth_1", "depth_2", "mask_1", "mask_2", "pose_1", "pose_2"))
    sa, sb = st(As), st(Bs)
    srand = S.draw_synthetic_multi_object_rand(B, H, W, TC, generator=gen)
    rows["synthetic_producer_ms"] = timed(lambda: S.synthetic_multi_object_batch(sa, sb, K, TC, generator=gen))
    rows["synthetic_producer_call_ms"] = timed(lambda: S.synthetic_multi_object_batch(sa, sb, K, TC, rand=srand))
    n0 = N.launch_count()
    sout = S.synthetic_multi_object_batch(sa, sb, K, TC, rand=srand)
    rows["synthetic_launches_per_call"] = N.launch_count() - n0
    rows["synthetic_mean_counts"] = [float(c) for c in sout["counts"].double().mean(0).cpu()]
    rows["synthetic_step_ms"] = timed(lambda: step(sout))
    rows["synthetic_step_with_producer_ms"] = timed(lambda: step(S.synthetic_multi_object_batch(sa, sb, K, TC, generator=gen)))
    rows["gpu_after"] = gpu_info()
    print(json.dumps(rows))


if __name__ == "__main__":
    main()
