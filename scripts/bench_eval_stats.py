"""Descriptor statistics and the across-object best match at 640x480.

Rows (one JSON object on stdout; needs a GPU):
  stats_D{3,16}   100 images, one pdc_b200.descriptor_statistics launch over all of them, against the reference's
                  per-image torch loop (compute_descriptor_statistics, evaluation.py:2177-2219) on the same GPU.  The
                  achieved bandwidth counts the bytes the algorithm must read (descriptors once, the float32 mask once)
                  over the device time of the call, against the H100 SXM data-sheet 3.35 TB/s.
  across_D{3,16}  25 pairs x 100 sampled pixels: one pdc_b200.evaluation.best_match_batch launch, against one
                  find_best_matches_cuda call per pair.
Times are CUDA-event means over STATS_REPS calls after warm-up.  GPU name, SM clock and power limit are read from
nvidia-smi (query only) in the same run and printed beside the numbers."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import pdc_b200  # noqa: E402
from pdc_b200 import evaluation as E  # noqa: E402

NI, H, W = 100, 480, 640
PAIRS, SAMPLES = 25, 100
REPS, WARM = int(os.environ.get("STATS_REPS", "20")), 3
HBM_BYTES_PER_S = 3.35e12
DEV = torch.device("cuda", 0)


def gpu_info():
    try:
        q = "name,clocks.sm,clocks.max.sm,power.limit"
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as e:             # the numbers are still device-timed; only the label is missing
        return "nvidia-smi unavailable (%s); %s" % (e, torch.cuda.get_device_name(0))


def timed(fn, reps=REPS):
    for _ in range(WARM):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def reference_loop(res, mask):
    """compute_descriptor_statistics per image, as the reference runs it (its empty-mask test reads back a length)."""
    out = []
    for i in range(res.shape[0]):
        r = res[i]
        D = r.shape[2]
        flat = r.contiguous().view(-1, D)
        whole = (flat.min(0)[0], flat.max(0)[0], flat.mean(0))
        idx = torch.nonzero(mask[i].view(-1, 1).squeeze(1))
        if len(idx) == 0:
            out.append((whole, None))
            continue
        m = flat.index_select(0, idx.squeeze(1))
        out.append((whole, (m.min(0)[0], m.max(0)[0], m.mean(0))))
    return out


def main():
    rows = {"gpu": gpu_info(), "images": NI, "image": [H, W], "pairs": PAIRS, "samples_per_pair": SAMPLES}
    g = torch.Generator(device=DEV).manual_seed(0)
    mask = (torch.rand(NI, H, W, device=DEV, generator=g) < 0.3).to(torch.float32)
    for D in (3, 16):
        res = torch.randn(NI, D, H, W, device=DEV, generator=g).permute(0, 2, 3, 1)      # the network's NCHW output
        one = timed(lambda: E.descriptor_statistics(res, mask))
        loop = timed(lambda: reference_loop(res, mask), reps=max(1, REPS // 4))
        got = E.descriptor_statistics(res, mask)
        ref = reference_loop(res, mask)
        exact = all(torch.equal(got["min"][i], w[0]) and torch.equal(got["max"][i], w[1]) and
                    torch.equal(got["mask_min"][i], m[0]) and torch.equal(got["mask_max"][i], m[1]) for i, (w, m) in enumerate(ref))
        mean_err = max(float(((got["mean"][i] - w[2]).abs() / w[2].abs()).max()) for i, (w, _) in enumerate(ref))
        nbytes = NI * H * W * (D + 1) * 4
        rows["stats_D%d" % D] = {"one_launch_ms": round(one, 3), "reference_loop_ms": round(loop, 3),
                                 "speedup": round(loop / one, 1), "bytes_read": nbytes,
                                 "achieved_TB_per_s": round(nbytes / (one * 1e-3) / 1e12, 3),
                                 "share_of_3_35_TB_per_s": round(nbytes / (one * 1e-3) / HBM_BYTES_PER_S, 3),
                                 "min_max_equal_to_loop": exact, "max_rel_mean_diff_vs_loop": mean_err}
        del res

        ra = torch.randn(PAIRS, D, H, W, device=DEV, generator=g).permute(0, 2, 3, 1)
        rb = torch.randn(PAIRS, D, H, W, device=DEV, generator=g).permute(0, 2, 3, 1)
        flat = torch.randint(0, H * W, (PAIRS * SAMPLES,), device=DEV, generator=g)
        uv_a = torch.stack([flat % W, flat // W], 1)
        pair = torch.arange(PAIRS, device=DEV).repeat_interleave(SAMPLES)
        DCN = pdc_b200.DenseCorrespondenceNetwork
        sl = lambda p: slice(p * SAMPLES, (p + 1) * SAMPLES)
        batch = timed(lambda: E.best_match_batch(ra, rb, uv_a, pair))
        per_pair = timed(lambda: [DCN.find_best_matches_cuda(uv_a[sl(p)], ra[p], rb[p]) for p in range(PAIRS)])
        uv, _, _ = E.best_match_batch(ra, rb, uv_a, pair)
        agree = sum(int((uv[sl(p)] == DCN.find_best_matches_cuda(uv_a[sl(p)], ra[p], rb[p])[0]).all(1).sum()) for p in range(PAIRS))
        rows["across_D%d" % D] = {"one_launch_ms": round(batch, 3), "per_pair_find_best_matches_cuda_ms": round(per_pair, 3),
                                  "speedup": round(per_pair / batch, 2), "same_pixel_as_per_pair": "%d/%d" % (agree, PAIRS * SAMPLES)}
        del ra, rb
    print(json.dumps(rows))


if __name__ == "__main__":
    main()
