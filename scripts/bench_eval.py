"""Per-match evaluation statistics: 100 image pairs x 100 matches at 640x480, D = 3 and 16.

Rows (one JSON object on stdout; needs a GPU):
  device_one_launch   pdc_b200.match_statistics over all pairs in one call (CUDA events, ms per call)
  device_per_pair     the same, one call per pair
  unfused             find_best_matches_cuda(return_norm_diffs=True, mask_b) per pair + the remaining statistics in torch
  reference_numpy     the reference's per-match numpy (oracle/match_stats_oracle.one_match, the same numpy statements),
                      timed on a few matches on the host and scaled to 100 x 100; the host core count is printed
GPU name, SM clock and power limit are read from nvidia-smi (query only) and printed beside the numbers."""
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
from pdc_b200 import evaluation as E  # noqa: E402
from oracle import match_stats_oracle as MO  # noqa: E402

NP, NQ, H, W = int(os.environ.get("EVAL_PAIRS", "100")), int(os.environ.get("EVAL_MATCHES", "100")), 480, 640
REPS, WARM = int(os.environ.get("EVAL_REPS", "5")), 2
DEV = torch.device("cuda", 0)


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
    for _ in range(REPS):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / REPS


def unfused(res_a, res_b, uv_a, uv_b, mask, n):
    """find_best_matches_cuda with the distance maps, then the counts / sums / fractions in torch (no 3-D columns)."""
    DCN = pdc_b200.DenseCorrespondenceNetwork
    uv, diff, nd, uvm, diffm = DCN.find_best_matches_cuda(uv_a, res_a, res_b, return_norm_diffs=True, mask_b=mask)
    t = nd[torch.arange(nd.shape[0], device=DEV), uv_b[:, 1], uv_b[:, 0]]
    closer = nd < t[:, None, None]
    mnd = nd.double() + (1 - mask.double()) * 1e6
    closer_m = mnd < t.double()[:, None, None]
    vv, uu = torch.meshgrid(torch.arange(H, device=DEV), torch.arange(W, device=DEV), indexing="ij")
    dist = torch.sqrt(((uu[None] - uv_b[:, 0, None, None]) ** 2 + (vv[None] - uv_b[:, 1, None, None]) ** 2).double())
    return (closer.sum((1, 2)), (dist * closer).sum((1, 2)), closer_m.sum((1, 2)), (dist * closer_m).sum((1, 2)), uv, uvm)


def main():
    rng = np.random.default_rng(0)
    rows = {"gpu": gpu_info(), "pairs": NP, "matches_per_pair": NQ, "image": [H, W], "host_cores": os.cpu_count()}
    K = np.array([[533.6, 0, 319.4], [0, 534.8, 236.4], [0, 0, 1.0]])
    poses = np.repeat(np.eye(4)[None], NP, 0)
    mask = torch.from_numpy((rng.random((NP, H, W)) < 0.5).astype(np.float32)).to(DEV)
    depth = torch.from_numpy(rng.integers(0, 3000, (NP, H, W)).astype(np.float32)).to(DEV)
    pair = torch.arange(NP, device=DEV).repeat_interleave(NQ)
    uv_a = torch.stack([torch.randint(0, W, (NP * NQ,)), torch.randint(0, H, (NP * NQ,))], 1).to(DEV)
    uv_b = torch.stack([torch.randint(0, W, (NP * NQ,)), torch.randint(0, H, (NP * NQ,))], 1).to(DEV)
    for D in (3, 16):
        a = torch.randn(NP, D, H, W, device=DEV); b = torch.randn(NP, D, H, W, device=DEV)
        res_a, res_b = a.permute(0, 2, 3, 1), b.permute(0, 2, 3, 1)      # forward_single_image_tensor's layout
        one = timed(lambda: E.match_statistics(res_a, res_b, uv_a, uv_b, pair, mask, depth, depth, poses, poses, K))
        sl = lambda n: slice(n * NQ, (n + 1) * NQ)
        z = torch.zeros(NQ, dtype=torch.int64, device=DEV)
        per = timed(lambda: [E.match_statistics(res_a[n], res_b[n], uv_a[sl(n)], uv_b[sl(n)], z, mask[n], depth[n], depth[n],
                                                poses[n:n + 1], poses[n:n + 1], K) for n in range(NP)])
        unf = timed(lambda: [unfused(res_a[n], res_b[n], uv_a[sl(n)], uv_b[sl(n)], mask[n], n) for n in range(NP)])
        # the reference's numpy on the host: a few matches, scaled to NP x NQ
        ra, rb = res_a[0].cpu().numpy(), res_b[0].cpu().numpy()
        mk, dp = mask[0].cpu().numpy(), depth[0].cpu().numpy()
        ua, ub = uv_a[:NQ].cpu().numpy(), uv_b[:NQ].cpu().numpy()
        nh = 5
        t0 = time.perf_counter()
        for i in range(nh):
            MO.one_match(dp, dp, mk, tuple(ua[i]), tuple(ub[i]), poses[0], poses[0], ra, rb, K, threshold="reference")
        host = (time.perf_counter() - t0) / nh
        rows["D%d" % D] = {"device_one_launch_ms": round(one, 3), "device_per_pair_ms": round(per, 3), "unfused_ms": round(unf, 3),
                           "reference_numpy_ms_per_match": round(host * 1e3, 3),
                           "reference_numpy_s_for_all": round(host * NP * NQ, 1)}
    print(json.dumps(rows))


if __name__ == "__main__":
    main()
