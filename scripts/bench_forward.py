"""Forward-only throughput of Resnet34_8s at the north_star's forward target: D=3, 640x480, batch 16 (BASELINE.json north_star,
SURVEY.md 8d "forward-only target": imgs/s x 211.909 GFLOP / peak).

Rows: train-mode BN (batch statistics from the conv epilogue + one BN-apply pass per conv) and eval-mode BN (inference:
BN + residual + ReLU folded into the conv epilogue, dense_correspondence_network.py:265-299 forward_single_image_tensor /
evaluation).  Images are resident in HBM; whole forward timed with CUDA events on the current stream, the tensor-core conv
launches additionally timed one by one through ddn_profile_* (a separate pass, so the per-launch events do not perturb
the headline).  Prints one JSON object; needs a GPU."""
import json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import pdc_b200
from pdc_b200 import _native as N

pk = os.path.join(ROOT, "MEASURED_PEAKS.json")
peaks = json.load(open(pk)) if os.path.exists(pk) else {}
peak_tf = float(peaks.get("bf16_tflops_sustained", 989.0))      # else the H100 SXM data sheet, dense bf16
B, D, H, W = int(os.environ.get("FWD_BATCH", "16")), 3, 480, 640
GF_IMG = 211.909
steps, warmup = int(os.environ.get("FWD_STEPS", "20")), int(os.environ.get("FWD_WARMUP", "5"))

torch.manual_seed(0)
net = pdc_b200.Resnet34_8s(num_classes=D).cuda()
x = torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(1)).cuda()
rows = []
for mode in ("train", "eval"):
    net.train(mode == "train")
    with torch.no_grad():
        for _ in range(warmup):
            net(x)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        l0 = N.launch_count()
        e0.record()
        for _ in range(steps):
            y = net(x)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / steps
        launches = (N.launch_count() - l0) // steps
        N.lib.ddn_profile_reset(); N.lib.ddn_profile_enable(1)
        for _ in range(steps):
            net(x)
        torch.cuda.synchronize()
        N.lib.ddn_profile_enable(0)
    conv = N.profile_read()["conv_fwd_tc"]
    conv_ms = conv["ms"] / steps
    useful = conv["flops"] / (conv["ms"] * 1e-3) / 1e12
    rows.append({"bn_mode": mode, "batch": B, "ms_per_forward": ms, "imgs_per_s": B / (ms * 1e-3), "launches_per_forward": launches,
                 "whole_forward_useful_TFLOPs": B * GF_IMG / ms, "whole_forward_issued_frac_of_peak": 3 * B * GF_IMG / ms / peak_tf,
                 "conv_kernels_ms": conv_ms, "conv_share_of_forward": conv_ms / ms, "conv_useful_TFLOPs": useful,
                 "conv_issued_frac_of_peak": 3 * useful / peak_tf, "finite": bool(torch.isfinite(y).all())})
    print(rows[-1], file=sys.stderr, flush=True)
print(json.dumps({"workload": "Resnet34_8s forward only, D=3, 640x480, batch %d, bf16x3 (3 MMAs per useful MAC)" % B,
                  "peak_bf16_TFLOPs_sustained": peak_tf, "rows": rows}))
