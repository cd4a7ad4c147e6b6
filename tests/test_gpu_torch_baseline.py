"""BASELINE.json configs[1] asks for the fused step "vs reference GPU PyTorch": this times the ORACLE port (the reference's
modules restated in plain PyTorch: cuDNN convolutions, torch BatchNorm, index_select / norm / clamp loss with its host
syncs) on the same GPU, same workload as bench.py (8 pairs, 640x480, D=3, 1000 matches + 1000 masked + 1000 background
non-matches per pair, fwd A + fwd B + loss + backward), next to this library's step, and prints both as one JSON line.
It is a measurement, not a gate, so it only runs when DDN_TORCH_GPU_BASELINE=1
(`DDN_TORCH_GPU_BASELINE=1 python -m pytest tests/test_gpu_torch_baseline.py -m gpu -s`)."""
import json
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


def _time_steps(step, warmup, steps):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


@pytest.mark.skipif(os.environ.get("DDN_TORCH_GPU_BASELINE") != "1", reason="measurement run; set DDN_TORCH_GPU_BASELINE=1")
def test_torch_gpu_baseline_report():
    import pdc_b200
    from pdc_b200 import loss_composer, synthetic
    from oracle import loss_oracle as LO
    from oracle.resnet34_8s_oracle import seeded_oracle, process_network_output

    B, D, H, W = 8, 3, 480, 640
    dev = torch.device("cuda:0")
    host = synthetic.make_pair_batch(B, H, W, 1000, 1000, 1000, 0, seed=1)
    data = {k: v.to(dev) for k, v in host.items() if v is not None}
    rows = []

    # ---- the oracle port on cuDNN
    oracle = seeded_oracle(D=D, seed=0).to(dev).train()
    pcl_o = LO.TorchPixelwiseContrastiveLoss([H, W], dict(LO.DEFAULT_LOSS_CONFIG))

    def oracle_step():
        oracle.zero_grad(set_to_none=True)
        ya, yb = oracle(data["img_a"]), oracle(data["img_b"])
        five = LO.batched_within_scene_loss(pcl_o, process_network_output(ya, B, D, H, W), process_network_output(yb, B, D, H, W), data)
        five[0].backward()
        return five[0]

    torch.backends.cudnn.benchmark = True
    for tf32 in (False, True):
        torch.backends.cudnn.allow_tf32 = tf32
        torch.backends.cuda.matmul.allow_tf32 = tf32
        ms = _time_steps(oracle_step, 3, 10)
        rows.append({"impl": "oracle port on PyTorch/cuDNN, fp32%s" % (" with TF32 convolutions" if tf32 else " (TF32 off)"),
                     "ms_per_step": ms, "pairs_per_s": B / (ms * 1e-3)})
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    loss_ref = float(oracle_step())
    del oracle
    torch.cuda.empty_cache()

    # ---- this library, same weights, same batch
    dcn = pdc_b200.DenseCorrespondenceNetwork(pdc_b200.Resnet34_8s(num_classes=D), D, image_width=W, image_height=H).to(dev).train()
    dcn.fcn.load_state_dict(seeded_oracle(D=D, seed=0).state_dict())
    pcl = pdc_b200.PixelwiseContrastiveLoss([H, W], dict(LO.DEFAULT_LOSS_CONFIG))
    match_type = torch.zeros(B, dtype=torch.int64)
    blind = loss_composer.empty_tensor().to(dev)

    def our_step():
        dcn.zero_grad(set_to_none=True)
        pa = dcn.process_network_output(dcn.forward(data["img_a"]), B)
        pb = dcn.process_network_output(dcn.forward(data["img_b"]), B)
        five = loss_composer.get_loss(pcl, match_type, pa, pb, data["matches_a"], data["matches_b"], data["masked_a"], data["masked_b"],
                                      data["background_a"], data["background_b"], blind, blind)
        five[0].backward()
        return five[0]

    ms = _time_steps(our_step, 3, 10)
    rows.append({"impl": "libddn_b200 (bf16x3 on the wgmma tensor cores, fp32-equivalent)", "ms_per_step": ms, "pairs_per_s": B / (ms * 1e-3)})
    loss_ours = float(our_step())
    assert abs(loss_ours - loss_ref) <= 1e-3 * abs(loss_ref)       # two train-mode steps in: still the same computation

    out = {"workload": "configs[1]: 8 pairs, Resnet34_8s D=3, 640x480, fwd A + fwd B + loss + backward, inputs resident",
           "torch": torch.__version__, "cudnn": torch.backends.cudnn.version(), "rows": rows,
           "gpu": torch.cuda.get_device_name(dev), "loss_oracle_cudnn": loss_ref, "loss_libddn": loss_ours}
    print(json.dumps(out))
