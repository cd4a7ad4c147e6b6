"""Writes tests/golden/loss_unit_d4.npz and tests/golden/loss_unit_d16.npz: the reference's ``normalize`` option under its
own loss.

Needs a checkout of the reference (PDC_REFERENCE_ROOT=<dir>):   python oracle/make_golden_unit.py

For each case the REAL reference Resnet34_8s (oracle/ref_loader.py, seeded weights) runs on two seeded images, one forward
each (batch 1, as the reference trains).  The map its fc layer writes (the map the upsample blends) is captured with a
forward hook.  The reference's own normalisation lines (dense_correspondence_network.py:256-259, read from the checkout and
executed as they stand) turn each output into unit descriptors, and the executed reference get_loss (oracle/build_ref.py)
scores the pair.  Autograd gives the gradient with respect to the UN-normalised network outputs.

Stored per case: low_a / low_b [1, D, h, w] (the fc outputs), the index lists, the loss config overrides, the five values
get_loss returns, the three hard-negative counts (recounted by loss_oracle.np_within_scene_loss from the same unit
descriptors) and dA / dB
[1, D, H, W], the gradients of the loss with respect to the un-normalised outputs.  tests/test_unit_descriptors_cpu.py
checks oracle.unit_descriptor_oracle against them; tests/test_gpu_unit_descriptors.py checks the fused unit loss.
"""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import build_ref                    # noqa: E402
from oracle import loss_oracle as LO            # noqa: E402
from oracle import ref_loader                   # noqa: E402
from oracle.resnet34_8s_oracle import seeded_oracle, process_network_output  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
NET_PY = "dense_correspondence/network/dense_correspondence_network.py"
NORMALIZE_LINES = (256, 259, "        if self._normalize:")


def reference_normalize():
    """The reference's normalisation (net.py:256-259) as a function of ``res``: the lines are read from the checkout, checked
    against their expected first line, dedented and executed with ``self._normalize = True``."""
    a, b, first = NORMALIZE_LINES
    with open(os.path.join(build_ref.REF_ROOT, NET_PY)) as f:
        lines = f.read().split("\n")[a - 1:b]
    if not lines[0].startswith(first):
        raise RuntimeError("%s:%d expected %r, found %r" % (NET_PY, a, first, lines[0]))
    code = compile("\n".join(ln[8:] for ln in lines), NET_PY, "exec")
    me = types.SimpleNamespace(_normalize=True)

    def normalize(res):
        scope = {"self": me, "res": res, "torch": torch}
        exec(code, scope)
        return scope["res"]
    return normalize


def case(name, D, H, W, Nm, k_masked, k_bg, n_blind, cfg_over, seed):
    cfg = dict(LO.DEFAULT_LOSS_CONFIG); cfg.update(cfg_over)
    ref_net = ref_loader.reference_resnet34_8s(D, seeded_oracle(D=D, seed=0).state_dict())
    ref_net.train()
    lows = []
    hook = ref_net.resnet34_8s.fc.register_forward_hook(lambda m, i, o: lows.append(o.detach().clone()))
    g = torch.Generator().manual_seed(seed)
    P = H * W
    img_a = torch.randn(1, 3, H, W, generator=g); img_b = torch.randn(1, 3, H, W, generator=g)
    A = ref_net(img_a).detach().requires_grad_()
    Bt = ref_net(img_b).detach().requires_grad_()
    hook.remove()
    normalize = reference_normalize()
    ya, yb = normalize(A), normalize(Bt)
    pa = process_network_output(ya, 1, D, H, W); pb = process_network_output(yb, 1, D, H, W)
    ma = torch.randint(0, P, (Nm,), generator=g); mb = torch.randint(0, P, (Nm,), generator=g)
    na_m = ma.repeat_interleave(k_masked); nb_m = torch.randint(0, P, (Nm * k_masked,), generator=g)
    na_b = ma.repeat_interleave(k_bg); nb_b = torch.randint(0, P, (Nm * k_bg,), generator=g)
    if n_blind:
        xa = torch.randint(0, P, (n_blind,), generator=g); xb = torch.randint(0, P, (n_blind,), generator=g)
    else:
        xa = xb = LO.empty_tensor()
    ref = build_ref.load()
    mt = torch.tensor([ref.dataset.SpartanDatasetDataType.SINGLE_OBJECT_WITHIN_SCENE])
    five = ref.composer.get_loss(ref.pcl.PixelwiseContrastiveLoss([H, W], dict(cfg)), mt, pa, pb, ma, mb, na_m, nb_m, na_b, nb_b,
                                 xa, xb)
    five[0].reshape(()).backward()
    idx = dict(matches_a=ma.numpy(), matches_b=mb.numpy(), masked_a=na_m.numpy(), masked_b=nb_m.numpy(),
               background_a=na_b.numpy(), background_b=nb_b.numpy(), blind_a=xa.numpy(), blind_b=xb.numpy())
    An = pa.detach().numpy()[0]; Bn = pb.detach().numpy()[0]
    _, counts = LO.np_within_scene_loss(An, Bn, idx, cfg, W)
    assert min(counts[:2]) > 0, (name, counts)          # both hinge branches fire
    out = dict(idx)
    out.update(low_a=lows[0].numpy(), low_b=lows[1].numpy(), H=np.int64(H), W=np.int64(W),
               five=np.array([float(t) for t in five]), counts=np.array(counts), dA=A.grad.numpy(), dB=Bt.grad.numpy(),
               cfg_keys=np.array(sorted(cfg_over.keys())), cfg_vals=np.array([float(cfg_over[k]) for k in sorted(cfg_over)]))
    np.savez_compressed(os.path.join(GOLD, name + ".npz"), **out)
    print("wrote", name, "five", out["five"], "counts", counts, "bytes", os.path.getsize(os.path.join(GOLD, name + ".npz")))


if __name__ == "__main__":
    assert ref_loader.reference_available() and build_ref.reference_available(), "set PDC_REFERENCE_ROOT to a checkout of the reference"
    build_ref.build()
    torch.set_num_threads(os.cpu_count())
    os.makedirs(GOLD, exist_ok=True)
    # D = 4: the setting of the reference's normalize_descriptors experiment; margins wide enough for unit descriptors
    case("loss_unit_d4", 4, 48, 64, 50, 3, 2, 20, {"M_masked": 1.5, "M_background": 1.2}, 41)
    case("loss_unit_d16", 16, 32, 48, 40, 4, 4, 16,
         {"use_l2_pixel_loss_on_masked_non_matches": True, "use_l2_pixel_loss_on_background_non_matches": True,
          "M_pixel": 25, "M_masked": 1.6, "M_background": 1.3, "non_match_loss_weight": 2.0}, 42)
