"""CPU/float64 oracle for the Resnet50_8s backbone -- TEST INFRASTRUCTURE, NOT THE PRODUCT.

A plain PyTorch restatement of the reference's Bottleneck backbone (only ``tests/`` and oracle/make_golden_resnet50.py import it;
the latter pins it bit for bit against the executed reference):

  external/pytorch-segmentation-detection/vision/torchvision/models/resnet.py
      Bottleneck           :72-109   (conv1 1x1, conv2 3x3 carrying stride and dilation, conv3 1x1 -> 4 x planes)
      ResNet._make_layer   :183-229  (downsample whenever stride != 1 or inplanes != 4 x planes -- layer1 included;
                                      stride -> dilation once output_stride is hit, block 0 dilated too)
      resnet50             :317-335
  external/pytorch-segmentation-detection/pytorch_segmentation_detection/models/resnet_dilated.py
      Resnet50_8s          :399-435  (fc = Conv2d(2048, D, 1), N(0, 0.01) / 0 init, upsample_bilinear)
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle.resnet34_8s_oracle import conv3x3, perturbed_relus, process_network_output, rel  # noqa: F401


class Bottleneck(nn.Module):
    # resnet.py:72-109
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, downsample=None, dilation=1):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, kernel_size=1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = conv3x3(planes, planes, stride=stride, dilation=dilation)
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv3 = nn.Conv2d(planes, planes * 4, kernel_size=1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = downsample
        self.stride = stride

    def forward(self, x):
        residual = x
        out = self.relu(self.bn1(self.conv1(x)))
        out = self.relu(self.bn2(self.conv2(out)))
        out = self.bn3(self.conv3(out))
        if self.downsample is not None:
            residual = self.downsample(x)
        return self.relu(out + residual)


class ResNetFullyConv(nn.Module):
    """resnet.py:112-265 configured as resnet50(fully_conv=True, output_stride=8, remove_avg_pool_layer=True) with the fc
    already replaced by the 1x1 scoring conv (resnet_dilated.py:414)."""

    def __init__(self, layers=(3, 4, 6, 3), num_classes=3, output_stride=8):
        super().__init__()
        self.output_stride = output_stride
        self.current_stride = 4
        self.current_dilation = 1
        self.inplanes = 64
        self.conv1 = nn.Conv2d(3, 64, kernel_size=7, stride=2, padding=3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.relu = nn.ReLU(inplace=True)
        self.maxpool = nn.MaxPool2d(kernel_size=3, stride=2, padding=1)
        self.layer1 = self._make_layer(64, layers[0])
        self.layer2 = self._make_layer(128, layers[1], stride=2)
        self.layer3 = self._make_layer(256, layers[2], stride=2)
        self.layer4 = self._make_layer(512, layers[3], stride=2)
        self.fc = nn.Conv2d(2048, num_classes, 1)
        for m in self.modules():        # resnet.py:174-180
            if isinstance(m, nn.Conv2d):
                n = m.kernel_size[0] * m.kernel_size[1] * m.out_channels
                m.weight.data.normal_(0, math.sqrt(2. / n))
            elif isinstance(m, nn.BatchNorm2d):
                m.weight.data.fill_(1)
                m.bias.data.zero_()
        self.fc.weight.data.normal_(0, 0.01)      # resnet_dilated.py:420-423
        self.fc.bias.data.zero_()

    def _make_layer(self, planes, blocks, stride=1):
        # resnet.py:183-229
        downsample = None
        if stride != 1 or self.inplanes != planes * 4:
            if self.current_stride == self.output_stride:
                self.current_dilation = self.current_dilation * stride
                stride = 1
            else:
                self.current_stride = self.current_stride * stride
            downsample = nn.Sequential(
                nn.Conv2d(self.inplanes, planes * 4, kernel_size=1, stride=stride, bias=False),
                nn.BatchNorm2d(planes * 4))
        layers = [Bottleneck(self.inplanes, planes, stride, downsample, dilation=self.current_dilation)]
        self.inplanes = planes * 4
        for _ in range(1, blocks):
            layers.append(Bottleneck(self.inplanes, planes, dilation=self.current_dilation))
        return nn.Sequential(*layers)

    def forward(self, x):
        x = self.maxpool(self.relu(self.bn1(self.conv1(x))))
        x = self.layer4(self.layer3(self.layer2(self.layer1(x))))
        return self.fc(x)


class Resnet50_8s(nn.Module):
    """resnet_dilated.py:399-435.  State-dict keys are ``resnet50_8s.*`` (320 entries at any D)."""

    def __init__(self, num_classes=1000):
        super().__init__()
        self.resnet50_8s = ResNetFullyConv((3, 4, 6, 3), num_classes=num_classes)

    def forward(self, x):
        size = x.shape[2:]
        x = self.resnet50_8s(x)
        return F.interpolate(x, size=tuple(size), mode="bilinear", align_corners=True)


def seeded_oracle(D=3, seed=0):
    """The weights the Resnet50_8s parity tests use: the oracle's own init under a fixed CPU seed."""
    g = torch.random.get_rng_state()
    torch.manual_seed(seed)
    net = Resnet50_8s(num_classes=D)
    torch.random.set_rng_state(g)
    return net


STEM_PARAMS = ("resnet50_8s.conv1.weight", "resnet50_8s.bn1.weight", "resnet50_8s.bn1.bias")


def decisive_biases(net, amp=6.0, on_fraction=0.7, seed=5):
    """The Bottleneck version of resnet34_8s_oracle.decisive_biases: every BatchNorm bias becomes +-amp so that every ReLU
    input lies far from zero.  Each residual stage (stem + layer1, layer2, layer3, layer4) draws ONE sign mask, shared by the
    stem bn1 (stage 0), every bn3 of the stage and its downsample BatchNorm -- so no +amp meets a -amp at a residual add --
    while bn1 and bn2 of every block draw their own masks."""
    r = net.resnet50_8s
    g = torch.Generator().manual_seed(seed)

    def mask(bn):
        return (torch.rand(bn.num_features, generator=g) < on_fraction).to(bn.bias.dtype) * 2 - 1

    with torch.no_grad():
        for i, layer in enumerate((r.layer1, r.layer2, r.layer3, r.layer4)):
            s = mask(layer[0].bn3)
            if i == 0:
                r.bn1.bias.copy_(amp * mask(r.bn1))     # 64 channels: the stem enters layer1 only through convolutions
            for blk in layer:
                blk.bn1.bias.copy_(amp * mask(blk.bn1))
                blk.bn2.bias.copy_(amp * mask(blk.bn2))
                blk.bn3.bias.copy_(amp * s)
                if blk.downsample is not None:
                    blk.downsample[1].bias.copy_(amp * s)
    return net


def calibrated_state(state, D, x):
    """``state`` with its running statistics replaced by the batch statistics of ``x`` (one train-mode forward with
    momentum 1, in x's dtype): eval-mode BatchNorm that normalises.  With the initial (0, 1) statistics the decisive
    construction leaves eval-mode ReLU inputs within 1e-5 of zero."""
    o = seeded_oracle(D).to(x.device, x.dtype)
    o.load_state_dict(state)
    for m in o.modules():
        if isinstance(m, nn.BatchNorm2d):
            m.momentum = 1.0
    with torch.no_grad():
        o.train()(x)
    return {k: (v.float().cpu() if v.is_floating_point() else v.cpu()) for k, v in o.state_dict().items()}


def relu_margins(net, x):
    """min |ReLU input| / max |ReLU input| over every ReLU of the float64 forward of ``net`` on ``x``, per ReLU call."""
    out = []

    def hook(_m, inp):
        v = inp[0].detach().abs()
        out.append((float(v.min()), float(v.max())))
    hs = [m.register_forward_pre_hook(hook) for m in net.modules() if isinstance(m, nn.ReLU)]
    try:
        net(x)
    finally:
        for h in hs:
            h.remove()
    return out
