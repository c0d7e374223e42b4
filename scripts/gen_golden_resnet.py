#!/usr/bin/env python
"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/resnet.pt from torchvision's resnet101 and transforms in float64.

torchvision's models.resnet101() (no weights) is loaded with the seeded synthetic weights of tests/resnet_oracle.synth_weights(SEED),
cast to float64 and run in eval mode on the fp32 pixels of each case after transforms.CenterCrop (when the case crops) and
transforms.Normalize(ImageNet mean, std), both on float64 tensors.  Nothing reaches the network.

Recorded: SEED and, per case, its shape, crop, input seed (tests/resnet_oracle.case_inputs regenerates the pixels) and the float64
logits [B, 1000].  Cases: 256^2 with the 224 crop (torchvision's IMAGENET1K_V1 eval transform), 224^2 and 97 x 131 uncropped, 32^2 (the
smallest extent) and 512 x 256.  It also prints the RMS of the residual stream after each stage, which the synthetic weights keep O(1).

    python scripts/gen_golden_resnet.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import resnet_oracle as RO                                   # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "resnet.pt")
SEED = 71
CASES = [  # name, B, H, W, crop, input seed
    ("256_crop224", 2, 256, 256, 224, 301), ("224", 1, 224, 224, None, 302), ("97x131", 2, 97, 131, None, 303),
    ("32", 2, 32, 32, None, 304), ("512x256", 1, 512, 256, None, 305)]


def main():
    from torchvision import models, transforms
    torch.set_grad_enabled(False)
    sd = RO.synth_weights(SEED)
    net = models.resnet101()
    net.load_state_dict(sd, strict=True)
    net = net.double().eval()
    rms = {}
    for name in ("layer1", "layer2", "layer3", "layer4"):
        getattr(net, name).register_forward_hook(lambda m, i, o, name=name: rms.__setitem__(name, float(o.pow(2).mean().sqrt())))
    norm = transforms.Normalize(RO.MEAN, RO.STD)
    cases = []
    for name, B, H, W, crop, seed in CASES:
        case = dict(name=name, B=B, H=H, W=W, crop=crop, seed=seed)
        x = RO.case_inputs(case).double()
        if crop is not None:
            x = transforms.CenterCrop(crop)(x)
        lg = net(norm(x))
        case["logits"] = lg.clone()
        lp = torch.log_softmax(lg, 1)
        top2 = lg.topk(2, 1).values
        print("%-12s stage RMS %s  logits std %.3f  max log-prob %.3f  top-2 margin %s" % (
            name, " ".join("%.3f" % rms[k] for k in sorted(rms)), float(lg.std()), float(lp.max()),
            " ".join("%.4f" % float(m) for m in top2[:, 0] - top2[:, 1])))
        cases.append(case)
    torch.save(dict(seed=SEED, cases=cases), OUT)
    print("wrote %s (%d bytes)" % (OUT, os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
