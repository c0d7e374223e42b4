#!/usr/bin/env python
"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/lpips.pt from the UNMODIFIED reference rqvae/losses/vqgan/lpips.py.

The reference's losses package imports its optimizer and discriminator at package level, so lpips.py and lpips_utils.py are loaded by
file path under a stand-in package name.  models.vgg16 (this machine's torchvision 0.26 still takes pretrained=False, with a warning)
and get_ckpt_path are patched to return the synthetic weights of tests/lpips_oracle.synth_weights(SEED): nothing reaches the network.

Recorded, all computed in float64 by the reference LPIPS (eval mode):
  - the LPIPS state_dict key layout (keys and shapes, in order) for use_dropout=True and use_dropout=False;
  - per case (tests/lpips_oracle.case_inputs): the per-tap spatial averages [B, 5] (res[k] of the reference's forward) and the
    reduction='none' values [B]; cases 256^2 (B 2), 64^2, 16^2 (a 1 x 1 relu5_3), 100 x 70 (odd extents through the pools),
    512 x 256, an identical pair and a pair whose target is the input plus small seeded noise.

Needs the reference tree:   python scripts/gen_golden_lpips.py
"""
import importlib.util
import os
import sys
import tempfile
import types
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_loader as R                                  # noqa: E402
from tests import lpips_oracle as LO                                # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "lpips.pt")
SEED = 53
CASES = [  # name, B, H, W, kind, input seed
    ("256", 2, 256, 256, "random", 201), ("64", 1, 64, 64, "random", 202), ("16", 2, 16, 16, "random", 203),
    ("100x70", 1, 100, 70, "random", 204), ("512x256", 1, 512, 256, "random", 205), ("identical", 2, 64, 48, "identical", 206),
    ("noisy", 2, 64, 64, "noisy", 207)]


def load_reference_lpips():
    d = os.path.join(R.REFERENCE_ROOT, "rqvae", "losses", "vqgan")
    pkg = types.ModuleType("reflpips")
    pkg.__path__ = [d]
    sys.modules["reflpips"] = pkg
    mods = {}
    for name in ("lpips_utils", "lpips"):
        spec = importlib.util.spec_from_file_location("reflpips." + name, os.path.join(d, name + ".py"))
        m = importlib.util.module_from_spec(spec)
        sys.modules["reflpips." + name] = m
        spec.loader.exec_module(m)
        mods[name] = m
    return mods["lpips"]


def main():
    torch.set_num_threads(8)
    lp = load_reference_lpips()
    sd = LO.synth_weights(SEED)
    tv_models = lp.models

    def fake_vgg16(pretrained=True):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            m = tv_models.vgg16(pretrained=False)
        feats = {k.split(".", 2)[2]: v for k, v in sd.items() if k.startswith("net.")}
        m.features.load_state_dict(feats, strict=False)
        for k, v in feats.items():
            assert torch.equal(m.features.state_dict()[k], v), k
        return m
    lp.models = types.SimpleNamespace(vgg16=fake_vgg16)

    tmp = tempfile.mkdtemp()
    ckpt = os.path.join(tmp, "vgg.pth")
    torch.save({k: v for k, v in sd.items() if k.startswith("lin")}, ckpt)
    lp.get_ckpt_path = lambda name, root=None, check=False: ckpt

    layouts = {}
    for dropout in (True, False):
        m = lp.LPIPS(use_dropout=dropout)
        layouts[dropout] = [(k, list(v.shape)) for k, v in m.state_dict().items()]
    model = lp.LPIPS(use_dropout=True).eval()
    got = model.state_dict()
    for k, v in sd.items():
        assert torch.equal(got[k], v), k
    model = model.double()

    cases = []
    with torch.no_grad():
        for name, B, H, W, kind, seed in CASES:
            case = dict(name=name, B=B, H=H, W=W, kind=kind, seed=seed)
            x0, x1 = LO.case_inputs(case)
            x0, x1 = x0.double(), x1.double()
            # the reference's forward, keeping its per-tap spatial averages
            outs0, outs1 = model.net(model.scaling_layer(x0)), model.net(model.scaling_layer(x1))
            lins = [model.lin0, model.lin1, model.lin2, model.lin3, model.lin4]
            res = [lp.spatial_average(lins[k].model((lp.normalize_tensor(outs0[k]) - lp.normalize_tensor(outs1[k])) ** 2))
                   for k in range(5)]
            val = model(x0, x1, reduction="none")
            layers = torch.cat([r.reshape(B, 1) for r in res], 1)
            assert torch.equal(layers.sum(1), val.reshape(B)) or float((layers.sum(1) - val.reshape(B)).abs().max()) < 1e-15
            case.update(layers=layers, val=val.reshape(B), tap_shapes=[list(o.shape) for o in outs0])
            cases.append(case)
            print("%-10s val %s  taps %s" % (name, " ".join("%.6g" % float(v) for v in val.reshape(-1)),
                                              " ".join("%.3g" % float(t.mean()) for t in outs0)))

    torch.save(dict(seed=SEED, layouts={"dropout": layouts[True], "no_dropout": layouts[False]}, cases=cases), OUT)
    print("wrote %s (%.0f KB)" % (OUT, os.path.getsize(OUT) / 1024))


if __name__ == "__main__":
    main()
