#!/usr/bin/env python
"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/fid.pt from the UNMODIFIED reference rqvae/metrics/inception.py and fid.py.

The reference's metrics package imports clip at package level, so its inception.py and fid.py are loaded by file path (under a
stand-in package name, so fid.py's `from .inception import InceptionV3` resolves to the reference's file).  fid_inception_v3()
is built with that module's load_state_dict_from_url patched to return synthetic weights: nothing reaches the network.  It uses
this machine's torchvision (0.26 still takes the reference's pretrained=False, with a warning).

Weights: conv / fc from oracle/synth.py, the BN affine from synth.randn_seeded (tests/inception_oracle.synth_weights, seed SEED);
the BN running statistics from one train-mode pass (momentum 1) over a seeded calibration batch, so every layer's output stays
O(1) through the 94 convs.  The running statistics are stored (small); the weights are rebuilt from the seed.

Recorded, all computed in float64 by the reference InceptionV3(output_blocks=[0, 1, 2, 3]):
  - the reference InceptionV3 / InceptionWrapper state_dict key layout (keys and shapes, in order);
  - per case (seeded input in [0, 1)): block-3 features [B, 2048], logits [B, 1008], per-image channel means of blocks 0-2;
    cases 299^2 (B 2), 256^2, 64^2 and 192 x 128 resized; 75^2, 80 x 96 and 512^2 with resize_input=False;
  - mean_covar_numpy and frechet_distance on seeded well-conditioned Gaussians (d = 64, 200 samples each), and frechet_distance
    on the singular covariances of 20 of those samples (with whether the eps retry ran).  scipy >= 1.16 has no `disp` argument
    to sqrtm; the reference's call is adapted to it here.

Needs the reference tree:   python scripts/gen_golden_inception.py
"""
import importlib.util
import logging
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_loader as R                                  # noqa: E402
from tests import inception_oracle as IO                            # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "fid.pt")
SEED = 41
CASES = [  # name, B, H, W, resize_input, input seed
    ("299", 2, 299, 299, True, 101), ("256", 1, 256, 256, True, 102), ("64", 1, 64, 64, True, 103),
    ("192x128", 1, 192, 128, True, 104), ("75", 1, 75, 75, False, 105), ("80x96", 1, 80, 96, False, 106),
    ("512", 1, 512, 512, False, 107)]


def load_reference_metrics():
    d = os.path.join(R.REFERENCE_ROOT, "rqvae", "metrics")
    pkg = types.ModuleType("refmetrics")
    pkg.__path__ = [d]
    sys.modules["refmetrics"] = pkg
    mods = {}
    for name in ("inception", "fid"):
        spec = importlib.util.spec_from_file_location("refmetrics." + name, os.path.join(d, name + ".py"))
        m = importlib.util.module_from_spec(spec)
        sys.modules["refmetrics." + name] = m
        spec.loader.exec_module(m)
        mods[name] = m
    return mods["inception"], mods["fid"]


def main():
    torch.set_num_threads(8)
    inc, fid = load_reference_metrics()
    # scipy >= 1.16 dropped sqrtm's `disp` argument (and its second return value), which the reference passes
    sqrtm = fid.linalg.sqrtm
    fid.linalg = types.SimpleNamespace(sqrtm=lambda a, disp=True: (sqrtm(a), 0.0) if not disp else sqrtm(a))
    synth_tv = IO.to_torchvision_keys(IO.synth_weights(SEED))

    def fake_load(url, *a, **k):
        assert url == inc.FID_WEIGHTS_URL
        return {k: v.clone() for k, v in synth_tv.items()}
    inc.load_state_dict_from_url = fake_load

    model = fid.InceptionWrapper([0, 1, 2, 3])
    layout = [(k, list(v.shape)) for k, v in fid.InceptionWrapper([3]).state_dict().items()]
    assert [k for k, _ in layout] == list(IO.layout()), "the restatement's layout differs from the reference's"
    n_values = sum(int(np.prod(s)) for _, s in layout)
    print("InceptionWrapper: %d state_dict entries, %.1f M values" % (len(layout), n_values / 1e6))

    # calibration: BN running statistics = the statistics of a seeded batch, layer by layer
    model = model.double()
    for m in model.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.momentum = 1.0
    model.train()
    # half pixel noise, half smooth (64^2 noise upsampled): the resized cases' inputs are smooth
    gc = torch.Generator().manual_seed(SEED + 1)
    calib = torch.cat([torch.rand((4, 3, 299, 299), generator=gc),
                       torch.nn.functional.interpolate(torch.rand((4, 3, 64, 64), generator=gc), size=(299, 299), mode="bilinear",
                                                       align_corners=False)]).double()
    with torch.no_grad():
        model(calib)
    model.eval()
    stats = {k: v.float().clone() for k, v in model.state_dict().items() if "running_" in k}
    # the fixture's weights are float32: round the calibrated statistics and run the reference on exactly those
    sd = model.state_dict()
    for k, v in stats.items():
        sd[k].copy_(v.double())

    cases = []
    with torch.no_grad():
        for name, B, H, W, resize, seed in CASES:
            model.resize_input = resize
            x = torch.rand((B, 3, H, W), generator=torch.Generator().manual_seed(seed))
            outs, logits = inc.InceptionV3.forward(model, x.double(), return_logits=True)
            cases.append(dict(name=name, B=B, H=H, W=W, resize=resize, seed=seed,
                              features=outs[3].reshape(B, -1).float(), logits=logits.float(),
                              means=[o.mean((2, 3)).float() for o in outs[:3]],
                              block_shapes=[list(o.shape) for o in outs[:3]]))
            f = outs[3].reshape(B, -1)
            print("%-8s features rms %.3f  logits rms %.3f  block means %s" % (
                name, float(f.pow(2).mean().sqrt()), float(logits.pow(2).mean().sqrt()),
                " ".join("%.3f" % float(o.mean()) for o in outs[:3])))

    # Frechet distance on seeded Gaussians, d = 64
    g = np.random.default_rng(SEED)
    d = 64
    a1, a2 = g.normal(size=(d, d)) / np.sqrt(d), g.normal(size=(d, d)) / np.sqrt(d)
    x1 = g.normal(size=(200, d)) @ (np.eye(d) + 0.5 * a1) + g.normal(size=d)
    x2 = g.normal(size=(200, d)) @ (np.eye(d) + 0.5 * a2) + g.normal(size=d)
    mu1, s1 = fid.mean_covar_numpy(x1)
    mu2, s2 = fid.mean_covar_numpy(x2)
    fd = float(fid.frechet_distance(mu1, s1, mu2, s2))
    # singular covariances (20 samples in 64 dimensions), the situation of an FID over fewer images than features; with the eps
    # retry recorded when sqrtm of their product is not finite
    _, r1 = fid.mean_covar_numpy(x1[:20])
    _, r2 = fid.mean_covar_numpy(x2[:20])
    warned = []

    class _H(logging.Handler):
        def emit(self, rec):
            warned.append(rec.getMessage())
    logging.getLogger().addHandler(_H())
    fd_eps = float(fid.frechet_distance(mu1, r1, mu2, r2))
    print("frechet %.6f, singular-product case %.6f (retried with eps: %s)" % (fd, fd_eps, bool(warned)))
    frechet = dict(x1=torch.from_numpy(x1), x2=torch.from_numpy(x2), mu1=torch.from_numpy(mu1), sigma1=torch.from_numpy(s1),
                   mu2=torch.from_numpy(mu2), sigma2=torch.from_numpy(s2), fd=fd, n_singular=20,
                   fd_singular=fd_eps, eps_retried=bool(warned))

    torch.save(dict(seed=SEED, layout=layout, running_stats=stats, cases=cases, frechet=frechet), OUT)
    print("wrote %s (%.0f KB)" % (OUT, os.path.getsize(OUT) / 1024))


if __name__ == "__main__":
    main()
