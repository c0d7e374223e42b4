#!/usr/bin/env python
"""Throughput of the native ResNet-101 and of rejection sampling.

(a) ResNet-101 logits, B = 256 at 224^2 and B = 64 at 256^2 uncropped: the native engine's fast tier (split-fp16 wgmma) and exact tier
    (fp32 FFMA) against the torch restatement (tests/resnet_oracle.py: cuDNN at fp32 with TF32 off, with TF32 on, and under
    fp16 autocast), synthetic weights (the rate does not depend on them).  Cases run in ABBA order after a warm-up; each prints one
    JSON line with the card's name and power limit, ms per batch, images/s and the achieved TFLOP/s from the multiply-adds of the layer
    shapes (2 FLOP each).
(b) rejection_sample at the in1400m shapes bench.py builds (synthetic weights, fast tier), B = 64, candidates = 20, top-k 1024: accepted
    images/s and the classifier's share of the call (its time measured alone on the same 20 x 64 images).

    python scripts/bench_resnet.py [--reps 3] [--skip-rejection]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "rq-vae-transformer_b200")]

from rqvae.metrics.resnet import ResNet101                           # noqa: E402
from tests import resnet_oracle as RO                                # noqa: E402

CASES = ((224, 256), (256, 64))           # (extent, batch), no crop


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
    except Exception:
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def macs_per_image(H, W):
    """multiply-adds of the 104 convs and fc on one H x W image"""
    def out(n, k, s, p):
        return (n + 2 * p - k) // s + 1
    h, w = out(H, 7, 2, 3), out(W, 7, 2, 3)
    total = h * w * 3 * 64 * 49
    h, w = out(h, 3, 2, 1), out(w, 3, 2, 1)
    cin = 64
    for i, n in enumerate(RO.LAYERS):
        wd = 64 << i
        for b in range(n):
            s = 2 if (b == 0 and i > 0) else 1
            ho, wo = out(h, 3, s, 1), out(w, 3, s, 1)
            total += h * w * cin * wd + ho * wo * wd * wd * 9 + ho * wo * wd * 4 * wd
            if b == 0:
                total += ho * wo * cin * 4 * wd
            h, w, cin = ho, wo, 4 * wd
    return total + 2048 * 1000


def timed(fn, reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps


def bench_classifier(args, name, power):
    dev = "cuda:0"
    sd = RO.synth_weights(1)
    nets = {}
    for tier in ("fast", "exact"):
        m = ResNet101()
        m.load_state_dict(sd)
        m = m.to(dev)
        m.precision = tier
        nets[tier] = m
    sd32 = RO.sd_as(sd, torch.float32, dev)

    def torch_fn(mode):
        def f(x):
            torch.backends.cudnn.allow_tf32 = mode == "tf32"
            torch.backends.cuda.matmul.allow_tf32 = mode == "tf32"
            with torch.autocast("cuda", dtype=torch.float16, enabled=mode == "autocast"):
                return RO.logits(sd32, x, None)
        return f
    fns = {"native_fast": lambda x: nets["fast"](x, center_crop=None), "native_exact": lambda x: nets["exact"](x, center_crop=None),
           "torch_fp32": torch_fn("fp32"), "torch_tf32": torch_fn("tf32"), "torch_fp16_autocast": torch_fn("autocast")}
    with torch.no_grad():
        for S, B in CASES:
            x = torch.rand(B, 3, S, S, device=dev)
            for f in fns.values():
                f(x)
            times = {k: [] for k in fns}
            order = list(fns) + list(fns)[::-1]
            for _ in range(args.reps):
                for k in order:
                    times[k].append(timed(lambda: fns[k](x), 2))
            macs = macs_per_image(S, S) * B
            for k in fns:
                t = min(times[k])
                print(json.dumps(dict(case=k, gpu=name, power_limit=power, images=B, size="%dx%d" % (S, S), ms_per_batch=round(t * 1e3, 2),
                                      images_per_s=round(B / t, 1), tflops=round(2 * macs / t / 1e12, 1),
                                      gmacs_per_image=round(macs / B / 1e9, 3))), flush=True)
            torch.backends.cudnn.allow_tf32 = True
            torch.backends.cuda.matmul.allow_tf32 = False


def bench_rejection(args, name, power):
    import bench
    from rqvae.models.rqtransformer import rejection_sample
    dev = "cuda:0"
    ar, vae, _ = bench.build_models("in1400m", dev, "fast")
    clf = ResNet101()
    clf.load_state_dict(RO.synth_weights(1))
    clf = clf.to(dev)
    clf.precision = "fast"
    B, C = 64, 20
    labels = torch.arange(B, device=dev) * 7 % 1000
    kw = dict(top_k=1024, amp=True)
    with torch.no_grad():
        rejection_sample(ar, vae, clf, labels, candidates=2, **kw)                  # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        rejection_sample(ar, vae, clf, labels, candidates=C, **kw)
        torch.cuda.synchronize()
        t = time.perf_counter() - t0
        pix = torch.rand(B, 3, 256, 256, device=dev)
        tc = timed(lambda: clf.class_log_prob(pix, labels), C)
    print(json.dumps(dict(case="rejection_sample_in1400m", gpu=name, power_limit=power, images=B, candidates=C, top_k=1024, tier="fast",
                          seconds=round(t, 2), accepted_images_per_s=round(B / t, 2), classifier_ms_per_round=round(tc * 1e3, 2),
                          classifier_share=round(C * tc / t, 4))), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--skip-rejection", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_resnet: no CUDA device")
    name, power = gpu_info()
    bench_classifier(args, name, power)
    if not args.skip_rejection:
        bench_rejection(args, name, power)


if __name__ == "__main__":
    main()
