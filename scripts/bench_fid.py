#!/usr/bin/env python
"""Throughput of the FID feature pass: the native Inception engine's fast tier (split-fp16 wgmma) and exact tier (fp32 FFMA)
against the torch restatement (tests/inception_oracle.py, cuDNN fp32 with TF32 on and off) on the same GPU.  256 x 256 inputs
resized to 299 x 299, B = 250, synthetic weights (the rate does not depend on them).  Cases run in ABBA order after a warm-up;
each prints one JSON line with the card's name and power limit, images/s, and the achieved TFLOP/s from the multiply-adds of the
layer shapes (2 FLOP each).  The fast tier's share of the 989 TFLOP/s dense fp16 figure counts the three fp16 products split-fp16
forms per multiply-add of every conv but Conv2d_1a_3x3 (fp32).  Also: the fast tier at B = 64, the batch of bench.py's in1400m
sample + decode step, for the feature pass's share of such a step.

    python scripts/bench_fid.py [--batch 250] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "rq-vae-transformer_b200")]

from rqvae.metrics import inception as INC                           # noqa: E402
from tests import inception_oracle as IO                             # noqa: E402

FP32_PEAK = 67.0          # NVIDIA H100 SXM data sheet, dense FP32 TFLOP/s (700 W)
FP16_PEAK = 989.0         # the same sheet, dense FP16 tensor-core TFLOP/s


def macs_per_image():
    """multiply-adds of one 299 x 299 image: (all: every conv's output elements x Cin kh kw plus the fc, Conv2d_1a_3x3's alone)"""
    net = IO.Restated(IO.synth_weights(1))
    total = [0]
    stem = [0]
    conv = net.c

    def counting(n, x, stride=1, padding=0):
        y = conv(n, x, stride, padding)
        w = net.w[n]
        m = y.numel() * w.shape[1] * w.shape[2] * w.shape[3]
        total[0] += m
        if n == "blocks.0.0":
            stem[0] += m
        return y
    net.c = counting
    with torch.no_grad():
        net.forward(torch.zeros(1, 3, 299, 299))
    return total[0] + 2048 * 1008, stem[0]


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
    except Exception:
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def timed(fn, reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=250)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_fid: no CUDA device")
    dev = "cuda:0"
    torch.set_grad_enabled(False)
    sd = IO.synth_weights(3)
    with tempfile.TemporaryDirectory() as home:
        IO.write_weight_file(home, sd)
        os.environ["TORCH_HOME"] = home
        model = INC.InceptionV3([3]).to(dev)
        fast = INC.InceptionV3([3]).to(dev)
        os.environ.pop("TORCH_HOME")
    model.precision = "exact"
    fast.precision = "fast"
    net = IO.Restated({k: v.to(dev) for k, v in sd.items()})
    x = torch.rand((a.batch, 3, 256, 256), generator=torch.Generator().manual_seed(0)).to(dev)

    def native():
        model(x)

    def torch_ref(tf32):
        def f():
            torch.backends.cudnn.allow_tf32 = tf32
            net.forward(x)
        return f

    def native_fast():
        fast(x)
    x64 = x[:64].contiguous()

    def native_fast_b64():
        fast(x64)
    cases = {"native_fast": native_fast, "native_exact": native, "torch_cudnn_fp32": torch_ref(False), "torch_cudnn_tf32": torch_ref(True),
             "native_fast_b64": native_fast_b64}
    for fn in cases.values():                 # warm-up: module loads, cuDNN algorithm choice
        fn()
    times = {k: [] for k in cases}
    order = list(cases) + list(cases)[::-1]   # ABBA
    for k in order:
        times[k].append(timed(cases[k], a.reps))
    macs, stem = macs_per_image()
    name, power = gpu_info()
    for k, ts in times.items():
        t = min(ts)
        n = 64 if k.endswith("b64") else a.batch
        tflops = 2.0 * macs * n / t / 1e12
        row = dict(case=k, gpu=name, power_limit=power, batch=n, input="256x256 resized to 299x299", images_per_s=round(n / t, 1),
                   ms_per_batch=round(t * 1e3, 2), gmacs_per_image=round(macs / 1e9, 3), tflops=round(tflops, 2))
        if k.startswith("native_fast"):          # three fp16 products per multiply-add of the wgmma convs
            row["fp16_share_of_989tf"] = round(2.0 * 3 * (macs - stem - 2048 * 1008) * n / t / 1e12 / FP16_PEAK, 3)
        else:
            row["share_of_fp32_67tf"] = round(tflops / FP32_PEAK, 3)
        print(json.dumps(row))


if __name__ == "__main__":
    main()
