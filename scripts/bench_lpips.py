#!/usr/bin/env python
"""Throughput of LPIPS: the native engine's fast tier (split-fp16 wgmma) and exact tier (fp32 FFMA) against the torch restatement
(tests/lpips_oracle.py: cuDNN at fp32 with TF32 off, with TF32 on, and under fp16 autocast) on the same GPU, with synthetic weights
(the rate does not depend on them).  Main case B = 64 pairs of 256^2; also 512^2 (B = 16) and 1024^2 (B = 4).  Cases run in ABBA
order after a warm-up; each prints one JSON line with the card's name and power limit, ms per batch, pairs/s and the achieved TFLOP/s
from the multiply-adds of the layer shapes (2 FLOP each; both images of a pair).  The fast tier's share of the 989 TFLOP/s dense fp16
figure counts the three fp16 products split-fp16 forms per multiply-add of every conv but conv1_1 (fp32).  Also: one reconstruction-
evaluation step at B = 64 (the ImageNet RQ-VAE's fast-tier forward, synthetic weights, then LPIPS of its output against the input),
timed with and without the LPIPS call, so LPIPS's share of such a step is measured.

    python scripts/bench_lpips.py [--reps 3]
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

from rqvae.losses.vqgan import LPIPS                                 # noqa: E402
from tests import lpips_oracle as LO                                 # noqa: E402

FP32_PEAK = 67.0          # NVIDIA H100 SXM data sheet, dense FP32 TFLOP/s (700 W)
FP16_PEAK = 989.0         # the same sheet, dense FP16 tensor-core TFLOP/s
SIZES = ((256, 64), (512, 16), (1024, 4))


def macs_per_image(H, W):
    """multiply-adds of the 13 convs on one H x W image (the heads add under 0.1 %): (all, conv1_1's alone)"""
    total, stem = 0, 0
    for name, ci, co, tap in LO.CONVS:
        m = H * W * ci * co * 9
        total += m
        if ci == 3:
            stem = m
        if tap:
            H, W = H // 2, W // 2
    return total, stem


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


def imagenet_vae(dev):
    from rqvae.models import create_model
    from rqvae.utils.config import Config, augment_arch_defaults
    dd = dict(double_z=False, z_channels=256, resolution=256, in_channels=3, out_ch=3, ch=128, ch_mult=[1, 1, 2, 2, 4, 4],
              num_res_blocks=2, attn_resolutions=[8], dropout=0.0)
    cfg = augment_arch_defaults(Config(
        type="rq-vae", hparams=dict(bottleneck_type="rq", embed_dim=256, n_embed=16384, latent_shape=[8, 8, 256], code_shape=[8, 8, 4],
                                    shared_codebook=True, decay=0.99, restart_unused_codes=True, loss_type="mse", latent_loss_weight=0.25),
        ddconfig=dd))
    torch.manual_seed(0)
    with torch.device(dev):
        vae, _ = create_model(cfg)
    vae.eval().precision = "fast"
    return vae


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_lpips: no CUDA device")
    dev = "cuda:0"
    torch.set_grad_enabled(False)
    sd = LO.synth_weights(3)
    with tempfile.TemporaryDirectory() as home:
        LO.write_weight_files(home, sd)
        os.environ["TORCH_HOME"] = home
        exact = LPIPS().to(dev).eval()
        fast = LPIPS().to(dev).eval()
        os.environ.pop("TORCH_HOME")
    exact.precision = "exact"
    fast.precision = "fast"
    sd32 = {k: v.to(dev) for k, v in sd.items()}
    name, power = gpu_info()

    for S, B in SIZES:
        g = torch.Generator().manual_seed(S)
        x = (torch.rand((B, 3, S, S), generator=g) * 2 - 1).to(dev)
        y = (x + 0.1 * torch.randn((B, 3, S, S), generator=g).to(dev)).clamp(-1, 1)

        def torch_ref(tf32, amp=False):
            def f():
                torch.backends.cudnn.allow_tf32 = tf32
                with torch.autocast("cuda", dtype=torch.float16, enabled=amp):
                    LO.lpips(sd32, x, y)
            return f
        cases = {"native_fast": lambda: fast(x, y, reduction="none"), "native_exact": lambda: exact(x, y, reduction="none"),
                 "torch_cudnn_fp32": torch_ref(False), "torch_cudnn_tf32": torch_ref(True), "torch_cudnn_fp16_autocast": torch_ref(False, True)}
        for fn in cases.values():                 # warm-up: module loads, cuDNN algorithm choice
            fn()
        times = {k: [] for k in cases}
        order = list(cases) + list(cases)[::-1]   # ABBA
        for k in order:
            times[k].append(timed(cases[k], a.reps))
        macs, stem = macs_per_image(S, S)
        for k, ts in times.items():
            t = min(ts)
            tflops = 2.0 * macs * 2 * B / t / 1e12
            row = dict(case=k, gpu=name, power_limit=power, pairs=B, size="%dx%d" % (S, S), ms_per_batch=round(t * 1e3, 2),
                       pairs_per_s=round(B / t, 1), gmacs_per_image=round(macs / 1e9, 2), tflops=round(tflops, 2))
            if k == "native_fast":                 # three fp16 products per multiply-add of the wgmma convs
                row["fp16_share_of_989tf"] = round(2.0 * 3 * (macs - stem) * 2 * B / t / 1e12 / FP16_PEAK, 3)
            elif k in ("native_exact", "torch_cudnn_fp32"):
                row["share_of_fp32_67tf"] = round(tflops / FP32_PEAK, 3)
            print(json.dumps(row), flush=True)
        del x, y

    # a reconstruction-evaluation step at B = 64: the RQ-VAE forward alone, and followed by LPIPS of its output against the input
    vae = imagenet_vae(dev)
    g = torch.Generator().manual_seed(1)
    xs = (torch.rand((64, 3, 256, 256), generator=g) * 2 - 1).to(dev)

    def vae_only():
        vae(xs)

    def vae_lpips():
        recon = vae(xs)[0]
        fast(xs, recon, reduction="none")
    for fn in (vae_only, vae_lpips):
        fn()
    times = {"rqvae_forward": [], "rqvae_forward_plus_lpips_fast": []}
    for k, fn in (("rqvae_forward", vae_only), ("rqvae_forward_plus_lpips_fast", vae_lpips), ("rqvae_forward_plus_lpips_fast", vae_lpips),
                  ("rqvae_forward", vae_only)):
        times[k].append(timed(fn, a.reps))
    t0, t1 = min(times["rqvae_forward"]), min(times["rqvae_forward_plus_lpips_fast"])
    print(json.dumps(dict(case="recon_eval_step", gpu=name, power_limit=power, pairs=64, size="256x256", vae="imagenet (fast tier)",
                          ms_rqvae_forward=round(t0 * 1e3, 2), ms_rqvae_forward_plus_lpips=round(t1 * 1e3, 2),
                          lpips_share=round((t1 - t0) / t1, 3))), flush=True)


if __name__ == "__main__":
    main()
