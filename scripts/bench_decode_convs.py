#!/usr/bin/env python
"""bench_decode_convs.py -- where RQVAE.decode_code's time goes on the fast tier, conv shape by conv shape.

Runs decode_code of the ImageNet RQ-VAE (bench.py's decoder: ch 128, ch_mult (1, 1, 2, 2, 4, 4), 8x8x4 codes, random-init
weights) at B = 64 under torch.profiler (a run of its own, after warm-up and an untimed profiler-off run), matches the
implicit-GEMM conv kernels in launch order against the decoder's layer plan, and groups kernel time by conv shape.  For each
group it reports:

    tflops        algorithmic TFLOP/s: 2 * B * H * W * Cout * Cin * ks^2 * 3 (the three split-fp16 products) over kernel time
    l2_smem_tbps  the L2 -> shared-memory bytes the kernel's tile plan loads (computed from the shape, not measured) over kernel time

The tile plan is recognised from the kernel name: conv3x3_wreg_kernel (Cout % 128 == 0) and conv3x3_tc_kernel load one halo tile
per 64-channel slab and stream the nine taps' weight slabs; conv_tc_kernel loads an activation box and a weight slab per (tap,
slab).  Prints one JSON line with the card's name and power limit, read in this run.
Usage: python scripts/bench_decode_convs.py [--batch 64] [--reps 3]"""
import argparse
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "rq-vae-transformer_b200")
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

DD = dict(double_z=False, z_channels=256, resolution=256, in_channels=3, out_ch=3, ch=128, ch_mult=[1, 1, 2, 2, 4, 4],
          num_res_blocks=2, attn_resolutions=[8], dropout=0.0)
EMBED_DIM, CODE_SHAPE, N_EMBED = 256, (8, 8, 4), 16384
PASSES = 3


def gpu_identity():
    out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit",
                          "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    name, power = [s.strip() for s in out.split(",")]
    return {"gpu": name, "power_limit": power}


def conv_plan(dd=DD, embed_dim=EMBED_DIM):
    """(ks, H, W, Cin, Cout) of every conv decode_code launches, in launch order (csrc/vae_engine.cu decode)"""
    nl, nb = len(dd["ch_mult"]), dd["num_res_blocks"]
    res = dd["resolution"] >> (nl - 1)
    ch = dd["ch"] * dd["ch_mult"][-1]
    plan = [(1, res, res, embed_dim, dd["z_channels"]), (3, res, res, dd["z_channels"], ch)]

    def resblock(r, cin, cout):
        plan.append((3, r, r, cin, cout))
        if cin != cout:
            plan.append((1, r, r, cin, cout))
        plan.append((3, r, r, cout, cout))

    def attn(r, c):
        plan.extend([(1, r, r, c, 3 * c), (1, r, r, c, c)])

    resblock(res, ch, ch)
    attn(res, ch)
    resblock(res, ch, ch)
    for lvl in range(nl - 1, -1, -1):
        cout = dd["ch"] * dd["ch_mult"][lvl]
        for _ in range(nb + 1):
            resblock(res, ch, cout)
            ch = cout
            if res in dd["attn_resolutions"]:
                attn(res, ch)
        if lvl != 0:
            plan.append((3, 2 * res, 2 * res, ch, ch))
            res *= 2
    plan.append((3, res, res, ch, dd["out_ch"]))
    return plan


def block_n(kernel, cout):
    """output channels per tile (csrc/conv_tc.cu launch_conv_tc): 128 on conv3x3_wreg_kernel, at most 64 on conv3x3_tc_kernel"""
    if kernel == "conv3x3_wreg_kernel":
        return 128
    wide = cout % 256 == 0 and not kernel.startswith("conv3x3")
    return 16 if cout <= 16 else (256 if wide else (128 if cout % 128 == 0 else 64))


def cdiv(a, b):
    return -(-a // b)


def plan_bytes(kernel, B, ks, H, W, cin, cout):
    """L2 -> shared-memory bytes of one launch under the kernel's tile plan (hi and lo operands: PASSES == 3)"""
    ops = 2 if PASSES == 3 else 1
    bn = block_n(kernel, cout)
    n_tiles = cdiv(cout, bn)
    slabs = cin // 64
    if kernel.startswith("conv3x3"):
        th = 32 if H >= 32 and kernel == "conv3x3_wreg_kernel" else (16 if H >= 16 else 8)
        nbt = 2 if th == 8 else 1
        tiles = cdiv(W, 8) * cdiv(H, th) * cdiv(B, nbt) * n_tiles
        per_slab = 10 * (th + 2) * nbt * 128 + 9 * bn * 128
        return tiles * slabs * per_slab * ops
    tw = min(W, 16)
    th = min(128 // tw, H)
    nbt = 128 // (tw * th)
    tiles = (W // tw) * (H // th) * cdiv(B, nbt) * n_tiles
    return tiles * ks * ks * slabs * (128 * 128 + bn * 128) * ops


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--reps", type=int, default=3, help="profiler-off decode_code calls timed with CUDA events")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_decode_convs.py: no CUDA device")
    from torch.profiler import ProfilerActivity, profile
    from rqvae.models import create_model
    from rqvae.utils.config import Config, augment_arch_defaults

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.set_grad_enabled(False)
    ident = gpu_identity()
    B = args.batch
    cfg = augment_arch_defaults(Config(
        type="rq-vae", hparams=dict(bottleneck_type="rq", embed_dim=EMBED_DIM, n_embed=N_EMBED,
                                    latent_shape=[CODE_SHAPE[0], CODE_SHAPE[1], EMBED_DIM], code_shape=list(CODE_SHAPE),
                                    shared_codebook=True, decay=0.99, restart_unused_codes=True, loss_type="mse",
                                    latent_loss_weight=0.25), ddconfig=DD))
    torch.manual_seed(0)
    with torch.device(dev):
        vae, _ = create_model(cfg)
    vae.eval().precision = "fast"
    codes = torch.randint(0, N_EMBED, (B, *CODE_SHAPE), device=dev, generator=torch.Generator(device=dev).manual_seed(1234))

    for _ in range(2):
        vae.decode_code(codes)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.reps):
        vae.decode_code(codes)
    e1.record()
    torch.cuda.synchronize()
    decode_ms = e0.elapsed_time(e1) / args.reps

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        vae.decode_code(codes)
        torch.cuda.synchronize()
    kern = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA),
                  key=lambda e: e.time_range.start)
    total_us = sum(e.time_range.elapsed_us() for e in kern)
    convs = [(e, m.group(1)) for e in kern for m in [re.search(r"\b(conv_tc_kernel|conv3x3_tc_kernel|conv3x3_wreg_kernel)\b", e.name)] if m]
    plan = conv_plan()
    if len(convs) != len(plan):
        raise SystemExit("bench_decode_convs.py: %d conv kernels in the trace, the decoder plan has %d" % (len(convs), len(plan)))

    groups = {}
    for (e, kname), (ks, H, W, cin, cout) in zip(convs, plan):
        key = "%dx%d %dx%d %d->%d" % (ks, ks, H, W, cin, cout)
        g = groups.setdefault(key, {"shape": key, "kernel": kname, "bn": block_n(kname, cout), "launches": 0, "kernel_us": 0.0,
                                    "alg_flop": 0.0, "l2_smem_bytes": 0.0})
        g["launches"] += 1
        g["kernel_us"] += e.time_range.elapsed_us()
        g["alg_flop"] += 2.0 * B * H * W * cout * cin * ks * ks * PASSES
        g["l2_smem_bytes"] += plan_bytes(kname, B, ks, H, W, cin, cout)
    out = []
    for g in sorted(groups.values(), key=lambda g: -g["kernel_us"]):
        s = g["kernel_us"] * 1e-6
        out.append(dict(g, kernel_ms=g["kernel_us"] / 1e3, tflops=g["alg_flop"] / s / 1e12, l2_smem_tbps=g["l2_smem_bytes"] / s / 1e12,
                        flop_per_byte=g["alg_flop"] / g["l2_smem_bytes"]))
    conv_us = sum(g["kernel_us"] for g in groups.values())
    flop = sum(g["alg_flop"] for g in groups.values())
    line = dict(ident, B=B, decoder="ImageNet RQ-VAE, ch 128, ch_mult (1,1,2,2,4,4), 256x256, fast tier (split-fp16, 3 products)",
                decode_ms=decode_ms, kernel_ms=total_us / 1e3, conv_kernel_ms=conv_us / 1e3,
                conv_tflops=flop / (conv_us * 1e-6) / 1e12,
                conv_l2_smem_gb=sum(g["l2_smem_bytes"] for g in groups.values()) / 1e9, groups=out)
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
