#!/usr/bin/env python
"""bench_vae_sizes.py -- the RQ-VAE's fast tier at image sizes past its configured 256 x 256: the ImageNet VAE (f = 32, attention at
the 8 x 8 level) and the f8 VAE of scripts/bench_shapes.py (ch_mult 1,2,2,4, attention at the 32 x 32 level), at 256^2, 512^2 and
1024^2 with the same pixels per call (B = 16 / 4 / 1).  Synthetic weights, like bench.py.

Prints one JSON line per (VAE, size): the card's name and power limit (read in this run), encode and decode ms per call (CUDA
events over --steps calls after --warmup) and megapixels/s, and, from a torch.profiler run of its own, the spatial attention's
share of decode kernel time (over three calls) with the attention launches per call by name (vae_attn_kernel up to 1024 tokens, vae_attn_tc_kernel past it).
Then one line per attention shape, HW = 1024 and 4096 at C = 512: vae_attn_kernel against vae_attn_tc_kernel head to head (ms
per launch), and, for the f8 VAE at 512^2, the share of decode the fp32 kernel would take in place of the tensor-core one
(derived: the measured decode time with the measured attention time swapped for the fp32 kernel's).
Usage: python scripts/bench_vae_sizes.py [--steps 5] [--warmup 2]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "rq-vae-transformer_b200")
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

VAES = {
    # name: (ch_mult, attn_resolutions, code_shape)
    "imagenet": ((1, 1, 2, 2, 4, 4), (8,), (8, 8, 4)),
    "f8": ((1, 2, 2, 4), (32,), (32, 32, 4)),
}
SIZES = ((256, 16), (512, 4), (1024, 1))          # (pixels per side, B): 1 Mpx per call


def gpu_identity():
    out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit",
                          "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    name, power = [s.strip() for s in out.split(",")]
    return {"gpu": name, "power_limit": power}


def build(name, dev):
    from rqvae.models import create_model
    from rqvae.utils.config import Config, augment_arch_defaults
    ch_mult, attn, cs = VAES[name]
    dd = dict(double_z=False, z_channels=256, resolution=256, in_channels=3, out_ch=3, ch=128, ch_mult=list(ch_mult),
              num_res_blocks=2, attn_resolutions=list(attn), dropout=0.0)
    cfg = augment_arch_defaults(Config(
        type="rq-vae", hparams=dict(bottleneck_type="rq", embed_dim=256, n_embed=16384, latent_shape=[cs[0], cs[1], 256],
                                    code_shape=list(cs), shared_codebook=True, decay=0.99, restart_unused_codes=True,
                                    loss_type="mse", latent_loss_weight=0.25), ddconfig=dd))
    torch.manual_seed(0)
    with torch.device(dev):
        vae, _ = create_model(cfg)
    vae.eval().precision = "fast"
    return vae


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def attn_profile(fn, calls=3):
    """kernel time per call by torch.profiler over `calls` calls: total, and the spatial attention's kernels by name"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    total, attn, names = 0.0, 0.0, {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            us = e.time_range.elapsed_us()
            total += us
            if "vae_attn" in e.name:
                attn += us
                k = "vae_attn_tc_kernel" if "vae_attn_tc" in e.name else "vae_attn_kernel"
                names[k] = names.get(k, 0) + 1
    return {"attn_us": round(attn / calls, 1), "kernel_us": round(total / calls, 1), "share": round(attn / total, 4) if total else None,
            "attn_launches": {k: v / calls for k, v in names.items()}}


def attn_head_to_head(HW, C, steps, warmup, dev):
    from rqvae import _native as N
    g = torch.Generator(device=dev).manual_seed(HW)
    qkv = torch.randn(1, HW, 3 * C, device=dev, generator=g)
    out = torch.empty(1, HW, C, device=dev)
    res = {}
    for fn in ("rqb200_dbg_vae_attn", "rqb200_dbg_vae_attn_tc"):
        f = getattr(N.lib(), fn)
        res[fn[len("rqb200_dbg_"):] + "_ms"] = round(timed(lambda: N.check(f(N.ptr(qkv), N.ptr(out), 1, HW, C, N.stream_ptr()), fn),
                                                           steps, warmup), 4)
    flops = 4.0 * HW * HW * C
    res["tc_tflops"] = round(flops / (res["vae_attn_tc_ms"] * 1e-3) / 1e12, 1)
    res["speedup"] = round(res["vae_attn_ms"] / res["vae_attn_tc_ms"], 1)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--vaes", default=",".join(VAES))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vae_sizes.py: no CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.set_grad_enabled(False)
    ident = gpu_identity()
    f8_512 = None
    for name in args.vaes.split(","):
        vae = build(name, dev)
        f = vae.downsample_factor()
        for S, B in SIZES:
            x = torch.randn(B, 3, S, S, device=dev)
            z = vae.encode(x)
            enc_ms = timed(lambda: vae.encode(x), args.steps, args.warmup)
            dec_ms = timed(lambda: vae.decode(z), args.steps, args.warmup)
            prof = attn_profile(lambda: vae.decode(z))
            mpx = B * S * S / 1e6
            # both VAEs carry their attention at the latent level: (S / f)^2 tokens
            line = dict(ident, bench="vae_sizes", vae=name, size=S, B=B, latent=[S // f, S // f], attn_tokens=(S // f) ** 2,
                        encode_ms=round(enc_ms, 3), decode_ms=round(dec_ms, 3), encode_mpx_s=round(mpx / (enc_ms * 1e-3), 2),
                        decode_mpx_s=round(mpx / (dec_ms * 1e-3), 2), decode_attn=prof)
            print(json.dumps(line), flush=True)
            if name == "f8" and S == 512:
                f8_512 = dict(prof, B=B)
            del x, z
        del vae
        torch.cuda.empty_cache()
    for HW in (1024, 4096):
        line = dict(ident, bench="vae_attn_head_to_head", HW=HW, C=512, B=1, **attn_head_to_head(HW, 512, max(args.steps, 5), args.warmup, dev))
        if HW == 4096 and f8_512 is not None:
            n = sum(f8_512["attn_launches"].values())
            old_us = n * f8_512["B"] * line["vae_attn_ms"] * 1e3          # the fp32 kernel's time is linear in B
            rest = f8_512["kernel_us"] - f8_512["attn_us"]
            line["f8_512_decode_share_fp32_kernel_derived"] = round(old_us / (rest + old_us), 4)
            line["f8_512_decode_share_tc_kernel"] = f8_512["share"]
        print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
