#!/usr/bin/env python
"""bench_shapes.py -- the fast tier on the long-sequence and head-less shapes of the reference's throughput harness
(measure_throughput: f=8 RQ-VAEs give 32x32 code maps; every d=1 run drops the head stack).  Synthetic weights, like bench.py.

    f8_huge_d4     32x32x4 codes, `huge` RQ-Transformer (E 1536, 24 heads, 42 body + 6 head layers), f8 RQ-VAE decode
    f16_huge_d1    16x16x1 codes, `huge` head-less (48 body + 0 head layers), f16 RQ-VAE decode

Prints one JSON line per shape: the card's name and power limit (read in this run), and per batch size images/s of
sample + decode, AR ms per spatial position over the first and the last 64 positions, and decode ms; once per shape the
teacher-forced forward(amp=True) ms, the share of decode time spent in vae_attn_kernel (torch.profiler, a run of its own) and
the body step attention's achieved KV read rate at the last position (RQB200_TRACE=1 stamps, a run of its own).
Usage: python scripts/bench_shapes.py [--shapes f8_huge_d4,f16_huge_d1] [--steps 1] [--warmup 1]"""
import argparse
import ctypes as C
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

SHAPES = {
    # name: (E, heads, n_body, n_head_layers, V = K, (H, W, D), vae ch_mult, vae attn_resolutions, batch sizes, forward batch)
    # (forward batch: the [B, H, W, D, V] fp32 logits of a 32x32x4 grid take 268 MB per image, twice)
    "f8_huge_d4": (1536, 24, 42, 6, 16384, (32, 32, 4), (1, 2, 2, 4), (32,), (64, 100), 8),
    "f16_huge_d1": (1536, 24, 48, 0, 16384, (16, 16, 1), (1, 1, 2, 2, 4), (16,), (100, 200), 100),
}
N_CLASSES = 1000
DECODE_CHUNK = 32        # images per decode_code call: the decoder's workspace at 256x256 is ~0.6 GB per image, the KV cache stays


def gpu_identity():
    out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit",
                          "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    name, power = [s.strip() for s in out.split(",")]
    return {"gpu": name, "power_limit": power}


def build(shape, dev):
    from rqvae.models import create_model
    from rqvae.utils.config import Config, augment_arch_defaults
    E, nh, nb, nhl, V, bs, ch_mult, attn = SHAPES[shape][:8]
    ar_cfg = augment_arch_defaults(Config(
        type="rq-transformer", vocab_size=V, block_size=list(bs), vocab_size_cond=N_CLASSES, block_size_cond=1, embed_dim=E,
        input_embed_dim=256, shared_tok_emb=True, shared_cls_emb=True, input_emb_vqvae=True, head_emb_vqvae=True,
        cumsum_depth_ctx=True, body=dict(n_layer=nb, block=dict(n_head=nh)), head=dict(n_layer=nhl, block=dict(n_head=nh))))
    dd = dict(double_z=False, z_channels=256, resolution=256, in_channels=3, out_ch=3, ch=128, ch_mult=list(ch_mult),
              num_res_blocks=2, attn_resolutions=list(attn), dropout=0.0)
    vae_cfg = augment_arch_defaults(Config(
        type="rq-vae", hparams=dict(bottleneck_type="rq", embed_dim=256, n_embed=V, latent_shape=[bs[0], bs[1], 256],
                                    code_shape=list(bs), shared_codebook=True, decay=0.99, restart_unused_codes=True,
                                    loss_type="mse", latent_loss_weight=0.25), ddconfig=dd))
    torch.manual_seed(0)
    with torch.device(dev):
        ar, _ = create_model(ar_cfg)
        vae, _ = create_model(vae_cfg)
    ar.eval().precision = "fast"
    vae.eval().precision = "fast"
    return ar, vae


def elapsed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def per_position_ms(ar, vae, cond, B):
    """AR ms per spatial position over the first and the last 64 positions: the engine's span entry point over
    [0, 64), [64, HW - 64), [HW - 64, HW) on one workspace, CUDA events between the spans (top-k 1024, no noise: q = 1)"""
    from rqvae import _native as N
    H, W, D = ar.block_size
    HW, V = H * W, ar.vocab_size[0]
    eng = ar._engine(ar._codebook_of(vae, D), N.MODE_FAST, 0)
    need = N.lib().rqb200_ar_workspace_bytes(eng["handle"], B)
    if eng["ws"] is None or eng["ws"].numel() < need:
        eng["ws"] = torch.empty(need, dtype=torch.uint8, device=cond.device)
    part = torch.zeros(B, H, W, D, dtype=torch.int64, device=cond.device)
    out = torch.empty_like(part)
    kk = (C.c_int32 * D)(*([min(1024, V)] * D))
    pp = (C.c_float * D)(*([1.0] * D))
    st = torch.cuda.current_stream()
    null = C.c_void_p(0)

    def span(p0, p1, resume):
        N.check(N.lib().rqb200_ar_sample_span(eng["handle"], N.ptr(part), N.ptr(cond), B, p0, p1, resume, 1.0, kk, pp, null, 0, null,
                                              null, N.ptr(out), N.ptr(eng["ws"]), eng["ws"].numel(), C.c_void_p(st.cuda_stream),
                                              None, None, 0, C.c_float(0.0), C.c_int(H), C.c_int(W)),
                "ar_sample_span")

    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    ev[0].record()
    span(0, 64, 0)
    ev[1].record()
    span(64, HW - 64, 1)
    ev[2].record()
    span(HW - 64, HW, 1)
    ev[3].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / 64, ev[2].elapsed_time(ev[3]) / 64


def vae_attn_share(vae, codes):
    from torch.profiler import ProfilerActivity, profile
    vae.decode_code(codes)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        vae.decode_code(codes)
        torch.cuda.synchronize()
    total = attn = 0.0
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            us = e.time_range.elapsed_us()
            total += us
            if "vae_attn" in e.name:
                attn += us
    return {"vae_attn_us": attn, "kernel_us": total, "share": attn / total if total else None}


def step_attention(ar, vae, cond, B):
    """Per-launch time of the body step's attention at the last position (the last replay of the code-token graph), from the
    RQB200_TRACE=1 stamps: from its dependency resolving to the next launch's dependency resolving (= the whole grid done).
    KV bytes per launch = B * n_head * t * 128 B * 2 (K and V rows, t cached rows)."""
    os.environ["RQB200_TRACE"] = "1"
    ar._invalidate_native()
    try:
        H, W, D = ar.block_size
        ar.sample(torch.zeros(B, H, W, D, dtype=torch.long, device=cond.device), model_aux=vae, cond=cond, top_k=1024, amp=True)
        torch.cuda.synchronize()
        rows = sorted(ar.native_trace(), key=lambda r: r[5])
    finally:
        del os.environ["RQB200_TRACE"]
        ar._invalidate_native()
    code_graph = [r for r in rows if 1024 <= r[5] < 2048]          # trace slots of the code-token body graph (second quarter)
    durs = [nxt[2] - r[2] for r, nxt in zip(code_graph, code_graph[1:]) if r[0] == "attn"]
    nh, cl = ar.config.body.block.n_head, ar.block_size_cond
    t = cl + H * W - 2                                                # cached rows read by the last body step
    byts = B * nh * t * 128 * 2
    us = sorted(durs)[len(durs) // 2] / 1e3 if durs else None
    return {"t": t, "launches": len(durs), "median_us": us, "kv_bytes": byts, "gb_per_s": byts / (us * 1e3) if us else None,
            "kernel": "attn_fast_kernel" if t > 320 else "attn_fast2_kernel"}


def run_shape(shape, steps, warmup, dev, ident):
    E, nh, nb, nhl, V, bs, ch_mult, attn, batches, fwd_B = SHAPES[shape]
    H, W, D = bs
    ar, vae = build(shape, dev)
    torch.set_grad_enabled(False)
    line = dict(ident, shape=shape, grid="%dx%dx%d" % bs, model="E %d, %d heads, %d + %d layers, V %d" % (E, nh, nb, nhl, V),
                per_batch=[])
    gen = torch.Generator(device=dev).manual_seed(1234)
    for B in batches:
        cond = torch.randint(0, N_CLASSES, (B, 1), device=dev, generator=gen)
        part = torch.zeros(B, H, W, D, dtype=torch.long, device=dev)

        def step():
            a_ms, codes = elapsed(lambda: ar.sample(part, model_aux=vae, cond=cond, top_k=1024, amp=True))
            d_ms, _ = elapsed(lambda: [vae.decode_code(c) for c in codes.split(DECODE_CHUNK)])
            return a_ms, d_ms, codes

        for _ in range(warmup):
            step()
        res = [step() for _ in range(steps)]
        a_ms = sum(r[0] for r in res) / steps
        d_ms = sum(r[1] for r in res) / steps
        first, last = per_position_ms(ar, vae, cond, B)
        mem = torch.cuda.max_memory_allocated() / 2**30
        torch.cuda.reset_peak_memory_stats()
        line["per_batch"].append({"B": B, "peak_gib": mem, "images_per_s": B / ((a_ms + d_ms) / 1e3), "sample_ms": a_ms, "decode_ms": d_ms,
                                  "ar_ms_per_position_first64": first, "ar_ms_per_position_last64": last})
        codes = res[-1][2]
        ar._invalidate_native()
        torch.cuda.empty_cache()
    # teacher-forced forward (batched passes; the body pass over cond_len + H*W - 1 tokens)
    xs = codes[:fwd_B]
    fcond = torch.randint(0, N_CLASSES, (fwd_B, 1), device=dev, generator=gen)
    elapsed(lambda: ar(xs, model_aux=vae, cond=fcond, amp=True))
    f_ms, _ = elapsed(lambda: ar(xs, model_aux=vae, cond=fcond, amp=True))
    line["forward_amp"] = {"B": fwd_B, "ms": f_ms}
    ar._invalidate_native()
    torch.cuda.empty_cache()
    line["decode_vae_attn"] = dict(vae_attn_share(vae, codes[:batches[0]]), B=batches[0])
    line["step_attention"] = dict(step_attention(ar, vae, cond[:batches[0]], batches[0]), B=batches[0])
    print(json.dumps(line), flush=True)
    del ar, vae
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--steps", type=int, default=1)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_shapes.py: no CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    ident = gpu_identity()
    for shape in args.shapes.split(","):
        run_shape(shape, args.steps, args.warmup, dev, ident)
    return 0


if __name__ == "__main__":
    sys.exit(main())
