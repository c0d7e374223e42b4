#!/usr/bin/env python
"""Shared vs per-depth codebooks on the GPU.  Prints one JSON line per case with the card's name and power limit (read in this
run).  Each case times the two variants alternately in ABBA order after a warm-up and reports the median of the timed calls.

    rq_quantize   N = 4096, K = 16384, D = 4, C = 256 (an ImageNet B = 64 encode), the 2-CTA cluster kernel;
                  GFLOP/s = 2 N K C D / t (the distance GEMM's FLOPs)
    decode_code   the ImageNet-shaped RQ-VAE decoder on the fast tier at B = 64 (8x8x4 codes, K = 16384)

    python scripts/bench_rq_depthwise.py [--calls 24]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "rq-vae-transformer_b200")):
    sys.path.insert(0, p)

from oracle import synth                                     # noqa: E402
from rqvae.models import _bind as nb                         # noqa: E402
from rqvae.models import create_model                        # noqa: E402
from tests.helpers import vae_config                         # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit",
                          "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout.strip()
    name, power = [s.strip() for s in out.split(",")]
    return {"gpu": name, "power_limit": power}


def time_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def abba(fa, fb, calls, warmup=3):
    for _ in range(warmup):
        fa()
        fb()
    ta, tb = [], []
    for i in range(calls):
        for tag in ("ab" if i % 2 == 0 else "ba"):
            (ta if tag == "a" else tb).append(time_ms(fa if tag == "a" else fb))
    return statistics.median(ta), statistics.median(tb)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=24)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_rq_depthwise: needs a CUDA device")
    torch.set_grad_enabled(False)
    dev = "cuda"
    info = card()

    n, K, D = 4096, 16384, 4
    x = synth.randn_seeded((n, 256), 1).to(dev)
    tables = [synth.randn_seeded((K, 256), 10 + d).to(dev) for d in range(D)]
    same_codes = torch.equal(nb.rq_quantize(x, tables[0], D)[1], nb.rq_quantize(x, [tables[0].clone() for _ in range(D)], D)[1])
    ts, td = abba(lambda: nb.rq_quantize(x, tables[0], D), lambda: nb.rq_quantize(x, tables, D), args.calls)
    flop = 2.0 * n * K * 256 * D
    print(json.dumps(dict(case="rq_quantize", N=n, K=K, D=D, calls=args.calls, shared_ms=round(ts, 4), per_depth_ms=round(td, 4),
                          shared_gflops=round(flop / ts / 1e6, 1), per_depth_gflops=round(flop / td / 1e6, 1),
                          per_depth_over_shared=round(td / ts, 4), identical_tables_same_codes=same_codes, **info)), flush=True)

    cfg = vae_config("imagenet")
    with torch.device("meta"):
        shared, _ = create_model(cfg)
    sd = synth.synth_state_dict(synth.shapes_of(shared.state_dict()), 3)
    shared = shared.to_empty(device=dev)
    shared.load_state_dict({k: v.to(dev) for k, v in sd.items()})
    cfg.hparams.shared_codebook = False
    with torch.device("meta"):
        per_depth, _ = create_model(cfg)
    per_depth = per_depth.to_empty(device=dev)
    tabs = [synth.randn_seeded((K, 256), 20 + d) for d in range(D)]
    for d, t in enumerate(tabs):
        sd["quantizer.codebooks.%d.weight" % d] = torch.cat([t, torch.zeros(1, 256)], 0)
        sd["quantizer.codebooks.%d.embed_ema" % d] = t.clone()
    per_depth.load_state_dict({k: v.to(dev) for k, v in sd.items()})
    for m in (shared, per_depth):
        m.eval()
        m.precision = "fast"
    codes = synth.randint_seeded(0, K, (64, 8, 8, 4), 4).to(dev)
    ts, td = abba(lambda: shared.decode_code(codes), lambda: per_depth.decode_code(codes), args.calls)
    print(json.dumps(dict(case="decode_code_fast", B=64, K=K, D=D, calls=args.calls, shared_ms=round(ts, 3), per_depth_ms=round(td, 3),
                          per_depth_over_shared=round(td / ts, 4), **info)), flush=True)


if __name__ == "__main__":
    main()
