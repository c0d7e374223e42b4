#!/usr/bin/env python
"""bench_cached_forward.py -- the reference's own sampling loop (init_cache(), then cached_forward + sample_from_logits once per
token, transformers.py:343-369) on the fast tier, against sample() on the same model.  Synthetic weights, built as bench.py and
scripts/bench_shapes.py build them; top-k 1024, amp=True.

    in1400m       8x8x4 codes, the 1.4B ImageNet RQ-Transformer, B = 64 (bench.py's model)
    f8_huge_d4    32x32x4 codes, the `huge` RQ-Transformer of bench_shapes.py, at that script's first batch size (64)

Prints one JSON line per case: the card's name and power limit (read in this run); ms per token of the loop and of sample(),
timed with CUDA events in ABBA order (sample, loop, loop, sample) after one warm-up of each; the host time of each cached_forward
call (median and mean, us) and of the weight-change check inside it (param_fingerprint); the launches of a d = 0 and a d > 0
call; and at in1400m the stateless teacher-forced evaluation's time for one call at the first and at the last position (what every
call cost before the step kept its KV caches).
Usage: python scripts/bench_cached_forward.py [--cases in1400m,f8_huge_d4]"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "rq-vae-transformer_b200")
for p in (ROOT, PKG, os.path.join(ROOT, "scripts")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402
from rqvae import _native as N  # noqa: E402

CASES = ("in1400m", "f8_huge_d4")
TOP_K = 1024


def build(case, dev):
    if case == "in1400m":
        import bench
        ar, vae, _ = bench.build_models("in1400m", dev, "fast")
        return ar, vae, bench.MODELS["in1400m"][11]
    import bench_shapes
    ar, vae = bench_shapes.build(case, dev)
    return ar, vae, bench_shapes.SHAPES[case][8][0]


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def reference_loop(ar, vae, cond, B, stats=None):
    """transformers.py:343-369 through the public API"""
    from rqvae.utils.utils import sample_from_logits
    H, W, D = ar.block_size
    xs = torch.zeros(B, H, W, D, dtype=torch.long, device=cond.device)
    ar.init_cache()
    for h in range(H):
        for w in range(W):
            for d in range(D):
                t0 = time.perf_counter()
                logits = ar.cached_forward(xs[:, :h + 1], model_aux=vae, cond=cond, amp=True, sample_loc=(h, w, d))
                if stats is not None:
                    stats["host_s"].append(time.perf_counter() - t0)
                    if (h * W + w, d) in ((1, 0), (1, 1)):
                        stats["launches_d%d" % min(d, 1)] = ar.last_launches
                xs[:, h, w, d] = sample_from_logits(logits.to(torch.float32), 1.0, top_k=TOP_K, top_p=None)
    ar.init_cache()
    return xs


def run_case(case, dev, ident):
    ar, vae, B = build(case, dev)
    torch.set_grad_enabled(False)
    H, W, D = ar.block_size
    n_tok = H * W * D
    cond = torch.randint(0, 1000, (B, 1), device=dev, generator=torch.Generator(device=dev).manual_seed(1234))
    part = torch.zeros(B, H, W, D, dtype=torch.long, device=dev)
    sample = lambda: ar.sample(part, model_aux=vae, cond=cond, top_k=TOP_K, amp=True)  # noqa: E731
    stats = {"host_s": []}
    timed(sample)                                               # warm-up: engines, workspaces, graphs of both paths
    timed(lambda: reference_loop(ar, vae, cond, B))
    ms = {"sample": [], "loop": []}
    for which in ("sample", "loop", "loop", "sample"):
        t, _ = timed(sample if which == "sample" else (lambda: reference_loop(ar, vae, cond, B, stats)))
        ms[which].append(t)
    host_us = [s * 1e6 for s in stats["host_s"]]
    line = dict(ident, case=case, grid="%dx%dx%d" % (H, W, D), B=B, tokens=n_tok,
                loop_ms_per_token=sum(ms["loop"]) / len(ms["loop"]) / n_tok,
                sample_ms_per_token=sum(ms["sample"]) / len(ms["sample"]) / n_tok,
                loop_ms=ms["loop"], sample_ms=ms["sample"],
                host_us_per_call_median=statistics.median(host_us), host_us_per_call_mean=sum(host_us) / len(host_us),
                launches_d0=stats["launches_d0"], launches_d1=stats["launches_d1"])
    line["loop_over_sample"] = line["loop_ms_per_token"] / line["sample_ms_per_token"]
    t0 = time.perf_counter()
    for _ in range(20):
        N.param_fingerprint(ar)                                 # the weight-change check every call makes (RQTransformer._engine)
    line["param_fingerprint_us"] = (time.perf_counter() - t0) / 20 * 1e6
    if case == "in1400m":
        xs = sample()
        last = (H - 1, W - 1, D - 1)
        for name, loc in (("first", (0, 0, 0)), ("last", last)):
            call = lambda: ar._stateless_cached_forward(xs[:, :loc[0] + 1], vae, cond, True, loc)  # noqa: E731
            timed(call)
            t, _ = timed(call)
            line["stateless_ms_" + name] = t
        line["stateless_launches"] = ar.last_launches
    print(json.dumps(line), flush=True)
    ar._invalidate_native()
    del ar, vae
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default=",".join(CASES))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_cached_forward.py: no CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    import bench_shapes
    ident = bench_shapes.gpu_identity()
    for case in args.cases.split(","):
        run_case(case, dev, ident)
    return 0


if __name__ == "__main__":
    sys.exit(main())
