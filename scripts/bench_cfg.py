#!/usr/bin/env python
"""Classifier-free guidance on the fast AR tier, end to end: in1400m B 64, cc3m654m_16 B 16 and t2i3900m B 16, the models built as
bench.py builds them (default init under torch.manual_seed(0), the RQ-VAE of the same config), top-k 1024 and the config's top-p.
uncond is the all-zero condition (class 0, or the all-zero caption).

Three runs per case, alternated in ABBA order (median over --calls): unguided at B images, guided at B images (2B engine rows), and
unguided at 2B images.  Per run: images/s of sample + decode, AR ms per spatial position, and the kernels launched per sample call;
the guided / unguided AR time ratios beside them.  One JSON line per case with the card's name and power limit read in this run.

    python scripts/bench_cfg.py [--calls 4] [--cases in1400m,cc3m654m_16,t2i3900m]
"""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "rq-vae-transformer_b200")):
    sys.path.insert(0, p)

import bench                                                  # noqa: E402
from rqvae import _native as N                                # noqa: E402

CASES = {"in1400m": 64, "cc3m654m_16": 16, "t2i3900m": 16}
RUNS = ("unguided_B", "guided_B", "unguided_2B")


def card():
    out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit",
                          "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout.strip()
    name, power = [s.strip() for s in out.split(",")]
    return {"gpu": name, "power_limit": power}


def run_case(name, B, calls, scale, info):
    E, nh, nb, nhl, V, bs, vc, cl, attn, ch_mult, top_p = bench.MODELS[name][:11]
    ar, vae, _ = bench.build_models(name, "cuda", "fast")
    g = torch.Generator().manual_seed(11)
    cond = torch.randint(0, vc, (2 * B, cl), generator=g).to("cuda")
    uncond = torch.zeros(B, cl, dtype=torch.long, device="cuda")
    z = torch.zeros(2 * B, *bs, dtype=torch.long, device="cuda")
    kw = dict(model_aux=vae, top_k=min(1024, V), top_p=top_p, amp=True)
    args = {"unguided_B": dict(partial_sample=z[:B], cond=cond[:B]),
            "guided_B": dict(partial_sample=z[:B], cond=cond[:B], cfg_scale=scale, uncond=uncond),
            "unguided_2B": dict(partial_sample=z, cond=cond)}
    n_pos = bs[0] * bs[1]

    def step(r):
        a, b, c = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        n0 = N.launch_count["total"]
        a.record()
        codes = ar.sample(**args[r], **kw)
        b.record()
        launches = N.launch_count["total"] - n0
        vae.decode_code(codes)
        c.record()
        c.synchronize()
        return a.elapsed_time(c), a.elapsed_time(b), launches, codes.shape[0]

    for r in RUNS:                                            # engine builds, graph captures, warm-up
        step(r)
        step(r)
    res = {r: {"total": [], "ar": [], "launches": None, "images": None} for r in RUNS}
    for i in range(calls):
        for r in (RUNS if i % 2 == 0 else RUNS[::-1]):
            t, a, launches, n_img = step(r)
            res[r]["total"].append(t)
            res[r]["ar"].append(a)
            res[r]["launches"], res[r]["images"] = launches, n_img
    out = {}
    for r in RUNS:
        t, a = statistics.median(res[r]["total"]), statistics.median(res[r]["ar"])
        out[r] = dict(images=res[r]["images"], images_per_s=round(res[r]["images"] / t * 1e3, 2), ar_ms=round(a, 2),
                      ar_ms_per_position=round(a / n_pos, 4), launches_per_call=res[r]["launches"])
    ratio = dict(guided_vs_unguided_B=round(out["guided_B"]["ar_ms"] / out["unguided_B"]["ar_ms"], 3),
                 guided_vs_unguided_2B=round(out["guided_B"]["ar_ms"] / out["unguided_2B"]["ar_ms"], 3))
    print(json.dumps(dict(case=name, B=B, cfg_scale=scale, calls=calls, order="ABBA", **out, ar_time_ratio=ratio, **info)), flush=True)
    del ar, vae
    gc.collect()
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=4)
    ap.add_argument("--cases", default=",".join(CASES))
    ap.add_argument("--scale", type=float, default=3.0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_cfg: needs a CUDA device")
    torch.set_grad_enabled(False)
    info = card()
    for name in args.cases.split(","):
        run_case(name, CASES[name], args.calls, args.scale, info)


if __name__ == "__main__":
    main()
