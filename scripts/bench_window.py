#!/usr/bin/env python
"""Sliding-window sampling (`sample()` on a canvas larger than the model's grid) on the fast AR tier, end to end: in1400m as bench.py
builds it (synthetic weights, fp16, B = 64, top-k 1024), partial_sample a seeded random code map, seeded labels.

Cases (canvas of codes; 256 px per 8 codes):
    8x8            today's call on the grid (the baseline)
    8x16, 16x16    every canvas token sampled
    8x16_outpaint  the left half kept (an encoded 256x256 image extended to 256x512): only the right half is sampled

In ABBA order over the cases (median over --calls): AR ms per call, launches per call, window prefills per call (the segments of the
canvas walk, tests/window_oracle.py), ms per sampled position, and images/s of sample + decode at the canvas size (decode:
vae.decode of the summed code embeddings, the README's recipe, 16 images per call).  One JSON line per case with the card's name and
power limit read in this run.

    python scripts/bench_window.py [--calls 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "rq-vae-transformer_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from tests import window_oracle as WO  # noqa: E402

DECODE_CHUNK = 16           # images per decode call
CASES = {"8x8": ((8, 8), False), "8x16": ((8, 16), False), "16x16": ((16, 16), False), "8x16_outpaint": ((8, 16), True)}


def card():
    out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit",
                          "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout.strip()
    name, power = [s.strip() for s in out.split(",")]
    return {"gpu": name, "power_limit": power}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--B", type=int, default=64)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_window.py measures on a CUDA device; none is visible")
    torch.set_grad_enabled(False)
    import bench
    ar, vae, _ = bench.build_models("in1400m", "cuda", "fast")
    os.environ["RQB200_FAST_DTYPE"] = "fp16"
    ar._invalidate_native()
    H, W, D = ar.block_size
    V, B = ar.vocab_size[0], args.B
    g = torch.Generator().manual_seed(11)
    cond = torch.randint(0, ar.vocab_size_cond, (B, ar.block_size_cond), generator=g).to("cuda")
    inputs = {}
    for name, (canvas, outpaint) in CASES.items():
        partial = torch.randint(0, V, (B, *canvas, D), generator=g).to("cuda")
        keep = None
        if outpaint:
            keep = torch.zeros(*canvas, 1, dtype=torch.bool, device="cuda")
            keep[:, :canvas[1] // 2] = True
        inputs[name] = (partial, keep)

    def step(name):
        partial, keep = inputs[name]
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        ev[0].record()
        codes = ar.sample(partial, model_aux=vae, cond=cond, top_k=1024, amp=True, keep_mask=keep)
        ev[1].record()
        launches = ar.last_launches
        for c in codes.split(DECODE_CHUNK):                # (a 512x512 decode of all 64 images at once needs ~48 GB of workspace)
            pix = vae.decode(vae.quantizer.embed_code_with_depth(c, True)[0].sum(-2))
        ev[2].record()
        ev[2].synchronize()
        assert pix.shape[-2:] == (codes.shape[1] * 32, codes.shape[2] * 32)
        return ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), launches

    names = list(CASES)
    for n in names:                                    # engine build, graph captures, warm-up of every shape
        step(n)
    t_ar = {n: [] for n in names}
    t_dec = {n: [] for n in names}
    launches = {}
    for i in range(args.calls):
        for n in (names if i % 2 == 0 else names[::-1]):
            a, d, launches[n] = step(n)
            t_ar[n].append(a)
            t_dec[n].append(d)
    info = card()
    for n in names:
        canvas, outpaint = CASES[n]
        sampled = [not (outpaint and idx % canvas[1] < canvas[1] // 2) for idx in range(canvas[0] * canvas[1])]
        segs = WO.segments((H, W), canvas, sampled)
        n_pos = sum(sampled)
        ar_ms, dec_ms = statistics.median(t_ar[n]), statistics.median(t_dec[n])
        print(json.dumps(dict(case=n, model="in1400m", B=B, canvas=list(canvas), weights="fp16", top_k=1024, calls=args.calls,
                              order="ABBA", sampled_positions=n_pos, prefills_per_call=len(segs), launches_per_call=launches[n],
                              ar_ms=round(ar_ms, 1), ms_per_sampled_position=round(ar_ms / n_pos, 2), decode_ms=round(dec_ms, 1),
                              images_per_s=round(B / ((ar_ms + dec_ms) / 1000), 2),
                              pixels=[canvas[0] * 32, canvas[1] * 32], **info)), flush=True)


if __name__ == "__main__":
    main()
