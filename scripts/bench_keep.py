#!/usr/bin/env python
"""Masked completion (`sample(keep_mask=...)`) on the fast AR tier, end to end: in1400m B = 64 (fp16, and one FP8 line) and the
32x32x4 `f8_huge_d4` shape of bench_cached_forward.py at B = 16, models built as those scripts build them, top-k 1024 and the
config's top-p, partial_sample a seeded random code map.

Masks (True = keep):
    box       resample the centre box (4x4 of 8x8, 16x16 of 32x32)
    right     resample the right half
    quadrant  resample the bottom-right quadrant
    depth     keep depth 0, resample depths 1..D-1 (no position is skipped: the worst case)
    none      keep nothing (must cost what unmasked sampling costs)
and, with --sweep (in1400m fp16), runs_k: sample every depth at positions 0, k, 2k, ... only, so every append is a run of exactly k
kept positions -- the batched append against token-by-token appends at each k fixes the threshold in csrc/ar_fast.cu.

Two phases per case, each in ABBA order over [unmasked, mask...] (median over --calls): the shipped engine (batched appends) and
RQB200_SEQ_PREFILL=1 (every append token by token).  Per run: AR ms per call, launches per call, sampled positions; the masked /
unmasked ratio beside it.  --forward: forward(amp=True) ms at in1400m B = 64 only (run it in two trees to compare their attention
kernels).  One JSON line per case with the card's name and power limit read in this run.

    python scripts/bench_keep.py [--calls 4] [--cases in1400m,in1400m_fp8,f8_huge_d4] [--sweep] [--forward]
"""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "rq-vae-transformer_b200"), os.path.join(ROOT, "scripts")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

# case: (model, B, RQB200_FAST_DTYPE)
CASES = {"in1400m": ("in1400m", 64, "fp16"), "in1400m_fp8": ("in1400m", 64, "fp8"), "f8_huge_d4": ("f8_huge_d4", 16, "fp16")}
SWEEP_K = (2, 3, 4, 5, 6, 8, 16)


def card():
    out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit",
                          "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout.strip()
    name, power = [s.strip() for s in out.split(",")]
    return {"gpu": name, "power_limit": power}


def build(model):
    if model == "in1400m":
        import bench
        ar, vae, _ = bench.build_models("in1400m", "cuda", "fast")
        return ar, vae, bench.MODELS["in1400m"][10]
    import bench_shapes
    ar, vae = bench_shapes.build(model, "cuda")
    return ar, vae, None


def masks(bs, sweep):
    H, W, D = bs
    out = {}
    k = torch.ones(H, W, 1, dtype=torch.bool)
    k[H // 4:H - H // 4, W // 4:W - W // 4] = False
    out["box"] = k
    k = torch.ones(H, W, 1, dtype=torch.bool)
    k[:, W // 2:] = False
    out["right"] = k
    k = torch.ones(H, W, 1, dtype=torch.bool)
    k[H // 2:, W // 2:] = False
    out["quadrant"] = k
    k = torch.zeros(1, 1, 1, D, dtype=torch.bool)
    k[..., 0] = True
    out["depth"] = k
    out["none"] = torch.zeros(1, 1, 1, 1, dtype=torch.bool)
    for n in (SWEEP_K if sweep else ()):
        k = torch.ones(H * W, 1, dtype=torch.bool)
        k[::n] = False
        out["runs_%d" % n] = k.view(H, W, 1)
    return {name: m.to("cuda") for name, m in out.items()}


def with_env(ar, env, fn):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    ar._invalidate_native()
    try:
        return fn()
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
        ar._invalidate_native()


def phase(ar, vae, partial, cond, top_p, ms, calls):
    """{run: (median AR ms, launches)} over unmasked and every mask, ABBA"""
    kw = dict(model_aux=vae, cond=cond, top_k=1024, top_p=top_p, amp=True)
    runs = ["unmasked"] + list(ms)

    def step(r):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        ar.sample(partial, keep_mask=None if r == "unmasked" else ms[r], **kw)
        b.record()
        b.synchronize()
        return a.elapsed_time(b), ar.last_launches

    for r in runs:                                          # engine builds, graph captures, warm-up
        step(r)
    t = {r: [] for r in runs}
    launches = {}
    for i in range(calls):
        for r in (runs if i % 2 == 0 else runs[::-1]):
            ms_, launches[r] = step(r)
            t[r].append(ms_)
    return {r: (statistics.median(t[r]), launches[r]) for r in runs}


def run_case(case, calls, sweep, info):
    model, B, fmt = CASES[case]
    ar, vae, top_p = build(model)
    H, W, D = ar.block_size
    V = ar.vocab_size[0]
    g = torch.Generator().manual_seed(11)
    cond = torch.randint(0, ar.vocab_size_cond, (B, ar.block_size_cond), generator=g).to("cuda")
    partial = torch.randint(0, V, (B, H, W, D), generator=g).to("cuda")
    ms = masks((H, W, D), sweep)
    env = {"RQB200_FAST_DTYPE": fmt}
    fast = with_env(ar, env, lambda: phase(ar, vae, partial, cond, top_p, ms, calls))
    seq = with_env(ar, dict(env, RQB200_SEQ_PREFILL="1"), lambda: phase(ar, vae, partial, cond, top_p, ms, calls))
    rows = {}
    for name, m in [("unmasked", None)] + list(ms.items()):
        sampled = H * W if m is None else int((~m.expand(B, H, W, D)).reshape(B, H * W, D).any(2).any(0).sum())
        rows[name] = dict(sampled_positions=sampled, ar_ms=round(fast[name][0], 2), launches_per_call=fast[name][1],
                          vs_unmasked=round(fast[name][0] / fast["unmasked"][0], 3), seq_append_ar_ms=round(seq[name][0], 2),
                          seq_append_launches=seq[name][1], seq_vs_unmasked=round(seq[name][0] / seq["unmasked"][0], 3))
    print(json.dumps(dict(case=case, B=B, shape=[H, W, D], weights=fmt, calls=calls, order="ABBA", runs=rows, **info)), flush=True)
    del ar, vae
    gc.collect()
    torch.cuda.empty_cache()


def forward_ms(calls, info):
    """forward(amp=True) at in1400m B = 64: the batched passes' prefill attention kernel at T0 = 0"""
    ar, vae, _ = build("in1400m")
    B = 64
    H, W, D = ar.block_size
    g = torch.Generator().manual_seed(12)
    codes = torch.randint(0, ar.vocab_size[0], (B, H, W, D), generator=g).to("cuda")
    cond = torch.randint(0, ar.vocab_size_cond, (B, 1), generator=g).to("cuda")
    for _ in range(2):
        ar.forward(codes, model_aux=vae, cond=cond, amp=True)
    t = []
    for _ in range(calls):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        ar.forward(codes, model_aux=vae, cond=cond, amp=True)
        b.record()
        b.synchronize()
        t.append(a.elapsed_time(b))
    print(json.dumps(dict(case="forward_in1400m", B=B, calls=calls, forward_ms=round(statistics.median(t), 3),
                          tree=os.path.basename(ROOT), **info)), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=4)
    ap.add_argument("--cases", default=",".join(CASES))
    ap.add_argument("--sweep", action="store_true")
    ap.add_argument("--forward", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_keep: needs a CUDA device")
    torch.set_grad_enabled(False)
    info = card()
    if args.forward:
        forward_ms(max(args.calls, 10), info)
        return
    for case in args.cases.split(","):
        run_case(case, args.calls, args.sweep and case == "in1400m", info)


if __name__ == "__main__":
    main()
