#!/usr/bin/env python
"""fp16 against FP8 (E4M3) weights on the fast AR tier, end to end: in1400m B 64, t2i3900m B 16 and cc3m654m_16 B 16, the models
built as bench.py builds them (default init under torch.manual_seed(0), the RQ-VAE of the same config).  Both variants share one
set of parameters: one RQTransformer builds its engine with RQB200_FAST_DTYPE=fp16, a twin on the same tensors with fp8.

Per variant, calls alternated in ABBA order (median over --calls): images/s of sample + decode, AR ms per spatial position,
forward(amp=True) ms (cc3m654m_16 only), and the engine's streamed weight bytes.  In a separate traced run (RQB200_TRACE), per
position (one body-step replay + one head-step replay): the GEMM launches' device us (dependency resolved -> done, summed), the
traced step's us, and the GEMM share of it.  One JSON line per case with the card's name and power limit read in this run.

    python scripts/bench_fp8_sample.py [--calls 4] [--cases in1400m,t2i3900m,cc3m654m_16]
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

CASES = {"in1400m": 64, "t2i3900m": 16, "cc3m654m_16": 16}
GEMMS = ("qkv", "proj", "fc1", "fc2", "w_in", "w_head", "cls")
SLOTS_PER_GRAPH = 1024                   # ar_fast.cu: TR_CAP / G_COUNT trace slots per captured graph (0 cond, 1 body, 2-3 head)


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


def with_dtype(dt, fn):
    os.environ["RQB200_FAST_DTYPE"] = dt
    try:
        return fn()
    finally:
        del os.environ["RQB200_FAST_DTYPE"]


def trace_stats(model):
    """GEMM us and step us of one position from the last replays of the body-step and head-step graphs"""
    rows = model.native_trace()
    gemm_us, step_us = 0.0, 0.0
    for graph in (1, 2, 3):
        rs = [r for r in rows if r[5] // SLOTS_PER_GRAPH == graph]
        if not rs:
            continue
        gemm_us += sum((r[4] - r[2]) / 1e3 for r in rs if r[0] in GEMMS)
        step_us += (max(r[4] for r in rs) - min(r[1] for r in rs)) / 1e3
    return gemm_us, step_us


def run_case(name, B, calls, info):
    E, nh, nb, nhl, V, bs, vc, cl, attn, ch_mult, top_p = bench.MODELS[name][:11]
    ar, vae, _ = bench.build_models(name, "cuda", "fast")
    with torch.device("meta"):
        ar8 = type(ar)(ar.config)
    ar8.load_state_dict(ar.state_dict(), assign=True)             # the same parameter tensors
    ar8 = ar8.eval()
    ar8.precision = "fast"
    models = {"fp16": ar, "fp8": ar8}
    g = torch.Generator().manual_seed(11)
    cond = torch.randint(0, max(vc, 1), (B, cl), generator=g).to("cuda")
    z = torch.zeros(B, *bs, dtype=torch.long, device="cuda")
    kw = dict(top_k=min(1024, V), top_p=top_p, amp=True)
    n_pos = bs[0] * bs[1]

    def step(v):
        a, b, c = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        a.record()
        codes = models[v].sample(z, model_aux=vae, cond=cond, **kw)
        b.record()
        vae.decode_code(codes)
        c.record()
        c.synchronize()
        return a.elapsed_time(c), a.elapsed_time(b), codes

    def fwd(v, codes):
        return time_ms(lambda: models[v](codes, model_aux=vae, cond=cond, amp=True))

    names = ["fp16", "fp8"]
    codes = {v: with_dtype(v, lambda: step(v))[2] for v in names}      # engine builds + warm-up (graphs captured)
    do_fwd = name == "cc3m654m_16"
    if do_fwd:
        for v in names:
            fwd(v, codes[v])
    res = {v: {"total": [], "ar": [], "fwd": []} for v in names}
    for i in range(calls):
        for v in (names if i % 2 == 0 else names[::-1]):
            t, a, _ = step(v)
            res[v]["total"].append(t)
            res[v]["ar"].append(a)
            if do_fwd:
                res[v]["fwd"].append(fwd(v, codes[v]))
    wbytes = {v: models[v].native_weight_bytes()["streamed"] for v in names}
    os.environ["RQB200_TRACE"] = "1"
    tr = {}
    for v in names:
        models[v]._invalidate_native()
        with_dtype(v, lambda: models[v].sample(z, model_aux=vae, cond=cond, **kw))
        torch.cuda.synchronize()
        tr[v] = trace_stats(models[v])
        models[v]._invalidate_native()
    del os.environ["RQB200_TRACE"]
    out = {}
    for v in names:
        t, a = statistics.median(res[v]["total"]), statistics.median(res[v]["ar"])
        gemm_us, step_us = tr[v]
        out[v] = dict(images_per_s=round(B / t * 1e3, 2), ar_ms_per_position=round(a / n_pos, 4),
                      forward_ms=round(statistics.median(res[v]["fwd"]), 2) if do_fwd else None,
                      streamed_weight_gb=round(wbytes[v] / 1e9, 3), traced_gemm_us_per_position=round(gemm_us, 1),
                      traced_step_us_per_position=round(step_us, 1), gemm_share=round(gemm_us / step_us, 3) if step_us else None)
    print(json.dumps(dict(case=name, B=B, calls=calls, order="ABBA", **out, **info)), flush=True)
    del ar, ar8, vae, models
    gc.collect()
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=4)
    ap.add_argument("--cases", default=",".join(CASES))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8_sample: needs a CUDA device")
    torch.set_grad_enabled(False)
    info = card()
    for name in args.cases.split(","):
        run_case(name, CASES[name], args.calls, info)


if __name__ == "__main__":
    main()
