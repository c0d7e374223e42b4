#!/usr/bin/env python
"""bench_log_prob.py -- teacher-forced log-likelihoods of code maps: RQTransformer.log_prob(amp=True) against forward(amp=True)
followed by log_softmax and gather in torch.

    A   log_prob(amp=True): the forward's passes, the classifier in row chunks reduced in a bounded buffer (rqb200_ar_log_prob)
    B   forward(amp=True) -> [B,H,W,D,V] fp32 logits -> torch.log_softmax -> gather at the codes (and the cond logits likewise)

Cases: in1400m at B = 64 (fp16 and RQB200_FAST_DTYPE=fp8 weights), cc3m654m_16 at B = 16 (built as bench.py builds them) and the
`huge` 32x32x4 model of scripts/bench_shapes.py at B = 16.  Random codes (and cond tokens).  Per case, A and B alternate in ABBA order
for --calls rounds; CUDA events around each call.  Prints one JSON line per case with the card's name and power limit (read in this
run): median ms per call of each route and its peak allocated memory (torch.cuda.max_memory_allocated after a reset, minus what was
allocated before the call), and the largest |A - B| over the case.
Usage: python scripts/bench_log_prob.py [--calls 3] [--cases in1400m,in1400m_fp8,cc3m654m_16,huge]"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "rq-vae-transformer_b200")
for p in (ROOT, PKG, os.path.join(ROOT, "scripts")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

# case: (model, B, RQB200_FAST_DTYPE)
CASES = {"in1400m": ("in1400m", 64, "fp16"), "in1400m_fp8": ("in1400m", 64, "fp8"), "cc3m654m_16": ("cc3m654m_16", 16, "fp16"),
         "huge": ("huge", 16, "fp16")}


def build(model):
    if model == "huge":
        import bench_shapes
        ar, vae = bench_shapes.build("f8_huge_d4", "cuda")
        del vae
        vc, cl = bench_shapes.N_CLASSES, 1
    else:
        import bench
        ar, vae, _ = bench.build_models(model, "cuda", "fast")
        del vae
        vc, cl = bench.MODELS[model][6], bench.MODELS[model][7]
    torch.cuda.empty_cache()
    return ar, vc, cl


class Aux:
    class _Q:
        shared_codebook = True

        def __init__(self, t):
            self._t = t

        def _shared_table(self):
            return self._t

    def __init__(self, t):
        self.quantizer = Aux._Q(t)


def route_a(ar, aux, xs, cond):
    out = ar.log_prob(xs, model_aux=aux, cond=cond, amp=True)
    return out[0] if isinstance(out, tuple) else out


def route_b(ar, aux, xs, cond):
    out = ar(xs, model_aux=aux, cond=cond, amp=True)
    if isinstance(out, tuple):
        out, clg = out
        torch.log_softmax(clg, -1).gather(-1, cond[:, 1:, None])
    return torch.log_softmax(out, -1).gather(-1, xs[..., None]).squeeze(-1)


def timed(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    r = fn()
    e1.record()
    torch.cuda.synchronize()
    return r, e0.elapsed_time(e1), torch.cuda.max_memory_allocated() - base


def run_case(case, calls, ident):
    model, B, fmt = CASES[case]
    os.environ["RQB200_FAST_DTYPE"] = fmt
    ar, vc, cl = build(model)
    H, W, D = ar.block_size
    V = ar.vocab_size[0]
    g = torch.Generator(device="cuda").manual_seed(1)
    aux = Aux(torch.randn(V, 256, device="cuda", generator=g))
    xs = torch.randint(0, V, (B, H, W, D), device="cuda", generator=g)
    cond = torch.randint(0, vc, (B, cl), device="cuda", generator=g)
    routes = {"A": lambda: route_a(ar, aux, xs, cond), "B": lambda: route_b(ar, aux, xs, cond)}
    res = {k: routes[k]() for k in routes}                  # warm-up: engine build, graph-free first launches
    diff = float((res["A"] - res["B"]).abs().max())
    del res
    t, mem = {"A": [], "B": []}, {"A": 0, "B": 0}
    for _ in range(calls):
        for k in ("A", "B", "B", "A"):
            _, ms, peak = timed(routes[k])
            t[k].append(ms)
            mem[k] = max(mem[k], peak)
    a, b = statistics.median(t["A"]), statistics.median(t["B"])
    print(json.dumps(dict(ident, case=case, model=model, B=B, weights=fmt, log_prob_ms=round(a, 2), forward_log_softmax_ms=round(b, 2),
                          log_prob_over_forward=round(a / b, 3), log_prob_peak_mb=round(mem["A"] / 2**20, 1),
                          forward_peak_mb=round(mem["B"] / 2**20, 1), peak_reduction=round(mem["B"] / max(mem["A"], 1), 1),
                          max_abs_diff=diff, spread_ms={k: [round(min(v), 2), round(max(v), 2)] for k, v in t.items()})), flush=True)
    del ar
    os.environ.pop("RQB200_FAST_DTYPE", None)
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=3, help="ABBA rounds per case")
    ap.add_argument("--cases", default=",".join(CASES))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_log_prob.py: needs a CUDA device")
    torch.set_grad_enabled(False)
    from bench_shapes import gpu_identity
    ident = gpu_identity()
    for case in a.cases.split(","):
        run_case(case, a.calls, ident)


if __name__ == "__main__":
    main()
