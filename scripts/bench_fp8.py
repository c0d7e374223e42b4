#!/usr/bin/env python
"""bench_fp8.py -- the fp8 (E4M3) weight streamer against the fp16 one, at the AR step's GEMM shapes.

For each case it times, fp16 against fp8 in ABBA order, every weight GEMM of one body layer (qkv, proj, fc1, fc2).  The split
counts follow the rule of the engine's default (pick_split in csrc/ar_fast.cu: SMs / 128-row tiles, at least 1, at most K / 64),
restated here rather than read from an engine.  One launch per body layer, each on
that layer's own random weights (cold in L2, as in the step), captured in a CUDA graph and replayed; CUDA events on the
launching stream.  Per GEMM it reports:

    us         kernel time per launch (median over --calls ABBA rounds)
    gbps       algorithmic bytes (weights at their stored width -- fp8 adds the fp32 row scales -- + fp16 activations in +
               the fp32 split-K partials out) over that time

`cc3m654m_16` adds the teacher-forced forward's large-M shapes (M = B * (cond_len + H * W) rows): the persistent fp16 rows
GEMM, the fp16 streamer's and the fp8 streamer's row chunks.

The `sweep` leg separates per-launch cost from streaming cost: the in1400m fc2 shape (N_out 1536, B 64) at a fixed split of 11
with K = 704 * 2^i (1 .. 16 k blocks per split), enough layers for 160 MB of fp8 weights (cold in L2) per timing.  Per format
it prints every point and a least-squares fit us = fixed_us + bytes / rate over all points.

Prints one JSON line per (case, GEMM), sweep point and fit, with the card's name and power limit, read in this run.
Usage: python scripts/bench_fp8.py [--calls 3] [--reps 10]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "rq-vae-transformer_b200")
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from oracle.zoo import AR_ZOO  # noqa: E402
from rqvae import _native as N  # noqa: E402

CASES = [("in1400m", 64), ("t2i3900m", 16), ("cc3m654m_16", 16)]


def gpu_identity():
    out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit",
                          "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    name, power = [s.strip() for s in out.split(",")]
    return {"gpu": name, "power_limit": power}


def pick_split(n_tiles, nkb, n_sm):
    return max(1, min(n_sm // n_tiles, nkb))


def graph_ms(launch, reps):
    """ms per replay of a CUDA graph of `launch()`"""
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        launch()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            launch()
        for _ in range(3):
            g.replay()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            g.replay()
        e1.record()
        torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


class Layers:
    """n_layers distinct [N_out, K] weights as fp16 and as packed fp8 + scales"""

    def __init__(self, n_layers, N_out, K, seed):
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.w16, self.w8, self.s = [], [], []
        for _ in range(n_layers):
            w = torch.randn(N_out, K, device="cuda", generator=g) / K ** 0.5
            q, s = N.quantize_fp8_rows(w)
            self.w16.append(w.half())
            self.w8.append(N.pack_fp8_tiles(q))
            self.s.append(s)


def step_gemms(name, B, calls, reps, n_sm, ident):
    E, nh, nb = AR_ZOO[name][:3]
    L = N.lib()
    shapes = [("qkv", 3 * E, E), ("proj", E, E), ("fc1", 4 * E, E), ("fc2", E, 4 * E)]
    for gi, (gname, N_out, K) in enumerate(shapes):
        splits = pick_split(N_out // 128, K // 64, n_sm)
        lay = Layers(nb, N_out, K, 100 + gi)
        X = torch.randn(B, K, device="cuda").half()
        part = torch.empty(splits, B, N_out, device="cuda")

        def run16():
            for w in lay.w16:
                N.check(L.rqb200_dbg_gemm_tc(N.ptr(w), N.ptr(X), None, None, None, 0, 0, N.ptr(part), N_out, K, B, splits, 0,
                                             N.stream_ptr()), "dbg_gemm_tc")

        def run8():
            for w, s in zip(lay.w8, lay.s):
                N.check(L.rqb200_dbg_gemm_tc_fp8(N.ptr(w), N.ptr(s), N.ptr(X), None, None, None, 0, 0, N.ptr(part), N_out, K, B,
                                                 splits, N.stream_ptr()), "dbg_gemm_tc_fp8")

        t = {"fp16": [], "fp8": []}
        for _ in range(calls):
            for v in ("fp16", "fp8", "fp8", "fp16"):
                t[v].append(graph_ms(run16 if v == "fp16" else run8, reps) * 1e3 / nb)
        io = B * K * 2 + splits * B * N_out * 4
        b16, b8 = N_out * K * 2 + io, N_out * K + N_out * 4 + io
        us16, us8 = statistics.median(t["fp16"]), statistics.median(t["fp8"])
        print(json.dumps(dict(ident, case=name, leg="step", B=B, gemm=gname, N_out=N_out, K=K, splits=splits, ctas=N_out // 128 * splits,
                              fp16_us=round(us16, 2), fp8_us=round(us8, 2), fp16_gbps=round(b16 / us16 / 1e3, 1),
                              fp8_gbps=round(b8 / us8 / 1e3, 1), fp8_speedup=round(us16 / us8, 3),
                              spread_us={k: [round(min(v), 2), round(max(v), 2)] for k, v in t.items()})), flush=True)
        del lay


def forward_gemms(name, B, calls, reps, ident):
    E, nh, nb, nhl, V, bs, vc, cl = AR_ZOO[name]
    M = B * (cl + bs[0] * bs[1])
    Mp = -(-M // 128) * 128
    L = N.lib()
    n_layers = 4
    # (gemm, N_out, K, 16-bit output, gelu)
    for gi, (gname, N_out, K, o16, gelu) in enumerate([("qkv", 3 * E, E, 1, 0), ("proj", E, E, 0, 0), ("fc1", 4 * E, E, 1, 1),
                                                       ("fc2", E, 4 * E, 0, 0)]):
        lay = Layers(n_layers, N_out, K, 200 + gi)
        X = torch.zeros(Mp, K, device="cuda", dtype=torch.float16)
        X[:M] = torch.randn(M, K, device="cuda").half()
        bias = torch.randn(N_out, device="cuda")
        out = torch.empty(M, N_out, device="cuda", dtype=torch.float16 if o16 else torch.float32)

        def rows16():
            for w in lay.w16:
                N.check(L.rqb200_dbg_rows_gemm(N.ptr(X), N.ptr(w), N.ptr(bias), None, None if o16 else N.ptr(out),
                                               N.ptr(out) if o16 else None, gelu, 0, M, N_out, K, N.stream_ptr()), "dbg_rows_gemm")

        def stream16():
            for w in lay.w16:
                N.check(L.rqb200_dbg_gemm_tc(N.ptr(w), N.ptr(X), N.ptr(bias), None, N.ptr(out), o16, gelu, None, N_out, K, M, 1, 0,
                                             N.stream_ptr()), "dbg_gemm_tc")

        def stream8():
            for w, s in zip(lay.w8, lay.s):
                N.check(L.rqb200_dbg_gemm_tc_fp8(N.ptr(w), N.ptr(s), N.ptr(X), N.ptr(bias), None, N.ptr(out), o16, gelu, None, N_out,
                                                 K, M, 1, N.stream_ptr()), "dbg_gemm_tc_fp8")

        runs = {"rows_fp16": rows16, "stream_fp16": stream16, "stream_fp8": stream8}
        t = {k: [] for k in runs}
        for _ in range(calls):
            for v in ("rows_fp16", "stream_fp16", "stream_fp8", "stream_fp8", "stream_fp16", "rows_fp16"):
                t[v].append(graph_ms(runs[v], reps) * 1e3 / n_layers)
        flop = 2.0 * M * N_out * K
        med = {k: statistics.median(v) for k, v in t.items()}
        print(json.dumps(dict(ident, case=name, leg="forward", M=M, gemm=gname, N_out=N_out, K=K,
                              **{k + "_us": round(v, 2) for k, v in med.items()},
                              **{k + "_tflops": round(flop / v / 1e6, 1) for k, v in med.items()})), flush=True)
        del lay


def bytes_sweep(calls, reps, ident):
    L = N.lib()
    N_out, B, splits = 1536, 64, 11
    pts = {"fp16": [], "fp8": []}
    for i in range(5):
        K = 704 << i
        n = max(8, -(-(160 << 20) // (N_out * K)))
        lay = Layers(n, N_out, K, 300 + i)
        X = torch.randn(B, K, device="cuda").half()
        part = torch.empty(splits, B, N_out, device="cuda")

        def run16():
            for w in lay.w16:
                N.check(L.rqb200_dbg_gemm_tc(N.ptr(w), N.ptr(X), None, None, None, 0, 0, N.ptr(part), N_out, K, B, splits, 0,
                                             N.stream_ptr()), "dbg_gemm_tc")

        def run8():
            for w, s in zip(lay.w8, lay.s):
                N.check(L.rqb200_dbg_gemm_tc_fp8(N.ptr(w), N.ptr(s), N.ptr(X), None, None, None, 0, 0, N.ptr(part), N_out, K, B,
                                                 splits, N.stream_ptr()), "dbg_gemm_tc_fp8")

        t = {"fp16": [], "fp8": []}
        for _ in range(calls):
            for v in ("fp16", "fp8", "fp8", "fp16"):
                t[v].append(graph_ms(run16 if v == "fp16" else run8, reps) * 1e3 / n)
        wb = {"fp16": N_out * K * 2, "fp8": N_out * K + N_out * 4}
        for v in t:
            us = statistics.median(t[v])
            pts[v].append((wb[v], us))
            print(json.dumps(dict(ident, leg="sweep", fmt=v, N_out=N_out, K=K, B=B, splits=splits, layers=n, weight_bytes=wb[v],
                                  us=round(us, 2))), flush=True)
        del lay
    for v, p in pts.items():
        xs, ys = [x for x, _ in p], [y for _, y in p]
        mx, my = statistics.fmean(xs), statistics.fmean(ys)
        slope = sum((x - mx) * (y - my) for x, y in p) / sum((x - mx) ** 2 for x in xs)
        print(json.dumps(dict(ident, leg="sweep_fit", fmt=v, fixed_us=round(my - slope * mx, 2), rate_gbps=round(1e-3 / slope, 1),
                              max_residual_us=round(max(abs(y - (my + slope * (x - mx))) for x, y in p), 2))), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=3, help="ABBA rounds per GEMM")
    ap.add_argument("--reps", type=int, default=10, help="graph replays per timing")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8.py: needs a CUDA device")
    torch.set_grad_enabled(False)
    ident = gpu_identity()
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    for name, B in CASES:
        step_gemms(name, B, a.calls, a.reps, n_sm, ident)
        if name == "cc3m654m_16":
            forward_gemms(name, B, a.calls, a.reps, ident)
    bytes_sweep(a.calls, a.reps, ident)


if __name__ == "__main__":
    main()
