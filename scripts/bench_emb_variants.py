#!/usr/bin/env python
"""RQ-Transformer embedding / classifier variants on the fast tier at the in1400m widths (E 1536, 42 + 6 layers, V 16384, 8x8x4,
B 64, synthetic weights): the shipped flags (all five switches true), the reference's all-false default (own token tables, per-depth
classifiers, no model_aux) and shared_cls_emb = false alone.  Prints one JSON line per variant with the card's name and power limit
(read in this run): images/s and AR ms per position of sample() (median of the timed calls, variants alternated in ABBA order), and
the classifier launch's device time in us (median over the launches of one traced sample, RQB200_TRACE: dependency resolved ->
done, in a separate run).

Every depth step streams one [V,E] classifier in each variant; a shared one may partly stay in L2 between the D depth steps.

    python scripts/bench_emb_variants.py [--calls 6]
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
from tests import variants_oracle as VO                      # noqa: E402
from tests.helpers import CodebookAux                        # noqa: E402
from tests.test_oracle_variants import make_variant          # noqa: E402

SHAPE = (1536, 24, 42, 6, 16384, (8, 8, 4), 1000, 1)
B = 64
SHIPPED = VO.COMBOS[-1]
VARIANTS = [("shipped", SHIPPED), ("all_false", VO.ALL_FALSE), ("per_depth_cls", dict(SHIPPED, shared_cls_emb=False))]


def card():
    out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit",
                          "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout.strip()
    name, power = [s.strip() for s in out.split(",")]
    return {"gpu": name, "power_limit": power}


def build(flags, base):
    """the variant's layout on the GPU; tensors it shares with the shipped layout are the shipped model's, the rest synthetic"""
    m = make_variant(SHAPE, flags, "meta")
    shapes = synth.shapes_of(m.state_dict())
    own = {k: s for k, s in shapes.items() if k not in base or tuple(base[k].shape) != tuple(s)}
    sd = {k: base[k] for k in shapes if k not in own}
    sd.update({k: v.to("cuda") for k, v in VO.state_dict_of(own, 7).items()})
    m = m.to_empty(device="cuda")
    m.load_state_dict(sd)
    m = m.eval()
    m.precision = "fast"
    return m


def time_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=6)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_emb_variants: needs a CUDA device")
    torch.set_grad_enabled(False)
    info = card()
    with torch.device("meta"):
        shipped = make_variant(SHAPE, SHIPPED, "meta")
    base = {k: v.to("cuda") for k, v in synth.synth_state_dict(synth.shapes_of(shipped.state_dict()), 5).items()}
    models = {name: build(flags, base) for name, flags in VARIANTS}
    aux = CodebookAux(synth.randn_seeded((SHAPE[4], 256), 6).to("cuda"))
    cond = synth.randint_seeded(0, SHAPE[6], (B, 1), 8).to("cuda")
    z = torch.zeros(B, *SHAPE[5], dtype=torch.long, device="cuda")

    def run(name):
        flags = dict(VARIANTS)[name]
        return lambda: models[name].sample(z, model_aux=aux if VO.needs_codebook(flags) else None, cond=cond, top_k=1024, amp=True)

    names = [n for n, _ in VARIANTS]
    for n in names:
        run(n)()
    times = {n: [] for n in names}
    for i in range(args.calls):
        for n in (names if i % 2 == 0 else names[::-1]):
            times[n].append(time_ms(run(n)))
    cls_us = {}
    os.environ["RQB200_TRACE"] = "1"
    for n in names:
        models[n]._invalidate_native()
        run(n)()
        rows = [r for r in models[n].native_trace() if r[0] == "cls"]
        cls_us[n] = statistics.median((r[4] - r[2]) / 1e3 for r in rows) if rows else None
        models[n]._invalidate_native()
    del os.environ["RQB200_TRACE"]
    n_pos = SHAPE[5][0] * SHAPE[5][1]
    for n in names:
        t = statistics.median(times[n])
        print(json.dumps(dict(variant=n, B=B, E=SHAPE[0], layers=[SHAPE[2], SHAPE[3]], V=SHAPE[4], calls=args.calls,
                              images_per_s=round(B / t * 1e3, 2), ar_ms_per_position=round(t / n_pos, 4),
                              cls_launch_us=None if cls_us[n] is None else round(cls_us[n], 2), **info)), flush=True)


if __name__ == "__main__":
    main()
