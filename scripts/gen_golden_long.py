#!/usr/bin/env python
"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/ar4.pt from the UNMODIFIED reference classes: the long-sequence AR shapes.

    long32       32x32x4 codes behind a 32-token prefix (body T = 1056: the f=8 RQ-VAE's latent grid)
    headless16   16x16x1 codes, no head layers (measure_throughput's d = 1 runs)

Needs the reference tree (oracle/ref_loader.py):   python scripts/gen_golden_long.py
Same protocol as the AR fixtures of oracle/gen_golden.py: the file stores seeds / configs and the reference's outputs (a greedy
and a seeded top-k trajectory per shape with the logits of their first and last steps, and a start_loc resume); weights,
codebook, cond tokens and the per-token Exp(1) noise are regenerated from oracle/synth.py seeds.  The key / shape list of the
weights comes from the model itself, so these shapes stay out of oracle/zoo.py and state_dict_layouts.json.
"""
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_loader as R                                  # noqa: E402
from oracle import synth                                            # noqa: E402
from oracle.gen_golden import NoiseInjector, check_multinomial_identity   # noqa: E402

# (E, heads, n_body, n_head_layers, V, block_size, vocab_cond, cond_len), as in oracle/zoo.py's AR_ZOO
AR4_ZOO = {
    "long32": (128, 2, 1, 1, 512, (32, 32, 4), 64, 32),
    "headless16": (128, 2, 1, 0, 512, (16, 16, 1), 10, 1),
}
# name, B, settings, logits steps to keep
PLAN = [
    ("long32", 2, [dict(top_k=1), dict(top_k=100)], [0, 32 * 32 * 4 - 1]),
    ("headless16", 2, [dict(top_k=1), dict(top_k=100)], [0, 16 * 16 - 1]),
]


def gen_ar4(ns):
    res = {}
    for name, B, settings, keep in PLAN:
        t0 = time.time()
        E, nh, nb, nhl, V, bs, vc, cl = AR4_ZOO[name]
        model = ns.RQTransformer(R.transformer_cfg(E, nh, nb, nhl, V, block_size=bs, vocab_cond=vc, cond_len=cl)).eval()
        model.load_state_dict(synth.synth_state_dict(synth.shapes_of(model.state_dict()), 11))
        cb = synth.randn_seeded((V, 256), 12)

        class Aux:          # the only thing sample() needs from the RQ-VAE (transformers.py:109-111)
            def get_code_emb_with_depth(self, code):
                parts = [torch.nn.functional.embedding(c, cb) for c in torch.chunk(code, code.shape[-1], dim=-1)]
                return torch.cat(parts, dim=-2), None

        cond = synth.randint_seeded(0, max(vc, 1), (B, cl), 13) if vc > 1 else None
        runs = []
        for si, st in enumerate(settings):
            kept = {}
            orig_cf = model.cached_forward
            counter = [0]

            def spy(*a, **kw):
                lg = orig_cf(*a, **kw)
                if counter[0] in keep:
                    kept[counter[0]] = lg.clone()
                counter[0] += 1
                return lg

            model.cached_forward = spy
            with NoiseInjector(500 + si):
                codes = model.sample(torch.zeros(B, *bs, dtype=torch.long), model_aux=Aux(), cond=cond, **st)
            model.cached_forward = orig_cf
            runs.append(dict(setting=st, noise_seed=500 + si, codes=codes.to(torch.int32), logits=dict(kept)))
        # start_loc resume (image completion): keep the first rows of run 0, resample from (h0, w0)
        h0, w0 = bs[0] // 2, 1
        with NoiseInjector(900):
            codes2 = model.sample(runs[0]["codes"].long().clone(), model_aux=Aux(), cond=cond, start_loc=(h0, w0),
                                  top_k=settings[-1].get("top_k"))
        res[name] = dict(B=B, weight_seed=11, codebook_seed=12, cond_seed=13, runs=runs,
                         resume=dict(start_loc=(h0, w0), noise_seed=900, codes=codes2.to(torch.int32), top_k=settings[-1].get("top_k")))
        print("  ar %-10s %.1fs" % (name, time.time() - t0), flush=True)
    return {"shapes": dict(AR4_ZOO), "ar": res}


def main():
    torch.set_grad_enabled(False)
    ns = R.load_reference()
    check_multinomial_identity()
    torch.save(gen_ar4(ns), os.path.join(ROOT, "tests", "golden", "ar4.pt"))


if __name__ == "__main__":
    main()
