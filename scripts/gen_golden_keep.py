#!/usr/bin/env python
"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/keep.pt: masked-completion trajectories of the UNMODIFIED reference classes.

The reference has no keep mask, so this script drives its own per-token loop (transformers.py:294-369) with one change: after
sample_from_logits a kept token's code is overwritten with partial_sample's, xs[:, h, w, d] = where(keep, partial, drawn).  Sampling
runs under oracle/gen_golden.py's NoiseInjector (one seeded Exp(1) draw per image and token, kept or not).  The guided case runs two
reference instances with the same weights, one on cond and one on uncond, as scripts/gen_golden_cfg.py does.

    shapes    the zoo's tiny and tiny_txt
    cases     tests/keep_oracle.py's CASES: a box, depths >= 1, a seeded per-image random mask, all kept, a box with a start_loc
              resume, and (tiny) a box with guidance s = 1.5

Needs the reference tree (oracle/ref_loader.py):   python scripts/gen_golden_keep.py
Same protocol as oracle/gen_golden.py: weights, codebook, conditions, partial code maps and masks come from seeds; the file stores
the seeds, the case list and the reference's codes.
"""
import os
import sys
import time
from itertools import product

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import synth                                            # noqa: E402
from oracle import ref_loader as R                                  # noqa: E402
from oracle.gen_golden import NoiseInjector, build_ar               # noqa: E402
from oracle.zoo import AR_ZOO                                       # noqa: E402
from tests.keep_oracle import CASES, PLAN, mask_of, partial_of      # noqa: E402


def keep_sample(ns, mc, mu, partial, aux, cond, uncond, keep, s, top_k, top_p, start_loc):
    """the reference's sample() loop with the kept-token overwrite (and, s not None, the second branch of gen_golden_cfg.py)"""
    H, W, D = mc.block_size
    V = mc.vocab_size
    ks = [min(top_k, V[i]) for i in range(D)]
    ps = [min(top_p, 1.0) for _ in range(D)]
    xs = partial.clone()
    mc.init_cache()
    mu.init_cache()
    for (h, w, d) in product(range(H), range(W), range(D)):
        if (h, w) < (start_loc[0], start_loc[1]):
            continue
        lg = mc.cached_forward(xs[:, :h + 1], aux, cond=cond, sample_loc=(h, w, d))
        if s is not None:
            u = mu.cached_forward(xs[:, :h + 1], aux, cond=uncond, sample_loc=(h, w, d))
            lg = u + s * (lg - u)
        drawn = ns.sample_from_logits(lg, temperature=1.0, top_k=ks[d], top_p=ps[d])
        xs[:, h, w, d] = torch.where(keep[:, h, w, d], partial[:, h, w, d], drawn)
    mc.init_cache()
    mu.init_cache()
    return xs


def gen_shape(ns, name):
    P = PLAN
    mc, _ = build_ar(ns, name, seed=P["weight_seed"])
    mu, _ = build_ar(ns, name, seed=P["weight_seed"])
    E, nh, nb, nhl, V, bs, vc, cl = AR_ZOO[name]
    cb = synth.randn_seeded((V, 256), P["codebook_seed"])

    class Aux:          # the only thing sample() needs from the RQ-VAE (transformers.py:109-111)
        def get_code_emb_with_depth(self, code):
            parts = [torch.nn.functional.embedding(c, cb) for c in torch.chunk(code, code.shape[-1], dim=-1)]
            return torch.cat(parts, dim=-2), None

    B = P["B"]
    cond = synth.randint_seeded(0, vc, (B, cl), P["cond_seed"])
    uncond = synth.randint_seeded(0, vc, (B, cl), P["uncond_seed"])
    partial = partial_of(B, bs, V)
    runs = []
    for i, (spec, start, s) in enumerate(CASES[name]):
        keep = mask_of(spec, B, bs)
        with NoiseInjector(P["noise_seed"] + i):
            codes = keep_sample(ns, mc, mu, partial, Aux(), cond, uncond, keep, s, P["setting"]["top_k"], P["setting"]["top_p"], start)
        runs.append(dict(mask=spec, start_loc=start, scale=s, noise_seed=P["noise_seed"] + i, codes=codes.to(torch.int16)))
    return dict(runs=runs)


def main():
    torch.set_grad_enabled(False)
    ns = R.load_reference()
    res = {"plan": PLAN, "ar": {}}
    for name in CASES:
        t0 = time.time()
        res["ar"][name] = gen_shape(ns, name)
        print("  keep %-9s %.1fs" % (name, time.time() - t0), flush=True)
    torch.save(res, os.path.join(ROOT, "tests", "golden", "keep.pt"))


if __name__ == "__main__":
    main()
