#!/usr/bin/env python
"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/win.pt: sliding-window trajectories of the UNMODIFIED reference classes on canvases
larger than the model's grid (and on the grid itself).

The reference has no sliding window, so this script drives its own cached_forward (transformers.py:190-287) window by window: for every
canvas position (i, j) it calls init_cache(), then cached_forward on the window's codes at (i - r0, j - c0, d) for d = 0 .. D-1
(depth 0 prefills the window's prefix, depths > 0 continue on that cache as in the reference's own loop), and sample_from_logits under
oracle/gen_golden.py's NoiseInjector (one seeded Exp(1) draw per image and canvas token, kept or not).  The window origin and the cases
are tests/window_oracle.py's.  Outpainting overwrites a kept token with partial_sample's code, as scripts/gen_golden_keep.py does; the
guided case runs two reference instances with the same weights, one on cond and one on uncond, as scripts/gen_golden_cfg.py does.

Needs the reference tree (oracle/ref_loader.py):   python scripts/gen_golden_window.py
Same protocol as oracle/gen_golden.py: weights, codebook, conditions and partial code maps come from seeds; the file stores the seeds,
the case list and the reference's codes.
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
from tests.window_oracle import CASES, PLAN, mask_of, partial_of, window_of   # noqa: E402


def window_sample(ns, mc, mu, partial, aux, cond, uncond, keep, s, top_k, top_p, start_loc):
    """the window-by-window loop on the reference's cached_forward (and, s not None, the second branch of gen_golden_cfg.py)"""
    H, W, D = mc.block_size
    Ht, Wt = partial.shape[1:3]
    V = mc.vocab_size
    ks = [min(top_k, V[i]) for i in range(D)]
    ps = [min(top_p, 1.0) for _ in range(D)]
    xs = partial.clone()
    for (i, j) in product(range(Ht), range(Wt)):
        if (i, j) < tuple(start_loc):
            continue
        r0, c0, li, lj = window_of(i, j, (H, W), (Ht, Wt))
        mc.init_cache()
        mu.init_cache()
        for d in range(D):
            win = xs[:, r0:r0 + H, c0:c0 + W].contiguous()
            lg = mc.cached_forward(win[:, :li + 1], aux, cond=cond, sample_loc=(li, lj, d))
            if s is not None:
                u = mu.cached_forward(win[:, :li + 1], aux, cond=uncond, sample_loc=(li, lj, d))
                lg = u + s * (lg - u)
            drawn = ns.sample_from_logits(lg, temperature=1.0, top_k=ks[d], top_p=ps[d])
            xs[:, i, j, d] = drawn if keep is None else torch.where(keep[:, i, j, d], partial[:, i, j, d], drawn)
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

    B, D = P["B"], bs[2]
    cond = synth.randint_seeded(0, vc, (B, cl), P["cond_seed"])
    uncond = synth.randint_seeded(0, vc, (B, cl), P["uncond_seed"])
    runs = []
    for n, (canvas, spec, start, s) in enumerate(CASES[name]):
        partial = partial_of(B, canvas, D, V)
        keep = mask_of(spec, B, canvas, D)
        with NoiseInjector(P["noise_seed"] + n):
            codes = window_sample(ns, mc, mu, partial, Aux(), cond, uncond, keep, s, P["setting"]["top_k"], P["setting"]["top_p"], start)
        runs.append(dict(canvas=canvas, mask=spec, start_loc=start, scale=s, noise_seed=P["noise_seed"] + n, codes=codes.to(torch.int16)))
    return dict(runs=runs)


def main():
    torch.set_grad_enabled(False)
    ns = R.load_reference()
    res = {"plan": PLAN, "ar": {}}
    for name in CASES:
        t0 = time.time()
        res["ar"][name] = gen_shape(ns, name)
        print("  window %-9s %.1fs" % (name, time.time() - t0), flush=True)
    torch.save(res, os.path.join(ROOT, "tests", "golden", "win.pt"))


if __name__ == "__main__":
    main()
