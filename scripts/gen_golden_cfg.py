#!/usr/bin/env python
"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/cfg.pt: classifier-free guided trajectories of the UNMODIFIED reference classes.

The reference has no guidance, so this script drives its own per-token loop (transformers.py:294-369) for two branches: two
reference RQTransformer instances with the same weights, one conditioned on `cond`, one on `uncond`, each keeping its own
cached_forward cache.  Per token (h, w, d) it takes both branches' logits c and u, forms l = u + s * (c - u) in fp32 torch, samples
with the reference's sample_from_logits under oracle/gen_golden.py's NoiseInjector (one seeded Exp(1) draw per image and token), and
writes the code into the one code map both branches read.

    shapes    the zoo's tiny (class-conditional, uncond = other seeded classes) and tiny_txt (text-shaped, uncond = the all-zero
              caption)
    runs      s in {0, 1.5, 4} x {top-k, top-(k, p)}; the guided logits of one run (s = 1.5, top-k) are kept at a few steps
    resume    one start_loc resume from the first run's codes

Needs the reference tree (oracle/ref_loader.py):   python scripts/gen_golden_cfg.py
Same protocol as oracle/gen_golden.py: weights, codebook and conditions come from oracle/synth.py seeds; the file stores seeds and
the reference's outputs.
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

PLAN = dict(B=2, weight_seed=11, codebook_seed=12, cond_seed=13, uncond_seed=14, scales=[0.0, 1.5, 4.0],
            settings=[dict(top_k=64), dict(top_k=64, top_p=0.9)], noise_seed=600, keep_steps=[0, 1, 5, 35], logits_run=2,
            resume=dict(scale=1.5, setting=1, noise_seed=601))
SHAPES = ["tiny", "tiny_txt"]


def uncond_of(name, B=PLAN["B"]):
    """tiny: other seeded classes; tiny_txt: the all-zero caption"""
    vc, cl = AR_ZOO[name][6], AR_ZOO[name][7]
    if name == "tiny":
        return synth.randint_seeded(0, vc, (B, cl), PLAN["uncond_seed"])
    return torch.zeros(B, cl, dtype=torch.long)


def guided_sample(ns, mc, mu, partial, aux, cond, uncond, s, top_k, top_p, start_loc=(0, 0), keep=()):
    """the reference's sample() loop with two branches; returns (codes, {step: guided logits})"""
    H, W, D = mc.block_size
    V = mc.vocab_size
    ks = [min(top_k, V[i]) for i in range(D)]
    ps = [1.0 if top_p is None else min(top_p, 1.0) for _ in range(D)]
    xs = partial.clone()
    mc.init_cache()
    mu.init_cache()
    kept, step = {}, 0
    for (h, w, d) in product(range(H), range(W), range(D)):
        if (h, w) < (start_loc[0], start_loc[1]):
            continue
        c = mc.cached_forward(xs[:, :h + 1], aux, cond=cond, sample_loc=(h, w, d))
        u = mu.cached_forward(xs[:, :h + 1], aux, cond=uncond, sample_loc=(h, w, d))
        lg = u + s * (c - u)
        if step in keep:
            kept[step] = lg.clone()
        xs[:, h, w, d] = ns.sample_from_logits(lg, temperature=1.0, top_k=ks[d], top_p=ps[d])
        step += 1
    mc.init_cache()
    mu.init_cache()
    return xs, kept


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

    cond = synth.randint_seeded(0, vc, (P["B"], cl), P["cond_seed"])
    uncond = uncond_of(name)
    zeros = torch.zeros(P["B"], *bs, dtype=torch.long)
    runs = []
    for i, (s, st) in enumerate(product(P["scales"], range(len(P["settings"])))):
        setting = P["settings"][st]
        with NoiseInjector(P["noise_seed"]):
            codes, kept = guided_sample(ns, mc, mu, zeros, Aux(), cond, uncond, s, setting["top_k"], setting.get("top_p"),
                                        keep=P["keep_steps"] if i == P["logits_run"] else ())
        runs.append(dict(scale=s, setting=setting, codes=codes.to(torch.int16), logits=kept or None))
    rs = P["resume"]
    h0, w0 = bs[0] // 2, 1
    setting = P["settings"][rs["setting"]]
    with NoiseInjector(rs["noise_seed"]):
        codes2, _ = guided_sample(ns, mc, mu, runs[0]["codes"].long(), Aux(), cond, uncond, rs["scale"], setting["top_k"],
                                  setting.get("top_p"), start_loc=(h0, w0))
    return dict(runs=runs, resume=dict(start_loc=(h0, w0), scale=rs["scale"], setting=setting, noise_seed=rs["noise_seed"],
                                       codes=codes2.to(torch.int16)))


def main():
    torch.set_grad_enabled(False)
    ns = R.load_reference()
    res = {"plan": PLAN, "ar": {}}
    for name in SHAPES:
        t0 = time.time()
        res["ar"][name] = gen_shape(ns, name)
        print("  cfg %-9s %.1fs" % (name, time.time() - t0), flush=True)
    torch.save(res, os.path.join(ROOT, "tests", "golden", "cfg.pt"))


if __name__ == "__main__":
    main()
