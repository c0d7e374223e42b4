"""Masked completion (RQTransformer.sample(keep_mask=...)) in plain torch: the reference's per-token loop
(transformers.py:294-369) on oracle/rq_oracle.py's cached forward, with one change -- after sample_from_logits a kept token's code is
overwritten with partial_sample's.  Every token still takes its noise draw.  Also the keep masks of tests/golden/keep.pt
(scripts/gen_golden_keep.py), rebuilt from their specs: the fixture stores seeds and codes only."""
from itertools import product

import torch

from oracle import rq_oracle as O
from oracle import synth

# the cases of keep.pt: (mask spec, start_loc, guidance scale or None); shape names of oracle/zoo.py
PLAN = dict(B=2, weight_seed=11, codebook_seed=12, cond_seed=13, uncond_seed=14, partial_seed=21, mask_seed=22, noise_seed=700,
            setting=dict(top_k=64, top_p=0.9))
CASES = {
    "tiny": [("box", (0, 0), None), ("depth", (0, 0), None), ("random", (0, 0), None), ("all", (0, 0), None),
             ("box", (1, 2), None), ("box", (0, 0), 1.5)],
    "tiny_txt": [("box", (0, 0), None), ("depth", (0, 0), None), ("random", (0, 0), None), ("all", (0, 0), None),
                 ("box", (1, 2), None)],
}


def mask_of(spec, B, bs, seed=PLAN["mask_seed"]):
    """bool [B, H, W, D], True = keep.  box: resample positions [1, 3) x [1, 3) at every depth; depth: keep depth 0, resample the
    others; random: a seeded per-image, per-token mask; all: keep everything"""
    H, W, D = bs
    if spec == "box":
        k = torch.ones(B, H, W, D, dtype=torch.bool)
        k[:, 1:3, 1:3, :] = False
    elif spec == "depth":
        k = torch.zeros(B, H, W, D, dtype=torch.bool)
        k[..., 0] = True
    elif spec == "random":
        k = synth.randn_seeded((B, H, W, D), seed) > 0.3
    elif spec == "all":
        k = torch.ones(B, H, W, D, dtype=torch.bool)
    else:
        raise ValueError(spec)
    return k


def partial_of(B, bs, V, seed=PLAN["partial_seed"]):
    return synth.randint_seeded(0, V, (B, *bs), seed)


def ar_sample_keep(sd, cfg, partial_sample, codebook, keep, cond=None, start_loc=(0, 0), top_k=None, top_p=None, noise=None,
                   scale=None, uncond=None):
    """rq_oracle.ar_sample with the kept-token overwrite; noise(step, B, V) -> q.  scale / uncond: classifier-free guidance, the
    guided logits l = u + s (c - u) from a second cached state conditioned on uncond"""
    H, W, D = cfg.block_size
    ks = O._per_depth(top_k, cfg.V, D, cfg.V)
    ps = O._per_depth(top_p, 1.0, D, 1.0)
    xs = partial_sample.clone()
    sc, su = O.new_state(cfg), O.new_state(cfg)
    step = 0
    for (h, w, d) in product(range(H), range(W), range(D)):
        if (h, w) < (start_loc[0], start_loc[1]):
            continue
        lg = O.ar_cached_forward(sd, cfg, sc, xs[:, :h + 1], codebook, cond, (h, w, d))
        if scale is not None:
            u = O.ar_cached_forward(sd, cfg, su, xs[:, :h + 1], codebook, uncond, (h, w, d))
            lg = u + scale * (lg - u)
        drawn = O.sample_from_logits(lg, 1.0, ks[d], ps[d], q=noise(step, lg.shape[0], lg.shape[1]))
        xs[:, h, w, d] = torch.where(keep[:, h, w, d], partial_sample[:, h, w, d], drawn)
        step += 1
    return xs
