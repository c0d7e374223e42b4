"""Sliding-window sampling (RQTransformer.sample on a canvas larger than the model's grid) in plain torch, and the cases of
tests/golden/win.pt (scripts/gen_golden_window.py): the fixture stores seeds, the case list and codes only.

The rule (Taming Transformers' sliding window, kept in bounds at odd sizes): the canvas token (i, j, d) of an Ht x Wt canvas is sampled as
the model's token (i - r0, j - c0, d) of the H x W window with origin

    r0 = clamp(i - H // 2, 0, Ht - H),   c0 = clamp(j - W // 2, 0, Wt - W),

seeing exactly what the reference's cached_forward sees for the window's codes at (i - r0, j - c0, d): the cond prefix, the window's
positions before it in window raster order and its own depths < d, read from the canvas as it stands.  Canvas tokens are sampled in
canvas raster order with one Exp(1) draw each (kept or not, none before start_loc), as sample() does on the grid.

The engine walks the canvas in segments: consecutive sampled positions whose windows share an origin continue one KV cache; a new
origin starts a new segment with a prefill of the window's prefix."""
from itertools import product

import torch

from oracle import rq_oracle as O
from oracle import synth

PLAN = dict(B=2, weight_seed=11, codebook_seed=12, cond_seed=13, uncond_seed=14, partial_seed=31, noise_seed=900,
            setting=dict(top_k=64, top_p=0.9))
# per zoo shape: (canvas (Ht, Wt), mask spec, start_loc, guidance scale or None).  "plain" samples every token, "outpaint" keeps the left
# half of the canvas (an encoded image extended to the right); the canvas == grid cases are sample() itself.
CASES = {
    "tiny": [((4, 8), "plain", (0, 0), None), ((8, 4), "plain", (0, 0), None), ((7, 9), "plain", (0, 0), None),
             ((10, 10), "plain", (0, 0), None), ((4, 8), "outpaint", (0, 0), None), ((7, 9), "plain", (2, 3), None),
             ((4, 8), "plain", (0, 0), 1.5), ((4, 4), "plain", (0, 0), None), ((4, 4), "outpaint", (0, 0), None)],
    "tiny_txt": [((5, 7), "plain", (0, 0), None), ((5, 7), "outpaint", (0, 0), None), ((3, 3), "plain", (0, 0), None)],
}


def origin(i, n, nt):
    """the window origin along one axis: n cells with floor(n/2) of them before coordinate i, clamped to [0, nt - n]"""
    return min(max(i - n // 2, 0), nt - n)


def taming_origin(i, n, nt):
    """Taming Transformers' three-branch rule (sample_conditional / make_video, even n): the reference for origin() at even sizes"""
    if i <= n // 2:
        return 0
    if nt - i < n // 2:
        return nt - n
    return i - n // 2


def window_of(i, j, grid, canvas):
    """canvas position (i, j) -> (r0, c0, li, lj): its window's origin and its position inside the window"""
    H, W = grid
    Ht, Wt = canvas
    r0, c0 = origin(i, H, Ht), origin(j, W, Wt)
    return r0, c0, i - r0, j - c0


def segments(grid, canvas, sampled=None, start=0):
    """the engine's segment plan: [(origin (r0, c0), [canvas positions])] over the canvas positions >= start that are sampled
    (sampled: a bool sequence over the Ht * Wt positions, None: all)"""
    Ht, Wt = canvas
    out = []
    for idx in range(start, Ht * Wt):
        if sampled is not None and not sampled[idx]:
            continue
        r0, c0, _, _ = window_of(idx // Wt, idx % Wt, grid, canvas)
        if out and out[-1][0] == (r0, c0):
            out[-1][1].append(idx)
        else:
            out.append(((r0, c0), [idx]))
    return out


def mask_of(spec, B, canvas, D):
    """bool [B, Ht, Wt, D] (True = keep) or None: outpaint keeps the left floor(Wt / 2) columns"""
    if spec == "plain":
        return None
    if spec == "outpaint":
        k = torch.zeros(B, *canvas, D, dtype=torch.bool)
        k[:, :, :canvas[1] // 2] = True
        return k
    raise ValueError(spec)


def partial_of(B, canvas, D, V, seed=PLAN["partial_seed"]):
    return synth.randint_seeded(0, V, (B, *canvas, D), seed)


def window_sample(sd, cfg, partial_sample, codebook, keep=None, cond=None, start_loc=(0, 0), top_k=None, top_p=None, noise=None,
                  scale=None, uncond=None, logits_hook=None):
    """the sliding-window loop on oracle/rq_oracle.py's cached forward: a fresh cache per canvas position, the window's codes as the
    model's code map; noise(step, B, V) -> q, one step per canvas token from start_loc on.  keep: the kept-token overwrite of
    tests/keep_oracle.py.  scale / uncond: classifier-free guidance, l = u + s (c - u).  logits_hook(step, (i, j, d), logits)."""
    H, W, D = cfg.block_size
    Ht, Wt = partial_sample.shape[1:3]
    ks = O._per_depth(top_k, cfg.V, D, cfg.V)
    ps = O._per_depth(top_p, 1.0, D, 1.0)
    xs = partial_sample.clone()
    step = 0
    for (i, j) in product(range(Ht), range(Wt)):
        if (i, j) < tuple(start_loc):
            continue
        r0, c0, li, lj = window_of(i, j, (H, W), (Ht, Wt))
        win = xs[:, r0:r0 + H, c0:c0 + W]                  # a view: the depths written below are seen by the next ones
        sc, su = O.new_state(cfg), O.new_state(cfg)
        for d in range(D):
            lg = O.ar_cached_forward(sd, cfg, sc, win[:, :li + 1], codebook, cond, (li, lj, d))
            if scale is not None:
                u = O.ar_cached_forward(sd, cfg, su, win[:, :li + 1], codebook, uncond, (li, lj, d))
                lg = u + scale * (lg - u)
            if logits_hook is not None:
                logits_hook(step, (i, j, d), lg)
            drawn = O.sample_from_logits(lg, 1.0, ks[d], ps[d], q=noise(step, lg.shape[0], lg.shape[1]))
            xs[:, i, j, d] = drawn if keep is None else torch.where(keep[:, i, j, d], partial_sample[:, i, j, d], drawn)
            step += 1
    return xs
