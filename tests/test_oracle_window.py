"""tests/window_oracle.py's sliding-window loop on oracle/rq_oracle.py against the unmodified reference's trajectories in
tests/golden/win.pt (scripts/gen_golden_window.py), bit for bit, before any GPU runs; and on the grid itself the loop is sample()'s."""
import pytest
import torch

from oracle import rq_oracle as O
from oracle import synth
from oracle.zoo import AR_ZOO
from tests import keep_oracle as KO
from tests import window_oracle as WO


def _setup(golden, layouts, name):
    fx = golden("win")
    P, runs = fx["plan"], fx["ar"][name]["runs"]
    E, nh, nb, nhl, V, bs, vc, cl = AR_ZOO[name]
    cfg = O.ArConfig(E, nh, nb, nhl, V, bs, vc, cl)
    sd = synth.synth_state_dict(layouts["ar/" + name], P["weight_seed"])
    cb = synth.randn_seeded((V, 256), P["codebook_seed"])
    B = P["B"]
    cond = synth.randint_seeded(0, vc, (B, cl), P["cond_seed"])
    uncond = synth.randint_seeded(0, vc, (B, cl), P["uncond_seed"])
    return P, runs, cfg, sd, cb, cond, uncond, bs, V


@pytest.mark.parametrize("name", ["tiny", "tiny_txt"])
def test_window_oracle_matches_reference(golden, layouts, name):
    P, runs, cfg, sd, cb, cond, uncond, bs, V = _setup(golden, layouts, name)
    B, D = P["B"], bs[2]
    assert [(tuple(r["canvas"]), r["mask"], tuple(r["start_loc"]), r["scale"]) for r in runs] == WO.CASES[name]
    for r in runs:
        canvas = tuple(r["canvas"])
        partial = WO.partial_of(B, canvas, D, V)
        keep = WO.mask_of(r["mask"], B, canvas, D)
        codes = WO.window_sample(sd, cfg, partial, cb, keep, cond=cond, start_loc=r["start_loc"], scale=r["scale"], uncond=uncond,
                                 noise=lambda step, B_, V_, s=r["noise_seed"]: synth.exp_noise(s, step, B_, V_), **P["setting"])
        assert codes.shape == (B, *canvas, D)
        assert torch.equal(codes.to(torch.int16), r["codes"]), (canvas, r["mask"], r["start_loc"], r["scale"])
        if keep is not None:
            assert torch.equal(codes[keep], partial[keep])
        pre = torch.zeros(canvas[0] * canvas[1], dtype=torch.bool)
        pre[:r["start_loc"][0] * canvas[1] + r["start_loc"][1]] = True
        assert torch.equal(codes.view(B, -1, D)[:, pre], partial.view(B, -1, D)[:, pre])


@pytest.mark.parametrize("name", ["tiny", "tiny_txt"])
def test_grid_canvas_is_the_keep_protocol(golden, layouts, name):
    """canvas == grid: the window loop (a fresh cache per position) gives the codes of keep.pt's protocol (one cache for the whole
    grid, tests/keep_oracle.py) on the same inputs"""
    P, runs, cfg, sd, cb, cond, uncond, bs, V = _setup(golden, layouts, name)
    B, D = P["B"], bs[2]
    grid = [r for r in runs if tuple(r["canvas"]) == tuple(bs[:2])]
    assert grid
    for r in grid:
        partial = WO.partial_of(B, bs[:2], D, V)
        keep = WO.mask_of(r["mask"], B, bs[:2], D)
        noise = lambda step, B_, V_, s=r["noise_seed"]: synth.exp_noise(s, step, B_, V_)      # noqa: E731
        one = KO.ar_sample_keep(sd, cfg, partial, cb, torch.zeros(B, *bs, dtype=torch.bool) if keep is None else keep, cond=cond,
                                noise=noise, **P["setting"])
        assert torch.equal(one.to(torch.int16), r["codes"]), r["mask"]
