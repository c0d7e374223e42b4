"""tests/keep_oracle.py's masked-completion loop on oracle/rq_oracle.py against the unmodified reference's trajectories in
tests/golden/keep.pt (scripts/gen_golden_keep.py), bit for bit, before any GPU runs."""
import pytest
import torch

from oracle import rq_oracle as O
from oracle import synth
from oracle.zoo import AR_ZOO
from tests import keep_oracle as KO


@pytest.mark.parametrize("name", ["tiny", "tiny_txt"])
def test_keep_oracle_matches_reference(golden, layouts, name):
    fx = golden("keep")
    P, runs = fx["plan"], fx["ar"][name]["runs"]
    E, nh, nb, nhl, V, bs, vc, cl = AR_ZOO[name]
    cfg = O.ArConfig(E, nh, nb, nhl, V, bs, vc, cl)
    sd = synth.synth_state_dict(layouts["ar/" + name], P["weight_seed"])
    cb = synth.randn_seeded((V, 256), P["codebook_seed"])
    B = P["B"]
    cond = synth.randint_seeded(0, vc, (B, cl), P["cond_seed"])
    uncond = synth.randint_seeded(0, vc, (B, cl), P["uncond_seed"])
    partial = KO.partial_of(B, bs, V)
    assert [(r["mask"], tuple(r["start_loc"]), r["scale"]) for r in runs] == KO.CASES[name]
    for r in runs:
        keep = KO.mask_of(r["mask"], B, bs)
        codes = KO.ar_sample_keep(sd, cfg, partial, cb, keep, cond=cond, start_loc=r["start_loc"], noise=lambda step, B_, V_, s=r["noise_seed"]:
                                  synth.exp_noise(s, step, B_, V_), scale=r["scale"], uncond=uncond, **P["setting"])
        assert torch.equal(codes.to(torch.int16), r["codes"]), (r["mask"], r["start_loc"], r["scale"])
        assert torch.equal(codes[keep], partial[keep])
        H, W, D = bs
        pre = torch.zeros(H * W, dtype=torch.bool)
        pre[:r["start_loc"][0] * W + r["start_loc"][1]] = True
        assert torch.equal(codes.view(B, H * W, D)[:, pre], partial.view(B, H * W, D)[:, pre])
