"""Pins the CPU oracle against the long-sequence fixtures of the unmodified reference (tests/golden/ar4.pt): a 32x32x4 grid behind
a 32-token prefix (body T = 1056) and a head-less (n_head_layers = 0) 16x16x1 model.  CPU only."""
import pytest
import torch

from oracle import rq_oracle as O
from oracle import synth
from rqvae.models import create_model
from tests.test_gpu_long import _ar_config

torch.set_grad_enabled(False)


@pytest.mark.parametrize("name", ["long32", "headless16"])
def test_ar_long_sample_matches_reference(golden, name):
    fx = golden("ar4")
    g = fx["ar"][name]
    E, nh, nb, nhl, V, bs, vc, cl = shape = fx["shapes"][name]
    with torch.device("meta"):
        model, _ = create_model(_ar_config(*shape))
    sd = synth.synth_state_dict(synth.shapes_of(model.state_dict()), g["weight_seed"])
    cfg = O.ArConfig(E, nh, nb, nhl, V, bs, vc, cl)
    cb = synth.randn_seeded((V, 256), g["codebook_seed"])
    cond = synth.randint_seeded(0, max(vc, 1), (g["B"], cl), g["cond_seed"]) if vc > 1 else None
    for run in g["runs"]:
        kept = {}
        codes = O.ar_sample(sd, cfg, torch.zeros(g["B"], *bs, dtype=torch.long), cb, cond=cond,
                            noise=lambda step, B, V_, s=run["noise_seed"]: synth.exp_noise(s, step, B, V_),
                            logits_hook=lambda step, loc, lg: kept.__setitem__(step, lg.clone()) if step in run["logits"] else None,
                            **run["setting"])
        assert torch.equal(codes.to(torch.int32), run["codes"])
        for step, lg in run["logits"].items():
            torch.testing.assert_close(kept[step], lg, rtol=1e-5, atol=1e-5)
    rs = g["resume"]
    codes2 = O.ar_sample(sd, cfg, g["runs"][0]["codes"].long(), cb, cond=cond, start_loc=rs["start_loc"], top_k=rs["top_k"],
                         noise=lambda step, B, V_: synth.exp_noise(rs["noise_seed"], step, B, V_))
    assert torch.equal(codes2.to(torch.int32), rs["codes"])
