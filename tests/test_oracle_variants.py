"""CPU: the variants oracle (tests/variants_oracle.py) reproduces the reference's RQ-Transformer trajectories for every combination of
the five embedding / classifier switches (tests/golden/arv.pt), and the product's RQTransformer builds the reference's state_dict
layout and seeded default initialisation for all of them."""
import pytest
import torch

from oracle import rq_oracle as O
from oracle import synth
from rqvae.models import create_model
from rqvae.utils.config import Config, augment_arch_defaults
from tests import variants_oracle as VO

torch.set_grad_enabled(False)


def variant_config(shape, flags):
    E, nh, nb, nhl, V, bs, vc, cl = shape
    cfg = Config(type="rq-transformer", vocab_size=V, block_size=list(bs), vocab_size_cond=vc, block_size_cond=cl, embed_dim=E,
                 input_embed_dim=256, body=dict(n_layer=nb, block=dict(n_head=nh)), head=dict(n_layer=nhl, block=dict(n_head=nh)),
                 **flags)
    return augment_arch_defaults(cfg)


def make_variant(shape, flags, device="cpu"):
    with torch.device(device):
        model, _ = create_model(variant_config(shape, flags))
    return model.eval()


def oracle_model(shape, flags):
    E, nh, nb, nhl, V, bs, vc, cl = shape
    cfg = O.ArConfig(E, nh, nb, nhl, V, bs, vc, cl)
    shapes = synth.shapes_of(make_variant(shape, flags, "meta").state_dict())
    return cfg, VO.state_dict_of(shapes, VO.PLAN["weight_seed"])


def table():
    return synth.randn_seeded((VO.TINY[4], 256), VO.PLAN["table_seed"])


def check_runs(shape, flags, runs, codebook):
    cfg, sd = oracle_model(shape, flags)
    cond = synth.randint_seeded(0, shape[6], (VO.PLAN["B"], shape[7]), VO.PLAN["cond_seed"])
    for run in runs:
        kept = {}
        codes = VO.ar_sample(sd, cfg, flags, torch.zeros(VO.PLAN["B"], *shape[5], dtype=torch.long), codebook, cond=cond,
                             noise=lambda s, B, V: synth.exp_noise(run["noise_seed"], s, B, V),
                             logits_hook=lambda s, loc, lg: kept.__setitem__(s, lg.clone()), **run["setting"])
        assert torch.equal(codes, run["codes"].long()), (VO.combo_name(flags), run["setting"])
        for s, ref in zip(run["logit_steps"], run["logits"]):
            torch.testing.assert_close(kept[s], ref, rtol=0, atol=1e-5)
    return cfg, sd, cond


@pytest.mark.parametrize("name", [VO.combo_name(f) for f in VO.COMBOS])
def test_oracle_reproduces_reference_variant_runs(golden, name):
    rec = golden("arv")["combos"][name]
    check_runs(VO.TINY, rec["flags"], rec["runs"], table() if VO.needs_codebook(rec["flags"]) else None)


def test_oracle_reproduces_text_resume_forward_and_headless(golden):
    g = golden("arv")
    t = g["text"]
    cfg, sd, cond = check_runs(VO.TEXT, VO.ALL_FALSE, t["runs"], None)
    rs = VO.PLAN["resume"]
    codes2 = VO.ar_sample(sd, cfg, VO.ALL_FALSE, t["runs"][1]["codes"].long(), None, cond=cond, start_loc=rs["start_loc"],
                          noise=lambda s, B, V: synth.exp_noise(rs["noise_seed"], s, B, V), **VO.PLAN["settings"][1])
    assert torch.equal(codes2, t["resume"]["codes"].long())
    logits, cond_logits = VO.ar_forward(sd, cfg, VO.ALL_FALSE, t["runs"][0]["codes"][:1].long(), None, cond[:1], with_cond_logits=True)
    torch.testing.assert_close(logits, t["forward"], rtol=0, atol=1e-5)
    torch.testing.assert_close(cond_logits, t["cond_logits"], rtol=0, atol=1e-5)
    check_runs(VO.HEADLESS, VO.ALL_FALSE, g["headless"]["runs"], None)


def assert_init(sd, ref):
    """sd equals the reference's seeded initialisation: every tensor's shape and fp64 sum, and the sampled values"""
    got = synth.state_dict_sample(sd, VO.PLAN["init_sample"])
    assert torch.equal(torch.tensor([v[1] for v in got.values()], dtype=torch.float64), ref["sums"])
    assert torch.equal(torch.cat([v[2].reshape(-1) for v in got.values()]), ref["values"])


@pytest.mark.parametrize("name", [VO.combo_name(f) for f in VO.COMBOS])
def test_variant_layout_and_seeded_init_equal_reference(golden, name):
    rec = golden("arv")["combos"][name]
    m = make_variant(VO.TINY, rec["flags"], "meta")
    assert [(k, list(v.shape)) for k, v in m.state_dict().items()] == golden("arv")["layouts"][rec["layout"]]
    torch.manual_seed(VO.PLAN["init_seed"])
    assert_init(make_variant(VO.TINY, rec["flags"]).state_dict(), rec["init"])


def test_unequal_vocabularies_build_and_load_but_do_not_compute(golden):
    g = golden("arv")["unequal"]
    U = VO.UNEQUAL
    torch.manual_seed(VO.PLAN["init_seed"])
    m = make_variant(U["shape"], U["flags"])
    assert [(k, list(v.shape)) for k, v in m.state_dict().items()] == g["layout"]
    assert_init(m.state_dict(), g["init"])
    vs = U["shape"][4]
    sd = VO.state_dict_of(synth.shapes_of(m.state_dict()), 3, vs)
    m.load_state_dict(sd)
    assert m.tok_emb.offsets.tolist() == [0, 512, 768, 1152]
    xs = torch.zeros(1, *U["shape"][5], dtype=torch.long)
    with pytest.raises(NotImplementedError, match="LogitMask"):
        m.sample(xs)
    with pytest.raises(NotImplementedError, match="LogitMask"):
        m(xs)


def test_model_aux_none_is_rejected_when_a_codebook_is_needed():
    for flags in VO.COMBOS:
        m = make_variant(VO.TINY, flags)
        if VO.needs_codebook(flags):
            with pytest.raises(ValueError, match="model_aux"):
                m._codebook_of(None, VO.TINY[5][2])
        else:
            assert m._codebook_of(None, VO.TINY[5][2]) is None


def test_embed_variant_bits_match_the_header():
    import os
    import re
    from rqvae import _native as N
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "rqb200.h")).read()
    bits = {n: int(v) for n, v in re.findall(r"#define\s+RQB200_(EMB_[A-Z0-9_]+)\s+(\d+)", hdr)}
    assert set(bits) == {"EMB_TOK_INPUT", "EMB_TOK_HEAD", "EMB_NO_CUMSUM", "EMB_TUPLE", "EMB_CLS_PER_DEPTH"}
    for name, value in bits.items():
        assert getattr(N, name) == value, name
    # the shipped family is variant 0; the reference's defaults set every token-source bit
    assert make_variant(VO.TINY, VO.COMBOS[-1], "meta")._embed_variant() == 0
    assert make_variant(VO.TINY, VO.ALL_FALSE, "meta")._embed_variant() == (N.EMB_TOK_INPUT | N.EMB_TOK_HEAD | N.EMB_TUPLE |
                                                                           N.EMB_CLS_PER_DEPTH)
