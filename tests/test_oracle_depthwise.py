"""CPU: the per-depth-codebook oracle (tests/depthwise_oracle.py) reproduces the reference's outputs in tests/golden/rqd.pt, and
the product's RQ-VAE with shared_codebook=False has the reference's state_dict layout and seeded default initialisation."""
import torch

from oracle import rq_oracle as O
from oracle import synth
from oracle.zoo import VAE_ZOO, vae_ddconfig
from rqvae.models import create_model
from rqvae.utils.config import Config, augment_arch_defaults
from tests import depthwise_oracle as DO

torch.set_grad_enabled(False)


def assert_sample(t, ref, tol=1e-5):
    total, values = ref
    s, v = (float(t.double().sum()), t.reshape(-1)[torch.randint(0, t.numel(), (values.numel(),),
                                                                 generator=torch.Generator().manual_seed(t.numel()))])
    torch.testing.assert_close(v, values, rtol=0, atol=tol)
    assert abs(s - total) <= tol * (1.0 + abs(total))


def make_depthwise_vae(device="cpu"):
    kw = VAE_ZOO["tiny"]
    cs = kw["code_shape"]
    cfg = Config(type="rq-vae", hparams=dict(bottleneck_type="rq", embed_dim=256, n_embed=kw["K"], latent_shape=[cs[0], cs[1], 256],
                                             code_shape=list(cs), shared_codebook=False, decay=0.99, restart_unused_codes=True,
                                             loss_type="mse", latent_loss_weight=0.25),
                 ddconfig=vae_ddconfig(**kw))
    with torch.device(device):
        model, _ = create_model(augment_arch_defaults(cfg))
    return model


def test_oracle_reproduces_reference_rq_runs(golden):
    g = golden("rqd")
    for name, rec in g["rq"].items():
        tables, x = DO.rq_inputs(name)
        quants, codes = DO.rq_quantize(x, tables)
        assert torch.equal(codes, rec["codes"].long()), name
        for a, ref in zip(quants, rec["agg_sums"]):
            assert abs(float(a.double().sum()) - ref) <= 1e-5 * (1.0 + abs(ref)), name
        assert_sample(quants[-1], rec["last"])
        assert_sample(DO.embed_code(codes, tables), rec["embed_code"])
        assert_sample(DO.embed_code_with_depth(codes, tables), rec["embed_code_with_depth"])
        for (typ, i), ref in rec["partial"].items():
            assert_sample(DO.embed_partial_code(codes, tables, i, typ), ref)
        if "soft" in rec:
            soft, scodes = DO.rq_soft_codes(x[:2], tables)
            assert torch.equal(scodes, codes[:2])
            assert_sample(soft, rec["soft"])
    # the tie case: every table-2 code is a first index (rows 256.. repeat rows 0..255); the planted input hits row 5 of table 0
    ties = g["rq"]["ties"]["codes"].long()
    assert int(ties[..., 2].max()) < 256 and int(ties[0, 0, 0, 0]) == 5


def test_depthwise_vae_layout_and_seeded_init_equal_reference(golden):
    g = golden("rqd")["vae"]
    m = make_depthwise_vae("meta")
    assert {k: list(v.shape) for k, v in m.state_dict().items()} == g["layout"]
    torch.manual_seed(0)
    sd = make_depthwise_vae().state_dict()
    assert sorted(sd) == sorted(g["init"])
    cbs = make_depthwise_vae("meta").quantizer.codebooks
    assert len({id(c) for c in cbs}) == len(cbs)
    for k, (shape, total, values) in synth.state_dict_sample(sd).items():
        ref = g["init"][k]
        assert shape == ref[0], k
        assert torch.equal(values, ref[2]), k
        assert abs(total - ref[1]) <= 1e-9 * (1.0 + abs(ref[1])), k


def test_oracle_decode_code_matches_reference(golden):
    g = golden("rqd")["vae"]
    sd = DO.depthwise_vae_state({k: tuple(v) for k, v in g["layout"].items()}, g["weight_seed"], g["table_seed"])
    tables = [sd["quantizer.codebooks.%d.weight" % d][:-1] for d in range(4)]
    codes = synth.randint_seeded(0, 512, (2, 4, 4, 4), g["codes_seed"])
    pix = DO.vae_decode_code(sd, vae_ddconfig(**VAE_ZOO["tiny"]), codes, tables)
    torch.testing.assert_close(pix, g["pixels"], rtol=0, atol=1e-5)


def test_oracle_ar_over_per_depth_tables_matches_reference(golden):
    g = golden("rqd")["ar"]
    P = DO.AR_PLAN
    E, nh, nb, nhl, V, bs, vc, cl = DO.AR_SHAPE
    cfg = O.ArConfig(E, nh, nb, nhl, V, bs, vc, cl)
    sd = synth.synth_state_dict(synth.shapes_of(make_ar_meta().state_dict()), P["weight_seed"])
    tables = DO.tables_of([V] * bs[2], P["table_seed"])
    cond = synth.randint_seeded(0, vc, (P["B"], cl), P["cond_seed"])
    for run in g["runs"]:
        kept = {}
        codes = DO.ar_sample(sd, cfg, torch.zeros(P["B"], *bs, dtype=torch.long), tables, cond=cond,
                             noise=lambda step, B, V_, s=run["noise_seed"]: synth.exp_noise(s, step, B, V_),
                             logits_hook=lambda step, loc, lg: kept.__setitem__(step, lg) if step in run["logits"] else None,
                             **run["setting"])
        assert torch.equal(codes, run["codes"].long()), run["setting"]
        for step, lg in run["logits"].items():
            torch.testing.assert_close(kept[step], lg, rtol=0, atol=1e-5)
    rs = P["resume"]
    codes2 = DO.ar_sample(sd, cfg, g["runs"][1]["codes"].long(), tables, cond=cond, start_loc=rs["start_loc"],
                          noise=lambda step, B, V_: synth.exp_noise(rs["noise_seed"], step, B, V_), **P["settings"][1])
    assert torch.equal(codes2, g["resume"]["codes"].long())
    assert not torch.equal(codes2, g["runs"][1]["codes"].long())      # the resume resampled the tail


def make_ar_meta():
    E, nh, nb, nhl, V, bs, vc, cl = DO.AR_SHAPE
    cfg = Config(type="rq-transformer", vocab_size=V, block_size=list(bs), vocab_size_cond=vc, block_size_cond=cl, embed_dim=E,
                 input_embed_dim=256, shared_tok_emb=True, shared_cls_emb=True, input_emb_vqvae=True, head_emb_vqvae=True,
                 cumsum_depth_ctx=True, body=dict(n_layer=nb, block=dict(n_head=nh)), head=dict(n_layer=nhl, block=dict(n_head=nh)))
    with torch.device("meta"):
        model, _ = create_model(augment_arch_defaults(cfg))
    return model
