"""GPU: one codebook per depth (RQBottleneck(shared_codebook=False)) through the RQ search kernels, the code embeddings, the
RQ-VAE engine and the AR engine -- against the reference's outputs (tests/golden/rqd.pt), the per-depth oracle
(tests/depthwise_oracle.py) and the shared-codebook path on identical values."""
import pytest
import torch

from oracle import rq_oracle as O
from oracle import synth
from oracle.zoo import AR_ZOO, VAE_ZOO, vae_ddconfig
from rqvae import _native as N
from rqvae.models import _bind as nb
from rqvae.models import create_model
from rqvae.models.rqvae.quantizations import RQBottleneck
from rqvae.utils.config import Config, augment_arch_defaults
from tests import depthwise_oracle as DO
from tests.helpers import ar_config, noise_tensor
from tests.test_gpu_parity import audit_code_flips

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
DEV = "cuda"


def bottleneck(ks, tables):
    q = RQBottleneck(latent_shape=[8, 8, 256], code_shape=[8, 8, len(ks)], n_embed=list(ks), shared_codebook=False).to(DEV).eval()
    for d, t in enumerate(tables):
        q.codebooks[d].weight[:-1] = t.to(DEV)
    return q


def sample_of(t, n):
    flat = t.reshape(-1)
    return flat[torch.randint(0, flat.numel(), (n,), generator=torch.Generator().manual_seed(flat.numel()))]


def dbg_quantize(form, x, tables):
    n, D = x.shape[0], len(tables)
    _tabs, ptrs, ks = nb.tables(tables)
    codes = torch.empty(n, D, dtype=torch.int64, device=DEV)
    ql = torch.empty(D, n, 256, device=DEV)
    res = torch.empty(n, 256, device=DEV)
    N.check(N.lib().rqb200_dbg_rq_quantize_depthwise(form, N.ptr(x), ptrs, ks, n, 256, D, N.ptr(codes), N.ptr(ql), N.ptr(res), None),
            "dbg_rq_quantize_depthwise")
    torch.cuda.synchronize()
    return codes, ql, res


# ------------------------------------------------------------------------------------------------ RQ search + embeddings
@pytest.mark.parametrize("name", list(DO.RQ_CASES))
def test_rq_search_and_embeddings_match_reference(golden, name):
    rec = golden("rqd")["rq"][name]
    ks = DO.RQ_CASES[name][0]
    tables, x = DO.rq_inputs(name)
    q = bottleneck(ks, tables)
    quants, codes = q.quantize(x.to(DEV))
    assert torch.equal(codes.cpu(), rec["codes"].long())
    for a, ref in zip(quants, rec["agg_sums"]):
        assert abs(float(a.double().sum()) - ref) <= 1e-5 * (1.0 + abs(ref))
    oq, _ = DO.rq_quantize(x, tables)
    torch.testing.assert_close(quants[-1].cpu(), oq[-1], rtol=0, atol=2e-6)
    # embeddings are gathers / <= D fp32 adds in depth order: equal to the oracle, and to the reference's sampled values
    torch.testing.assert_close(q.embed_code(codes).cpu(), DO.embed_code(codes.cpu(), tables), rtol=0, atol=0)
    torch.testing.assert_close(sample_of(q.embed_code(codes).cpu(), 256), rec["embed_code"][1], rtol=0, atol=1e-6)
    emb, _ = q.embed_code_with_depth(codes)
    torch.testing.assert_close(emb.cpu(), DO.embed_code_with_depth(codes.cpu(), tables), rtol=0, atol=0)
    for (typ, i), ref in rec["partial"].items():
        got = q.embed_partial_code(codes, i, typ).cpu()
        torch.testing.assert_close(got, DO.embed_partial_code(codes.cpu(), tables, i, typ), rtol=0, atol=0)
        torch.testing.assert_close(sample_of(got, 256), ref[1], rtol=0, atol=1e-6)
    if "soft" in rec:
        x2 = x[:2]                                               # the fixture's soft codes cover the first two images
        soft, scodes = q.get_soft_codes(x2.to(DEV))
        rs, rc = DO.rq_soft_codes(x2, tables)
        assert torch.equal(scodes.cpu(), rc)
        # soft = softmax(-d): a distance error of e moves a soft code by a relative e.  Both sides round d = ||r||^2 + ||e||^2 - 2 r.e
        # in fp32 with different summation orders, so the bound is 8 ulp of the largest ||r||^2 + ||e||^2 (the near-tie bound of
        # test_gpu_parity.audit_rq_codes), and never tighter than the shared-codebook test's 2e-4
        oq, _ = DO.rq_quantize(x2, tables)
        scale = max(float((x2 - (oq[d - 1] if d else 0)).pow(2).sum(-1).max() + t.pow(2).sum(-1).max()) for d, t in enumerate(tables))
        rtol = max(2e-4, 8 * 2.0 ** -23 * scale)
        torch.testing.assert_close(soft.cpu(), rs, rtol=rtol, atol=1e-6)
        torch.testing.assert_close(sample_of(soft.cpu(), 256), rec["soft"][1], rtol=rtol, atol=1e-6)
        s2, c2 = q.get_soft_codes(x2.to(DEV), stochastic=True)
        assert s2.shape == soft.shape and int(c2.max()) < ks[0]
        torch.testing.assert_close(s2[..., 0, :], soft[..., 0, :], rtol=0, atol=0)


@pytest.mark.parametrize("ks,n", [([2048] * 4, 1000), ([512, 1000, 2048, 300], 517), ([16384] * 4, 4096), ([300, 16384, 7, 256], 130)])
def test_rq_search_forms_bit_identical_on_separate_tables(ks, n):
    """the 2x4-tile kernel and the 2-CTA cluster kernel on per-depth tables in separate allocations: identical bits"""
    tables = [synth.randn_seeded((k, 256), 40 + d).to(DEV) for d, k in enumerate(ks)]
    x = synth.randn_seeded((n, 256), 50).to(DEV)
    c1, q1, r1 = dbg_quantize(1, x, tables)
    c2, q2, r2 = dbg_quantize(2, x, tables)
    assert torch.equal(c1, c2)
    assert torch.equal(q1, q2) and torch.equal(r1, r2)
    _, co = DO.rq_quantize(x.cpu(), [t.cpu() for t in tables])
    assert torch.equal(c1.cpu(), co)


@pytest.mark.parametrize("form", [1, 2])
def test_identical_tables_give_the_shared_bits(form):
    """D distinct allocations holding one table's values: the per-depth path computes exactly what the shared call computes"""
    cb = synth.randn_seeded((4096, 256), 60).to(DEV)
    x = synth.randn_seeded((777, 256), 61).to(DEV)
    c, ql, res = dbg_quantize(form, x, [cb.clone() for _ in range(4)])
    codes = torch.empty_like(c)
    ql0, res0 = torch.empty_like(ql), torch.empty_like(res)
    N.check(N.lib().rqb200_dbg_rq_quantize(form, N.ptr(x), N.ptr(cb), 777, 4096, 256, 4, N.ptr(codes), N.ptr(ql0), N.ptr(res0), None),
            "dbg_rq_quantize")
    torch.cuda.synchronize()
    assert torch.equal(c, codes) and torch.equal(ql, ql0) and torch.equal(res, res0)
    s = nb.rq_embed(c, cb, summed=True)
    assert torch.equal(nb.rq_embed(c, [cb.clone() for _ in range(4)], summed=True), s)


# ------------------------------------------------------------------------------------------------ RQ-VAE
def depthwise_vae(golden):
    g = golden("rqd")["vae"]
    kw = VAE_ZOO["tiny"]
    cs = kw["code_shape"]
    cfg = Config(type="rq-vae", hparams=dict(bottleneck_type="rq", embed_dim=256, n_embed=kw["K"], latent_shape=[cs[0], cs[1], 256],
                                             code_shape=list(cs), shared_codebook=False, decay=0.99, restart_unused_codes=True,
                                             loss_type="mse", latent_loss_weight=0.25),
                 ddconfig=vae_ddconfig(**kw))
    model, _ = create_model(augment_arch_defaults(cfg))
    sd = DO.depthwise_vae_state({k: tuple(v) for k, v in g["layout"].items()}, g["weight_seed"], g["table_seed"])
    model.load_state_dict(sd)
    return model.to(DEV).eval(), sd, g


def test_depthwise_vae_decode_get_codes_forward(golden):
    model, sd, g = depthwise_vae(golden)
    tables = [sd["quantizer.codebooks.%d.weight" % d][:-1] for d in range(4)]
    codes = synth.randint_seeded(0, 512, (2, 4, 4, 4), g["codes_seed"]).to(DEV)
    model.precision = "exact"
    pix = model.decode_code(codes).cpu()
    rel = float((pix - g["pixels"]).norm() / g["pixels"].norm())
    assert rel < 1e-4, "exact decode rel-L2 %.3g" % rel
    # fast tier: decode_code's per-depth embedding is the same gather as embed_code, so it equals decode(embed_code(codes))
    model.precision = "fast"
    pix_f = model.decode_code(codes)
    torch.testing.assert_close(pix_f, model.decode(model.quantizer.embed_code(codes)), rtol=0, atol=0)
    model.precision = "exact"
    img = synth.randn_seeded((2, 3, 16, 16), g["image_seed"], 0.5).to(DEV)
    got = model.get_codes(img)
    z = model.encode(img).cpu()
    z_ref = O.vae_encode(sd, vae_ddconfig(**VAE_ZOO["tiny"]), img.cpu())
    ref = g["get_codes"].long()
    # per-depth flip audit: stack the tables and offset codes so the audit's shared-table arithmetic selects table d at depth d
    offs = torch.arange(4) * 512
    n_flip = audit_code_flips(z_ref, z, torch.cat(tables, 0), ref + offs, got.cpu() + offs)
    print("per-depth tiny VAE get_codes: %d audited near-tie flips" % n_flip)
    out, loss, c_fwd = model(img)
    assert torch.equal(c_fwd, got) and out.shape == img.shape and torch.isfinite(out).all()


def test_depthwise_vae_fast_tier_decode_within_1e3():
    """fast-tier decode_code of a per-depth RQ-VAE whose decoder runs on the wgmma convs (every channel count a multiple of 128;
    the tiny zoo VAE's ch = 32 falls back to FFMA on fp16-rounded weights) against the per-depth oracle"""
    dd = dict(double_z=False, z_channels=256, resolution=16, in_channels=3, out_ch=3, ch=128, ch_mult=[1, 2], num_res_blocks=1,
              attn_resolutions=[8], dropout=0.0)
    torch.manual_seed(3)
    model, _ = create_model(augment_arch_defaults(Config(type="rq-vae", ddconfig=dd, hparams=dict(
        bottleneck_type="rq", embed_dim=256, n_embed=[512, 300, 1000, 64], latent_shape=[8, 8, 256], code_shape=[8, 8, 4],
        shared_codebook=False, decay=0.99, restart_unused_codes=True, loss_type="mse", latent_loss_weight=0.25))))
    tables = DO.tables_of([512, 300, 1000, 64], 7)
    for d, t in enumerate(tables):
        model.quantizer.codebooks[d].weight[:-1] = t
    model = model.to(DEV).eval()
    sd = {k: v.detach().cpu() for k, v in model.state_dict().items()}
    codes = torch.stack([synth.randint_seeded(0, k, (2, 8, 8), 8 + d) for d, k in enumerate([512, 300, 1000, 64])], -1)
    ref = DO.vae_decode_code(sd, dd, codes, tables)
    for prec, bound in (("exact", 1e-4), ("fast", 1e-3)):
        model.precision = prec
        pix = model.decode_code(codes.to(DEV)).cpu()
        rel = float((pix - ref).norm() / ref.norm())
        print("per-depth VAE (ch 128, unequal K) %s decode rel-L2 %.2e" % (prec, rel))
        assert rel < bound


# ------------------------------------------------------------------------------------------------ AR over per-depth tables
class TablesAux:
    """stand-in RQ-VAE whose quantizer holds D per-depth tables"""

    def __init__(self, tables):
        self.quantizer = RQBottleneck(latent_shape=[4, 4, 256], code_shape=[4, 4, len(tables)], n_embed=[t.shape[0] for t in tables],
                                      shared_codebook=False).to(DEV).eval()
        for d, t in enumerate(tables):
            self.quantizer.codebooks[d].weight[:-1] = t.to(DEV)


def tiny_ar():
    E, nh, nbody, nhl, V, bs, vc, cl = AR_ZOO["tiny"]
    torch.manual_seed(5)
    model, _ = create_model(ar_config("tiny"))
    model = model.to(DEV).eval()
    sd = {k: v.detach().cpu() for k, v in model.state_dict().items()}
    return model, sd, O.ArConfig(E, nh, nbody, nhl, V, bs, vc, cl)


def test_ar_exact_tier_trajectories_match_reference(golden):
    """greedy and top-k/top-p trajectories and a start_loc resume of a transformer whose model_aux holds per-depth tables: codes
    bit-exact against the reference's (tests/golden/rqd.pt), under the same per-token Exp(1) noise"""
    g = golden("rqd")["ar"]
    P = DO.AR_PLAN
    E, nh, nb, nhl, V, bs, vc, cl = DO.AR_SHAPE
    with torch.device("meta"):
        model, _ = create_model(_ar_config(*DO.AR_SHAPE))
    sd = synth.synth_state_dict(synth.shapes_of(model.state_dict()), P["weight_seed"])
    model = model.to_empty(device=DEV)
    model.load_state_dict({k: v.to(DEV) for k, v in sd.items()})
    model = model.eval()
    model.precision = "exact"
    aux = TablesAux(DO.tables_of([V] * bs[2], P["table_seed"]))
    cond = synth.randint_seeded(0, vc, (P["B"], cl), P["cond_seed"]).to(DEV)
    n_tok = bs[0] * bs[1] * bs[2]
    for run in g["runs"]:
        st = run["setting"]
        codes, logits = model._native_sample(torch.zeros(P["B"], *bs, dtype=torch.long, device=DEV), aux, cond, (0, 0), 1.0,
                                             st.get("top_k"), st.get("top_p"), False,
                                             noise=noise_tensor(run["noise_seed"], n_tok, P["B"], V), return_logits=True)
        for step, lg in run["logits"].items():
            torch.testing.assert_close(logits[step].cpu(), lg, rtol=1e-4, atol=2e-4)
        d = (codes.cpu() != run["codes"].long()).flatten(1).any(0).nonzero()
        assert len(d) == 0, "%s: first divergent token %d of %d" % (st, int(d[0]), n_tok)
    rs = P["resume"]
    st = P["settings"][1]
    codes2 = model._native_sample(g["runs"][1]["codes"].long().to(DEV), aux, cond, rs["start_loc"], 1.0, st["top_k"], st["top_p"],
                                  False, noise=noise_tensor(rs["noise_seed"], n_tok, P["B"], V))
    assert torch.equal(codes2.cpu(), g["resume"]["codes"].long())


def _ar_config(E, nh, nb, nhl, V, bs, vc, cl):
    return augment_arch_defaults(Config(
        type="rq-transformer", vocab_size=V, block_size=list(bs), vocab_size_cond=vc, block_size_cond=cl, embed_dim=E,
        input_embed_dim=256, shared_tok_emb=True, shared_cls_emb=True, input_emb_vqvae=True, head_emb_vqvae=True,
        cumsum_depth_ctx=True, body=dict(n_layer=nb, block=dict(n_head=nh)), head=dict(n_layer=nhl, block=dict(n_head=nh))))


def test_ar_per_depth_tables():
    model, sd, cfg = tiny_ar()
    V, bs = cfg.V, cfg.block_size
    tables = [synth.randn_seeded((V, 256), 70 + d) for d in range(bs[2])]
    aux = TablesAux(tables)
    cond = synth.randint_seeded(0, cfg.vocab_cond, (2, cfg.cond_len), 13)
    xs = synth.randint_seeded(0, V, (2, *bs), 71)
    ref = DO.ar_forward(sd, cfg, xs, tables, cond)
    # exact tier: teacher-forced replay against the oracle
    model.precision = "exact"
    lg = model(xs.to(DEV), model_aux=aux, cond=cond.to(DEV))
    torch.testing.assert_close(lg.cpu(), ref, rtol=1e-4, atol=2e-4)
    # identical values in D separate tables: bit-identical to the shared engine, sampled codes included
    same = TablesAux([tables[0]] * bs[2])
    shared = TablesAux.__new__(TablesAux)
    shared.quantizer = RQBottleneck(latent_shape=[4, 4, 256], code_shape=[4, 4, bs[2]], n_embed=V, shared_codebook=True).to(DEV).eval()
    shared.quantizer.codebooks[0].weight[:-1] = tables[0].to(DEV)
    for amp in (False, True):
        a = model.sample(torch.zeros(2, *bs, dtype=torch.long, device=DEV), model_aux=same, cond=cond.to(DEV), top_k=1, amp=amp)
        b = model.sample(torch.zeros(2, *bs, dtype=torch.long, device=DEV), model_aux=shared, cond=cond.to(DEV), top_k=1, amp=amp)
        assert torch.equal(a, b)
    # fast tier: batched forward and the teacher-forced step replay, fp16 and bf16, against the oracle
    model.precision = "fast"
    import os
    for dt in ("fp16", "bf16"):
        os.environ["RQB200_FAST_DTYPE"] = dt
        model._invalidate_native()
        try:
            fwd = model(xs.to(DEV), model_aux=aux, cond=cond.to(DEV), amp=True).cpu()
            _, step = model._native_sample(xs.to(DEV), aux, cond.to(DEV), (0, 0), 1.0, None, None, True, noise=False,
                                           return_logits=True, force_codes=xs.to(DEV))
        finally:
            del os.environ["RQB200_FAST_DTYPE"]
            model._invalidate_native()
        n_tok = bs[0] * bs[1] * bs[2]
        want = ref.reshape(2, n_tok, V).permute(1, 0, 2)
        err_fwd = float((fwd - ref).abs().max()) / float(ref.std())
        err_step = float((step.cpu() - want).abs().max()) / float(want.std())
        print("per-depth AR fast tier %s: forward %.4f sigma, step replay %.4f sigma" % (dt, err_fwd, err_step))
        assert err_fwd < 0.02 and err_step < 0.02


def test_ar_engine_reuse_and_rebuild_on_table_edit():
    model, sd, cfg = tiny_ar()
    V, bs = cfg.V, cfg.block_size
    aux = TablesAux([synth.randn_seeded((V, 256), 80 + d) for d in range(bs[2])])
    model.precision = "exact"
    z = torch.zeros(2, *bs, dtype=torch.long, device=DEV)
    model.sample(z, model_aux=aux, top_k=1)
    eng = dict(model._eng)
    model.sample(z, model_aux=aux, top_k=1)
    assert len(model._eng) == 1 and list(model._eng) == list(eng)
    assert next(iter(model._eng.values()))["handle"] == next(iter(eng.values()))["handle"]
    xs = synth.randint_seeded(0, V, (2, *bs), 81).to(DEV)
    before = model(xs, model_aux=aux)
    fp = model._eng_fp
    aux.quantizer.codebooks[2].weight[:V] += 0.5                   # in place: bumps the table's version counter
    after = model(xs, model_aux=aux)
    assert model._eng_fp != fp and len(model._eng) == 1             # the engine was rebuilt from the edited table
    assert torch.equal(before[:, 0, 0, 0], after[:, 0, 0, 0])       # the first token reads no code
    assert not torch.equal(before[..., 3, :], after[..., 3, :])     # depth 3's head input sums table 2's row


def test_ar_refuses_unequal_tables():
    model, _, cfg = tiny_ar()
    bs = cfg.block_size
    aux = TablesAux([synth.randn_seeded((k, 256), 90) for k in (cfg.V, cfg.V, 256, cfg.V)])
    with pytest.raises(ValueError):
        model.sample(torch.zeros(1, *bs, dtype=torch.long, device=DEV), model_aux=aux)
