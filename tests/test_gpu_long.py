"""Long sequences and head-less models on both tiers: a 32x32x4 code grid behind a 32-token prefix (body T = 1056, the f=8
RQ-VAE's latent grid) and a 16x16x1 model without head layers (measure_throughput's d = 1 runs), against the trajectories and
logits the unmodified reference stored in tests/golden/ar4.pt; the f=8 RQ-VAE's decoder; the fast tier's shape limits."""
import pytest
import torch

from oracle import rq_oracle as O
from oracle import synth
from oracle.zoo import vae_ddconfig
from rqvae import _native as N
from rqvae.models import create_model
from rqvae.utils.config import Config, augment_arch_defaults
from tests.helpers import CodebookAux, noise_tensor
from tests.test_gpu_fast import _with_env, fast_tier_parity_stats

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
DEV = "cuda"


def _ar_config(E, nh, nb, nhl, V, bs, vc, cl):
    return augment_arch_defaults(Config(
        type="rq-transformer", vocab_size=V, block_size=list(bs), vocab_size_cond=vc, block_size_cond=cl, embed_dim=E,
        input_embed_dim=256, shared_tok_emb=True, shared_cls_emb=True, input_emb_vqvae=True, head_emb_vqvae=True,
        cumsum_depth_ctx=True, body=dict(n_layer=nb, block=dict(n_head=nh)), head=dict(n_layer=nhl, block=dict(n_head=nh))))


def _build(shape, seed):
    """product model with the synthetic weights of `seed`; key / shape list from the product model itself"""
    with torch.device("meta"):
        model, _ = create_model(_ar_config(*shape))
    sd = synth.synth_state_dict(synth.shapes_of(model.state_dict()), seed)
    model = model.to_empty(device=DEV)
    model.load_state_dict({k: v.to(DEV) for k, v in sd.items()})
    return model.eval()


def _case(name, golden):
    fx = golden("ar4")
    g = fx["ar"][name]
    shape = fx["shapes"][name]
    E, nh, nb, nhl, V, bs, vc, cl = shape
    model = _build(shape, g["weight_seed"])
    cb = synth.randn_seeded((V, 256), g["codebook_seed"]).to(DEV)
    cond = synth.randint_seeded(0, max(vc, 1), (g["B"], cl), g["cond_seed"]).to(DEV) if vc > 1 else None
    return g, shape, model, CodebookAux(cb), cond, bs, V


NAMES = ["long32", "headless16"]


@pytest.mark.parametrize("name", NAMES)
def test_exact_tier_matches_reference(golden, name):
    g, shape, model, aux, cond, bs, V = _case(name, golden)
    model.precision = "exact"
    B = g["B"]
    n_tok = bs[0] * bs[1] * bs[2]
    for run in g["runs"]:
        st = run["setting"]
        codes, logits = model._native_sample(torch.zeros(B, *bs, dtype=torch.long, device=DEV), aux, cond, (0, 0), 1.0,
                                             st.get("top_k"), st.get("top_p"), False, noise=noise_tensor(run["noise_seed"], n_tok, B, V),
                                             return_logits=True)
        for step, lg in run["logits"].items():
            torch.testing.assert_close(logits[step].cpu(), lg, rtol=1e-4, atol=2e-4)
        d = (codes.cpu() != run["codes"].long()).flatten(1).any(0).nonzero()
        assert len(d) == 0, "%s %s: first divergent token %d of %d" % (name, st, int(d[0]), n_tok)
    rs = g["resume"]
    codes2 = model._native_sample(g["runs"][0]["codes"].long().to(DEV), aux, cond, rs["start_loc"], 1.0, rs["top_k"], None, False,
                                  noise=noise_tensor(rs["noise_seed"], n_tok, B, V))
    assert torch.equal(codes2.cpu().to(torch.int32), rs["codes"])


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("fmt", ["fp16", "bf16"])
def test_fast_tier_teacher_forced_step_parity(golden, name, fmt):
    g, shape, model, aux, cond, bs, V = _case(name, golden)
    r = _with_env(model, {"RQB200_FAST_DTYPE": fmt}, lambda: fast_tier_parity_stats(model, aux, cond, g, bs, V))
    print("%s %s: logits std %.3f, fast-tier error rms %.5f max %.5f; %d / %d greedy indices differ, %d outside the margin bound"
          % (name, fmt, r["std"], r["rms"], r["max"], r["flips"], r["n"], r["flips_outside_margin"]))
    k = 1.0 if fmt == "bf16" else 0.25
    assert r["rms"] < 0.02 * k * r["std"] and r["max"] < 0.15 * k * r["std"]
    assert r["flips_outside_margin"] == 0, "index flip outside the arithmetic error bound"
    for step, lg in g["runs"][-1]["logits"].items():
        assert float((r["lg16"][step].cpu() - lg).abs().max()) < 0.15 * k * r["std"] + 2e-4, step


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("fmt", ["fp16", "bf16"])
def test_fast_tier_batched_forward(golden, name, fmt):
    """forward(amp=True): the body pass over T = cond_len + H*W - 1 tokens (1055 for long32: the tiled attention kernel) against
    the same tier's sequential replay and the CPU oracle, cond_classifier logits included"""
    g, shape, model, aux, cond, bs, V = _case(name, golden)
    E, nh, nb, nhl, V_, bs_, vc, cl = shape
    codes = g["runs"][-1]["codes"].long().to(DEV)
    B = codes.shape[0]
    model.precision = "fast"

    def run():
        out = model(codes, model_aux=aux, cond=cond, amp=True)
        _, seq = model._native_sample(codes, aux, cond, (0, 0), 1.0, None, None, True, noise=False, return_logits=True, force_codes=codes)
        return out, seq.reshape(*bs, B, V).permute(3, 0, 1, 2, 4)

    out, seq = _with_env(model, {"RQB200_FAST_DTYPE": fmt}, run)
    out, cond_logits = out if isinstance(out, tuple) else (out, None)
    assert out.shape == (B, *bs, V)
    std = float(seq.std())
    d = float((out - seq).abs().max())
    print("%s %s: batched forward vs sequential replay: max logit difference %.2e (std %.3f)" % (name, fmt, d, std))
    assert d < (0.02 if fmt == "fp16" else 0.15) * std
    if fmt == "bf16":
        return
    sd = {k: v.cpu() for k, v in model.state_dict().items()}
    cfg = O.ArConfig(E, nh, nb, nhl, V, bs, vc, cl)
    table = aux.quantizer._shared_table().cpu()
    cpu_cond = None if cond is None else cond.cpu()
    if cl > 1:
        ref, cref = O.ar_forward(sd, cfg, codes.cpu(), table, cpu_cond, with_cond_logits=True)
        assert cond_logits is not None and cond_logits.shape == (B, cl - 1, vc)
        e = float((cond_logits.cpu() - cref).abs().max())
        print("%s: cond_logits vs oracle: max error %.2e (std %.3f)" % (name, e, float(cref.std())))
        assert e < 0.04 * float(cref.std())
    else:
        ref = O.ar_forward(sd, cfg, codes.cpu(), table, cpu_cond)
    assert float((out.cpu() - ref).abs().max()) < 0.04 * std


def test_fast_tier_resume_after_long_prefix(golden):
    """start_loc = (20, 3): a 675-token prefix, prefilled in one batched pass (tiled attention, KV cache written by query tile)"""
    g, shape, model, aux, cond, bs, V = _case("long32", golden)
    model.precision = "fast"
    B = g["B"]
    n_tok = bs[0] * bs[1] * bs[2]
    noise = noise_tensor(91, n_tok, B, V)
    part = torch.zeros(B, *bs, dtype=torch.long, device=DEV)
    a = model._native_sample(part, aux, cond, (0, 0), 1.0, 100, None, True, noise=noise)
    h0, w0 = 20, 3
    skip = (h0 * bs[1] + w0) * bs[2]
    tail = noise[skip:].contiguous()
    rb = model._native_sample(a, aux, cond, (h0, w0), 1.0, 100, None, True, noise=tail, return_logits=True)
    rs = _with_env(model, {"RQB200_SEQ_PREFILL": "1"},
                   lambda: model._native_sample(a, aux, cond, (h0, w0), 1.0, 100, None, True, noise=tail, return_logits=True))
    assert torch.equal(rs[0], a), "sequential-prefill resume must reproduce the trajectory bit for bit"
    std = float(rs[1].std())
    d = float((rb[1][0] - rs[1][0]).abs().max())
    print("resume at (%d,%d), prefix %d tokens: batched vs sequential prefill, first-step max logit difference %.2e (std %.3f)"
          % (h0, w0, shape[7] + h0 * bs[1] + w0, d, std))
    assert d < 0.02 * std
    assert torch.equal(rb[0].flatten(1)[:, :skip], a.flatten(1)[:, :skip])


def test_fast_tier_scheduling_has_no_effect_at_32x32(golden):
    g, shape, model, aux, cond, bs, V = _case("long32", golden)
    model.precision = "fast"
    B = g["B"]
    D = bs[2]
    n_tok = bs[0] * bs[1] * D
    noise = noise_tensor(92, n_tok, B, V)
    part = torch.zeros(B, *bs, dtype=torch.long, device=DEV)
    a = model._native_sample(part, aux, cond, (0, 0), 1.0, 100, 0.95, True, noise=noise)
    b = model._native_sample(part, aux, cond, (0, 0), 1.0, 100, 0.95, True, noise=noise)
    assert torch.equal(a, b), "fast tier is not run-to-run deterministic"
    for var in ("RQB200_NO_GRAPH", "RQB200_NO_PDL", "RQB200_TRACE"):
        c = _with_env(model, {var: "1"}, lambda: model._native_sample(part, aux, cond, (0, 0), 1.0, 100, 0.95, True, noise=noise))
        assert torch.equal(a, c), var
    # noise drawn span by span (bounded buffer, KV state resumed between spans) == one call with the whole noise tensor
    torch.manual_seed(4321)
    full = torch.empty(n_tok, B, V, device=DEV)
    for t in range(n_tok):
        full[t].exponential_(1)
    want = model._native_sample(part, aux, cond, (0, 0), 1.0, 100, 0.95, True, noise=full)
    model.noise_budget_bytes = 100 * D * B * V * 4              # 100 positions per span
    torch.manual_seed(4321)
    got = model._native_sample(part, aux, cond, (0, 0), 1.0, 100, 0.95, True)
    model.noise_budget_bytes = 256 << 20
    assert torch.equal(got, want)


def test_fast_tier_headless_large_batch_is_chunked(golden):
    g, shape, model, aux, cond, bs, V = _case("headless16", golden)
    model.precision = "fast"
    B = 300
    n_tok = bs[0] * bs[1] * bs[2]
    noise = torch.empty(n_tok, B, V, device=DEV).exponential_(1, generator=torch.Generator(DEV).manual_seed(3))
    cond = torch.randint(0, shape[6], (B, 1), device=DEV, generator=torch.Generator(DEV).manual_seed(4))
    part = torch.zeros(B, *bs, dtype=torch.long, device=DEV)
    full = model._native_sample(part, aux, cond, (0, 0), 1.0, 64, None, True, noise=noise)
    sub = model._native_sample(part[140:160], aux, cond[140:160], (0, 0), 1.0, 64, None, True, noise=noise[:, 140:160].contiguous())
    assert torch.equal(full[140:160], sub)


# the f=8 RQ-VAE (32x32x4 codes; its AttnBlocks attend over 1024 positions).  ch = 128: the fast tier runs its convs on wgmma only
# when every decoder channel count is a multiple of 128 (narrower decoders run the FFMA kernels on fp16-rounded weights)
F8_VAE = dict(K=512, code_shape=(32, 32, 4), ch=128, ch_mult=(1, 2, 2, 4), attn_resolutions=(32,), resolution=256)


def test_f8_vae_decode_vs_oracle():
    kw = F8_VAE
    dd = vae_ddconfig(**kw)
    cs = kw["code_shape"]
    cfg = augment_arch_defaults(Config(type="rq-vae", ddconfig=dd, hparams=dict(
        bottleneck_type="rq", embed_dim=256, n_embed=kw["K"], latent_shape=[cs[0], cs[1], 256], code_shape=list(cs),
        shared_codebook=True, decay=0.99, restart_unused_codes=True, loss_type="mse", latent_loss_weight=0.25)))
    with torch.device("meta"):
        model, _ = create_model(cfg)
    sd = synth.synth_state_dict(synth.shapes_of(model.state_dict()), 61)
    model = model.to_empty(device=DEV)
    model.load_state_dict({k: v.to(DEV) for k, v in sd.items()})
    model = model.eval()
    codes = synth.randint_seeded(0, kw["K"], (2, *cs), 62)
    ref = O.vae_decode_code(sd, dd, codes)
    assert ref.shape == (2, 3, 256, 256)
    for precision, bound in (("exact", 1e-4), ("fast", 1e-3)):
        model.precision = precision
        pix = model.decode_code(codes.to(DEV)).cpu()
        rel = float((pix - ref).norm() / ref.norm())
        print("f8 decode, %s tier: rel-L2 %.3e" % (precision, rel))
        assert rel < bound, (precision, rel)


def test_fast_tier_limits():
    V = 512
    cb = CodebookAux(synth.randn_seeded((V, 256), 1).to(DEV))
    # cond_len + H*W = 1 + 2048 = 2049: one past the fast tier's sequence limit
    model = _build((128, 2, 1, 1, V, (32, 64, 1), 10, 1), 5)
    codes = torch.zeros(1, 32, 64, 1, dtype=torch.long, device=DEV)
    with pytest.raises(N.NativeError, match="cond_len \\+ H\\*W <= 2048"):
        model(codes, model_aux=cb, amp=True)
    # no body layers: refused before anything runs
    model = _build((128, 2, 0, 1, V, (4, 4, 1), 10, 1), 5)
    with pytest.raises(N.NativeError, match="n_body >= 1"):
        model(torch.zeros(1, 4, 4, 1, dtype=torch.long, device=DEV), model_aux=cb, amp=True)
    # head dimension other than 64 (vqgan_large: E = 1664, 16 heads): the existing error
    model = _build((1664, 16, 1, 0, V, (4, 4, 1), 10, 1), 5)
    with pytest.raises(N.NativeError, match="embed_dim must be n_head\\*64"):
        model(torch.zeros(1, 4, 4, 1, dtype=torch.long, device=DEV), model_aux=cb, amp=True)
