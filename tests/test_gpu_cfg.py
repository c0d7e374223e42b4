"""Classifier-free guidance in RQTransformer.sample on both tiers: image b runs a cond and an uncond branch as rows b and n + b of one
native batch, and the sampler draws from l = u + s (c - u) formed in fp32 as three rounded operations.  Checked bit for bit against
torch's own `u + s * (c - u)` on the engine's raw logits, against unguided 2n-row runs that must give the same logits or codes, and
against the guided trajectories of the unmodified reference (tests/golden/cfg.pt, scripts/gen_golden_cfg.py)."""
import pytest
import torch

from oracle import synth
from oracle.zoo import AR_ZOO
from rqvae import _native as N
from rqvae.models import _bind as nb
from tests import variants_oracle as VO
from tests.fp8_helpers import dequantised_copy
from tests.helpers import CodebookAux, build_ar, noise_tensor
from tests.test_gpu_fast import _with_env
from tests.test_gpu_long import _build as _build_long, _case as _long_case
from tests.test_gpu_variants import aux_for, build as build_variant

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
DEV = "cuda"
# tier -> (precision, amp, RQB200_FAST_DTYPE)
TIERS = {"exact": ("exact", False, None), "fp16": ("fast", True, "fp16"), "bf16": ("fast", True, "bf16"), "fp8": ("fast", True, "fp8")}


def _run(model, tier, fn):
    prec, amp, fmt = TIERS[tier]
    model.precision = prec
    try:
        return _with_env(model, {"RQB200_FAST_DTYPE": fmt} if fmt else {}, lambda: fn(amp))
    finally:
        model.precision = None


def _zoo(name, layouts, B=3, seed=11):
    E, nh, nb_, nhl, V, bs, vc, cl = AR_ZOO[name]
    model, _ = build_ar(name, layouts, seed)
    aux = CodebookAux(synth.randn_seeded((V, 256), 12).to(DEV))
    cond = synth.randint_seeded(0, vc, (B, cl), 13).to(DEV)
    uncond = synth.randint_seeded(0, vc, (B, cl), 14).to(DEV)
    return model, aux, cond, uncond, bs, V


def _guided(model, aux, cond, uncond, bs, s, noise, k=None, p=None, amp=False, start=(0, 0), partial=None, force=None):
    B = cond.shape[0]
    part = torch.zeros(B, *bs, dtype=torch.long, device=DEV) if partial is None else partial
    return model._native_sample(part, aux, cond, start, 1.0, k, p, amp, noise=noise, return_logits=True, force_codes=force,
                                guidance=(s, uncond.reshape(B, -1).long()))


def _unguided(model, aux, cond, bs, noise, k=None, p=None, amp=False, partial=None, force=None, logits=True):
    B = cond.shape[0]
    part = torch.zeros(B, *bs, dtype=torch.long, device=DEV) if partial is None else partial
    return model._native_sample(part, aux, cond, (0, 0), 1.0, k, p, amp, noise=noise, return_logits=logits, force_codes=force)


def _check_composition(model, aux, cond, uncond, bs, V, s, k, p, amp, noise):
    """(1) torch's u + s*(c - u) on the returned raw logits, sampled with nb.sample_logits and the same noise row, gives every code the
    engine wrote; (2) the raw logits equal an unguided teacher-forced 2n-row call with cond = cat(c, u) and the guided codes in both
    halves, and a guided teacher-forced call returns them too -- so the uncond branch consumed the same codes"""
    n = cond.shape[0]
    H, W, D = bs
    codes, lg = _guided(model, aux, cond, uncond, bs, s, noise, k, p, amp)
    assert lg.shape == (H * W * D, 2 * n, V)
    ks, ps = model._lists(k, p)
    flat = codes.reshape(n, -1)
    for t in range(H * W * D):
        c, u = lg[t, :n], lg[t, n:]
        want = nb.sample_logits(u + s * (c - u), 1.0, ks[t % D], ps[t % D], q=noise[t])
        assert torch.equal(want, flat[:, t]), "token %d" % t
    both = torch.cat([codes, codes])
    c2 = torch.cat([cond.reshape(n, -1), uncond.reshape(n, -1)])
    out2, lg2 = _unguided(model, aux, c2, bs, False, amp=amp, partial=both, force=both)
    assert torch.equal(out2, both) and torch.equal(lg2, lg)
    out3, lg3 = _guided(model, aux, cond, uncond, bs, s, False, amp=amp, partial=codes, force=both)
    assert torch.equal(out3, codes) and torch.equal(lg3, lg)
    return codes


@pytest.mark.parametrize("tier", list(TIERS))
@pytest.mark.parametrize("name", ["tiny", "tiny_txt"])
def test_guided_codes_are_torch_composition_bit_for_bit(layouts, name, tier):
    model, aux, cond, uncond, bs, V = _zoo(name, layouts)
    if name == "tiny_txt":
        uncond = torch.zeros_like(cond)                       # the all-zero caption
    n_tok = bs[0] * bs[1] * bs[2]
    noise = noise_tensor(31, n_tok, cond.shape[0], V)
    for s, k, p in ((1.5, 64, None), (3.0, 100, 0.9), (-0.5, None, None)):
        _run(model, tier, lambda amp: _check_composition(model, aux, cond, uncond, bs, V, s, k, p, amp, noise))


@pytest.mark.parametrize("tier", ["exact", "fp16", "fp8"])
def test_guided_embedding_variant_headless_and_32x32(golden, tier):
    """the reference's all-false embedding switches (own token tables, per-depth classifiers), a head-less 16x16x1 model and a
    32x32x4 map behind a 32-token prefix"""
    vm, _ = build_variant(VO.TINY, VO.ALL_FALSE)
    vc, cl = VO.TINY[6], VO.TINY[7]
    cases = [(vm, aux_for(VO.ALL_FALSE), VO.TINY[5], VO.TINY[4], vc, cl)]
    for nm in ("headless16", "long32"):
        g, shape, model, aux, cond, bs, V = _long_case(nm, golden)
        cases.append((model, aux, bs, V, shape[6], shape[7]))
    for model, aux, bs, V, vc, cl in cases:
        cond = synth.randint_seeded(0, vc, (2, cl), 51).to(DEV)
        uncond = synth.randint_seeded(0, vc, (2, cl), 52).to(DEV)
        noise = noise_tensor(53, bs[0] * bs[1] * bs[2], 2, V)
        _run(model, tier, lambda amp: _check_composition(model, aux, cond, uncond, bs, V, 2.0, 100, 0.95, amp, noise))


@pytest.mark.parametrize("tier", ["exact", "fp16"])
def test_scale_zero_is_the_uncond_branch(layouts, tier):
    """s = 0: guided codes == rows [n, 2n) of an unguided 2n-row sample with cond = cat(c, u) and noise cat(q, q)"""
    model, aux, cond, uncond, bs, V = _zoo("tiny", layouts)
    n = cond.shape[0]
    q = noise_tensor(32, bs[0] * bs[1] * bs[2], n, V)

    def go(amp):
        g, _ = _guided(model, aux, cond, uncond, bs, 0.0, q, 100, 0.9, amp)
        u, _ = _unguided(model, aux, torch.cat([cond, uncond]), bs, torch.cat([q, q], 1), 100, 0.9, amp)
        assert torch.equal(g, u[n:])
    _run(model, tier, go)


@pytest.mark.parametrize("tier", ["exact", "fp16"])
def test_uncond_equal_to_cond_is_unguided(layouts, tier):
    """uncond == cond: guided codes at any s == rows [0, n) of an unguided 2n-row sample with cond = cat(c, c) and noise cat(q, q);
    on the exact tier also == unguided sampling of the n images"""
    model, aux, cond, _, bs, V = _zoo("tiny", layouts)
    n = cond.shape[0]
    q = noise_tensor(33, bs[0] * bs[1] * bs[2], n, V)

    def go(amp):
        u, _ = _unguided(model, aux, torch.cat([cond, cond]), bs, torch.cat([q, q], 1), 100, 0.9, amp)
        one, _ = _unguided(model, aux, cond, bs, q, 100, 0.9, amp)
        for s in (0.0, 1.5, 4.0):
            g, _ = _guided(model, aux, cond, cond, bs, s, q, 100, 0.9, amp)
            assert torch.equal(g, u[:n]), s
            if not amp:
                assert torch.equal(g, one), s
    _run(model, tier, go)


def _fixture_case(name, golden, layouts):
    fx = golden("cfg")
    P, g = fx["plan"], fx["ar"][name]
    E, nh, nb_, nhl, V, bs, vc, cl = AR_ZOO[name]
    model, _ = build_ar(name, layouts, P["weight_seed"])
    aux = CodebookAux(synth.randn_seeded((V, 256), P["codebook_seed"]).to(DEV))
    cond = synth.randint_seeded(0, vc, (P["B"], cl), P["cond_seed"]).to(DEV)
    uncond = (synth.randint_seeded(0, vc, (P["B"], cl), P["uncond_seed"]) if name == "tiny" else torch.zeros(P["B"], cl, dtype=torch.long))
    return P, g, model, aux, cond, uncond.to(DEV), bs, V


def _first_diff(a, b):
    d = (a != b).flatten(1).any(0).nonzero()
    return int(d[0]) if len(d) else -1


@pytest.mark.parametrize("name", ["tiny", "tiny_txt"])
def test_exact_tier_guided_codes_match_reference(golden, layouts, name):
    """fp32 tier, the reference's injected Exp(1) noise: codes equal the reference's guided trajectories token for token; the kept
    guided logits agree within fp32 summation order (scaled by |s| + |1 - s|, the factor l = s c + (1 - s) u carries errors by)"""
    P, g, model, aux, cond, uncond, bs, V = _fixture_case(name, golden, layouts)
    model.precision = "exact"
    B, n_tok = P["B"], bs[0] * bs[1] * bs[2]
    for run in g["runs"]:
        s, st = run["scale"], run["setting"]
        noise = noise_tensor(P["noise_seed"], n_tok, B, V)
        codes, lg = _guided(model, aux, cond, uncond, bs, s, noise, st.get("top_k"), st.get("top_p"))
        if run["logits"]:
            amp_ = abs(s) + abs(1 - s)
            for step, want in run["logits"].items():
                c, u = lg[step, :B], lg[step, B:]
                torch.testing.assert_close((u + s * (c - u)).cpu(), want, rtol=1e-4 * amp_, atol=2e-4 * amp_)
        fd = _first_diff(codes.cpu(), run["codes"].long())
        assert fd < 0, "%s s=%s %s: first divergent token %d of %d" % (name, s, st, fd, n_tok)
    rs = g["resume"]
    noise = noise_tensor(rs["noise_seed"], n_tok, B, V)
    codes2, _ = _guided(model, aux, cond, uncond, bs, rs["scale"], noise, rs["setting"].get("top_k"), rs["setting"].get("top_p"),
                        start=rs["start_loc"], partial=g["runs"][0]["codes"].long().to(DEV))
    assert torch.equal(codes2.cpu().to(torch.int16), rs["codes"])


def _guided_logits(lg, s):
    n = lg.shape[1] // 2
    c, u = lg[:, :n], lg[:, n:]
    return u + s * (c - u)


@pytest.mark.parametrize("fmt", ["fp16", "fp8"])
@pytest.mark.parametrize("name", ["tiny", "tiny_txt"])
def test_fast_tier_guided_logits_vs_exact(golden, layouts, name, fmt):
    """teacher-forced on the reference's guided trajectories: the fast tier's guided logits within its existing bounds of the exact
    tier's (fp16 against the same weights, E4M3 against its dequantised model, as tests/test_gpu_fp8_tier.py), in units of the raw
    logits' std and scaled by |s| + |1 - s|; no greedy flip outside the fp32 decision margin"""
    P, g, model, aux, cond, uncond, bs, V = _fixture_case(name, golden, layouts)
    ref_model = dequantised_copy(model) if fmt == "fp8" else model
    rms_k, max_k = 0.005, 0.0375             # the fp16 tier's rms / max bounds (0.02 / 0.15 of the std, 4x tighter than bf16's)
    for run in g["runs"]:
        s = run["scale"]
        codes = run["codes"].long().to(DEV)
        both = torch.cat([codes, codes])
        ref_model.precision = "exact"
        _, lg32 = _guided(ref_model, aux, cond, uncond, bs, s, False, partial=codes, force=both)
        model.precision = "fast"
        _, lg16 = _with_env(model, {"RQB200_FAST_DTYPE": fmt}, lambda: _guided(model, aux, cond, uncond, bs, s, False, amp=True,
                                                                             partial=codes, force=both))
        model.precision = None
        std = float(lg32.std())
        l32, l16 = _guided_logits(lg32, s), _guided_logits(lg16, s)
        err = (l16 - l32).abs()
        amp_ = abs(s) + abs(1 - s)
        assert float(err.pow(2).mean().sqrt()) < rms_k * amp_ * std and float(err.max()) < max_k * amp_ * std, (s, float(err.max()), std)
        top2 = l32.topk(2, dim=-1).values
        differ = l16.argmax(-1) != l32.argmax(-1)
        outside = differ & (top2[..., 0] - top2[..., 1] > 2 * err.amax(-1))
        assert int(outside.sum()) == 0, "greedy flip outside the fp32 decision margin (s=%s)" % s


def test_fast_tier_chunks_of_128_images(layouts):
    """B = 300 images on the fast tier (three chunks of 100 images, 200 rows each) == the same images run chunk by chunk; guided costs
    the launches of an unguided call at 2n rows"""
    model, aux, _, _, bs, V = _zoo("tiny", layouts)
    vc, cl = AR_ZOO["tiny"][6], AR_ZOO["tiny"][7]
    B, n_tok = 300, bs[0] * bs[1] * bs[2]
    cond = synth.randint_seeded(0, vc, (B, cl), 61).to(DEV)
    uncond = synth.randint_seeded(0, vc, (B, cl), 62).to(DEV)
    q = noise_tensor(63, n_tok, B, V)
    model.precision = "fast"
    part = torch.zeros(B, *bs, dtype=torch.long, device=DEV)
    whole = model._native_sample(part, aux, cond, (0, 0), 1.0, 100, 0.9, True, noise=q, guidance=(2.5, uncond))
    for lo in range(0, B, 100):
        sl = slice(lo, lo + 100)
        piece = model._native_sample(part[sl], aux, cond[sl], (0, 0), 1.0, 100, 0.9, True, noise=q[:, sl].contiguous(),
                                     guidance=(2.5, uncond[sl]))
        assert torch.equal(piece, whole[sl]), lo
        guided_launches = model.last_launches
    model._native_sample(torch.zeros(200, *bs, dtype=torch.long, device=DEV), aux, torch.cat([cond[:100], uncond[:100]]), (0, 0), 1.0,
                         100, 0.9, True, noise=False)
    assert guided_launches == model.last_launches
    # through the public API, drawing its own noise: the default scale is unguided and consumes the RNG as before
    torch.manual_seed(5)
    a = model.sample(part[:4], model_aux=aux, cond=cond[:4], top_k=100, top_p=0.9, amp=True)
    torch.manual_seed(5)
    b = model.sample(part[:4], model_aux=aux, cond=cond[:4], top_k=100, top_p=0.9, amp=True, cfg_scale=None, uncond=None)
    torch.manual_seed(5)
    c = model.sample(part[:4], model_aux=aux, cond=cond[:4], top_k=100, top_p=0.9, amp=True, cfg_scale=2.5, uncond=uncond[:4])
    torch.manual_seed(5)
    d = model._native_sample(part[:4], aux, cond[:4], (0, 0), 1.0, 100, 0.9, True, guidance=(2.5, uncond[:4]))
    assert torch.equal(a, b) and torch.equal(c, d) and c.shape == a.shape
    model.precision = None


def test_guidance_errors_raise_before_any_kernel(layouts):
    model, aux, cond, uncond, bs, V = _zoo("tiny", layouts)
    part = torch.zeros(3, *bs, dtype=torch.long, device=DEV)
    cl, vc = AR_ZOO["tiny"][7], AR_ZOO["tiny"][6]
    bad = [dict(cfg_scale=1.5), dict(uncond=uncond), dict(cfg_scale=1.5, uncond=uncond[:2]),
           dict(cfg_scale=1.5, uncond=torch.full((3, cl), -1, device=DEV)), dict(cfg_scale=1.5, uncond=torch.full((3, cl), vc, device=DEV))]
    launches = N.launch_count["total"]
    for kw in bad:
        with pytest.raises(ValueError):
            model.sample(part, model_aux=aux, cond=cond, **kw)
    unconditional = _build_long((128, 2, 1, 1, 512, (4, 4, 4), 1, 1), 7)          # vocab_size_cond == 1
    with pytest.raises(ValueError):
        unconditional.sample(part, model_aux=aux, cfg_scale=1.5, uncond=torch.zeros(3, 1, dtype=torch.long, device=DEV))
    assert N.launch_count["total"] == launches
