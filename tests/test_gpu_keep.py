"""Masked completion (RQTransformer.sample(keep_mask=...)) on both tiers: kept tokens hold partial_sample's codes, the other tokens are
sampled as the reference's loop with a kept-token overwrite samples them (tests/golden/keep.pt, scripts/gen_golden_keep.py), positions
where nothing is sampled skip the head, and the fast tier appends runs of kept positions to the body's KV cache in one batched pass
(rqb200_dbg_append_attn: the tiled causal attention at a sequence offset T0, checked against an fp64 reference here)."""
import pytest
import torch

from oracle import synth
from oracle.zoo import AR_ZOO
from rqvae import _native as N
from tests import ar_kernels_ref as R
from tests import keep_oracle as KO
from tests.fp8_helpers import dequantised_copy
from tests.helpers import CodebookAux, build_ar, noise_tensor
from tests.test_gpu_ar_kernels import bits, guard_intact, guarded, run_prefill, within
from tests.test_gpu_cfg import TIERS, _run
from tests.test_gpu_fast import _with_env
from tests.test_gpu_long import _case as _long_case

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
DEV = "cuda"


def _fixture(name, golden, layouts):
    fx = golden("keep")
    P = fx["plan"]
    E, nh, nb_, nhl, V, bs, vc, cl = AR_ZOO[name]
    model, _ = build_ar(name, layouts, P["weight_seed"])
    aux = CodebookAux(synth.randn_seeded((V, 256), P["codebook_seed"]).to(DEV))
    B = P["B"]
    cond = synth.randint_seeded(0, vc, (B, cl), P["cond_seed"]).to(DEV)
    uncond = synth.randint_seeded(0, vc, (B, cl), P["uncond_seed"]).to(DEV)
    partial = KO.partial_of(B, bs, V).to(DEV)
    return P, fx["ar"][name]["runs"], model, aux, cond, uncond, partial, bs, V


def _sample(model, aux, cond, partial, keep_mask, start=(0, 0), noise=False, amp=False, k=64, p=0.9, guidance=None, force=None,
            logits=True):
    keep = None if keep_mask is None else model._keep_mask(keep_mask, partial.shape[0], start)
    return model._native_sample(partial, aux, cond, start, 1.0, k, p, amp, noise=noise, return_logits=logits, force_codes=force,
                                guidance=guidance, keep=keep)


def _evaluated(keep, bs):
    """[H*W*D] bool: the tokens whose logits a masked call computes (every depth of a position some row samples at some depth)"""
    H, W, D = bs
    pos = (~keep).reshape(keep.shape[0], H * W, D).any(2).any(0)
    return pos.repeat_interleave(D)


@pytest.mark.parametrize("name", ["tiny", "tiny_txt"])
def test_exact_tier_matches_reference(golden, layouts, name):
    """fp32 tier, the reference's injected noise: every case of keep.pt (box, depths >= 1, per-image random, all kept, a box with a
    start_loc resume, a guided box) equals the reference's codes token for token; kept tokens hold partial_sample's codes"""
    P, runs, model, aux, cond, uncond, partial, bs, V = _fixture(name, golden, layouts)
    model.precision = "exact"
    H, W, D = bs
    B = P["B"]
    for r in runs:
        keep = KO.mask_of(r["mask"], B, bs).to(DEV)
        start = tuple(r["start_loc"])
        n_tok = (H * W - start[0] * W - start[1]) * D
        noise = noise_tensor(r["noise_seed"], n_tok, B, V)
        g = None if r["scale"] is None else (r["scale"], uncond)
        codes, _ = _sample(model, aux, cond, partial, keep, start, noise, guidance=g, k=P["setting"]["top_k"], p=P["setting"]["top_p"])
        assert torch.equal(codes.cpu().to(torch.int16), r["codes"]), (name, r["mask"], start, r["scale"])
        assert torch.equal(codes[keep], partial[keep])
    model.precision = None


@pytest.mark.parametrize("tier", list(TIERS))
def test_all_false_mask_is_unmasked_sampling(layouts, tier):
    """a mask that keeps nothing: the codes and every returned logit of sample() without a mask, bit for bit, at the same launch
    count; unguided and guided"""
    E, nh, nb_, nhl, V, bs, vc, cl = AR_ZOO["tiny"]
    model, _ = build_ar("tiny", layouts, KO.PLAN["weight_seed"])
    aux = CodebookAux(synth.randn_seeded((V, 256), 12).to(DEV))
    B = 3
    cond = synth.randint_seeded(0, vc, (B, cl), 41).to(DEV)
    uncond = synth.randint_seeded(0, vc, (B, cl), 42).to(DEV)
    partial = KO.partial_of(B, bs, V, seed=43).to(DEV)
    noise = noise_tensor(44, bs[0] * bs[1] * bs[2], B, V)
    none = torch.zeros(B, *bs, dtype=torch.bool, device=DEV)
    for g in (None, (1.5, uncond)):
        def both(amp):
            a = _sample(model, aux, cond, partial, None, noise=noise, amp=amp, guidance=g)
            la = model.last_launches
            b = _sample(model, aux, cond, partial, none, noise=noise, amp=amp, guidance=g)
            return a, la, b, model.last_launches
        (ca, lga), la, (cb, lgb), lb = _run(model, tier, both)
        assert torch.equal(ca, cb) and torch.equal(lga, lgb) and la == lb, (tier, g is not None)


@pytest.mark.parametrize("tier", ["exact", "fp16", "fp8"])
def test_all_true_mask_returns_partial_without_launches(layouts, tier):
    model, _ = build_ar("tiny", layouts, KO.PLAN["weight_seed"])
    E, nh, nb_, nhl, V, bs, vc, cl = AR_ZOO["tiny"]
    aux = CodebookAux(synth.randn_seeded((V, 256), 12).to(DEV))
    B = 4
    cond = synth.randint_seeded(0, vc, (B, cl), 45).to(DEV)
    partial = KO.partial_of(B, bs, V, seed=46).to(DEV)
    everything = torch.ones(1, 1, 1, 1, dtype=torch.bool, device=DEV)

    def go(amp):
        out = model.sample(partial, model_aux=aux, cond=cond, top_k=64, amp=amp, keep_mask=everything)
        return out, model.last_launches
    out, launches = _run(model, tier, go)
    assert torch.equal(out, partial) and out.data_ptr() != partial.data_ptr() and launches == 0


@pytest.mark.parametrize("fmt", ["fp16", "fp8"])
@pytest.mark.parametrize("name", ["tiny", "tiny_txt"])
def test_fast_tier_logits_vs_exact_on_reference_cases(golden, layouts, name, fmt):
    """teacher-forced on the reference's masked trajectories: the fast tier's logits at every evaluated token (its batched appends
    included) within the fast tier's existing bounds of the exact tier's (E4M3 against its dequantised model), in units of the logits'
    std; no greedy flip outside the fp32 decision margin; kept tokens equal partial_sample"""
    P, runs, model, aux, cond, uncond, partial, bs, V = _fixture(name, golden, layouts)
    ref_model = dequantised_copy(model) if fmt == "fp8" else model
    rms_k, max_k = 0.005, 0.0375
    B = P["B"]
    for r in runs:
        keep = KO.mask_of(r["mask"], B, bs).to(DEV)
        if bool(keep.all()):
            continue
        start = tuple(r["start_loc"])
        codes = r["codes"].long().to(DEV)
        g = None if r["scale"] is None else (r["scale"], uncond)
        force = codes if g is None else torch.cat([codes, codes])
        ref_model.precision = "exact"
        c32, lg32 = _sample(ref_model, aux, cond, partial, keep, start, guidance=g, force=force)
        model.precision = "fast"
        c16, lg16 = _with_env(model, {"RQB200_FAST_DTYPE": fmt}, lambda: _sample(model, aux, cond, partial, keep, start, amp=True,
                                                                                 guidance=g, force=force))
        model.precision = None
        assert torch.equal(c32, codes) and torch.equal(c16, codes)
        ev = _evaluated(keep, bs)[start[0] * bs[1] * bs[2] + start[1] * bs[2]:]
        l32, l16 = lg32[ev], lg16[ev]
        std = float(l32.std())
        err = (l16 - l32).abs()
        assert float(err.pow(2).mean().sqrt()) < rms_k * std and float(err.max()) < max_k * std, (r["mask"], float(err.max()), std)
        top2 = l32.topk(2, dim=-1).values
        outside = (l16.argmax(-1) != l32.argmax(-1)) & (top2[..., 0] - top2[..., 1] > 2 * err.amax(-1))
        assert int(outside.sum()) == 0, r["mask"]


def test_batched_append_vs_token_by_token_at_32x32(golden):
    """32x32x4 codes behind 32 cond tokens, teacher-forced: sampled positions 3, 70, 200, 333 and 1023 leave runs of 67, 130, 133 and
    690 kept positions, appended at T0 = 35, 102, 232 and 365 (no multiple of 64; every run crosses 64-key tiles).  The batched appends'
    logits at the sampled positions stay within the batched-vs-sequential prefill bound of tests/test_gpu_long.py; the codes are equal"""
    g, shape, model, aux, cond, bs, V = _long_case("long32", golden)
    H, W, D = bs
    B = g["B"]
    codes = synth.randint_seeded(0, V, (B, *bs), 47).to(DEV)
    keep = torch.ones(H * W, 1, dtype=torch.bool, device=DEV)
    keep[[3, 70, 200, 333, 1023]] = False
    keep = keep.view(H, W, 1)
    model.precision = "fast"
    rb = _sample(model, aux, cond, codes, keep, amp=True, force=codes, k=100, p=None)
    rs = _with_env(model, {"RQB200_SEQ_PREFILL": "1"}, lambda: _sample(model, aux, cond, codes, keep, amp=True, force=codes, k=100, p=None))
    model.precision = None
    assert torch.equal(rb[0], codes) and torch.equal(rs[0], codes)
    ev = _evaluated(keep.expand(B, H, W, D), bs)
    std = float(rs[1][ev].std())
    d = float((rb[1][ev] - rs[1][ev]).abs().max())
    print("batched vs token-by-token appends at 32x32: max logit difference %.2e (std %.3f)" % (d, std))
    assert d < 0.02 * std


@pytest.mark.parametrize("tier", ["exact", "fp16"])
def test_spans_give_the_codes_of_one_span(layouts, tier):
    """public API drawing its own noise: a noise budget of two positions (spans that end inside runs of kept positions, runs long
    enough for batched appends) gives the codes of one span bit for bit"""
    model, _ = build_ar("tiny", layouts, KO.PLAN["weight_seed"])
    E, nh, nb_, nhl, V, bs, vc, cl = AR_ZOO["tiny"]
    H, W, D = bs
    aux = CodebookAux(synth.randn_seeded((V, 256), 12).to(DEV))
    B = 3
    cond = synth.randint_seeded(0, vc, (B, cl), 48).to(DEV)
    partial = KO.partial_of(B, bs, V, seed=49).to(DEV)
    keep = torch.ones(B, H * W, D, dtype=torch.bool)
    keep[:, [0, 7, 15], :] = synth.randn_seeded((B, 3, D), 50) > 0
    keep[0, 7, 1] = False
    keep = keep.view(B, H, W, D).to(DEV)

    def go(amp):
        outs = []
        for budget in (1 << 30, 2 * D * B * V * 4):
            model.noise_budget_bytes = budget
            torch.manual_seed(9)
            outs.append(model.sample(partial, model_aux=aux, cond=cond, top_k=64, top_p=0.9, amp=amp, keep_mask=keep))
        model.noise_budget_bytes = 256 << 20
        return outs
    one, many = _run(model, tier, go)
    assert torch.equal(one, many)
    assert torch.equal(one[keep], partial[keep])


def test_fast_tier_chunks_with_a_per_image_mask(layouts):
    """B = 300 images on the fast tier (two chunks of 150) with a per-image mask == each chunk run alone"""
    model, _ = build_ar("tiny", layouts, KO.PLAN["weight_seed"])
    E, nh, nb_, nhl, V, bs, vc, cl = AR_ZOO["tiny"]
    aux = CodebookAux(synth.randn_seeded((V, 256), 12).to(DEV))
    B, n_tok = 300, bs[0] * bs[1] * bs[2]
    cond = synth.randint_seeded(0, vc, (B, cl), 51).to(DEV)
    partial = KO.partial_of(B, bs, V, seed=52).to(DEV)
    keep = (synth.randn_seeded((B, *bs), 53) > 0.5).to(DEV)
    q = noise_tensor(54, n_tok, B, V)
    model.precision = "fast"
    whole = _sample(model, aux, cond, partial, keep, noise=q, amp=True, k=100, logits=False)
    for lo in (0, 150):
        sl = slice(lo, lo + 150)
        piece = _sample(model, aux, cond[sl], partial[sl], keep[sl], noise=q[:, sl].contiguous(), amp=True, k=100, logits=False)
        assert torch.equal(piece, whole[sl]), lo
    model.precision = None
    assert torch.equal(whole[keep], partial[keep])


# ---------------------------------------------------------------------------------------------------------------- append attention
def append_ref(qkv, kc, vc, G, T0, T, E, fmt):
    """fp64 causal attention of T new tokens at offset T0: keys / values = the cache rows [0, T0) then the new tokens' -> (ref, slack)"""
    nh = E // 64
    x = qkv.view(T, G, 3, nh, 64).double()
    q = x[:, :, 0].permute(1, 2, 0, 3).reshape(G * nh, T, 64)
    k = torch.cat([kc[:, :, :T0].double(), x[:, :, 1].permute(1, 2, 0, 3)], 2).reshape(G * nh, T0 + T, 64)
    v = torch.cat([vc[:, :, :T0].double(), x[:, :, 2].permute(1, 2, 0, 3)], 2).reshape(G * nh, T0 + T, 64)
    mask = torch.arange(T0 + T, device=qkv.device)[None, :] <= (T0 + torch.arange(T, device=qkv.device))[:, None]
    ref = R.attend(q, k, v, mask).view(G, nh, T, 64).permute(2, 0, 1, 3).reshape(T * G, E)
    slack = R.attn_slack(q, k, v, mask, fmt, True).view(G, nh, T, 1).expand(G, nh, T, 64).permute(2, 0, 1, 3).reshape(T * G, E)
    return ref, slack


def run_append(qkv, kc, vc, G, T0, T, E, Tmax, fmt):
    bufs = [guarded(c) for c in (kc, vc)]
    afull, att = guarded(torch.full((T * G, E), float("nan"), dtype=R.DT[fmt], device=DEV))
    N.check(N.lib().rqb200_dbg_append_attn(N.ptr(qkv), N.ptr(bufs[0][1]), N.ptr(bufs[1][1]), N.ptr(att), G, T0, T, E, Tmax, fmt,
                                           N.stream_ptr()), "dbg_append_attn")
    torch.cuda.synchronize()
    assert guard_intact(afull, T * G * E)
    return att, bufs


APPEND_CASES = [(0, 65, 102), (5, 1, 64), (100, 1, 128), (7, 65, 100), (63, 70, 170), (64, 64, 128), (65, 129, 300),
                (2048 - 65, 65, 2048), (2047, 1, 2048)]


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("T0,T,Tmax", APPEND_CASES)
def test_append_attention(T0, T, Tmax, fmt):
    """rqb200_dbg_append_attn against the fp64 reference at the tile edges (T0 = 63, 64, 65; k = 1 and 65; T0 + k = Tmax = 2048): the
    attention within the flash kernel's bound; cache rows [T0, T0 + k) = the new K / V, every other row and the guard untouched; at
    T0 = 0 the prefill's launch bit for bit"""
    G, E = 3, 128
    nh = E // 64
    gen = torch.Generator(DEV).manual_seed(T0 * 7 + T)
    qkv = torch.randn(T * G, 3 * E, generator=gen, device=DEV).to(R.DT[fmt])
    kc, vc = (torch.randn(G, nh, Tmax, 64, generator=gen, device=DEV).to(R.DT[fmt]) for _ in range(2))
    att, bufs = run_append(qkv, kc, vc, G, T0, T, E, Tmax, fmt)
    ref, slack = append_ref(qkv, kc, vc, G, T0, T, E, fmt)
    within(att, ref, slack, fmt, "T0 %d T %d fmt %d" % (T0, T, fmt))
    for m, (full, c) in enumerate(bufs):
        want = (kc, vc)[m].clone()
        want[:, :, T0:T0 + T] = qkv[:, (m + 1) * E:(m + 2) * E].view(T, G, nh, 64).permute(1, 2, 0, 3)
        assert torch.equal(bits(c), bits(want)), "K" if m == 0 else "V"
        assert guard_intact(full, G * nh * Tmax * 64)
    if T0 == 0:
        att_p, _, _ = run_prefill(qkv, G, T, E, Tmax, fmt)
        assert torch.equal(bits(att), bits(att_p))


def test_keep_mask_errors_raise_before_any_kernel(layouts):
    model, _ = build_ar("tiny", layouts, KO.PLAN["weight_seed"])
    E, nh, nb_, nhl, V, bs, vc, cl = AR_ZOO["tiny"]
    aux = CodebookAux(synth.randn_seeded((V, 256), 12).to(DEV))
    part = torch.zeros(3, *bs, dtype=torch.long, device=DEV)
    cond = synth.randint_seeded(0, vc, (3, cl), 55).to(DEV)
    bad = [torch.ones(*bs, dtype=torch.uint8, device=DEV), torch.ones(4, *bs, dtype=torch.bool, device=DEV),
           torch.ones(*bs, dtype=torch.bool)]
    launches = N.launch_count["total"]
    for k in bad:
        with pytest.raises(ValueError):
            model.sample(part, model_aux=aux, cond=cond, keep_mask=k)
    assert N.launch_count["total"] == launches
