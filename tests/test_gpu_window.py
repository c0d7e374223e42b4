"""Sliding-window sampling (RQTransformer.sample on a canvas larger than the model's grid) on both tiers: the exact tier's codes equal the
unmodified reference's window-by-window trajectories (tests/golden/win.pt, scripts/gen_golden_window.py) token for token, the fast tier's
teacher-forced canvas logits stay within the fast tier's existing bounds of the exact tier's, and a canvas equal to the grid is sample()
itself."""
import pytest
import torch

from oracle import synth
from oracle.zoo import AR_ZOO
from tests import window_oracle as WO
from tests.fp8_helpers import dequantised_copy
from tests.helpers import CodebookAux, build_ar, noise_tensor
from tests.test_gpu_cfg import TIERS, _run
from tests.test_gpu_fast import _with_env

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
DEV = "cuda"


def _fixture(name, golden, layouts):
    fx = golden("win")
    P = fx["plan"]
    E, nh, nb_, nhl, V, bs, vc, cl = AR_ZOO[name]
    model, _ = build_ar(name, layouts, P["weight_seed"])
    aux = CodebookAux(synth.randn_seeded((V, 256), P["codebook_seed"]).to(DEV))
    B = P["B"]
    cond = synth.randint_seeded(0, vc, (B, cl), P["cond_seed"]).to(DEV)
    uncond = synth.randint_seeded(0, vc, (B, cl), P["uncond_seed"]).to(DEV)
    return P, fx["ar"][name]["runs"], model, aux, cond, uncond, bs, V


def _sample(model, aux, cond, partial, keep_mask=None, start=(0, 0), noise=False, amp=False, k=64, p=0.9, guidance=None, force=None,
            logits=True):
    keep = None if keep_mask is None else model._keep_mask(keep_mask, partial.shape[0], start, canvas=tuple(partial.shape[1:3]))
    return model._native_sample(partial, aux, cond, start, 1.0, k, p, amp, noise=noise, return_logits=logits, force_codes=force,
                                guidance=guidance, keep=keep)


def _run_inputs(r, P, bs, V):
    canvas = tuple(r["canvas"])
    B, D = P["B"], bs[2]
    partial = WO.partial_of(B, canvas, D, V).to(DEV)
    keep = WO.mask_of(r["mask"], B, canvas, D)
    return canvas, partial, None if keep is None else keep.to(DEV)


@pytest.mark.parametrize("name", ["tiny", "tiny_txt"])
def test_exact_tier_matches_reference(golden, layouts, name):
    """fp32 tier, the reference's injected noise: every case of win.pt (canvases 4x8, 8x4, 7x9, 10x10 and 5x7 with an odd window,
    outpainting, a start_loc resume, guidance, and the grid itself) equals the reference's codes token for token"""
    P, runs, model, aux, cond, uncond, bs, V = _fixture(name, golden, layouts)
    model.precision = "exact"
    B, D = P["B"], bs[2]
    for r in runs:
        canvas, partial, keep = _run_inputs(r, P, bs, V)
        start = tuple(r["start_loc"])
        n_tok = (canvas[0] * canvas[1] - start[0] * canvas[1] - start[1]) * D
        noise = noise_tensor(r["noise_seed"], n_tok, B, V)
        g = None if r["scale"] is None else (r["scale"], uncond)
        codes, _ = _sample(model, aux, cond, partial, keep, start, noise, guidance=g, k=P["setting"]["top_k"], p=P["setting"]["top_p"])
        assert codes.shape == (B, *canvas, D)
        assert torch.equal(codes.cpu().to(torch.int16), r["codes"]), (name, canvas, r["mask"], start, r["scale"])
        if keep is not None:
            assert torch.equal(codes[keep], partial[keep])
    model.precision = None


@pytest.mark.parametrize("fmt", ["fp16", "fp8"])
@pytest.mark.parametrize("name", ["tiny", "tiny_txt"])
def test_fast_tier_logits_vs_exact_on_reference_cases(golden, layouts, name, fmt):
    """teacher-forced on the reference's canvas trajectories: the fast tier's logits at every sampled token (its prefills of every
    window's prefix and batched appends included) within the fast tier's existing bounds of the exact tier's (E4M3 against its
    dequantised model), in units of the logits' std; no greedy flip outside the fp32 decision margin; free-running codes differ from
    the exact tier's only where the fp32 decision margin allows"""
    P, runs, model, aux, cond, uncond, bs, V = _fixture(name, golden, layouts)
    ref_model = dequantised_copy(model) if fmt == "fp8" else model
    rms_k, max_k = 0.005, 0.0375
    B, D = P["B"], bs[2]
    for r in runs:
        canvas, partial, keep = _run_inputs(r, P, bs, V)
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
        ev = torch.ones(canvas[0] * canvas[1], dtype=torch.bool, device=DEV)
        if keep is not None:
            ev = (~keep).reshape(B, -1, D).any(2).any(0)
        ev = ev.repeat_interleave(D)[(start[0] * canvas[1] + start[1]) * D:]
        l32, l16 = lg32[ev], lg16[ev]
        std = float(l32.std())
        err = (l16 - l32).abs()
        print("%s %s %s %s: rms %.2e max %.2e (std %.3f)" % (name, fmt, canvas, r["mask"], float(err.pow(2).mean().sqrt()),
                                                              float(err.max()), std))
        assert float(err.pow(2).mean().sqrt()) < rms_k * std and float(err.max()) < max_k * std, (canvas, r["mask"])
        top2 = l32.topk(2, dim=-1).values
        outside = (l16.argmax(-1) != l32.argmax(-1)) & (top2[..., 0] - top2[..., 1] > 2 * err.amax(-1))
        assert int(outside.sum()) == 0, (canvas, r["mask"])
        if g is None and start == (0, 0):
            # free-running greedy on the fast tier against the exact tier's teacher-forced logits of that same trajectory: every code is
            # the exact tier's argmax unless its top-2 gap is within the logits' error there
            model.precision = "fast"
            f16 = _with_env(model, {"RQB200_FAST_DTYPE": fmt}, lambda: _sample(model, aux, cond, partial, keep, amp=True, k=1, p=None,
                                                                               logits=False))
            ref_model.precision = "exact"
            _, lf = _sample(ref_model, aux, cond, partial, keep, force=f16, k=1, p=None)
            model.precision = "fast"                                   # (for fp16, ref_model is model)
            _, lf16 = _with_env(model, {"RQB200_FAST_DTYPE": fmt}, lambda: _sample(model, aux, cond, partial, keep, amp=True, force=f16,
                                                                                   k=1, p=None))
            model.precision = ref_model.precision = None
            toks = f16.reshape(B, -1).t()                              # [n_tok, B], token-major like the logits
            ev_all = torch.ones_like(toks, dtype=torch.bool) if keep is None else ~keep.reshape(B, -1).t()
            top2 = lf.topk(2, dim=-1).values
            gap = top2[..., 0] - top2[..., 1]
            e = (lf16 - lf).abs().amax(-1)
            flip = (toks != lf.argmax(-1)) & ev_all & (gap > 2 * e)
            assert int(flip.sum()) == 0, (canvas, r["mask"])


@pytest.mark.parametrize("tier", list(TIERS))
def test_grid_canvas_is_sample(layouts, tier):
    """a canvas equal to the grid through the public sample() gives the codes and the launch count of the unmasked native call, and of
    the masked call with a mask that keeps nothing (one segment at origin (0, 0): the grid graphs and today's launches)"""
    E, nh, nb_, nhl, V, bs, vc, cl = AR_ZOO["tiny"]
    model, _ = build_ar("tiny", layouts, WO.PLAN["weight_seed"])
    aux = CodebookAux(synth.randn_seeded((V, 256), 12).to(DEV))
    B, H, W, D = 3, *bs
    cond = synth.randint_seeded(0, vc, (B, cl), 61).to(DEV)
    grid = WO.partial_of(B, (H, W), D, V, seed=62).to(DEV)
    none = torch.zeros(B, H, W, D, dtype=torch.bool, device=DEV)

    def go(amp):
        torch.manual_seed(5)
        a = model.sample(grid, model_aux=aux, cond=cond, top_k=64, top_p=0.9, amp=amp)
        la = model.last_launches
        torch.manual_seed(5)
        b = model.sample(grid, model_aux=aux, cond=cond, top_k=64, top_p=0.9, amp=amp, keep_mask=none)
        lb = model.last_launches
        noise = noise_tensor(64, H * W * D, B, V)
        c = _sample(model, aux, cond, grid, noise=noise, amp=amp, logits=False)
        lc = model.last_launches
        d = model._native_sample(grid, aux, cond, (0, 0), 1.0, 64, 0.9, amp, noise=noise)
        return a, la, b, lb, c, lc, d, model.last_launches
    a, la, b, lb, c, lc, d, ld = _run(model, tier, go)
    assert torch.equal(a, b) and la == lb, (la, lb)
    assert torch.equal(c, d) and lc == ld == la, (lc, ld, la)


def test_fast_tier_chunks_match_per_chunk_calls(layouts):
    """B = 300 images on a 6 x 7 canvas on the fast tier (two chunks of 150) == each chunk run alone"""
    model, _ = build_ar("tiny", layouts, WO.PLAN["weight_seed"])
    E, nh, nb_, nhl, V, bs, vc, cl = AR_ZOO["tiny"]
    aux = CodebookAux(synth.randn_seeded((V, 256), 12).to(DEV))
    B, canvas, D = 300, (6, 7), bs[2]
    cond = synth.randint_seeded(0, vc, (B, cl), 65).to(DEV)
    partial = WO.partial_of(B, canvas, D, V, seed=66).to(DEV)
    q = noise_tensor(67, canvas[0] * canvas[1] * D, B, V)
    model.precision = "fast"
    whole = _sample(model, aux, cond, partial, noise=q, amp=True, k=100, logits=False)
    for lo in (0, 150):
        sl = slice(lo, lo + 150)
        piece = _sample(model, aux, cond[sl], partial[sl], noise=q[:, sl].contiguous(), amp=True, k=100, logits=False)
        assert torch.equal(piece, whole[sl]), lo
    model.precision = None


@pytest.mark.parametrize("tier", ["exact", "fp16", "fp8"])
def test_all_kept_canvas_returns_partial_without_launches(layouts, tier):
    model, _ = build_ar("tiny", layouts, WO.PLAN["weight_seed"])
    E, nh, nb_, nhl, V, bs, vc, cl = AR_ZOO["tiny"]
    aux = CodebookAux(synth.randn_seeded((V, 256), 12).to(DEV))
    B = 4
    cond = synth.randint_seeded(0, vc, (B, cl), 68).to(DEV)
    partial = WO.partial_of(B, (7, 9), bs[2], V, seed=69).to(DEV)
    everything = torch.ones(1, 1, 1, 1, dtype=torch.bool, device=DEV)

    def go(amp):
        out = model.sample(partial, model_aux=aux, cond=cond, top_k=64, amp=amp, keep_mask=everything)
        return out, model.last_launches
    out, launches = _run(model, tier, go)
    assert torch.equal(out, partial) and out.data_ptr() != partial.data_ptr() and launches == 0


@pytest.mark.parametrize("tier", ["exact", "fp16"])
def test_spans_give_the_codes_of_one_span(layouts, tier):
    """public API drawing its own noise on an outpainting canvas: a noise budget of two positions (spans that end inside segments and
    at their edges) gives the codes of one span bit for bit"""
    model, _ = build_ar("tiny", layouts, WO.PLAN["weight_seed"])
    E, nh, nb_, nhl, V, bs, vc, cl = AR_ZOO["tiny"]
    D = bs[2]
    aux = CodebookAux(synth.randn_seeded((V, 256), 12).to(DEV))
    B, canvas = 3, (5, 9)
    cond = synth.randint_seeded(0, vc, (B, cl), 70).to(DEV)
    partial = WO.partial_of(B, canvas, D, V, seed=71).to(DEV)
    keep = torch.zeros(*canvas, 1, dtype=torch.bool, device=DEV)
    keep[:, :4] = True

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
    assert torch.equal(one[:, :, :4], partial[:, :, :4])


def test_in1400m_16x16_canvas_fast_vs_exact(layouts):
    """the in1400m shape (8x8x4 grid, V = 16384) on a 16x16 canvas, synthetic weights, B = 4, teacher-forced on seeded codes: the fast
    tier's logits of all 1024 canvas tokens (144 window prefills) against the exact tier's within the fast tier's bounds"""
    E, nh, nb_, nhl, V, bs, vc, cl = AR_ZOO["in1400m"]
    model, _ = build_ar("in1400m", layouts, 11)
    aux = CodebookAux(synth.randn_seeded((V, 256), 12).to(DEV))
    B, canvas, D = 4, (16, 16), bs[2]
    cond = synth.randint_seeded(0, vc, (B, cl), 72).to(DEV)
    codes = WO.partial_of(B, canvas, D, V, seed=73).to(DEV)
    model.precision = "exact"
    c32, lg32 = _sample(model, aux, cond, codes, force=codes, k=1024, p=None)
    model.precision = "fast"
    c16, lg16 = _sample(model, aux, cond, codes, amp=True, force=codes, k=1024, p=None)
    model.precision = None
    assert torch.equal(c32, codes) and torch.equal(c16, codes)
    std = float(lg32.std())
    err = (lg16 - lg32).abs()
    print("in1400m 16x16: rms %.2e max %.2e (std %.3f)" % (float(err.pow(2).mean().sqrt()), float(err.max()), std))
    assert float(err.pow(2).mean().sqrt()) < 0.005 * std and float(err.max()) < 0.0375 * std
