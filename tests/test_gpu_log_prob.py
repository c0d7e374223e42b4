"""GPU: teacher-forced log-likelihoods (RQTransformer.log_prob, rqb200_ar_log_prob) and the row-wise log-softmax gather behind them
(rqb200_dbg_log_prob_rows).  log_prob must equal the log-softmax of forward's logits gathered at the codes on each tier, the exact tier
must match the logits the unmodified reference stored in the golden fixtures, the fast tier must stay near the exact one, its memory
must not grow with the logits, and its results must be deterministic and independent of the batch they were computed in."""
import contextlib
import gc

import pytest
import torch

from oracle import synth
from rqvae import _native as N
from rqvae.models import create_model
from tests import depthwise_oracle as DO
from tests import variants_oracle as VO
from tests.fp8_helpers import dequantised_copy
from tests.helpers import CodebookAux
from tests.test_gpu_depthwise import TablesAux, _ar_config
from tests.test_gpu_fast import _case as _zoo_case
from tests.test_gpu_fast import _with_env
from tests.test_gpu_long import _case as _long_case
from tests.test_gpu_variants import aux_for, build as build_variant, cond_of

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
DEV = "cuda"
ENV = {"fp16": {}, "bf16": {"RQB200_FAST_DTYPE": "bf16"}, "fp8": {"RQB200_FAST_DTYPE": "fp8"}}


def _free():
    gc.collect()
    torch.cuda.empty_cache()


def _ref_lp(logits, idx):
    """fp64 log-softmax of logits [..., V] gathered at idx [...], and the logsumexp"""
    lg = logits.double()
    return torch.log_softmax(lg, -1).gather(-1, idx[..., None].long()).squeeze(-1), torch.logsumexp(lg, -1)


def _assert_kernel_tol(got, logits, idx, what=""):
    want, lse = _ref_lp(logits, idx)
    err = (got.double() - want).abs()
    tol = 1e-5 * lse.abs().clamp_min(1.0)
    assert bool((err <= tol).all()), "%s: max |dlog p| %.3g (worst tolerance ratio %.3g)" % (what, float(err.max()), float((err / tol).max()))


def _dbg_rows(lg, V, tgt):
    rows, ld = lg.shape
    out = torch.full((rows,), 123.0, device=DEV)
    N.check(N.lib().rqb200_dbg_log_prob_rows(N.ptr(lg), ld, V, rows, N.ptr(tgt), N.ptr(out), N.stream_ptr()), "dbg_log_prob_rows")
    return out


# ------------------------------------------------------------------------------------------------ 1. the reduction kernel
@pytest.mark.parametrize("V", [512, 2048, 16384])
@pytest.mark.parametrize("pad", [0, 68])
def test_kernel_matches_fp64_log_softmax(V, pad):
    rows = 41
    lg = synth.randn_seeded((rows, V + pad), V + pad, 3.0).to(DEV)
    lg[3, ::5] = -1e6                                   # LogitMask's value
    lg[4] *= 1e4 / 3.0                                  # entries of magnitude 1e4
    lg[5, : V // 2] = -1e6
    lg[:, V:] = float("nan")                            # beyond V: never read
    tgt = synth.randint_seeded(0, V, (rows,), 7).to(DEV)
    tgt[5] = V // 2 + 1
    got = _dbg_rows(lg, V, tgt)
    _assert_kernel_tol(got, lg[:, :V], tgt, "V=%d ld=%d" % (V, V + pad))
    assert torch.equal(got, _dbg_rows(lg, V, tgt))     # run to run


@pytest.mark.parametrize("V", [512, 16384])
def test_kernel_out_of_range_target_gives_nan_for_that_row_only(V):
    rows = 12
    lg = synth.randn_seeded((rows, V), 3, 2.0).to(DEV)
    tgt = synth.randint_seeded(0, V, (rows,), 4).to(DEV)
    good = _dbg_rows(lg, V, tgt)
    bad_tgt = tgt.clone()
    bad_tgt[4], bad_tgt[7] = -1, V
    bad = _dbg_rows(lg, V, bad_tgt)
    assert bool(bad[4].isnan()) and bool(bad[7].isnan())
    keep = torch.ones(rows, dtype=torch.bool, device=DEV)
    keep[4] = keep[7] = False
    assert torch.equal(bad[keep], good[keep])


def test_kernel_result_of_a_row_does_not_depend_on_its_neighbours():
    lg = synth.randn_seeded((300, 2048), 9, 4.0).to(DEV)
    tgt = synth.randint_seeded(0, 2048, (300,), 10).to(DEV)
    full = _dbg_rows(lg, 2048, tgt)
    part = _dbg_rows(lg[117:250].contiguous(), 2048, tgt[117:250].contiguous())
    assert torch.equal(full[117:250], part)


# ------------------------------------------------------------------------------------------------ 2. fast tier == its own forward
def _fast_vs_forward(model, aux, xs, cond, what):
    model.precision = "fast"
    out = model(xs, model_aux=aux, cond=cond, amp=True)
    lp = model.log_prob(xs, model_aux=aux, cond=cond, amp=True)
    if isinstance(out, tuple):
        (lg, clg), (lp, clp) = out, lp
        assert clp.shape == (xs.shape[0], model.block_size_cond - 1)
        _assert_kernel_tol(clp, clg, cond[:, 1:], what + " cond")
    assert lp.shape == xs.shape and lp.dtype == torch.float32
    _assert_kernel_tol(lp, out[0] if isinstance(out, tuple) else out, xs, what)


@pytest.mark.parametrize("fmt", ["fp16", "bf16", "fp8"])
@pytest.mark.parametrize("name", ["tiny", "tiny_txt", "cc3m654m", "in1400m"])
def test_fast_log_prob_equals_forward_zoo(golden, layouts, name, fmt):
    g, model, aux, cond, bs, V = _zoo_case(name, golden, layouts)
    xs = g["runs"][-1]["codes"].long().to(DEV)
    _with_env(model, ENV[fmt], lambda: _fast_vs_forward(model, aux, xs, cond, "%s %s" % (name, fmt)))
    _free()


@pytest.mark.parametrize("fmt", ["fp16", "bf16", "fp8"])
@pytest.mark.parametrize("name", [VO.combo_name(f) for f in VO.COMBOS])
def test_fast_log_prob_equals_forward_embedding_variants(golden, name, fmt):
    rec = golden("arv")["combos"][name]
    model, _ = build_variant(VO.TINY, rec["flags"])
    xs = rec["runs"][1]["codes"].long().to(DEV)
    _with_env(model, ENV[fmt], lambda: _fast_vs_forward(model, aux_for(rec["flags"]), xs, cond_of(VO.TINY), name))


def _depthwise_case():
    P = DO.AR_PLAN
    with torch.device("meta"):
        model, _ = create_model(_ar_config(*DO.AR_SHAPE))
    sd = synth.synth_state_dict(synth.shapes_of(model.state_dict()), P["weight_seed"])
    model = model.to_empty(device=DEV)
    model.load_state_dict({k: v.to(DEV) for k, v in sd.items()})
    bs, V, vc, cl = DO.AR_SHAPE[5], DO.AR_SHAPE[4], DO.AR_SHAPE[6], DO.AR_SHAPE[7]
    aux = TablesAux(DO.tables_of([V] * bs[2], P["table_seed"]))
    cond = synth.randint_seeded(0, vc, (P["B"], cl), P["cond_seed"]).to(DEV)
    return model.eval(), aux, cond


@pytest.mark.parametrize("fmt", ["fp16", "bf16", "fp8"])
def test_fast_log_prob_equals_forward_per_depth_codebooks(golden, fmt):
    model, aux, cond = _depthwise_case()
    xs = golden("rqd")["ar"]["runs"][1]["codes"].long().to(DEV)
    _with_env(model, ENV[fmt], lambda: _fast_vs_forward(model, aux, xs, cond, "rqd " + fmt))


@pytest.mark.parametrize("fmt", ["fp16", "bf16", "fp8"])
@pytest.mark.parametrize("name", ["long32", "headless16"])
def test_fast_log_prob_equals_forward_long_and_headless(golden, name, fmt):
    g, shape, model, aux, cond, bs, V = _long_case(name, golden)
    xs = g["runs"][0]["codes"].long().to(DEV)
    _with_env(model, ENV[fmt], lambda: _fast_vs_forward(model, aux, xs, cond, name + " " + fmt))
    _free()


# ------------------------------------------------------------------------------------------------ 3. exact tier
def _without_cond_classifier(model):
    """the exact tier has no cond classifier: evaluate a text model's code log-likelihoods on the module without it (the code
    log-likelihoods do not read it).  For models built by the test itself."""
    if hasattr(model, "cond_classifier"):
        del model.cond_classifier
    return model


@contextlib.contextmanager
def _no_cond_classifier(model):
    """_without_cond_classifier for the memoised zoo models: the cond classifier is put back afterwards"""
    cc = model._modules.pop("cond_classifier", None)
    try:
        yield model
    finally:
        if cc is not None:
            model.cond_classifier = cc
        model._invalidate_native()


def _exact_copy(model, dequantise):
    """a separate module with the weights of `model` (the memoised zoo models keep theirs), without the cond classifier; dequantise:
    every streamed weight replaced by the q * s the FP8 tier computes with"""
    m = dequantised_copy(model) if dequantise else None
    if m is None:
        with torch.device("meta"):
            m = type(model)(model.config)
        m = m.to_empty(device=model.pos_emb_hw.device)
        m.load_state_dict(model.state_dict())
    return _without_cond_classifier(m.eval())


def _exact_checks(model, aux, xs, cond, steps, what, repeat=True):
    """log_prob(amp=False) against forward(amp=False) (kernel tolerance) and against the reference's stored logits of `steps`
    ({token step: [B,V]}) on the trajectory xs (the exact-tier logits gate carried through both terms); repeat: and run to run"""
    model.precision = "exact"
    lp = model.log_prob(xs, model_aux=aux, cond=cond, amp=False)
    B, H, W, D = xs.shape
    _, lg = model._native_sample(xs, aux, cond, (0, 0), 1.0, None, None, False, noise=False, return_logits=True, force_codes=xs)
    lg = lg.reshape(H, W, D, B, -1).permute(3, 0, 1, 2, 4)
    _assert_kernel_tol(lp, lg, xs, what)
    flat_lp, flat_xs = lp.reshape(B, -1), xs.reshape(B, -1)
    for step, ref in steps.items():
        ref = ref.to(DEV).double()
        t = flat_xs[:, step]
        lt = ref.gather(-1, t[:, None]).squeeze(-1)
        want = lt - torch.logsumexp(ref, -1)
        err = (flat_lp[:, step].double() - want).abs()
        tol = 4e-4 + 1e-4 * (lt.abs() + torch.logsumexp(ref, -1).abs())
        assert bool((err <= tol).all()), "%s step %d: |dlog p| %.3g" % (what, step, float(err.max()))
    if repeat:
        assert torch.equal(lp, model.log_prob(xs, model_aux=aux, cond=cond, amp=False))   # run to run
    return lp


@pytest.mark.parametrize("name", ["tiny", "tiny_txt"])
def test_exact_log_prob_matches_forward_and_reference_zoo(golden, layouts, name):
    g, model, aux, cond, bs, V = _zoo_case(name, golden, layouts)
    with _no_cond_classifier(model):
        for run in g["runs"]:
            _exact_checks(model, aux, run["codes"].long().to(DEV), cond, run["logits"] or {}, name)


@pytest.mark.parametrize("name", ["cc3m654m", "cc3m654m_16", "t2i3900m"])
def test_exact_log_prob_matches_reference_text_models(golden, layouts, name):
    """the text-conditioned shapes of ar2.pt / ar3.pt, on the last trajectory with stored logits.  cc3m654m_16 at B = 2 (V = 16384,
    D = 4: 512 KB of logits per position) replays as two spans of 128 positions, and its stored step 1023 lies in the second: the
    span resume and the output offsets of a later span are checked against the reference there"""
    g, model, aux, cond, bs, V = _zoo_case(name, golden, layouts)
    run = [r for r in g["runs"] if r["logits"]][-1]
    with _no_cond_classifier(model):
        _exact_checks(model, aux, run["codes"].long().to(DEV), cond, run["logits"], name, repeat=False)
    _free()


def test_exact_log_prob_matches_reference_embedding_variants(golden):
    g = golden("arv")
    for name in [VO.combo_name(f) for f in VO.COMBOS]:
        rec = g["combos"][name]
        model, _ = build_variant(VO.TINY, rec["flags"])
        for run in rec["runs"]:
            _exact_checks(model, aux_for(rec["flags"]), run["codes"].long().to(DEV), cond_of(VO.TINY),
                          dict(zip(run["logit_steps"], run["logits"])), name)
    for key, shape in (("text", VO.TEXT), ("headless", VO.HEADLESS)):
        model, _ = build_variant(shape, VO.ALL_FALSE)
        model = _without_cond_classifier(model)
        for run in g[key]["runs"]:
            _exact_checks(model, None, run["codes"].long().to(DEV), cond_of(shape), dict(zip(run["logit_steps"], run["logits"])), key)


def test_exact_log_prob_matches_reference_per_depth_codebooks(golden):
    model, aux, cond = _depthwise_case()
    model = _without_cond_classifier(model)
    for run in golden("rqd")["ar"]["runs"]:
        _exact_checks(model, aux, run["codes"].long().to(DEV), cond, run["logits"], "rqd")


@pytest.mark.parametrize("name", ["long32", "headless16"])
def test_exact_log_prob_matches_reference_long_and_headless(golden, name):
    g, shape, model, aux, cond, bs, V = _long_case(name, golden)
    model = _without_cond_classifier(model)
    run = g["runs"][0]
    _exact_checks(model, aux, run["codes"].long().to(DEV), cond, run["logits"], name)
    _free()


def test_exact_tier_refuses_cond_log_likelihoods(golden, layouts):
    g, model, aux, cond, bs, V = _zoo_case("tiny_txt", golden, layouts)
    model.precision = "exact"
    with pytest.raises(NotImplementedError):
        model.log_prob(g["runs"][0]["codes"].long().to(DEV), model_aux=aux, cond=cond, amp=False)


# ------------------------------------------------------------------------------------------------ 4. fast vs exact
@pytest.mark.parametrize("fmt", ["fp16", "fp8"])
@pytest.mark.parametrize("name", ["tiny", "tiny_txt", "cc3m654m", "in1400m"])
def test_fast_log_prob_near_exact(golden, layouts, name, fmt):
    g, model, aux, cond, bs, V = _zoo_case(name, golden, layouts)
    xs = g["runs"][-1]["codes"].long().to(DEV)
    ref_model = _exact_copy(model, dequantise=fmt == "fp8")                   # FP8 against the dequantised exact tier
    ref_model.precision = "exact"
    lp32 = ref_model.log_prob(xs, model_aux=aux, cond=cond, amp=False)
    _, lg32 = ref_model._native_sample(xs, aux, cond, (0, 0), 1.0, None, None, False, noise=False, return_logits=True, force_codes=xs)
    std = float(lg32.std())
    del ref_model, lg32
    _free()
    model.precision = "fast"
    lp16 = _with_env(model, ENV[fmt], lambda: model.log_prob(xs, model_aux=aux, cond=cond, amp=True))
    lp16 = lp16[0] if isinstance(lp16, tuple) else lp16
    err = (lp16.double() - lp32.double()).abs()
    print("%s %s: fast vs exact log p: rms %.3g, max %.3g (logit std %.3f)" % (name, fmt, float(err.pow(2).mean().sqrt()), float(err.max()), std))
    assert float(err.max()) < 0.075 * std
    _free()


# ------------------------------------------------------------------------------------------------ 5. losses agree
@pytest.mark.parametrize("fmt", ["fp16", "fp8"])
def test_losses_agree_with_log_prob(golden, layouts, fmt):
    g, model, aux, cond, bs, V = _zoo_case("tiny_txt", golden, layouts)
    xs = g["runs"][-1]["codes"].long().to(DEV)
    model.precision = "fast"

    def run():
        return model(xs, model_aux=aux, cond=cond, amp=True), model.log_prob(xs, model_aux=aux, cond=cond, amp=True)

    (lg, clg), (lp, clp) = _with_env(model, ENV[fmt], run)
    D = bs[2]

    def close(a, b):
        assert abs(float(a) - float(b)) <= 1e-5 * abs(float(b)), (float(a), float(b))

    close(-lp.double().mean(), model.compute_loss(lg, xs))
    cb = model.compute_codebook_loss(lg, xs)
    for d in range(D):
        close(-lp.double().reshape(-1, D).mean(0)[d], cb[d])
    close(-clp.double().mean(), model.compute_cond_loss(clg, cond))


# ------------------------------------------------------------------------------------------------ 6. bounded memory
def _big_model():
    cfg = _ar_config(128, 2, 2, 2, 16384, (32, 32, 4), 1, 1)
    with torch.device("meta"):
        model, _ = create_model(cfg)
    sd = synth.synth_state_dict(synth.shapes_of(model.state_dict()), 77)
    model = model.to_empty(device=DEV)
    model.load_state_dict({k: v.to(DEV) for k, v in sd.items()})
    return model.eval()


@pytest.mark.parametrize("tier", ["fast", "exact"])
def test_log_prob_memory_is_bounded(tier):
    model = _big_model()
    model.precision = tier
    aux = CodebookAux(synth.randn_seeded((16384, 256), 78).to(DEV))
    B = 8
    xs = synth.randint_seeded(0, 16384, (B, 32, 32, 4), 79).to(DEV)
    amp = tier == "fast"
    first = model.log_prob(xs, model_aux=aux, amp=amp)                     # engine build outside the measurement
    _free()
    eng = model._engine(model._codebook_of(aux, 4), model._mode(amp))
    ws = N.lib().rqb200_ar_log_prob_workspace_bytes(eng["handle"], B)
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    lp = model.log_prob(xs, model_aux=aux, amp=amp)
    peak = torch.cuda.max_memory_allocated() - base
    logits_bytes = B * 32 * 32 * 4 * 16384 * 4
    out_bytes = lp.numel() * 4
    print("%s tier: peak increase %.1f MB, workspace %.1f MB, logits would be %.1f MB" % (tier, peak / 2**20, ws / 2**20, logits_bytes / 2**20))
    assert peak <= ws + out_bytes + (64 << 20)
    assert peak < logits_bytes / 4
    assert torch.equal(first, lp)
    lg = model(xs[:1], model_aux=aux, amp=amp)                                # (one image's logits: 268 MB)
    _assert_kernel_tol(lp[:1], lg, xs[:1], "%s 32x32x4 V=16384 B=%d" % (tier, B))
    if tier == "exact":
        # the exact tier replays in spans of 64 MB of logits: 32 spans of 32 positions at B = 8 (above), 4 of 256 positions at B = 1
        _assert_kernel_tol(model.log_prob(xs[:1], model_aux=aux, amp=False), lg, xs[:1], "exact 32x32x4 V=16384 B=1")


# ------------------------------------------------------------------------------------------------ 7. self-consistency
def test_fast_log_prob_batch_independent_and_deterministic(golden, layouts):
    g, model, aux, cond, bs, V = _zoo_case("tiny", golden, layouts)
    model.precision = "fast"
    xs = synth.randint_seeded(0, V, (300, *bs), 81).to(DEV)
    full = model.log_prob(xs, model_aux=aux, amp=True)
    assert torch.equal(full, model.log_prob(xs, model_aux=aux, amp=True))
    halves = torch.cat([model.log_prob(xs[:150], model_aux=aux, amp=True), model.log_prob(xs[150:], model_aux=aux, amp=True)])
    assert torch.equal(full, halves)


@pytest.mark.parametrize("amp", [True, False])
def test_out_of_range_codes_raise_before_any_kernel(golden, layouts, amp):
    g, model, aux, cond, bs, V = _zoo_case("tiny", golden, layouts)
    xs = g["runs"][0]["codes"].long().to(DEV)
    model.log_prob(xs, model_aux=aux, amp=amp)                              # (engine built)
    for bad in (-1, V):
        ys = xs.clone()
        ys[1, 2, 3, 1] = bad
        before = N.launch_count["total"]
        with pytest.raises(ValueError):
            model.log_prob(ys, model_aux=aux, amp=amp)
        assert N.launch_count["total"] == before
