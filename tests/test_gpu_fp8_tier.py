"""FP8 (E4M3) tier of the fast AR engine (RQB200_FAST_DTYPE=fp8): every streamed weight is E4M3 with one fp32 scale per output row,
activations and the KV cache fp16, accumulation fp32.  FP8 changes the model, so the gate is against the DEQUANTISED model -- the
same module with every streamed weight replaced by q * s in fp32 -- on the exact tier.  Each E4M3 x fp16 product is exact in fp32,
so the FP8 tier may differ from that reference only the way the fp16 tier differs from fp32: the fp16 tier's bounds apply.  How far
FP8 moves the logits from the original weights is printed, not gated (synthetic weights say nothing about a trained checkpoint)."""
import ctypes as C
import gc
import os

import pytest
import torch

from oracle import rq_oracle as O
from oracle import synth
from oracle.zoo import AR_ZOO
from rqvae import _native as N
from tests import variants_oracle as VO
from tests.fp8_helpers import dequantised_copy, packed_bytes, streamed_weights
from tests.helpers import noise_tensor
from tests.test_gpu_fast import _case as _zoo_case
from tests.test_gpu_fast import _with_env
from tests.test_gpu_long import _case as _long_case
from tests.test_gpu_variants import aux_for, build as build_variant, cond_of

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
DEV = "cuda"
FP8 = {"RQB200_FAST_DTYPE": "fp8"}


def _free():
    gc.collect()
    torch.cuda.empty_cache()


def _teacher_forced(model, aux, cond, codes, amp):
    out, lg = model._native_sample(codes, aux, cond, (0, 0), 1.0, None, None, amp, noise=False, return_logits=True, force_codes=codes)
    assert torch.equal(out, codes)
    return lg


def _stats(ref, got):
    err = (got - ref).abs()
    top2 = ref.topk(2, dim=-1).values
    differ = got.argmax(-1) != ref.argmax(-1)
    outside = differ & (top2[..., 0] - top2[..., 1] > 2 * err.amax(-1))
    return dict(std=float(ref.std()), rms=float(err.pow(2).mean().sqrt()), max=float(err.max()), flips=int(differ.sum()),
                outside=int(outside.sum()), n=differ.numel())


def fp8_parity(label, model, aux, cond, codes):
    """fast_tier_parity_stats' protocol (teacher-forced on a reference trajectory) with the FP8 tier against the exact tier on the
    dequantised model; the distance to the original weights' exact logits is printed beside it"""
    dq = dequantised_copy(model)
    dq.precision = "exact"
    lg_dq = _teacher_forced(dq, aux, cond, codes, False)
    del dq
    _free()
    model.precision = "exact"
    lg32 = _teacher_forced(model, aux, cond, codes, False)
    model._invalidate_native()
    model.precision = "fast"
    lg8 = _with_env(model, FP8, lambda: _teacher_forced(model, aux, cond, codes, True))
    r, o = _stats(lg_dq, lg8), _stats(lg32, lg8)
    print("%s fp8: vs dequantised exact: std %.3f rms %.5f max %.5f, %d / %d greedy flips, %d outside the margin | vs original "
          "weights (reported): rms %.5f max %.5f (%.4f / %.4f std), %d greedy flips"
          % (label, r["std"], r["rms"], r["max"], r["flips"], r["n"], r["outside"], o["rms"], o["max"], o["rms"] / o["std"],
             o["max"] / o["std"], o["flips"]))
    model.precision = None
    del lg_dq, lg32, lg8
    _free()
    return r


def _gate(r):
    assert r["rms"] < 0.005 * r["std"] and r["max"] < 0.0375 * r["std"], r
    assert r["outside"] == 0, "index flip outside the arithmetic error bound"


@pytest.mark.parametrize("name", ["tiny", "tiny_txt", "ffhq355m", "in1400m", "cc3m654m", "t2i3900m"])
def test_fp8_teacher_forced_step_parity(golden, layouts, name):
    g, model, aux, cond, bs, V = _zoo_case(name, golden, layouts)
    _gate(fp8_parity(name, model, aux, cond, g["runs"][-1]["codes"].long().to(DEV)))


@pytest.mark.parametrize("name", ["long32", "headless16"])
def test_fp8_teacher_forced_step_parity_long_and_headless(golden, name):
    g, shape, model, aux, cond, bs, V = _long_case(name, golden)
    _gate(fp8_parity(name, model, aux, cond, g["runs"][-1]["codes"].long().to(DEV)))


@pytest.mark.parametrize("name", [VO.combo_name(f) for f in VO.COMBOS])
def test_fp8_teacher_forced_step_parity_embedding_variants(golden, name):
    rec = golden("arv")["combos"][name]
    model, _ = build_variant(VO.TINY, rec["flags"])
    _gate(fp8_parity(name, model, aux_for(rec["flags"]), cond_of(VO.TINY), rec["runs"][1]["codes"].long().to(DEV)))


def _forward_vs_replay(model, aux, cond, codes):
    def run():
        out = model(codes, model_aux=aux, cond=cond, amp=True)
        fwd, cl = out if isinstance(out, tuple) else (out, None)
        seq = _teacher_forced(model, aux, cond, codes, True)
        return fwd, cl, seq
    model.precision = "fast"
    fwd, cond_logits, seq = _with_env(model, FP8, run)
    B, H, W, D = codes.shape
    seq = seq.reshape(H, W, D, B, -1).permute(3, 0, 1, 2, 4)
    std = float(seq.std())
    d = float((fwd - seq).abs().max())
    return d, std, cond_logits


@pytest.mark.parametrize("name", ["tiny", "tiny_txt", "cc3m654m"])
def test_fp8_batched_forward(golden, layouts, name):
    """forward(amp=True) on FP8 (every large-M pass on the FP8 streamer's 128-row chunks) against the FP8 sequential replay; the
    cond_classifier's logits against the oracle's forward of the dequantised weights"""
    g, model, aux, cond, bs, V = _zoo_case(name, golden, layouts)
    E, nh, nb_, nhl, V_, bs_, vc, cl = AR_ZOO[name]
    codes = g["runs"][-1]["codes"].long().to(DEV)
    d, std, cond_logits = _forward_vs_replay(model, aux, cond, codes)
    print("%s fp8: batched forward vs sequential replay: max logit difference %.2e (std %.3f)" % (name, d, std))
    assert d < 0.02 * std
    if cl > 1:
        dq = dequantised_copy(model)
        sd = {k: v.cpu() for k, v in dq.state_dict().items()}
        del dq
        _free()
        _, cref = O.ar_forward(sd, O.ArConfig(E, nh, nb_, nhl, V_, bs_, vc, cl), codes.cpu(), aux.quantizer._shared_table().cpu(),
                               cond.cpu(), with_cond_logits=True)
        e = float((cond_logits.cpu() - cref).abs().max())
        print("%s fp8: cond_logits vs oracle on the dequantised weights: max error %.2e (std %.3f)" % (name, e, float(cref.std())))
        assert cond_logits.shape == (codes.shape[0], cl - 1, vc) and e < 0.04 * float(cref.std())


def test_fp8_batched_forward_per_depth_classifier_and_cond_logits():
    """the reference's all-false default on the text-shaped model: per-depth classifiers (each depth's own [V,E] E4M3 slice and
    scales) and the zero-padded cond classifier (padding rows s = 1, q = 0)"""
    E, nh, nb, nhl, V, bs, vc, cl = VO.TEXT
    model, sd = build_variant(VO.TEXT, VO.ALL_FALSE)
    xs = synth.randint_seeded(0, V, (3, *bs), 44).to(DEV)
    cond = synth.randint_seeded(0, vc, (3, cl), 45).to(DEV)
    d, std, cond_logits = _forward_vs_replay(model, None, cond, xs)
    assert d < 0.02 * std, (d, std)
    dq = dequantised_copy(model)
    dsd = {k: v.cpu() for k, v in dq.state_dict().items()}
    _, ref_c = VO.ar_forward(dsd, O.ArConfig(E, nh, nb, nhl, V, bs, vc, cl), VO.ALL_FALSE, xs.cpu(), None, cond.cpu(), with_cond_logits=True)
    e = float((cond_logits.cpu() - ref_c).abs().max()) / float(ref_c.std())
    print("all-false text model fp8: forward vs replay %.2e (std %.3f); cond logits vs oracle %.4f std" % (d, std, e))
    assert e < 0.02


def test_fp8_free_running_consistency(golden, layouts):
    """deterministic; graph / no graph / no PDL / trace give the same codes; noise drawn span by span == one noise tensor; a
    sequential-prefill resume reproduces the trajectory bit for bit; B = 300 runs in chunks with rows independent"""
    g, model, aux, cond, bs, V = _zoo_case("tiny", golden, layouts)
    B = g["B"]
    n_tok = bs[0] * bs[1] * bs[2]
    noise = noise_tensor(77, n_tok, B, V)
    part = torch.zeros(B, *bs, dtype=torch.long, device=DEV)
    model.precision = "fast"

    def sample(start=(0, 0), src=part, nz=noise, c=cond, **kw):
        return model._native_sample(src, aux, c, start, 1.0, 100, 0.95, True, noise=nz, **kw)

    def fp8(fn, **extra):
        return _with_env(model, dict(FP8, **extra), fn)

    a = fp8(lambda: (sample(), sample()))
    assert torch.equal(a[0], a[1]), "FP8 tier is not run-to-run deterministic"
    a = a[0]
    assert int(a.min()) >= 0 and int(a.max()) < V
    for var in ("RQB200_NO_GRAPH", "RQB200_NO_PDL", "RQB200_TRACE"):
        assert torch.equal(fp8(sample, **{var: "1"}), a), var
    h0, w0 = bs[0] // 2, 1
    skip = (h0 * bs[1] + w0) * bs[2]
    c = fp8(lambda: sample((h0, w0), a, noise[skip:].contiguous()), RQB200_SEQ_PREFILL="1")
    assert torch.equal(c, a), "sequential-prefill resume must reproduce the trajectory bit for bit"
    cb = fp8(lambda: sample((h0, w0), a, noise[skip:].contiguous()))
    assert torch.equal(cb.flatten(1)[:, :skip], a.flatten(1)[:, :skip])

    torch.manual_seed(4321)
    full = torch.empty(n_tok, B, V, device=DEV)
    for t in range(n_tok):
        full[t].exponential_(1)

    def spans():
        want = sample(nz=full)
        got = []
        for budget in (1, 3 * 4 * B * V * 4):
            model.noise_budget_bytes = budget
            torch.manual_seed(4321)
            got.append(sample(nz=None))
        model.noise_budget_bytes = 256 << 20
        return want, got
    want, got = fp8(spans)
    for x in got:
        assert torch.equal(x, want)

    Bl = 300
    nl = torch.empty(n_tok, Bl, V, device=DEV).exponential_(1, generator=torch.Generator(DEV).manual_seed(3))
    cl = torch.randint(0, 10, (Bl, 1), device=DEV)
    pl = torch.zeros(Bl, *bs, dtype=torch.long, device=DEV)
    full_b, sub = fp8(lambda: (sample(src=pl, nz=nl, c=cl), sample(src=pl[140:160], nz=nl[:, 140:160].contiguous(), c=cl[140:160])))
    assert torch.equal(full_b[140:160], sub)


@pytest.mark.parametrize("name", ["tiny_txt", "in1400m"])
def test_fp8_engine_keeps_packed_weights_only(golden, layouts, name):
    """kept bytes = sum of N*K + 4N over the streamed weights + the fp32 small tensors, no 16-bit copy; the device memory the build
    allocates is no more than that"""
    g, model, aux, cond, bs, V = _zoo_case(name, golden, layouts)
    model.precision = "fast"
    model._invalidate_native()
    _free()
    before = torch.cuda.memory_stats()["requested_bytes.all.current"]      # (bytes requested: no allocator rounding)
    os.environ.update(FP8)
    try:
        model._engine(aux.quantizer._shared_table(), N.MODE_FAST)
    finally:
        del os.environ["RQB200_FAST_DTYPE"]
    grown = torch.cuda.memory_stats()["requested_bytes.all.current"] - before
    held = model.native_weight_bytes()
    kept = [t for e in model._eng.values() for t in e["keep"] if isinstance(t, torch.Tensor)]
    snames = {n + ".weight" for n, _ in streamed_weights(model)}
    small = sum(4 * p.numel() for n, p in model.named_parameters() if n not in snames) + 4 * aux.quantizer._shared_table().numel()
    if model.block_size_cond > 1:
        small += 4 * (-model.vocab_size_cond % 128)             # the cond classifier's bias, zero-padded to 128 rows
    print("%s fp8 engine: streamed %.1f MB (fp16 would be %.1f MB), fp32 %.1f MB, device memory grown by %.1f MB"
          % (name, held["streamed"] / 1e6, sum(2 * w.numel() for _, w in streamed_weights(model)) / 1e6, held["fp32"] / 1e6, grown / 1e6))
    assert held["streamed"] == packed_bytes(model)
    assert held["fp32"] == small
    assert not any(t.dtype in (torch.float16, torch.bfloat16) for t in kept)
    assert grown <= held["streamed"] + held["fp32"], (grown, held)
    model._invalidate_native()


def test_fp8_refusals(golden, layouts):
    """rqb200_ar_create refuses E4M3 on the exact tier, a missing scale and a misaligned packed pointer (NULL + message);
    precision = 'exact' ignores RQB200_FAST_DTYPE=fp8"""
    g, model, aux, cond, bs, V = _zoo_case("tiny_txt", golden, layouts)
    L = N.lib()
    cb = aux.quantizer._shared_table()
    os.environ.update(FP8)
    try:
        cfg, w, keep, _ = model._engine_structs(cb, N.MODE_FAST)
    finally:
        del os.environ["RQB200_FAST_DTYPE"]

    def create():
        h = L.rqb200_ar_create(C.byref(cfg), C.byref(w))
        if h:
            L.rqb200_ar_destroy(h)
            return None
        return L.rqb200_last_error().decode()

    assert create() is None                                          # the unmodified structs are accepted
    cfg.mode = N.MODE_EXACT
    assert "fast-tier" in create()
    cfg.mode = N.MODE_FAST
    for field in ("s_cls", "s_in", "s_head", "s_ccls"):
        saved = getattr(w, field)
        setattr(w, field, None)
        msg = create()
        assert msg is not None and field in msg, (field, msg)
        setattr(w, field, saved)
    saved = w.body[1].s1
    w.body[1].s1 = None
    assert "body block" in create()
    w.body[1].s1 = saved
    saved = w.head[0].sqkv
    w.head[0].sqkv = None
    assert "head block" in create()
    w.head[0].sqkv = saved
    saved = w.w_cls
    w.w_cls = saved + 8                                              # 8-byte aligned, not 16
    assert "16-byte" in create()
    w.w_cls = saved
    saved = w.body[0].w2
    w.body[0].w2 = saved + 1
    assert "16-byte" in create()
    w.body[0].w2 = saved
    assert create() is None
    # the exact tier ignores the FP8 switch: fp32 weights, the same codes
    n_tok = bs[0] * bs[1] * bs[2]
    noise = noise_tensor(5, n_tok, g["B"], V)
    z = torch.zeros(g["B"], *bs, dtype=torch.long, device=DEV)
    model.precision = "exact"
    want = model._native_sample(z, aux, cond, (0, 0), 1.0, 100, 0.95, False, noise=noise)

    def run():
        got = model._native_sample(z, aux, cond, (0, 0), 1.0, 100, 0.95, False, noise=noise)
        return got, [e["weight_dtype"] for e in model._eng.values()]
    got, dts = _with_env(model, FP8, run)
    assert dts == [N.F32] and torch.equal(got, want)
    model.precision = None
