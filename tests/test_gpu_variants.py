"""GPU: RQ-Transformers under every combination of the five embedding / classifier switches (tests/variants_oracle.py) on both
tiers -- exact-tier codes bit-exact against the reference's trajectories (tests/golden/arv.pt), fast-tier logits against the exact
tier and the reference, the batched forward against the oracle, and the per-depth classifier at production widths."""
import os

import pytest
import torch

from oracle import rq_oracle as O
from oracle import synth
from tests import variants_oracle as VO
from tests.helpers import CodebookAux, noise_tensor
from tests.test_oracle_variants import make_variant

pytestmark = pytest.mark.gpu
DEV = "cuda"
torch.set_grad_enabled(False)
NAMES = [VO.combo_name(f) for f in VO.COMBOS]


def build(shape, flags, seed=VO.PLAN["weight_seed"]):
    m = make_variant(shape, flags, "meta")
    sd = VO.state_dict_of(synth.shapes_of(m.state_dict()), seed)
    m = m.to_empty(device=DEV)
    m.load_state_dict({k: v.to(DEV) for k, v in sd.items()})
    return m.eval(), sd


def aux_for(flags):
    return CodebookAux(synth.randn_seeded((VO.TINY[4], 256), VO.PLAN["table_seed"]).to(DEV)) if VO.needs_codebook(flags) else None


def cond_of(shape, B=VO.PLAN["B"]):
    return synth.randint_seeded(0, shape[6], (B, shape[7]), VO.PLAN["cond_seed"]).to(DEV)


class env:
    """fast-tier engine options read from the environment at engine build"""

    def __init__(self, model, **kv):
        self.model, self.kv = model, kv

    def __enter__(self):
        os.environ.update(self.kv)
        self.model._invalidate_native()

    def __exit__(self, *a):
        for k in self.kv:
            del os.environ[k]
        self.model._invalidate_native()


def exact_runs(model, shape, runs, aux):
    bs, B = shape[5], VO.PLAN["B"]
    n_tok = bs[0] * bs[1] * bs[2]
    model.precision = "exact"
    for run in runs:
        st = run["setting"]
        codes, logits = model._native_sample(torch.zeros(B, *bs, dtype=torch.long, device=DEV), aux, cond_of(shape), (0, 0), 1.0,
                                             st.get("top_k"), st.get("top_p"), False,
                                             noise=noise_tensor(run["noise_seed"], n_tok, B, shape[4]), return_logits=True)
        for s, lg in zip(run["logit_steps"], run["logits"]):
            torch.testing.assert_close(logits[s].cpu(), lg, rtol=1e-4, atol=2e-4)
        d = (codes.cpu() != run["codes"].long()).flatten(1).any(0).nonzero()
        assert len(d) == 0, "%s: first divergent token %d of %d" % (st, int(d[0]), n_tok)


@pytest.mark.parametrize("name", NAMES)
def test_exact_tier_codes_match_reference(golden, name):
    rec = golden("arv")["combos"][name]
    model, _ = build(VO.TINY, rec["flags"])
    exact_runs(model, VO.TINY, rec["runs"], aux_for(rec["flags"]))


def test_exact_tier_text_resume_and_headless(golden):
    g = golden("arv")
    model, _ = build(VO.TEXT, VO.ALL_FALSE)
    exact_runs(model, VO.TEXT, g["text"]["runs"], None)
    rs, st = VO.PLAN["resume"], VO.PLAN["settings"][1]
    bs = VO.TEXT[5]
    codes2 = model._native_sample(g["text"]["runs"][1]["codes"].long().to(DEV), None, cond_of(VO.TEXT), rs["start_loc"], 1.0,
                                  st["top_k"], st["top_p"], False,
                                  noise=noise_tensor(rs["noise_seed"], bs[0] * bs[1] * bs[2], VO.PLAN["B"], VO.TEXT[4]))
    assert torch.equal(codes2.cpu(), g["text"]["resume"]["codes"].long())
    model, _ = build(VO.HEADLESS, VO.ALL_FALSE)
    exact_runs(model, VO.HEADLESS, g["headless"]["runs"], None)


def teacher_forced(model, aux, xs, cond, amp):
    _, lg = model._native_sample(xs, aux, cond, (0, 0), 1.0, None, None, amp, noise=False, return_logits=True, force_codes=xs)
    return lg


def greedy_flips(ref, got, bound):
    """argmax disagreements where the fp32 logits' top-2 margin exceeds the error bound (flips inside it are allowed)"""
    top2 = ref.topk(2, dim=-1).values
    margin = top2[..., 0] - top2[..., 1]
    return int(((ref.argmax(-1) != got.argmax(-1)) & (margin > 2 * bound)).sum())


@pytest.mark.parametrize("dt", ["fp16", "bf16"])
@pytest.mark.parametrize("name", NAMES)
def test_fast_tier_logits_match_exact_tier_and_reference(golden, name, dt):
    rec = golden("arv")["combos"][name]
    model, _ = build(VO.TINY, rec["flags"])
    aux = aux_for(rec["flags"])
    run = rec["runs"][1]
    xs, cond = run["codes"].long().to(DEV), cond_of(VO.TINY)
    model.precision = "exact"
    ex = teacher_forced(model, aux, xs, cond, False)
    model.precision = "fast"
    with env(model, RQB200_FAST_DTYPE=dt):
        fa = teacher_forced(model, aux, xs, cond, True)
    sig = float(ex.std())
    err = float((fa - ex).abs().max()) / sig
    bound = (0.02 if dt == "fp16" else 0.06) * sig
    print("%s %s: fast vs exact %.4f sigma" % (name, dt, err))
    assert err < bound / sig
    assert greedy_flips(ex, fa, bound) == 0
    for s, lg in zip(run["logit_steps"], run["logits"]):
        assert float((fa[s].cpu() - lg).abs().max()) < bound


def test_fast_forward_matches_oracle_with_cond_logits():
    """forward(amp=True) of every variant on the text-shaped model, cond logits included, against the oracle"""
    E, nh, nb, nhl, V, bs, vc, cl = VO.TEXT
    cfg = O.ArConfig(E, nh, nb, nhl, V, bs, vc, cl)
    xs = synth.randint_seeded(0, V, (3, *bs), 44)
    cond = synth.randint_seeded(0, vc, (3, cl), 45)
    table = synth.randn_seeded((V, 256), VO.PLAN["table_seed"])
    for flags in VO.COMBOS:
        model, sd = build(VO.TEXT, flags)
        need = VO.needs_codebook(flags)
        ref, ref_c = VO.ar_forward(sd, cfg, flags, xs, table if need else None, cond, with_cond_logits=True)
        got, got_c = model(xs.to(DEV), model_aux=CodebookAux(table.to(DEV)) if need else None, cond=cond.to(DEV), amp=True)
        err = float((got.cpu() - ref).abs().max()) / float(ref.std())
        err_c = float((got_c.cpu() - ref_c).abs().max()) / float(ref_c.std())
        assert err < 0.02 and err_c < 0.02, (VO.combo_name(flags), err, err_c)


def test_sample_without_model_aux_both_tiers():
    model, _ = build(VO.TINY, VO.ALL_FALSE)
    z = torch.zeros(2, *VO.TINY[5], dtype=torch.long, device=DEV)
    for amp in (False, True):
        out = model.sample(z, cond=cond_of(VO.TINY), top_k=1, amp=amp)
        assert out.shape == z.shape and int(out.min()) >= 0 and int(out.max()) < VO.TINY[4]
    with pytest.raises(ValueError, match="model_aux"):
        build(VO.TINY, VO.COMBOS[-1])[0].sample(z, top_k=1)


def test_fast_tier_batch_over_256_runs_in_chunks():
    """B = 300 runs as two chunks of 150: identical to two separate calls of 150 rows"""
    model, _ = build(VO.TINY, VO.ALL_FALSE)
    model.precision = "fast"
    bs = VO.TINY[5]
    cond = synth.randint_seeded(0, VO.TINY[6], (300, 1), 46).to(DEV)
    z = torch.zeros(300, *bs, dtype=torch.long, device=DEV)
    out = model.sample(z, cond=cond, top_k=1, amp=True)
    a = model.sample(z[:150], cond=cond[:150], top_k=1, amp=True)
    b = model.sample(z[150:], cond=cond[150:], top_k=1, amp=True)
    assert torch.equal(out, torch.cat([a, b]))


def test_all_false_graph_pdl_determinism_and_sequential_prefill():
    model, _ = build(VO.TINY, VO.ALL_FALSE)
    model.precision = "fast"
    bs, V = VO.TINY[5], VO.TINY[4]
    cond = cond_of(VO.TINY)
    n_tok = bs[0] * bs[1] * bs[2]
    noise = noise_tensor(9, n_tok, 2, V)

    def run(start=(0, 0), part=None):
        p = torch.zeros(2, *bs, dtype=torch.long, device=DEV) if part is None else part
        skip = (start[0] * bs[1] + start[1]) * bs[2]
        return model._native_sample(p, None, cond, start, 1.0, 100, 0.95, True, noise=noise[skip:].contiguous())

    base = run()
    assert torch.equal(run(), base)                                       # run to run
    with env(model, RQB200_NO_GRAPH="1"):
        assert torch.equal(run(), base)
    with env(model, RQB200_NO_PDL="1"):
        assert torch.equal(run(), base)
    res = run((2, 1), base)
    with env(model, RQB200_SEQ_PREFILL="1"):
        assert torch.equal(run((2, 1), base), res)                        # prefill token by token == one batched pass


def test_per_depth_classifier_at_production_width():
    """shared_cls_emb = false at V 16384, E 1536 (2 + 2 layers, synthetic weights): the per-depth tensor maps of the step and both
    classifier GEMMs of the forward (B 2: 128 rows per depth, weight streamer; B 8: 512 rows per depth, rows GEMM) against the exact
    tier"""
    flags = dict(VO.COMBOS[-1], shared_cls_emb=False)
    shape = (1536, 24, 2, 2, 16384, (8, 8, 4), 1000, 1)
    model, _ = build(shape, flags, seed=47)
    table = CodebookAux(synth.randn_seeded((16384, 256), 48).to(DEV))
    for B in (2, 8):
        xs = synth.randint_seeded(0, 16384, (B, 8, 8, 4), 49).to(DEV)
        cond = synth.randint_seeded(0, 1000, (B, 1), 50).to(DEV)
        model.precision = "exact"
        ex = teacher_forced(model, table, xs, cond, False)
        model.precision = "fast"
        fwd = model(xs, model_aux=table, cond=cond, amp=True)
        sig = float(ex.std())
        want = ex.reshape(8, 8, 4, B, -1).permute(3, 0, 1, 2, 4)
        err_fwd = float((fwd - want).abs().max()) / sig
        assert err_fwd < 0.02, err_fwd
        if B == 2:
            step = teacher_forced(model, table, xs, cond, True)
            err_step = float((step - ex).abs().max()) / sig
            assert err_step < 0.02, err_step
        print("per-depth classifier V 16384 E 1536 B %d: forward %.4f sigma" % (B, err_fwd))
