"""GPU: the stateful RQTransformer.cached_forward (one rqb200_ar_step per call after init_cache()) driven by the reference's own
sampling loop through the public API.  Exact tier: codes equal to the reference's trajectories (tests/golden/ar.pt, ar4.pt) and
logits within the exact-tier bounds.  Fast tier: every step's logits bit-identical to the fused sampling loop's under teacher
forcing, for every weight format and model family the fast tier samples.  Plus: O(1) launches and memory per call, isolation of the
step's KV state from other calls, the stateless fallback, and invalidation on new weights."""
import pytest
import torch

from oracle import synth
from oracle.zoo import AR_ZOO
from rqvae.models import _bind as nb
from rqvae.models import create_model
from tests import depthwise_oracle as DO
from tests import variants_oracle as VO
from tests.helpers import CodebookAux, ar_config, noise_tensor
from tests.test_gpu_depthwise import TablesAux, _ar_config as _dw_config
from tests.test_gpu_fast import _case as _zoo_case, _with_env
from tests.test_gpu_long import _case as _ar4_case
from tests.test_gpu_variants import build as _variant, cond_of as _variant_cond

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
DEV = "cuda"


def raster(bs, start=(0, 0)):
    H, W, D = bs
    return [(h, w, d) for h in range(H) for w in range(W) for d in range(D) if (h, w) >= tuple(start)]


def stepped_loop(model, xs0, aux, cond, amp, start=(0, 0), force=None, noise=None, ks=None, ps=None):
    """the reference's sample loop (transformers.py:343-369): init_cache(), then for every (h, w, d) cached_forward on the rows
    up to h, a sampler on its logits and the code written into xs.  force: teacher forcing (the code written is force's).
    Returns (codes, [n_tok, B, V] logits, launches of every call)."""
    xs = xs0.clone()
    model.init_cache()
    logits, launches = [], []
    for t, (h, w, d) in enumerate(raster(model.block_size, start)):
        lg = model.cached_forward(xs[:, :h + 1], model_aux=aux, cond=cond, amp=amp, sample_loc=(h, w, d))
        launches.append(model.last_launches)
        logits.append(lg.clone())
        if force is not None:
            xs[:, h, w, d] = force[:, h, w, d]
        else:
            xs[:, h, w, d] = nb.sample_logits(lg, 1.0, ks[d], ps[d], q=None if noise is None else noise[t])
    return xs, torch.stack(logits), launches


def teacher_forced(model, codes, aux, cond, start=(0, 0)):
    _, lg = model._native_sample(codes, aux, cond, start, 1.0, None, None, True, noise=False, return_logits=True, force_codes=codes)
    return lg


def assert_fast_bit_identical(model, codes, aux, cond, start=(0, 0), label=""):
    model.precision = "fast"
    want = teacher_forced(model, codes, aux, cond, start)
    got, lg, launches = stepped_loop(model, codes, aux, cond, True, start, force=codes)
    assert torch.equal(got, codes)
    bad = (lg != want).flatten(1).any(1).nonzero()
    assert len(bad) == 0, "%s: first token with different logits: %d of %d" % (label, int(bad[0]), len(lg))
    return launches


# ------------------------------------------------------------------------------------------------ exact tier vs the reference
@pytest.mark.parametrize("name", ["tiny", "tiny_txt", "ffhq355m"])
def test_exact_tier_stepped_loop_matches_reference(golden, layouts, name):
    g, model, aux, cond, bs, V = _zoo_case(name, golden, layouts)
    model.precision = "exact"
    B = g["B"]
    n_tok = bs[0] * bs[1] * bs[2]
    zero = torch.zeros(B, *bs, dtype=torch.long, device=DEV)
    for run in g["runs"]:
        st = run["setting"]
        ks, ps = model._lists(st.get("top_k"), st.get("top_p"))
        codes, logits, _ = stepped_loop(model, zero, aux, cond, False, noise=noise_tensor(run["noise_seed"], n_tok, B, V), ks=ks, ps=ps)
        for step, lg in (run["logits"] or {}).items():
            torch.testing.assert_close(logits[step].cpu(), lg, rtol=1e-4, atol=2e-4)
        d = (codes.cpu() != run["codes"].long()).flatten(1).any(0).nonzero()
        assert len(d) == 0, "%s %s: first divergent token %d of %d" % (name, st, int(d[0]), n_tok)
    rs = g["resume"]
    ks, ps = model._lists(rs["top_k"], None)
    codes2, _, _ = stepped_loop(model, g["runs"][0]["codes"].long().to(DEV), aux, cond, False, start=rs["start_loc"],
                                noise=noise_tensor(rs["noise_seed"], n_tok, B, V), ks=ks, ps=ps)
    assert torch.equal(codes2.cpu().to(torch.int32), rs["codes"])


# ------------------------------------------------------------------------------------------------ fast tier == the sampling loop
@pytest.mark.parametrize("name", ["tiny", "tiny_txt", "cc3m654m"])
@pytest.mark.parametrize("fmt", ["fp16", "fp8"])
def test_fast_tier_step_logits_bit_identical_to_sampling_loop(golden, layouts, name, fmt):
    """cc3m654m: the 32-token prefix goes through the batched prefill on the restart call"""
    g, model, aux, cond, bs, V = _zoo_case(name, golden, layouts)
    codes = g["runs"][-1]["codes"].long().to(DEV)
    _with_env(model, {"RQB200_FAST_DTYPE": fmt}, lambda: assert_fast_bit_identical(model, codes, aux, cond, label="%s %s" % (name, fmt)))


def test_fast_tier_step_per_depth_codebooks(golden):
    """model_aux with one codebook per depth (tests/golden/rqd.pt's model)"""
    P = DO.AR_PLAN
    E, nh, nb_, nhl, V, bs, vc, cl = DO.AR_SHAPE
    with torch.device("meta"):
        model, _ = create_model(_dw_config(*DO.AR_SHAPE))
    sd = synth.synth_state_dict(synth.shapes_of(model.state_dict()), P["weight_seed"])
    model = model.to_empty(device=DEV)
    model.load_state_dict({k: v.to(DEV) for k, v in sd.items()})
    model = model.eval()
    aux = TablesAux(DO.tables_of([V] * bs[2], P["table_seed"]))
    cond = synth.randint_seeded(0, vc, (P["B"], cl), P["cond_seed"]).to(DEV)
    codes = golden("rqd")["ar"]["runs"][1]["codes"].long().to(DEV)
    assert_fast_bit_identical(model, codes, aux, cond, label="per-depth codebooks")


def test_fast_tier_step_all_false_embeddings_without_model_aux(golden):
    """the reference's default embedding flags (own token tables, per-depth classifiers): model_aux=None"""
    rec = golden("arv")["combos"][VO.combo_name(VO.ALL_FALSE)]
    model, _ = _variant(VO.TINY, VO.ALL_FALSE)
    codes = rec["runs"][1]["codes"].long().to(DEV)
    cond = _variant_cond(VO.TINY)
    assert_fast_bit_identical(model, codes, None, cond, label="all-false")
    _with_env(model, {"RQB200_FAST_DTYPE": "fp8"}, lambda: assert_fast_bit_identical(model, codes, None, cond, label="all-false fp8"))


def test_fast_tier_step_headless(golden):
    """16x16x1 without head layers (tests/golden/ar4.pt headless16): each step is body step + classifier"""
    g, shape, model, aux, cond, bs, V = _ar4_case("headless16", golden)
    codes = g["runs"][-1]["codes"].long().to(DEV)
    launches = assert_fast_bit_identical(model, codes, aux, cond, label="headless16")
    assert len(set(launches[1:])) == 1


def test_fast_tier_step_start_after_origin_and_two_chunks(golden, layouts):
    g, model, aux, cond, bs, V = _zoo_case("tiny", golden, layouts)
    codes = g["runs"][-1]["codes"].long().to(DEV)
    # first call at (2, 1, 0) after init_cache(): prefill of the 9 positions before it, as sample(start_loc=(2, 1)) does
    assert_fast_bit_identical(model, codes, aux, cond, start=(2, 1), label="start (2, 1)")
    # B = 300: two engine slots of 150 rows, each bit-identical to a 150-row sampling loop
    B = 300
    gen = torch.Generator(DEV).manual_seed(7)
    codes = torch.randint(0, V, (B, *bs), device=DEV, generator=gen)
    cnd = torch.randint(0, AR_ZOO["tiny"][6], (B, 1), device=DEV, generator=gen)
    model.precision = "fast"
    got, lg, _ = stepped_loop(model, codes, aux, cnd, True, force=codes)
    for lo, hi in ((0, 150), (150, 300)):
        want = teacher_forced(model, codes[lo:hi].contiguous(), aux, cnd[lo:hi].contiguous())
        assert torch.equal(lg[:, lo:hi], want), (lo, hi)


# ------------------------------------------------------------------------------------------------ O(1) per call
def test_step_cost_is_constant_per_call():
    """in1400m at B = 8: a call's launches do not depend on the position, and far below a stateless re-evaluation's; a call after
    the first allocates only its [B, V] output"""
    torch.manual_seed(0)
    with torch.device(DEV):
        model, _ = create_model(ar_config("in1400m"))
    model = model.eval()
    model.precision = "fast"
    H, W, D = model.block_size
    V, B = model.vocab_size[0], 8
    aux = CodebookAux(torch.randn(V, 256, device=DEV))
    gen = torch.Generator(DEV).manual_seed(1)
    codes = torch.randint(0, V, (B, H, W, D), device=DEV, generator=gen)
    cond = torch.randint(0, 1000, (B, 1), device=DEV, generator=gen)
    model.init_cache()
    at = {}
    for (h, w, d) in raster(model.block_size):
        if (h, w, d) == (0, 1, 1):
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            before = torch.cuda.memory_allocated()
        model.cached_forward(codes[:, :h + 1], aux, cond, True, (h, w, d))
        if (h, w, d) == (0, 1, 1):
            torch.cuda.synchronize()
            grew = torch.cuda.max_memory_allocated() - before
        at[(h, w, d)] = model.last_launches
    for d in range(D):                                                      # (d = D-1 also advances the position counter)
        assert at[(0, 1, d)] == at[(H - 1, W - 1, d)], (d, at[(0, 1, d)], at[(H - 1, W - 1, d)])
    model.cached_forward(codes[:, :1], aux, cond, True, (0, 0, 2))         # out of order: stateless
    stateless = model.last_launches
    print("in1400m B=8 launches per call: d=0 %d, d>0 %d, stateless %d; peak growth of a d>0 call %d bytes ([B,V] = %d)"
          % (at[(0, 1, 0)], at[(0, 1, 1)], stateless, grew, B * V * 4))
    assert 10 * at[(0, 1, 0)] < stateless and 10 * at[(0, 1, 1)] < stateless
    assert grew <= 4 * B * V * 4
    model._invalidate_native()


# ------------------------------------------------------------------------------------------------ isolation, fallback, invalidation
def test_step_state_isolation_fallback_and_invalidation(golden, layouts):
    g, model, aux, cond, bs, V = _zoo_case("tiny", golden, layouts)
    H, W, D = bs
    codes = g["runs"][-1]["codes"].long().to(DEV)
    model.precision = "fast"
    want = teacher_forced(model, codes, aux, cond)
    toks = raster(bs)

    def cf(t, x=codes, c=cond):
        h, w, d = toks[t]
        return model.cached_forward(x[:, :h + 1], aux, c, True, (h, w, d))

    # a forward(amp=True) and a stateless cached_forward (another batch), both on other engine slots, between two steps
    model.init_cache()
    for t in range(22):
        assert torch.equal(cf(t), want[t]), t
    step_launches = model.last_launches
    model(codes, model_aux=aux, cond=cond, amp=True)
    lg1 = cf(5, x=codes[:1], c=None if cond is None else cond[:1])
    assert torch.equal(lg1, teacher_forced(model, codes[:1].contiguous(), aux, None if cond is None else cond[:1].contiguous())[5])
    for t in range(22, 30):
        assert torch.equal(cf(t), want[t]), t
        assert model.last_launches <= step_launches + 64           # still the native step, not a re-evaluation
    # out of order: a repeated token and a skipped one return the stateless teacher-forced logits
    assert torch.equal(cf(29), want[29])
    assert torch.equal(cf(31), want[31])
    assert torch.equal(cf(32), want[32])
    # ... and init_cache() restarts cleanly at the next (h, w, 0)
    model.init_cache()
    h0, w0 = toks[32][:2]
    resume = teacher_forced(model, codes, aux, cond, (h0, w0))
    for t in range(32, 40):
        assert torch.equal(cf(t), resume[t - 32]), t
    # new weights: the next call does not reuse the caches built with the old ones
    sd = {k: (v * 1.01 if v.is_floating_point() else v) for k, v in model.state_dict().items()}
    model.load_state_dict(sd)
    want2 = teacher_forced(model, codes, aux, cond)
    assert not torch.equal(want2[40], want[40])
    assert torch.equal(cf(40), want2[40])
    model.init_cache()
    for t in range(0, 8):
        assert torch.equal(cf(t), want2[t]), t


# ------------------------------------------------------------------------------------------------ 32x32x4 behind a 32-token prefix
def test_long32_stepped_loop_both_tiers(golden):
    """long32 (tests/golden/ar4.pt): 4096 steps over body KV caches up to 1056 rows kept between calls.  Exact tier: the reference's
    codes; fast tier: _native_sample's codes under the same injected noise"""
    g, shape, model, aux, cond, bs, V = _ar4_case("long32", golden)
    B = g["B"]
    n_tok = bs[0] * bs[1] * bs[2]
    zero = torch.zeros(B, *bs, dtype=torch.long, device=DEV)
    run = g["runs"][-1]
    st = run["setting"]
    ks, ps = model._lists(st.get("top_k"), st.get("top_p"))
    noise = noise_tensor(run["noise_seed"], n_tok, B, V)
    model.precision = "exact"
    codes, _, _ = stepped_loop(model, zero, aux, cond, False, noise=noise, ks=ks, ps=ps)
    d = (codes.cpu() != run["codes"].long()).flatten(1).any(0).nonzero()
    assert len(d) == 0, "exact tier: first divergent token %d of %d" % (int(d[0]), n_tok)
    model.precision = "fast"
    want = model._native_sample(zero, aux, cond, (0, 0), 1.0, st.get("top_k"), st.get("top_p"), True, noise=noise)
    codes, _, _ = stepped_loop(model, zero, aux, cond, True, noise=noise, ks=ks, ps=ps)
    d = (codes != want).flatten(1).any(0).nonzero()
    assert len(d) == 0, "fast tier: first divergent token %d of %d" % (int(d[0]), n_tok)
