"""CLIP on the native engine (H100): the fused preprocessing bit for bit against the reference's PIL / torchvision route, both tiers'
image and text features and cosines against the float64 fixture (tests/golden/clip.pt, scripts/gen_golden_clip.py) on three
geometries, fast-tier ranking, chunked batches, and the new kernels against float64: the QuickGELU epilogues of the weight streamer
and the rows GEMM, the non-causal tiled flash attention and the exact tier's fp32 attention."""
import hashlib
import os

import pytest
import torch

from rqvae import _native as N
from rqvae.metrics import clip_score as CS
from tests import clip_oracle as CO

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# CLIP's merge list reduced to the merges of the texts the tests tokenize, every merge at its own rank (scripts/gen_golden_clip.py)
BPE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "clip_bpe_subset.txt.gz")
# measured maxima on an H100 are in README.md (CLIP score); the bounds hold them with margin
BOUND = {"exact": (1e-5, 1e-6), "fast": (1.5e-3, 4e-4)}        # features rel-L2 per row, |cosine| error


@pytest.fixture(scope="module")
def fixture(golden):
    return golden("clip")


_models = {}


def model_of(fixture, g, precision):
    if g not in _models:
        m = CS.build_model(CO.synth_state_dict(g, fixture["seeds"][g])).to(DEV)
        m.bpe_path = BPE
        _models[g] = m
    m = _models[g]
    m.precision = precision
    return m


def sha256(t):
    return hashlib.sha256(t.cpu().contiguous().numpy().tobytes()).hexdigest()


def row_rel(a, b):
    return ((a.double().cpu() - b.double()).norm(dim=1) / b.double().norm(dim=1)).max().item()


def test_preprocess_bit_exact(fixture):
    L = CS._lib()
    for name, case in fixture["pix"].items():
        x = CO.pixels(case["seed"], 1, case["H"], case["W"]).to(DEV)
        u8 = torch.empty(1, 3, 224, 224, dtype=torch.uint8, device=DEV)
        nrm = torch.empty(1, 3, 224, 224, dtype=torch.float32, device=DEV)
        N.check(L.rqb200_dbg_clip_preprocess(N.ptr(x), 1, case["H"], case["W"], 224, N.ptr(u8), N.ptr(nrm), N.stream_ptr()), "preprocess")
        assert torch.equal(u8[:, :, :4].cpu(), case["u8_head"]), name               # (a readable diff of the first rows)
        assert sha256(u8) == case["u8_sha256"], name
        assert sha256(nrm) == case["norm_sha256"], name


def test_preprocess_clamps_out_of_range():
    x = torch.full((1, 3, 224, 224), 2.0, device=DEV)
    x[:, :, :112] = -1.0
    u8 = torch.empty(1, 3, 224, 224, dtype=torch.uint8, device=DEV)
    N.check(CS._lib().rqb200_dbg_clip_preprocess(N.ptr(x), 1, 224, 224, 224, N.ptr(u8), None, N.stream_ptr()), "preprocess")
    assert (u8[:, :, :112] == 0).all() and (u8[:, :, 112:] == 255).all()


@pytest.mark.parametrize("precision", ["exact", "fast"])
@pytest.mark.parametrize("g", ["tiny", "b32", "b16n"])
def test_features_and_cosines(fixture, g, precision):
    f = fixture["feat"][g]
    m = model_of(fixture, g, precision)
    H, W, ps = f["pix"]
    B0 = len(f["caps"])
    px = CO.pixels(ps, B0, H, W)
    fb, cb = BOUND[precision]
    report = []
    for reps in (1, 14):                                        # B = 5 and 70 (not a multiple of 64); and B = 1 below
        pix = px.repeat(reps, 1, 1, 1).to(DEV)
        tok = f["tokens"].repeat(reps, 1).to(DEV)
        ei = row_rel(m.encode_pixels(pix), f["image"].repeat(reps, 1))
        et = row_rel(m.encode_text(tok), f["text"].repeat(reps, 1))
        ec = (CS.clip_score(pix, tok, m, None).double().cpu() - f["cos"].repeat(reps)).abs().max().item()
        report.append((ei, et, ec))
        assert ei < fb and et < fb and ec < cb, (g, precision, reps, ei, et, ec)
    one = CS.clip_score(px[:1].to(DEV), f["tokens"][:1].to(DEV), m, None)
    assert one.dim() == 0 and abs(float(one) - float(f["cos"][0])) < cb
    print("CLIP %s %s: max image rel-L2 %.2e, text %.2e, cosine %.2e" % (g, precision, max(r[0] for r in report),
                                                                          max(r[1] for r in report), max(r[2] for r in report)))


def test_encode_image_takes_normalised_batch(fixture):
    f = fixture["feat"]["tiny"]
    m = model_of(fixture, "tiny", "exact")
    H, W, ps = f["pix"]
    px = CO.pixels(ps, len(f["caps"]), H, W).to(DEV)
    nrm = torch.empty(px.shape[0], 3, 32, 32, device=DEV)
    N.check(CS._lib().rqb200_dbg_clip_preprocess(N.ptr(px), px.shape[0], H, W, 32, None, N.ptr(nrm), N.stream_ptr()), "preprocess")
    assert torch.equal(m.encode_image(nrm), m.encode_pixels(px))


def test_clip_score_with_captions(fixture):
    f = fixture["feat"]["tiny"]
    m = model_of(fixture, "tiny", "exact")
    H, W, ps = f["pix"]
    caps = [fixture["captions"][c] for c in f["caps"]]
    s = CS.clip_score(CO.pixels(ps, len(caps), H, W).to(DEV), caps, m, CS.ClipPreprocess(32))
    assert (s.double().cpu() - f["cos"]).abs().max() < BOUND["exact"][1]


def test_fast_ranking_matches_exact(fixture):
    m = model_of(fixture, "tiny", "exact")
    px = CO.pixels(77, 16, 64, 64).to(DEV)
    tok = fixture["feat"]["tiny"]["tokens"][:1].repeat(16, 1).to(DEV)
    se = CS.clip_score(px, tok, m, None).double().cpu()
    m.precision = "fast"
    sf = CS.clip_score(px, tok, m, None).double().cpu()
    bound = BOUND["fast"][1]
    assert (se - sf).abs().max() < bound
    for i in range(16):
        for j in range(16):
            if se[i] - se[j] > 2 * bound:
                assert sf[i] > sf[j], (i, j)
    close = sum(1 for i in range(16) for j in range(i) if abs(se[i] - se[j]) <= 2 * bound)
    print("fast ranking: %d of 120 pairs closer than twice the bound" % close)


@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_chunked_batch_equals_separate_calls(fixture, precision):
    m = model_of(fixture, "tiny", precision)
    B = CS.CHUNK + 7
    px = CO.pixels(78, B, 40, 48).to(DEV)
    tok = CS.tokenize(["a photo of number %d" % i for i in range(B)], bpe_path=BPE).to(DEV)
    whole_i, whole_t = m.encode_pixels(px), m.encode_text(tok)
    parts_i = torch.cat([m.encode_pixels(px[:CS.CHUNK]), m.encode_pixels(px[CS.CHUNK:])])
    parts_t = torch.cat([m.encode_text(tok[:CS.CHUNK]), m.encode_text(tok[CS.CHUNK:])])
    assert torch.equal(whole_i, parts_i) and torch.equal(whole_t, parts_t)


def test_engine_rebuilt_after_load_state_dict(fixture):
    m = CS.build_model(CO.synth_state_dict("tiny", 21)).to(DEV)
    tok = torch.zeros(1, 77, dtype=torch.long, device=DEV)
    tok[0, :2] = torch.tensor([CS.SOT, CS.EOT])
    a = m.encode_text(tok)
    sd2 = CO.synth_state_dict("tiny", 22)
    m.load_state_dict(sd2)
    b = m.encode_text(tok)
    want = CO.encode_text(sd2, "tiny", tok.cpu())
    assert row_rel(b, want) < BOUND["exact"][0] and not torch.equal(a, b)


# ---- kernels against float64
def _qgelu(x):
    return x * torch.sigmoid(1.702 * x)


@pytest.mark.parametrize("M", [1, 37, 200, 256, 300, 700])
@pytest.mark.parametrize("Nout", [128, 384])
def test_quick_gelu_epilogues(M, Nout):
    K = 192
    g = torch.Generator(device="cpu").manual_seed(M * 7 + Nout)
    W = (torch.randn(Nout, K, generator=g) / K ** 0.5).half().to(DEV)
    X = torch.randn(((M + 127) // 128) * 128, K, generator=g).half().to(DEV)
    bias = (0.3 * torch.randn(Nout, generator=g)).to(DEV)
    ref = _qgelu(X[:M].double() @ W.double().t() + bias.double())
    L = N.lib()
    out = torch.zeros(M, Nout, dtype=torch.float16, device=DEV)
    N.check(L.rqb200_dbg_gemm_tc(N.ptr(W), N.ptr(X), N.ptr(bias), None, N.ptr(out), 1, 2, None, Nout, K, M, 1, 0, N.stream_ptr()), "gemm_tc")
    err = ((out.double() - ref).abs() / (ref.abs() + 1)).max().item()
    assert err < 2e-3, ("streamer", err)
    out2 = torch.zeros(M, Nout, dtype=torch.float16, device=DEV)
    N.check(L.rqb200_dbg_rows_gemm(N.ptr(X), N.ptr(W), N.ptr(bias), None, None, N.ptr(out2), 2, 0, M, Nout, K, N.stream_ptr()), "rows")
    err2 = ((out2.double() - ref).abs() / (ref.abs() + 1)).max().item()
    assert err2 < 2e-3, ("rows GEMM", err2)
    pre = X[:M].double() @ W.double().t() + bias.double()       # the exact GELU in place of QuickGELU would miss the bound
    assert ((torch.nn.functional.gelu(pre) - ref).abs() / (ref.abs() + 1)).max().item() > 1e-2


def _attn_ref(qkv, G, T, E, causal):
    q, k, v = qkv.double().reshape(T, G, 3, E // 64, 64).unbind(2)
    s = torch.einsum("tghd,sghd->ghts", q, k) * 0.125
    if causal:
        s = s + torch.full((T, T), float("-inf"), dtype=torch.float64, device=s.device).triu(1)
    return torch.einsum("ghts,sghd->tghd", s.softmax(-1), v).reshape(T * G, E)


@pytest.mark.parametrize("T", [17, 50, 64, 65, 77, 197, 257])
@pytest.mark.parametrize("causal", [0, 1])
def test_attention_kernels(T, causal):
    G, E = 3, 128
    g = torch.Generator(device="cpu").manual_seed(T * 2 + causal)
    qkv = (2 * torch.randn(T * G, 3 * E, generator=g)).to(DEV)
    ref = _attn_ref(qkv, G, T, E, causal)
    out = torch.empty(T * G, E, device=DEV)
    N.check(CS._lib().rqb200_dbg_clip_attn(N.ptr(qkv), N.ptr(out), G, T, E, causal, N.stream_ptr()), "clip_attn")
    assert (out.double() - ref).abs().max().item() < 1e-5
    q16 = qkv.half()
    ref16 = _attn_ref(q16, G, T, E, causal)
    a16 = torch.full((T * G, E), float("nan"), dtype=torch.float16, device=DEV)
    N.check(CS._lib().rqb200_dbg_clip_attn_flash(N.ptr(q16), N.ptr(a16), G, T, E, causal, N.stream_ptr()), "clip_attn_flash")
    assert (a16.double() - ref16).abs().max().item() < 4e-3
    if not causal:                                              # the causal result would fail the non-causal reference
        assert (_attn_ref(q16, G, T, E, 1) - ref16).abs().max().item() > 1e-2
