"""RQVAE at any image size on the GPU: encode / decode / forward on maps other than the configured resolution, against the reference
fixture tests/golden/vaesz.pt (scripts/gen_golden_vae_sizes.py), on both tiers; the per-extent entry points at the configured
extent against the original ones, bit for bit; batch independence and fused vs stand-alone GroupNorm statistics at a non-square
size; the tensor-core spatial attention (rqb200_dbg_vae_attn_tc) against the float64 reference of tests/vae_kernels_ref.py; and a
1024 x 1024 fast-tier decode of the f8 VAE (16384 attention tokens, past the exact tier's shared-memory limit)."""
import math
import os

import pytest
import torch

from oracle import rq_oracle as O
from oracle import synth
from oracle.zoo import VAE_ZOO, vae_ddconfig
from rqvae import _native as N
from rqvae.models import create_model
from rqvae.utils.config import Config, augment_arch_defaults
from tests import vae_kernels_ref as R
from tests.test_gpu_parity import audit_code_flips
from tests.test_gpu_tc_kernels import check_conv
from tests.test_gpu_vae_kernels import twice, within

pytestmark = pytest.mark.gpu
DEV = "cuda"
F8 = dict(K=16384, code_shape=(32, 32, 4), ch_mult=(1, 2, 2, 4), attn_resolutions=(32,))


def vae_kw(name, golden):
    return dict(golden("vaesz")[name]["vae"]) if name == "f8" else VAE_ZOO[name]


_MODELS = {}


def build(name, kw, seed):
    """the product RQVAE of a VAE_ZOO-style kwargs dict with the fixture's synthetic weights (memoised per session)"""
    key = (name, seed)
    if key not in _MODELS:
        cs = kw.get("code_shape", (8, 8, 4))
        dd = vae_ddconfig(**kw)
        cfg = augment_arch_defaults(Config(type="rq-vae", ddconfig=dd, hparams=dict(
            bottleneck_type="rq", embed_dim=256, n_embed=kw["K"], latent_shape=[cs[0], cs[1], 256], code_shape=list(cs),
            shared_codebook=True, decay=0.99, restart_unused_codes=True, loss_type="mse", latent_loss_weight=0.25)))
        with torch.device("meta"):
            model, _ = create_model(cfg)
        sd = synth.synth_state_dict(synth.shapes_of(model.state_dict()), seed)
        model = model.to_empty(device=DEV)
        model.load_state_dict({k: v.to(DEV) for k, v in sd.items()})
        _MODELS.clear()
        _MODELS[key] = (model.eval(), sd)
    return _MODELS[key]


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def cases(names):
    """(name, case index) of every fixture size of the named VAEs"""
    g = torch.load(os.path.join(os.path.dirname(__file__), "golden", "vaesz.pt"), weights_only=False)
    return [(n, i) for n in names for i in range(len(g[n]["cases"]))]


def inputs(model, c, kw):
    f = model.downsample_factor()
    x = synth.randn_seeded((c["B"], 3, c["H"], c["W"]), c["x_seed"]).to(DEV)
    code = synth.randint_seeded(0, kw["K"], (c["B"], c["H"] // f, c["W"] // f, kw.get("code_shape", (8, 8, 4))[-1]), c["codes_seed"])
    zq = model.quantizer.embed_code_with_depth(code.to(DEV), True)[0].sum(-2)
    return x, zq


def check_against_fixture(name, idx, precision, golden, bar):
    g = golden("vaesz")[name]
    c, kw, zs = g["cases"][idx], vae_kw(name, golden), g["z_stride"]
    model, sd = build(name, kw, g["weight_seed"])
    model.precision = precision
    x, zq = inputs(model, c, kw)
    st, what = c["stride"], "%s %s %dx%d" % (precision, name, c["H"], c["W"])
    # decode of a code map of this size's grid (the reference's route for codes off code_shape)
    pix = model.decode(zq)
    assert pix.shape == (c["B"], 3, c["H"], c["W"])
    r_dec = rel(pix.cpu()[:, :, ::st, ::st], c["pixels_sub"])
    mx = float(((pix.cpu()[:, :, ::st, ::st] * 0.5 + 0.5).clamp(0, 1) - (c["pixels_sub"] * 0.5 + 0.5).clamp(0, 1)).abs().max())
    assert abs(float(pix.double().pow(2).sum().sqrt()) - c["pixels_l2"]) < bar * c["pixels_l2"]
    # encode
    z_e = model.encode(x)
    assert z_e.shape == (c["B"], c["H"] // model.downsample_factor(), c["W"] // model.downsample_factor(), 256) and z_e.is_contiguous()
    z_sub = z_e.cpu()[:, ::zs, ::zs]
    r_enc = rel(z_sub, c["z_e_sub"])
    # forward: codes audited where the fixture holds z_e, the reconstruction compared when every code agrees
    out, _, codes_fwd = model(x)
    cf, cr = codes_fwd.cpu(), c["codes_fwd"].long()
    n_flip = audit_code_flips(c["z_e_sub"], z_sub, O.codebook_of(sd), cr[:, ::zs, ::zs], cf[:, ::zs, ::zs])
    n_diff = int((cf != cr).any(-1).sum())
    assert torch.equal(model.get_codes(x), codes_fwd)
    r_rec = rel(out.cpu()[:, :, ::st, ::st], c["recon_sub"]) if n_diff == 0 else float("nan")
    print("%s: decode rel-L2 %.2e (max abs after clamp %.2e), encode %.2e, forward %.2e; %d audited near-tie flip(s), %d vector(s) "
          "differ" % (what, r_dec, mx, r_enc, r_rec, n_flip, n_diff))
    assert r_dec < bar and r_enc < bar, what
    if precision == "fast":
        assert mx < 1e-3, what
    if zs == 1:
        assert n_diff == n_flip
    if n_diff == 0:
        assert r_rec < bar, what
    soft, scodes = model.get_soft_codes(x)
    assert soft.shape[:3] == codes_fwd.shape[:3] and torch.equal(scodes, codes_fwd)


@pytest.mark.parametrize("name,idx", cases(["tiny", "tiny_attn_mid", "imagenet", "f8"]))
def test_exact_tier_any_size_matches_reference(golden, name, idx):
    check_against_fixture(name, idx, "exact", golden, 1e-4)


@pytest.mark.parametrize("name,idx", cases(["imagenet", "f8"]))
def test_fast_tier_any_size_within_1e3(golden, name, idx):
    check_against_fixture(name, idx, "fast", golden, 1e-3)


# ------------------------------------------------------------------------------------------------ wgmma convs off powers of two
# (B, H, W, Cin, Cout, ks, stride, gn): H, W the output extent.  conv_tc_kernel's 128-pixel tile has power-of-two sides that may
# overhang the map; the TMA box reads zeros there (for stride 2 through the element-strided map) and the epilogue stores nothing.
CONV_ANY_CASES = [
    (2, 6, 10, 128, 128, 3, 2, 0),     # Downsample of a 12 x 20 map: one 16 x 8 box over the 10 x 6 output
    (1, 12, 40, 128, 256, 3, 2, 0),    # three 16-wide tiles, the last one half past the right edge; two 8-row tiles, the last half
    (3, 3, 5, 256, 256, 3, 2, 0),      # a 3 x 5 output: 8 x 4 boxes of four images, odd B
    (2, 3, 5, 256, 768, 1, 1, 0),      # the AttnBlock's q|k|v 1x1 conv on a 3 x 5 latent
    (2, 12, 20, 128, 128, 1, 1, 0),    # W = 20: two 16-wide tiles
    (1, 24, 48, 128, 128, 3, 2, 1),    # tiles cover the map exactly: GroupNorm statistics from the epilogue
]


@pytest.mark.parametrize("c", CONV_ANY_CASES, ids=str)
def test_conv_tc_any_extent(c):
    B, H, W, Cin, Cout, ks, stride, gn = c
    check_conv("tc", B, H, W, Cin, Cout, ks, stride, gn=bool(gn), seed=H * 100 + W)


# ------------------------------------------------------------------------------------------------ the per-extent entry points
def raw_call(model, fn, x, B, ext, out_shape, ws_hw):
    eng = model._engine(x.device)
    L = N.lib()
    need = L.rqb200_vae_workspace_bytes(eng["handle"], B) if ws_hw is None else L.rqb200_vae_workspace_bytes_hw(eng["handle"], B, *ws_hw)
    ws = torch.full((need,), 0x7F, dtype=torch.uint8, device=DEV)
    out = torch.full(out_shape, float("nan"), device=DEV)
    N.check(getattr(L, fn)(eng["handle"], N.ptr(x), B, *ext, N.ptr(out), N.ptr(ws), need, N.stream_ptr()), fn)
    torch.cuda.synchronize()
    return out, need, L.rqb200_vae_last_launches(eng["handle"])


@pytest.mark.parametrize("name,precision", [("tiny", "exact"), ("tiny_attn_mid", "exact"), ("imagenet", "exact"), ("imagenet", "fast")])
def test_hw_entry_points_equal_the_configured_ones(golden, name, precision):
    """at the configured extent, rqb200_vae_encode_hw / decode_hw are rqb200_vae_encode / decode: same bits, same launch count, same
    workspace size"""
    kw = VAE_ZOO[name]
    model, _ = build(name, kw, 41)
    model.precision = precision
    Rz, f = vae_ddconfig(**kw)["resolution"], model.downsample_factor()
    r, B = Rz // f, 2
    x = synth.randn_seeded((B, 3, Rz, Rz), 42).to(DEV)
    z = synth.randn_seeded((B, r, r, 256), 43).to(DEV)
    a, na, la = raw_call(model, "rqb200_vae_encode", x, B, (), (B, r, r, 256), None)
    b, nb, lb = raw_call(model, "rqb200_vae_encode_hw", x, B, (Rz, Rz), (B, r, r, 256), (Rz, Rz))
    assert torch.equal(a, b) and la == lb and na == nb and la > 0
    a, na, la = raw_call(model, "rqb200_vae_decode", z, B, (), (B, 3, Rz, Rz), None)
    b, nb, lb = raw_call(model, "rqb200_vae_decode_hw", z, B, (r, r), (B, 3, Rz, Rz), (Rz, Rz))
    assert torch.equal(a, b) and la == lb and na == nb and la > 0
    assert not torch.isnan(a).any()
    # and the Python surface, which calls the per-extent entry points at every size
    assert torch.equal(model.decode(z), a) and model.last_launches == la


def test_hw_entry_points_refuse_bad_extents():
    kw = VAE_ZOO["tiny"]
    model, _ = build("tiny", kw, 41)
    model.precision = "exact"
    eng = model._engine(torch.device(DEV))
    L = N.lib()
    ws = torch.empty(1 << 20, dtype=torch.uint8, device=DEV)
    x = torch.zeros(1, 3, 16, 16, device=DEV)
    for H, W in ((10, 16), (16, 6), (0, 16), (16, -4)):
        assert L.rqb200_vae_workspace_bytes_hw(eng["handle"], 1, H, W) == 0
        assert L.rqb200_vae_encode_hw(eng["handle"], N.ptr(x), 1, H, W, N.ptr(x), N.ptr(ws), ws.numel(), N.stream_ptr()) == N.EINVAL
    for h, w in ((0, 4), (4, 0), (-1, 2)):
        assert L.rqb200_vae_decode_hw(eng["handle"], N.ptr(x), 1, h, w, N.ptr(x), N.ptr(ws), ws.numel(), N.stream_ptr()) == N.EINVAL


def test_fast_tier_non_square_batch_independence_and_gn_statistics():
    """imagenet VAE, 12 x 8 latent (384 x 256 pixels): image 1 of a 3-image batch equals image 1 of a 2-image batch, bit for bit;
    GroupNorm statistics from the conv epilogues (where the tiles cover the map exactly) vs the stand-alone pass within 1e-4"""
    kw = VAE_ZOO["imagenet"]
    model, _ = build("imagenet", kw, 41)
    model.precision = "fast"
    z = synth.randn_seeded((3, 12, 8, 256), 44).to(DEV)
    x = synth.randn_seeded((3, 3, 384, 256), 45).to(DEV)
    p2, p3 = model.decode(z[:2]), model.decode(z)
    assert torch.equal(p3[:2], p2) and torch.isfinite(p3).all()
    e2, e3 = model.encode(x[:2]), model.encode(x)
    assert torch.equal(e3[:2], e2)
    os.environ["RQB200_GN_FUSE"] = "0"
    model._invalidate_native()
    try:
        p_unf, e_unf = model.decode(z), model.encode(x)
    finally:
        del os.environ["RQB200_GN_FUSE"]
        model._invalidate_native()
    d_dec, d_enc = float((p_unf - p3).abs().max()), float((e_unf - e3).abs().max() / e3.abs().max())
    print("fused vs stand-alone GroupNorm statistics, 384x256: decode max pixel difference %.2e, encode %.2e of max |z_e|" % (d_dec, d_enc))
    assert d_dec < 1e-4 and d_enc < 1e-4


def test_fast_tier_f8_decode_1024():
    """the f8 VAE's decoder at 1024 x 1024 (a 128 x 128 latent: 16384 attention tokens at C = 512) runs on the fast tier"""
    model, _ = build("f8", F8, 46)
    model.precision = "fast"
    z = synth.randn_seeded((1, 128, 128, 256), 47).to(DEV)
    pix = model.decode(z)
    assert pix.shape == (1, 3, 1024, 1024) and bool(torch.isfinite(pix).all())
    # the exact tier keeps the fp32 attention and its shared-memory limit: a clean NativeError, nothing launched past it
    model.precision = "exact"
    with pytest.raises(N.NativeError):
        model.decode(z)


# ------------------------------------------------------------------------------------------------ tensor-core attention
U16 = 2.0 ** -11           # fp16 unit roundoff


def attn_tc_slack(qkv, B, HW, C, mutation=None, rows=1024):
    """float64 bound [B, HW, C] on |rqb200_dbg_vae_attn_tc - attn_ref| (csrc/vae_attn_tc.cu), derived as attn_ref's is:
      operands.  q, k, v are rounded to fp16: relative U16 each, or an absolute 2^-25 below fp16's normal range;
      score.  q16 k16 is exact in fp32, the tensor core sums the C products in fp32 (2 u per addition, allowing truncation) and the
        scale adds one rounding: |d s_ij| <= A_ij = (2.001 U16 + (2 C + 4) u) s sum_c |q_c k_jc| + 2^-25 s sum_c (|q_c| + |k_jc|);
      exp.  expf (2 ulp) of s_ij - m_t (one rounding of the argument, m_t <= m the running maximum), and at most one rescale
        exp(m_old - m_new) and product per key tile: a relative 4 u + u (m - s_ij) + 6 n_t u on key j's weight, n_t = ceil(HW / 32);
      softmax.  Score errors e_j with |e_j| <= A'_j (the exp errors folded in) move a softmax weight by the factor exp(e_j) / sum_k
        p_k exp(e_k), within expm1(A'_j + max_k A'_k) of 1 -- not first order: A reaches ~0.4 on the needle rows of |score| ~100;
      the rest.  fp16(p) (U16, or 2^-25 absolute), fp16(v) (U16), the row sum l ((3 n_t + 12) u), the fp32 P V sums over HW keys
        (2 u per addition) and the final division (u): e2 = 2.001 U16 + (3 n_t + 2 HW + 20) u.
      |d out_ic| <= ((P (1 + dlt)) |v|)_ic (1 + e2) - (P |v|)_ic + 2^-25 (sum_j |v_jc| + 1),   dlt_ij = expm1(A'_ij + max_j A'_ij)."""
    x = qkv.reshape(B, HW, 3, C).double()
    q, k, v = x[:, :, 0], x[:, :, 1], x[:, :, 2]
    s = 0.125 if mutation == "scale_one_eighth" else R.attn_scale(C)
    U, nt = R.U32, math.ceil(HW / 32)
    va = v.abs()
    slack = torch.empty(B, HW, C, dtype=torch.float64, device=qkv.device)
    ksum = k.abs().sum(-1)
    e2 = 2.001 * U16 + (3 * nt + 2 * HW + 20) * U
    for i0 in range(0, HW, rows):
        qi = q[:, i0:i0 + rows]
        S = (qi @ k.transpose(1, 2)) * s
        if mutation == "last_key_dropped":
            S[..., -1] = float("-inf")
        m = S.amax(-1, keepdim=True)
        P = torch.softmax(S, -1)
        A = (2.001 * U16 + (2 * C + 4) * U) * s * (qi.abs() @ k.abs().transpose(1, 2)) + \
            2.0 ** -25 * s * (qi.abs().sum(-1, keepdim=True) + ksum[:, None, :])
        A = A + 4 * U + U * (m - S).nan_to_num(posinf=0.0) + 6 * nt * U
        dlt = torch.expm1(A + A.amax(-1, keepdim=True))
        slack[:, i0:i0 + rows] = ((P * (1 + dlt)) @ va) * (1 + e2) - P @ va + 2.0 ** -25 * (va.sum(1, keepdim=True) + 1)
    return slack


def run_attn_tc(qkv, B, HW, C):
    (out,) = twice(lambda o: N.lib().rqb200_dbg_vae_attn_tc(N.ptr(qkv), N.ptr(o), B, HW, C, N.stream_ptr()), ((B, HW, C), torch.float32))
    return out


ATTN_TC_CASES = [(1, 1025, 512, False), (3, 2047, 256, False), (2, 4096, 512, False), (1, 16384, 512, False), (2, 1500, 128, True),
                 (2, 7, 128, True), (1, 33, 384, False)]


@pytest.mark.parametrize("B,HW,C,needles", ATTN_TC_CASES)
def test_vae_attention_tc(B, HW, C, needles):
    qkv = R.attn_inputs(B, HW, C, seed=HW + C, needles=needles, device=DEV)
    out = run_attn_tc(qkv, B, HW, C)
    ref, _ = R.attn_ref(qkv, B, HW, C)
    slack = attn_tc_slack(qkv, B, HW, C)
    err = (out.double() - ref).abs()
    print("attn_tc B %d HW %d C %d: max |err| %.2e, max |err| / slack %.3f" % (B, HW, C, float(err.max()), float((err / slack).max())))
    within(out, ref, slack, "attn_tc B %d HW %d C %d" % (B, HW, C))


def test_vae_attention_tc_rejects_mutations():
    B, HW, C = 2, 1500, 128
    qkv = R.attn_inputs(B, HW, C, seed=2, needles=True, device=DEV)
    out = run_attn_tc(qkv, B, HW, C)
    ref, _ = R.attn_ref(qkv, B, HW, C)
    within(out, ref, attn_tc_slack(qkv, B, HW, C), "needles")
    for mutation in R.ATTN_MUTATIONS:
        mut, _ = R.attn_ref(qkv, B, HW, C, mutation=mutation)
        mslack = attn_tc_slack(qkv, B, HW, C, mutation=None if mutation == "softmax_over_queries" else mutation)
        assert R.excess(out, mut, mslack) > 0, mutation
