"""The tensor-core kernels, one launch per case through the engine's launchers (rqb200_dbg_gemm_tc_epi -> launch_gemm_tc,
rqb200_dbg_rows_gemm -> launch_rows_gemm_tc, rqb200_dbg_conv_tc / _gn -> launch_conv_tc), against the float64 references and derived
bounds of tests/tc_kernels_ref.py.  Every output starts as NaN with a guard region behind it: the output lies within the bound, the
guard keeps its bits, and a second launch gives the same bits.  The cases are named by the instantiation they run:
  gemm_tc_kernel<BN, WF>        BN 16 / 32 / 64 / 128 / 256 (16-bit) and 16 .. 128 (E4M3) on both sides of every chunk switch, ragged
                                multi-chunk tails, every epilogue mode, k-block counts around each ring depth, the engine's uneven splits
                                and N_out, and the engine's epilogue options (bias_scale, res_div, a device row index, ld_res);
  conv_tc_kernel<BN, S, 1>      the rows GEMM, BN 128 / 256 over several n tiles, M around the 128-row tiles;
  conv_tc_kernel<BN, S, 3>      1x1 and stride-2 convs with NB > 1 images per tile, BN 16 / 64 / 128 / 256, fused GroupNorm at cg 4 / 8 / 16;
  conv3x3_tc_kernel<BN, S>      Cout 3 (NCHW) and 64, TH 16 and 8 x 2;
  conv3x3_wreg_kernel<TH, NB, S> all three forms, Cout 384 / 640 / 768, odd slab counts, W < 8, NCHW output, GroupNorm partials, more
                                tiles than SMs at B >= 8;
and every wgmma conv geometry of the FFHQ and ImageNet layer plans.  Each family's *_rejects_mutations test shows the bound rejecting
the named mistakes of tc_kernels_ref on needle inputs.  Run with -s to see each family's largest |err| / bound."""
import collections

import pytest
import torch

from oracle.zoo import VAE_ZOO, vae_ddconfig
from rqvae import _native as N
from tests import tc_kernels_ref as R
from tests import vae_kernels_ref as V
from tests.test_gpu_vae_kernels import guard_intact, nan_guarded, twice

pytestmark = pytest.mark.gpu
DEV = "cuda"
FMT = {"fp16": 0, "bf16": 1, "e4m3": 0}
RATIO = collections.defaultdict(float)


@pytest.fixture(scope="module", autouse=True)
def report_ratios():
    yield
    for fam in sorted(RATIO):
        print("tc kernels: %-12s max |err| / bound = %.3g" % (fam, RATIO[fam]))


def within(fam, got, ref, tol, what):
    d = (got.double() - ref).abs()
    RATIO[fam] = max(RATIO[fam], float(torch.nan_to_num(d / tol, nan=float("inf")).max()))
    e = R.excess(got, ref, tol)
    assert e <= 0, "%s: %.3g beyond the bound" % (what, e)


# ---------------------------------------------------------------------------------------------------------------- streamer
def streamer_operands(fmt, N_out, K, B, seed):
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(N_out, K, generator=g) / K ** 0.5
    w[::5] *= 8.0                                                   # rows of different scales
    X = R.r16(torch.randn(B, K, generator=g), FMT[fmt]).to(DEV)
    bias = torch.randn(N_out, generator=g).to(DEV)
    if fmt == "e4m3":
        q, s = N.quantize_fp8_rows(w.to(DEV))
        return q, s, X, bias
    return R.r16(w, FMT[fmt]).to(DEV), None, X, bias


def run_streamer(fmt, W, s, X, mode, bias=None, bias_scale=1.0, residual=None, ld_res=0, res_div=0, row_idx=None, res_row_stride=0,
                 splits=1, in_place=False):
    """two guarded launches of rqb200_dbg_gemm_tc_epi; in_place: out is the residual buffer (the batched passes' x += ...)"""
    N_out, K = W.shape
    B = X.shape[0]
    Wp = N.pack_fp8_tiles(W) if s is not None else W
    dt = torch.float32 if mode in (0, 3) else R.DT[FMT[fmt]]
    shape = (splits, B, N_out) if mode == 3 else (B, N_out)
    rp = torch.tensor([row_idx], dtype=torch.int32, device=DEV) if row_idx is not None else None

    def launch(o):
        res = residual
        if in_place:
            o.copy_(residual)
            res = o
        return N.lib().rqb200_dbg_gemm_tc_epi(N.ptr(Wp), N.ptr(s), N.ptr(X), mode, N.ptr(bias), bias_scale, N.ptr(res), ld_res, res_div,
                                              N.ptr(rp), res_row_stride, None if mode == 3 else N.ptr(o), N.ptr(o) if mode == 3 else None,
                                              N_out, K, B, splits, FMT[fmt], N.stream_ptr())

    (out,) = twice(launch, (shape, dt))
    return out


def streamer_cases():
    cases = []
    engine = [(3072, 1024), (1280, 5120), (4608, 1536), (2560, 2560), (1536, 6144), (5120, 1280), (10240, 2560), (1024, 4096)]
    bs = [1, 16, 17, 32, 33, 64, 65, 128, 129, 256, 257, 300, 520]
    for fmt in ("fp16", "bf16", "e4m3"):
        for i, B in enumerate(bs):                  # every chunk switch, every mode, the engine's N_out
            N_out, K = engine[(i + len(fmt)) % len(engine)]
            cases.append((fmt, B, N_out, K, ("f32", "f32_res", "f32_inplace", "h16", "gelu")[i % 5], 1))
        for bn in (16, 32, 64, 128, 256):           # k-block counts around the ring depth
            if fmt == "e4m3" and bn == 256:
                continue
            st = R.stages(bn, fmt == "e4m3")
            for nkb in (st - 1, st, st + 1):
                cases.append((fmt, bn - (nkb % 3) * (bn // 16 - 1 if bn > 16 else 0), 256, 64 * nkb, "f32_res", 1))
        for N_out, K, splits, B in ((1536, 1536, 11, 17), (1536, 6144, 11, 64), (1280, 1280, 13, 1), (1280, 5120, 13, 33),
                                    (4608, 1536, 2, 128), (1536, 576, 9, 256)):
            cases.append((fmt, B, N_out, K, "partial", splits))
    return cases


def case_id(c):
    fmt, B, N_out, K, mode, splits = c
    bn = R.chunk_rows(B, fmt == "e4m3")
    return "gemm_tc_kernel<%d,%s>-%s-B%d-N%d-K%d-%s-s%d" % (bn, "E4M3" if fmt == "e4m3" else "W16", fmt, B, N_out, K, mode, splits)


@pytest.mark.parametrize("case", streamer_cases(), ids=case_id)
def test_streamer(case):
    fmt, B, N_out, K, mode, splits = case
    W, s, X, bias = streamer_operands(fmt, N_out, K, B, seed=B + N_out + K + splits)
    code = {"f32": 0, "f32_res": 0, "f32_inplace": 0, "h16": 1, "gelu": 2, "partial": 3}[mode]
    res = torch.randn(B, N_out, generator=torch.Generator(DEV).manual_seed(B), device=DEV) if mode in ("f32_res", "f32_inplace") else None
    kw = dict(bias=bias if code != 3 else None, residual=res, ld_res=N_out if res is not None else 0, splits=splits)
    out = run_streamer(fmt, W, s, X, code, in_place=mode == "f32_inplace", **kw)
    ref, slack = R.gemm_ref(W, X, code, scale=s, fmt=FMT[fmt], **kw)
    within("streamer" + ("16" if code in (1, 2) else ""), out, ref, slack, case_id(case))


# the AR engine's epilogues: w_in of the single-token step (bias x D, the position row at a device index, broadcast: ld_res = 0), w_in of
# the batched body pass (bias x D, row b of the residual for rows b * res_div ..), w_head (broadcast depth row)
EPI_CASES = [("w_in_step", 16, 4), ("w_in_step", 33, 8), ("w_in_batched", 64, 4), ("w_in_batched", 300, 2), ("w_head", 17, 1),
             ("w_in_batched", 129, 3)]


@pytest.mark.parametrize("fmt", ["fp16", "bf16", "e4m3"])
@pytest.mark.parametrize("kind,B,D", EPI_CASES)
def test_streamer_engine_epilogues(fmt, kind, B, D):
    N_out, K, HW = 1280, 256, 40
    W, s, X, bias = streamer_operands(fmt, N_out, K, B, seed=B + D)
    pos = torch.randn(HW, N_out, generator=torch.Generator(DEV).manual_seed(D), device=DEV)
    if kind == "w_in_step":
        kw = dict(bias_scale=float(D), residual=pos, ld_res=0, row_idx=HW - 3, res_row_stride=N_out)
    elif kind == "w_in_batched":
        kw = dict(bias_scale=float(D), residual=pos[1:], ld_res=N_out, res_div=max(1, B // (HW - 1) + 1))
    else:
        kw = dict(residual=pos[D], ld_res=0)
    out = run_streamer(fmt, W, s, X, 0, bias=bias, **kw)
    row0 = kw.pop("row_idx", None)
    ref, slack = R.gemm_ref(W, X, 0, scale=s, bias=bias, res_row0=row0 or 0, **kw)
    within("streamer_epi", out, ref, slack, "%s %s B %d" % (kind, fmt, B))


@pytest.mark.parametrize("mutation", R.GEMM_MUTATIONS)
def test_streamer_rejects_mutations(mutation):
    case = R.GEMM_MUTATION_CASES[mutation]
    W, s, X, bias, res = R.gemm_case_operands(case, seed=11, device=DEV)
    fmt = "e4m3" if case["e4m3"] else "fp16"
    kw = dict(bias=bias, bias_scale=case.get("bias_scale", 1.0), residual=res, ld_res=case["N"] if res is not None else 0,
              res_div=case.get("res_div", 0), splits=case["splits"])
    out = run_streamer(fmt, W, s, X, case["mode"], **kw)
    ref, slack = R.gemm_ref(W, X, case["mode"], scale=s, **kw)
    within("streamer_mut", out, ref, slack, mutation + " needles")
    mut, mslack = R.gemm_ref(W, X, case["mode"], scale=s, mutation=mutation, **kw)
    assert R.excess(out, mut, mslack) > 0, mutation


# ---------------------------------------------------------------------------------------------------------------- rows GEMM
@pytest.mark.parametrize("fmt", ["fp16", "bf16"])
@pytest.mark.parametrize("M,N_out,K", [(1, 384, 128), (127, 512, 256), (128, 384, 64), (129, 768, 192), (300, 1280, 320),
                                       (1000, 384, 512)])
def test_rows_gemm(fmt, M, N_out, K):
    """conv_tc_kernel<128, 6, 1> (N_out % 256 != 0) and <256, 4, 1>: fp32 in place over a residual, and 16-bit GELU; nothing past row M"""
    W, _, Xm, bias = streamer_operands(fmt, N_out, K, M, seed=M + N_out)
    Mp = -(-M // 128) * 128
    X = torch.zeros(Mp, K, dtype=Xm.dtype, device=DEV)
    X[:M] = Xm
    res = torch.randn(M, N_out, generator=torch.Generator(DEV).manual_seed(M), device=DEV)
    L = N.lib()

    def f32(o):
        o.copy_(res)
        return L.rqb200_dbg_rows_gemm(N.ptr(X), N.ptr(W), N.ptr(bias), N.ptr(o), N.ptr(o), None, 0, FMT[fmt], M, N_out, K, N.stream_ptr())

    (out,) = twice(f32, ((M, N_out), torch.float32))
    ref, slack = R.gemm_ref(W, Xm, 0, bias=bias, residual=res, ld_res=N_out)
    within("rows", out, ref, slack, "rows f32 M %d N %d" % (M, N_out))
    (o16,) = twice(lambda o: L.rqb200_dbg_rows_gemm(N.ptr(X), N.ptr(W), N.ptr(bias), None, None, N.ptr(o), 1, FMT[fmt], M, N_out, K,
                                                    N.stream_ptr()), ((M, N_out), R.DT[FMT[fmt]]))
    ref, slack = R.gemm_ref(W, Xm, 2, bias=bias, fmt=FMT[fmt])
    within("rows16", o16, ref, slack, "rows gelu M %d N %d" % (M, N_out))


# ---------------------------------------------------------------------------------------------------------------- convs
def run_conv(ops, bias, res, B, H, W, Cin, Cout, ks, stride, nchw=False, gn=False):
    """two guarded launches of rqb200_dbg_conv_tc_gn -> (out, gn partials [B, H W / 32, 32, 2] or None)"""
    x_hi, x_lo, w_hi, w_lo = ops
    flags = int(nchw) | (stride << 8 if stride > 1 else 0)
    shape = (B, Cout, H, W) if nchw else (B, H, W, Cout)

    def launch(o, part):
        return N.lib().rqb200_dbg_conv_tc_gn(N.ptr(x_hi), N.ptr(w_hi), N.ptr(x_lo), N.ptr(w_lo), N.ptr(bias), N.ptr(res), N.ptr(o),
                                             N.ptr(part), B, H, W, Cin, Cout, ks, flags, N.stream_ptr())

    out, part = twice(launch, (shape, torch.float32), ((B, H * W // 32, 32, 2) if gn else None, torch.float64))
    return out, part


def check_conv(fam, B, H, W, Cin, Cout, ks, stride, nchw=False, resid=False, gn=False, seed=0):
    x_hi, x_lo, w_hi, w_lo, bias, res = R.conv_operands(B, H, W, Cin, Cout, ks, stride, seed, DEV, resid=resid)
    if gn:
        bias = R.gn_needles_bias(Cout, seed, DEV)
    out, part = run_conv((x_hi, x_lo, w_hi, w_lo), bias, res, B, H, W, Cin, Cout, ks, stride, nchw, gn)
    ref, slack = R.conv_ref(x_hi, x_lo, w_hi, w_lo, bias, res, B, H, W, Cin, Cout, ks, stride, nchw)
    what = "%s B %d %dx%d %d->%d ks %d s %d" % (R.conv_kernel(H, W, Cout, ks, stride), B, H, W, Cin, Cout, ks, stride)
    within(fam, out, ref, slack, what)
    if gn:
        TW, TH, _ = R.conv_tile(H, W, Cout, ks, stride)
        kern = "wreg" if fam == "wreg" else "tc"
        gref, mag = R.gn_partials_ref(out, TW, TH)
        within(fam + "_gn", part, gref, R.gn_depth(kern, Cout) * R.U32 * mag + 1e-300, what + " GroupNorm partials")
    return out, part


# (B, H, W, Cin, Cout, ks, stride, nchw, resid, gn): H, W the output extent
CONV_TC_CASES = [
    (3, 1, 1, 64, 256, 3, 2, 0, 1, 0),      # Downsample to 1 x 1: NB = 128 images per tile, odd B
    (3, 2, 2, 128, 128, 3, 2, 0, 0, 0),     # NB = 32, the last tile's images past B
    (3, 8, 8, 128, 128, 3, 2, 0, 0, 1),     # NB = 2, odd B, GroupNorm cg = 4
    (5, 4, 4, 64, 64, 3, 2, 0, 1, 0),       # BN = 64, NB = 8
    (1, 8, 8, 512, 512, 1, 1, 0, 1, 1),     # 1x1, NB = 2 with one image, BN = 256, cg = 16
    (3, 8, 8, 128, 384, 1, 1, 0, 0, 0),     # BN = 128 over three n tiles (AttnBlock's q|k|v at C = 128)
    (2, 16, 16, 256, 256, 1, 1, 0, 1, 1),   # TW 16 x TH 8, cg = 8
    (2, 8, 8, 64, 3, 1, 1, 1, 0, 0),        # BN = 16, NCHW
    (1, 64, 64, 128, 128, 3, 2, 0, 0, 1),   # the encoder's first Downsample shape
]


@pytest.mark.parametrize("c", CONV_TC_CASES, ids=lambda c: "%s-%s" % (R.conv_kernel(c[1], c[2], c[4], c[5], c[6]), c))
def test_conv_tc(c):
    B, H, W, Cin, Cout, ks, stride, nchw, resid, gn = c
    check_conv("conv_tc", B, H, W, Cin, Cout, ks, stride, nchw, resid, gn, seed=sum(c))


CONV3X3_TC_CASES = [(2, 16, 16, 64, 64, 0, 1), (3, 8, 8, 128, 64, 0, 0), (1, 32, 32, 64, 3, 1, 0), (3, 4, 4, 64, 3, 1, 0),
                    (2, 16, 8, 192, 64, 0, 1)]


@pytest.mark.parametrize("c", CONV3X3_TC_CASES, ids=lambda c: "%s-%s" % (R.conv_kernel(c[1], c[2], c[4], 3, 1), c))
def test_conv3x3_tc(c):
    B, H, W, Cin, Cout, nchw, resid = c
    check_conv("conv3x3_tc", B, H, W, Cin, Cout, 3, 1, nchw, resid, seed=sum(c))


# (B, H, W, Cin, Cout, nchw, resid, gn)
WREG_CASES = [
    (1, 32, 32, 64, 128, 0, 1, 1),          # TH 32, one slab (9 k blocks: frag[0] across the tile boundary)
    (2, 32, 16, 192, 384, 0, 0, 0),         # three slabs, three n tiles
    (1, 64, 32, 128, 640, 0, 1, 0),         # five n tiles
    (2, 16, 16, 64, 768, 0, 0, 0),          # TH 16, six n tiles
    (3, 8, 8, 192, 256, 0, 1, 1),           # TH 8 x NB 2, odd B, cg = 8
    (2, 32, 4, 64, 128, 0, 0, 0),           # W < 8 at TH 32
    (2, 16, 4, 128, 256, 0, 1, 0),          # W < 8 at TH 16
    (2, 16, 16, 64, 128, 1, 0, 0),          # NCHW output
    (1, 16, 16, 128, 512, 0, 0, 1),         # cg = 16
    (8, 32, 32, 64, 640, 0, 1, 0),          # 160 tiles over 132 SMs, five n tiles
    (64, 16, 16, 64, 256, 0, 0, 1),         # the engine's B = 64: 256 tiles, two n tiles
]


@pytest.mark.parametrize("c", WREG_CASES, ids=lambda c: "%s-%s" % (R.conv_kernel(c[1], c[2], c[4], 3, 1), c))
def test_conv3x3_wreg(c):
    B, H, W, Cin, Cout, nchw, resid, gn = c
    check_conv("wreg", B, H, W, Cin, Cout, 3, 1, nchw, resid, gn, seed=sum(c))


def plan_geometries():
    """every wgmma conv of the FFHQ and ImageNet encoder + decoder plans: (H, W, Cin, Cout, ks, stride, nchw) with H, W the output
    extent (the fp32 conv_in, Cin = 3, is not one)"""
    geos = set()
    for name in ("ffhq", "imagenet"):
        for H, W, Cin, Cout, ks, stride, up, in_nchw, out_nchw in V.conv_plan(vae_ddconfig(**VAE_ZOO[name]))["conv"]:
            if in_nchw or Cin % 64:
                continue
            Ho, Wo, _ = V.conv_geom(H, W, ks, stride, up)
            geos.add((Ho, Wo, Cin, Cout, ks, stride, out_nchw))
    return sorted(geos)


@pytest.mark.parametrize("g", plan_geometries(), ids=lambda g: "%s-%s" % (R.conv_kernel(g[0], g[1], g[3], g[4], g[5]), g))
def test_conv_layer_plans(g):
    H, W, Cin, Cout, ks, stride, nchw = g
    B = 1 if H >= 64 else 2
    gn = not nchw and Cout in (128, 256, 512) and (ks, stride) != (3, 1) or (ks == 3 and stride == 1 and Cout % 128 == 0 and H <= 32)
    fam = "wreg" if ks == 3 and stride == 1 and Cout % 128 == 0 else "plan"
    check_conv(fam, B, H, W, Cin, Cout, ks, stride, nchw, resid=not nchw and H % 2 == 0, gn=gn, seed=H + Cin + Cout)


@pytest.mark.parametrize("mutation", R.CONV_MUTATIONS)
def test_conv_rejects_mutations(mutation):
    B, H, W, Cin, Cout, ks, stride = R.CONV_MUTATION_CASES[mutation]
    x_hi, x_lo, w_hi, w_lo, bias = R.conv_needles(B, H, W, Cin, Cout, ks, stride, seed=4, device=DEV)
    out, _ = run_conv((x_hi, x_lo, w_hi, w_lo), bias, None, B, H, W, Cin, Cout, ks, stride)
    ref, slack = R.conv_ref(x_hi, x_lo, w_hi, w_lo, bias, None, B, H, W, Cin, Cout, ks, stride, 0)
    within("conv_mut", out, ref, slack, mutation + " needles")
    mut, mslack = R.conv_ref(x_hi, x_lo, w_hi, w_lo, bias, None, B, H, W, Cin, Cout, ks, stride, 0, mutation=mutation)
    assert R.excess(out, mut, mslack) > 0, mutation


@pytest.mark.parametrize("mutation", R.GN_MUTATIONS)
def test_groupnorm_partials_reject_mutations(mutation):
    B, H, W, Cin, Cout, ks, stride = R.GN_MUTATION_CASES[mutation]
    out, part = check_conv("gn_mut", B, H, W, Cin, Cout, ks, stride, gn=True, seed=6)
    TW, TH, _ = R.conv_tile(H, W, Cout, ks, stride)
    kern = "wreg" if ks == 3 and stride == 1 and Cout % 128 == 0 else "tc"
    mut, mmag = R.gn_partials_ref(out, TW, TH, mutation)
    assert R.excess(part, mut, R.gn_depth(kern, Cout) * R.U32 * mmag) > 0, mutation


def test_conv_refuses_nhwc_cout3_without_writing():
    """an NHWC Cout = 3 output (the 16-channel epilogue would store past it) is refused, and nothing is written"""
    B, H, W, Cin = 2, 16, 16, 128
    x_hi, x_lo, w_hi, w_lo, bias, _ = R.conv_operands(B, H, W, Cin, 3, 3, 1, 5, DEV)
    full, out = nan_guarded((B, H, W, 3), torch.float32)
    assert N.lib().rqb200_dbg_conv_tc(N.ptr(x_hi), N.ptr(w_hi), N.ptr(x_lo), N.ptr(w_lo), N.ptr(bias), None, N.ptr(out), B, H, W, Cin, 3,
                                      3, 0, N.stream_ptr()) == N.EINVAL
    torch.cuda.synchronize()
    assert bool(torch.isnan(out).all()) and guard_intact(full, out.numel())
