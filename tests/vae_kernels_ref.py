"""float64 references of the VAE engine's kernels between its convs and of the exact tier's conv (csrc/conv_kernels.cu: the fp32
FFMA implicit-GEMM conv, GroupNorm(32) + SiLU, the AttnBlock core; csrc/conv_tc.cu: the fast tier's GroupNorm and cast operand
producers), the error bounds the tests hold them to, and the needle inputs on which a named mistake becomes visible.

Every reference starts from what the kernel reads: the fp32 activation and the stored weight, both converted to float64 exactly.  For
the fp16 outputs the bound covers the kernel's own rounding to fp16.  u = 2^-24 is the fp32 unit roundoff.  Every bound below is a
worst-case bound (first order in u), so it cannot fail by chance.

conv (conv_igemm_kernel).  One fp32 accumulator per output takes fmaf over the K = ks^2 Cin products in k order (a tap outside the
  input adds an exact zero), then bias and residual are added with one rounding each:
    |err| <= gamma_K sum_k |a_k w_k| + u (|conv + bias| + |out|) <= (K + 2) u (sum_k |a_k w_k| + |bias| + |residual|).
  K u < 3e-4 at K = 9 * 512, which is what lets the + 2 absorb gamma_K's 1 / (1 - K u).

GroupNorm.  Per (image, group): n = HW cg values x, mean mu, variance var, S1 = sum |x|, S2 = sum x^2 = n (var + mu^2).
  Statistics.  Each partial sum is formed in fp32 to depth d, then carried in fp64:
    gn_stats_kernel (exact tier; fast tier form 1): one pixel's cg channels per lane, d = cg;
    the wgmma conv epilogue (fast tier form 2): cg channels per lane, then 5 shuffle-add levels over a 32-pixel chunk, d = cg + 5.
  So |d sum| <= d u S1 and |d sumsq| <= d u S2; the fp64 levels add below 2^-40 of that and are covered by a term of 2^-45.  The
  kernels form var = sumsq / n - mean^2, so
    |d mean| <= d u S1 / n,   |d var| <= d u (S2 / n + 2 |mu| S1 / n) ~ d u var (3 + r^2) + ...,   r = |mu| / sqrt(var):
  the relative error of the variance grows with 1 + r^2 -- the cancellation term.  `cancel=False` replaces it with 3 d u var, what
  the same sums would give on centred data, to show where the kernels stop meeting that tighter bound.
  rstd = 1 / sqrt(var + eps) is evaluated in fp64 and cast to fp32; mean is cast to fp32:
    d_rstd / rstd <= |d var| / (2 (var + eps)) + u / 2,   d_mu <= |d mean| + u |mu| / 2.
  Normalisation, exact tier (gn_apply_kernel): scale = rstd gamma, shift = fmaf(-scale, mean, beta), v = fmaf(x, scale, shift),
  one rounding each:
    |d v| <= rstd |gamma| (|x - mu| (d_rstd / rstd + u) + d_mu) + u (|beta| + rstd |gamma| |mu|) + u |v|.
  Fast tier (gn_apply_f16_kernel): v = (x - mean) * rstd * gamma + beta, at most four roundings:
    |d v| <= rstd |gamma| (|x - mu| (d_rstd / rstd + 3 u) + d_mu) + 2 u |v|.
  SiLU z = v / (1 + exp(-v)): |d z| <= 1.1 |d v| (silu' <= 1.0998) + (e + 3 u) |z|, e the relative error of exp: expf 2 ulp (e = 4 u,
  exact tier), __expf 2 + 1.173 |v| ulp (e = (4 + 2.35 |v|) u, fast tier), and 3 u for the sum, the division and v's own rounding.
  fp32 output (form 0): that bound.  fp16 outputs (forms 1, 2): hi + lo is held to it plus half an ulp of lo (lo is the fp16 rounding
  of v - hi, which fp32 holds exactly); hi to one ulp16 of the reference plus it (tol16); and hi must be a nearest fp16 of
  float(hi) + float(lo) with |lo| at most half the gap to hi's neighbour on lo's side -- the promise the split-product conv relies on.
  (This is fp16-RNE of float(hi) + float(lo) except at an exact tie: when v - hi lies within an fp32 ulp of half a gap, lo rounds to
  exactly half a gap and the sum is a tie that RNE may resolve to hi's odd neighbour.)

cast / upsample (cast_f16_kernel): bit-exact: hi = x.half(), lo = (x - hi.float()).half(), the upsample repeat_interleave(2) on H and W.

spatial attention (vae_attn_kernel): softmax over the HW keys of (q k^T * s) v, s = float(1 / sqrt(double C)).  Per query i and key j,
  with A_ij = (ceil(C / 32) + 6) u s sum_c |q_c k_jc| the error of a score (a lane's fma chain of ceil(C / 32) terms, 5 shuffle-add
  levels, the scale) and m the row's maximum score:
    e_ij = exp(s_ij - m) is off by delta_ij = 4 u (expf) + A_ij + max_j A_ij + u (m - s_ij) relative,
    their sum (a thread's ceil(HW / 256) terms, 10 block-reduction levels) by delta_s = max_j delta_ij + (ceil(HW / 256) + 10) u,
    p_ij = e_ij / sum by delta_ij + delta_s + u, and the output's fma chain over the HW keys adds gamma_HW sum_j p_ij |v_jc|:
    |d out_ic| <= sum_j p_ij |v_jc| (delta_ij + delta_s + (HW + 2) u).
"""
import math

import torch
import torch.nn.functional as F

from tests.ar_kernels_ref import excess, tol16, ulp16  # noqa: F401  (the GPU tests' tolerance helpers, shared with the AR tier)

U32 = 2.0 ** -24
GN_EPS = 1e-6
GN_PIX = 256                 # pixels per gn_stats_kernel chunk
FUSED_PIX = 32               # pixels per conv-epilogue chunk


# ---------------------------------------------------------------------------------------------------------------- layer plans
def conv_plan(dd, embed_dim=256):
    """the convs, GroupNorms, attention cores and fp16 casts of RQVAE decode + encode for a ddconfig, in the engine's walk
    (csrc/vae_engine.cu VaeRun.decode / encode) -> dict of sets: conv (H, W, Cin, Cout, ks, stride, upsample, in_nchw, out_nchw) with H, W
    the input extent, gn (HW, C), attn (HW, C), cast (H, W, C, upsample)"""
    out = {"conv": set(), "gn": set(), "attn": set(), "cast": set()}
    nl, nb, ch0, mult, z = len(dd["ch_mult"]), dd["num_res_blocks"], dd["ch"], dd["ch_mult"], dd["z_channels"]
    conv = lambda *g: out["conv"].add(g)

    def resblock(r, cin, cout):
        out["gn"].update({(r * r, cin), (r * r, cout)})
        conv(r, r, cin, cout, 3, 1, 0, 0, 0)
        if cin != cout:
            out["cast"].add((r, r, cin, 0))
            conv(r, r, cin, cout, 1, 1, 0, 0, 0)
        conv(r, r, cout, cout, 3, 1, 0, 0, 0)

    def attnblock(r, c):
        out["gn"].add((r * r, c))
        out["attn"].add((r * r, c))
        out["cast"].add((r, r, c, 0))
        conv(r, r, c, 3 * c, 1, 1, 0, 0, 0)
        conv(r, r, c, c, 1, 1, 0, 0, 0)

    res, ch = dd["resolution"] >> (nl - 1), ch0 * mult[-1]
    out["cast"].update({(res, res, embed_dim, 0), (res, res, z, 0)})
    conv(res, res, embed_dim, z, 1, 1, 0, 0, 0)
    conv(res, res, z, ch, 3, 1, 0, 0, 0)
    resblock(res, ch, ch)
    attnblock(res, ch)
    resblock(res, ch, ch)
    for lvl in reversed(range(nl)):
        cout = ch0 * mult[lvl]
        for _ in range(nb + 1):
            resblock(res, ch, cout)
            ch = cout
            if res in dd["attn_resolutions"]:
                attnblock(res, ch)
        if lvl:
            out["cast"].add((res, res, ch, 1))
            conv(res, res, ch, ch, 3, 1, 1, 0, 0)
            res *= 2
    out["gn"].add((res * res, ch))
    conv(res, res, ch, dd["out_ch"], 3, 1, 0, 0, 1)
    res, ch = dd["resolution"], ch0
    conv(res, res, dd["in_channels"], ch, 3, 1, 0, 1, 0)
    for lvl in range(nl):
        cout = ch0 * mult[lvl]
        for _ in range(nb):
            resblock(res, ch, cout)
            ch = cout
            if res in dd["attn_resolutions"]:
                attnblock(res, ch)
        if lvl != nl - 1:
            out["cast"].add((res, res, ch, 0))
            conv(res, res, ch, ch, 3, 2, 0, 0, 0)
            res //= 2
    resblock(res, ch, ch)
    attnblock(res, ch)
    resblock(res, ch, ch)
    out["gn"].add((res * res, ch))
    conv(res, res, ch, z, 3, 1, 0, 0, 0)
    out["cast"].add((res, res, z, 0))
    conv(res, res, z, embed_dim, 1, 1, 0, 0, 0)
    return out


# ---------------------------------------------------------------------------------------------------------------- conv
CONV_MUTATIONS = ("flipped_taps", "pad_wrong_side", "upsample_round_up", "bias_dropped", "nhwc_as_nchw")


def conv_geom(H, W, ks, stride, upsample):
    """(Ho, Wo, pad): the engine's rule (vae_conv_geom)"""
    Hv, Wv = (2 * H, 2 * W) if upsample else (H, W)
    return Hv // stride, Wv // stride, 1 if (ks == 3 and stride == 1) else 0


def conv_ref(x, w, bias, resid, B, H, W, Cin, Cout, ks, stride, upsample, in_nchw, out_nchw, mutation=None):
    """(ref, slack) float64 of rqb200_dbg_vae_conv, laid out as the kernel's output.  x: the stored activation (NHWC, or NCHW when
    in_nchw), w: the stored OHWI weight in its own dtype, bias / resid nullable.  Taps are gathered with the kernel's own index rule
    (virtual input row uy = oy * stride + ky - pad, source row uy >> 1 under the upsample, zero outside the virtual extent)."""
    if in_nchw and mutation != "nhwc_as_nchw":
        X = x.reshape(B, Cin, H, W).permute(0, 2, 3, 1)
    else:
        X = x.reshape(B, H, W, Cin)
    X = F.pad(X.double(), (0, 0, 0, 1, 0, 1))          # one zero row and column at index H / W: every tap outside the input
    Wd = w.double().reshape(Cout, ks, ks, Cin)
    if mutation == "flipped_taps":
        Wd = Wd.flip(1, 2)
    Ho, Wo, pad = conv_geom(H, W, ks, stride, upsample)
    if mutation == "pad_wrong_side" and stride == 2:
        pad = 1
    Hv, Wv = (2 * H, 2 * W) if upsample else (H, W)
    dev = X.device

    def src(n_out, k, n_in, nv):
        u = torch.arange(n_out, device=dev) * stride + k - pad
        i = ((u + 1) >> 1 if mutation == "upsample_round_up" else u >> 1) if upsample else u
        return torch.where((u >= 0) & (u < nv) & (i < n_in), i, torch.full_like(i, n_in))

    out = torch.zeros(B, Ho, Wo, Cout, dtype=torch.float64, device=dev)
    mag = torch.zeros_like(out)
    for ky in range(ks):
        iy = src(Ho, ky, H, Hv)
        for kx in range(ks):
            tap = X[:, iy][:, :, src(Wo, kx, W, Wv)]
            wt = Wd[:, ky, kx]
            out += tap @ wt.t()
            mag += tap.abs() @ wt.abs().t()
    if bias is not None:
        mag += bias.double().abs()
        if mutation != "bias_dropped":
            out += bias.double()
    if resid is not None:
        out += resid.double().reshape(B, Ho, Wo, Cout)
        mag += resid.double().abs().reshape(B, Ho, Wo, Cout)
    slack = (ks * ks * Cin + 2) * U32 * mag
    if out_nchw:
        return out.permute(0, 3, 1, 2), slack.permute(0, 3, 1, 2)
    return out, slack


# ---------------------------------------------------------------------------------------------------------------- GroupNorm
GN_MUTATIONS = ("eps_1e-5", "unbiased_variance", "group_c_mod_32", "last_chunk_dropped")


def silu64(v):
    return v / (1 + torch.exp(-v))


def gn_ref(x, gamma, beta, silu, mutation=None, chunk=GN_PIX):
    """GroupNorm(32, eps 1e-6) (+ SiLU) in float64 of x [B, HW, C] -> dict: y (the output), v (before SiLU), and per (image, group)
    [B, 1, 32, 1]: mean, var, rstd, m1 = mean |x|, m2 = mean x^2.  chunk: the statistics' pixel chunk, which the mutation
    last_chunk_dropped leaves out of them (256 for gn_stats_kernel, 32 for the conv epilogue)."""
    B, HW, C = x.shape
    cg = C // 32
    xd = x.double()
    c = torch.arange(C, device=x.device)
    perm = torch.argsort(c % 32 if mutation == "group_c_mod_32" else c // cg, stable=True)   # channels grouped
    xg = xd[..., perm].reshape(B, HW, 32, cg)
    xs = xg
    if mutation == "last_chunk_dropped":
        xs = xg[:, :(math.ceil(HW / chunk) - 1) * chunk]
    n = xs.shape[1] * cg
    mean = xs.mean((1, 3), keepdim=True)
    var = ((xs - mean) ** 2).sum((1, 3), keepdim=True) / (n - 1 if mutation == "unbiased_variance" else n)
    rstd = 1 / torch.sqrt(var + (1e-5 if mutation == "eps_1e-5" else GN_EPS))
    inv = torch.argsort(perm)
    v = ((xg - mean) * rstd).reshape(B, HW, C)[..., inv] * gamma.double() + beta.double()
    return dict(y=silu64(v) if silu else v, v=v, mean=mean, var=var, rstd=rstd, m1=xs.abs().mean((1, 3), keepdim=True),
                m2=(xs * xs).mean((1, 3), keepdim=True), perm=perm, inv=inv)


def gn_depth(C, fused):
    return C // 32 + (5 if fused else 0)


def gn_slack(x, gamma, beta, silu, ref, fused, fast, cancel=True):
    """the bound of the module docstring [B, HW, C] for the output of a GroupNorm path: fused (statistics from the conv epilogue) or
    not, fast (gn_apply_f16_kernel, __expf) or exact (gn_apply_kernel, expf).  cancel=False: the variance term without 1 + r^2."""
    B, HW, C = x.shape
    cg = C // 32
    d = gn_depth(C, fused) * U32
    mean, var, rstd, m1, m2 = (ref[k] for k in ("mean", "var", "rstd", "m1", "m2"))
    dmean = d * m1 + 2.0 ** -45 * m1
    dvar = d * (m2 + 2 * mean.abs() * m1) if cancel else 3 * d * var
    dvar = dvar + 2.0 ** -45 * m2
    drel = dvar / (2 * (var + GN_EPS)) + U32 / 2
    dmu = dmean + U32 / 2 * mean.abs()
    group = lambda t: t.expand(B, 1, 32, cg).reshape(B, 1, C)[..., ref["inv"]]      # per-group value at each channel
    ga, be = gamma.double().abs(), beta.double().abs()
    dx = (x.double() - group(mean)).abs()
    rg = group(rstd) * ga
    v = ref["v"]
    if fast:
        sv = rg * (dx * (group(drel) + 3 * U32) + group(dmu)) + 2 * U32 * v.abs()
    else:
        sv = rg * (dx * (group(drel) + U32) + group(dmu)) + U32 * (be + rg * group(mean).abs()) + U32 * v.abs()
    if not silu:
        return sv
    e = (4 + 2.35 * v.abs()) * U32 if fast else 4 * U32
    return 1.1 * sv + (e + 3 * U32) * ref["y"].abs()


def gn_inputs(B, HW, C, seed, r=None, device="cpu"):
    """(x [B, HW, C] f32, gamma, beta [C]).  Group g of image b: mean mu_bg (N(0, 2^2), or +-r with r given: r = |mean| / std), std
    in [0.5, 2) (1 with r given), except group 0 of image 0, which is the constant 0.75 (its sums are exact, var = 0, rstd = 1000).
    gamma in [0.5, 1.5) and beta N(0, 1), per channel."""
    g = torch.Generator().manual_seed(seed)
    cg = C // 32
    if r is None:
        mu = torch.randn(B, 1, 32, 1, generator=g) * 2
        sd = torch.rand(B, 1, 32, 1, generator=g) * 1.5 + 0.5
    else:
        mu = r * (torch.randint(0, 2, (B, 1, 32, 1), generator=g) * 2 - 1).float()
        sd = torch.ones(B, 1, 32, 1)
    x = (torch.randn(B, HW, 32, cg, generator=g) * sd + mu).reshape(B, HW, C)
    x[0, :, :cg] = 0.75
    gamma = torch.rand(C, generator=g) + 0.5
    beta = torch.randn(C, generator=g)
    return x.to(device), gamma.to(device), beta.to(device)


def gn_needles(B, HW, C, seed, device="cpu"):
    """gn_inputs with group 1 of every image at std 1e-3 (var 1e-6: eps decides rstd) and the last pixel of every image offset by
    +40 in groups 2..31 (the chunk it sits in moves their mean and variance)"""
    x, gamma, beta = gn_inputs(B, HW, C, seed)
    cg = C // 32
    x[:, :, cg:2 * cg] = 0.3 + 1e-3 * torch.randn(B, HW, cg, generator=torch.Generator().manual_seed(seed + 1))
    if HW > 1:
        x[:, -1, 2 * cg:] += 40.0
    return x.to(device), gamma.to(device), beta.to(device)


def half_gap(hi, lo):
    """float64: half the gap between fp16 hi and its neighbour on lo's side"""
    b = hi.view(torch.int16).int()
    mag = b & 0x7FFF
    toward = torch.where((lo >= 0) == (b >= 0), mag + 1, mag - 1).clamp_min(0)      # neighbour magnitude on lo's side
    nb = torch.where(b < 0, toward | 0x8000, toward).to(torch.int16).view(torch.float16)
    g = (nb.double() - hi.double()).abs() / 2
    return torch.where(mag == 0, torch.full_like(g, 2.0 ** -25), g)


def split_ok(hi, lo):
    """hi is a nearest fp16 of float(hi) + float(lo): |lo| <= half the gap on lo's side"""
    return bool((lo.double().abs() <= half_gap(hi, lo)).all())


# ---------------------------------------------------------------------------------------------------------------- cast
CAST_MUTATIONS = ("last_row_wrong_source", "last_col_wrong_source")


def cast_ref(x, upsample, with_lo, mutation=None):
    """x [B, H, W, C] f32 -> (hi, lo or None) fp16, bit for bit the kernel's output"""
    hi = x.half()
    lo = (x - hi.float()).half() if with_lo else None
    up = lambda t: t.repeat_interleave(2, 1).repeat_interleave(2, 2) if upsample else t
    hi, lo = up(hi), up(lo) if lo is not None else None
    for t in (hi, lo):
        if t is None:
            continue
        if mutation == "last_row_wrong_source" and t.shape[1] > 2:
            t[:, -1] = t[:, -3]
        elif mutation == "last_col_wrong_source" and t.shape[2] > 2:
            t[:, :, -1] = t[:, :, -3]
    return hi, lo


# ---------------------------------------------------------------------------------------------------------------- attention
ATTN_MUTATIONS = ("scale_one_eighth", "last_key_dropped", "softmax_over_queries")


def attn_scale(C):
    """the kernel's scale: 1 / sqrt(C) in double, cast to float"""
    return float(torch.tensor(1.0 / math.sqrt(C), dtype=torch.float32))


def attn_ref(qkv, B, HW, C, mutation=None, rows=1024):
    """(ref, slack) [B, HW, C] float64 of rqb200_dbg_vae_attn on qkv [B, HW, 3C] f32, in chunks of query rows"""
    x = qkv.reshape(B, HW, 3, C).double()
    q, k, v = x[:, :, 0], x[:, :, 1], x[:, :, 2]
    s = 0.125 if mutation == "scale_one_eighth" else attn_scale(C)
    ref = torch.empty(B, HW, C, dtype=torch.float64, device=qkv.device)
    slack = torch.empty_like(ref)
    for i0 in range(0, HW, rows):
        qi = q[:, i0:i0 + rows]
        S = (qi @ k.transpose(1, 2)) * s
        if mutation == "last_key_dropped":
            S[..., -1] = float("-inf")
        m = S.amax(-1, keepdim=True)
        P = torch.softmax(S, -1)
        A = (math.ceil(C / 32) + 6) * U32 * s * (qi.abs() @ k.abs().transpose(1, 2))
        dlt = 4 * U32 + A + A.amax(-1, keepdim=True) + U32 * (m - S).nan_to_num(posinf=0.0)
        ds = dlt.amax(-1, keepdim=True) + (math.ceil(HW / 256) + 10) * U32
        ref[:, i0:i0 + rows] = P @ v
        slack[:, i0:i0 + rows] = (P * dlt) @ v.abs() + (ds + (HW + 2) * U32) * (P @ v.abs())
    if mutation == "softmax_over_queries":           # column-normalised weights need every query row at once; the slack stays
        ref = torch.softmax((q @ k.transpose(1, 2)) * s, dim=1) @ v
    return ref, slack


def attn_inputs(B, HW, C, seed, needles=False, device="cpu"):
    """qkv [B, HW, 3C] f32: q, k, v N(0, 1).  needles: query i by i % 5 -- 0: one dominant random key (score 16), 1: q = 0 (all scores
    equal), 2: q * 30 (|scores| up to ~100), 3: the last key dominant (score 16), 4: as drawn (scores ~ N(0, 1))"""
    g = torch.Generator().manual_seed(seed)
    q, k, v = (torch.randn(B, HW, C, generator=g, dtype=torch.float64) for _ in range(3))
    if needles:
        s = attn_scale(C)
        for i in range(HW):
            rule = i % 5
            if rule == 0 or rule == 3:
                j = HW - 1 if rule == 3 else int(torch.randint(0, HW, (1,), generator=g))
                q[:, i] = k[:, j] * 16.0 / (s * (k[:, j] * k[:, j]).sum(-1, keepdim=True))
            elif rule == 1:
                q[:, i] = 0
            elif rule == 2:
                q[:, i] *= 30
    return torch.cat([q, k, v], -1).float().to(device)
