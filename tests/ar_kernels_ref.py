"""float64 references of the fast AR tier's non-GEMM kernels (csrc/ar_fast.cu: step attention, prefill attention, LayerNorm with the
split-K reduction, act_reduce), the error bounds the tests hold them to, and the needle inputs on which a named mistake becomes visible.

Every reference starts from the operands the kernel sees: the 16-bit-rounded q / k / v and the fp32 sums, formed here in the kernels'
order (fp32 additions are correctly rounded on both sides, so those sums are bit-exact).

Tolerance of a 16-bit output o against its reference r: ulp16(|r| + slack) + slack -- the final rounding to 16 bits (half an ulp, a
whole one when the fp32 value crossed a binade) plus `slack`, a bound on the kernel's fp32 error before that rounding:
  attention   max|v| * u * (16 sqrt(n) + 134 a + 11 + 16 (n / 64 + 1))  with u = 2^-24, n attended keys, a = max_j sum_i |q_i k_ji| / 8:
              the fp32 sums of p_j v_j and of p_j over n terms (probabilistic bound 8 sqrt(n) u each), a 64-term fp32 score dot
              (8 * 8 u * a, entering the weights and the max twice), __expf (2^-22 relative plus the rounded argument, 1.44 |s - m| u),
              the reciprocal and the final product (3 u), and per 64-key tile the online softmax's rescale (16 u);
              prefill_attn_flash_kernel also rounds P to 16 bits before P V: + max|v| * (2^-11 fp16 / 2^-8 bf16), and fp16 P below
              2^-24 flushes: + n 2^-25 max|v|;
  LayerNorm   |g| rstd dmean + |g d rstd| (depth / 2 + 6) u + 2 u (|g d rstd| + |b|)  with d = x - mean, dmean = (depth + 1) u mean|x|:
              the fp32 reduction tree of `depth` sequential additions for the mean and the variance (16 for ln_reduce_kernel, NV + 8
              for ln_rows_kernel<NV>), rsqrtf (2 ulp), the normalisation's three roundings;
  GELU        (4 |x| + 2 |r|) u: erff (2 ulp of a value below 1), its rounded argument, 1 + erf and the products.
"""
import math

import torch

U32 = 2.0 ** -24
DT = {0: torch.float16, 1: torch.bfloat16}
MANT = {0: 10, 1: 7}                       # explicit mantissa bits
MIN_SUB = {0: 2.0 ** -24, 1: 2.0 ** -133}  # smallest subnormal
P_ROUND = {0: 2.0 ** -11, 1: 2.0 ** -8}    # half-ulp relative rounding of P in the flash kernel
LN_EPS = 1e-5


def r16(x, fmt):
    """x rounded to the 16-bit format (round to nearest even, as __floats2half2_rn / __floats2bfloat162_rn)"""
    return x.to(DT[fmt])


def split_sum_f32(*terms):
    """the fp32 sum of the given terms left to right (None terms skipped): the kernels' split-K order bias, p_0, ..., p_{S-1}"""
    acc = None
    for t in terms:
        if t is None:
            continue
        acc = t.float().clone() if acc is None else acc + t.float()
    return acc


def ulp16(x, fmt):
    """spacing of the 16-bit format at |x| (float64 tensor)"""
    a = x.abs().double()
    e = torch.frexp(a)[1].double() - 1                   # floor(log2 |x|) for x != 0
    u = torch.pow(2.0, e - MANT[fmt]).clamp_min(MIN_SUB[fmt])
    return torch.where(a > 0, u, torch.full_like(u, MIN_SUB[fmt]))


def tol16(ref, slack, fmt):
    return ulp16(ref.abs() + slack, fmt) + slack


def excess(got, ref, tol):
    """max over elements of |got - ref| - tol (<= 0: every element within tolerance); NaN counts as a miss"""
    d = (got.double() - ref.double()).abs() - tol
    return float(torch.nan_to_num(d, nan=float("inf")).max())


# ---------------------------------------------------------------------------------------------------------------- attention
def attend(q, k, v, mask):
    """q [P, Tq, 64], k / v [P, Tk, 64] float64, mask [Tq, Tk] or [P, Tq, Tk] (True = attended) -> softmax(q k^T / 8) v [P, Tq, 64];
    a row with no attended key gives 0 (a mutated mask may empty one)"""
    s = (q @ k.transpose(1, 2)) / 8
    s = s.masked_fill(~mask, float("-inf"))
    m = s.amax(-1, keepdim=True).clamp_min(-1e300)
    p = torch.exp(s - m).masked_fill(~mask, 0.0)
    den = p.sum(-1, keepdim=True)
    return (p @ v) / torch.where(den > 0, den, torch.ones_like(den))


def attn_slack(q, k, v, mask, fmt, flash=False):
    """the fp32 error bound of the module docstring, per query row: [P, Tq, 1]"""
    n = mask.expand(q.shape[0], q.shape[1], k.shape[1]).sum(-1, keepdim=True).double()
    a = ((q.abs() @ k.abs().transpose(1, 2)) / 8).masked_fill(~mask, 0.0).amax(-1, keepdim=True)
    vmax = v.abs().amax(dim=(1, 2)).view(-1, 1, 1)
    s = U32 * (16 * n.sqrt() + 134 * a + 11 + 16 * (n / 64 + 1))
    if flash:
        s = s + P_ROUND[fmt] + (n * 2.0 ** -25 if fmt == 0 else 0.0)
    return vmax * s


PREFILL_MUTATIONS = ("exclude_diagonal", "include_next_key", "drop_tile_edge_key", "neighbour_group")


def prefill_mask(T, mutation=None, device="cpu"):
    m = torch.ones(T, T, dtype=torch.bool, device=device).tril()
    if mutation == "exclude_diagonal":
        m = m.tril(-1)
    elif mutation == "include_next_key":
        m = torch.ones(T, T, dtype=torch.bool, device=device).tril(1)
    elif mutation == "drop_tile_edge_key":
        m[:, 63::64] = False                              # key 64k - 1 for every k
    return m


def prefill_ref(qkv, G, T, E, fmt, mutation=None, flash=None, max_bytes=1 << 27):
    """causal attention of the batched passes over qkv [T*G, 3E] (16-bit, token-major) -> (ref [T*G, E], slack [T*G, E]) float64, in
    chunks of (group, head) pairs of about max_bytes of float64 operands and scores.  flash: the T > 8 kernel's bound (default: T > 8)."""
    if flash is None:
        flash = T > 8
    nh = E // 64
    x = qkv.view(T, G, 3, nh, 64)
    mask = prefill_mask(T, mutation, qkv.device)
    ref = torch.empty(T, G * nh, 64, dtype=torch.float64, device=qkv.device)
    slack = torch.empty(T, G * nh, 1, dtype=torch.float64, device=qkv.device)
    step = max(1, max_bytes // (8 * T * (4 * T + 3 * 64)))
    for p0 in range(0, G * nh, step):
        p = torch.arange(p0, min(G * nh, p0 + step), device=qkv.device)
        g, h = p // nh, p % nh
        gk = (g + 1) % G if mutation == "neighbour_group" else g      # keys / values of group g+1
        q, k, v = (x[:, gg, i, h].double().permute(1, 0, 2) for i, gg in ((0, g), (1, gk), (2, gk)))
        ref[:, p0:p0 + len(p)] = attend(q, k, v, mask).permute(1, 0, 2)
        slack[:, p0:p0 + len(p)] = attn_slack(q, k, v, mask, fmt, flash).permute(1, 0, 2)
    return ref.view(T * G, E), slack.expand(T, G * nh, 64).reshape(T * G, E)


STEP_MUTATIONS = ("drop_key_t_minus_1", "drop_new_token", "omit_last_partial", "neighbour_head_keys")


def step_qkv(part, bqkv, fmt, n_parts=None):
    """q, k, v of the new token: round16(bqkv + part[0] + ... + part[n_parts-1]) in fp32, split order -> three [B, E] 16-bit tensors"""
    S = part.shape[0] if n_parts is None else n_parts
    x = r16(split_sum_f32(bqkv, *[part[s] for s in range(S)]), fmt)
    E = bqkv.numel() // 3
    return x[:, :E], x[:, E:2 * E], x[:, 2 * E:]


def step_ref(part, bqkv, kc, vc, t, fmt, mutation=None, b_chunk=None):
    """one step attention (rqb200_dbg_attn_step) against the caches as they were BEFORE the launch (kc / vc [B, nh, Tmax, 64] 16-bit,
    rows [0, t) read) -> (ref [B, E], slack [B, E]) float64"""
    B, nh = kc.shape[0], kc.shape[1]
    E = nh * 64
    q, kn, vn = step_qkv(part, bqkv, fmt, part.shape[0] - 1 if mutation == "omit_last_partial" else None)
    mask = torch.ones(1, t + 1, dtype=torch.bool, device=kc.device)
    if mutation == "drop_key_t_minus_1":
        mask[0, t - 1] = False
    elif mutation == "drop_new_token":
        mask[0, t] = False
    if b_chunk is None:
        b_chunk = max(1, (1 << 28) // (nh * (t + 1) * 64 * 8 * 3))
    ref = torch.empty(B, E, dtype=torch.float64, device=kc.device)
    slack = torch.empty_like(ref)
    for b0 in range(0, B, b_chunk):
        bs = slice(b0, b0 + b_chunk)
        kk, vv = kc[bs, :, :t], vc[bs, :, :t]
        if mutation == "neighbour_head_keys":
            kk = kk.roll(-1, 1)
        nb = kk.shape[0]
        keys = torch.cat([kk.double(), kn[bs].double().view(nb, nh, 1, 64)], 2).view(nb * nh, t + 1, 64)
        vals = torch.cat([vv.double(), vn[bs].double().view(nb, nh, 1, 64)], 2).view(nb * nh, t + 1, 64)
        qq = q[bs].double().view(nb * nh, 1, 64)
        ref[bs] = attend(qq, keys, vals, mask).view(nb, E)
        slack[bs] = attn_slack(qq, keys, vals, mask, fmt).expand(-1, -1, 64).reshape(nb, E)
    return ref, slack


def needle_query(gen, n, scale=2.0, score=16.0):
    """n query vectors q (N(0, scale^2) entries) and their needle keys k* = q * 8 score / |q|^2, so that q . k* / 8 = score"""
    q = torch.randn(n, 64, generator=gen, dtype=torch.float64) * scale
    return q, q * (8 * score) / (q * q).sum(-1, keepdim=True)


def step_inputs(B, E, Tmax, t, S, fmt, seed, needles=False, noise=0.1):
    """(part [S, B, 3E] f32, bqkv [3E] f32, kc, vc [B, nh, Tmax, 64] 16-bit) on the CPU.  Cached rows [0, t) random, rows [t, Tmax) NaN
    (a kernel that reads past row t - 1, or a cache row it did not write, shows NaN).  needles: in head h of every row, the query's
    needle key sits at cache row t - 1 (h % 4 == 0), at the new token (1), at a random cached row (2) or nowhere (3); the needle q / k / v
    come in partial 0, the other partials are N(0, noise^2)."""
    g = torch.Generator().manual_seed(seed)
    nh = E // 64
    part = torch.randn(S, B, 3 * E, generator=g) * (noise if needles else 1.0 / math.sqrt(max(S, 1)))
    bqkv = torch.randn(3 * E, generator=g) * (noise if needles else 0.5)
    kc = torch.randn(B, nh, Tmax, 64, generator=g)
    vc = torch.randn(B, nh, Tmax, 64, generator=g)
    kc[:, :, t:] = float("nan")
    vc[:, :, t:] = float("nan")
    if needles:
        q, ks = needle_query(g, B * nh)
        q, ks = q.float().view(B, nh, 64), ks.float().view(B, nh, 64)
        knew = torch.randn(B, nh, 64, generator=g)
        for h in range(nh):
            rule = h % 4
            if rule == 0 and t > 0:
                kc[:, h, t - 1] = ks[:, h]
            elif rule == 1:
                knew[:, h] = ks[:, h]
            elif rule == 2 and t > 0:
                j = int(torch.randint(0, t, (1,), generator=g))
                kc[:, h, j] = ks[:, h]
        part[0, :, :E] = q.reshape(B, E)
        part[0, :, E:2 * E] = knew.reshape(B, E)
        part[0, :, 2 * E:] = torch.randn(B, E, generator=g)
    return part, bqkv, r16(kc, fmt), r16(vc, fmt)


def prefill_needles(G, T, E, fmt, seed):
    """qkv [T*G, 3E] 16-bit whose query row r of head h puts its weight on one key: r itself (h % 4 == 0), r + 1 (1; the next key,
    outside the causal window), the last key 64k - 1 of the tile before r's (2; rows >= 64) or a random key <= r (3)"""
    g = torch.Generator().manual_seed(seed)
    nh = E // 64
    k = torch.randn(G, nh, T, 64, generator=g, dtype=torch.float64)
    v = torch.randn(G, nh, T, 64, generator=g, dtype=torch.float64)
    q = torch.empty_like(k)
    for h in range(nh):
        for r in range(T):
            rule = h % 4
            j = r if rule == 0 else min(r + 1, T - 1) if rule == 1 else (r // 64) * 64 - 1 if (rule == 2 and r >= 64) else \
                int(torch.randint(0, r + 1, (1,), generator=g))
            kk = k[:, h, j]
            q[:, h, r] = kk * (8 * 16.0) / (kk * kk).sum(-1, keepdim=True)     # q . k_j / 8 = 16
    tm = lambda x: x.permute(2, 0, 1, 3).reshape(T * G, E)
    return r16(torch.cat([tm(q), tm(k), tm(v)], 1), fmt)


# ---------------------------------------------------------------------------------------------------------------- LayerNorm / GELU
LN_MUTATIONS = ("omit_last_partial", "eps_outside_sqrt", "unbiased_variance")


def layer_norm64(x, g, b, mutation=None):
    """LayerNorm (eps 1e-5) in float64 of the fp32 rows x [rows, E]; -> (y, mean, rstd)"""
    x = x.double()
    mean = x.mean(-1, keepdim=True)
    d = x - mean
    E = x.shape[-1]
    var = (d * d).sum(-1, keepdim=True) / (E - 1 if mutation == "unbiased_variance" else E)
    rstd = 1.0 / (var.sqrt() + LN_EPS) if mutation == "eps_outside_sqrt" else 1.0 / (var + LN_EPS).sqrt()
    return d * rstd * g.double() + b.double(), mean, rstd


def ln_slack(x, g, b, depth):
    """the LayerNorm bound of the module docstring for rows x [rows, E] of a kernel whose reductions are `depth` additions deep"""
    x = x.double()
    y, mean, rstd = layer_norm64(x, torch.ones_like(g), torch.zeros_like(b))
    gd = (g.double() * y).abs()
    dmean = (depth + 1) * U32 * x.abs().mean(-1, keepdim=True)
    return g.double().abs() * rstd * dmean + gd * (depth / 2 + 6) * U32 + 2 * U32 * (gd + b.double().abs())


def ln_depth(form, E):
    """addition depth of the fp32 reduction tree: ln_reduce_kernel<384, 3> (form 1) or ln_rows_kernel<NV> (form 2)"""
    if form == 1:
        return 16
    nv = -(-E // 128)
    return next(n for n in (8, 12, 20, 36) if nv <= n) + 8


def ln_rows_ref(x_out, g, b, form, mutation_x=None, mutation=None, chunk=2048):
    """(ref, slack) [rows, E] float64 of xn = LN(x) in row chunks; x = x_out, or mutation_x (a mutated sum) for the reference"""
    x = x_out if mutation_x is None else mutation_x
    ref = torch.empty(x.shape, dtype=torch.float64, device=x.device)
    slack = torch.empty_like(ref)
    depth = ln_depth(form, x.shape[1])
    for r0 in range(0, x.shape[0], chunk):
        ref[r0:r0 + chunk] = layer_norm64(x[r0:r0 + chunk], g, b, mutation)[0]
        slack[r0:r0 + chunk] = ln_slack(x_out[r0:r0 + chunk], g, b, depth)
    return ref, slack


def ln_rows_input(rows, E, seed, device="cpu"):
    """[rows, E] f32 rows N(0, 1), with row 1 at mean 10^3 (std 1), row 2 carrying one outlier of +300 and row 3 of variance ~1e-8
    (0.5 + small multiples of 2^-14: where eps decides rstd), when there are such rows"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, E, generator=g)
    if rows > 1:
        x[1] += 1000.0
    if rows > 2:
        x[2, E // 3] += 300.0
    if rows > 3:
        x[3] = 0.5 + torch.randint(-3, 4, (E,), generator=g).float() * 2.0 ** -14
    return x.to(device)


def dyadic(n, seed, scale=1024):
    """n values that are multiples of 1/scale (exact in fp32, and so are their sums and differences with 0.5)"""
    g = torch.Generator().manual_seed(seed)
    return torch.round(torch.randn(n, generator=g) * scale) / scale


def gelu64(x, mutation=None):
    x = x.double()
    if mutation == "tanh_gelu":
        return 0.5 * x * (1 + torch.tanh(math.sqrt(2 / math.pi) * (x + 0.044715 * x ** 3)))
    return 0.5 * x * (1 + torch.erf(x / math.sqrt(2)))


def gelu_slack(x, ref):
    return (4 * x.double().abs() + 2 * ref.abs()) * U32
