"""The fast AR tier's non-GEMM kernels (csrc/ar_fast.cu), one launch each through the engine's own launchers (rqb200_dbg_attn_step,
rqb200_dbg_prefill_attn, rqb200_dbg_ln, rqb200_dbg_act_reduce), against the float64 references of tests/ar_kernels_ref.py at the
shapes where the kernels switch form, tile or pass: outputs within the derived tolerance (ar_kernels_ref's docstring), cache writes and
fp32 sums bit for bit, every other byte untouched, and for each family a set of named mistakes that the tolerance rejects."""
import pytest
import torch

from rqvae import _native as N
from tests import ar_kernels_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda"
GUARD = 512                     # elements behind every output buffer that no launch may touch


def bits(x):
    return x.view(torch.int16) if x.element_size() == 2 else x.view(torch.int32)


def guarded(x):
    """x copied into the front of a device buffer with GUARD sentinel elements behind it -> (buffer, view of x's shape)"""
    full = torch.empty(x.numel() + GUARD, dtype=x.dtype, device=DEV)
    full[:x.numel()].copy_(x.reshape(-1))
    bits(full)[x.numel():] = 0x5A5A
    return full, full[:x.numel()].view(x.shape)


def guard_intact(full, n):
    return bool((bits(full)[n:] == 0x5A5A).all())


def within(got, ref, slack, fmt, what):
    e = R.excess(got, ref, R.tol16(ref, slack, fmt))
    assert e <= 0, "%s: %.3g beyond tolerance" % (what, e)


# ---------------------------------------------------------------------------------------------------------------- step attention
def run_step(form, part, bqkv, kc, vc, B, E, Tmax, t, fmt, t_dev=None):
    """(rc, att, kc_buf, vc_buf, att_buf): one launch on fresh guarded copies of the caches"""
    kfull, kcd = guarded(kc)
    vfull, vcd = guarded(vc)
    afull, att = guarded(torch.full((B, E), float("nan"), dtype=R.DT[fmt]))
    td = torch.tensor([t], dtype=torch.int32, device=DEV) if t_dev else None
    rc = N.lib().rqb200_dbg_attn_step(form, N.ptr(part), part.shape[0], N.ptr(bqkv), N.ptr(kcd), N.ptr(vcd), N.ptr(att), B, E, Tmax,
                                      N.ptr(td), -1 if t_dev else t, fmt, N.stream_ptr())
    torch.cuda.synchronize()
    return rc, att, kfull, vfull, afull


def check_step(form, B, E, Tmax, t, S, fmt, seed, needles=False):
    """one (form, shape, fmt) case, t from the host and from the device, each launched twice; returns the first launch's att and the
    reference"""
    part, bqkv, kc, vc = R.step_inputs(B, E, Tmax, t, S, fmt, seed, needles)
    part, bqkv = part.to(DEV), bqkv.to(DEV)
    nh, n = E // 64, kc.numel()
    ref, slack = R.step_ref(part, bqkv, kc.to(DEV), vc.to(DEV), t, fmt)
    _, kn, vn = R.step_qkv(part, bqkv, fmt)
    kc_want, vc_want = kc.clone(), vc.clone()                     # the caches after the step: row t = the new k / v, nothing else
    kc_want[:, :, t] = kn.view(B, nh, 64).cpu()
    vc_want[:, :, t] = vn.view(B, nh, 64).cpu()
    first = None
    for t_dev in (False, True):
        for rep in range(2):
            rc, att, kfull, vfull, afull = run_step(form, part, bqkv, kc, vc, B, E, Tmax, t, fmt, t_dev)
            N.check(rc, "dbg_attn_step")
            what = "form %d B %d E %d Tmax %d t %d S %d fmt %d t_dev %d" % (form, B, E, Tmax, t, S, fmt, t_dev)
            assert torch.equal(bits(kfull[:n]).cpu(), bits(kc_want).reshape(-1)), what + ": K cache"
            assert torch.equal(bits(vfull[:n]).cpu(), bits(vc_want).reshape(-1)), what + ": V cache"
            assert guard_intact(kfull, n) and guard_intact(vfull, n) and guard_intact(afull, B * E), what + ": guard"
            if first is None:
                within(att, ref, slack, fmt, what)
                first = att.clone()
            else:                                                 # run-to-run and t source: the same bits
                assert torch.equal(bits(att), bits(first)), what + ": not bit-identical to the first launch"
    return first, (part, bqkv, kc, vc, ref, slack)


STEP_T = [0, 1, 7, 31, 32, 33, 63, 64, 65, 127, 128, 319, 320]
BE = [(1, 128), (3, 128), (64, 1536), (16, 4608)]      # (1, 128) and (3, 128): part of attn_fast_kernel's last CTA idle
SPLITS = [1, 3, 11, 24]


def step_cases():
    """every t of each form at one (B, E) and S, cycling through both lists; Tmax alternates between the tightest cache (t + 1; at
    least 16 for form 2, which the engine runs from there) and the form's largest (321 / 2048).  t = 1023 / 2047 need Tmax = 2048; the
    (64, 1536) cache there is 2 x 403 MB, the largest case."""
    cases, i = [], 0
    for form in (2, 1):
        for t in STEP_T + ([1023, 2047] if form == 1 else []):
            B, E = (64, 1536) if t == 2047 else (3, 128) if t == 1023 else BE[i % 4]
            Tmax = 2048 if t >= 1023 else (max(t + 1, 16) if i % 2 == 0 else (321 if form == 2 else 2048 if B * E <= 3 * 128 else 400))
            cases.append((form, B, E, Tmax, t, SPLITS[(i + i // 4) % 4]))
            i += 1
    for D in (1, 4, 8):                                    # the head stack: Tmax = D rows, attn_fast_kernel
        for t in sorted({0, D // 2, D - 1}):
            B, E = BE[i % 4]
            cases.append((1, B, E, D, t, SPLITS[i % 4]))
            i += 1
    return cases


@pytest.mark.parametrize("form,B,E,Tmax,t,S", step_cases())
@pytest.mark.parametrize("fmt", [0, 1])
def test_step_attention(form, B, E, Tmax, t, S, fmt):
    check_step(form, B, E, Tmax, t, S, fmt, seed=1000 * t + 7 * B + S)


@pytest.mark.parametrize("Tmax", [15, 16, 321, 322])
@pytest.mark.parametrize("fmt", [0, 1])
def test_step_attention_form_choice(Tmax, fmt):
    """form 0 (the engine's choice) is attn_fast2_kernel exactly for 16 <= Tmax <= 321: bit for bit the forced form"""
    want = 2 if 16 <= Tmax <= 321 else 1
    B, E, t, S = 16, 1536, Tmax - 1, 4
    part, bqkv, kc, vc = R.step_inputs(B, E, Tmax, t, S, fmt, seed=Tmax)
    part, bqkv = part.to(DEV), bqkv.to(DEV)
    outs = []
    for form in (0, want):
        rc, att, kfull, vfull, _ = run_step(form, part, bqkv, kc, vc, B, E, Tmax, t, fmt)
        N.check(rc, "dbg_attn_step")
        outs.append((bits(att).clone(), bits(kfull).clone(), bits(vfull).clone()))
    assert all(torch.equal(a, b) for a, b in zip(*outs))
    if Tmax > 321:                                         # form 2 refuses more than 320 cached rows
        rc, *_ = run_step(2, part, bqkv, kc, vc, B, E, Tmax, t, fmt)
        assert rc == N.EINVAL


@pytest.mark.parametrize("form", [1, 2])
@pytest.mark.parametrize("fmt", [0, 1])
def test_step_attention_rejects_mutations(form, fmt):
    """needle inputs (tests/ar_kernels_ref.step_inputs): the kernel is within tolerance of the reference and outside it for each mistake"""
    B, E, Tmax, t, S = 4, 256, 100, 70, 3
    att, (part, bqkv, kc, vc, _, _) = check_step(form, B, E, Tmax, t, S, fmt, seed=11, needles=True)
    for mutation in R.STEP_MUTATIONS:
        mut, mslack = R.step_ref(part, bqkv, kc.to(DEV), vc.to(DEV), t, fmt, mutation=mutation)
        assert R.excess(att, mut, R.tol16(mut, mslack, fmt)) > 0, mutation


# ---------------------------------------------------------------------------------------------------------------- prefill attention
def run_prefill(qkv, G, T, E, Tmax, fmt, with_cache=True, seed=0):
    nh = E // 64
    gen = torch.Generator(DEV).manual_seed(seed)
    cache0 = [torch.randn(G, nh, Tmax, 64, generator=gen, device=DEV).to(R.DT[fmt]) for _ in range(2)]
    bufs = [guarded(c) for c in cache0] if with_cache else [(None, None), (None, None)]
    afull, att = guarded(torch.full((T * G, E), float("nan"), dtype=R.DT[fmt]))
    N.check(N.lib().rqb200_dbg_prefill_attn(N.ptr(qkv), N.ptr(bufs[0][1]), N.ptr(bufs[1][1]), N.ptr(att), G, T, E, Tmax, fmt,
                                            N.stream_ptr()), "dbg_prefill_attn")
    torch.cuda.synchronize()
    assert guard_intact(afull, T * G * E)
    return att, cache0, bufs


def prefill_cases():
    """each T with one case of G > 1 and Tmax = T + 37 and one of G = 64, E = 128, Tmax = T, in alternating formats"""
    cases = []
    for i, T in enumerate([1, 2, 4, 5, 8, 9, 63, 64, 65, 127, 128, 129, 320, 1000, 2047, 2048]):
        cases.append((T, 64 if T <= 128 else 3, 1536, T + 37, i % 2))
        cases.append((T, 64, 128, T, (i + 1) % 2))
    cases += [(4, 4096, 1536, 4, 0), (4, 4096, 1536, 4, 1)]     # the forward's head stack (D = 4 tokens per group)
    return cases


@pytest.mark.parametrize("T,G,E,Tmax,fmt", prefill_cases())
def test_prefill_attention(T, G, E, Tmax, fmt):
    gen = torch.Generator(DEV).manual_seed(T * 131 + G)
    qkv = torch.randn(T * G, 3 * E, generator=gen, device=DEV).to(R.DT[fmt])
    att, cache0, bufs = run_prefill(qkv, G, T, E, Tmax, fmt, seed=T)
    ref, slack = R.prefill_ref(qkv, G, T, E, fmt)
    within(att, ref, slack, fmt, "T %d G %d E %d fmt %d" % (T, G, E, fmt))
    nh, n = E // 64, G * (E // 64) * Tmax * 64
    for m, (full, c) in enumerate(bufs):                   # rows [0, T): the K / V slices of qkv; rows [T, Tmax) and the guard untouched
        want = cache0[m].clone()
        want[:, :, :T] = qkv[:, (m + 1) * E:(m + 2) * E].view(T, G, nh, 64).permute(1, 2, 0, 3)
        assert torch.equal(bits(c), bits(want)), "K" if m == 0 else "V"
        assert guard_intact(full, n)
    att_nc, _, _ = run_prefill(qkv, G, T, E, Tmax, fmt, with_cache=False)
    assert torch.equal(bits(att_nc), bits(att))


@pytest.mark.parametrize("T", [8, 130])
@pytest.mark.parametrize("fmt", [0, 1])
def test_prefill_attention_rejects_mutations(T, fmt):
    G, E = 2, 256
    qkv = R.prefill_needles(G, T, E, fmt, seed=3).to(DEV)
    att, _, _ = run_prefill(qkv, G, T, E, T, fmt)
    ref, slack = R.prefill_ref(qkv, G, T, E, fmt)
    within(att, ref, slack, fmt, "needles")
    for mutation in R.PREFILL_MUTATIONS:
        if mutation == "drop_tile_edge_key" and T <= 64:
            continue                                       # (no key 63 to drop)
        mut, mslack = R.prefill_ref(qkv, G, T, E, fmt, mutation=mutation)
        assert R.excess(att, mut, R.tol16(mut, mslack, fmt)) > 0, mutation


# ---------------------------------------------------------------------------------------------------------------- LayerNorm
def ln_inputs(rows, E, S, fmt, seed, with_bias, with_extra):
    """x_in with the rows of ar_kernels_ref.ln_rows_input and a last row whose sum is exactly 0.5 everywhere (bias / extra / x_in dyadic,
    its partials 0): mean exactly 0.5, so xn = beta bit for bit"""
    x = R.ln_rows_input(rows, E, seed)
    part = torch.randn(S, rows, E, generator=torch.Generator().manual_seed(seed + 1)) / max(S, 1) ** 0.5
    bias = R.dyadic(E, seed + 2) if with_bias else None
    extra = R.dyadic(E, seed + 3) if with_extra else None
    c = rows - 1 if rows >= 5 else None
    if c is not None:
        part[:, c] = 0
        x[c] = 0.5 - (bias if bias is not None else 0) - (extra if extra is not None else 0)
    gen = torch.Generator().manual_seed(seed + 4)
    g, b = torch.rand(E, generator=gen) + 0.5, torch.randn(E, generator=gen)
    return x, part, bias, extra, g, b, c


def run_ln(form, x, part, bias, extra, g, b, fmt, in_place, with_xn, with_x_out=True):
    rows, E = x.shape
    S = part.shape[0] if part is not None else 0
    xfull, xd = guarded(x)
    ofull, od = (xfull, xd) if in_place else guarded(torch.zeros(rows, E)) if with_x_out else (None, None)
    nfull, xn = guarded(torch.zeros(rows, E, dtype=R.DT[fmt])) if with_xn else (None, None)
    d = lambda a: a.to(DEV) if a is not None else None
    pd, bd, ed, gd, bbd = d(part), d(bias), d(extra), d(g), d(b)
    N.check(N.lib().rqb200_dbg_ln(form, N.ptr(xd), N.ptr(pd), S, N.ptr(bd), N.ptr(ed), N.ptr(od), N.ptr(gd), N.ptr(bbd), N.ptr(xn),
                                  rows, E, fmt, N.stream_ptr()), "dbg_ln")
    torch.cuda.synchronize()
    n = rows * E
    assert guard_intact(xfull, n) and (ofull is None or guard_intact(ofull, n)) and (nfull is None or guard_intact(nfull, n))
    return od, xn, xd


def check_ln(form, x_sum, xn, g, b, fmt, c, what):
    for r0 in range(0, x_sum.shape[0], 2048):
        ref, slack = R.ln_rows_ref(x_sum[r0:r0 + 2048], g.to(DEV), b.to(DEV), 1 if form == 1 else 2)
        within(xn[r0:r0 + 2048], ref, slack, fmt, what)
    if c is not None:                                     # mean exactly 0.5: xn = beta
        assert torch.equal(bits(xn[c]), bits(R.r16(b.to(DEV), fmt))), what + ": constant row"


def ln_step_cases():
    rows, S, E = [1, 64, 256, 511], [0, 1, 11, 12, 13, 24], [128, 1536, 1664, 4608]
    return [(rows[i % 4], S[i % 6], E[(i + i // 4) % 4]) for i in range(12)]


@pytest.mark.parametrize("rows,S,E", ln_step_cases())
@pytest.mark.parametrize("pattern", ["ln1_first", "in_place", "no_xn"])
@pytest.mark.parametrize("fmt", [0, 1])
def test_ln_reduce(rows, S, E, pattern, fmt):
    """ln_reduce_kernel in the engine's argument patterns: block 0's LN1 (x_src + extra into x, no partials), LN1 / LN2 in place with
    the previous GEMM's partials and bias, and the stack's finalize without xn"""
    first = pattern == "ln1_first"
    x, part, bias, extra, g, b, c = ln_inputs(rows, E, 0 if first else S, fmt, rows + S + E, not first, first)
    x_out, xn, _ = run_ln(1, x, part, bias, extra, g, b, fmt, in_place=not first, with_xn=pattern != "no_xn")
    want = R.split_sum_f32(x, bias, *part, extra).to(DEV)
    assert torch.equal(bits(x_out), bits(want)), "x_out is not the fp32 sum in split order"
    if xn is not None:
        check_ln(1, want, xn, g, b, fmt, c, "ln_reduce rows %d S %d E %d %s" % (rows, S, E, pattern))


@pytest.mark.parametrize("E", [1024, 1152, 1536, 2560, 2688, 4608])     # both sides of every NV step (8, 12, 20, 36 float4 per lane)
@pytest.mark.parametrize("rows", [512, 1000, 8449, 20001])              # 8449, 20001: more rows than one pass of 132 * 8 CTAs x 8
def test_ln_rows(E, rows):
    fmt = (E + rows) % 2
    big = rows * E > 8_000_000
    x, part, _, extra, g, b, c = ln_inputs(rows, E, 0, fmt, rows + E, False, not big)
    x_out, xn, xd = run_ln(2, x, None, None, extra, g, b, fmt, in_place=False, with_xn=True, with_x_out=not big)
    want = R.split_sum_f32(xd, extra.to(DEV)) if extra is not None else xd
    if x_out is not None:
        assert torch.equal(bits(x_out), bits(want))
    check_ln(2, want, xn, g, b, fmt, c, "ln_rows rows %d E %d" % (rows, E))


@pytest.mark.parametrize("rows,form", [(511, 1), (512, 2)])
@pytest.mark.parametrize("fmt", [0, 1])
def test_ln_form_choice(rows, form, fmt):
    """form 0 (the batched passes' choice): ln_reduce_kernel below 512 rows, ln_rows_kernel from 512 -- bit for bit the forced form"""
    x, _, _, extra, g, b, c = ln_inputs(rows, 1536, 0, fmt, rows, False, True)
    o0, n0, _ = run_ln(0, x, None, None, extra, g, b, fmt, in_place=False, with_xn=True)
    o1, n1, _ = run_ln(form, x, None, None, extra, g, b, fmt, in_place=False, with_xn=True)
    assert torch.equal(bits(o0), bits(o1)) and torch.equal(bits(n0), bits(n1))
    check_ln(form, o0, n0, g, b, fmt, c, "form 0 rows %d" % rows)


@pytest.mark.parametrize("form", [1, 2])
@pytest.mark.parametrize("fmt", [0, 1])
def test_ln_rejects_mutations(form, fmt):
    """E = 128; row 3 has variance ~1e-8 (eps decides rstd) and no partials"""
    E, rows, S = 128, 8 if form == 1 else 512, 3 if form == 1 else 0
    x = R.ln_rows_input(rows, E, seed=7)
    part = torch.randn(S, rows, E, generator=torch.Generator().manual_seed(8))
    part[:, 3] = 0
    gen = torch.Generator().manual_seed(9)
    g, b = torch.rand(E, generator=gen) + 0.5, torch.randn(E, generator=gen)
    _, xn, _ = run_ln(form, x, part if S else None, None, None, g, b, fmt, in_place=True, with_xn=True)
    x_sum = R.split_sum_f32(x, *part).to(DEV)
    gd, bd = g.to(DEV), b.to(DEV)
    ref, slack = R.ln_rows_ref(x_sum, gd, bd, form)
    within(xn, ref, slack, fmt, "needles")
    for mutation in R.LN_MUTATIONS:
        if mutation == "omit_last_partial" and not S:
            continue
        xm = R.split_sum_f32(x, *part[:-1]).to(DEV) if mutation == "omit_last_partial" else None
        mut, mslack = R.ln_rows_ref(x_sum, gd, bd, form, mutation_x=xm, mutation=None if xm is not None else mutation)
        assert R.excess(xn, mut, R.tol16(mut, mslack, fmt)) > 0, mutation


# ---------------------------------------------------------------------------------------------------------------- act_reduce
def run_act(part, bias, B, N_, fmt):
    hfull, h = guarded(torch.full((B, N_), float("nan"), dtype=R.DT[fmt]))
    N.check(N.lib().rqb200_dbg_act_reduce(N.ptr(part), part.shape[0], N.ptr(bias), N.ptr(h), B, N_, fmt, N.stream_ptr()), "dbg_act_reduce")
    torch.cuda.synchronize()
    assert guard_intact(hfull, B * N_)
    return h


@pytest.mark.parametrize("S", [2, 3, 4, 5, 8, 13])        # past 4: the partials beyond the unrolled loads
@pytest.mark.parametrize("B", [1, 64, 256])
@pytest.mark.parametrize("N_", [512, 6144, 18432])        # B = 256 with N = 6144 and up: grid-strided (1184 CTAs)
@pytest.mark.parametrize("fmt", [0, 1])
def test_act_reduce(S, B, N_, fmt):
    gen = torch.Generator(DEV).manual_seed(S * 1000 + B + N_)
    part = torch.randn(S, B, N_, generator=gen, device=DEV) * (2.0 / S ** 0.5)
    bias = torch.randn(N_, generator=gen, device=DEV)
    h = run_act(part, bias, B, N_, fmt)
    v = R.split_sum_f32(bias, *part)
    ref = R.gelu64(v)
    within(h, ref, R.gelu_slack(v, ref), fmt, "S %d B %d N %d" % (S, B, N_))


@pytest.mark.parametrize("fmt", [0, 1])
def test_act_reduce_rejects_mutations(fmt):
    S, B, N_ = 5, 2, 512
    part = torch.randn(S, B, N_, generator=torch.Generator(DEV).manual_seed(1), device=DEV)
    bias = torch.linspace(-4, 4, N_, device=DEV)
    h = run_act(part, bias, B, N_, fmt)
    v = R.split_sum_f32(bias, *part)
    ref = R.gelu64(v)
    within(h, ref, R.gelu_slack(v, ref), fmt, "needles")
    tanh = R.gelu64(v, "tanh_gelu")
    assert R.excess(h, tanh, R.tol16(tanh, R.gelu_slack(v, tanh), fmt)) > 0
    vm = R.split_sum_f32(bias, *part[:-1])
    om = R.gelu64(vm)
    assert R.excess(h, om, R.tol16(om, R.gelu_slack(vm, om), fmt)) > 0
