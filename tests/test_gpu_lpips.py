"""The native LPIPS on the GPU: against the reference's fixture (tests/golden/lpips.pt) on both tiers, the exact identities (x against
itself, symmetry, batch independence, chunking), against the float64 torch restatement (tests/lpips_oracle.py) at shapes the fixture
does not hold, every VGG conv geometry on both conv kernels, and the new kernels against float64 at their edges."""
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import synth
from rqvae import _native as N
from rqvae.losses.vqgan import LPIPS
from rqvae.losses.vqgan import lpips as LP
from rqvae.metrics import inception as INC
from tests import lpips_oracle as LO

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# rel-L2 of the per-tap averages and of the values against float64, per tier.  On an H100 the fixture's cases and the restatement's
# shapes measured at most 8.0e-8 on the exact tier (fp32 FFMA through 13 convs) and 4.0e-7 on the fast tier (split-fp16 operands,
# which drop the lo x lo product)
EXACT_BOUND = 1e-6
FAST_BOUND = 5e-6
# the near-identical pair (target = input + 0.01 noise): its value is a difference of nearly equal normalised features, so the fp32
# head's rounding weighs about |f| / |f0 - f1| times more; measured 4.2e-6 (exact) and 4.1e-6 (fast)
EXACT_NOISY_BOUND = 4e-5
FAST_NOISY_BOUND = 4e-5


def rel(a, b):
    return float((a.double().cpu() - b.double().cpu()).norm() / b.double().cpu().norm())


@pytest.fixture(scope="module")
def fixture(golden):
    return golden("lpips")


@pytest.fixture(scope="module")
def weights(fixture):
    return LO.synth_weights(fixture["seed"])


def build(home, precision):
    old = os.environ.get("TORCH_HOME")
    os.environ["TORCH_HOME"] = home
    try:
        m = LPIPS().to(DEV).eval()
    finally:
        if old is None:
            del os.environ["TORCH_HOME"]
        else:
            os.environ["TORCH_HOME"] = old
    m.precision = precision
    return m


@pytest.fixture(scope="module")
def torch_home(tmp_path_factory, weights):
    home = str(tmp_path_factory.mktemp("torch_home"))
    LO.write_weight_files(home, weights)
    return home


@pytest.fixture(scope="module")
def exact(torch_home):
    return build(torch_home, "exact")


@pytest.fixture(scope="module")
def fast(torch_home):
    return build(torch_home, "fast")


@pytest.fixture(scope="module")
def sd64(weights):
    return {k: v.double().to(DEV) for k, v in weights.items()}


def bounds(tier, kind):
    if kind == "noisy":
        return EXACT_NOISY_BOUND if tier == "exact" else FAST_NOISY_BOUND
    return EXACT_BOUND if tier == "exact" else FAST_BOUND


@pytest.mark.parametrize("tier", ["exact", "fast"])
@pytest.mark.parametrize("idx", range(7))
def test_matches_reference_fixture(exact, fast, fixture, tier, idx):
    m = exact if tier == "exact" else fast
    case = fixture["cases"][idx]
    x0, x1 = LO.case_inputs(case)
    with torch.no_grad():
        layers, val = m._run(x0.to(DEV), x1.to(DEV))
        none = m(x0.to(DEV), x1.to(DEV), reduction="none")
    assert none.shape == (case["B"], 1, 1, 1) and torch.equal(none.reshape(-1), val)
    if case["kind"] == "identical":
        assert torch.equal(val, torch.zeros_like(val)) and torch.equal(layers, torch.zeros_like(layers))
        return
    b = bounds(tier, case["kind"])
    e_layers, e_val = rel(layers, case["layers"]), rel(val, case["val"])
    print("LPIPS %s %s: per-tap rel-L2 %.3g, value rel-L2 %.3g" % (tier, case["name"], e_layers, e_val))
    assert e_layers <= b and e_val <= b, (e_layers, e_val, b)


@pytest.mark.parametrize("tier", ["exact", "fast"])
def test_reductions(exact, fast, tier):
    m = exact if tier == "exact" else fast
    x0 = synth.randn_seeded((3, 3, 32, 48), 1).tanh().to(DEV)
    x1 = synth.randn_seeded((3, 3, 32, 48), 2).tanh().to(DEV)
    with torch.no_grad():
        v = m(x0, x1, reduction="none")
        assert torch.equal(m(x0, x1), torch.mean(v)) and m(x0, x1).dim() == 0
        assert torch.equal(m(x0, x1, reduction="sum"), torch.sum(v))


# ------------------------------------------------------------------------------------------------ exact identities
@pytest.mark.parametrize("tier", ["exact", "fast"])
def test_identities_are_exact(exact, fast, tier):
    m = exact if tier == "exact" else fast
    x = synth.randn_seeded((4, 3, 72, 56), 3).tanh().to(DEV)
    y = synth.randn_seeded((4, 3, 72, 56), 4).tanh().to(DEV)
    with torch.no_grad():
        assert torch.equal(m(x, x, reduction="none"), torch.zeros(4, 1, 1, 1, device=DEV))
        lxy, vxy = m._run(x, y)
        lyx, vyx = m._run(y, x)
        assert torch.equal(vxy, vyx) and torch.equal(lxy, lyx)
        for i in (0, 3):
            li, vi = m._run(x[i:i + 1], y[i:i + 1])
            assert torch.equal(vi[0], vxy[i]) and torch.equal(li[0], lxy[i])


@pytest.mark.parametrize("tier", ["exact", "fast"])
def test_chunked_batch_gives_the_bits_of_its_pieces(exact, fast, tier, sd64):
    """40 pairs of 256^2 pass the 2 GiB chunk (31 pairs per chunk on the exact tier, 21 on the fast)"""
    m = exact if tier == "exact" else fast
    x = synth.randn_seeded((40, 3, 256, 256), 5).tanh().to(DEV)
    y = (x + 0.1 * synth.randn_seeded((40, 3, 256, 256), 6).to(DEV)).clamp(-1, 1)
    with torch.no_grad():
        layers, val = m._run(x, y)
        for a, b in ((0, 13), (13, 31), (31, 40), (20, 22)):
            lp, vp = m._run(x[a:b], y[a:b])
            assert torch.equal(vp, val[a:b]) and torch.equal(lp, layers[a:b]), (a, b)
        pick = [0, 20, 21, 30, 31, 39]
        rl, rv = LO.lpips(sd64, x[pick].double(), y[pick].double())
    b = bounds(tier, "random")
    assert rel(layers[pick], rl) <= b and rel(val[pick], rv) <= b


# ------------------------------------------------------------------------------------------------ against the restatement
@pytest.mark.parametrize("tier", ["exact", "fast"])
@pytest.mark.parametrize("B,H,W", [(3, 97, 131), (1, 1024, 1024), (2, 17, 33)])
def test_matches_restatement(exact, fast, sd64, tier, B, H, W):
    m = exact if tier == "exact" else fast
    x = synth.randn_seeded((B, 3, H, W), 7).tanh().to(DEV)
    y = synth.randn_seeded((B, 3, H, W), 8).tanh().to(DEV)
    with torch.no_grad():
        layers, val = m._run(x, y)
        rl, rv = LO.lpips(sd64, x.double(), y.double())
    b = bounds(tier, "random")
    e = (rel(layers, rl), rel(val, rv))
    print("LPIPS %s %dx%dx%d against the restatement: per-tap %.3g, value %.3g" % (tier, B, H, W, *e))
    assert e[0] <= b and e[1] <= b, e


def test_engine_rebuilds_after_load_state_dict(exact, weights):
    x = synth.randn_seeded((2, 3, 32, 32), 9).tanh().to(DEV)
    y = synth.randn_seeded((2, 3, 32, 32), 10).tanh().to(DEV)
    with torch.no_grad():
        before = exact(x, y, reduction="none").clone()
        sd = {k: v.clone() for k, v in exact.state_dict().items()}
        sd["lin0.model.1.weight"] = sd["lin0.model.1.weight"] * 2
        exact.load_state_dict(sd)
        after = exact(x, y, reduction="none")
        l0 = exact._run(x, y)[0][:, 0]
        exact.load_state_dict({k: v.to(DEV) for k, v in weights.items()}, strict=False)
        again = exact(x, y, reduction="none")
    assert not torch.equal(before, after)
    assert torch.allclose(after.reshape(-1), before.reshape(-1) + l0 / 2, rtol=1e-5)
    assert torch.equal(again, before)


# ------------------------------------------------------------------------------------------------ every VGG conv geometry
def conv_geometries():
    """(name, Cin, Cout, H, W) of every conv at a 16^2 input (down to the 2x2 and 1x1 maps of slice 4 and 5) and at 100 x 70"""
    out = []
    for H0, W0 in ((16, 16), (100, 70)):
        H, W, s = H0, W0, 0
        for name, ci, co, tap in LO.CONVS:
            out.append((name, ci, co, H, W))
            if tap:
                H, W = H // 2, W // 2
    return out


@pytest.mark.parametrize("g", conv_geometries(), ids=lambda g: "%s_%dto%d_%dx%d" % g)
def test_conv_every_geometry(g):
    name, ci, co, H, W = g
    B = 2
    x = synth.randn_seeded((B, ci, H, W), 11).abs().to(DEV)
    w = synth.randn_seeded((co, ci, 3, 3), 12, (2.0 / (9 * ci)) ** 0.5).to(DEV)
    b = synth.randn_seeded((co,), 13, 0.01).to(DEV)
    ref = F.relu(F.conv2d(x.double(), w.double(), b.double(), padding=1)).permute(0, 2, 3, 1)
    xn, wn = x.permute(0, 2, 3, 1).contiguous(), w.permute(0, 2, 3, 1).contiguous()
    out = torch.zeros(B, H, W, co, device=DEV)
    N.check(INC._lib().rqb200_dbg_inception_conv(N.ptr(xn), N.ptr(wn), N.ptr(b), N.ptr(out), B, H, W, ci, co, 3, 3, 1, 1, 1, co, 0,
                                                 N.stream_ptr()), "dbg_inception_conv")
    assert float((out.double() - ref).abs().max()) <= 1e-5 * float(ref.abs().max()) + 1e-6
    if ci == 3:
        return                                        # conv1_1 runs the fp32 FFMA kernel on both tiers
    xh, xl = xn.half(), (xn - xn.half().float()).half()
    wh, wl = wn.half(), (wn - wn.half().float()).half()
    out = torch.zeros(B, H, W, co, device=DEV)
    oh = torch.full((B, H, W, co), 7.0, device=DEV, dtype=torch.half)
    ol = torch.full((B, H, W, co), 7.0, device=DEV, dtype=torch.half)
    N.check(INC._lib().rqb200_dbg_inception_conv_tc(N.ptr(xh), N.ptr(xl), N.ptr(wh), N.ptr(wl), N.ptr(b), N.ptr(out), N.ptr(oh), N.ptr(ol),
                                                    B, H, W, ci, co, 3, 3, 1, 1, 1, co, 0, N.stream_ptr()), "dbg_inception_conv_tc")
    ref16 = F.relu(F.conv2d((xh.double() + xl.double()).permute(0, 3, 1, 2), (wh.double() + wl.double()).permute(0, 3, 1, 2), b.double(),
                            padding=1)).permute(0, 2, 3, 1)
    assert float((out.double() - ref16).abs().max()) <= 2e-5 * float(ref16.abs().max()) + 1e-6
    assert torch.equal(oh, out.half()) and torch.equal(ol, (out - out.half().float()).half())


# ------------------------------------------------------------------------------------------------ the new kernels
@pytest.mark.parametrize("n,H,W", [(1, 16, 16), (3, 37, 20), (2, 1, 5)])
def test_input_kernel(n, H, W):
    x0 = synth.randn_seeded((n, 3, H, W), 14).to(DEV)
    x1 = synth.randn_seeded((n, 3, H, W), 15).to(DEV)
    shift = torch.tensor(LO.SHIFT, device=DEV)
    scale = torch.tensor(LO.SCALE, device=DEV)
    y = torch.empty(2 * n, H, W, 3, device=DEV)
    N.check(LP._lib().rqb200_dbg_lpips_input(N.ptr(x0), N.ptr(x1), N.ptr(shift), N.ptr(scale), N.ptr(y), n, H, W, N.stream_ptr()),
            "dbg_lpips_input")
    ref = (torch.cat([x0, x1]) - shift.reshape(1, 3, 1, 1)) / scale.reshape(1, 3, 1, 1)    # torch's fp32 ScalingLayer
    assert torch.equal(y, ref.permute(0, 2, 3, 1))


@pytest.mark.parametrize("N_,H,W,C", [(2, 16, 16, 64), (3, 7, 5, 128), (1, 2, 2, 512), (2, 3, 3, 256), (1, 101, 70, 64)])
def test_pool_kernel(N_, H, W, C):
    x = synth.randn_seeded((N_, H, W, C), 16).relu().to(DEV)
    Ho, Wo = H // 2, W // 2
    y = torch.full((N_, Ho, Wo, C), 7.0, device=DEV)
    yh = torch.full((N_, Ho, Wo, C), 7.0, device=DEV, dtype=torch.half)
    yl = torch.full((N_, Ho, Wo, C), 7.0, device=DEV, dtype=torch.half)
    N.check(LP._lib().rqb200_dbg_lpips_pool(N.ptr(x), N.ptr(y), N.ptr(yh), N.ptr(yl), N_, H, W, C, N.stream_ptr()), "dbg_lpips_pool")
    ref = F.max_pool2d(x.permute(0, 3, 1, 2).double(), 2, 2).permute(0, 2, 3, 1)
    assert torch.equal(y.double(), ref)
    assert torch.equal(yh, y.half()) and torch.equal(yl, (y - y.half().float()).half())
    y2 = torch.full_like(y, 7.0)
    N.check(LP._lib().rqb200_dbg_lpips_pool(N.ptr(x), N.ptr(y2), None, None, N_, H, W, C, N.stream_ptr()), "dbg_lpips_pool")
    assert torch.equal(y2, y)


def head_ref(Fm, w, n):
    a, t = Fm[:n].double(), Fm[n:].double()
    na = a.pow(2).sum(-1, keepdim=True).sqrt() + 1e-10
    nt = t.pow(2).sum(-1, keepdim=True).sqrt() + 1e-10
    return ((a / na - t / nt) ** 2 * w.double()).sum(-1)


def dbg_head(Fm, w, n, hw, C):
    d = torch.full((n, hw), 7.0, device=DEV)
    N.check(LP._lib().rqb200_dbg_lpips_head(N.ptr(Fm), N.ptr(w), N.ptr(d), n, hw, C, N.stream_ptr()), "dbg_lpips_head")
    return d


@pytest.mark.parametrize("C", [64, 128, 256, 512])
@pytest.mark.parametrize("near", [False, True])
def test_head_kernel(C, near):
    n, hw = 3, 37
    a = synth.randn_seeded((n, hw, C), 17).relu()
    t = a + 1e-3 * synth.randn_seeded((n, hw, C), 18) if near else synth.randn_seeded((n, hw, C), 18).relu()
    t = t.relu()
    a[1, 5] = 0.0                                       # all-zero feature pixels normalise to 0
    t[2, 7] = 0.0
    a[0, 3] = 0.0
    t[0, 3] = 0.0
    Fm = torch.cat([a, t]).to(DEV)
    w = synth.randn_seeded((C,), 19, 0.1).abs().to(DEV)
    d = dbg_head(Fm, w, n, hw, C)
    ref = head_ref(Fm, w, n)
    assert float(d[0, 3]) == 0.0
    err = float(((d.double() - ref).abs() / ref.abs().clamp_min(1e-30)).max())
    assert err <= (1e-3 if near else 1e-5), err
    swapped = dbg_head(torch.cat([t, a]).to(DEV), w, n, hw, C)
    assert torch.equal(swapped, d)


def test_mean_kernel():
    n, hw = 3, 1000
    d = synth.randn_seeded((n, hw), 20).abs().to(DEV)
    tm = torch.zeros(n, 5, dtype=torch.float64, device=DEV)
    lo = torch.zeros(n, 5, device=DEV)
    val = torch.full((n,), 7.0, device=DEV)
    for k in range(5):
        dk = d * (k + 1)
        N.check(LP._lib().rqb200_dbg_lpips_mean(N.ptr(dk), n, hw, k, N.ptr(tm), N.ptr(lo), N.ptr(val), N.stream_ptr()), "dbg_lpips_mean")
        ref = dk.double().mean(1)
        assert float((tm[:, k] - ref).abs().max()) <= 1e-15 * float(ref.abs().max())
        assert torch.equal(lo[:, k], tm[:, k].float())
    acc = tm[:, 0].clone()
    for k in range(1, 5):
        acc = acc + tm[:, k]                        # the kernel's order: tap 0 + tap 1 + ... + tap 4
    assert torch.equal(val, acc.float())
    one = torch.full((1, 1), 0.25, device=DEV)
    N.check(LP._lib().rqb200_dbg_lpips_mean(N.ptr(one), 1, 1, 0, N.ptr(tm), None, None, N.stream_ptr()), "dbg_lpips_mean")
    assert float(tm[0, 0]) == 0.25
