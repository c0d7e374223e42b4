"""The native FID Inception-v3 on the GPU: against the reference's fixture (tests/golden/fid.pt) per image, against the torch
restatement (tests/inception_oracle.py, float64 on the GPU) at batches and sizes the fixture does not hold, batch independence,
each kernel against float64, and the FID functions end to end."""
import os
import pickle

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import synth
from rqvae import _native as N
from rqvae.metrics import fid as FID
from rqvae.metrics import inception as INC
from tests import inception_oracle as IO

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# whole-network bound of the exact tier against float64: fp32 FFMA through 94 convs whose folded BatchNorms rescale each channel
# (up to 3.8e-5 rel-L2 on the fixture's images on an H100)
NET_BOUND = 1e-4
# the fast tier's whole-network bound: split-fp16 operands drop the lo x lo product and carry small activations' lo halves as fp16
# subnormals; through 93 wgmma convs that measured 7.4e-5 to 4.4e-4 rel-L2 on the fixture's images on an H100
FAST_BOUND = 1e-3


def rel(a, b):
    return float((a.double().cpu() - b.double().cpu()).norm() / b.double().cpu().norm())


@pytest.fixture(scope="module")
def fixture(golden):
    return golden("fid")


@pytest.fixture(scope="module")
def weights(fixture):
    return IO.fixture_state_dict(fixture)


@pytest.fixture(scope="module")
def torch_home(tmp_path_factory, weights):
    home = str(tmp_path_factory.mktemp("torch_home"))
    IO.write_weight_file(home, weights)
    return home


@pytest.fixture(scope="module")
def model(torch_home):
    old = os.environ.get("TORCH_HOME")
    os.environ["TORCH_HOME"] = torch_home
    try:
        m = INC.InceptionV3([0, 1, 2, 3]).to(DEV)
    finally:
        if old is None:
            del os.environ["TORCH_HOME"]
        else:
            os.environ["TORCH_HOME"] = old
    m.precision = "exact"
    return m


@pytest.fixture(scope="module")
def fast_model(torch_home):
    old = os.environ.get("TORCH_HOME")
    os.environ["TORCH_HOME"] = torch_home
    try:
        m = INC.InceptionV3([0, 1, 2, 3]).to(DEV)
    finally:
        if old is None:
            del os.environ["TORCH_HOME"]
        else:
            os.environ["TORCH_HOME"] = old
    m.precision = "fast"
    return m


@pytest.fixture(scope="module")
def restated(weights):
    return IO.Restated({k: v.double().to(DEV) for k, v in weights.items()})


def run(model, x, resize=True):
    model.resize_input = resize
    outs, lg = model(x.to(DEV), return_logits=True)
    return outs, lg


@pytest.mark.parametrize("idx", range(7))
def test_exact_tier_matches_reference_fixture(model, fixture, idx):
    case = fixture["cases"][idx]
    outs, lg = run(model, IO.fixture_input(case), case["resize"])
    for b in range(case["B"]):          # per image
        assert rel(outs[3][b].reshape(-1), case["features"][b]) <= NET_BOUND
        assert rel(lg[b], case["logits"][b]) <= NET_BOUND
        for k in range(3):
            assert list(outs[k].shape) == case["block_shapes"][k]
            assert rel(outs[k][b].mean((1, 2)), case["means"][k][b]) <= NET_BOUND


@pytest.mark.parametrize("idx", range(7))
def test_fast_tier_matches_reference_fixture(fast_model, fixture, idx):
    case = fixture["cases"][idx]
    outs, lg = run(fast_model, IO.fixture_input(case), case["resize"])
    for b in range(case["B"]):
        assert rel(outs[3][b].reshape(-1), case["features"][b]) <= FAST_BOUND
        assert rel(lg[b], case["logits"][b]) <= FAST_BOUND
        for k in range(3):
            assert list(outs[k].shape) == case["block_shapes"][k]
            assert rel(outs[k][b].mean((1, 2)), case["means"][k][b]) <= FAST_BOUND


@pytest.mark.parametrize("B, H, W, resize", [(1, 299, 299, True), (2, 97, 131, False), (3, 33, 517, True), (300, 256, 256, True)])
def test_fast_tier_matches_restatement_and_batch_independence(fast_model, restated, B, H, W, resize):
    x = synth.randn_seeded((B, 3, H, W), 11 + H).sigmoid()
    outs, lg = run(fast_model, x, resize)
    pick = list(range(B)) if B <= 3 else [0, 150, 299]
    with torch.no_grad():
        ro, rl = restated.forward(x[pick].double().to(DEV), resize_input=resize)
    for k in range(4):
        assert rel(outs[k][pick], ro[k]) <= FAST_BOUND, k
    assert rel(lg[pick], rl) <= FAST_BOUND
    o1, _ = run(fast_model, x[pick[-1]:pick[-1] + 1], resize)
    assert torch.equal(o1[3][0], outs[3][pick[-1]])


@pytest.mark.parametrize("B, H, W, resize", [(1, 299, 299, True), (2, 97, 131, False), (3, 33, 517, True)])
def test_exact_tier_matches_restatement(model, restated, B, H, W, resize):
    x = synth.randn_seeded((B, 3, H, W), 7 + H).sigmoid()
    outs, lg = run(model, x, resize)
    with torch.no_grad():
        ro, rl = restated.forward(x.double().to(DEV), resize_input=resize)
    for k in range(4):
        assert outs[k].shape == ro[k].shape
        assert rel(outs[k], ro[k]) <= NET_BOUND, k
    assert rel(lg, rl) <= NET_BOUND


def test_chunked_batch_of_300(model, restated):
    x = synth.randn_seeded((300, 3, 256, 256), 301).sigmoid()
    model.resize_input = True
    feats = model(x.to(DEV))[3].reshape(300, -1)
    pick = [0, 91, 92, 183, 184, 275, 276, 299]       # across the chunk boundaries (92 images of 299^2 per 2 GiB chunk)
    with torch.no_grad():
        ro, _ = restated.forward(x[pick].double().to(DEV))
    assert rel(feats[pick], ro[3].reshape(len(pick), -1)) <= NET_BOUND
    alone = model(x[299:300].to(DEV))[3].reshape(1, -1)
    assert torch.equal(alone, feats[299:300])


def test_batch_independence_bitwise(model):
    x = synth.randn_seeded((5, 3, 160, 200), 17).sigmoid().to(DEV)
    outs, lg = run(model, x)
    for i in (0, 3):
        o1, l1 = run(model, x[i:i + 1])
        for k in range(4):
            assert torch.equal(o1[k][0], outs[k][i]), k
        assert torch.equal(l1[0], lg[i])


# ------------------------------------------------------------------------------------------------ kernels against float64
STRIDE2 = {"blocks.0.0", "blocks.2.3.branch3x3", "blocks.2.3.branch3x3dbl_3", "blocks.3.0.branch3x3_2", "blocks.3.0.branch7x7x3_4"}
VALID = STRIDE2 | {"blocks.0.1", "blocks.1.1"}                   # no padding
EXTENT = {"blocks.0.0": 299, "blocks.0.1": 149, "blocks.0.2": 147, "blocks.1.0": 73, "blocks.1.1": 73}


def plan_convs():
    """every conv of the plan with its real input extent at 299 x 299: (name, Cout, Cin, kh, kw, pad_h, pad_w, stride, H, W)"""
    out = []
    for n, co, ci, kh, kw in IO.conv_list():
        p = ".".join(n.split(".")[:3])
        H = EXTENT.get(n) or (35 if p <= "blocks.2.3" else 17 if p <= "blocks.3.0" else 8)
        ph, pw = (0, 0) if n in VALID else (kh // 2, kw // 2)
        out.append((n, co, ci, kh, kw, ph, pw, 2 if n in STRIDE2 else 1, H, H))
    return out


def geometries():
    seen, out = set(), []
    for c in plan_convs():
        if c[1:] not in seen:
            seen.add(c[1:])
            out.append(c)
    return out


def dbg_conv(X, Wt, b, B, H, W, Cin, Cout, kh, kw, ph, pw, s, out=None, ldy=None, yoff=0):
    L = INC._lib()
    Ho, Wo = (H + 2 * ph - kh) // s + 1, (W + 2 * pw - kw) // s + 1
    ldy = ldy or Cout
    if out is None:
        out = torch.zeros(B, Ho, Wo, ldy, device=DEV)
    N.check(L.rqb200_dbg_inception_conv(N.ptr(X), N.ptr(Wt), N.ptr(b), N.ptr(out), B, H, W, Cin, Cout, kh, kw, ph, pw, s, ldy, yoff,
                                        N.stream_ptr()), "dbg_inception_conv")
    return out


@pytest.mark.parametrize("g", geometries(), ids=lambda g: "%s_%dx%d_s%d_%dto%d_%d" % (g[0], g[3], g[4], g[7], g[2], g[1], g[8]))
def test_conv_every_plan_geometry(g):
    name, co, ci, kh, kw, ph, pw, s, H, W = g
    B = 2 if H <= 73 else 1
    x = synth.randn_seeded((B, ci, H, W), 5).to(DEV)
    w = synth.randn_seeded((co, ci, kh, kw), 6, (ci * kh * kw) ** -0.5).to(DEV)
    b = synth.randn_seeded((co,), 7, 0.1).to(DEV)
    got = dbg_conv(x.permute(0, 2, 3, 1).contiguous(), w.permute(0, 2, 3, 1).contiguous(), b, B, H, W, ci, co, kh, kw, ph, pw, s)
    ref = F.relu(F.conv2d(x.double(), w.double(), b.double(), stride=s, padding=(ph, pw))).permute(0, 2, 3, 1)
    assert got.shape == ref.shape
    err = float((got.double() - ref).abs().max())
    bound = 1e-5 * float(ref.abs().max()) + 1e-5
    assert err <= bound, (err, bound)


def split16(t):
    hi = t.half()
    return hi.contiguous(), (t - hi.float()).half().contiguous()


def dbg_conv_tc(x, w, b, B, H, W, ci, co, kh, kw, ph, pw, s, ldy=None, yoff=0, out=None, out16=True):
    """x NHWC f32, w OHWI f32 -> (out f32, hi, lo) [B, Ho, Wo, ldy] through the fast tier's conv"""
    Ho, Wo = (H + 2 * ph - kh) // s + 1, (W + 2 * pw - kw) // s + 1
    ldy = ldy or co
    xh, xl = split16(x)
    wh, wl = split16(w)
    if out is None:
        out = torch.zeros(B, Ho, Wo, ldy, device=DEV)
    oh = torch.full((B, Ho, Wo, ldy), 7.0, device=DEV, dtype=torch.half) if out16 else None
    ol = torch.full((B, Ho, Wo, ldy), 7.0, device=DEV, dtype=torch.half) if out16 else None
    N.check(INC._lib().rqb200_dbg_inception_conv_tc(N.ptr(xh), N.ptr(xl), N.ptr(wh), N.ptr(wl), N.ptr(b), N.ptr(out), N.ptr(oh), N.ptr(ol),
                                                    B, H, W, ci, co, kh, kw, ph, pw, s, ldy, yoff, N.stream_ptr()), "dbg_inception_conv_tc")
    return out, oh, ol


@pytest.mark.parametrize("g", geometries(), ids=lambda g: "%s_%dx%d_s%d_%dto%d_%d" % (g[0], g[3], g[4], g[7], g[2], g[1], g[8]))
def test_fast_conv_every_plan_geometry(g):
    """the split-fp16 wgmma conv of every conv geometry of the plan but the Cin = 3 stem conv (fp32 FFMA on both tiers), at its real
    extent, against float64 on the operands it is given (their hi + lo)"""
    name, co, ci, kh, kw, ph, pw, s, H, W = g
    if ci == 3:
        pytest.skip("Conv2d_1a_3x3 runs the fp32 FFMA kernel on both tiers")
    B = 2 if H <= 73 else 1
    x = synth.randn_seeded((B, H, W, ci), 15).to(DEV)
    w = synth.randn_seeded((co, kh, kw, ci), 16, (ci * kh * kw) ** -0.5).to(DEV)
    b = synth.randn_seeded((co,), 17, 0.1).to(DEV)
    got, oh, ol = dbg_conv_tc(x, w, b, B, H, W, ci, co, kh, kw, ph, pw, s)
    ref = F.relu(F.conv2d(x.permute(0, 3, 1, 2).double(), w.permute(0, 3, 1, 2).double(), b.double(), stride=s,
                          padding=(ph, pw))).permute(0, 2, 3, 1)
    assert got.shape == ref.shape
    err = float((got.double() - ref).abs().max())
    bound = 2e-5 * float(ref.abs().max()) + 1e-5
    assert err <= bound, (err, bound)
    # the epilogue's fp16 operand halves are the split of the fp32 output
    eh, el = split16(got)
    assert torch.equal(oh, eh) and torch.equal(ol, el)


def test_fast_conv_channel_offset_store_leaves_neighbours():
    B, H, W, ci, co, ld, off = 2, 17, 17, 160, 192, 768, 384
    x = synth.randn_seeded((B, H, W, ci), 18).to(DEV)
    w = synth.randn_seeded((co, 1, 7, ci), 19, (7 * ci) ** -0.5).to(DEV)
    b = synth.randn_seeded((co,), 20, 0.1).to(DEV)
    out = torch.full((B, H, W, ld), 123.5, device=DEV)
    got, oh, ol = dbg_conv_tc(x, w, b, B, H, W, ci, co, 1, 7, 0, 3, 1, ldy=ld, yoff=off, out=out)
    for t, fill in ((out, 123.5), (oh, 7.0), (ol, 7.0)):
        assert bool((t[..., :off] == fill).all()) and bool((t[..., off + co:] == fill).all())
    ref = F.relu(F.conv2d(x.permute(0, 3, 1, 2).double(), w.permute(0, 3, 1, 2).double(), b.double(), padding=(0, 3)))
    assert rel(out[..., off:off + co], ref.permute(0, 2, 3, 1)) <= 2e-5


def test_conv_channel_offset_store_leaves_neighbours():
    B, H, W, ci, co, ld, off = 2, 17, 17, 96, 192, 768, 384
    x = synth.randn_seeded((B, H, W, ci), 8).to(DEV)
    w = synth.randn_seeded((co, 7, 1, ci), 9, (7 * ci) ** -0.5).to(DEV)
    b = synth.randn_seeded((co,), 10, 0.1).to(DEV)
    out = torch.full((B, H, W, ld), 123.5, device=DEV)
    dbg_conv(x, w, b, B, H, W, ci, co, 7, 1, 3, 0, 1, out=out, ldy=ld, yoff=off)
    assert bool((out[..., :off] == 123.5).all()) and bool((out[..., off + co:] == 123.5).all())
    ref = F.relu(F.conv2d(x.permute(0, 3, 1, 2).double(), w.permute(0, 3, 1, 2).double(), b.double(), padding=(3, 0)))
    assert rel(out[..., off:off + co], ref.permute(0, 2, 3, 1)) <= 1e-6


@pytest.mark.parametrize("mode, stride, pad, H, W, C, ldy, yoff", [
    (0, 2, 0, 147, 147, 64, 64, 0), (0, 2, 0, 35, 35, 288, 768, 480), (0, 2, 0, 17, 16, 768, 1280, 512), (0, 1, 1, 8, 8, 2048, 2048, 0),
    (1, 1, 1, 35, 35, 192, 192, 0), (1, 1, 1, 17, 17, 768, 768, 0), (1, 1, 1, 3, 5, 1280, 1280, 0), (0, 1, 1, 1, 1, 8, 8, 0)])
def test_pools(mode, stride, pad, H, W, C, ldy, yoff):
    B = 2
    x = synth.randn_seeded((B, C, H, W), 11).to(DEV)
    Ho, Wo = (H + 2 * pad - 3) // stride + 1, (W + 2 * pad - 3) // stride + 1
    out = torch.full((B, Ho, Wo, ldy), -7.25, device=DEV)
    N.check(INC._lib().rqb200_dbg_inception_pool(mode, N.ptr(x.permute(0, 2, 3, 1).contiguous()), N.ptr(out), B, H, W, C, stride, pad,
                                                 ldy, yoff, N.stream_ptr()), "dbg_inception_pool")
    xd = x.double()
    ref = F.max_pool2d(xd, 3, stride, pad) if mode == 0 else F.avg_pool2d(xd, 3, stride, pad, count_include_pad=False)
    got = out[..., yoff:yoff + C].permute(0, 3, 1, 2)
    assert float((got.double() - ref).abs().max()) <= 1e-6
    if ldy > C:
        assert bool((out[..., :yoff] == -7.25).all()) and bool((out[..., yoff + C:] == -7.25).all())


@pytest.mark.parametrize("H, W, resize, normalize", [(256, 256, 1, 1), (64, 64, 1, 1), (192, 128, 1, 0), (1, 1, 1, 1), (299, 299, 1, 1),
                                                     (512, 300, 1, 1), (80, 96, 0, 1), (75, 75, 0, 0)])
def test_input_stage(H, W, resize, normalize):
    B = 2
    x = torch.rand((B, 3, H, W), generator=torch.Generator().manual_seed(H * 7 + W)).to(DEV)
    Ho, Wo = (299, 299) if resize else (H, W)
    y = torch.empty(B, Ho, Wo, 3, device=DEV)
    N.check(INC._lib().rqb200_dbg_inception_input(N.ptr(x), N.ptr(y), B, H, W, resize, normalize, N.stream_ptr()), "dbg_inception_input")
    ref = x.double()
    if resize:
        ref = F.interpolate(ref, size=(299, 299), mode="bilinear", align_corners=False)
    if normalize:
        ref = 2 * ref - 1
    assert float((y.permute(0, 3, 1, 2).double() - ref).abs().max()) <= 2e-6


@pytest.mark.parametrize("B, HW, C", [(3, 64, 2048), (1, 1, 2048), (2, 196, 2048), (2, 5, 100)])
def test_global_average_pool(B, HW, C):
    x = synth.randn_seeded((B, HW, C), 12).to(DEV)
    y = torch.empty(B, C, device=DEV)
    N.check(INC._lib().rqb200_dbg_inception_gap(N.ptr(x), N.ptr(y), B, HW, C, N.stream_ptr()), "dbg_inception_gap")
    assert float((y.double() - x.double().mean(1)).abs().max()) <= 1e-6


# ------------------------------------------------------------------------------------------------ FID end to end
@pytest.fixture
def hub(torch_home, monkeypatch):
    monkeypatch.setenv("TORCH_HOME", torch_home)


def write_samples(path, n_files, per_file, seed):
    """samples*.pkl as main_sampling_fid.py writes them: uint8-free float arrays [n, 3, H, W] in [0, 1]"""
    xs = []
    for i in range(n_files):
        x = synth.randn_seeded((per_file, 3, 64, 64), seed + i).sigmoid()
        xs.append(x)
        with open(os.path.join(path, "samples_%d.pkl" % i), "wb") as f:
            pickle.dump(x.numpy(), f)
    return torch.cat(xs)


def test_statistics_from_files_and_compute_fid(hub, tmp_path, restated):
    fake = tmp_path / "fake"
    fake.mkdir()
    xs = write_samples(str(fake), 3, 4, 40)
    mu, sigma, acts = FID.compute_statistics_from_files(str(fake), batch_size=5, device=torch.device(DEV), return_acts=True)
    # glob order is the file order the statistics saw
    import glob
    order = [int(os.path.basename(p)[8:-4]) for p in glob.glob(os.path.join(str(fake), "samples*.pkl"))]
    xs_in = torch.cat([xs[4 * i:4 * i + 4] for i in order])
    with torch.no_grad():
        ro, _ = restated.forward(xs_in.double().to(DEV))
    ref = ro[3].reshape(12, -1).cpu()
    assert rel(acts, ref) <= NET_BOUND
    rmu, rsigma = FID.mean_covar_numpy(ref.numpy())
    assert np.abs(mu - rmu).max() <= 1e-4 * np.abs(rmu).max()
    assert np.abs(sigma - rsigma).max() <= 1e-4 * np.abs(rsigma).max()
    ref_stats = tmp_path / "ref.npz"
    g = np.random.default_rng(3)
    np.savez(ref_stats, mu=rmu + 0.01 * g.normal(size=rmu.shape), sigma=rsigma * 1.1)
    value = FID.compute_fid(str(fake), str(ref_stats), batch_size=5, device=torch.device(DEV))
    saved = np.load(fake / "acts.npz")
    assert set(saved.files) == {"acts", "mu", "sigma"}
    st = np.load(ref_stats)
    assert value == FID.frechet_distance(st["mu"], st["sigma"], saved["mu"], saved["sigma"])


def test_compute_rfid_with_a_zoo_rqvae(hub, restated):
    from tests.test_gpu_vae_sizes import build
    from oracle.zoo import VAE_ZOO
    vae, _ = build("tiny", VAE_ZOO["tiny"], 71)
    vae.precision = "exact"
    imgs = synth.randn_seeded((10, 3, 16, 16), 72).tanh()
    data = torch.utils.data.TensorDataset(imgs, torch.zeros(10, dtype=torch.long))
    value = FID.compute_rfid(data, vae, batch_size=4, device=torch.device(DEV))
    # the restatement's features of the originals and of the reconstructions (one image per RQVAE call, as the reference does)
    xs = torch.clamp(imgs * 0.5 + 0.5, 0, 1).to(DEV)
    with torch.no_grad():
        recon = torch.cat([vae(2. * xs[i:i + 1] - 1.)[0] for i in range(10)])
        recon = torch.clamp(recon * 0.5 + 0.5, 0, 1)
        fo = restated.forward(xs.double())[0][3].reshape(10, -1).cpu().numpy()
        fr = restated.forward(recon.double())[0][3].reshape(10, -1).cpu().numpy()
    mo, so = FID.mean_covar_numpy(fo)
    mr, sr = FID.mean_covar_numpy(fr)
    got = FID.compute_statistics_dataset(data, batch_size=4, stage1_model=vae, device=torch.device(DEV))
    for a, b in zip(got, (mo, so, mr, sr)):
        assert np.linalg.norm(a - b) <= 1e-4 * np.linalg.norm(b)
    assert value == FID.frechet_distance(*got)


def test_native_vae_reconstructs_each_image_on_its_own():
    from tests.test_gpu_vae_sizes import build
    from oracle.zoo import VAE_ZOO
    vae, _ = build("tiny", VAE_ZOO["tiny"], 71)
    for p in ("exact", "fast"):
        vae.precision = p
        x = synth.randn_seeded((6, 3, 16, 16), 73).tanh().to(DEV)
        whole = vae(x)[0]
        for i in (0, 5):
            assert torch.equal(vae(x[i:i + 1])[0][0], whole[i]), p
