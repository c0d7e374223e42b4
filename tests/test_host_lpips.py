"""LPIPS on the host (no GPU): the torch restatement against the reference's fixture (tests/golden/lpips.pt, scripts/gen_golden_lpips.py),
the state_dict layout and weight loading, the argument checks (all before any native call), and the engine's C exports."""
import ctypes
import os

import pytest
import torch

from rqvae import _native as N
from rqvae.losses import LPIPS as LPIPS_pkg
from rqvae.losses.vqgan import LPIPS
from rqvae.losses.vqgan import lpips as LP
from rqvae.losses.vqgan import lpips_utils as LU
from tests import lpips_oracle as LO


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


@pytest.fixture(scope="module")
def fixture(golden):
    return golden("lpips")


@pytest.fixture(scope="module")
def weights(fixture):
    return LO.synth_weights(fixture["seed"])


@pytest.fixture(scope="module")
def torch_home(tmp_path_factory, weights):
    home = str(tmp_path_factory.mktemp("torch_home"))
    LO.write_weight_files(home, weights)
    return home


@pytest.fixture
def hub(torch_home, monkeypatch):
    monkeypatch.setenv("TORCH_HOME", torch_home)
    return torch_home


@pytest.mark.parametrize("idx", range(7))
def test_restatement_matches_reference_fixture(fixture, weights, idx):
    case = fixture["cases"][idx]
    sd = {k: v.double() for k, v in weights.items()}
    x0, x1 = LO.case_inputs(case)
    with torch.no_grad():
        layers, val = LO.lpips(sd, x0.double(), x1.double())
        taps = LO.features(sd, x0.double())
    assert [list(t.shape) for t in taps] == case["tap_shapes"]
    if case["kind"] == "identical":
        assert torch.equal(val, torch.zeros_like(val)) and torch.equal(case["val"], torch.zeros_like(case["val"]))
        return
    assert rel(layers, case["layers"]) <= 1e-10
    assert rel(val, case["val"]) <= 1e-10


@pytest.mark.parametrize("dropout", [True, False])
def test_state_dict_layout_equals_the_reference(hub, fixture, dropout):
    m = LPIPS(use_dropout=dropout)
    got = [(k, list(v.shape)) for k, v in m.state_dict().items()]
    assert got == [(k, list(s)) for k, s in fixture["layouts"]["dropout" if dropout else "no_dropout"]]
    assert got[0][0] == "scaling_layer.shift" and got[2][0] == "net.slice1.0.weight" and got[27][0] == "net.slice5.28.bias"
    assert ("lin0.model.1.weight" if dropout else "lin0.model.0.weight") in dict(got)


def test_weight_files_fill_every_parameter(hub, weights):
    sd = LPIPS().state_dict()
    for k, v in weights.items():
        assert torch.equal(sd[k].reshape(v.shape), v), k
    assert not any(p.requires_grad for p in LPIPS().parameters())


def test_lpips_file_lookup_order():
    paths = LU.ckpt_candidates("vgg_lpips")
    assert paths[0].endswith(os.path.join("rqvae", "losses", "vqgan", ".caches", "vgg.pth"))
    assert paths[1] == os.path.join(torch.hub.get_dir(), "checkpoints", "vgg.pth")
    assert LU.ckpt_candidates("vgg_lpips", root="/x") == ["/x/vgg.pth"]


def test_missing_weight_files_name_every_path(tmp_path, monkeypatch):
    monkeypatch.setenv("TORCH_HOME", str(tmp_path))
    with pytest.raises(FileNotFoundError) as e:
        LPIPS()
    assert os.path.join(str(tmp_path), "hub", "checkpoints", "vgg16-397923af.pth") in str(e.value)
    assert LU.VGG16_URL in str(e.value)
    LO.write_weight_files(str(tmp_path), LO.synth_weights(1))
    os.remove(os.path.join(str(tmp_path), "hub", "checkpoints", "vgg.pth"))
    with pytest.raises(FileNotFoundError) as e:
        LPIPS()
    for p in LU.ckpt_candidates("vgg_lpips"):
        assert p in str(e.value)
    assert LU.URL_MAP["vgg_lpips"] in str(e.value)


def test_md5_check(tmp_path):
    (tmp_path / "vgg.pth").write_bytes(b"not the published file")
    with pytest.raises(ValueError, match="md5"):
        LU.get_ckpt_path("vgg_lpips", root=str(tmp_path), check=True)
    assert LU.get_ckpt_path("vgg_lpips", root=str(tmp_path)) == str(tmp_path / "vgg.pth")


@pytest.fixture
def model(hub, monkeypatch):
    m = LPIPS().eval()

    def no_native(*a, **k):
        raise AssertionError("a native call was made")
    monkeypatch.setattr(LP, "_lib", no_native)
    monkeypatch.setattr(m, "_engine", no_native)
    return m


class _FakeCuda(torch.Tensor):
    """a CPU tensor that claims to live on a CUDA device, to reach the checks that follow the device check"""
    @property
    def is_cuda(self):
        return True


@pytest.mark.parametrize("a_shape,b_shape", [((3, 16, 16), (3, 16, 16)), ((1, 4, 16, 16), (1, 4, 16, 16)),
                                             ((2, 3, 16, 16), (1, 3, 16, 16)), ((1, 3, 16, 16), (1, 3, 16, 17)),
                                             ((1, 3, 15, 16), (1, 3, 15, 16)), ((1, 3, 64, 8), (1, 3, 64, 8)),
                                             ((0, 3, 16, 16), (0, 3, 16, 16))])
def test_bad_shapes_raise_before_any_native_call(model, a_shape, b_shape):
    with pytest.raises(ValueError):
        model(torch.zeros(a_shape), torch.zeros(b_shape))


def test_unknown_reduction_raises(model):
    x = torch.zeros(1, 3, 16, 16)
    with pytest.raises(ValueError, match="reduction"):
        model(x, x, reduction="max")


def test_cpu_tensor_raises(model):
    x = torch.zeros(1, 3, 16, 16)
    with pytest.raises(ValueError, match="CUDA"):
        model(x, x, reduction="none")


def test_training_mode_with_dropout_raises(model):
    x = torch.zeros(1, 3, 16, 16).as_subclass(_FakeCuda)
    model.train()
    with pytest.raises(NotImplementedError, match="eval"):
        model(x, x)


def test_training_mode_without_dropout_reaches_the_engine(hub, monkeypatch):
    m = LPIPS(use_dropout=False).train()
    called = []
    monkeypatch.setattr(m, "_engine", lambda dev: called.append(dev) or (_ for _ in ()).throw(RuntimeError("engine")))
    x = torch.zeros(1, 3, 16, 16).as_subclass(_FakeCuda)
    with pytest.raises(RuntimeError, match="engine"):
        m(x, x)
    assert called


def test_requires_grad_raises(model):
    x = torch.zeros(1, 3, 16, 16).as_subclass(_FakeCuda)
    y = torch.zeros(1, 3, 16, 16, requires_grad=True).as_subclass(_FakeCuda)
    with torch.enable_grad():
        with pytest.raises(RuntimeError, match="backward"):
            model(x, y)
        with pytest.raises(RuntimeError, match="backward"):
            model(y, x)


def test_tier_selection(model, monkeypatch):
    monkeypatch.delenv("RQB200_PRECISION", raising=False)
    assert model._mode() == N.MODE_EXACT
    monkeypatch.setenv("RQB200_PRECISION", "fast")
    assert model._mode() == N.MODE_FAST
    model.precision = "exact"
    assert model._mode() == N.MODE_EXACT


def test_helpers_are_the_references(fixture):
    x = torch.randn(2, 8, 3, 5, dtype=torch.float64)
    assert torch.equal(LP.normalize_tensor(x), LO.normalize_tensor(x))
    assert torch.equal(LP.spatial_average(x), x.mean([2, 3], keepdim=True))
    s = LP.ScalingLayer()
    assert torch.equal(s(x[:, :3]), (x[:, :3] - s.shift) / s.scale)
    assert LPIPS_pkg is LPIPS


def test_lpips_exports_exist():
    lib = ctypes.CDLL(N.LIB_PATH)
    for name in [e for e in N.EXPORTS if "lpips" in e]:
        assert hasattr(lib, name), name
    assert len(LP.EXPORTS) == 12
    assert N.lib().rqb200_version() >= 118

