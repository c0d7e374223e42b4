"""FID Inception-v3 and FID statistics on the host (no GPU): the torch restatement against the reference's fixture
(tests/golden/fid.pt, scripts/gen_golden_inception.py), the InceptionV3 state_dict layout and weight loading, the input checks,
frechet_distance / mean_covar_*, and the engine's C exports."""
import ctypes
import logging
import os
import socket

import numpy as np
import pytest
import torch

from rqvae import _native as N
from rqvae.metrics import fid as FID
from rqvae.metrics import inception as INC
from tests import inception_oracle as IO


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


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


@pytest.fixture
def model(torch_home, monkeypatch):
    monkeypatch.setenv("TORCH_HOME", torch_home)
    return INC.InceptionV3([0, 1, 2, 3])


@pytest.mark.parametrize("idx", range(7))
def test_restatement_matches_reference_fixture(fixture, weights, idx):
    case = fixture["cases"][idx]
    net = IO.Restated({k: v.double() for k, v in weights.items()})
    with torch.no_grad():
        outs, logits = net.forward(IO.fixture_input(case).double(), resize_input=case["resize"])
    assert rel(outs[3].reshape(case["B"], -1), case["features"]) <= 1e-5
    assert rel(logits, case["logits"]) <= 1e-5
    for k in range(3):
        assert list(outs[k].shape) == case["block_shapes"][k]
        assert rel(outs[k].mean((2, 3)), case["means"][k]) <= 1e-5


def test_block_extents_match_the_reference(fixture):
    for case in fixture["cases"]:
        ext = INC.block_extents(case["H"], case["W"], case["resize"])
        assert [list(e) for e in ext] == [s[2:] for s in case["block_shapes"]]


def test_state_dict_layout_equals_the_reference(model, fixture):
    got = [(k, list(v.shape)) for k, v in model.state_dict().items()]
    assert got == [(k, list(s)) for k, s in fixture["layout"]]
    assert len(got) == 566
    wrapper = FID.InceptionWrapper([3])
    assert [k for k in wrapper.state_dict()] == [k for k, _ in fixture["layout"]]


def test_weight_file_fills_every_parameter(model, weights):
    sd = model.state_dict()
    for k, v in weights.items():
        if k.endswith("num_batches_tracked"):
            continue
        assert torch.equal(sd[k], v), k


def test_partial_output_blocks_hold_only_their_blocks(torch_home, monkeypatch):
    monkeypatch.setenv("TORCH_HOME", torch_home)
    m = INC.InceptionV3([1])
    assert {k.split(".")[1] for k in m.state_dict() if k.startswith("blocks.")} == {"0", "1"}
    assert FID.get_inception_model(768).output_blocks == [2]


def test_missing_weight_file_names_the_hub_path_and_never_connects(tmp_path, monkeypatch):
    def no_network(*a, **k):
        raise AssertionError("a network connection was attempted")
    monkeypatch.setattr(socket.socket, "connect", no_network)
    monkeypatch.setattr(socket.socket, "connect_ex", no_network)
    monkeypatch.setenv("TORCH_HOME", str(tmp_path))
    want = os.path.join(str(tmp_path), "hub", "checkpoints", "pt_inception-2015-12-05-6726825d.pth")
    assert INC.fid_weights_path() == want
    with pytest.raises(FileNotFoundError, match=want.replace(".", r"\.")):
        INC.InceptionV3()
    with pytest.raises(FileNotFoundError, match="elsewhere.pth"):
        INC.fid_inception_v3(str(tmp_path / "elsewhere.pth"))


def test_explicit_weight_path(torch_home, weights):
    inc = INC.fid_inception_v3(os.path.join(torch_home, "hub", "checkpoints", INC.FID_WEIGHTS_FILE))
    assert torch.equal(inc.Mixed_7c.branch_pool.bn.running_var, weights["blocks.3.2.branch_pool.bn.running_var"])


def test_torchvision_imagenet_inception_is_refused(torch_home, monkeypatch):
    monkeypatch.setenv("TORCH_HOME", torch_home)
    with pytest.raises(NotImplementedError, match="torchvision"):
        INC.InceptionV3(use_fid_inception=False)


@pytest.mark.parametrize("shape, resize", [((3, 299, 299), True), ((1, 2, 3, 299, 299), True), ((1, 4, 299, 299), True),
                                           ((1, 1, 299, 299), True), ((0, 3, 299, 299), True), ((1, 3, 0, 5), True),
                                           ((1, 3, 74, 74), False), ((1, 3, 75, 74), False), ((1, 3, 74, 200), False)])
def test_bad_inputs_raise_value_error_before_any_native_call(model, shape, resize):
    model.resize_input = resize
    with pytest.raises(ValueError):
        model(torch.zeros(shape))


def test_return_logits_needs_block_3(torch_home, monkeypatch):
    monkeypatch.setenv("TORCH_HOME", torch_home)
    with pytest.raises(ValueError, match="block 3"):
        INC.InceptionV3([2])(torch.zeros(1, 3, 299, 299), return_logits=True)


def test_precision_selects_the_tier(model, monkeypatch):
    monkeypatch.delenv("RQB200_PRECISION", raising=False)
    assert model._mode() == N.MODE_EXACT
    monkeypatch.setenv("RQB200_PRECISION", "fast")
    assert model._mode() == N.MODE_FAST
    model.precision = "exact"
    assert model._mode() == N.MODE_EXACT


def test_mean_covar_and_frechet_match_the_reference(fixture):
    f = fixture["frechet"]
    mu1, s1 = FID.mean_covar_numpy(f["x1"].numpy())
    np.testing.assert_allclose(mu1, f["mu1"].numpy(), rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(s1, f["sigma1"].numpy(), rtol=1e-12, atol=1e-14)
    mu_t, s_t = FID.mean_covar_torch(f["x1"])
    np.testing.assert_allclose(mu_t.numpy()[0], f["mu1"].numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(s_t.numpy(), f["sigma1"].numpy(), rtol=1e-10, atol=1e-12)
    mu2, s2 = FID.mean_covar_numpy(f["x2"])
    fd = FID.frechet_distance(mu1, s1, mu2, s2)
    assert fd == pytest.approx(f["fd"], rel=1e-9)
    n = f["n_singular"]
    _, r1 = FID.mean_covar_numpy(f["x1"][:n])
    _, r2 = FID.mean_covar_numpy(f["x2"][:n])
    assert FID.frechet_distance(mu1, r1, mu2, r2) == pytest.approx(f["fd_singular"], rel=1e-6)


def test_frechet_retries_with_eps_when_sqrtm_is_not_finite(fixture, monkeypatch, caplog):
    f = fixture["frechet"]
    mu1, s1, mu2, s2 = (f[k].numpy() for k in ("mu1", "sigma1", "mu2", "sigma2"))
    calls = []
    real = FID._sqrtm

    def first_not_finite(a):
        calls.append(a.copy())
        return np.full_like(a, np.nan) if len(calls) == 1 else real(a)
    monkeypatch.setattr(FID, "_sqrtm", first_not_finite)
    eps = 1e-3
    with caplog.at_level(logging.WARNING):
        got = FID.frechet_distance(mu1, s1, mu2, s2, eps=eps)
    assert "singular product" in caplog.text
    off = np.eye(s1.shape[0]) * eps
    np.testing.assert_array_equal(calls[1], (s1 + off).dot(s2 + off))
    d = mu1 - mu2
    want = d.dot(d) + np.trace(s1) + np.trace(s2) - 2 * np.trace(np.real(real((s1 + off).dot(s2 + off))))
    assert got == pytest.approx(want, rel=1e-12)


def test_compute_is_and_clip_score_stay_placeholders():
    import rqvae.metrics as M
    for fn in (M.compute_IS, M.compute_clip_score):
        with pytest.raises(NotImplementedError):
            fn()
    assert M.compute_fid is FID.compute_fid


def test_inception_exports_exist():
    lib = ctypes.CDLL(N.LIB_PATH)
    for name in INC.EXPORTS:
        assert hasattr(lib, name), name
    assert N.lib().rqb200_version() >= 116
