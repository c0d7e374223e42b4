"""ResNet-101 and rejection sampling without a GPU: the state_dict layout against torchvision's, the weight lookup, every argument error,
the exports, and the float64 restatement pinned to the torchvision fixture (tests/golden/resnet.pt)."""
import os

import pytest
import torch

from rqvae import _native as N
from rqvae.metrics import resnet as RN
from rqvae.metrics.resnet import ResNet101, get_resnet101, resnet101_weights_path
from tests import resnet_oracle as RO
from tests.helpers import ar_config


def test_state_dict_matches_torchvision_and_its_file_loads_strictly(tmp_path):
    tv = pytest.importorskip("torchvision")
    ref = tv.models.resnet101().state_dict()
    ours = ResNet101().state_dict()
    assert list(ours) == list(ref)
    assert all(ours[k].shape == ref[k].shape and ours[k].dtype == ref[k].dtype for k in ref)
    assert {k: tuple(v.shape) for k, v in ours.items()} == RO.state_dict_shapes()
    path = str(tmp_path / "r101.pth")
    torch.save(RO.synth_weights(3), path)
    m = get_resnet101(path)
    assert torch.equal(m.layer3[22].bn3.running_var, RO.synth_weights(3)["layer3.22.bn3.running_var"])
    assert not any(p.requires_grad for p in m.parameters()) and not m.training


def test_weight_path_and_missing_file(tmp_path, monkeypatch):
    monkeypatch.setenv("TORCH_HOME", str(tmp_path))
    p = resnet101_weights_path()
    assert p == os.path.join(torch.hub.get_dir(), "checkpoints", "resnet101-63fe2227.pth")
    with pytest.raises(FileNotFoundError) as e:
        get_resnet101()
    assert p in str(e.value) and RN.RESNET101_URL in str(e.value)
    with pytest.raises(FileNotFoundError, match="nowhere.pth"):
        get_resnet101(str(tmp_path / "nowhere.pth"))


@pytest.mark.parametrize("shape,crop,what", [
    ((3, 32, 32), None, "4-D"), ((1, 1, 32, 32), None, "channels"), ((1, 4, 64, 64), None, "channels"),
    ((1, 3, 31, 64), None, ">= 32"), ((1, 3, 64, 16), None, ">= 32"), ((1, 3, 200, 256), 224, "smaller than center_crop"),
    ((1, 3, 256, 223), 224, "smaller than center_crop"), ((1, 3, 64, 64), 16, "center_crop must be"),
    ((1, 3, 64, 64), 32.0, "center_crop must be"), ((1, 3, 64, 64), True, "center_crop must be"), ((1, 3, 64, 64), None, "CUDA")])
def test_value_errors_before_any_native_call(shape, crop, what):
    m = ResNet101()
    x = torch.rand(*shape)
    with pytest.raises(ValueError, match=what):
        m(x, center_crop=crop)
    with pytest.raises(ValueError, match=what):
        m.class_log_prob(x, torch.zeros(shape[0] if len(shape) == 4 else 1, dtype=torch.long), center_crop=crop)
    assert m._eng == {}


@pytest.mark.parametrize("labels,what", [
    (torch.zeros(2, dtype=torch.float32), "integer"), (torch.zeros(2, 1, dtype=torch.long), "integer"),
    (torch.zeros(3, dtype=torch.long), "integer"), (torch.zeros(2, dtype=torch.bool), "integer"), ([0, 1], "integer"),
    (torch.tensor([0, 1000]), r"\[0, 1000\)"), (torch.tensor([-1, 3]), r"\[0, 1000\)")])
def test_label_errors(labels, what):
    m = ResNet101()
    with pytest.raises(ValueError, match=what):
        m.class_log_prob(torch.rand(2, 3, 64, 64), labels, center_crop=None)


def test_exports():
    from rqvae.metrics import resnet
    from rqvae.models.rqtransformer import rejection_sample
    from rqvae.models.rqtransformer.rejection import rejection_sample as rs
    assert rejection_sample is rs
    assert resnet.ResNet101 is ResNet101
    L = RN._lib()
    for name in RN.EXPORTS:
        assert hasattr(L, name), name
    assert len(RN.EXPORTS) == 11 and "rqb200_resnet_create" in N.EXPORTS
    assert L.rqb200_version() == 118


def test_torchvision_is_not_imported():
    src = open(RN.__file__).read()
    assert "import torchvision" not in src and "from torchvision" not in src


@pytest.mark.slow
def test_oracle_matches_torchvision_fixture(golden):
    fx = golden("resnet")
    sd = RO.sd_as(RO.synth_weights(fx["seed"]))
    torch.set_grad_enabled(False)
    for case in fx["cases"]:
        x = RO.case_inputs(case).double()
        got = RO.logits(sd, x, case["crop"])
        err = float((got - case["logits"]).norm() / case["logits"].norm())
        assert err <= 1e-10, (case["name"], err)


# ------------------------------------------------------------------------------------------------ rejection_sample arguments
class _Clf:
    def class_log_prob(self, *a, **k):
        raise AssertionError("nothing may run before the arguments are checked")


def _ar(name="tiny"):
    from rqvae.models import create_model
    with torch.device("meta"):
        ar, _ = create_model(ar_config(name))
    return ar


@pytest.mark.parametrize("kw,what", [
    (dict(candidates=0), "candidates"), (dict(candidates=-3), "candidates"), (dict(candidates=2.0), "candidates"),
    (dict(candidates=True), "candidates"), (dict(batch_size=0), "batch_size"),
    (dict(labels=torch.tensor([0, 10])), r"\[0, 10\)"), (dict(labels=torch.tensor([-1])), r"\[0, 10\)"),
    (dict(labels=torch.zeros(2, 1, dtype=torch.long)), "integer"), (dict(labels=torch.zeros(2)), "integer"),
    (dict(labels=torch.zeros(0, dtype=torch.long)), "non-empty")])
def test_rejection_sample_argument_checks(kw, what):
    from rqvae.models.rqtransformer import rejection_sample
    args = dict(labels=torch.tensor([0, 9]), candidates=2)
    args.update(kw)
    labels = args.pop("labels")
    with pytest.raises(ValueError, match=what):
        rejection_sample(_ar(), None, _Clf(), labels, **args)


def test_rejection_sample_needs_a_class_condition():
    from rqvae.models import create_model
    from rqvae.models.rqtransformer import rejection_sample
    cfg = ar_config("tiny")
    cfg.vocab_size_cond = 1
    with torch.device("meta"):
        ar, _ = create_model(cfg)
    with pytest.raises(ValueError, match="no class condition"):
        rejection_sample(ar, None, _Clf(), torch.tensor([0]))
    with pytest.raises(ValueError, match="no class condition"):
        rejection_sample(_ar("tiny_txt"), None, _Clf(), torch.tensor([0]))
