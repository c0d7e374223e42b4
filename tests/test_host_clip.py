"""CLIP score on the host (no GPU): the tokenizer against the reference SimpleTokenizer's ids (tests/golden/clip.pt), geometry inference
from state_dicts, the weight and vocabulary lookups, clip_score's argument checks, the engine's resize plan against PIL, tier
selection and the C exports."""
import ctypes
import hashlib
import os

import numpy as np
import pytest
import torch
from PIL import Image

from rqvae import _native as N
from rqvae.metrics import clip_score as CS
from tests import clip_oracle as CO

# CLIP's merge list reduced to the merges the fixture's texts use, every merge at its own rank (scripts/gen_golden_clip.py)
BPE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "clip_bpe_subset.txt.gz")


@pytest.fixture(scope="module")
def fixture(golden):
    return golden("clip")


def test_tokenizer_reproduces_reference_ids(fixture):
    for cap, ids in zip(fixture["captions"], fixture["caption_ids"]):
        if len(ids) <= 77:
            got = CS.tokenize([cap], bpe_path=BPE)[0]
            assert got[:len(ids)].tolist() == ids, cap
            assert not got[len(ids):].any()
    assert CS.tokenize("a photo of a cat", bpe_path=BPE).shape == (1, 77)


def test_tokenizer_too_long_and_truncate(fixture):
    cap, ids = fixture["captions"][-1], fixture["caption_ids"][-1]
    assert len(ids) > 77
    with pytest.raises(RuntimeError, match="too long for context length 77"):
        CS.tokenize([cap], bpe_path=BPE)
    got = CS.tokenize([cap], truncate=True, bpe_path=BPE)[0].tolist()
    assert got == ids[:76] + [CS.EOT]
    assert CS.tokenize([cap], context_length=len(ids), bpe_path=BPE)[0].tolist() == ids


def test_vocab_lookup_raises_file_not_found(tmp_path):
    missing = str(tmp_path / "nope.txt.gz")
    with pytest.raises(FileNotFoundError, match="nope.txt.gz"):
        CS.tokenize(["x"], bpe_path=missing)


def test_weight_lookup_raises_file_not_found(tmp_path, monkeypatch):
    monkeypatch.setenv("HOME", str(tmp_path))
    with pytest.raises(FileNotFoundError, match=str(tmp_path / ".cache" / "clip" / "ViT-B-32.pt")):
        CS.get_clip(bpe_path=BPE)
    with pytest.raises(FileNotFoundError, match="given.pt"):
        CS.get_clip(path=str(tmp_path / "given.pt"), bpe_path=BPE)
    assert CS.clip_weights_path("ViT-L/14@336px").endswith("ViT-L-14-336px.pt")


def test_geometry_inference():
    for g, G in CO.GEOMS.items():
        if g == "b32":
            sd = {k: torch.empty(s) for k, s in CO.shapes(g)}
        else:
            sd = CO.synth_state_dict(g, 1)
        cfg = CS.clip_config_of(sd)
        assert cfg == dict(embed_dim=G["embed"], vision_width=G["vw"], vision_layers=G["vl"], vision_patch_size=G["patch"],
                           context_length=G["ctx"], vocab_size=G["vocab"], transformer_width=G["tw"], transformer_layers=G["tl"],
                           image_resolution=G["res"])


def test_build_model_round_trip_and_attributes():
    sd = CO.synth_state_dict("tiny", 3)
    m = CS.build_model(dict(sd, input_resolution=torch.tensor(32), context_length=torch.tensor(77), vocab_size=torch.tensor(49408)))
    assert m.visual.input_resolution == 32 and m.context_length == 77 and m.vocab_size == 49408
    got = m.state_dict()
    assert set(got) == set(sd)
    assert all(torch.equal(got[k], sd[k]) for k in sd)


def test_resnet_and_width_errors():
    with pytest.raises(ValueError, match="ResNet"):
        CS.clip_config_of({"visual.layer1.0.conv1.weight": torch.empty(1), "text_projection": torch.empty(1, 1)})
    sd = {k: torch.empty(s) for k, s in CO.shapes(dict(CO.GEOMS["tiny"], vw=96))}
    with pytest.raises(ValueError, match="vision_width 96"):
        CS.clip_config_of(sd)
    with pytest.raises(ValueError, match="ResNet"):
        CS.CLIP(512, 224, (3, 4, 6, 3), 64, None, 77, 49408, 512, 8, 12)


def test_get_clip_reads_torchscript_and_plain_files(tmp_path):
    sd = CO.synth_state_dict("tiny", 4)
    plain = tmp_path / "plain.pt"
    torch.save({k: v.half() for k, v in sd.items()}, plain)
    m, pre = CS.get_clip(path=str(plain), bpe_path=BPE)
    assert all(torch.equal(m.state_dict()[k], sd[k]) for k in sd)
    assert isinstance(pre, CS.ClipPreprocess) and pre.n_px == 32

    class Holder(torch.nn.Module):
        def __init__(self):
            super().__init__()
            for k, v in sd.items():
                self.register_buffer(k.replace(".", "__"), v.half())
    scripted = torch.jit.script(Holder())
    # a TorchScript archive whose state_dict carries OpenAI's keys: a scripted CLIP from a renamed holder
    arch = tmp_path / "ViT-T-8.pt"
    scripted.save(str(arch))
    got = CS.load_state_dict_file(str(arch))
    assert {k.replace("__", ".") for k in got} == set(sd)


def _score_args():
    sd = CO.synth_state_dict("tiny", 5)
    m = CS.build_model(sd)
    m.bpe_path = BPE
    return m, CS.ClipPreprocess(32)


def test_clip_score_value_errors():
    m, pre = _score_args()
    ok = torch.rand(2, 3, 40, 40)
    with pytest.raises(ValueError, match="4-D"):
        CS.clip_score(torch.rand(3, 40, 40), ["a", "b"], m, pre)
    with pytest.raises(ValueError, match="channels"):
        CS.clip_score(torch.rand(2, 4, 40, 40), ["a", "b"], m, pre)
    with pytest.raises(ValueError, match="empty"):
        CS.clip_score(torch.rand(0, 3, 40, 40), [], m, pre)
    with pytest.raises(ValueError, match="3 captions for 2 images"):
        CS.clip_score(ok, ["a", "b", "c"], m, pre)
    bad = torch.zeros(2, 77, dtype=torch.long)
    bad[1, 3] = 49408
    with pytest.raises(ValueError, match=r"\[0, 49408\)"):
        CS.clip_score(ok, bad, m, pre)
    with pytest.raises(ValueError, match=r"\[0, 49408\)"):
        CS.clip_score(ok, -torch.ones(2, 77, dtype=torch.long), m, pre)
    with pytest.raises(ValueError, match="for 2 images"):
        CS.clip_score(ok, torch.zeros(3, 77, dtype=torch.long), m, pre)


@pytest.mark.parametrize("H,W", [(256, 256), (224, 224), (512, 512), (384, 256), (255, 257), (200, 300), (64, 64), (300, 200), (223, 225)])
def test_resize_plan_matches_pil(H, W):
    from torchvision import transforms as T
    R = 224
    img = Image.fromarray(np.zeros((H, W, 3), np.uint8))
    resized = T.Resize(R, interpolation=T.InterpolationMode.BICUBIC)(img)
    Hr, Wr, top, left, ksh, ksv = CS.resize_plan(H, W, R)
    assert (Wr, Hr) == resized.size
    assert (Hr, Wr) == CS.resized_extent(H, W, R)
    assert (top, left) == CS.crop_offsets(Hr, Wr, R)
    # CenterCrop's box, by a crop of an image whose pixels are their own coordinates
    yy, xx = np.meshgrid(np.arange(Hr) % 256, np.arange(Wr) % 256, indexing="ij")
    coords = Image.fromarray(np.stack([yy, xx, yy * 0], -1).astype(np.uint8))
    c = np.asarray(T.CenterCrop(R)(coords))
    assert c[0, 0, 0] == top % 256 and c[0, 0, 1] == left % 256
    assert (ksh == 0) == (Wr == W) and (ksv == 0) == (Hr == H)


def test_host_preprocess_matches_reference_route(fixture):
    for name, case in fixture["pix"].items():
        x = CO.pixels(case["seed"], 1, case["H"], case["W"])
        img = Image.fromarray((np.transpose(x[0].numpy(), (1, 2, 0)) * 255).astype(np.uint8))
        got = CS.ClipPreprocess(224)(img)
        assert hashlib.sha256(got.numpy().tobytes()).hexdigest() == case["norm_sha256"], name


def test_tier_selection(monkeypatch):
    m, _ = _score_args()
    monkeypatch.delenv("RQB200_PRECISION", raising=False)
    assert m._mode() == N.MODE_EXACT
    monkeypatch.setenv("RQB200_PRECISION", "fast")
    assert m._mode() == N.MODE_FAST
    m.precision = "exact"
    assert m._mode() == N.MODE_EXACT
    monkeypatch.delenv("RQB200_PRECISION")
    m.precision = "fast"
    assert m._mode() == N.MODE_FAST


def test_clip_exports_exist():
    lib = ctypes.CDLL(N.LIB_PATH)
    for name in [e for e in N.EXPORTS if "clip" in e]:
        assert hasattr(lib, name), name
    assert N.lib().rqb200_version() == 118
