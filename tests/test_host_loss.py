"""The reference's stage-2 losses (RQTransformer.compute_loss / compute_cond_loss / compute_codebook_loss, transformers.py:371-410) on
CPU tensors, against the values the unmodified reference computed on the same inputs (tests/golden/loss.pt, scripts/gen_golden_loss.py)."""
import os

import pytest
import torch

from rqvae.models import create_model
from rqvae.models.ema import ExponentialMovingAverage
from rqvae.utils.config import Config, augment_arch_defaults

GOLDEN = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "loss.pt"), weights_only=False)
CASES = sorted(GOLDEN)


def _model(case):
    g = GOLDEN[case]
    cfg = Config(type="rq-transformer", vocab_size=g["vocab"], block_size=list(g["block_size"]), vocab_size_cond=g["vocab_cond"],
                 block_size_cond=g["cond_len"], embed_dim=128, input_embed_dim=256, shared_tok_emb=True, shared_cls_emb=True,
                 input_emb_vqvae=True, head_emb_vqvae=True, cumsum_depth_ctx=True,
                 body=dict(n_layer=1, block=dict(n_head=2)), head=dict(n_layer=1, block=dict(n_head=2)))
    with torch.device("meta"):
        model, _ = create_model(augment_arch_defaults(cfg))
    return model


def _close(got, want):
    got, want = got.double(), want.double()
    assert got.shape == want.shape
    assert torch.all((got - want).abs() <= 1e-6 * want.abs().clamp_min(1e-30)), (got, want)


@pytest.mark.parametrize("case", CASES)
def test_compute_loss_matches_reference(case):
    m, g = _model(case), GOLDEN[case]
    x = g["inputs"]
    _close(m.compute_loss(x["logits"], x["targets"]), g["ref"]["loss"])
    _close(m.compute_loss(x["logits"], x["soft_targets"], use_soft_target=True), g["ref"]["loss_soft"])


@pytest.mark.parametrize("case", CASES)
def test_compute_cond_loss_matches_reference(case):
    m, g = _model(case), GOLDEN[case]
    _close(m.compute_cond_loss(g["inputs"]["cond_logits"], g["inputs"]["conds"]), g["ref"]["cond_loss"])


@pytest.mark.parametrize("case", CASES)
def test_compute_codebook_loss_matches_reference(case):
    m, g = _model(case), GOLDEN[case]
    x = g["inputs"]
    _close(m.compute_codebook_loss(x["logits"], x["targets"]), g["ref"]["codebook_loss"])
    _close(m.compute_codebook_loss(x["logits"], x["soft_targets"], use_soft_target=True), g["ref"]["codebook_loss_soft"])


def test_hard_target_loss_is_plain_cross_entropy():
    """compute_loss with hard targets is F.cross_entropy over the flattened logits, bit for bit"""
    x = GOLDEN["unit"]["inputs"]
    want = torch.nn.functional.cross_entropy(x["logits"].reshape(-1, x["logits"].shape[-1]), x["targets"].reshape(-1))
    assert torch.equal(_model("unit").compute_loss(x["logits"], x["targets"]), want)


def test_losses_reach_through_the_ema_wrapper():
    """the EMA wrapper forwards attributes to the wrapped model: the three losses are callable through it"""
    ema = ExponentialMovingAverage(_model("unit"), 0.999)
    g = GOLDEN["unit"]
    x = g["inputs"]
    _close(ema.compute_cond_loss(x["cond_logits"], x["conds"]), g["ref"]["cond_loss"])
    _close(ema.compute_codebook_loss(x["logits"], x["targets"]), g["ref"]["codebook_loss"])
