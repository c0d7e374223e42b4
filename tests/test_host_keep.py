"""Masked completion on the host: the entry points are declared, exported and bound; sample()'s keep_mask is checked (bool, broadcasts
to [B, H, W, D], the model's device) and laid out for the engine (uint8, the start_loc prefix kept) before anything reaches a device."""
import ctypes as C
import os
import re

import pytest
import torch

from rqvae import _native as N
from tests.test_host_cpu import make_ar

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_sample_span_takes_the_keep_arguments_and_append_attn_is_bound():
    hdr = open(os.path.join(ROOT, "include", "rqb200.h")).read()
    L = N.lib()
    for name in ("rqb200_ar_sample_span", "rqb200_dbg_append_attn"):
        assert re.search(r"\bint %s\s*\(" % name, hdr)
        assert name in N.EXPORTS
        assert hasattr(C.CDLL(N.LIB_PATH), name)
    assert L.rqb200_ar_sample_span.argtypes[-4:] == [C.c_void_p, C.c_void_p, C.c_int, C.c_float]     # keep, sampled_host, cfg_n, cfg_scale
    assert L.rqb200_version() >= 112


def _forbid_native(monkeypatch):
    def boom(*a, **k):
        raise AssertionError("a native call was reached")
    monkeypatch.setattr(N, "lib", boom)


@pytest.mark.parametrize("name", ["tiny", "tiny_txt"])
def test_bad_keep_masks_raise_before_any_native_call(name, monkeypatch):
    model = make_ar(name)
    B = 3
    H, W, D = model.block_size
    part = torch.zeros(B, H, W, D, dtype=torch.long)
    _forbid_native(monkeypatch)
    bad = [torch.ones(H, W, D, dtype=torch.uint8), torch.ones(H, W, D), [[True]], torch.ones(B + 1, H, W, D, dtype=torch.bool),
           torch.ones(H, W + 1, 1, dtype=torch.bool), torch.ones(2, B, H, W, D, dtype=torch.bool), torch.ones(D + 1, dtype=torch.bool),
           torch.ones(H, W, D, dtype=torch.bool, device="meta")]
    for k in bad:
        with pytest.raises(ValueError):
            model.sample(part, keep_mask=k)


def test_keep_mask_broadcasts_and_keeps_the_prefix():
    model = make_ar("tiny")
    B = 3
    H, W, D = model.block_size
    region = torch.zeros(H, W, 1, dtype=torch.bool)
    region[0, 0] = True
    k = model._keep_mask(region, B, (0, 0))
    assert k.dtype == torch.uint8 and k.is_contiguous() and k.shape == (B, H, W, D)
    assert torch.equal(k, region.expand(B, H, W, D).to(torch.uint8))
    depth = torch.tensor([True] + [False] * (D - 1)).view(1, 1, 1, D)
    k = model._keep_mask(depth, B, (1, 2))
    flat = k.view(B, H * W, D)
    assert bool((flat[:, :W + 2] == 1).all())                          # positions before start_loc are kept whole
    assert torch.equal(flat[:, W + 2:], depth.view(1, 1, D).expand(B, H * W - W - 2, D).to(torch.uint8))
    per_image = torch.rand(B, H, W, D) > 0.5
    assert torch.equal(model._keep_mask(per_image, B, (0, 0)).bool(), per_image)
    assert model._keep_mask(None, B, (0, 0)) is None
