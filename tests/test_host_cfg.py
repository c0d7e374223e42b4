"""Classifier-free guidance on the host: the one sampling entry point is declared, exported and bound with its guidance arguments, the
entry points it replaced are gone, sample() refuses bad guidance arguments with ValueError before anything reaches a device, the native
entry refuses a row count that is not 2 cfg_n before any CUDA call, and a guided fast-tier call is split into equal chunks of at most
128 images."""
import ctypes as C
import os
import re

import pytest
import torch

from rqvae import _native as N
from rqvae.models.rqtransformer.transformers import _chunk_bounds
from tests.test_host_cpu import make_ar

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SPAN = "rqb200_ar_sample_span"
PREFIX = SPAN[:-len("_span")]
# the entry points rqb200_ar_sample_span replaced: the start_loc form, the guided form and the masked form
REMOVED = (PREFIX, SPAN + "_cfg", SPAN + "_keep")


def test_sample_span_is_the_one_sampling_entry_and_takes_guidance():
    hdr = open(os.path.join(ROOT, "include", "rqb200.h")).read()
    assert re.search(r"\bint %s\s*\(" % SPAN, hdr)
    assert SPAN in N.EXPORTS
    so = C.CDLL(N.LIB_PATH)
    assert hasattr(so, SPAN)
    L = N.lib()
    argtypes = getattr(L, SPAN).argtypes
    assert len(argtypes) == 22 and argtypes[-4:] == [C.c_void_p, C.c_void_p, C.c_int, C.c_float]     # keep, sampled_host, cfg_n, cfg_scale
    assert set(re.findall(r"\b(%s\w*)\s*\(" % PREFIX, hdr)) == {SPAN}
    assert {n for n in N.EXPORTS if n.startswith(PREFIX)} == {SPAN}
    for name in REMOVED:
        assert not hasattr(so, name), name
    assert L.rqb200_version() >= 113


def _errors(model, B, cl):
    part = torch.zeros(B, *model.block_size, dtype=torch.long)
    good = torch.zeros(B, cl, dtype=torch.long)
    cases = [dict(cfg_scale=1.5), dict(uncond=good), dict(cfg_scale=1.5, uncond=torch.zeros(B + 1, cl, dtype=torch.long)),
             dict(cfg_scale=1.5, uncond=torch.full((B, cl), -1)), dict(cfg_scale=1.5, uncond=torch.full((B, cl), model.vocab_size_cond)),
             dict(cfg_scale=1.5, uncond=good.float()), dict(cfg_scale="2", uncond=good), dict(cfg_scale=None, uncond=None, _ok=True)]
    return part, cases


@pytest.mark.parametrize("name", ["tiny", "tiny_txt"])
def test_guidance_arguments_are_checked_first(name):
    model = make_ar(name)
    cl = model.block_size_cond
    part, cases = _errors(model, 3, cl)
    for kw in cases:
        if kw.pop("_ok", False):
            assert model._guidance(3, **kw) is None
            continue
        with pytest.raises(ValueError):
            model.sample(part, cond=torch.zeros(3, cl, dtype=torch.long), **kw)
    # anything that reshapes to [B, cond_len] is accepted: [B * cond_len] and [B, 1, cond_len]
    s, u = model._guidance(3, 2, torch.ones(3 * cl, dtype=torch.int32))
    assert s == 2.0 and isinstance(s, float) and u.shape == (3, cl) and u.dtype == torch.int64
    assert model._guidance(3, 0.0, torch.zeros(3, 1, cl, dtype=torch.long))[0] == 0.0


def test_guidance_needs_a_conditional_model():
    model = make_ar("ffhq355m", "meta")          # vocab_size_cond == 1
    with pytest.raises(ValueError):
        model.sample(torch.zeros(2, *model.block_size, dtype=torch.long), cfg_scale=1.5, uncond=torch.zeros(2, 1, dtype=torch.long))


def test_guided_chunks_hold_at_most_128_images():
    assert _chunk_bounds(300, N.MODE_FAST, 128) == [(0, 100), (100, 200), (200, 300)]
    assert _chunk_bounds(256, N.MODE_FAST, 128) == [(0, 128), (128, 256)]
    assert _chunk_bounds(128, N.MODE_FAST, 128) == [(0, 128)]
    assert _chunk_bounds(300, N.MODE_EXACT, 128) == [(0, 300)]
    assert _chunk_bounds(300, N.MODE_FAST) == [(0, 150), (150, 300)]        # unguided: unchanged


def test_sample_span_refuses_rows_other_than_2_cfg_n_before_any_cuda_call():
    """B must be 2 cfg_n rows when cfg_n > 0, and cfg_n >= 0: refused with EINVAL before the device is looked at (no GPU here)"""
    torch.manual_seed(0)
    model = make_ar("tiny")
    cfg, w, keep, _ = model._engine_structs(torch.randn(model.vocab_size[0], 256), N.MODE_EXACT)
    L = N.lib()
    h = L.rqb200_ar_create(C.byref(cfg), C.byref(w))
    assert h, L.rqb200_last_error().decode()
    try:
        kk, pp = (C.c_int32 * 4)(*[512] * 4), (C.c_float * 4)(*[1.0] * 4)
        buf = C.create_string_buffer(64)
        for B, cfg_n in ((0, 1), (1, 1), (3, 1), (4, 1), (2, -1)):
            rc = L.rqb200_ar_sample_span(h, buf, None, B, 0, 16, 0, 1.0, kk, pp, None, 0, None, None, buf, buf, 64, None, None, None,
                                         cfg_n, C.c_float(1.5))
            assert rc == N.EINVAL, (B, cfg_n)
            assert B < 1 or "2n rows" in L.rqb200_last_error().decode(), (B, cfg_n)
    finally:
        L.rqb200_ar_destroy(h)
