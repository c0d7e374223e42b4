"""Sliding-window sampling on the host: the window origin rule, the segment plan, the one sampling entry point with its canvas extents,
and sample()'s canvas checks, all before anything reaches a device."""
import ctypes as C
import os
import re

import pytest
import torch

from rqvae import _native as N
from rqvae.models.rqtransformer.transformers import CANVAS_MAX_CODES
from tests import window_oracle as WO
from tests.test_host_cpu import make_ar

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SPAN = "rqb200_ar_sample_span"
PREFIX = SPAN[:-len("_span")]
# the entry points rqb200_ar_sample_span replaced: the start_loc form, the guided form and the masked form
REMOVED = (PREFIX, SPAN + "_cfg", SPAN + "_keep")


@pytest.mark.parametrize("n", [2, 4, 8, 16])
def test_origin_is_tamings_rule_at_even_sizes(n):
    for nt in range(n, 3 * n + 1):
        for i in range(nt):
            assert WO.origin(i, n, nt) == WO.taming_origin(i, n, nt), (i, n, nt)


@pytest.mark.parametrize("n", [1, 3, 5, 7])
def test_origin_stays_in_bounds_at_odd_sizes(n):
    for nt in range(n, 3 * n + 1):
        for i in range(nt):
            o = WO.origin(i, n, nt)
            assert 0 <= o <= nt - n and o <= i < o + n, (i, n, nt)
            if n // 2 <= i <= nt - n + n // 2:
                assert i - o == n // 2            # away from the edges the token sits floor(n/2) cells into its window


def test_segment_counts():
    segs = WO.segments((8, 8), (16, 16))
    assert len(segs) == 144
    for row in range(16):
        assert sum(1 for _, pos in segs if pos[0] // 16 == row) == 9
    assert sum(len(p) for _, p in segs) == 256
    assert len(WO.segments((8, 8), (8, 8))) == 1                       # the grid: one segment, today's call
    assert len(WO.segments((8, 8), (8, 16))) == 8 * 9
    # outpainting the right half of 8 x 16: columns 8..11 each open a window, 12..15 share the last one
    sampled = [idx % 16 >= 8 for idx in range(8 * 16)]
    segs = WO.segments((8, 8), (8, 16), sampled)
    assert len(segs) == 8 * 5 and sum(len(p) for _, p in segs) == 64
    # tall canvas with the grid's width: whole rows share an origin while it does not move
    assert len(WO.segments((4, 4), (8, 4))) == 5
    # a resume: positions before start are not planned
    assert sum(len(p) for _, p in WO.segments((4, 4), (7, 9), start=2 * 9 + 3)) == 7 * 9 - 21


def test_segments_are_consecutive_in_their_window():
    """inside a segment the window positions increase (the KV cache continues), and every segment's positions lie in its window"""
    for grid, canvas in (((8, 8), (16, 16)), ((3, 3), (5, 7)), ((4, 4), (7, 9)), ((4, 4), (10, 10))):
        for (r0, c0), pos in WO.segments(grid, canvas):
            local = []
            for idx in pos:
                i, j = divmod(idx, canvas[1])
                rr, cc, li, lj = WO.window_of(i, j, grid, canvas)
                assert (rr, cc) == (r0, c0) and 0 <= li < grid[0] and 0 <= lj < grid[1]
                local.append(li * grid[1] + lj)
            assert local == sorted(local) and len(set(local)) == len(local)


def test_sample_span_takes_the_canvas_extents():
    """ABI 117: rqb200_ar_sample_span's last two arguments are canvas_h and canvas_w, still the one sampling entry point; the binding
    declares the arguments up to cfg_scale and the callers pass the extents after them as C int"""
    hdr = open(os.path.join(ROOT, "include", "rqb200.h")).read()
    assert re.search(r"int cfg_n, float cfg_scale, int canvas_h, int canvas_w\);", hdr)
    assert re.search(r"#define RQB200_CANVAS_MAX_CODES 2147483647LL", hdr)
    assert set(re.findall(r"\b(%s\w*)\s*\(" % PREFIX, hdr)) == {SPAN}
    so = C.CDLL(N.LIB_PATH)
    for name in REMOVED:
        assert not hasattr(so, name), name
    L = N.lib()
    assert getattr(L, SPAN).argtypes[-4:] == [C.c_void_p, C.c_void_p, C.c_int, C.c_float]
    assert L.rqb200_version() >= 117


def test_sample_span_refuses_bad_rows_and_canvases_before_any_cuda_call():
    """B must be 2 cfg_n rows when cfg_n > 0, cfg_n >= 0, and the canvas at least the grid and at most RQB200_CANVAS_MAX_CODES codes
    per row: refused with EINVAL before the device is looked at (no GPU here)"""
    torch.manual_seed(0)
    model = make_ar("tiny")
    cfg, w, keep, _ = model._engine_structs(torch.randn(model.vocab_size[0], 256), N.MODE_EXACT)
    L = N.lib()
    h = L.rqb200_ar_create(C.byref(cfg), C.byref(w))
    assert h, L.rqb200_last_error().decode()
    try:
        kk, pp = (C.c_int32 * 4)(*[512] * 4), (C.c_float * 4)(*[1.0] * 4)
        buf = C.create_string_buffer(64)

        def call(B, cfg_n, Ht=4, Wt=4, idx_end=16):
            return L.rqb200_ar_sample_span(h, buf, None, B, 0, idx_end, 0, 1.0, kk, pp, None, 0, None, None, buf, buf, 64, None, None,
                                           None, cfg_n, C.c_float(1.5), C.c_int(Ht), C.c_int(Wt))
        for B, cfg_n in ((0, 1), (1, 1), (3, 1), (4, 1), (2, -1)):
            assert call(B, cfg_n) == N.EINVAL, (B, cfg_n)
            assert B < 1 or "2n rows" in L.rqb200_last_error().decode(), (B, cfg_n)
        for Ht, Wt in ((3, 4), (4, 3), (0, 0), (2, 8)):
            assert call(1, 0, Ht, Wt) == N.EINVAL, (Ht, Wt)
            assert "at least the model's grid" in L.rqb200_last_error().decode()
        assert call(1, 0, 1 << 15, 1 << 14) == N.EINVAL                   # 2^29 positions x D = 4: 2^31 codes
        assert "RQB200_CANVAS_MAX_CODES" in L.rqb200_last_error().decode()
        assert call(1, 0, 4, 8, idx_end=33) == N.EINVAL                    # the span counts canvas positions
        assert "span" in L.rqb200_last_error().decode()
    finally:
        L.rqb200_ar_destroy(h)


def _forbid_native(monkeypatch):
    def boom(*a, **k):
        raise AssertionError("a native call was reached")
    monkeypatch.setattr(N, "lib", boom)


@pytest.mark.parametrize("name", ["tiny", "tiny_txt"])
def test_canvas_checks_come_before_any_native_call(name, monkeypatch):
    model = make_ar(name)
    H, W, D = model.block_size
    B = 2
    _forbid_native(monkeypatch)
    # smaller than the grid, or another D: AssertionError as before
    for shape in ((B, H - 1, W + 4, D), (B, H + 4, W - 1, D), (B, H + 1, W + 1, D + 1), (B, H + 1, W + 1, D - 1), (H, W, D)):
        with pytest.raises(AssertionError):
            model.sample(torch.zeros(shape, dtype=torch.long))
    # a keep_mask that broadcasts to the grid but not to the canvas
    part = torch.zeros(B, H + 2, W + 3, D, dtype=torch.long)
    for k in (torch.ones(H, W, D, dtype=torch.bool), torch.ones(B, H, W + 3, D, dtype=torch.bool), torch.ones(H + 2, W + 3, D),
              torch.ones(B + 1, H + 2, W + 3, D, dtype=torch.bool)):
        with pytest.raises(ValueError):
            model.sample(part, keep_mask=k)
    # past the engine's index range (a meta tensor: nothing is allocated)
    big = torch.empty(1, 1 << 15, 1 << 16, D, dtype=torch.long, device="meta")
    assert big.shape[1] * big.shape[2] * D > CANVAS_MAX_CODES
    with pytest.raises(ValueError, match="index range"):
        model.sample(big)


def test_keep_mask_is_laid_out_over_the_canvas():
    """a [Ht, Wt, 1] region broadcasts to [B, Ht, Wt, D]; the start_loc prefix (canvas coordinates) is kept"""
    model = make_ar("tiny")
    H, W, D = model.block_size
    keep = torch.zeros(6, 10, 1, dtype=torch.bool)
    keep[:, :5] = True
    k = model._keep_mask(keep, 3, (1, 2), canvas=(6, 10))
    assert k.shape == (3, 6, 10, D) and k.dtype == torch.uint8 and k.is_contiguous()
    want = keep.expand(3, 6, 10, D).clone()
    want.view(3, 60, D)[:, :12] = True
    assert torch.equal(k.bool(), want)
