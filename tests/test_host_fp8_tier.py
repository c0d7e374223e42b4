"""FP8 (E4M3) tier of the fast AR engine, host side: the C ABI's weight format and scale fields against the ctypes binding, the
RQB200_FAST_DTYPE parsing, the quantisation identities the dequantised-model oracle relies on, and the engine structs an FP8 build
hands to rqb200_ar_create (no kernels are launched)."""
import os
import re

import pytest
import torch

from rqvae import _native as N
from tests import fp8_helpers as F
from tests.test_host_cpu import make_ar
from tests.test_oracle_variants import make_variant
from tests import variants_oracle as VO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header():
    return open(os.path.join(ROOT, "include", "rqb200.h")).read()


def _struct_fields(hdr, name):
    """field names of `typedef struct name { ... } name;` in declaration order"""
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), hdr, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    out = []
    for decl in body.split(";"):
        if decl.strip():
            out += [re.search(r"(\w+)\s*$", part).group(1) for part in decl.split(",")]
    return out


def test_header_weight_format_and_struct_layouts_match_the_binding():
    hdr = _header()
    assert int(re.search(r"#define RQB200_E4M3 (\d+)", hdr).group(1)) == N.E4M3 == 3
    assert {N.F32, N.BF16, N.F16, N.E4M3} == {0, 1, 2, 3}
    for cname, cls in (("rqb200_block_weights", N.BlockWeights), ("rqb200_ar_weights", N.ArWeights)):
        assert _struct_fields(hdr, cname) == [f[0] for f in cls._fields_], cname
    # the scale pointers trail both structs (a caller built against the older layout ends before them)
    assert [f[0] for f in N.BlockWeights._fields_][-4:] == ["sqkv", "sproj", "s1", "s2"]
    assert [f[0] for f in N.ArWeights._fields_][-4:] == ["s_in", "s_head", "s_cls", "s_ccls"]


@pytest.mark.parametrize("value,fmt,act", [(None, "fp16", torch.float16), ("fp16", "fp16", torch.float16), ("fp8", "fp8", torch.float16),
                                           ("FP8", "fp8", torch.float16), ("Fp8", "fp8", torch.float16), ("bf16", "bf16", torch.bfloat16),
                                           ("bfloat16", "bf16", torch.bfloat16), ("e4m3", "fp16", torch.float16),
                                           ("int8", "fp16", torch.float16)])
def test_fast_dtype_env_parsing(monkeypatch, value, fmt, act):
    if value is None:
        monkeypatch.delenv("RQB200_FAST_DTYPE", raising=False)
    else:
        monkeypatch.setenv("RQB200_FAST_DTYPE", value)
    assert N.fast_weight_format() == fmt
    assert N.fast_dtype() == act              # the activation format: fp8 weights keep fp16 activations


def test_quantising_concatenated_qkv_rows_equals_per_matrix_quantisation():
    g = torch.Generator().manual_seed(3)
    E = 256
    mats = [torch.randn(E, E, generator=g) * sc for sc in (0.02, 1.0, 7.0)]
    mats[1][5] = 0.0                                                   # an all-zero row keeps s = 1 in either form
    q, s = N.quantize_fp8_rows(torch.cat(mats, 0))
    parts = [N.quantize_fp8_rows(m) for m in mats]
    assert torch.equal(q.view(torch.uint8), torch.cat([p[0] for p in parts]).view(torch.uint8))
    assert torch.equal(s, torch.cat([p[1] for p in parts]))
    # and the packed stream of the concatenation is the row-tile concatenation of the packed parts (3E rows, E % 128 == 0)
    packed, s2 = N.pack_fp8_weight(torch.cat(mats, 0))
    assert torch.equal(packed, torch.cat([N.pack_fp8_tiles(p[0]) for p in parts])) and torch.equal(s2, s)


def test_per_depth_classifier_slices_unpack_to_each_depths_quantisation():
    g = torch.Generator().manual_seed(4)
    D, E, V = 3, 128, 256
    weight = torch.randn(D, E, V, generator=g) / E ** 0.5                # BatchLinear layout: [D, in, out]
    weight[1] *= 50.0
    packed, s = N.pack_fp8_weight(weight.transpose(1, 2))
    assert packed.numel() == D * V * E and s.shape == (D, V)
    for d in range(D):
        q, sd = N.quantize_fp8_rows(weight[d].t())
        got = N.unpack_fp8_tiles(packed[d * V * E:(d + 1) * V * E], V, E)
        assert torch.equal(got.view(torch.uint8), q.view(torch.uint8)), d
        assert torch.equal(s[d], sd), d


def _structs(model, codebook, mode, fmt, monkeypatch):
    monkeypatch.setenv("RQB200_FAST_DTYPE", fmt)
    return model._engine_structs(codebook, mode)


def _blocks(w, n_body, n_head):
    return [w.body[i] for i in range(n_body)] + [w.head[i] for i in range(n_head)]


@pytest.mark.parametrize("name", ["tiny", "tiny_txt"])
def test_fp8_engine_structs_hold_packed_weights_and_scales_only(monkeypatch, name):
    """an FP8 build keeps the packed E4M3 streams and their fp32 scales -- sum of N*K + 4N bytes -- and no 16-bit copy; every
    present weight has its scale pointer, and every packed stream is 16-byte aligned"""
    torch.manual_seed(0)
    model = make_ar(name)
    cb = torch.randn(model.vocab_size[0], 256)
    cfg, w, keep, streamed = _structs(model, cb, N.MODE_FAST, "fp8", monkeypatch)
    assert cfg.weight_dtype == N.E4M3
    assert {t.dtype for t in keep if isinstance(t, torch.Tensor)} == {torch.float32, torch.uint8}
    assert sum(t.numel() * t.element_size() for t in streamed) == F.packed_bytes(model)
    nb, nh = cfg.n_body, cfg.n_head_layers
    for b in _blocks(w, nb, nh):
        for q, s in ((b.wqkv, b.sqkv), (b.wproj, b.sproj), (b.w1, b.s1), (b.w2, b.s2)):
            assert q and s and q % 16 == 0
    for q, s in ((w.w_in, w.s_in), (w.w_head, w.s_head), (w.w_cls, w.s_cls)):
        assert q and s and q % 16 == 0
    assert bool(w.w_ccls) == bool(w.s_ccls) == (model.block_size_cond > 1)


def test_per_depth_classifier_engine_struct(monkeypatch):
    model = make_variant(VO.TINY, VO.ALL_FALSE)
    cfg, w, keep, streamed = _structs(model, None, N.MODE_FAST, "fp8", monkeypatch)
    D, V, E = VO.TINY[5][2], VO.TINY[4], VO.TINY[0]
    scales = [t for t in streamed if t.data_ptr() == w.s_cls][0]
    packed = [t for t in streamed if t.data_ptr() == w.w_cls][0]
    assert scales.shape == (D, V) and packed.numel() == D * V * E
    assert not w.w_in and not w.s_in and not w.w_head and not w.s_head     # own token tables: no input / head MLP


def test_16bit_and_exact_builds_leave_the_scales_unset(monkeypatch):
    torch.manual_seed(0)
    model = make_ar("tiny")
    cb = torch.randn(512, 256)
    for mode, fmt, want in ((N.MODE_FAST, "fp16", N.F16), (N.MODE_FAST, "bf16", N.BF16), (N.MODE_EXACT, "fp8", N.F32)):
        cfg, w, keep, _ = _structs(model, cb, mode, fmt, monkeypatch)
        assert cfg.weight_dtype == want, (mode, fmt)                     # the exact tier ignores RQB200_FAST_DTYPE
        assert not any(getattr(b, f) for b in _blocks(w, cfg.n_body, cfg.n_head_layers) for f in ("sqkv", "sproj", "s1", "s2"))
        assert not (w.s_in or w.s_head or w.s_cls or w.s_ccls)
        assert torch.uint8 not in {t.dtype for t in keep if isinstance(t, torch.Tensor)}
