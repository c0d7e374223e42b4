"""rqb200_ar_step on the host: the header, library and binding agree on it, its argument and sequence checks answer before any
CUDA call, and RQTransformer.cached_forward routes each call to the stateful native step or to the stateless evaluation."""
import ctypes as C
import os
import re

import pytest
import torch

from rqvae import _native as N
from tests.helpers import CodebookAux
from tests.test_host_cpu import make_ar

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_step_is_declared_exported_and_bound():
    hdr = open(os.path.join(ROOT, "include", "rqb200.h")).read()
    assert re.search(r"\bint rqb200_ar_step\s*\(", hdr)
    assert "rqb200_ar_step" in N.EXPORTS
    L = N.lib()
    assert hasattr(C.CDLL(N.LIB_PATH), "rqb200_ar_step")
    assert L.rqb200_ar_step.argtypes is not None and len(L.rqb200_ar_step.argtypes) == 13
    assert L.rqb200_version() >= 107


@pytest.fixture
def exact_engine():
    """an exact-tier handle over host tensors: its creation touches no device, and every call below is refused before one would"""
    torch.manual_seed(0)
    model = make_ar("tiny")
    cfg, w, keep, _ = model._engine_structs(torch.randn(model.vocab_size[0], 256), N.MODE_EXACT)
    L = N.lib()
    h = L.rqb200_ar_create(C.byref(cfg), C.byref(w))
    assert h, L.rqb200_last_error().decode()
    yield L, h, model.block_size
    L.rqb200_ar_destroy(h)


def _step(L, h, pos, restart, stride=4 * 4 * 4, B=2):
    xs = (C.c_int64 * (B * stride))()
    out = (C.c_float * 4)()
    ws = (C.c_uint8 * 256)()
    rc = L.rqb200_ar_step(h, xs, stride, None, B, pos[0], pos[1], pos[2], restart, out, ws, 256, None)
    return rc, L.rqb200_last_error().decode()


def test_step_refuses_bad_arguments_and_broken_sequences(exact_engine):
    L, h, (H, W, D) = exact_engine
    assert _step(L, None, (0, 0, 0), 1)[0] == N.EINVAL
    rc, msg = _step(L, h, (0, 0, 1), 1)
    assert rc == N.EINVAL and "d must be 0" in msg
    for pos in ((H, 0, 0), (0, W, 0), (0, 0, D), (-1, 0, 0), (0, -1, 0), (0, 0, -1)):
        rc, msg = _step(L, h, pos, 0)
        assert rc == N.EINVAL and "out of range" in msg, pos
    rc, msg = _step(L, h, (1, 1, 2), 0, stride=(1 * W + 1) * D + 1)      # reads (1*W+1)*D + 2 codes per row
    assert rc == N.EINVAL and "xs_batch_stride" in msg
    # no step has run on this handle: nothing to continue
    for pos in ((0, 0, 1), (0, 1, 0), (2, 3, 3)):
        rc, msg = _step(L, h, pos, 0)
        assert rc == N.ESTATE and "restart" in msg, pos


@pytest.mark.skipif(N.lib().rqb200_device_count() > 0, reason="a device is present: the call would run")
def test_step_without_a_device_is_enodev(exact_engine):
    L, h, _ = exact_engine
    assert _step(L, h, (0, 0, 0), 1)[0] == N.ENODEV


# ------------------------------------------------------------------------------------------------ cached_forward routing
class _Spy:
    """stands in for the native step and the stateless evaluation: records which one each cached_forward call reached"""

    def __init__(self, model):
        self.calls = []
        model._native_step = lambda route, xs, cb, cond, mode, loc: self.calls.append((route, loc)) or "step"
        model._stateless_cached_forward = lambda xs, aux, cond, amp, loc: self.calls.append(("stateless", loc)) or "stateless"

    def take(self):
        c, self.calls = self.calls, []
        return c


def test_cached_forward_routes_in_order_calls_to_the_step():
    torch.manual_seed(0)
    model = make_ar("tiny")
    H, W, D = model.block_size
    aux = CodebookAux(torch.randn(model.vocab_size[0], 256))
    spy = _Spy(model)
    xs = torch.zeros(3, H, W, D, dtype=torch.long)
    cond = torch.zeros(3, 1, dtype=torch.long)

    def cf(loc, x=xs, c=cond, amp=False, rows=None):
        return model.cached_forward(x[:, :loc[0] + 1] if rows is None else x[:, :rows], aux, c, amp, loc)

    def raster(h0, w0, d0, n):
        t0 = (h0 * W + w0) * D + d0
        return [((t // D) // W, (t // D) % W, t % D) for t in range(t0, t0 + n)]

    cf((0, 0, 0))                                                   # no init_cache(): stateless
    assert spy.take() == [("stateless", (0, 0, 0))]

    model.init_cache()
    locs = raster(0, 0, 0, 6)
    for loc in locs:
        assert cf(loc) == "step"
    assert spy.take() == [("restart", locs[0])] + [("continue", l) for l in locs[1:]]

    # another batch / cond tensor / tier in between: stateless, the sequence goes on
    cf((0, 1, 2), x=xs[:1], c=cond[:1])
    cf((0, 1, 2), c=cond.clone())
    cf((0, 1, 2), amp=True)
    cf((0, 1, 2))
    assert spy.take() == [("stateless", (0, 1, 2))] * 3 + [("continue", (0, 1, 2))]

    # a repeated token: stateless, and the sequence ends
    cf((0, 1, 2))
    cf((0, 1, 3))
    assert spy.take() == [("stateless", (0, 1, 2)), ("stateless", (0, 1, 3))]

    # a skipped token ends it too; init_cache() lets the next (h, w, 0) restart
    model.init_cache()
    cf((1, 2, 0))
    cf((1, 2, 1))
    cf((1, 2, 3))
    cf((1, 3, 0))
    model.init_cache()
    cf((1, 3, 0))
    cf((1, 3, 1))
    assert spy.take() == [("restart", (1, 2, 0)), ("continue", (1, 2, 1)), ("stateless", (1, 2, 3)), ("stateless", (1, 3, 0)),
                          ("restart", (1, 3, 0)), ("continue", (1, 3, 1))]

    # the first call after init_cache() must begin a position (d == 0); an out-of-range position never steps (nor ends a sequence)
    model.init_cache()
    cf((2, 1, 1))
    cf((2, 1, 2))
    model.init_cache()
    cf((0, 0, 0))
    cf((0, 0, D))
    cf((0, 0, 1))
    assert spy.take() == [("stateless", (2, 1, 1)), ("stateless", (2, 1, 2)), ("restart", (0, 0, 0)), ("stateless", (0, 0, D)),
                          ("continue", (0, 0, 1))]

    # xs without the codes a step reads: stateless (zero-padded), and the sequence ends
    model.init_cache()
    cf((2, 0, 0), rows=2)                                           # reads positions [0, 8): the two rows hold them
    cf((2, 0, 1), rows=2)                                           # reads position 8's first code: not in xs
    cf((2, 0, 2))
    assert spy.take() == [("restart", (2, 0, 0)), ("stateless", (2, 0, 1)), ("stateless", (2, 0, 2))]

    # new weights drop the sequence with the engines
    model.init_cache()
    cf((0, 0, 0))
    model.load_state_dict(model.state_dict())
    cf((0, 0, 1))
    assert spy.take() == [("restart", (0, 0, 0)), ("stateless", (0, 0, 1))]
