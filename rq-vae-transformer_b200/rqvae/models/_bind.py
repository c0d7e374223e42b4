"""Thin tensor-level wrappers over the C ABI (pointers + sizes in, freshly allocated torch tensors out)."""
import ctypes

import torch

from .. import _native as N


def _prep(t, dtype):
    N.require_cuda(t)
    if t.dtype != dtype:
        t = t.to(dtype)
    return t.contiguous()


def tables(codebooks):
    """a list of D [K_d,C] tables -> (the f32 contiguous tables, host pointer array, host K array) for the *_depthwise entries"""
    tabs = [_prep(t, torch.float32) for t in codebooks]
    ptrs = (ctypes.c_void_p * len(tabs))(*[t.data_ptr() for t in tabs])
    ks = (ctypes.c_int32 * len(tabs))(*[t.shape[0] for t in tabs])
    return tabs, ptrs, ks


def rq_quantize(x, codebook, depth, want_list=True):
    """x [n,C], codebook [K,C] (shared by every depth) or a list of D tables [K_d,C] (table d at depth d)
    -> (quant_list [D,n,C] or None, codes [n,D] int64)"""
    x = _prep(x, torch.float32)
    n, C = x.shape
    codes = torch.empty(n, depth, dtype=torch.int64, device=x.device)
    ql = torch.empty(depth, n, C, dtype=torch.float32, device=x.device) if want_list else None
    with torch.cuda.device(x.device):
        if isinstance(codebook, (list, tuple)):
            if len(codebook) != depth:
                raise ValueError("rq_quantize: %d codebooks for depth %d" % (len(codebook), depth))
            _tabs, ptrs, ks = tables(codebook)
            rc = N.lib().rqb200_rq_quantize_depthwise(N.ptr(x), ptrs, ks, n, C, depth, N.ptr(codes), N.ptr(ql), None,
                                                      N.stream_ptr(x.device))
        else:
            cb = _prep(codebook, torch.float32)
            rc = N.lib().rqb200_rq_quantize(N.ptr(x), N.ptr(cb), n, cb.shape[0], C, depth, N.ptr(codes), N.ptr(ql), None,
                                            N.stream_ptr(x.device))
        N.check(rc, "rq_quantize")
    N.launch_count["total"] += 1 if n else 0
    return ql, codes


def rq_embed(codes, codebook, summed):
    """codes [n,D] int64 -> [n,C] (summed over depth) or [n,D,C]; codebook [K,C] or a list of D tables (code d from table d)"""
    codes = _prep(codes, torch.int64)
    n, D = codes.shape
    L = N.lib()
    with torch.cuda.device(codes.device):
        if isinstance(codebook, (list, tuple)):
            if len(codebook) != D:
                raise ValueError("rq_embed: %d codebooks for %d codes per vector" % (len(codebook), D))
            _tabs, ptrs, ks = tables(codebook)
            C = _tabs[0].shape[1]
            out = torch.empty((n, C) if summed else (n, D, C), dtype=torch.float32, device=codes.device)
            fn = L.rqb200_rq_embed_sum_depthwise if summed else L.rqb200_rq_embed_depth_depthwise
            rc = fn(N.ptr(codes), ptrs, ks, n, D, C, N.ptr(out), N.stream_ptr(codes.device))
        else:
            cb = _prep(codebook, torch.float32)
            K, C = cb.shape
            out = torch.empty((n, C) if summed else (n, D, C), dtype=torch.float32, device=codes.device)
            fn = L.rqb200_rq_embed_sum if summed else L.rqb200_rq_embed_depth
            rc = fn(N.ptr(codes), N.ptr(cb), n, D, K, C, N.ptr(out), N.stream_ptr(codes.device))
        N.check(rc, "rq_embed")
    N.launch_count["total"] += 1 if n else 0
    return out


def sample_logits(logits, temperature=1.0, top_k=None, top_p=None, q=None):
    logits = _prep(logits, torch.float32)
    B, V = logits.shape
    if q is not None:
        q = _prep(q, torch.float32)
    out = torch.empty(B, dtype=torch.int64, device=logits.device)
    k = 0 if top_k is None else int(top_k)
    p = 1.0 if top_p is None else float(top_p)
    with torch.cuda.device(logits.device):
        N.check(N.lib().rqb200_sample_logits(N.ptr(logits), N.ptr(q), B, V, float(temperature), k, p, N.ptr(out),
                                             N.stream_ptr(logits.device)), "sample_logits")
    N.launch_count["total"] += 1
    return out


def rq_soft(residual, codebook, temp=1.0, want_logits=False):
    """residual [n,C] -> softmax(-distances / temp) [n,K] (and optionally the logits -d/temp)"""
    r = _prep(residual, torch.float32)
    cb = _prep(codebook, torch.float32)
    n, C = r.shape
    K = cb.shape[0]
    soft = torch.empty(n, K, dtype=torch.float32, device=r.device)
    logits = torch.empty(n, K, dtype=torch.float32, device=r.device) if want_logits else None
    with torch.cuda.device(r.device):
        N.check(N.lib().rqb200_rq_soft_codes(N.ptr(r), N.ptr(cb), n, K, C, float(temp), N.ptr(soft), N.ptr(logits),
                                             N.stream_ptr(r.device)), "rq_soft_codes")
    N.launch_count["total"] += 1 if n else 0
    return (soft, logits) if want_logits else soft
