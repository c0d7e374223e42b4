"""FP8 (E4M3) tier helpers: the dequantised model the FP8 tier is checked against, and the byte count of its packed weights."""
import torch
import torch.nn as nn

from rqvae import _native as N
from rqvae.models.rqtransformer.primitives import BatchLinear


def streamed_weights(model):
    """every weight the fast tier streams, as [N,K] (nn.Linear) or [D,N,K] views (BatchLinear: depth d's [E,V] transposed); the rest
    of the model (embeddings, positional tables, LayerNorms, biases) stays fp32 in every tier"""
    out = []
    for name, m in model.named_modules():
        if isinstance(m, nn.Linear):
            out.append((name, m.weight))
        elif isinstance(m, BatchLinear):
            out.append((name, m.weight.transpose(1, 2)))
    return out


def dequantise_(w):
    """w <- q * s in place, with (q, s) = quantize_fp8_rows of each [N,K] row block ([D,N,K]: of each depth's)"""
    for wd in (w if w.dim() == 3 else [w]):
        q, s = N.quantize_fp8_rows(wd)
        wd.copy_(q.float() * s[:, None])


@torch.no_grad()
def dequantised_copy(model):
    """a new model with the weights of `model`, every streamed weight replaced by the fp32 values q * s the FP8 tier computes with.
    A separate copy: the memoised test models must keep their own weights.  Free it when done (3.9 B parameters are 15.6 GB)."""
    with torch.device("meta"):
        m = type(model)(model.config)
    m = m.to_empty(device=model.pos_emb_hw.device)
    m.load_state_dict(model.state_dict())
    for _, w in streamed_weights(m):
        dequantise_(w)
    return m.eval()


def packed_bytes(model):
    """sum of N*K + 4*N over the streamed weights: the E4M3 values and one fp32 scale per output row (the cond classifier's rows
    padded to a multiple of 128)"""
    total = 0
    for name, w in streamed_weights(model):
        n, k = w.shape[-2:]
        if name == "cond_classifier.linear":
            n = -(-n // 128) * 128
        total +=(w.shape[0] if w.dim() == 3 else 1) * (n * k + 4 * n)
    return total
