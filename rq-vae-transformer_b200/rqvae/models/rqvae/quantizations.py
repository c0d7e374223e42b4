"""Residual quantiser -- host-side mirror of rqvae/models/rqvae/quantizations.py (VQEmbedding :24, RQBottleneck :149).

Parameters / buffers keep the reference's names and shapes (``codebooks.{i}.weight`` [K+1, C] with a zero padding row,
``cluster_size_ema``, ``embed_ema``) so checkpoints load unchanged; the numeric work is done by
``rqb200_rq_quantize`` / ``rqb200_rq_embed_sum`` / ``rqb200_rq_embed_depth`` (csrc/rq_search.cu), or their ``*_depthwise``
forms when every depth has its own codebook (``shared_codebook=False``)."""
from typing import Iterable

import numpy as np
import torch
from torch import nn

from .. import _bind as nb


class VQEmbedding(nn.Embedding):
    """codebook holder (quantizations.py:24-41).  EMA training updates (:80-129) are out of scope."""

    def __init__(self, n_embed, embed_dim, ema=True, decay=0.99, restart_unused_codes=True, eps=1e-5):
        super().__init__(n_embed + 1, embed_dim, padding_idx=n_embed)
        self.ema, self.decay, self.eps = ema, decay, eps
        self.restart_unused_codes = restart_unused_codes
        self.n_embed = n_embed
        if ema:
            for p in self.parameters():
                p.requires_grad_(False)
            self.register_buffer("cluster_size_ema", torch.zeros(n_embed))
            self.register_buffer("embed_ema", self.weight[:-1, :].detach().clone())

    def codebook(self):
        """[K, C] view without the padding row (quantizations.py:45)"""
        return self.weight[:-1, :]

    @torch.no_grad()
    def find_nearest_embedding(self, inputs):
        """quantizations.py:64-69 -- one-depth search through the fused kernel"""
        _, codes = nb.rq_quantize(inputs.reshape(-1, inputs.shape[-1]), self.codebook(), 1)
        return codes.reshape(inputs.shape[:-1])

    @torch.no_grad()
    def embed(self, idxs):
        """quantizations.py:144-146"""
        flat = idxs.reshape(-1, 1)
        out = nb.rq_embed(flat, self.codebook(), summed=True)
        return out.reshape(*idxs.shape, -1)

    def forward(self, inputs):
        if self.training:
            raise NotImplementedError("rqb200: EMA codebook training is out of scope; call .eval()")
        idx = self.find_nearest_embedding(inputs)
        return self.embed(idx), idx


class RQBottleneck(nn.Module):
    """quantizations.py:149-214 (constructor semantics incl. the shared-codebook aliasing :199-205)"""

    def __init__(self, latent_shape, code_shape, n_embed, decay=0.99, shared_codebook=False, restart_unused_codes=True,
                 commitment_loss="cumsum"):
        super().__init__()
        if not len(code_shape) == len(latent_shape) == 3:
            raise ValueError("incompatible code shape or latent shape")
        if any(y % x != 0 for x, y in zip(code_shape[:2], latent_shape[:2])):
            raise ValueError("incompatible code shape or latent shape")
        embed_dim = int(np.prod(latent_shape[:2]) // np.prod(code_shape[:2]) * latent_shape[2])
        self.latent_shape = torch.Size(latent_shape)
        self.code_shape = torch.Size(code_shape)
        self.shape_divisor = torch.Size([latent_shape[i] // code_shape[i] for i in range(3)])
        self.shared_codebook = shared_codebook
        if shared_codebook and (isinstance(n_embed, Iterable) or isinstance(decay, Iterable)):
            raise ValueError("Shared codebooks are incompatible with list types of momentums or sizes: Change it into int")
        depth = self.code_shape[-1]
        self.restart_unused_codes = restart_unused_codes
        self.n_embed = list(n_embed) if isinstance(n_embed, Iterable) else [n_embed] * depth
        self.decay = list(decay) if isinstance(decay, Iterable) else [decay] * depth
        assert len(self.n_embed) == depth and len(self.decay) == depth
        if shared_codebook:
            one = VQEmbedding(self.n_embed[0], embed_dim, decay=self.decay[0], restart_unused_codes=restart_unused_codes)
            self.codebooks = nn.ModuleList([one] * depth)
        else:
            self.codebooks = nn.ModuleList([
                VQEmbedding(self.n_embed[i], embed_dim, decay=self.decay[i], restart_unused_codes=restart_unused_codes)
                for i in range(depth)])
        self.commitment_loss = commitment_loss

    # -- identity reshapes whenever rH = rW = 1 (every shipped config); general form kept (quantizations.py:216-235)
    def to_code_shape(self, x):
        B, H, W, D = x.shape
        rH, rW, _ = self.shape_divisor
        x = x.reshape(B, H // rH, rH, W // rW, rW, D).permute(0, 1, 3, 2, 4, 5)
        return x.reshape(B, H // rH, W // rW, -1)

    def to_latent_shape(self, x):
        B, h, w, _ = x.shape
        _, _, D = self.latent_shape
        rH, rW, _ = self.shape_divisor
        x = x.reshape(B, h, w, rH, rW, D).permute(0, 1, 3, 2, 4, 5)
        return x.reshape(B, h * rH, w * rW, D)

    def _shared_table(self):
        if not self.shared_codebook:
            raise ValueError("rqb200: this quantizer has one codebook per depth (use _tables())")
        return self.codebooks[0].codebook()

    def _tables(self):
        """what the kernels search and embed with: the one [K,C] table of a shared codebook, else the list of the D per-depth
        [K_d,C] tables (views of codebooks[d].weight without the padding row; no copies)"""
        if self.shared_codebook:
            return self.codebooks[0].codebook()
        return [cb.codebook() for cb in self.codebooks]

    @torch.no_grad()
    def quantize(self, x):
        """quantizations.py:237-271.  x [B,h,w,C] -> (list of D cumulative aggregates [B,h,w,C], codes [B,h,w,D] int64)."""
        B, h, w, C = x.shape
        depth = self.code_shape[-1]
        quants, codes = nb.rq_quantize(x.reshape(-1, C), self._tables(), depth)
        return [quants[i].reshape(B, h, w, C) for i in range(depth)], codes.reshape(B, h, w, depth)

    def forward(self, x):
        x_r = self.to_code_shape(x)
        quant_list, codes = self.quantize(x_r)
        loss = self.compute_commitment_loss(x_r, quant_list)
        q = self.to_latent_shape(quant_list[-1])
        q = x + (q - x).detach()                       # straight-through form, quantizations.py:279
        return q, loss, codes

    def compute_commitment_loss(self, x, quant_list):
        """quantizations.py:283-295 (torch elementwise glue on tiny tensors; not on the sampling path)"""
        return torch.mean(torch.stack([(x - q.detach()).pow(2.0).mean() for q in quant_list]))

    @torch.no_grad()
    def get_soft_codes(self, x, temp=1.0, stochastic=False):
        """quantizations.py:371-399: per depth softmax(-distances/temp) over the codebook ([B,h,w,D,K]) and the codes taken along
        the way -- argmin (then identical to ``quantize``) or, stochastic, one multinomial draw per vector from the soft code."""
        x = self.to_code_shape(x)
        B, h, w, C = x.shape
        depth = self.code_shape[-1]
        tabs = self._tables()
        cb = tabs if isinstance(tabs, list) else [tabs] * depth      # table of depth d
        if len({t.shape[0] for t in cb}) != 1:
            raise ValueError("get_soft_codes: the per-depth codebooks must have equal sizes (the soft codes are stacked)")
        flat = x.reshape(-1, C).float().contiguous()
        softs, codes = [], []
        if not stochastic:
            ql, code = nb.rq_quantize(flat, tabs, depth)
            for d in range(depth):
                softs.append(nb.rq_soft(flat if d == 0 else flat - ql[d - 1], cb[d], temp))
            codes = code
        else:
            res = flat.clone()
            for d in range(depth):
                soft, logits = nb.rq_soft(res, cb[d], temp, want_logits=True)
                q = torch.empty_like(soft).exponential_(1)        # the draw torch.multinomial(soft, 1) makes
                idx = nb.sample_logits(logits, 1.0, None, None, q=q)
                res = res - nb.rq_embed(idx.reshape(-1, 1), cb[d], summed=True)
                softs.append(soft)
                codes.append(idx.unsqueeze(-1))
            codes = torch.cat(codes, -1)
        soft = torch.stack(softs, dim=1).reshape(B, h, w, depth, -1)
        return soft, codes.reshape(B, h, w, depth)

    @torch.no_grad()
    def embed_code(self, code):
        """quantizations.py:297-311"""
        assert code.shape[1:] == self.code_shape
        out = nb.rq_embed(code.reshape(-1, code.shape[-1]), self._tables(), summed=True)
        return self.to_latent_shape(out.reshape(*code.shape[:-1], -1))

    @torch.no_grad()
    def embed_code_with_depth(self, code, to_latent_shape=False):
        """quantizations.py:313-334 -> ([..., D, C], None)"""
        assert code.shape[-1] == self.code_shape[-1]
        out = nb.rq_embed(code.reshape(-1, code.shape[-1]), self._tables(), summed=False)
        out = out.reshape(*code.shape, -1)
        if to_latent_shape:
            out = torch.stack([self.to_latent_shape(out[..., d, :]) for d in range(code.shape[-1])], dim=-2)
        return out, None

    @torch.no_grad()
    def embed_partial_code(self, code, code_idx, decode_type="select"):
        """quantizations.py:336-369"""
        assert code.shape[1:] == self.code_shape and code_idx < code.shape[-1]
        tabs = self._tables()
        if decode_type == "select":
            sub = code[..., code_idx:code_idx + 1]
            if isinstance(tabs, list):
                tabs = tabs[code_idx:code_idx + 1]
        elif decode_type == "add":
            sub = code[..., :code_idx + 1]
            if isinstance(tabs, list):
                tabs = tabs[:code_idx + 1]
        else:
            raise NotImplementedError(f"{decode_type} is not implemented in partial decoding")
        out = nb.rq_embed(sub.reshape(-1, sub.shape[-1]).contiguous(), tabs, summed=True)
        return self.to_latent_shape(out.reshape(*code.shape[:-1], -1))
