"""TEST INFRASTRUCTURE ONLY -- the oracle's residual quantisation, code embeddings, decode and teacher-forced AR forward for an
RQBottleneck with one codebook per depth (shared_codebook=False): depth d searches, subtracts and embeds with tables[d]
(reference: rqvae/models/rqvae/quantizations.py:237-271, 297-399).  Built on oracle/rq_oracle.py's primitives; the shared
case stays there.  Pinned to the reference by tests/golden/rqd.pt (scripts/gen_golden_depthwise.py)."""
from itertools import product

import torch
import torch.nn.functional as F

from oracle import rq_oracle as O
from oracle import synth


def rq_quantize(x, tables):
    """x [..., C] -> (list of D cumulative aggregates, codes [..., D] int64); the reference's update order"""
    residual = x.detach().clone()
    agg = torch.zeros_like(x)
    quants, codes = [], []
    for cb in tables:
        idx = O.vq_distances(residual, cb).argmin(dim=-1)
        q = F.embedding(idx, cb)
        residual.sub_(q)
        agg.add_(q)
        quants.append(agg.clone())
        codes.append(idx.unsqueeze(-1))
    return quants, torch.cat(codes, dim=-1)


def rq_soft_codes(x, tables, temp=1.0):
    """get_soft_codes(stochastic=False): [..., D, K] soft codes (equal K) and the argmin codes"""
    residual = x.detach().clone()
    softs, codes = [], []
    for cb in tables:
        d = O.vq_distances(residual, cb)
        softs.append(F.softmax(-d / temp, dim=-1).unsqueeze(-2))
        idx = d.argmin(dim=-1)
        residual.sub_(F.embedding(idx, cb))
        codes.append(idx.unsqueeze(-1))
    return torch.cat(softs, dim=-2), torch.cat(codes, dim=-1)


def embed_code_with_depth(codes, tables):
    parts = [F.embedding(c, tables[i]) for i, c in enumerate(torch.chunk(codes, codes.shape[-1], dim=-1))]
    return torch.cat(parts, dim=-2)


def embed_code(codes, tables):
    return embed_code_with_depth(codes, tables).sum(-2)


def embed_partial_code(codes, tables, code_idx, decode_type):
    emb = embed_code_with_depth(codes, tables)
    if decode_type == "select":
        return emb[..., code_idx, :]
    return emb[..., :code_idx + 1, :].sum(-2)


def vae_decode_code(sd, dd, codes, tables):
    return O.vae_decode(sd, dd, embed_code(codes, tables))


def _stacked(xs, tables):
    """per-depth tables of one size K as one [D*K, C] table: code d of xs indexes rows d*K.., so the shared-table oracle computes
    exactly the per-depth embeddings"""
    offs = torch.arange(len(tables), dtype=xs.dtype) * tables[0].shape[0]
    return xs + offs, torch.cat(tables, 0)


def ar_sample(sd, cfg, partial_sample, tables, cond=None, start_loc=(0, 0), temperature=1.0, top_k=None, top_p=None, noise=None,
              logits_hook=None):
    """oracle/rq_oracle.py's ar_sample (transformers.py:294-369) with model_aux embedding code d from tables[d]; ``noise`` is a
    callable noise(step, B, V) -> q"""
    H, W, D = cfg.block_size
    ks = O._per_depth(top_k, cfg.V, D, cfg.V)
    ps = O._per_depth(top_p, 1.0, D, 1.0)
    xs = partial_sample.clone()
    state = O.new_state(cfg)
    step = 0
    for (h, w, d) in product(range(H), range(W), range(D)):
        if (h, w) < (start_loc[0], start_loc[1]):
            continue
        xo, table = _stacked(xs[:, :h + 1], tables)
        logits = O.ar_cached_forward(sd, cfg, state, xo, table, cond, (h, w, d))
        if logits_hook is not None:
            logits_hook(step, (h, w, d), logits)
        xs[:, h, w, d] = O.sample_from_logits(logits, temperature, ks[d], ps[d], q=noise(step, logits.shape[0], logits.shape[1]))
        step += 1
    return xs


def ar_forward(sd, cfg, xs, tables, cond=None):
    """teacher-forced logits [B,H,W,D,V] with code d embedded from tables[d]"""
    xo, table = _stacked(xs, tables)
    return O.ar_forward(sd, cfg, xo, table, cond)


def tables_of(sizes, seed):
    """the seeded per-depth tables of the fixture: table d = randn(K_d, 256) from seed + d"""
    return [synth.randn_seeded((k, 256), seed + d) for d, k in enumerate(sizes)]


def depthwise_vae_state(shapes, seed, table_seed):
    """synth.synth_state_dict with every depth's codebook its own seeded table (synth aliases them into one)"""
    sd = synth.synth_state_dict(shapes, seed)
    D = sum(1 for k in shapes if k.startswith("quantizer.codebooks.") and k.endswith(".weight"))
    K = shapes["quantizer.codebooks.0.weight"][0] - 1
    for d, t in enumerate(tables_of([K] * D, table_seed)):
        sd["quantizer.codebooks.%d.weight" % d] = torch.cat([t, torch.zeros(1, t.shape[1])], 0)
        sd["quantizer.codebooks.%d.embed_ema" % d] = t.clone()
    return sd


# RQ runs of the fixture -- name: (K per depth, B, table seed, input seed, tie case); codes maps are 8x8xD
RQ_CASES = {
    "k2048": ([2048] * 4, 2, 100, 200, False),
    "k16384_b64": ([16384] * 4, 64, 110, 210, False),
    "unequal": ([512, 1000, 2048, 300], 2, 120, 220, False),
    "ties": ([512] * 4, 2, 130, 230, True),
}


def rq_inputs(name):
    """(tables, x [B,8,8,256]) of one case, regenerated from its seeds"""
    ks, B, ts, xs, tie = RQ_CASES[name]
    tables = tables_of(ks, ts)
    x = synth.randn_seeded((B, 8, 8, 256), xs)
    if tie:
        tables[2][256:] = tables[2][:256]          # every table-2 argmin is a tie: the first index must win
        x[0, 0, 0] = tables[0][5]                  # distance exactly 0 to row 5 of table 0
    return tables, x


# AR trajectories of the fixture: a tiny transformer over per-depth tables -- (E, heads, n_body, n_head_layers, V, block_size,
# vocab_cond, cond_len), the AR_ZOO tuple layout of oracle/zoo.py
AR_SHAPE = (128, 2, 2, 2, 512, (8, 8, 4), 16, 4)
AR_PLAN = dict(B=2, weight_seed=31, table_seed=400, cond_seed=32, settings=[dict(top_k=1), dict(top_k=100, top_p=0.95)],
               noise_seeds=[600, 601], resume=dict(start_loc=(4, 1), noise_seed=902))
