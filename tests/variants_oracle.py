"""TEST INFRASTRUCTURE ONLY -- the oracle's cached AR step, sampling loop and teacher-forced forward for every combination of the
RQ-Transformer's five embedding / classifier switches (reference: rqvae/models/rqtransformer/transformers.py:63-105, 113-287;
primitives.py): input_emb_vqvae, head_emb_vqvae, cumsum_depth_ctx, shared_tok_emb, shared_cls_emb.  Built on oracle/rq_oracle.py's
primitives; the shipped family (all five true) stays there.  Pinned to the reference by tests/golden/arv.pt
(scripts/gen_golden_variants.py)."""
from itertools import product

import torch
import torch.nn.functional as F

from oracle import rq_oracle as O

FLAG_NAMES = ("input_emb_vqvae", "head_emb_vqvae", "cumsum_depth_ctx", "shared_tok_emb", "shared_cls_emb")
COMBOS = [dict(zip(FLAG_NAMES, bits)) for bits in product((False, True), repeat=5)]


def combo_name(flags):
    return "".join("1" if flags[n] else "0" for n in FLAG_NAMES)


def _tok(sd, xs):
    """tok_emb(xs) [..., D, E]: nn.Embedding (shared) or TupleEmbedding (rows offsets[d] + code)"""
    off = sd.get("tok_emb.offsets")
    return F.embedding(xs if off is None else xs + off, sd["tok_emb.weight"])


def _body_emb(sd, flags, xs, codebook):
    if flags["input_emb_vqvae"]:
        return O._linear(sd, "input_mlp", O.embed_code_with_depth(xs, codebook))          # :219-220
    return _tok(sd, xs)                                                                    # :222


def _head_emb(sd, flags, xs, codebook):
    if flags["head_emb_vqvae"]:
        e = O.embed_code_with_depth(xs, codebook)
        if flags["cumsum_depth_ctx"]:
            e = torch.cumsum(e, dim=-2)
        return O._linear(sd, "head_mlp", e)                                                # :250-255
    return _tok(sd, xs)                                                                    # :257


def _classify(sd, flags, x, depths):
    """x [N, n, E] -> logits [N, n, V]; depth of slot i = depths[i] (BatchLinear's einsum, :278-283 / :183)"""
    x = O._layer_norm(sd, "classifier.layer_norm", x)
    if flags["shared_cls_emb"]:
        return O._linear(sd, "classifier.linear", x)
    w, b = sd["classifier.linear.weight"], sd["classifier.linear.bias"]
    if len(depths) != w.shape[0]:
        w, b = w[depths], b[depths]
    return torch.einsum("bij,ijk->bik", x.view(-1, x.shape[-2], x.shape[-1]), w) + b.unsqueeze(0)


def ar_cached_forward(sd, cfg, flags, state, xs, codebook, cond, loc):
    """transformers.py:190-287 for any flag combination; ``codebook`` may be None when no code goes through it"""
    h, w, d = loc
    B, H, W, D = xs.shape
    idx = h * W + w
    xs = xs.clone().reshape(B, -1, D)[:, :idx + 1]
    cond = torch.zeros(B, cfg.cond_len, dtype=torch.long) if cond is None else cond.reshape(B, cfg.cond_len)
    seq_len, cond_len = xs.shape[1], cond.shape[1]
    if d == 0:
        emb = _body_emb(sd, flags, xs, codebook)
        c_emb = F.embedding(cond, sd["cond_emb.weight"]) + sd["pos_emb_cond"][:, :cond_len, :]
        emb = emb.sum(dim=-2) + sd["pos_emb_hw"][:, :seq_len, :]
        lat = torch.cat([c_emb, emb[:, :-1, :]], dim=1)[:, :cond_len + idx, :]
        if state["ctx"] is None:
            out = O.stack(sd, "body_transformer", lat, cfg.n_body, cfg.nh, state["body"])
            ctx = out[:, -1, :].unsqueeze(1)
        else:
            ctx = O.stack(sd, "body_transformer", lat[:, -1, :].unsqueeze(1), cfg.n_body, cfg.nh, state["body"])
        state["ctx"] = ctx
    ctx = state["ctx"]
    dctx = _head_emb(sd, flags, xs, codebook)[:, idx, :]
    full = torch.cat([ctx.view(B, 1, -1), dctx[:, :-1, :]], dim=-2) + sd["pos_emb_d"][:, :D, :]
    tok = full[:, d, :].unsqueeze(1)
    if d == 0:
        state["head"] = [[None] for _ in range(cfg.n_headl)]
    out = O.stack(sd, "head_transformer", tok, cfg.n_headl, cfg.nh, state["head"])
    return _classify(sd, flags, out, [d]).reshape(B, -1)


def ar_sample(sd, cfg, flags, partial_sample, codebook, cond=None, start_loc=(0, 0), temperature=1.0, top_k=None, top_p=None,
              noise=None, logits_hook=None):
    """transformers.py:294-369; ``noise`` is a callable noise(step, B, V) -> q"""
    H, W, D = cfg.block_size
    ks = O._per_depth(top_k, cfg.V, D, cfg.V)
    ps = O._per_depth(top_p, 1.0, D, 1.0)
    xs = partial_sample.clone()
    state = O.new_state(cfg)
    step = 0
    for (h, w, d) in product(range(H), range(W), range(D)):
        if (h, w) < (start_loc[0], start_loc[1]):
            continue
        logits = ar_cached_forward(sd, cfg, flags, state, xs[:, :h + 1], codebook, cond, (h, w, d))
        if logits_hook is not None:
            logits_hook(step, (h, w, d), logits)
        xs[:, h, w, d] = O.sample_from_logits(logits, temperature, ks[d], ps[d], q=noise(step, logits.shape[0], logits.shape[1]))
        step += 1
    return xs


def ar_forward(sd, cfg, flags, xs, codebook, cond=None, with_cond_logits=False):
    """transformers.py:113-188 for any flag combination"""
    B, H, W, D = xs.shape
    xs = xs.reshape(B, H * W, D)
    cond = torch.zeros(B, cfg.cond_len, dtype=torch.long) if cond is None else cond.reshape(B, cfg.cond_len)
    L, cl = xs.shape[1], cond.shape[1]
    emb = _body_emb(sd, flags, xs, codebook)
    c_emb = F.embedding(cond, sd["cond_emb.weight"]) + sd["pos_emb_cond"][:, :cl, :]
    emb = emb.sum(dim=-2) + sd["pos_emb_hw"][:, :L, :]
    lat = O.stack(sd, "body_transformer", torch.cat([c_emb, emb[:, :-1, :]], dim=1), cfg.n_body, cfg.nh)
    sp = lat[:, cl - 1:]
    dctx = _head_emb(sd, flags, xs, codebook)
    full = torch.cat([sp.view(B, L, 1, -1), dctx[:, :, :-1, :]], dim=-2).reshape(B * L, D, -1) + sd["pos_emb_d"][:, :D, :]
    out = O.stack(sd, "head_transformer", full, cfg.n_headl, cfg.nh).reshape(B, H, W, D, -1)
    logits = _classify(sd, flags, out.reshape(-1, D, out.shape[-1]), list(range(D))).reshape(B, H, W, D, -1)
    if with_cond_logits and cl > 1:
        return logits, O._linear(sd, "cond_classifier.linear", O._layer_norm(sd, "cond_classifier.layer_norm", lat[:, :cl - 1]))
    return logits


def needs_codebook(flags):
    return flags["input_emb_vqvae"] or flags["head_emb_vqvae"]


def state_dict_of(shapes, seed, vocab_sizes=None):
    """oracle/synth.py's seeded weights for a variant layout, with tok_emb.offsets set to the real row offsets (synth would draw
    random floats for the buffer)"""
    from oracle import synth
    sd = synth.synth_state_dict(shapes, seed)
    if "tok_emb.offsets" in sd:
        D = shapes["tok_emb.offsets"][0]
        vs = vocab_sizes or [shapes["tok_emb.weight"][0] // D] * D
        sd["tok_emb.offsets"] = torch.tensor([sum(vs[:d]) for d in range(D)], dtype=torch.long)
    return sd


# fixture plan (tests/golden/arv.pt) -- shapes in oracle/zoo.py's AR_ZOO tuple layout (E, heads, n_body, n_head_layers, V, block_size,
# vocab_cond, cond_len)
TINY = (128, 2, 2, 2, 512, (4, 4, 4), 10, 1)
TEXT = (128, 2, 2, 2, 512, (3, 3, 4), 16, 4)
HEADLESS = (128, 2, 2, 0, 512, (4, 4, 1), 10, 1)
UNEQUAL = dict(shape=(128, 2, 1, 1, [512, 256, 384, 128], (4, 4, 4), 10, 1), flags=dict(
    input_emb_vqvae=False, head_emb_vqvae=False, cumsum_depth_ctx=False, shared_tok_emb=False, shared_cls_emb=False))
ALL_FALSE = COMBOS[0]
PLAN = dict(B=2, weight_seed=41, table_seed=42, cond_seed=43, settings=[dict(top_k=1), dict(top_k=100, top_p=0.95)],
            noise_seeds=[700, 701], resume=dict(start_loc=(1, 2), noise_seed=702), init_seed=0, init_sample=16)
