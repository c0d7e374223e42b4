"""RQTransformer -- host-side mirror of rqvae/models/rqtransformer/transformers.py:34-369 over the native AR engine.

Boundary kept (SURVEY.md section 8b): constructor from an ``RQTransformerConfig``-shaped object, parameter names
(state_dict layout A.3), ``sample`` :294-307 (same signature; ``fast``/``cached``/``is_tqdm``/``desc`` accepted),
``cached_forward`` :191 (stateful after ``init_cache``: one native token step per call, ``rqb200_ar_step``), ``init_cache`` :289, ``get_block_size``, attributes ``block_size`` / ``block_size_cond`` /
``vocab_size``, the losses ``compute_loss`` / ``compute_cond_loss`` / ``compute_codebook_loss`` :371-410, and ``log_prob`` (teacher-forced
log-likelihoods without the logits, ``rqb200_ar_log_prob``).  The (h,w,d) loop, KV caches, embedding glue, classifier and ``sample_from_logits`` all run inside
``rqb200_ar_sample_span`` (csrc/ar_engine.cu): one native call per batch chunk and span of positions, no per-token host work.

Arithmetic tiers: ``amp=False`` -> 'exact' (fp32 weights/activations, FFMA -- the tier the bit-exact-indices gate is
defined on); ``amp=True`` -> 'fast' (fp16 weights / activations / KV on wgmma tensor cores, fp32 accumulate -- the
reference's own amp class is fp16 autocast, transformers.py:114,206; RQB200_FAST_DTYPE=bf16 selects bf16 instead,
RQB200_FAST_DTYPE=fp8 E4M3 weights with one fp32 scale per output row and fp16 activations / KV).
``self.precision`` ('exact' | 'fast') or RQB200_PRECISION overrides the ``amp`` mapping."""
import ctypes as C
import os
from collections import OrderedDict
from itertools import product

import torch
import torch.nn as nn

from ... import _native as N
from ..interfaces import Stage2Model
from .primitives import BatchLinear, LogitMask, TupleEmbedding


class _Holder(nn.Module):
    def forward(self, *a, **k):
        raise RuntimeError("rqb200: parameter holder -- compute runs in the native engine (RQTransformer.sample)")


class _Attn(_Holder):
    def __init__(self, E, n_head, bias):
        super().__init__()
        self.key, self.query, self.value = nn.Linear(E, E, bias=bias), nn.Linear(E, E, bias=bias), nn.Linear(E, E, bias=bias)
        self.proj = nn.Linear(E, E, bias)
        self.n_head = n_head


class _Block(_Holder):
    def __init__(self, cfg):
        super().__init__()
        E = cfg.embed_dim
        assert E % cfg.n_head == 0
        self.ln1, self.ln2 = nn.LayerNorm(E), nn.LayerNorm(E)
        self.attn = _Attn(E, cfg.n_head, cfg.attn_bias)
        # indices 0 / 2 carry the weights (attentions.py:117-122); 1 / 3 are GELU / dropout in the reference
        self.mlp = nn.Sequential(nn.Linear(E, 4 * E, bias=cfg.mlp_bias), nn.Identity(), nn.Linear(4 * E, E, bias=cfg.mlp_bias),
                                 nn.Identity())
        if cfg.gelu != "v1":
            raise NotImplementedError("rqb200: only the exact-erf GELU ('v1') is implemented (all shipped configs)")


class _Stack(_Holder):
    def __init__(self, cfg):
        super().__init__()
        self.blocks = nn.ModuleList([_Block(cfg.block) for _ in range(cfg.n_layer)])


class RQTransformer(N.EngineCache, Stage2Model):
    def __init__(self, config):
        super().__init__()
        self.config = config = config.copy()
        if len(config.block_size) != 3:
            raise ValueError("incompatible block size")
        self.block_size = torch.Size(config.block_size)
        if isinstance(config.vocab_size, int):
            config.vocab_size = [config.vocab_size] * config.block_size[2]
        vs = list(config.vocab_size)
        if config.shared_tok_emb or config.shared_cls_emb:
            assert [vs[0]] * len(vs) == vs, "shared token / classifier embeddings need one vocabulary size for every depth"
        self.vocab_size = vs
        E = config.embed_dim
        self.vocab_size_cond = max(config.vocab_size_cond, 1)
        self.block_size_cond = max(config.block_size_cond, 1)
        assert not (self.block_size_cond > 1 and self.vocab_size_cond == 1)
        # modules in the reference's order (transformers.py:60-105): same state_dict order, same draws under a seed
        self.cond_emb = nn.Embedding(self.vocab_size_cond, E)
        self.tok_emb, self.input_mlp, self.head_mlp = None, None, None
        if config.input_emb_vqvae:
            self.input_mlp = nn.Linear(config.input_embed_dim, E)
        if config.head_emb_vqvae:
            self.head_mlp = nn.Linear(config.input_embed_dim, E)
        if not (config.input_emb_vqvae and config.head_emb_vqvae):
            self.tok_emb = nn.Embedding(vs[0], E) if config.shared_tok_emb else TupleEmbedding(vs, E)
        self.pos_emb_cond = nn.Parameter(torch.zeros(1, self.block_size_cond, E))
        self.pos_emb_hw = nn.Parameter(torch.zeros(1, self.block_size[0] * self.block_size[1], E))
        self.pos_emb_d = nn.Parameter(torch.zeros(1, self.block_size[2], E))
        for p in (self.pos_emb_cond, self.pos_emb_hw, self.pos_emb_d):
            p.data.normal_(mean=0.0, std=0.02)
        self.body_transformer = _Stack(config.body)
        self.head_transformer = _Stack(config.head)
        cls = nn.Linear(E, vs[0]) if config.shared_cls_emb else BatchLinear(self.block_size[2], E, max(vs))
        self.classifier = nn.Sequential(OrderedDict([("layer_norm", nn.LayerNorm(E)), ("linear", cls),
                                                     ("logit_mask", LogitMask(vs, value=-1e6))]))
        if config.block_size_cond > 1:
            self.cond_classifier = nn.Sequential(OrderedDict([("layer_norm", nn.LayerNorm(E)),
                                                              ("linear", nn.Linear(E, config.vocab_size_cond))]))
        self.noise_budget_bytes = 256 << 20      # bound on the Exp(1) noise buffer sample() draws per span of positions
        self._cache = None
        self._step = None                        # the stepped cached_forward sequence (init_cache / _step_route)

    # ------------------------------------------------------------------ native engine plumbing
    _DESTROY = "rqb200_ar_destroy"

    def _invalidate_native(self):
        super()._invalidate_native()
        self._step = None                        # its KV caches lived in the engines' workspaces

    def _mode(self, amp):
        p = self.precision or N.default_precision()
        if p == "auto":
            p = "fast" if amp else "exact"
        return N.MODE_FAST if p == "fast" else N.MODE_EXACT

    def _embed_variant(self):
        """rqb200_ar_config.embed_variant of this model's five embedding / classifier switches (0: the shipped family)"""
        c = self.config
        v = 0 if c.input_emb_vqvae else N.EMB_TOK_INPUT
        v |= 0 if c.head_emb_vqvae else N.EMB_TOK_HEAD
        v |= N.EMB_NO_CUMSUM if (c.head_emb_vqvae and not c.cumsum_depth_ctx) else 0
        v |= N.EMB_TUPLE if (self.tok_emb is not None and not c.shared_tok_emb) else 0
        v |= 0 if c.shared_cls_emb else N.EMB_CLS_PER_DEPTH
        return v

    def _check_computable(self):
        if [self.vocab_size[0]] * len(self.vocab_size) != self.vocab_size:
            raise NotImplementedError("rqb200: per-depth vocabularies of different sizes (%s) can be built and loaded but not sampled "
                                      "or evaluated: the reference's LogitMask indexes the logits of one depth as if they held all "
                                      "depths and raises IndexError in both sample and forward, so there is no behaviour to "
                                      "reproduce" % (self.vocab_size,))

    def _codebook_of(self, model_aux, depth):
        """the table(s) behind model_aux.get_code_emb_with_depth (transformers.py:109-111): the [K,C] tensor of a shared codebook,
        or the list of the D per-depth [K,C] tables, each K equal to the vocabulary.  None when the model embeds its codes with its
        own tok_emb only (input_emb_vqvae and head_emb_vqvae both false): model_aux is not needed then."""
        if self.input_mlp is None and self.head_mlp is None:
            return None
        if model_aux is None:
            raise ValueError("rqb200: this model embeds codes through model_aux's codebooks (input_emb_vqvae or head_emb_vqvae "
                             "is true): pass the RQ-VAE as model_aux")
        q = getattr(model_aux, "quantizer", None)
        if q is not None and hasattr(q, "_tables"):
            tabs = q._tables()
            if isinstance(tabs, list) and (len(tabs) != depth or any(t.shape[0] != self.vocab_size[0] for t in tabs)):
                raise ValueError("rqb200: model_aux's per-depth codebooks must number %d, each of the vocabulary's size %d (got %s)"
                                 % (depth, self.vocab_size[0], [t.shape[0] for t in tabs]))
            return tabs
        if q is not None and hasattr(q, "_shared_table"):
            return q._shared_table()
        if q is not None and getattr(q, "shared_codebook", False):
            return q.codebooks[0].weight[:-1]
        raise NotImplementedError("rqb200: model_aux must be an RQ-VAE (its quantizer holds the codebooks)")

    def _engine(self, codebook, mode, slot=0):
        """codebook: one [K,C] table, a list of D per-depth tables, or None (a model that needs none).  Engines are keyed by the
        tables' storage and rebuilt when any of them is written in place (per-depth tables are stacked into one [D,K,C] copy per
        engine build)."""
        dev = self.pos_emb_hw.device
        per_depth = isinstance(codebook, list)
        if codebook is None:
            fp = (N.param_fingerprint(self), None)
            cb_id = None
        elif per_depth:
            fp = (N.param_fingerprint(self), tuple(t._version for t in codebook))
            cb_id = tuple(t.data_ptr() for t in codebook)
        else:
            fp = (N.param_fingerprint(self), codebook._version)
            cb_id = codebook.data_ptr()
        return self._cached_engine((str(dev), mode, cb_id, slot), fp, lambda: self._build_engine(codebook, mode, slot))

    def _build_engine(self, codebook, mode, slot):
        if slot != 0:
            # engines of one model share the packed weights of slot 0; each slot owns its workspace, KV cache and graphs
            base = self._engine(codebook, mode, 0)
            return dict(base, handle=base["make"](), ws=None)
        N.require_cuda(self.pos_emb_hw, *(codebook if isinstance(codebook, list) else [codebook]))
        self._check_computable()
        L = N.lib()
        cfg, w, keep, streamed = self._engine_structs(codebook, mode)

        def make():
            hnd = L.rqb200_ar_create(C.byref(cfg), C.byref(w))
            if not hnd:
                raise N.NativeError("rqb200_ar_create: " + L.rqb200_last_error().decode())
            return hnd

        return {"handle": make(), "keep": keep, "ws": None, "make": make, "weight_dtype": cfg.weight_dtype, "streamed": streamed}

    def _engine_structs(self, codebook, mode):
        """the rqb200_ar_config / rqb200_ar_weights of one engine build and the tensors they point into: (cfg, w, keep, streamed),
        streamed = the tensors of the streamed weights (a subset of keep).  The fast tier's streamed weights (every nn.Linear / BatchLinear weight) are copied in its weight format:
        fp16 or bf16, or (RQB200_FAST_DTYPE=fp8) packed E4M3 tiles plus fp32 row scales and no 16-bit copy; everything else is
        read as fp32.  Host-only: runs on CPU tensors too."""
        per_depth = isinstance(codebook, list)
        fmt = N.fast_weight_format() if mode == N.MODE_FAST else "fp32"
        wdt = {"fp32": torch.float32, "fp16": torch.float16, "bf16": torch.bfloat16, "fp8": None}[fmt]
        keep, streamed = [], []

        def f32(t):
            t = t.detach().float().contiguous()
            keep.append(t)
            return t.data_ptr()

        def wt(t):
            """one streamed weight ([N,K], or [D,N,K] per-depth) -> (weight pointer, row-scale pointer or None)"""
            if fmt == "fp8":
                q, sc = N.pack_fp8_weight(t.detach())
                keep.extend([q, sc])
                streamed.extend([q, sc])
                return q.data_ptr(), sc.data_ptr()
            t = t.detach().to(wdt).contiguous()
            keep.append(t)
            streamed.append(t)
            return t.data_ptr(), None

        def blocks(stack):
            arr = (N.BlockWeights * len(stack.blocks))()
            for i, b in enumerate(stack.blocks):
                a = b.attn
                wqkv = torch.cat([a.query.weight, a.key.weight, a.value.weight], 0)
                bqkv = torch.cat([a.query.bias, a.key.bias, a.value.bias], 0)
                (arr[i].wqkv, arr[i].sqkv), arr[i].bqkv = wt(wqkv), f32(bqkv)
                del wqkv
                (arr[i].w1, arr[i].s1), arr[i].b1 = wt(b.mlp[0].weight), f32(b.mlp[0].bias)
                (arr[i].wproj, arr[i].sproj), arr[i].bproj = wt(a.proj.weight), f32(a.proj.bias)
                (arr[i].w2, arr[i].s2), arr[i].b2 = wt(b.mlp[2].weight), f32(b.mlp[2].bias)
                arr[i].ln1_w, arr[i].ln1_b = f32(b.ln1.weight), f32(b.ln1.bias)
                arr[i].ln2_w, arr[i].ln2_b = f32(b.ln2.weight), f32(b.ln2.bias)
            return arr

        cfg = N.ArConfig()
        c = self.config
        cfg.embed_dim, cfg.n_head = c.embed_dim, c.body.block.n_head
        cfg.n_body, cfg.n_head_layers = len(self.body_transformer.blocks), len(self.head_transformer.blocks)
        cfg.vocab, cfg.H, cfg.W, cfg.D = self.vocab_size[0], self.block_size[0], self.block_size[1], self.block_size[2]
        cfg.vocab_cond, cfg.cond_len = self.vocab_size_cond, self.block_size_cond
        if codebook is None:
            cfg.code_dim, cfg.codebook_size = 64, self.vocab_size[0]        # (unused: no code goes through a codebook)
        else:
            table0 = codebook[0] if per_depth else codebook
            cfg.code_dim, cfg.codebook_size = table0.shape[1], table0.shape[0]
        cfg.codebook_per_depth = int(per_depth)
        cfg.mode, cfg.weight_dtype = mode, N.E4M3 if fmt == "fp8" else N._DT[wdt]
        cfg.flags = N.ar_engine_options() if mode == N.MODE_FAST else 0      # (the split_* fields stay 0: the engine fills the SMs)
        cfg.embed_variant = self._embed_variant()
        if c.head.block.n_head != c.body.block.n_head:
            raise NotImplementedError("rqb200: body and head stacks must share n_head")
        w = N.ArWeights()
        w.pos_emb_cond, w.pos_emb_hw, w.pos_emb_d = f32(self.pos_emb_cond), f32(self.pos_emb_hw), f32(self.pos_emb_d)
        w.cond_emb = f32(self.cond_emb.weight)
        if self.input_mlp is not None:
            (w.w_in, w.s_in), w.b_in = wt(self.input_mlp.weight), f32(self.input_mlp.bias)
        if self.head_mlp is not None:
            (w.w_head, w.s_head), w.b_head = wt(self.head_mlp.weight), f32(self.head_mlp.bias)
        if self.tok_emb is not None:
            te = self.tok_emb
            if isinstance(te, TupleEmbedding):
                V, D = self.vocab_size[0], self.block_size[2]
                if te.offsets.tolist() != [d * V for d in range(D)]:
                    raise ValueError("rqb200: tok_emb.offsets must be [0, V, 2V, ...] (got %s)" % te.offsets.tolist())
            w.tok_emb = f32(te.weight)
        lin = self.classifier.linear
        if isinstance(lin, BatchLinear):
            # [D,E,V] (input-major) -> one [D,V,E] copy per engine build: depth d's classifier is a row-major [V,E] slice (E4M3:
            # quantised by its own V rows, scales [D,V])
            (w.w_cls, w.s_cls), w.b_cls = wt(lin.weight.detach().transpose(1, 2)), f32(lin.bias)
        else:
            (w.w_cls, w.s_cls), w.b_cls = wt(lin.weight), f32(lin.bias)
        w.cls_ln_w, w.cls_ln_b = f32(self.classifier.layer_norm.weight), f32(self.classifier.layer_norm.bias)
        if codebook is not None:
            w.codebook = f32(torch.stack(codebook)) if per_depth else f32(codebook)
        if hasattr(self, "cond_classifier") and mode == N.MODE_FAST:
            pad = -self.vocab_size_cond % 128            # classifier rows padded with zeros up to the 128-feature wgmma tile
            pw = torch.nn.functional.pad(self.cond_classifier.linear.weight.detach(), (0, 0, 0, pad))
            pb = torch.nn.functional.pad(self.cond_classifier.linear.bias.detach(), (0, pad))
            (w.w_ccls, w.s_ccls), w.b_ccls = wt(pw), f32(pb)      # (E4M3: the zero rows get s = 1, q = 0)
            w.ccls_ln_w, w.ccls_ln_b = f32(self.cond_classifier.layer_norm.weight), f32(self.cond_classifier.layer_norm.bias)
        body, head = blocks(self.body_transformer), blocks(self.head_transformer)
        w.body, w.head = C.cast(body, C.POINTER(N.BlockWeights)), C.cast(head, C.POINTER(N.BlockWeights))
        keep.extend([body, head, cfg, w])
        return cfg, w, keep, streamed

    def native_weight_bytes(self):
        """bytes of the tensors the native engines of this model hold, each build counted once (engine slots share one):
        {"streamed": the weight copies the fast tier streams, in its format (E4M3: packed bytes + 4 per row scale), "fp32": the
        fp32 tensors they read (embeddings, biases, LayerNorms, codebook; mostly the module's own parameters)}"""
        seen, out = set(), {"streamed": 0, "fp32": 0}
        for eng in self._eng.values():
            if id(eng["keep"]) in seen:
                continue
            seen.add(id(eng["keep"]))
            sids = {id(t) for t in eng["streamed"]}
            for t in eng["keep"]:
                if isinstance(t, torch.Tensor):
                    out["streamed" if id(t) in sids else "fp32"] += t.numel() * t.element_size()
        return out

    # ------------------------------------------------------------------ reference surface
    def init_cache(self):
        """transformers.py:289-292 -- ends any stepped cached_forward sequence; the next cached_forward at some (h, w, 0) starts a
        new one (sample() keeps its KV state inside its own native call)"""
        self._cache = {"spatial_ctx_hw": None}
        self._step = {"armed": True}

    def _lists(self, top_k, top_p):
        D = self.block_size[2]
        V = self.vocab_size
        if top_k is None:
            ks = [V[i] for i in range(D)]
        elif isinstance(top_k, int):
            ks = [min(top_k, V[i]) for i in range(D)]
        elif len(top_k) == 1:
            ks = [min(top_k[0], V[i]) for i in range(D)]
        else:
            ks = [min(top_k[i], V[i]) for i in range(D)]
        if top_p is None:
            ps = [1.0] * D
        elif isinstance(top_p, float):
            ps = [min(top_p, 1.0)] * D
        elif len(top_p) == 1:
            ps = [min(top_p[0], 1.0)] * D
        else:
            ps = [min(top_p[i], 1.0) for i in range(D)]
        return ks, ps

    def _guidance(self, B, cfg_scale, uncond):
        """sample()'s classifier-free guidance arguments checked before any kernel runs: None (unguided) or (s, uncond [B, cond_len]
        int64).  Raises ValueError for a scale without uncond or the reverse, an unconditional model, an uncond that does not reshape
        to [B, cond_len] or is not integer, and entries outside [0, vocab_size_cond) (one host read)."""
        if cfg_scale is None and uncond is None:
            return None
        if cfg_scale is None or uncond is None:
            raise ValueError("rqb200: classifier-free guidance needs both cfg_scale and uncond")
        if self.vocab_size_cond == 1:
            raise ValueError("rqb200: classifier-free guidance needs a conditional model (vocab_size_cond > 1)")
        if isinstance(cfg_scale, bool) or not isinstance(cfg_scale, (int, float)):
            raise ValueError("rqb200: cfg_scale must be a float, got %r" % (cfg_scale,))
        cl = self.block_size_cond
        if not isinstance(uncond, torch.Tensor) or uncond.dtype.is_floating_point or uncond.dtype.is_complex or \
                uncond.dtype == torch.bool or uncond.numel() != B * cl:
            raise ValueError("rqb200: uncond must be an integer tensor that reshapes to cond's [%d, %d], got %s %s"
                             % (B, cl, getattr(uncond, "dtype", type(uncond)), tuple(getattr(uncond, "shape", ()))))
        u = uncond.reshape(B, cl).to(torch.int64)
        if bool(((u < 0) | (u >= self.vocab_size_cond)).any()):
            raise ValueError("rqb200: uncond entries must lie in [0, %d)" % self.vocab_size_cond)
        return float(cfg_scale), u

    def _keep_mask(self, keep_mask, B, start_loc, canvas=None):
        """sample()'s keep_mask checked before any kernel runs and laid out for the engine: None, or a contiguous uint8 [B, H, W, D] with
        the start_loc prefix kept too.  Raises ValueError for a mask that is not a bool tensor, does not broadcast to [B, H, W, D] or lies
        on another device than the model.  canvas: (Ht, Wt) of a canvas larger than the grid, which then takes the place of (H, W)."""
        if keep_mask is None:
            return None
        H, W, D = self.block_size
        if canvas is not None:
            H, W = canvas
        if not isinstance(keep_mask, torch.Tensor) or keep_mask.dtype != torch.bool:
            raise ValueError("rqb200: keep_mask must be a torch.bool tensor, got %s" % getattr(keep_mask, "dtype", type(keep_mask)))
        if keep_mask.device != self.pos_emb_hw.device:
            raise ValueError("rqb200: keep_mask is on %s, the model on %s" % (keep_mask.device, self.pos_emb_hw.device))
        want = (B, H, W, D)
        try:
            ok = tuple(torch.broadcast_shapes(tuple(keep_mask.shape), want)) == want
        except RuntimeError:
            ok = False
        if not ok:
            raise ValueError("rqb200: keep_mask of shape %s does not broadcast to [B, H, W, D] = %s" % (tuple(keep_mask.shape), want))
        keep = keep_mask.expand(want).to(torch.uint8).contiguous()
        idx0 = min(start_loc[0] * W + start_loc[1], H * W)
        keep.view(B, H * W, D)[:, :idx0] = 1
        return keep

    @torch.no_grad()
    def _native_sample(self, partial, model_aux, cond, start_loc, temperature, top_k, top_p, amp, noise=None,
                       return_logits=False, force_codes=None, guidance=None, keep=None):
        """guidance: None, or (s, uncond [B, cond_len] int64) from _guidance -- classifier-free guidance: every image runs a cond and an
        uncond branch as rows [cond | uncond] of one native call (cfg_n = rows / 2), noise stays per image [n_tok, B, V],
        logits (return_logits) and force_codes hold both branches' rows [2B]: [cond rows | uncond rows].
        keep: None, or uint8 [B, H, W, D] from _keep_mask -- masked completion (keep, sampled_host): each batch chunk passes its
        rows of the mask (guided: in both branches' rows) and the positions where any of its rows samples any depth; those position
        lists are formed on the device and read to the host once per call.  The logits of positions a chunk skips are not written."""
        H, W, D = partial.shape[1:]         # the canvas: the model's grid, or larger (sliding-window sampling)
        B = partial.shape[0]
        dev = self.pos_emb_hw.device
        self._check_computable()
        N.require_cuda(partial, cond, self.pos_emb_hw, None if guidance is None else guidance[1])
        ks, ps = self._lists(top_k, top_p)
        codebook = self._codebook_of(model_aux, D)
        mode = self._mode(amp)
        partial = partial.to(torch.int64).contiguous()
        cl = self.block_size_cond
        cond_t = None if cond is None else cond.reshape(B, cl).to(torch.int64).contiguous()
        idx0 = start_loc[0] * W + start_loc[1]
        n_tok = max(H * W - idx0, 0) * D
        V = self.vocab_size[0]
        HWD = H * W * D
        R = B if guidance is None else 2 * B          # batch rows of the engine: one per image, or one per image and branch
        with torch.cuda.device(dev):
            draw = noise is None            # draw the Exp(1) noise here, exactly as torch.multinomial would (utils.py:114)
            if noise is False:
                noise = None
            logits = torch.empty(n_tok, R, V, dtype=torch.float32, device=dev) if return_logits else None
            out = torch.empty_like(partial)
            kk = (C.c_int32 * D)(*[int(k) for k in ks])
            pp = (C.c_float * D)(*[float(p) for p in ps])
            fc = None if force_codes is None else force_codes.to(torch.int64).contiguous()
            # images per native call: the fast tier runs at most 256 rows, so a guided call takes at most 128 images
            bounds = _chunk_bounds(B, mode, 256 if guidance is None else 128)
            if len(bounds) > 1 and return_logits:
                raise N.NativeError("rqb200: return_logits with more than one batch chunk (B > %d) is not supported on the fast tier"
                                    % (256 if guidance is None else 128))
            # per chunk: (rows, partial, cond, force, out) as the native call reads them, each row 0 the chunk's first
            if guidance is None:
                calls = [(hi - lo, _rows(partial, lo), _rows(cond_t, lo), _rows(fc, lo), _rows(out, lo)) for lo, hi in bounds]
            else:
                u = guidance[1]
                cu = torch.zeros(B, cl, dtype=torch.int64, device=dev) if cond_t is None else cond_t
                calls = [(2 * (hi - lo), torch.cat([partial[lo:hi], partial[lo:hi]]), torch.cat([cu[lo:hi], u[lo:hi]]),
                          None if fc is None else torch.cat([fc[lo:hi], fc[B + lo:B + hi]]),
                          torch.empty(2 * (hi - lo), H, W, D, dtype=torch.int64, device=dev)) for lo, hi in bounds]
            plans = [(None, None)] * len(bounds)                    # per chunk: (sampled_host, keep rows), NULL unless masked
            if keep is not None:
                HW = H * W
                sampled = torch.stack([(keep[lo:hi] == 0).reshape(hi - lo, HW, D).any(2).any(0) for lo, hi in bounds])
                sampled = sampled.to(torch.uint8).cpu()                 # the call's one host read
                plans = [((C.c_uint8 * HW)(*sampled[i].tolist()),
                          keep[lo:hi] if guidance is None else torch.cat([keep[lo:hi], keep[lo:hi]]).contiguous())
                         for i, (lo, hi) in enumerate(bounds)]
            # position spans: when the noise is drawn here it is drawn span by span into one bounded buffer (noise_budget_bytes)
            # instead of one [n_tok,B,V] tensor (1 GB at 8x8x4, B=64, V=16384); every batch chunk keeps its own engine slot
            # (workspace + KV state) so that all chunks can resume on the next span
            n_pos = H * W - idx0
            per_pos = max(1, D * B * V * 4)
            span = max(1, min(n_pos, int(self.noise_budget_bytes) // per_pos)) if draw else max(n_pos, 1)
            if draw and n_tok > 0:
                noise = torch.empty(min(span, n_pos) * D, B, V, dtype=torch.float32, device=dev)
            st = torch.cuda.current_stream(dev)
            launches = 0
            engines = []
            for slot, call in enumerate(calls):
                eng = self._engine(codebook, mode, slot)
                _workspace(eng, N.lib().rqb200_ar_workspace_bytes(eng["handle"], call[0]), dev)
                engines.append(eng)

            def off(t, lo, row_elems, esize, extra=0):
                return C.c_void_p(t.data_ptr() + (lo * row_elems + extra) * esize) if t is not None else C.c_void_p(0)

            for p0 in range(idx0, H * W, span):
                p1 = min(p0 + span, H * W)
                if draw:
                    # one exponential_ per token, in (h,w,d) order: the draws torch.multinomial would make
                    for t in range((p1 - p0) * D):
                        noise[t].exponential_(1)
                tok0 = 0 if draw else (p0 - idx0) * D                  # first token of this span inside `noise`
                for i, (eng, (lo, hi), (rows, part_c, cond_c, fc_c, out_c)) in enumerate(zip(engines, bounds, calls)):
                    N.check(N.lib().rqb200_ar_sample_span(
                        eng["handle"], off(part_c, 0, HWD, 8), off(cond_c, 0, cl, 8), rows, p0, p1, int(p0 > idx0),
                        float(temperature), kk, pp, off(noise, lo, V, 4, tok0 * B * V), 0 if noise is None else B * V,
                        off(logits, 0, V, 4, (p0 - idx0) * D * R * V), off(fc_c, 0, HWD, 8), off(out_c, 0, HWD, 8),
                        N.ptr(eng["ws"]), eng["ws"].numel(), C.c_void_p(st.cuda_stream), N.ptr(plans[i][1]), plans[i][0],
                        0 if guidance is None else rows // 2, C.c_float(0.0 if guidance is None else guidance[0]), C.c_int(H), C.c_int(W)), "ar_sample")
                    launches += N.lib().rqb200_ar_last_launches(eng["handle"])
            if n_tok == 0:
                out.copy_(partial)
            elif guidance is not None:
                for (lo, hi), call in zip(bounds, calls):
                    out[lo:hi] = call[4][:hi - lo]
        self.last_launches = launches
        N.launch_count["total"] += launches
        return (out, logits) if return_logits else out

    def native_trace(self):
        """diagnostics (RQB200_TRACE=1, fast tier): [(name, t_entry, t_dependency_resolved, t_mid, t_done)] in ns for every launch
        slot of the last replay of each captured graph -- where the time of one AR position goes"""
        rows = []
        for key, eng in self._eng.items():
            cap = 12288                          # TR_CAP of csrc/ar_fast.cu: 1024 slots for each of its 12 graphs
            buf = (C.c_longlong * (4 * cap))()
            names = C.create_string_buffer(cap * 16)
            n = N.lib().rqb200_ar_trace(eng["handle"], buf, cap, names, len(names))
            nm = names.value.decode().split("\n")
            for i in range(max(n, 0)):
                if buf[4 * i]:
                    rows.append((nm[i] if i < len(nm) else "?", buf[4 * i], buf[4 * i + 1], buf[4 * i + 2], buf[4 * i + 3], i))
        return rows

    @torch.no_grad()
    def sample(self, partial_sample, model_aux=None, cond=None, start_loc=(0, 0), temperature=1.0, top_k=None, top_p=None,
               amp=False, cached=True, is_tqdm=False, desc="Sampling", fast=True, cfg_scale=None, uncond=None, keep_mask=None):
        """transformers.py:294-369.  Returns LongTensor [B,H,W,D]; ``partial_sample`` is not modified.
        Classifier-free guidance: with a float ``cfg_scale`` s and ``uncond`` (cond's shape: an unconditional or negative condition
        per image), every token is drawn from l = u + s * (c - u) -- c the logits under ``cond``, u under ``uncond`` -- then
        temperature, top-k and top-p as unguided, with one Exp(1) draw per image and token.  Both branches share the
        partial_sample / start_loc prefix and every drawn code.  The default ``cfg_scale=None`` samples unguided.
        Masked completion (editing): ``keep_mask``, a torch.bool tensor on the model's device that broadcasts to [B, H, W, D] (e.g.
        [H, W, 1] for a region of every image, [1, 1, 1, D] for depths), keeps partial_sample's code wherever it is True; the positions
        before start_loc are kept as always.  Every other token is sampled as sample() would, seeing the kept codes before it in raster
        order (and none after it), and every token still takes its Exp(1) draw.  Positions where nothing is sampled skip the head stack;
        their codes reach the body in one batched pass per run on the fast tier.  Which positions those are is read to the host once
        per call.  Composes with guidance, both tiers and every fast weight format.
        Canvases larger than the grid (sliding-window sampling): ``partial_sample`` [B, Ht, Wt, D] with Ht >= H, Wt >= W returns
        [B, Ht, Wt, D].  The token at canvas (i, j, d) is sampled as the model's token (i - r0, j - c0, d) of the H x W window with origin
        r0 = clamp(i - H // 2, 0, Ht - H), c0 = clamp(j - W // 2, 0, Wt - W) (Taming Transformers' rule at even sizes), seeing the cond
        prefix, the window's positions before it and its own depths < d, read from the canvas as it stands -- nothing outside its
        window.  ``start_loc`` is in canvas coordinates and ``keep_mask`` broadcasts to [B, Ht, Wt, D] (outpainting: keep the encoded
        part).  Ht * Wt * D may not exceed 2^31 - 1.  On the grid itself this is the call above, launch for launch."""
        shp = partial_sample.shape
        assert len(shp) == 4 and shp[1] >= self.block_size[0] and shp[2] >= self.block_size[1] and shp[3] == self.block_size[2]
        if shp[1] * shp[2] * shp[3] > CANVAS_MAX_CODES:
            raise ValueError("rqb200: a canvas of %d x %d x %d codes is past the engine's index range (Ht * Wt * D <= 2^31 - 1)"
                             % (shp[1], shp[2], shp[3]))
        guidance = self._guidance(partial_sample.shape[0], cfg_scale, uncond)
        keep = self._keep_mask(keep_mask, partial_sample.shape[0], start_loc, canvas=(shp[1], shp[2]))
        self.init_cache()
        out = self._native_sample(partial_sample, model_aux, cond, start_loc, temperature, top_k, top_p, amp, guidance=guidance,
                                  keep=keep)
        self.init_cache()
        return out

    def _step_key(self, B, mode, codebook, cond, device):
        """what a stepped sequence must keep from call to call: batch, tier, the codebook tables and the cond tensor (compared by
        storage, not by value: reading them back would synchronise every call)"""
        tabs = None if codebook is None else (tuple(t.data_ptr() for t in codebook) if isinstance(codebook, list) else codebook.data_ptr())
        cnd = None if cond is None else (cond.data_ptr(), tuple(cond.shape), cond.dtype)
        return (B, mode, tabs, cnd, str(device))

    def _step_route(self, key, loc, n_codes):
        """'restart', 'continue' or None (stateless evaluation) for a cached_forward at loc = (h, w, d) with the sequence key `key`
        over xs holding n_codes codes per batch row; updates the sequence record.
          restart:  the first call after init_cache(), at some (h, w, 0) -- the reference prefills the prefix then (:237-239);
          continue: the token after the previous call's, in raster order, with the same key.
        Any other call is evaluated statelessly.  One with the sequence's key ends the sequence (the reference would append a
        duplicate or misplaced KV entry, or fail); one with another key (another batch, tier, cond or codebook) leaves it alone."""
        H, W, D = self.block_size
        h, w, d = loc
        st = self._step
        if st is None:
            return None
        if not (0 <= h < H and 0 <= w < W and 0 <= d < D):
            return None
        t = (h * W + w) * D + d
        if n_codes < (t if d > 0 else (h * W + w) * D):          # xs lacks codes the step reads: let the stateless path zero-pad
            if not st.get("armed") and st["key"] == key:
                self._step = None
            return None
        if st.get("armed"):
            if d != 0:
                self._step = None
                return None
            self._step = {"key": key, "next": t + 1, "engines": None}
            return "restart"
        if st["key"] != key:
            return None
        if st["next"] != t:
            self._step = None
            return None
        st["next"] = t + 1
        return "continue"

    @torch.no_grad()
    def cached_forward(self, xs, model_aux=None, cond=None, amp=False, sample_loc=(0, 0, 0)):
        """transformers.py:190-287 -- logits [B,V] for one (h,w,d).
        After init_cache(), calls in raster order from some (h, w, 0) (the reference's own loop) run one native token step each
        (rqb200_ar_step): the first prefills cond and the positions before it from ``xs``, every later one appends one body token
        (d == 0) and runs one head depth, on KV caches kept in engine slots of their own.  Like the reference, ``cond`` is read by
        the first call only and later calls read only the codes the step consumes.  Any other call pattern is evaluated
        statelessly: the prefix in ``xs`` is teacher-forced through the native loop and the requested step's logits returned."""
        h, w, d = (int(v) for v in sample_loc)
        H, W, D = self.block_size
        B = xs.shape[0]
        route = None
        if self._step is not None and xs.dim() == 4 and tuple(xs.shape[2:]) == (W, D):
            codebook = self._codebook_of(model_aux, D)
            mode = self._mode(amp)
            key = self._step_key(B, mode, codebook, cond, xs.device)
            route = self._step_route(key, (h, w, d), xs.shape[1] * W * D)
        if route is not None:
            out = self._native_step(route, xs, codebook, cond, mode, (h, w, d))
            if out is not None:
                return out
        return self._stateless_cached_forward(xs, model_aux, cond, amp, (h, w, d))

    def _stateless_cached_forward(self, xs, model_aux, cond, amp, sample_loc):
        h, w, d = sample_loc
        H, W, D = self.block_size
        B = xs.shape[0]
        full = torch.zeros(B, H, W, D, dtype=torch.int64, device=xs.device)
        full[:, :xs.shape[1]] = xs
        _, logits = self._native_sample(full, model_aux, cond, (0, 0), 1.0, None, None, amp, noise=False,
                                        return_logits=True, force_codes=full)
        return logits[(h * W + w) * D + d]

    @torch.no_grad()
    def _native_step(self, route, xs, codebook, cond, mode, loc):
        """one rqb200_ar_step per batch chunk (fast tier: equal chunks of at most 256 rows, as _native_sample), each on its own
        engine slot ("step", chunk).  None when the slots were rebuilt since the sequence began (weights written, .to(...)): the
        stale caches are gone and the caller evaluates statelessly."""
        H, W, D = self.block_size
        h, w, d = loc
        B, V, cl = xs.shape[0], self.vocab_size[0], self.block_size_cond
        dev = self.pos_emb_hw.device
        N.require_cuda(xs, cond, self.pos_emb_hw)
        bounds = _chunk_bounds(B, mode)
        st = self._step
        restart = route == "restart"
        try:
            engines = [self._engine(codebook, mode, ("step", i)) for i in range(len(bounds))]
            if self._step is not st:                 # _engine found the weights changed and dropped every engine and the sequence
                if not restart:
                    return None
                self._step = st                      # (a sequence that begins now has no stale state)
            if restart:
                st["engines"] = engines
            elif any(a is not b for a, b in zip(engines, st["engines"])):
                self._step = None
                return None
            if xs.dtype != torch.int64 or xs.stride()[1:] != (W * D, D, 1):
                xs = xs.to(torch.int64).contiguous()
            stride = xs.stride(0) if B > 1 else xs.shape[1] * W * D
            cond_t = None if (cond is None or not restart) else cond.reshape(B, cl).to(torch.int64).contiguous()
            out = torch.empty(B, V, dtype=torch.float32, device=dev)
            L = N.lib()
            launches = 0
            with torch.cuda.device(dev):
                stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
                for eng, (lo, hi) in zip(engines, bounds):
                    if restart:                      # (sized when a sequence begins; its batch stays until the next one)
                        _workspace(eng, L.rqb200_ar_workspace_bytes(eng["handle"], hi - lo), dev)
                    N.check(L.rqb200_ar_step(
                        eng["handle"], C.c_void_p(xs.data_ptr() + lo * stride * 8), stride,
                        C.c_void_p(cond_t.data_ptr() + lo * cl * 8) if cond_t is not None else C.c_void_p(0), hi - lo, h, w, d,
                        int(restart), C.c_void_p(out.data_ptr() + lo * V * 4), N.ptr(eng["ws"]), eng["ws"].numel(), stream), "ar_step")
                    launches += L.rqb200_ar_last_launches(eng["handle"])
        except BaseException:
            self._step = None
            raise
        self.last_launches = launches
        N.launch_count["total"] += launches
        return out

    def forward(self, xs, model_aux=None, cond=None, amp=False):
        """transformers.py:113-188 -- teacher-forced logits [B,H,W,D,V]; with cond_len > 1 also the cond logits
        [B,cond_len-1,vocab_cond] (the reference's return convention :185-188).
        Fast tier (amp=True): all positions at once -- the body over B*(cond_len+H*W-1) rows, the head over B*H*W*D rows, as
        large-M wgmma GEMMs + causal attention (rqb200_ar_forward).  Exact tier: the sequential teacher-forced replay."""
        B, H, W, D = xs.shape
        self._check_computable()
        if self._mode(amp) == N.MODE_FAST:
            return self._native_forward(xs, model_aux, cond)
        if self.block_size_cond > 1:
            raise NotImplementedError("rqb200: cond_logits (cond_len > 1) are produced by the fast tier only (amp=True)")
        _, logits = self._native_sample(xs, model_aux, cond, (0, 0), 1.0, None, None, amp, noise=False,
                                        return_logits=True, force_codes=xs)
        return logits.reshape(H, W, D, B, -1).permute(3, 0, 1, 2, 4).contiguous()

    @torch.no_grad()
    def _native_forward(self, xs, model_aux, cond):
        H, W, D = self.block_size
        B = xs.shape[0]
        dev = self.pos_emb_hw.device
        N.require_cuda(xs, cond, self.pos_emb_hw)
        codebook = self._codebook_of(model_aux, D)
        eng = self._engine(codebook, N.MODE_FAST)
        xs = xs.to(torch.int64).contiguous()
        cl, V = self.block_size_cond, self.vocab_size[0]
        cond_t = None if cond is None else cond.reshape(B, cl).to(torch.int64).contiguous()
        want_cond = cl > 1 and hasattr(self, "cond_classifier")
        with torch.cuda.device(dev):
            ws = _workspace(None, N.lib().rqb200_ar_forward_workspace_bytes(eng["handle"], B), dev)
            logits = torch.empty(D, H * W, B, V, dtype=torch.float32, device=dev)
            vcp = -(-self.vocab_size_cond // 128) * 128
            cond_logits = torch.empty(cl - 1, B, vcp, dtype=torch.float32, device=dev) if want_cond else None
            N.check(N.lib().rqb200_ar_forward(eng["handle"], N.ptr(xs), N.ptr(cond_t), B, N.ptr(logits), N.ptr(cond_logits), N.ptr(ws),
                                              ws.numel(), N.stream_ptr(dev)), "ar_forward")
            self.last_launches = N.lib().rqb200_ar_last_launches(eng["handle"])
            N.launch_count["total"] += self.last_launches
        out = logits.permute(2, 1, 0, 3).reshape(B, H, W, D, V).contiguous()
        if want_cond:
            return out, cond_logits[..., :self.vocab_size_cond].permute(1, 0, 2).contiguous()
        return out

    @torch.no_grad()
    def log_prob(self, xs, model_aux=None, cond=None, amp=False):
        """teacher-forced log-likelihoods log p(x_{h,w,d} | x before it, cond) [B,H,W,D] fp32: forward's logits log-softmaxed and gathered
        at xs, computed without the [B,H,W,D,V] logits (rqb200_ar_log_prob: fast tier, the classifier in bounded row chunks; exact tier,
        the teacher-forced replay in bounded spans).  Tiers and return convention as forward: with cond_len > 1 and a cond classifier
        (fast tier) also the cond log-likelihoods [B,cond_len-1] of cond[:, 1:].  Codes outside [0, V) (and cond entries outside
        [0, vocab_size_cond)) raise ValueError before any kernel runs."""
        H, W, D = self.block_size
        if xs.dim() != 4 or tuple(xs.shape[1:]) != (H, W, D):
            raise ValueError("rqb200: log_prob expects codes [B,%d,%d,%d], got %s" % (H, W, D, tuple(xs.shape)))
        B = xs.shape[0]
        self._check_computable()
        mode = self._mode(amp)
        cl, V = self.block_size_cond, self.vocab_size[0]
        want_cond = cl > 1 and hasattr(self, "cond_classifier")
        if mode == N.MODE_EXACT and want_cond:
            raise NotImplementedError("rqb200: cond log-likelihoods (cond_len > 1) are produced by the fast tier only (amp=True)")
        N.require_cuda(xs, cond, self.pos_emb_hw)
        dev = self.pos_emb_hw.device
        xs = xs.to(torch.int64).contiguous()
        cond_t = None if cond is None else cond.reshape(B, cl).to(torch.int64).contiguous()
        if want_cond and cond_t is None:
            cond_t = torch.zeros(B, cl, dtype=torch.int64, device=dev)        # (forward's cond = None: zeros)
        bad = ((xs < 0) | (xs >= V)).any()
        if cond_t is not None:
            bad = bad | ((cond_t < 0) | (cond_t >= self.vocab_size_cond)).any()
        if bool(bad):                                                       # one reduction, one host read per call
            raise ValueError("rqb200: log_prob: codes must lie in [0, %d) and cond in [0, %d)" % (V, self.vocab_size_cond))
        codebook = self._codebook_of(model_aux, D)
        eng = self._engine(codebook, mode)
        L = N.lib()
        with torch.cuda.device(dev):
            ws = _workspace(None, L.rqb200_ar_log_prob_workspace_bytes(eng["handle"], B), dev)
            logp = torch.empty(D, H * W, B, dtype=torch.float32, device=dev)
            cond_logp = torch.empty(cl - 1, B, dtype=torch.float32, device=dev) if want_cond else None
            N.check(L.rqb200_ar_log_prob(eng["handle"], N.ptr(xs), N.ptr(cond_t), B, N.ptr(logp), N.ptr(cond_logp), N.ptr(ws), ws.numel(),
                                         N.stream_ptr(dev)), "ar_log_prob")
            self.last_launches = L.rqb200_ar_last_launches(eng["handle"])
            N.launch_count["total"] += self.last_launches
        out = logp.permute(2, 1, 0).reshape(B, H, W, D)
        if want_cond:
            return out, cond_logp.t().contiguous()
        return out

    # ------------------------------------------------------------------ stage-2 losses (transformers.py:371-410), torch over given logits
    def compute_loss(self, logits, targets, use_soft_target=False):
        if use_soft_target:
            return _soft_target_cross_entropy(logits.reshape(-1, logits.shape[-1]), targets.reshape(-1, targets.shape[-1]))
        return torch.nn.functional.cross_entropy(logits.reshape(-1, logits.shape[-1]), targets.reshape(-1))

    def compute_cond_loss(self, cond_logits, conds):
        assert cond_logits.shape[1] == (conds.shape[1] - 1)
        targets = conds[:, 1:].contiguous()
        return torch.nn.functional.cross_entropy(cond_logits.reshape(-1, cond_logits.shape[-1]), targets.reshape(-1))

    @torch.no_grad()
    def compute_codebook_loss(self, logits, targets, use_soft_target=False):
        """the cross-entropy of each depth's codes [D] (the reference logs it)"""
        B, H, W, D, _ = logits.shape
        logits = logits.reshape(-1, logits.shape[-1])
        if use_soft_target:
            tokenwise = _soft_target_cross_entropy(logits, targets.reshape(-1, targets.shape[-1]), reduction="none")
        else:
            tokenwise = torch.nn.functional.cross_entropy(logits, targets.reshape(-1), reduction="none")
        return tokenwise.reshape(-1, D).mean(dim=0)


# the engine's canvas limit (RQB200_CANVAS_MAX_CODES, include/rqb200.h): Ht * Wt * D, the codes of one batch row of a canvas
CANVAS_MAX_CODES = (1 << 31) - 1


def _chunk_bounds(B, mode, limit=256):
    """the batch chunks [(lo, hi)] of one native call each: the fast tier takes at most 256 batch rows per call (wgmma N <= 256), so
    a larger batch runs as equal chunks back to back.  limit: images per call (128 when each image takes two rows)"""
    n = max(1, -(-B // limit)) if mode == N.MODE_FAST else 1
    return [(i * B // n, (i + 1) * B // n) for i in range(n)]


def _rows(t, lo):
    """the rows of t from row lo on (a view), or None"""
    return None if t is None else t[lo:]


def _workspace(eng, need, dev):
    """a workspace of at least `need` bytes on dev: the engine slot's own (it holds the KV state between calls), replaced when too
    small; eng = None: one for this call only (forward / log_prob, whose activation rows would otherwise stay allocated)"""
    if eng is None:
        return torch.empty(need, dtype=torch.uint8, device=dev)
    if eng["ws"] is None or eng["ws"].numel() < need:
        eng["ws"] = torch.empty(need, dtype=torch.uint8, device=dev)
    return eng["ws"]


_REDUCE = {"mean": torch.mean, "sum": torch.sum, "none": lambda t: t}


def _soft_target_cross_entropy(logits, target, reduction="mean"):
    """cross-entropy of each row of `logits` [N,V] against a distribution `target` [N,V]: -(target * log p).sum(-1), reduced by
    `reduction`.  log p is the log-softmax the reference's soft-target loss uses (rqvae/optimizer/loss.py:68-84): logits shifted by
    their row maximum, with 1e-7 added to the sum of exponentials before the log."""
    if reduction not in _REDUCE:
        raise ValueError(reduction)
    shifted = logits - logits.amax(dim=-1, keepdim=True)
    log_p = shifted - (shifted.exp().sum(dim=-1, keepdim=True) + 1e-7).log()
    return _REDUCE[reduction]((target * log_p).sum(dim=-1).neg())
