"""RQVAE -- host-side mirror of rqvae/models/rqvae/rqvae.py:26-168 over the native conv engine.

Boundary kept (SURVEY.md section 8b): ``encode`` :80, ``decode`` :85, ``forward`` :74, ``get_codes`` :91, ``decode_code`` :105,
``get_code_emb_with_depth`` :146, ``decode_partial_code`` :150, ``get_recon_imgs`` :111, attribute ``code_shape`` and the
state_dict key layout.  ``precision``: 'exact' = fp32 FFMA kernels, 'fast' = fp16-operand / fp32-accumulate wgmma
implicit GEMM (the reference's own GPU decode runs cuDNN with TF32 allowed -- same 10-bit mantissa class)."""
import ctypes as C
import os

import torch
from torch import nn
from torch.nn import functional as F

from ... import _native as N
from ..interfaces import Stage1Model
from .modules import Decoder, Encoder, ResnetBlock
from .quantizations import RQBottleneck


class RQVAE(N.EngineCache, Stage1Model):
    def __init__(self, *, embed_dim=64, n_embed=512, decay=0.99, loss_type="mse", latent_loss_weight=0.25,
                 bottleneck_type="rq", ddconfig=None, checkpointing=False, **kwargs):
        super().__init__()
        assert loss_type in ("mse", "l1")
        ddconfig = dict(ddconfig)
        self.ddconfig = ddconfig
        self.encoder = Encoder(**ddconfig)
        self.decoder = Decoder(**ddconfig)
        if bottleneck_type != "rq":
            raise ValueError("invalid 'bottleneck_type' (must be 'rq')")
        self.quantizer = RQBottleneck(latent_shape=kwargs["latent_shape"], code_shape=kwargs["code_shape"], n_embed=n_embed,
                                      decay=decay, shared_codebook=kwargs["shared_codebook"],
                                      restart_unused_codes=kwargs["restart_unused_codes"])
        self.code_shape = kwargs["code_shape"]
        self.embed_dim = embed_dim
        self.quant_conv = nn.Conv2d(ddconfig["z_channels"], embed_dim, 1)
        self.post_quant_conv = nn.Conv2d(embed_dim, ddconfig["z_channels"], 1)
        self.loss_type, self.latent_loss_weight = loss_type, latent_loss_weight

    # ------------------------------------------------------------------ native engine plumbing
    _DESTROY = "rqb200_vae_destroy"

    def _engine(self, device):
        mode = self._mode()
        return self._cached_engine((str(device), mode), N.param_fingerprint(self), lambda: self._build_engine(mode))

    def _build_engine(self, mode):
        L = N.lib()
        dd = self.ddconfig
        cfg = N.VaeConfig()
        cfg.ch, cfg.n_levels, cfg.num_res_blocks = dd["ch"], len(dd["ch_mult"]), dd["num_res_blocks"]
        for i, m in enumerate(dd["ch_mult"]):
            cfg.ch_mult[i] = m
        cfg.n_attn_res = len(dd["attn_resolutions"])
        for i, r in enumerate(dd["attn_resolutions"]):
            cfg.attn_resolutions[i] = r
        cfg.resolution, cfg.z_channels, cfg.embed_dim = dd["resolution"], dd["z_channels"], self.embed_dim
        cfg.in_channels, cfg.out_ch = dd["in_channels"], dd["out_ch"]
        cfg.codebook_size, cfg.depth, cfg.mode = self.quantizer.n_embed[0], self.code_shape[-1], mode
        if os.environ.get("RQB200_GN_FUSE", "1") == "0":      # diagnostics: stand-alone GroupNorm statistics pass
            cfg.mode |= 0x100
        handle = L.rqb200_vae_create(C.byref(cfg))
        if not handle:
            raise N.NativeError("rqb200_vae_create: " + L.rqb200_last_error().decode())
        wdt = torch.float16 if mode == N.MODE_FAST else torch.float32
        keep = {}

        def reg(name, t):
            t = t.detach().contiguous()
            keep[name] = t
            N.check(L.rqb200_vae_set_tensor(handle, name.encode(), N.ptr(t), N.dtype_code(t), t.numel()), "vae_set_tensor")

        def reg_conv(name, w_oihw):
            """conv weight OIHW -> OHWI in the engine's dtype; fast tier: fp16 hi + lo halves (split-fp16 products)"""
            w = w_oihw.detach().permute(0, 2, 3, 1).contiguous().float()
            # fast tier: every conv but the encoder's Cin = 3 conv_in runs on the wgmma conv path
            if mode == N.MODE_FAST and not name.startswith("encoder.conv_in"):
                hi = w.to(torch.float16)
                reg(name, hi)
                reg(name + "_lo", (w - hi.float()).to(torch.float16))
            else:
                reg(name, w)          # exact tier, and the encoder's conv_in in every tier (fp32 FFMA kernels)

        sd = {k: v for k, v in self.state_dict().items()}
        for k, v in sd.items():
            if not (k.startswith("encoder.") or k.startswith("decoder.") or k.startswith("quant_conv") or
                    k.startswith("post_quant_conv")):
                continue
            N.require_cuda(v)
            if v.dim() == 4:                                   # conv weight OIHW -> OHWI in the engine's weight dtype
                if k.endswith((".q.weight", ".k.weight", ".v.weight")):
                    continue
                reg_conv(k, v)
            elif k.endswith((".q.bias", ".k.bias", ".v.bias")):
                continue
            else:
                reg(k, v.float())
        for k in [k for k in sd if k.endswith(".q.weight")]:   # fused q|k|v 1x1 conv (layers.py:161-163)
            base = k[:-len(".q.weight")]
            w = torch.cat([sd[base + ".q.weight"], sd[base + ".k.weight"], sd[base + ".v.weight"]], 0)
            b = torch.cat([sd[base + ".q.bias"], sd[base + ".k.bias"], sd[base + ".v.bias"]], 0)
            reg_conv(base + ".qkv.weight", w)
            reg(base + ".qkv.bias", b.float())
        tabs = self.quantizer._tables()
        if isinstance(tabs, list):                             # one table per depth (shared_codebook=False)
            for d, t in enumerate(tabs):
                reg("codebook.%d" % d, t.float())
        else:
            reg("codebook", tabs.float())
        N.check(L.rqb200_vae_finalize(handle), "vae_finalize")
        return {"handle": handle, "keep": keep, "ws": None}

    def _run(self, fn_name, x, out_shape, hw, ext=()):
        """one native call on x -> out_shape.  hw: the call's pixel extent (H, W); ext: the extent arguments the *_hw entry points
        take after B"""
        N.require_cuda(x)
        eng = self._engine(x.device)
        B = x.shape[0]
        out = torch.empty(out_shape, dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            # no refusal message: only decode_code of an empty batch gets a zero size, and the engine's own call reports it
            ws = N.workspace(eng, N.lib().rqb200_vae_workspace_bytes_hw(eng["handle"], B, *hw), x.device)
            fn = getattr(N.lib(), fn_name)
            N.check(fn(eng["handle"], N.ptr(x), B, *ext, N.ptr(out), N.ptr(ws), ws.numel(), N.stream_ptr(x.device)), fn_name)
        self.last_launches = N.lib().rqb200_vae_last_launches(eng["handle"])
        N.launch_count["total"] += self.last_launches
        return out

    # ------------------------------------------------------------------ reference surface
    def downsample_factor(self):
        """f = 2^(len(ch_mult) - 1): an image of H x W pixels has an H/f x W/f latent"""
        return 2 ** (len(self.ddconfig["ch_mult"]) - 1)

    def _check_input(self, t, channels, what, f):
        """ValueError unless t is [B, ..] 4-D with `channels` at dim 1 (what == 'image', NCHW) or dim 3 (NHWC latent) and both spatial
        extents positive multiples of f -> (H, W)"""
        if t.dim() != 4:
            raise ValueError("RQVAE: the %s must be 4-D, got shape %s" % (what, tuple(t.shape)))
        nchw = what == "image"
        c = t.shape[1] if nchw else t.shape[3]
        H, W = (t.shape[2], t.shape[3]) if nchw else (t.shape[1], t.shape[2])
        if c != channels:
            raise ValueError("RQVAE: the %s has %d channels, the model takes %d (shape %s)" % (what, c, channels, tuple(t.shape)))
        if t.shape[0] < 1 or H < 1 or W < 1 or H % f or W % f:
            raise ValueError("RQVAE: the %s's extent %d x %d is not a positive multiple of %d (shape %s)" % (what, H, W, f, tuple(t.shape)))
        return H, W

    @torch.no_grad()
    def encode(self, x):
        """rqvae.py:80-83: [B,in_channels,H,W] -> z_e [B,H/f,W/f,embed_dim] NHWC contiguous, at any H, W the downsampling
        factor f = downsample_factor() divides (the reference's encoder is fully convolutional)"""
        f = self.downsample_factor()
        H, W = self._check_input(x, self.ddconfig["in_channels"], "image", f)
        x = x.float().contiguous()
        return self._run("rqb200_vae_encode_hw", x, (x.shape[0], H // f, W // f, self.embed_dim), (H, W), (H, W))

    @torch.no_grad()
    def decode(self, z_q):
        """rqvae.py:85-89: z_q [B,h,w,embed_dim] NHWC -> [B,out_ch,h f,w f], at any latent extent h, w >= 1.  A code map of
        another grid than code_shape decodes as decode(quantizer.embed_code_with_depth(code, True)[0].sum(-2)), as in the
        reference (decode_code itself keeps the configured code_shape)."""
        h, w = self._check_input(z_q, self.embed_dim, "latent", 1)
        z_q = z_q.float().contiguous()
        f = self.downsample_factor()
        return self._run("rqb200_vae_decode_hw", z_q, (z_q.shape[0], self.ddconfig["out_ch"], h * f, w * f), (h * f, w * f), (h, w))

    @torch.no_grad()
    def forward(self, xs):
        """rqvae.py:74-78 (inference; gradients are out of scope)"""
        z_e = self.encode(xs)
        z_q, quant_loss, code = self.quantizer(z_e)
        return self.decode(z_q), quant_loss, code

    @torch.no_grad()
    def get_codes(self, xs):
        z_e = self.encode(xs)
        _, codes = self.quantizer.quantize(self.quantizer.to_code_shape(z_e))
        return codes

    @torch.no_grad()
    def decode_code(self, code):
        """rqvae.py:105-109 -- embed_code + decode in one native call"""
        assert code.shape[1:] == torch.Size(self.code_shape)
        code = code.to(torch.int64).contiguous()
        dd = self.ddconfig
        if tuple(self.quantizer.shape_divisor[:2]) != (1, 1):
            return self.decode(self.quantizer.embed_code(code))
        R = dd["resolution"]
        return self._run("rqb200_vae_decode_code", code, (code.shape[0], dd["out_ch"], R, R), (R, R))

    def get_recon_imgs(self, xs_real, xs_recon):
        return xs_real * 0.5 + 0.5, torch.clamp(xs_recon * 0.5 + 0.5, 0, 1)

    def compute_loss(self, out, quant_loss, code, xs=None, valid=False):
        """rqvae.py:119-141 (torch glue; evaluation only)"""
        loss_recon = F.mse_loss(out, xs) if self.loss_type == "mse" else F.l1_loss(out, xs)
        loss_latent = quant_loss
        if valid:
            loss_recon = loss_recon * xs.shape[0] * xs.shape[1]
            loss_latent = loss_latent * xs.shape[0]
        return {"loss_total": loss_recon + self.latent_loss_weight * loss_latent, "loss_recon": loss_recon,
                "loss_latent": loss_latent, "codes": [code]}

    def get_last_layer(self):
        return self.decoder.conv_out.weight

    @torch.no_grad()
    def get_code_emb_with_depth(self, code):
        return self.quantizer.embed_code_with_depth(code)

    @torch.no_grad()
    def decode_partial_code(self, code, code_idx, decode_type="select"):
        return self.decode(self.quantizer.embed_partial_code(code, code_idx, decode_type))

    @torch.no_grad()
    def forward_partial_code(self, xs, code_idx, decode_type="select"):
        return self.decode_partial_code(self.get_codes(xs), code_idx, decode_type)

    @torch.no_grad()
    def get_soft_codes(self, xs, temp=1.0, stochastic=False):
        """rqvae.py:97-103"""
        z_e = self.encode(xs)
        return self.quantizer.get_soft_codes(z_e, temp=temp, stochastic=stochastic)
