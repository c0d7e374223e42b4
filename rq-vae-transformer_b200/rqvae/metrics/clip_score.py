"""CLIP score -- the reference's rqvae/metrics/clip_score.py surface over the native CLIP engine (csrc/clip_engine.cu).

``get_clip()`` returns ``(model_clip, preprocess_clip)`` as ``clip.load("ViT-B/32")`` does, from the weight file ``clip.load`` caches
(``~/.cache/clip/ViT-B-32.pt``); nothing is ever downloaded.  ``clip_score(pixels, texts, model_clip, preprocess_clip)`` gives the
reference's per-pair cosine of image and caption features, with preprocessing, both encoders and the cosine on the GPU: no PIL round
trip.  The preprocessing is bit-exact to the reference's route -- ``(pixel * 255).astype(np.uint8)``, ``Image.fromarray``, Pillow's
bicubic resize of the shorter side to the model's resolution, centre crop, ``ToTensor``, ``Normalize`` -- for pixels in [0, 1].
Pixels outside [0, 1] are clamped first; there numpy's cast to uint8 is undefined, so the reference has no defined value to match.

``tokenize`` is ``clip.tokenize``: CLIP's byte-level BPE over ``bpe_simple_vocab_16e6.txt.gz`` with the start / end tokens 49406 /
49407 and zero padding.  Text is cleaned with ``ftfy.fix_text`` when ftfy is installed; without it, text that ftfy would repair
(curly quotes, mojibake) may tokenize differently, and one warning says so.

Tiers (``CLIP.precision``, else ``RQB200_PRECISION``): 'exact' (the default) runs fp32 FFMA throughout; 'fast' runs the transformer
GEMMs with fp16 operands and fp32 accumulation.  OpenAI's released weights are stored in fp16, so the fast tier's fp16 weight copies
of them are exact; its error comes from rounding activations to fp16.  ResNet CLIPs are not supported."""
import ctypes as C
import functools
import gzip
import html
import importlib.util
import logging
import os
from collections import OrderedDict

import numpy as np
import torch
from torch import nn

from .. import _native as N

log = logging.getLogger(__name__)

PREPROCESS = 1                         # rqb200_clip_encode_image flag: pixels in [0, 1] at any size
CHUNK = 1024                           # images or captions per native call: bounds the workspace
MEAN = (0.48145466, 0.4578275, 0.40821073)
STD = (0.26862954, 0.26130258, 0.27577711)
SOT, EOT = 49406, 49407


# ---------------------------------------------------------------------------------------------------------------- tokenizer
def _byte_symbols():
    """the 256 bytes -> printable unicode characters, in vocabulary order: the bytes that are printable latin-1 keep their own
    character and come first; the rest follow in byte order as chr(256 + i)"""
    keep = list(range(ord("!"), ord("~") + 1)) + list(range(ord("\xa1"), ord("\xac") + 1)) + list(range(ord("\xae"), ord("\xff") + 1))
    rest = [b for b in range(256) if b not in keep]
    return dict([(b, chr(b)) for b in keep] + [(b, chr(256 + i)) for i, b in enumerate(rest)])


def _ftfy():
    try:
        import ftfy
        return ftfy.fix_text
    except ImportError:
        log.warning("rqvae.metrics.clip_score: ftfy is not installed; captions that ftfy would repair (curly quotes, mojibake) may "
                    "tokenize differently from clip.tokenize")
        return lambda s: s


class BpeTokenizer:
    """CLIP's byte-level BPE tokenizer over a bpe_simple_vocab_16e6.txt.gz merge list"""

    def __init__(self, bpe_path):
        import regex
        with gzip.open(bpe_path) as f:
            lines = f.read().decode("utf-8").split("\n")
        merges = [tuple(line.split()) for line in lines[1:49152 - 256 - 2 + 1]]
        self.byte_sym = _byte_symbols()
        syms = list(self.byte_sym.values())
        vocab = syms + [s + "</w>" for s in syms] + ["".join(m) for m in merges] + ["<|startoftext|>", "<|endoftext|>"]
        self.ids = {s: i for i, s in enumerate(vocab)}
        self.rank = {m: i for i, m in enumerate(merges)}
        self.pattern = regex.compile(r"""<\|startoftext\|>|<\|endoftext\|>|'s|'t|'re|'ve|'m|'ll|'d|[\p{L}]+|[\p{N}]|[^\s\p{L}\p{N}]+""",
                                     regex.IGNORECASE)
        self.ws = regex.compile(r"\s+")
        self.fix_text = _ftfy()
        self.sot, self.eot = self.ids["<|startoftext|>"], self.ids["<|endoftext|>"]

    @functools.lru_cache(maxsize=1 << 16)
    def _merge(self, word):
        """the BPE symbols of one pre-token (already mapped to byte symbols): repeatedly join the adjacent pair of lowest rank"""
        if word in ("<|startoftext|>", "<|endoftext|>"):
            return (word,)
        parts = list(word[:-1]) + [word[-1] + "</w>"]
        while len(parts) > 1:
            ranked = [(self.rank.get((a, b), None), a, b) for a, b in zip(parts, parts[1:])]
            ranked = [r for r in ranked if r[0] is not None]
            if not ranked:
                break
            _, a, b = min(ranked)
            out, i = [], 0
            while i < len(parts):
                if i + 1 < len(parts) and parts[i] == a and parts[i + 1] == b:
                    out.append(a + b)
                    i += 2
                else:
                    out.append(parts[i])
                    i += 1
            parts = out
        return tuple(parts)

    def encode(self, text):
        text = html.unescape(html.unescape(self.fix_text(text))).strip()
        text = self.ws.sub(" ", text).strip().lower()
        ids = []
        for tok in self.pattern.findall(text):
            word = "".join(self.byte_sym[b] for b in tok.encode("utf-8"))
            ids.extend(self.ids[s] for s in self._merge(word))
        return ids


def default_bpe_path():
    """the vocab file the installed `clip` package ships, or None"""
    spec = importlib.util.find_spec("clip")
    if spec is None or spec.origin is None:
        return None
    return os.path.join(os.path.dirname(spec.origin), "bpe_simple_vocab_16e6.txt.gz")


@functools.lru_cache(maxsize=4)
def _tokenizer(bpe_path):
    return BpeTokenizer(bpe_path)


def get_tokenizer(bpe_path=None):
    path = bpe_path or default_bpe_path()
    if path is None or not os.path.isfile(path):
        raise FileNotFoundError("rqb200: CLIP's BPE vocabulary %s is not there; pass bpe_path= (the file is "
                                "bpe_simple_vocab_16e6.txt.gz of OpenAI's clip package)" % (path or "(no clip package installed)"))
    return _tokenizer(os.path.abspath(path))


def tokenize(texts, context_length=77, truncate=False, bpe_path=None):
    """clip.tokenize: [len(texts), context_length] int64 of SOT + BPE ids + EOT, zero-padded.  A text longer than the context raises
    RuntimeError unless truncate, which keeps the first context_length ids with EOT last."""
    tok = get_tokenizer(bpe_path)
    if isinstance(texts, str):
        texts = [texts]
    out = torch.zeros(len(texts), context_length, dtype=torch.long)
    for i, text in enumerate(texts):
        ids = [tok.sot] + tok.encode(text) + [tok.eot]
        if len(ids) > context_length:
            if not truncate:
                raise RuntimeError(f"Input {texts[i]} is too long for context length {context_length}")
            ids = ids[:context_length]
            ids[-1] = tok.eot
        out[i, :len(ids)] = torch.tensor(ids)
    return out


# ---------------------------------------------------------------------------------------------------------------- preprocessing
def resized_extent(H, W, R):
    """torchvision Resize(R) on an H x W image: the shorter side becomes R, the longer int(R * long / short)"""
    return (int(R * H / W), R) if W <= H else (R, int(R * W / H))


def crop_offsets(Hr, Wr, R):
    """torchvision CenterCrop(R): (top, left) = int(round((n - R) / 2)), Python's round (half to even)"""
    return int(round((Hr - R) / 2.0)), int(round((Wr - R) / 2.0))


class ClipPreprocess:
    """the reference's preprocess_clip for PIL images, restated on the host: Pillow's bicubic resize of the shorter side to R,
    centre crop, ToTensor, Normalize with CLIP's mean and std.  [3, R, R] fp32."""

    def __init__(self, n_px):
        self.n_px = n_px

    def __call__(self, image):
        from PIL import Image
        R = self.n_px
        image = image.convert("RGB")
        W, H = image.size
        Hr, Wr = resized_extent(H, W, R)
        if (Wr, Hr) != (W, H):
            image = image.resize((Wr, Hr), Image.BICUBIC)
        top, left = crop_offsets(Hr, Wr, R)
        u = np.array(image, dtype=np.uint8)[top:top + R, left:left + R]
        x = torch.from_numpy(np.ascontiguousarray(u)).permute(2, 0, 1).float().div(255)
        mean = torch.as_tensor(MEAN, dtype=torch.float32)[:, None, None]
        std = torch.as_tensor(STD, dtype=torch.float32)[:, None, None]
        return x.sub(mean).div(std)


# ---------------------------------------------------------------------------------------------------------------- model
class _Holder(nn.Module):
    def forward(self, *a, **k):
        raise RuntimeError("rqb200: parameter holder -- compute runs in the native CLIP engine (CLIP.encode_image / encode_text)")


class QuickGELU(_Holder):
    pass


class ResidualAttentionBlock(_Holder):
    def __init__(self, d_model, n_head):
        super().__init__()
        self.attn = nn.MultiheadAttention(d_model, n_head)
        self.ln_1 = nn.LayerNorm(d_model)
        self.mlp = nn.Sequential(OrderedDict([("c_fc", nn.Linear(d_model, d_model * 4)), ("gelu", QuickGELU()),
                                              ("c_proj", nn.Linear(d_model * 4, d_model))]))
        self.ln_2 = nn.LayerNorm(d_model)


class Transformer(_Holder):
    def __init__(self, width, layers, heads):
        super().__init__()
        self.width, self.layers = width, layers
        self.resblocks = nn.Sequential(*[ResidualAttentionBlock(width, heads) for _ in range(layers)])


class VisionTransformer(_Holder):
    def __init__(self, input_resolution, patch_size, width, layers, heads, output_dim):
        super().__init__()
        self.input_resolution = input_resolution
        self.output_dim = output_dim
        self.conv1 = nn.Conv2d(3, width, kernel_size=patch_size, stride=patch_size, bias=False)
        scale = width ** -0.5
        self.class_embedding = nn.Parameter(scale * torch.randn(width))
        self.positional_embedding = nn.Parameter(scale * torch.randn((input_resolution // patch_size) ** 2 + 1, width))
        self.ln_pre = nn.LayerNorm(width)
        self.transformer = Transformer(width, layers, heads)
        self.ln_post = nn.LayerNorm(width)
        self.proj = nn.Parameter(scale * torch.randn(width, output_dim))


def clip_config_of(state_dict):
    """the geometry of a ViT CLIP state_dict, inferred as OpenAI's build_model infers it"""
    sd = state_dict
    if "visual.proj" not in sd:
        if any(k.startswith("visual.layer1") for k in sd):
            raise ValueError("rqb200: this is a ResNet CLIP (visual.layer1...); only ViT CLIPs are supported")
        raise ValueError("rqb200: not a CLIP ViT state_dict (no visual.proj)")
    vision_width = sd["visual.conv1.weight"].shape[0]
    cfg = dict(
        embed_dim=sd["text_projection"].shape[1],
        vision_width=vision_width,
        vision_layers=len([k for k in sd if k.startswith("visual.") and k.endswith(".attn.in_proj_weight")]),
        vision_patch_size=sd["visual.conv1.weight"].shape[-1],
        context_length=sd["positional_embedding"].shape[0],
        vocab_size=sd["token_embedding.weight"].shape[0],
        transformer_width=sd["ln_final.weight"].shape[0],
        transformer_layers=len(set(k.split(".")[2] for k in sd if k.startswith("transformer.resblocks"))))
    grid = round((sd["visual.positional_embedding"].shape[0] - 1) ** 0.5)
    cfg["image_resolution"] = cfg["vision_patch_size"] * grid
    for name in ("vision_width", "transformer_width"):
        if cfg[name] % 64:
            raise ValueError("rqb200: %s %d is not a multiple of 64; the engine's attention has head dim 64 (heads = width / 64)"
                             % (name, cfg[name]))
    return cfg


class CLIP(N.EngineCache, nn.Module):
    """OpenAI's CLIP (ViT image tower) with its state_dict layout; encode_image / encode_text run in the native engine.

    ``precision``: None (the default: RQB200_PRECISION, 'auto' = exact) or 'exact' runs fp32 FFMA; 'fast' runs the transformer GEMMs
    with fp16 operands (fp32 accumulate, residual stream, LayerNorm and softmax)."""

    def __init__(self, embed_dim, image_resolution, vision_layers, vision_width, vision_patch_size, context_length, vocab_size,
                 transformer_width, transformer_heads, transformer_layers):
        super().__init__()
        if not isinstance(vision_layers, int):
            raise ValueError("rqb200: ResNet CLIPs (vision_layers as a tuple) are not supported")
        for name, w in (("vision_width", vision_width), ("transformer_width", transformer_width)):
            if w % 64:
                raise ValueError("rqb200: %s %d is not a multiple of 64 (heads = width / 64)" % (name, w))
        self.context_length = context_length
        self.vocab_size = vocab_size
        self.visual = VisionTransformer(image_resolution, vision_patch_size, vision_width, vision_layers, vision_width // 64, embed_dim)
        self.transformer = Transformer(transformer_width, transformer_layers, transformer_heads)
        self.token_embedding = nn.Embedding(vocab_size, transformer_width)
        self.positional_embedding = nn.Parameter(torch.empty(context_length, transformer_width))
        self.ln_final = nn.LayerNorm(transformer_width)
        self.text_projection = nn.Parameter(torch.empty(transformer_width, embed_dim))
        self.logit_scale = nn.Parameter(torch.ones([]) * np.log(1 / 0.07))
        self.embed_dim = embed_dim

    # ------------------------------------------------------------------ native engine plumbing
    _DESTROY = "rqb200_clip_destroy"

    def _config(self, mode):
        v = self.visual
        return ClipConfig(v.conv1.weight.shape[0], len(v.transformer.resblocks), v.conv1.weight.shape[-1], v.input_resolution,
                          self.ln_final.weight.shape[0], len(self.transformer.resblocks), self.context_length, self.vocab_size,
                          self.embed_dim, mode)

    def _engine(self, device):
        mode = self._mode()
        return self._cached_engine((str(device), mode), N.param_fingerprint(self), lambda: N.plan_engine(
            _lib(), "clip", self._config(mode), {k: v for k, v in self.state_dict().items() if k != "logit_scale"}, device))

    @staticmethod
    def _workspace(eng, need, device):
        return N.workspace(eng, need, device, "rqb200_clip: the engine refused the input's extent")

    @torch.no_grad()
    def _encode_images(self, x, flags):
        N.require_cuda(x)
        x = x.float().contiguous()
        B, _, H, W = x.shape
        eng = self._engine(x.device)
        L = _lib()
        out = torch.empty(B, self.embed_dim, dtype=torch.float32, device=x.device)
        launches = 0
        with torch.cuda.device(x.device):
            for b0 in range(0, B, CHUNK):
                n = min(CHUNK, B - b0)
                ws = self._workspace(eng, L.rqb200_clip_workspace_bytes(eng["handle"], n, H, W, flags), x.device)
                N.check(L.rqb200_clip_encode_image(eng["handle"], N.ptr(x[b0:b0 + n]), n, H, W, flags, N.ptr(out[b0:b0 + n]), N.ptr(ws),
                                                   ws.numel(), N.stream_ptr(x.device)), "clip_encode_image")
                launches += L.rqb200_clip_last_launches(eng["handle"])
        self.last_launches = launches
        N.launch_count["total"] += launches
        return out

    def encode_image(self, image):
        """image features [B, embed_dim] of an already-normalised [B, 3, R, R] batch (what preprocess_clip produces)"""
        R = self.visual.input_resolution
        if not isinstance(image, torch.Tensor) or image.dim() != 4 or tuple(image.shape[1:]) != (3, R, R) or image.shape[0] < 1:
            raise ValueError("CLIP.encode_image: need a [B, 3, %d, %d] tensor, got %s"
                             % (R, R, tuple(image.shape) if isinstance(image, torch.Tensor) else type(image).__name__))
        return self._encode_images(image, 0)

    def encode_pixels(self, pixels):
        """image features of [B, 3, H, W] pixels in [0, 1] at any size: the reference's preprocessing, fused into the engine"""
        _check_pixels(pixels)
        return self._encode_images(pixels, PREPROCESS)

    @torch.no_grad()
    def encode_text(self, text):
        """text features [N, embed_dim] of tokens [N, context_length] (tokenize's output), pooled at the end-of-text token"""
        tokens = self._check_tokens(text)
        N.require_cuda(tokens)
        tokens = tokens.long().contiguous()
        eng = self._engine(tokens.device)
        L = _lib()
        n_all = tokens.shape[0]
        out = torch.empty(n_all, self.embed_dim, dtype=torch.float32, device=tokens.device)
        launches = 0
        with torch.cuda.device(tokens.device):
            for b0 in range(0, n_all, CHUNK):
                n = min(CHUNK, n_all - b0)
                ws = self._workspace(eng, L.rqb200_clip_text_workspace_bytes(eng["handle"], n), tokens.device)
                N.check(L.rqb200_clip_encode_text(eng["handle"], N.ptr(tokens[b0:b0 + n]), n, N.ptr(out[b0:b0 + n]), N.ptr(ws), ws.numel(),
                                                  N.stream_ptr(tokens.device)), "clip_encode_text")
                launches += L.rqb200_clip_last_launches(eng["handle"])
        self.last_launches = launches
        N.launch_count["total"] += launches
        return out

    def _check_tokens(self, tokens):
        if not isinstance(tokens, torch.Tensor) or tokens.dim() != 2 or tokens.shape[1] != self.context_length or tokens.shape[0] < 1:
            raise ValueError("CLIP.encode_text: need an [N, %d] integer tensor, got %s"
                             % (self.context_length, tuple(tokens.shape) if isinstance(tokens, torch.Tensor) else type(tokens).__name__))
        if tokens.dtype.is_floating_point or tokens.dtype == torch.bool:
            raise ValueError("CLIP.encode_text: token ids must be integers, got %s" % tokens.dtype)
        lo, hi = int(tokens.min()), int(tokens.max())
        if lo < 0 or hi >= self.vocab_size:
            raise ValueError("CLIP.encode_text: token ids must lie in [0, %d), got [%d, %d]" % (self.vocab_size, lo, hi))
        return tokens


def _check_pixels(pixels):
    if not isinstance(pixels, torch.Tensor) or pixels.dim() != 4:
        raise ValueError("clip_score: pixels must be a 4-D [B, 3, H, W] tensor, got %s"
                         % (str(tuple(pixels.shape)) if isinstance(pixels, torch.Tensor) else type(pixels).__name__))
    B, c, H, W = pixels.shape
    if c != 3:
        raise ValueError("clip_score: pixels have %d channels, CLIP takes 3 (shape %s)" % (c, tuple(pixels.shape)))
    if B < 1 or H < 1 or W < 1:
        raise ValueError("clip_score: empty input, shape %s" % (tuple(pixels.shape),))


def build_model(state_dict):
    """a CLIP with the geometry of a ViT CLIP state_dict (OpenAI's build_model), its weights loaded in fp32"""
    sd = {k: v for k, v in state_dict.items() if k not in ("input_resolution", "context_length", "vocab_size")}
    cfg = clip_config_of(sd)
    model = CLIP(cfg["embed_dim"], cfg["image_resolution"], cfg["vision_layers"], cfg["vision_width"], cfg["vision_patch_size"],
                 cfg["context_length"], cfg["vocab_size"], cfg["transformer_width"], cfg["transformer_width"] // 64,
                 cfg["transformer_layers"])
    model.load_state_dict({k: v.float() for k, v in sd.items()})
    return model.eval()


def clip_weights_path(name="ViT-B/32"):
    """where clip.load caches a model's weights: ~/.cache/clip/<name with '/' and '@' as '-'>.pt"""
    return os.path.join(os.path.expanduser("~/.cache/clip"), name.replace("/", "-").replace("@", "-") + ".pt")


def load_state_dict_file(path):
    """the state_dict of clip.load's TorchScript archive, or of a plain state_dict file"""
    try:
        return torch.jit.load(path, map_location="cpu").state_dict()
    except RuntimeError:
        return torch.load(path, map_location="cpu", weights_only=True)


def get_clip(name="ViT-B/32", path=None, bpe_path=None):
    """(model_clip, preprocess_clip) as the reference's get_clip returns them, from the weight file clip.load caches (or `path`).  Never
    downloads: a missing weight file or vocabulary raises FileNotFoundError naming the path looked at.  The model stays on the CPU
    until moved, as clip.load(..., device='cpu') leaves it."""
    path = path or clip_weights_path(name)
    if not os.path.isfile(path):
        raise FileNotFoundError("rqb200: the CLIP weights %s are not there.  This package never downloads; copy them from another "
                                "machine's clip cache (clip.load puts them there) or pass path=" % path)
    get_tokenizer(bpe_path)
    model = build_model(load_state_dict_file(path))
    model.bpe_path = bpe_path
    return model, ClipPreprocess(model.visual.input_resolution)


@torch.no_grad()
def clip_score(pixels, texts, model_clip, preprocess_clip, device=torch.device('cuda')):
    """per-pair cosine of CLIP image and caption features (the reference's clip_score).  pixels [B, 3, H, W] in [0, 1]; texts a list of
    B captions or a [B, context_length] token tensor.  Returns F.cosine_similarity(...).squeeze(): [B], or 0-d for one image."""
    _check_pixels(pixels)
    B = pixels.shape[0]
    if isinstance(texts, torch.Tensor):
        tokens = texts
    else:
        texts = [texts] if isinstance(texts, str) else list(texts)
        if len(texts) != B:
            raise ValueError("clip_score: %d captions for %d images" % (len(texts), B))
        tokens = tokenize(texts, model_clip.context_length, bpe_path=getattr(model_clip, "bpe_path", None))
    if tokens.dim() != 2 or tokens.shape[0] != B:
        raise ValueError("clip_score: token tensor of shape %s for %d images" % (tuple(tokens.shape), B))
    model_clip._check_tokens(tokens)
    if not pixels.is_cuda:
        pixels = pixels.to(device)
    tokens = tokens.to(pixels.device)
    img = model_clip.encode_pixels(pixels)
    txt = model_clip.encode_text(tokens)
    return cosine_similarity(img, txt).squeeze()


def cosine_similarity(a, b):
    """F.cosine_similarity(a, b) of [n, d] fp32 rows on the device (eps 1e-8), natively"""
    N.require_cuda(a, b)
    a, b = a.float().contiguous(), b.float().contiguous()
    out = torch.empty(a.shape[0], dtype=torch.float32, device=a.device)
    with torch.cuda.device(a.device):
        N.check(_lib().rqb200_clip_cosine(N.ptr(a), N.ptr(b), a.shape[0], a.shape[1], N.ptr(out), N.stream_ptr(a.device)), "clip_cosine")
    return out


class ClipConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("vision_width", "vision_layers", "vision_patch", "vision_resolution", "text_width", "text_layers",
                                          "context_length", "vocab_size", "embed_dim", "mode")]


def _lib():
    L = N.lib()
    if not getattr(L, "_clip_bound", False):
        N.bind_plan_engine(L, "clip", ClipConfig)
        L.rqb200_clip_workspace_bytes.restype = C.c_size_t
        L.rqb200_clip_workspace_bytes.argtypes = [C.c_void_p] + [C.c_int] * 4
        L.rqb200_clip_text_workspace_bytes.restype = C.c_size_t
        L.rqb200_clip_text_workspace_bytes.argtypes = [C.c_void_p, C.c_int]
        L.rqb200_clip_encode_image.argtypes = [C.c_void_p, C.c_void_p] + [C.c_int] * 4 + [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
        L.rqb200_clip_encode_text.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
        L.rqb200_clip_cosine.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        L.rqb200_clip_resize_plan.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p]
        L.rqb200_dbg_clip_preprocess.argtypes = [C.c_void_p] + [C.c_int] * 4 + [C.c_void_p, C.c_void_p, C.c_void_p]
        L.rqb200_dbg_clip_attn.argtypes = [C.c_void_p, C.c_void_p] + [C.c_int] * 4 + [C.c_void_p]
        L.rqb200_dbg_clip_attn_flash.argtypes = [C.c_void_p, C.c_void_p] + [C.c_int] * 4 + [C.c_void_p]
        L._clip_bound = True
    return L


def resize_plan(H, W, R):
    """the engine's host resize plan: (resized H, resized W, crop top, crop left, horizontal taps, vertical taps); taps 0 = no pass"""
    out = (C.c_int32 * 6)()
    N.check(_lib().rqb200_clip_resize_plan(H, W, R, out), "clip_resize_plan")
    return tuple(out)
