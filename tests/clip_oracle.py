"""float64 torch restatement of OpenAI's CLIP ViT (image and text towers, cosine), and the synthetic CLIP weights of the tests.

Geometries (GEOMS): `tiny` (width 128, 2 heads, 2 layers, patch 8 at 32^2), `b32` (ViT-B/32 exactly) and `b16n` (patch 16 at 224^2,
width 128: 197 tokens, four 64-query tiles).  Weights are rebuilt from a seed in OpenAI's state_dict layout and rounded to fp16, as
OpenAI's released weights are stored.  scripts/gen_golden_clip.py pins this restatement to transformers.CLIPModel in float64."""
import torch

GEOMS = {
    #        vision width, layers, patch, resolution, text width, layers, context, vocab, embed
    "tiny": dict(vw=128, vl=2, patch=8, res=32, tw=128, tl=2, ctx=77, vocab=49408, embed=128),
    "b32": dict(vw=768, vl=12, patch=32, res=224, tw=512, tl=12, ctx=77, vocab=49408, embed=512),
    "b16n": dict(vw=128, vl=2, patch=16, res=224, tw=128, tl=2, ctx=77, vocab=49408, embed=128),
}
MEAN = (0.48145466, 0.4578275, 0.40821073)
STD = (0.26862954, 0.26130258, 0.27577711)


def _block_shapes(pre, width, layers):
    out = []
    for i in range(layers):
        p = "%stransformer.resblocks.%d." % (pre, i)
        out += [(p + "ln_1.weight", (width,)), (p + "ln_1.bias", (width,)), (p + "attn.in_proj_weight", (3 * width, width)),
                (p + "attn.in_proj_bias", (3 * width,)), (p + "attn.out_proj.weight", (width, width)), (p + "attn.out_proj.bias", (width,)),
                (p + "ln_2.weight", (width,)), (p + "ln_2.bias", (width,)), (p + "mlp.c_fc.weight", (4 * width, width)),
                (p + "mlp.c_fc.bias", (4 * width,)), (p + "mlp.c_proj.weight", (width, 4 * width)), (p + "mlp.c_proj.bias", (width,))]
    return out


def shapes(g):
    G = GEOMS[g] if isinstance(g, str) else g
    vw, tw, P = G["vw"], G["tw"], G["patch"]
    n = (G["res"] // P) ** 2 + 1
    return ([("visual.class_embedding", (vw,)), ("visual.positional_embedding", (n, vw)), ("visual.proj", (vw, G["embed"])),
             ("visual.conv1.weight", (vw, 3, P, P)), ("visual.ln_pre.weight", (vw,)), ("visual.ln_pre.bias", (vw,))]
            + _block_shapes("visual.", vw, G["vl"])
            + [("visual.ln_post.weight", (vw,)), ("visual.ln_post.bias", (vw,)), ("text_projection", (tw, G["embed"])),
               ("positional_embedding", (G["ctx"], tw)), ("token_embedding.weight", (G["vocab"], tw)), ("logit_scale", ())]
            + _block_shapes("", tw, G["tl"]) + [("ln_final.weight", (tw,)), ("ln_final.bias", (tw,))])


def synth_state_dict(g, seed):
    """seeded weights in OpenAI's layout, fp16-representable, scaled so every layer's activations stay O(1)"""
    gen = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shp in shapes(g):
        r = torch.randn(shp, generator=gen, dtype=torch.float64)
        if k == "logit_scale":
            v = torch.tensor(4.6052)
        elif "ln_" in k and k.endswith(".weight"):
            v = 1.0 + 0.1 * r
        elif k.endswith("bias"):
            v = 0.05 * r
        elif k == "visual.conv1.weight":
            v = r / (shp[1] * shp[2] * shp[3]) ** 0.5
        elif len(shp) == 2 and ("weight" in k) and "embedding" not in k:
            v = r / shp[1] ** 0.5
        elif k in ("visual.proj", "text_projection"):
            v = r / shp[0] ** 0.5
        else:                                   # class / positional / token embeddings
            v = 0.5 * r
        sd[k] = v.half().float()
    return sd


def _ln(x, sd, p):
    return torch.nn.functional.layer_norm(x, x.shape[-1:], sd[p + ".weight"].to(x.dtype), sd[p + ".bias"].to(x.dtype), 1e-5)


def _blocks(x, sd, pre, layers, causal):
    """x [B, T, E] float64 through the residual blocks (nn.MultiheadAttention: q scaled by 1/sqrt(64) before q k^T)"""
    B, T, E = x.shape
    nh = E // 64
    mask = torch.full((T, T), float("-inf"), dtype=x.dtype, device=x.device).triu(1) if causal else None
    for i in range(layers):
        p = "%stransformer.resblocks.%d." % (pre, i)
        h = _ln(x, sd, p + "ln_1")
        qkv = h @ sd[p + "attn.in_proj_weight"].to(x.dtype).t() + sd[p + "attn.in_proj_bias"].to(x.dtype)
        q, k, v = qkv.split(E, -1)
        q, k, v = (t.reshape(B, T, nh, 64).transpose(1, 2) for t in (q, k, v))
        s = (q * 0.125) @ k.transpose(-1, -2)
        if mask is not None:
            s = s + mask
        a = (s.softmax(-1) @ v).transpose(1, 2).reshape(B, T, E)
        x = x + a @ sd[p + "attn.out_proj.weight"].to(x.dtype).t() + sd[p + "attn.out_proj.bias"].to(x.dtype)
        h = _ln(x, sd, p + "ln_2")
        h = h @ sd[p + "mlp.c_fc.weight"].to(x.dtype).t() + sd[p + "mlp.c_fc.bias"].to(x.dtype)
        h = h * torch.sigmoid(1.702 * h)
        x = x + h @ sd[p + "mlp.c_proj.weight"].to(x.dtype).t() + sd[p + "mlp.c_proj.bias"].to(x.dtype)
    return x


def encode_image(sd, g, images, dtype=torch.float64):
    """images [B, 3, R, R] already normalised -> [B, embed] (float64; another dtype on the GPU for the benchmark's torch restatement)"""
    G = GEOMS[g] if isinstance(g, str) else g
    x = torch.nn.functional.conv2d(images.to(dtype), sd["visual.conv1.weight"].to(dtype), stride=G["patch"])
    x = x.flatten(2).transpose(1, 2)
    cls = sd["visual.class_embedding"].to(x.dtype).expand(x.shape[0], 1, -1)
    x = torch.cat([cls, x], 1) + sd["visual.positional_embedding"].to(x.dtype)
    x = _ln(x, sd, "visual.ln_pre")
    x = _blocks(x, sd, "visual.", G["vl"], False)
    return _ln(x[:, 0], sd, "visual.ln_post") @ sd["visual.proj"].to(x.dtype)


def encode_text(sd, g, tokens, dtype=torch.float64):
    G = GEOMS[g] if isinstance(g, str) else g
    x = sd["token_embedding.weight"].to(dtype)[tokens] + sd["positional_embedding"].to(dtype)
    x = _blocks(x, sd, "", G["tl"], True)
    x = _ln(x, sd, "ln_final")
    return x[torch.arange(x.shape[0]), tokens.argmax(-1)] @ sd["text_projection"].to(x.dtype)


def cosine(a, b):
    return torch.nn.functional.cosine_similarity(a.double(), b.double())


def normalise(u8):
    """ToTensor + Normalize of a uint8 [.., 3, R, R] crop, in fp32 as torchvision computes it"""
    x = u8.float().div(255)
    mean = torch.as_tensor(MEAN, dtype=torch.float32)[:, None, None]
    std = torch.as_tensor(STD, dtype=torch.float32)[:, None, None]
    return x.sub(mean).div(std)


def pixels(seed, B, H, W):
    """seeded pixels in [0, 1) fp32 with the boundary values 0, 1 and k/255 written into the first row of every plane"""
    x = torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(seed))
    edge = torch.tensor([0.0, 1.0] + [k / 255.0 for k in range(0, 256, 5)], dtype=torch.float32)
    n = min(W, edge.numel())
    x[:, :, 0, :n] = edge[:n]
    return x
