#!/usr/bin/env python
"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/clip.pt on the CPU.

  - seeds of the synthetic CLIP weights of three geometries (tests/clip_oracle.GEOMS; the tests rebuild the weights from them);
  - per geometry, float64 image features of pixels run through the literal reference preprocessing (below), text features of five
    captions and their cosines, from tests/clip_oracle.py -- asserted here to match transformers.CLIPModel in float64, loaded with
    the same weights, to <= 1e-10;
  - for pixel inputs of 256^2, 224^2, 512^2, 384 x 256, 255 x 257, 200 x 300 and 64^2 (an upscale), with the boundary values 0, 1 and
    k/255 in fp32, the reference's route: (pixel * 255).astype(np.uint8), Image.fromarray, torchvision Resize(224, BICUBIC),
    CenterCrop(224), ToTensor, Normalize.  Stored are the SHA-256 digests of the uint8 crop's bytes and of the normalised fp32
    tensor's bytes (a bit-exact check at a few bytes per case), and the crop's first four rows for a readable failure message.
  - the token ids of the captions from the reference's own SimpleTokenizer (rqvae/txtimg_datasets/tokenizers/simple_tokenizer.py,
    loaded by file path, with an identity ftfy stub when ftfy is absent; every caption is one fix_text leaves unchanged).

It also writes tests/golden/clip_bpe_subset.txt.gz: CLIP's merge list (bpe_simple_vocab_16e6.txt.gz, 1.3 MB) with every merge that
the BPE of BPE_TEXTS never sees as a candidate pair replaced by a placeholder that matches nothing.  Every merge keeps its line, so
its rank and its token id are the full list's; on these texts the BPE takes the same steps and gives the same ids as with the full
list (asserted here against the reference tokenizer).  Users' tokenizers read the full list from the installed clip package.

Needs the reference tree:   python scripts/gen_golden_clip.py"""
import gzip
import hashlib
import importlib.util
import os
import sys
import types

import numpy as np
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_loader as R                                  # noqa: E402
from tests import clip_oracle as CO                                 # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "clip.pt")
BPE_OUT = os.path.join(ROOT, "tests", "golden", "clip_bpe_subset.txt.gz")
SEEDS = {"tiny": 11, "b32": 12, "b16n": 13}
PIX_CASES = [("256", 256, 256, 201), ("224", 224, 224, 202), ("512", 512, 512, 203), ("384x256", 384, 256, 204),
             ("255x257", 255, 257, 205), ("200x300", 200, 300, 206), ("64", 64, 64, 207)]
FEAT_PIX = {"tiny": (40, 48, 301), "b32": (256, 256, 302), "b16n": (256, 256, 303)}   # H, W, seed of the feature cases' pixels
CAPTIONS = [
    "a photo of a cat", "A dog running on the beach.", "two red apples on a wooden table", "an oil painting of a lighthouse at dusk",
    "the quick brown fox jumps over the lazy dog", "It's a sunny day, isn't it?", "a bowl of soup with 3 spoons",
    "A man riding a horse   in the mountains", "close-up of a bee on a sunflower", "Tom & Jerry &amp; friends",
    "a street sign that reads STOP", "city skyline at night, 2019", "a cup of coffee; latte art", "mountains reflected in a lake",
    "children playing soccer in a park", "a vintage car parked outside a diner", "we'll meet at 10:30 pm", "a plate of sushi",
    "snow-covered pine trees", "an astronaut riding a horse on mars", "a watercolor painting of a fox", "\tleading tab and trailing  ",
    "UPPER CASE CAPTION", "a cat sitting on a keyboard", "macro photo of a water droplet", "a red double-decker bus in london",
    "a glass of red wine", "fireworks over the harbour", "a hot air balloon festival", "a bicycle leaning against a brick wall",
    "a bowl of ramen, top view", "they're here", "you've got mail", "I'm fine", "a 3d render of a cube", "an old map of the world",
    "a koala sleeping in a tree", "a steaming cup of tea & a book", "a field of tulips in the netherlands", "a train crossing a bridge",
    "a cozy living room with a fireplace", "a robot painting a portrait", "graffiti on a concrete wall", "a lemon cut in half",
    "an aerial view of a winding river", "a chess board mid-game", "a frog on a lily pad", "neon lights in the rain",
    "a slice of pepperoni pizza",
    "a very long caption " + " ".join("word%d" % i for i in range(90)),
]


def sha256(t):
    return hashlib.sha256(t.contiguous().numpy().tobytes()).hexdigest()


def bpe_texts():
    """every text the tests and scripts/bench_clip.py tokenize with the subset list"""
    return (CAPTIONS + ["a photo of number %d" % i for i in range(1100)]
            + ["a photo of a %s on a table" % w for w in ("cat", "dog", "cup", "book", "lamp")] + ["a", "b", "x"])


def write_bpe_subset(tok, texts, path):
    """the merge list with the merges these texts' BPE never considers replaced by placeholders (same line = same rank and id)"""
    import regex
    from rqvae.metrics import clip_score as CS
    seen = set()
    for text in texts:
        for t in regex.findall(tok.pat, sys.modules["reftok.simple_tokenizer"].whitespace_clean(
                sys.modules["reftok.simple_tokenizer"].basic_clean(text)).lower()):
            word = "".join(tok.byte_encoder[b] for b in t.encode("utf-8"))
            parts = list(word[:-1]) + [word[-1] + "</w>"]
            while len(parts) > 1:                      # the reference's merge loop, recording every ranked candidate pair
                ranked = [(tok.bpe_ranks[p], p) for p in zip(parts, parts[1:]) if p in tok.bpe_ranks]
                seen.update(p for _, p in ranked)
                if not ranked:
                    break
                a, b = min(ranked)[1]
                out, i = [], 0
                while i < len(parts):
                    if i + 1 < len(parts) and parts[i] == a and parts[i + 1] == b:
                        out.append(a + b)
                        i += 2
                    else:
                        out.append(parts[i])
                        i += 1
                parts = out
    with gzip.open(os.path.join(os.path.dirname(sys.modules["reftok.utils"].__file__), "pretrained", "bpe_simple_vocab_16e6.txt.gz")) as f:
        lines = f.read().decode("utf-8").split("\n")
    keep = lines[:1]
    for i, line in enumerate(lines[1:49152 - 256 - 2 + 1]):
        keep.append(line if tuple(line.split()) in seen else "\u2400%x \u2401" % i)
    with open(path, "wb") as f:                       # mtime 0: the file is the same bytes on every run
        with gzip.GzipFile(fileobj=f, mode="wb", mtime=0) as g:
            g.write("\n".join(keep).encode("utf-8"))
    CS._tokenizer.cache_clear()
    for text in texts:
        want = [49406] + tok._encode(text) + [49407]
        got = CS.tokenize([text], context_length=max(77, len(want)), bpe_path=path)[0, :len(want)].tolist()
        assert got == want, text
    print("wrote", path, os.path.getsize(path), "bytes;", len(seen), "merges kept")


def reference_tokenizer():
    if importlib.util.find_spec("ftfy") is None:
        sys.modules["ftfy"] = types.SimpleNamespace(fix_text=lambda s: s)
    d = os.path.join(R.REFERENCE_ROOT, "rqvae", "txtimg_datasets", "tokenizers")
    pkg = types.ModuleType("reftok")
    pkg.__path__ = [d]
    sys.modules["reftok"] = pkg
    for name in ("utils", "simple_tokenizer"):
        spec = importlib.util.spec_from_file_location("reftok." + name, os.path.join(d, name + ".py"))
        m = importlib.util.module_from_spec(spec)
        sys.modules["reftok." + name] = m
        spec.loader.exec_module(m)
    return sys.modules["reftok.simple_tokenizer"].SimpleTokenizer()


def reference_crop(x):
    """the reference's route for one [3, H, W] fp32 image: uint8 cast, PIL, torchvision Resize(224, BICUBIC) + CenterCrop(224)"""
    from torchvision import transforms as T
    arr = np.transpose(x.numpy(), (1, 2, 0))
    img = Image.fromarray((arr * 255).astype(np.uint8))
    img = T.CenterCrop(224)(T.Resize(224, interpolation=T.InterpolationMode.BICUBIC)(img))
    return torch.from_numpy(np.asarray(img).copy()).permute(2, 0, 1).contiguous()


def reference_preprocess(x, R):
    from torchvision import transforms as T
    arr = np.transpose(x.numpy(), (1, 2, 0))
    img = Image.fromarray((arr * 255).astype(np.uint8))
    tf = T.Compose([T.Resize(R, interpolation=T.InterpolationMode.BICUBIC), T.CenterCrop(R), T.ToTensor(),
                    T.Normalize(CO.MEAN, CO.STD)])
    return tf(img)


def hf_features(sd, g, images, tokens):
    """transformers.CLIPModel in float64 with the same weights"""
    from transformers import CLIPConfig, CLIPModel
    G = CO.GEOMS[g]
    cfg = CLIPConfig(
        text_config=dict(hidden_size=G["tw"], intermediate_size=4 * G["tw"], num_attention_heads=G["tw"] // 64,
                         num_hidden_layers=G["tl"], max_position_embeddings=G["ctx"], vocab_size=G["vocab"], hidden_act="quick_gelu",
                         layer_norm_eps=1e-5, eos_token_id=2),
        vision_config=dict(hidden_size=G["vw"], intermediate_size=4 * G["vw"], num_attention_heads=G["vw"] // 64,
                           num_hidden_layers=G["vl"], image_size=G["res"], patch_size=G["patch"], hidden_act="quick_gelu",
                           layer_norm_eps=1e-5),
        projection_dim=G["embed"])
    m = CLIPModel(cfg).double().eval()
    hf = {}
    for tower, pre, L in (("vision_model", "visual.", G["vl"]), ("text_model", "", G["tl"])):
        for i in range(L):
            p, q = "%stransformer.resblocks.%d." % (pre, i), "%s.encoder.layers.%d." % (tower, i)
            w, b = sd[p + "attn.in_proj_weight"].chunk(3), sd[p + "attn.in_proj_bias"].chunk(3)
            for j, n in enumerate("qkv"):
                hf[q + "self_attn.%s_proj.weight" % n], hf[q + "self_attn.%s_proj.bias" % n] = w[j], b[j]
            for a, c in (("attn.out_proj", "self_attn.out_proj"), ("ln_1", "layer_norm1"), ("ln_2", "layer_norm2"),
                         ("mlp.c_fc", "mlp.fc1"), ("mlp.c_proj", "mlp.fc2")):
                hf[q + c + ".weight"], hf[q + c + ".bias"] = sd[p + a + ".weight"], sd[p + a + ".bias"]
    hf.update({
        "vision_model.embeddings.class_embedding": sd["visual.class_embedding"],
        "vision_model.embeddings.patch_embedding.weight": sd["visual.conv1.weight"],
        "vision_model.embeddings.position_embedding.weight": sd["visual.positional_embedding"],
        "vision_model.pre_layrnorm.weight": sd["visual.ln_pre.weight"], "vision_model.pre_layrnorm.bias": sd["visual.ln_pre.bias"],
        "vision_model.post_layernorm.weight": sd["visual.ln_post.weight"], "vision_model.post_layernorm.bias": sd["visual.ln_post.bias"],
        "visual_projection.weight": sd["visual.proj"].t(), "text_projection.weight": sd["text_projection"].t(),
        "text_model.embeddings.token_embedding.weight": sd["token_embedding.weight"],
        "text_model.embeddings.position_embedding.weight": sd["positional_embedding"],
        "text_model.final_layer_norm.weight": sd["ln_final.weight"], "text_model.final_layer_norm.bias": sd["ln_final.bias"],
        "logit_scale": sd["logit_scale"]})
    missing, _ = m.load_state_dict({k: v.double() for k, v in hf.items()}, strict=False)
    assert all("position_ids" in k for k in missing), missing
    with torch.no_grad():
        fi = m.get_image_features(pixel_values=images.double())
        ft = m.get_text_features(input_ids=tokens)
    fi = getattr(fi, "pooler_output", fi)
    ft = getattr(ft, "pooler_output", ft)
    return fi, ft


def main():
    tok = reference_tokenizer()
    sys.path.insert(0, os.path.join(ROOT, "rq-vae-transformer_b200"))
    write_bpe_subset(tok, bpe_texts(), BPE_OUT)
    ids = [[49406] + tok._encode(c) + [49407] for c in CAPTIONS]
    assert all(i[0] == 49406 for i in ids)
    golden = {"seeds": SEEDS, "captions": CAPTIONS, "caption_ids": ids, "pix": {}, "feat": {}}
    for name, H, W, seed in PIX_CASES:
        x = CO.pixels(seed, 1, H, W)
        u8 = reference_crop(x[0]).unsqueeze(0)
        nrm = reference_preprocess(x[0], 224).unsqueeze(0)
        assert torch.equal(nrm, CO.normalise(u8))
        golden["pix"][name] = dict(H=H, W=W, seed=seed, u8_sha256=sha256(u8), norm_sha256=sha256(nrm), u8_head=u8[:, :, :4].clone())
        print("pix", name, "ok")
    caps = [0, 1, 5, 9, 17]
    tokens = torch.zeros(len(caps), 77, dtype=torch.long)
    for r, c in enumerate(caps):
        tokens[r, :len(ids[c])] = torch.tensor(ids[c])
    for g, seed in SEEDS.items():
        sd = CO.synth_state_dict(g, seed)
        H, W, ps = FEAT_PIX[g]
        px = CO.pixels(ps, len(caps), H, W)
        images = torch.stack([reference_preprocess(px[i], CO.GEOMS[g]["res"]) for i in range(len(caps))])
        fi = CO.encode_image(sd, g, images)
        ft = CO.encode_text(sd, g, tokens)
        hi, ht = hf_features(sd, g, images, tokens)
        ei = float((hi - fi).abs().max() / fi.abs().max())
        et = float((ht - ft).abs().max() / ft.abs().max())
        print(g, "restatement vs transformers.CLIPModel (float64): image %.2e, text %.2e" % (ei, et))
        assert ei <= 1e-10 and et <= 1e-10
        golden["feat"][g] = dict(pix=(H, W, ps), caps=caps, tokens=tokens.clone(), image=fi, text=ft, cos=CO.cosine(fi, ft))
    torch.save(golden, OUT)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
