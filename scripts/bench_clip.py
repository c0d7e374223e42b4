#!/usr/bin/env python
"""Throughput of CLIP scoring (ViT-B/32 geometry, synthetic weights: the rate does not depend on them) on one GPU.

Cases, one JSON line each with the card's name and power limit:
  - clip_score at B = 100 (the reference's batch size) on 256 x 256 pixels with 100 captions, exact and fast tiers: images/s, the
    image and text encoders' ms, and achieved TFLOP/s from the multiply-adds of the layer shapes (macs(), 2 FLOP each);
  - the torch restatement (tests/clip_oracle.py) on the same card, fp32 with TF32 off and fp16 autocast, on the preprocessed batch,
    timed in ABBA order with the native tiers;
  - the reference route's host cost: PIL preprocessing of the 100 images (ClipPreprocess, Pillow's resize) plus the copy to the device.

    python scripts/bench_clip.py [--batch 100] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "rq-vae-transformer_b200")]

from rqvae import _native as N                                       # noqa: E402
from rqvae.metrics import clip_score as CS                           # noqa: E402
from tests import clip_oracle as CO                                  # noqa: E402

# the tests' reduced merge list, which covers the captions below; scoring your own captions needs the full list (bpe_path or the
# installed clip package)
BPE = os.path.join(ROOT, "tests", "golden", "clip_bpe_subset.txt.gz")


def macs(G):
    """multiply-adds of one image and one caption: conv1, per block qkv + attention (q k^T and p v) + out_proj + MLP, projection"""
    def tower(E, L, T):
        return L * (T * (3 * E * E + E * E + 8 * E * E) + 2 * T * T * E)
    g = G["res"] // G["patch"]
    T = g * g + 1
    img = g * g * 3 * G["patch"] ** 2 * G["vw"] + tower(G["vw"], G["vl"], T) + G["vw"] * G["embed"]
    txt = tower(G["tw"], G["tl"], G["ctx"]) + G["tw"] * G["embed"]
    return img, txt


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
    except Exception:
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def timed(fn, reps):
    """ms per call over reps calls, between two device synchronisations"""
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=100)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_clip: needs a CUDA device")
    torch.set_grad_enabled(False)
    dev = "cuda:0"
    name, power = gpu_info()
    G = CO.GEOMS["b32"]
    mi, mt = macs(G)
    B = a.batch
    sd = CO.synth_state_dict("b32", 12)
    model = CS.build_model(sd).to(dev)
    model.bpe_path = BPE
    sd_dev = {k: v.to(dev) for k, v in sd.items()}
    pix = CO.pixels(1, B, 256, 256).to(dev)
    caps = ["a photo of a %s on a table" % w for w in ("cat", "dog", "cup", "book", "lamp")] * (B // 5 + 1)
    caps = caps[:B]
    tokens = CS.tokenize(caps, bpe_path=BPE).to(dev)
    pre = CS.ClipPreprocess(224)
    from PIL import Image
    host = (np.transpose(pix.cpu().numpy(), (0, 2, 3, 1)) * 255).astype(np.uint8)
    images = torch.stack([pre(Image.fromarray(h)) for h in host]).to(dev)
    base = dict(gpu=name, power_limit=power, model="ViT-B/32 geometry", batch=B, pixels="256x256", macs_per_image=mi, macs_per_caption=mt)

    def native(prec):
        def run():
            model.precision = prec
            return CS.clip_score(pix, tokens, model, pre)
        return run

    def torch_ref(dtype_case):
        def run():
            if dtype_case == "fp16_autocast":
                with torch.autocast("cuda", dtype=torch.float16):
                    fi = CO.encode_image(sd_dev, "b32", images, torch.float32)
                    ft = CO.encode_text(sd_dev, "b32", tokens, torch.float32)
            else:
                fi = CO.encode_image(sd_dev, "b32", images, torch.float32)
                ft = CO.encode_text(sd_dev, "b32", tokens, torch.float32)
            return torch.nn.functional.cosine_similarity(fi.float(), ft.float())
        return run

    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    cases = {"native_exact": native("exact"), "native_fast": native("fast"), "torch_fp32": torch_ref("fp32"),
             "torch_fp16_autocast": torch_ref("fp16_autocast")}
    for fn in cases.values():                                  # warm-up: modules, engines, workspaces, cuBLAS heuristics
        fn()
        fn()
    order = list(cases) + list(cases)[::-1]
    ms = {k: [] for k in cases}
    for _ in range(a.reps):
        for k in order:
            ms[k].append(timed(cases[k], 3))
    parts = {}
    for prec in ("exact", "fast"):
        model.precision = prec
        parts[prec] = (timed(lambda: model.encode_pixels(pix), 5), timed(lambda: model.encode_text(tokens), 5))
    for k, v in ms.items():
        t = float(np.median(v))
        rec = dict(base, case=k, ms=round(t, 3), images_per_s=round(B * 1e3 / t, 1),
                   tflops=round(2 * B * (mi + mt) / (t * 1e-3) / 1e12, 2), spread_ms=[round(min(v), 3), round(max(v), 3)])
        if k.startswith("native"):
            pi, pt = parts[k.split("_")[1]]
            rec.update(image_ms=round(pi, 3), text_ms=round(pt, 3))
        else:
            rec.update(note="torch restatement on the preprocessed batch (no preprocessing)")
        print(json.dumps(rec), flush=True)
    # the reference route's host cost: PIL preprocessing of B images + the copy to the device
    def host_route():
        arr = (np.transpose(pix.cpu().numpy(), (0, 2, 3, 1)) * 255).astype(np.uint8)
        torch.stack([pre(Image.fromarray(h)) for h in arr]).to(dev)
    host_route()
    t = float(np.median([timed(host_route, 1) for _ in range(3)]))
    print(json.dumps(dict(base, case="reference_host_preprocess", ms=round(t, 3), images_per_s=round(B * 1e3 / t, 1),
                          note="PIL resize + crop + normalise of B images on the host, plus the copy to the device")), flush=True)


if __name__ == "__main__":
    main()
