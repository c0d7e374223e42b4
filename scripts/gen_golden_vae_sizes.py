#!/usr/bin/env python
"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/vaesz.pt from the UNMODIFIED reference RQVAE, run on images of other sizes than
its configured resolution (the reference's encoder and decoder are fully convolutional; which levels carry an AttnBlock is fixed
by the configured resolution at construction).

    tiny            f = 4:  8x8, 12x20, 32x16 (B 2)
    tiny_attn_mid   f = 8:  24x40 (B 2)
    imagenet        f = 32: 384x256 and 512x512 (B 1)
    f8              the f8 RQ-VAE of scripts/bench_shapes.py (ch_mult 1,2,2,4, attention at 32, 32x32x4 codes): 384x512 (B 1), a
                    48x64 latent = 3072 tokens at the attention of every decoder level 0 block

Per size: z_e = encode(x) (f8: every 4th latent row and column), forward(x)'s codes and reconstruction, and the decode of a seeded
code map of the size's latent grid through the reference's own route for such a map,
decode(quantizer.embed_code_with_depth(code, True)[0].sum(-2)); pixels every `stride`-th row and column (1, 8 or 16), with the
full L2.  About 0.9 MB.

Needs the reference tree (oracle/ref_loader.py):   python scripts/gen_golden_vae_sizes.py
Same protocol as oracle/gen_golden.py: weights from oracle/synth.py seeds (synth_state_dict of the model's own shapes), inputs from
synth.randn_seeded / randint_seeded; the file stores seeds and the reference's outputs.
"""
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_loader as R                                  # noqa: E402
from oracle import synth                                            # noqa: E402
from oracle.zoo import VAE_ZOO                                      # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "vaesz.pt")
F8 = dict(K=16384, code_shape=(32, 32, 4), ch_mult=(1, 2, 2, 4), attn_resolutions=(32,))
PLAN = {
    # name: (vae kwargs, B, [(H, W, pixel stride), ...], latent stride of the stored z_e)
    "tiny": (VAE_ZOO["tiny"], 2, [(8, 8, 1), (12, 20, 1), (32, 16, 1)], 1),
    "tiny_attn_mid": (VAE_ZOO["tiny_attn_mid"], 2, [(24, 40, 1)], 1),
    "imagenet": (VAE_ZOO["imagenet"], 1, [(384, 256, 8), (512, 512, 16)], 1),
    "f8": (F8, 1, [(384, 512, 16)], 4),
}
SEEDS = dict(weight_seed=31, x_seed=32, codes_seed=33)


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    ns = R.load_reference()
    res = {}
    for name, (zkw, B, sizes, zst) in PLAN.items():
        kw = R.vae_kwargs(**zkw)
        model = ns.RQVAE(**kw).eval()
        model.load_state_dict(synth.synth_state_dict(synth.shapes_of(model.state_dict()), SEEDS["weight_seed"]))
        f = 2 ** (len(kw["ddconfig"]["ch_mult"]) - 1)
        D = kw["code_shape"][-1]
        cases = []
        for (H, W, st) in sizes:
            t0 = time.time()
            x = synth.randn_seeded((B, 3, H, W), SEEDS["x_seed"] + H * 1000 + W)
            code = synth.randint_seeded(0, kw["n_embed"], (B, H // f, W // f, D), SEEDS["codes_seed"] + H * 1000 + W)
            with torch.no_grad():
                z_e = model.encode(x)
                recon, _, codes_fwd = model(x)
                pix = model.decode(model.quantizer.embed_code_with_depth(code, True)[0].sum(-2))
            assert z_e.shape == (B, H // f, W // f, kw["embed_dim"]) and pix.shape == (B, 3, H, W)
            cases.append(dict(H=H, W=W, B=B, stride=st, x_seed=SEEDS["x_seed"] + H * 1000 + W, codes_seed=SEEDS["codes_seed"] + H * 1000 + W,
                              z_e_sub=z_e[:, ::zst, ::zst].clone(), codes_fwd=codes_fwd.to(torch.int16),
                              pixels_sub=pix[:, :, ::st, ::st].clone(), pixels_l2=float(pix.double().pow(2).sum().sqrt()),
                              recon_sub=recon[:, :, ::st, ::st].clone(), recon_l2=float(recon.double().pow(2).sum().sqrt())))
            print("  vaesz %-14s %4dx%-4d %.1fs" % (name, H, W, time.time() - t0), flush=True)
        res[name] = dict(vae=dict(zkw), weight_seed=SEEDS["weight_seed"], z_stride=zst, cases=cases)
        del model
    torch.save(res, OUT)
    print("wrote %s (%.0f KB)" % (OUT, os.path.getsize(OUT) / 1024))


if __name__ == "__main__":
    main()
