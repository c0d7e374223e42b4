#!/usr/bin/env python
"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/loss.pt from the UNMODIFIED reference: RQTransformer.compute_loss (hard and soft
targets), compute_cond_loss and compute_codebook_loss (hard and soft) on seeded logits (transformers.py:371-410; the soft targets go
through rqvae/optimizer/loss.py:68-84).

    cases   logits [B,H,W,D,V] at unit and large scale (one with -1e6 entries, the LogitMask value), hard targets, soft targets (a
            softmax of seeded values), cond logits [B,cond_len-1,vocab_cond] and conds [B,cond_len].  Inputs are stored beside the
            reference's outputs (a few KB each), so the CPU test needs neither the reference nor a generator protocol.

Needs the reference tree (oracle/ref_loader.py):   python scripts/gen_golden_loss.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_loader as R                                  # noqa: E402
from oracle import synth                                            # noqa: E402

# (block size, V, vocab_cond, cond_len, logit scale, seed)
CASES = {
    "unit": ((2, 2, 4), 64, 50, 4, 1.0, 1),
    "wide": ((2, 3, 2), 300, 17, 3, 8.0, 2),
    "masked": ((1, 2, 4), 128, 10, 2, 30.0, 3),
}
B = 3


def make_inputs(bs, V, vc, cl, scale, seed):
    logits = synth.randn_seeded((B, *bs, V), seed, scale)
    if scale >= 30.0:
        logits[..., V // 2:] = -1e6                                 # LogitMask's value on the upper half of the vocabulary
    targets = synth.randint_seeded(0, V // 2 if scale >= 30.0 else V, (B, *bs), seed + 100)
    soft = torch.softmax(synth.randn_seeded((B, *bs, V), seed + 200, 2.0), dim=-1)
    cond_logits = synth.randn_seeded((B, cl - 1, vc), seed + 300, scale if scale < 30.0 else 1.0)
    conds = synth.randint_seeded(0, vc, (B, cl), seed + 400)
    return dict(logits=logits, targets=targets, soft_targets=soft, cond_logits=cond_logits, conds=conds)


def main():
    torch.set_grad_enabled(False)
    ns = R.load_reference()
    out = {}
    for name, (bs, V, vc, cl, scale, seed) in CASES.items():
        model = ns.RQTransformer(R.transformer_cfg(128, 2, 1, 1, V, block_size=bs, vocab_cond=vc, cond_len=cl)).eval()
        x = make_inputs(bs, V, vc, cl, scale, seed)
        res = dict(
            loss=model.compute_loss(x["logits"], x["targets"]),
            loss_soft=model.compute_loss(x["logits"], x["soft_targets"], use_soft_target=True),
            cond_loss=model.compute_cond_loss(x["cond_logits"], x["conds"]),
            codebook_loss=model.compute_codebook_loss(x["logits"], x["targets"]),
            codebook_loss_soft=model.compute_codebook_loss(x["logits"], x["soft_targets"], use_soft_target=True),
        )
        out[name] = dict(block_size=bs, vocab=V, vocab_cond=vc, cond_len=cl, inputs=x,
                         ref={k: v.detach().clone() for k, v in res.items()})
        print("  %-7s %s" % (name, {k: [round(float(t), 5) for t in v.reshape(-1)] for k, v in res.items()}), flush=True)
    torch.save(out, os.path.join(ROOT, "tests", "golden", "loss.pt"))


if __name__ == "__main__":
    main()
