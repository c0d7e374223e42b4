#!/usr/bin/env python
"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/rqd.pt from the UNMODIFIED reference classes: residual quantisation with one
codebook per depth (RQBottleneck(shared_codebook=False)).

    rq    RQBottleneck runs on 8x8xD code maps: K = [2048]*4 at B = 2, K = [16384]*4 at B = 64 (N = 4096), unequal
          K = [512, 1000, 2048, 300], and a tie case (rows 256.. of table 2 repeat rows 0..255; one input equals a row of
          table 0).  Codes, the fp64 sums of every aggregate, a sample of the last aggregate, and samples + fp64 sums of
          embed_code, embed_code_with_depth, embed_partial_code (select / add, every code_idx) and, for equal K, get_soft_codes of the
          first two images.
    vae   the "tiny" RQ-VAE of oracle/zoo.py with per-depth codebooks: its state_dict key / shape list, a sample of its default
          initialisation under torch.manual_seed(0), decode_code pixels of seeded codes and get_codes of a seeded image.
    ar    a tiny transformer (tests/depthwise_oracle.py AR_SHAPE: E 128, 2 heads, 2 + 2 layers, V 512, 8x8x4, a 4-token prefix)
          whose model_aux is the reference's own RQBottleneck(shared_codebook=False): greedy and top-k/top-p trajectories under
          oracle/gen_golden.py's NoiseInjector with the logits of their first and last steps, and one start_loc resume.

Needs the reference tree (oracle/ref_loader.py):   python scripts/gen_golden_depthwise.py
Same protocol as scripts/gen_golden_long.py: tables, inputs and weights are regenerated from oracle/synth.py seeds
(tests/depthwise_oracle.py: rq_inputs, depthwise_vae_state); the file stores seeds and the reference's outputs.
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
from tests import depthwise_oracle as DO                            # noqa: E402

N_SAMPLE = 256


def sample(t, n=N_SAMPLE):
    """(fp64 sum, n seeded values) -- positions depend on the size only"""
    flat = t.reshape(-1)
    g = torch.Generator().manual_seed(flat.numel())
    return float(t.double().sum()), flat[torch.randint(0, flat.numel(), (n,), generator=g)].clone()


def gen_rq(ns):
    RQB = ns.modules["rqvae.models.rqvae.quantizations"].RQBottleneck
    out = {}
    for name, (ks, B, _, _, _) in DO.RQ_CASES.items():
        t0 = time.time()
        tables, x = DO.rq_inputs(name)
        D = len(ks)
        q = RQB(latent_shape=[8, 8, 256], code_shape=[8, 8, D], n_embed=list(ks), shared_codebook=False).eval()
        for d, t in enumerate(tables):
            q.codebooks[d].weight.data[:-1] = t
        quants, codes = q.quantize(x)
        rec = dict(codes=codes.to(torch.int16), agg_sums=[float(a.double().sum()) for a in quants], last=sample(quants[-1]),
                   embed_code=sample(q.embed_code(codes)), embed_code_with_depth=sample(q.embed_code_with_depth(codes)[0]),
                   partial={(typ, i): sample(q.embed_partial_code(codes, i, typ)) for typ in ("select", "add") for i in range(D)})
        if len(set(ks)) == 1:           # soft codes of the first two images ([2,8,8,D,K]: 128 MB at K = 16384)
            soft, scodes = q.get_soft_codes(x[:2], temp=1.0, stochastic=False)
            assert torch.equal(scodes, codes[:2])
            rec["soft"] = sample(soft)
        out[name] = rec
        print("  rq %-12s %.1fs" % (name, time.time() - t0), flush=True)
    return out


def vae_kwargs():
    kw = R.vae_kwargs(**{k: v for k, v in VAE_ZOO["tiny"].items()})
    kw["shared_codebook"] = False
    return kw


def gen_vae(ns):
    torch.manual_seed(0)
    init = synth.state_dict_sample(ns.RQVAE(**vae_kwargs()).state_dict())
    m = ns.RQVAE(**vae_kwargs()).eval()
    shapes = synth.shapes_of(m.state_dict())
    m.load_state_dict(DO.depthwise_vae_state(shapes, 21, 300))
    codes = synth.randint_seeded(0, 512, (2, 4, 4, 4), 22)
    img = synth.randn_seeded((2, 3, 16, 16), 23, 0.5)
    return dict(layout={k: list(v) for k, v in shapes.items()}, init=init, weight_seed=21, table_seed=300, codes_seed=22,
                image_seed=23, pixels=m.decode_code(codes).detach().clone(), get_codes=m.get_codes(img).to(torch.int16))


def gen_ar(ns):
    """(c): greedy and top-k/top-p trajectories with the logits of their first and last steps, and one start_loc resume; model_aux is
    the reference's own RQBottleneck(shared_codebook=False)"""
    from oracle.gen_golden import NoiseInjector
    E, nh, nb, nhl, V, bs, vc, cl = DO.AR_SHAPE
    P = DO.AR_PLAN
    t0 = time.time()
    model = ns.RQTransformer(R.transformer_cfg(E, nh, nb, nhl, V, block_size=bs, vocab_cond=vc, cond_len=cl)).eval()
    model.load_state_dict(synth.synth_state_dict(synth.shapes_of(model.state_dict()), P["weight_seed"]))
    RQB = ns.modules["rqvae.models.rqvae.quantizations"].RQBottleneck
    q = RQB(latent_shape=[bs[0], bs[1], 256], code_shape=list(bs), n_embed=V, shared_codebook=False).eval()
    for d, t in enumerate(DO.tables_of([V] * bs[2], P["table_seed"])):
        q.codebooks[d].weight.data[:-1] = t

    class Aux:          # the only thing sample() needs from the RQ-VAE (transformers.py:109-111)
        def get_code_emb_with_depth(self, code):
            return q.embed_code_with_depth(code)

    cond = synth.randint_seeded(0, vc, (P["B"], cl), P["cond_seed"])
    keep = [0, bs[0] * bs[1] * bs[2] - 1]
    runs = []
    for st, seed in zip(P["settings"], P["noise_seeds"]):
        kept, counter, orig = {}, [0], model.cached_forward

        def spy(*a, **kw):
            lg = orig(*a, **kw)
            if counter[0] in keep:
                kept[counter[0]] = lg.clone()
            counter[0] += 1
            return lg

        model.cached_forward = spy
        with NoiseInjector(seed):
            codes = model.sample(torch.zeros(P["B"], *bs, dtype=torch.long), model_aux=Aux(), cond=cond, **st)
        model.cached_forward = orig
        runs.append(dict(setting=st, noise_seed=seed, codes=codes.to(torch.int16), logits=kept))
    rs = P["resume"]
    with NoiseInjector(rs["noise_seed"]):
        codes2 = model.sample(runs[1]["codes"].long(), model_aux=Aux(), cond=cond, start_loc=rs["start_loc"], **P["settings"][1])
    print("  ar %.1fs" % (time.time() - t0), flush=True)
    return dict(runs=runs, resume=dict(codes=codes2.to(torch.int16)))


def main():
    torch.set_grad_enabled(False)
    ns = R.load_reference()
    res = {"rq_cases": dict(DO.RQ_CASES), "rq": gen_rq(ns), "vae": gen_vae(ns), "ar": gen_ar(ns)}
    torch.save(res, os.path.join(ROOT, "tests", "golden", "rqd.pt"))


if __name__ == "__main__":
    main()
