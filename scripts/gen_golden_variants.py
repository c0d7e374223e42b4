#!/usr/bin/env python
"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/arv.pt from the UNMODIFIED reference classes: RQ-Transformers under every
combination of the five embedding / classifier switches (input_emb_vqvae, head_emb_vqvae, cumsum_depth_ctx, shared_tok_emb,
shared_cls_emb; tests/variants_oracle.py).

    combos    all 32 combinations on a tiny class-conditional model (variants_oracle.TINY: E 128, 2 heads, 2 + 2 layers, V 512,
              4x4x4).  For each: the state_dict key / shape list, a sample of the default initialisation under torch.manual_seed(0),
              greedy and top-k/top-p trajectories under oracle/gen_golden.py's NoiseInjector with the logits of their first and last
              steps.
    text      the all-false default on a text-shaped tiny model (variants_oracle.TEXT, cond_len 4): one start_loc resume and the
              forward logits with the cond logits of the greedy trajectory.
    headless  the all-false default on a 4x4x1 model without head layers (variants_oracle.HEADLESS).
    unequal   one layout with per-depth vocabularies of different sizes (construction only: the reference cannot sample it).

Needs the reference tree (oracle/ref_loader.py):   python scripts/gen_golden_variants.py
Same protocol as scripts/gen_golden_depthwise.py: weights come from oracle/synth.py seeds (variants_oracle.state_dict_of, which
restores the real tok_emb.offsets), the shared codebook from synth.randn_seeded; the file stores seeds and the reference's outputs.
"""
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_loader as R                                  # noqa: E402
from oracle import synth                                            # noqa: E402
from oracle.gen_golden import NoiseInjector                         # noqa: E402
from tests import variants_oracle as VO                             # noqa: E402


def cfg_of(shape, flags):
    E, nh, nb, nhl, V, bs, vc, cl = shape
    c = R.transformer_cfg(E, nh, nb, nhl, V, block_size=bs, vocab_cond=vc, cond_len=cl)
    c.update(flags)
    return c


def aux_of(table):
    class Aux:          # the only thing sample() needs from the RQ-VAE (transformers.py:109-111)
        def get_code_emb_with_depth(self, code):
            parts = [torch.nn.functional.embedding(c, table) for c in torch.chunk(code, code.shape[-1], dim=-1)]
            return torch.cat(parts, dim=-2), None
    return Aux()


def build(ns, shape, flags):
    model = ns.RQTransformer(cfg_of(shape, flags)).eval()
    shapes = synth.shapes_of(model.state_dict())
    model.load_state_dict(VO.state_dict_of(shapes, VO.PLAN["weight_seed"]))
    return model, shapes


def trajectories(ns, model, shape, flags, aux):
    P = VO.PLAN
    bs, vc, cl = shape[5], shape[6], shape[7]
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
            codes = model.sample(torch.zeros(P["B"], *bs, dtype=torch.long), model_aux=aux, cond=cond, **st)
        model.cached_forward = orig
        runs.append(dict(setting=st, noise_seed=seed, codes=codes.to(torch.int16), logit_steps=keep,
                         logits=torch.stack([kept[s] for s in keep])))
    return runs, cond


def init_sample(sd):
    """synth.state_dict_sample packed into two tensors (the file stays small): the fp64 sums and the concatenated sampled values, both
    in state_dict order (the layout gives keys and shapes)"""
    s = synth.state_dict_sample(sd, VO.PLAN["init_sample"])
    return dict(sums=torch.tensor([v[1] for v in s.values()], dtype=torch.float64),
                values=torch.cat([v[2].reshape(-1) for v in s.values()]))


def gen_combos(ns, aux, layouts):
    """layouts: list of the distinct state_dict layouts; each combo stores the index of its own"""
    out = {}
    for flags in VO.COMBOS:
        t0 = time.time()
        torch.manual_seed(VO.PLAN["init_seed"])
        init = init_sample(ns.RQTransformer(cfg_of(VO.TINY, flags)).state_dict())
        model, shapes = build(ns, VO.TINY, flags)
        runs, _ = trajectories(ns, model, VO.TINY, flags, aux if VO.needs_codebook(flags) else None)
        layout = [(k, list(v)) for k, v in shapes.items()]
        if layout not in layouts:
            layouts.append(layout)
        out[VO.combo_name(flags)] = dict(flags=flags, layout=layouts.index(layout), init=init, runs=runs)
        print("  combo %s %.1fs" % (VO.combo_name(flags), time.time() - t0), flush=True)
    return out


def gen_text(ns):
    model, _ = build(ns, VO.TEXT, VO.ALL_FALSE)
    runs, cond = trajectories(ns, model, VO.TEXT, VO.ALL_FALSE, None)
    rs = VO.PLAN["resume"]
    with NoiseInjector(rs["noise_seed"]):
        codes2 = model.sample(runs[1]["codes"].long(), model_aux=None, cond=cond, start_loc=rs["start_loc"], **VO.PLAN["settings"][1])
    logits, cond_logits = model(runs[0]["codes"][:1].long(), model_aux=None, cond=cond[:1])      # (batch row 0: the file stays small)
    return dict(runs=runs, resume=dict(codes=codes2.to(torch.int16)), forward=logits.detach().clone(),
                cond_logits=cond_logits.detach().clone())


def gen_headless(ns):
    model, _ = build(ns, VO.HEADLESS, VO.ALL_FALSE)
    runs, _ = trajectories(ns, model, VO.HEADLESS, VO.ALL_FALSE, None)
    return dict(runs=runs)


def gen_unequal(ns):
    U = VO.UNEQUAL
    torch.manual_seed(VO.PLAN["init_seed"])
    sd = ns.RQTransformer(cfg_of(U["shape"], U["flags"])).state_dict()
    return dict(layout=[(k, list(v.shape)) for k, v in sd.items()], init=init_sample(sd))


def main():
    torch.set_grad_enabled(False)
    ns = R.load_reference()
    table = synth.randn_seeded((VO.TINY[4], 256), VO.PLAN["table_seed"])
    layouts = []
    res = {"combos": gen_combos(ns, aux_of(table), layouts), "layouts": layouts, "text": gen_text(ns), "headless": gen_headless(ns),
           "unequal": gen_unequal(ns)}
    torch.save(res, os.path.join(ROOT, "tests", "golden", "arv.pt"))


if __name__ == "__main__":
    main()
