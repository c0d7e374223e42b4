"""GroupNorm statistics under a mean offset: for groups whose mean sits r standard deviations off zero, the error of each GroupNorm path
of the VAE engine next to torch's fp32 group_norm, both against float64.  Both kernel statistics paths form the variance as
E[x^2] - mean^2 from fp32 partial sums, whose relative error grows with 1 + r^2 (tests/vae_kernels_ref.py derives the bound).

One conv (fp16 wgmma, its epilogue emitting the GroupNorm partials; 2 images of 32 x 32 x 512, cg = 16) makes the input, with a bias
of +-r per group; its output then goes through the three paths:
  exact  gn_stats_kernel + gn_apply_kernel (fp32 out)
  stats  gn_stats_kernel + gn_finalize_kernel + gn_apply_f16_kernel (fp16 hi / lo out)
  fused  the conv epilogue's partials + gn_finalize_kernel + gn_apply_f16_kernel
Per path and r, one JSON line: var_rel (max relative error of the variance the kernel normalised with: from its fp64 rstd, or for
`exact` from its partial sums), torch_var_rel (the same for torch's fp32 rstd), out_err / torch_out_err (max |y - y64|, fp32 output
or hi + lo), hi_ulps (max |hi - fp16(y64)| in fp16 ulps of |(x - mean) rstd gamma| + |beta|), bound (max error / derived bound), bound_nc (the same against the bound
without the 1 + r^2 cancellation term).

usage: python scripts/gn_variance_sweep.py   (an H100; writes nothing)"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "rq-vae-transformer_b200")]

import torch  # noqa: E402

from tests import test_gpu_vae_kernels as T  # noqa: E402
from tests import vae_kernels_ref as R  # noqa: E402


def main():
    B, H, W, C = 2, 32, 32, 512
    HW = H * W
    print(json.dumps({"gpu": torch.cuda.get_device_name(0)}))
    for r in T.R_SWEEP:
        x, w, bias, _ = T.conv_gn_inputs(B, H, W, C, C, seed=r + 1, r=r)
        out, ws = T.fused_stats(x, w, bias, None, B, H, W, C, C)
        y = out.view(B, HW, C)
        gamma, beta = T.gn_affine(C, r)
        ref = R.gn_ref(y, gamma, beta, 0)
        var64 = ref["var"].view(B, 32)
        _, _, trstd = torch.ops.aten.native_group_norm(y.permute(0, 2, 1).contiguous(), gamma, beta, B, C, HW, 32, R.GN_EPS)
        torch_y = torch.nn.functional.group_norm(y.permute(0, 2, 1), 32, gamma, beta, R.GN_EPS).permute(0, 2, 1)
        torch_var = 1 / trstd.double().view(B, 32) ** 2 - R.GN_EPS
        for path, form in (("exact", 0), ("stats", 1), ("fused", 2)):
            n = T.ws_doubles(B, HW)
            wsp = ws if form == 2 else T.nan_guarded((n,), torch.float64)
            yk, hi, lo = T.run_gn(form, y, gamma, beta, 0, ws=wsp)
            stats = wsp[1]
            if form == 0:
                part = stats[:B * -(-HW // 256) * 64].view(B, -1, 32, 2).sum(1)
                var_k = part[..., 1] / (HW * C // 32) - (part[..., 0] / (HW * C // 32)) ** 2
            else:
                nchunks = HW // 32 if form == 2 else -(-HW // 256)
                fin = stats[B * nchunks * 64:B * nchunks * 64 + B * 64].view(B, 32, 2)
                var_k = 1 / fin[..., 1] ** 2 - R.GN_EPS
            got = yk.double() if form == 0 else hi.double() + lo.double()
            err = (got - ref["y"]).abs()
            s = R.gn_slack(y, gamma, beta, 0, ref, form == 2, form > 0)
            s_nc = R.gn_slack(y, gamma, beta, 0, ref, form == 2, form > 0, cancel=False)
            if form:
                s, s_nc = s + R.ulp16(lo.double(), 0) / 2, s_nc + R.ulp16(lo.double(), 0) / 2
            rel = lambda v: float(((v - var64) / var64)[:, 1:].abs().max())          # group 0 is constant (var 0)
            row = dict(path=path, r=r, var_rel=rel(var_k), torch_var_rel=rel(torch_var), out_err=float(err.max()),
                       torch_out_err=float((torch_y.double() - ref["y"]).abs().max()), bound=float((err / s).max()),
                       bound_nc=float((err / s_nc).max()))
            if form:                                  # in ulps of the affine step's terms, not of a y that cancels to ~0
                scale = ((y.double() - ref["mean"].expand(B, 1, 32, C // 32).reshape(B, 1, C)) * ref["rstd"].expand(B, 1, 32, C // 32)
                         .reshape(B, 1, C) * gamma.double()).abs() + beta.double().abs()
                row["hi_ulps"] = float(((hi.double() - ref["y"].half().double()).abs() / R.ulp16(scale, 0)).max())
            print(json.dumps(row))


if __name__ == "__main__":
    main()
