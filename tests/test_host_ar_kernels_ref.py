"""The float64 references of tests/test_gpu_ar_kernels.py (tests/ar_kernels_ref.py), pinned on the CPU: against torch's own float64
attention and LayerNorm, the split-order fp32 sum against an explicit loop, and every named mistake visible on its needle inputs -- its
reference lies more than both tolerances away from the correct one somewhere, so a kernel within tolerance of the correct reference is
outside tolerance of the mutated one."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import ar_kernels_ref as R


def separated(ref, slack, mut, mslack, fmt):
    return float(((ref - mut).abs() - R.tol16(ref, slack, fmt) - R.tol16(mut, mslack, fmt)).max()) > 0


@pytest.mark.parametrize("G,T,E", [(1, 1, 64), (3, 5, 128), (2, 70, 128), (1, 130, 64)])
def test_prefill_reference_is_causal_sdpa(G, T, E):
    qkv = torch.randn(T * G, 3 * E, generator=torch.Generator().manual_seed(T), dtype=torch.float64)
    ref, slack = R.prefill_ref(qkv, G, T, E, 0)
    q, k, v = (qkv[:, i * E:(i + 1) * E].view(T, G, E // 64, 64).permute(1, 2, 0, 3) for i in range(3))
    sd = F.scaled_dot_product_attention(q, k, v, is_causal=True, scale=0.125)          # [G, nh, T, 64]
    torch.testing.assert_close(ref, sd.permute(2, 0, 1, 3).reshape(T * G, E), rtol=1e-12, atol=1e-12)
    assert bool((slack > 0).all()) and float(slack.max()) < 1e-2


def test_step_reference_is_attention_over_cache_and_new_token():
    B, E, Tmax, t, S = 2, 128, 20, 9, 3
    part, bqkv, kc, vc = R.step_inputs(B, E, Tmax, t, S, 0, seed=1)
    ref, _ = R.step_ref(part, bqkv, kc, vc, t, 0)
    q, kn, vn = R.step_qkv(part, bqkv, 0)
    for b in range(B):
        for h in range(E // 64):
            keys = torch.cat([kc[b, h, :t].double(), kn[b, h * 64:(h + 1) * 64].double()[None]])
            vals = torch.cat([vc[b, h, :t].double(), vn[b, h * 64:(h + 1) * 64].double()[None]])
            w = torch.softmax(keys @ q[b, h * 64:(h + 1) * 64].double() / 8, 0)
            torch.testing.assert_close(ref[b, h * 64:(h + 1) * 64], w @ vals, rtol=1e-12, atol=1e-12)


def test_split_sum_is_the_fp32_loop_in_split_order():
    g = torch.Generator().manual_seed(0)
    terms = [torch.randn(5, generator=g) * 10 ** e for e in (0, 6, -3, 4, 0)]
    got = R.split_sum_f32(terms[0], None, *terms[1:])
    for i in range(5):
        acc = np.float32(terms[0][i])
        for t in terms[1:]:
            acc = np.float32(acc + np.float32(t[i]))
        assert got[i].item() == float(acc)
    assert got.dtype == torch.float32


@pytest.mark.parametrize("E", [128, 1536])
def test_layer_norm_reference_is_torch_layer_norm(E):
    x = R.ln_rows_input(6, E, seed=E)
    g, b = torch.randn(E, dtype=torch.float64), torch.randn(E, dtype=torch.float64)
    y, _, _ = R.layer_norm64(x, g, b)
    torch.testing.assert_close(y, F.layer_norm(x.double(), (E,), g, b, eps=R.LN_EPS), rtol=1e-10, atol=1e-10)


def test_ulp16():
    for fmt, dt in R.DT.items():
        x = torch.tensor([1.0, 1.5, 3.0, 1e-3, 0.0, -2.0])
        a = x.abs().to(dt)
        nxt = torch.nextafter(a, torch.full_like(a, 1e4)).double() - a.double()        # the spacing above |x|
        assert torch.equal(R.ulp16(x.double(), fmt), nxt)


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("mutation", R.STEP_MUTATIONS)
def test_step_mutations_are_visible_on_needles(mutation, fmt):
    part, bqkv, kc, vc = R.step_inputs(2, 256, 100, 70, 3, fmt, seed=5, needles=True)
    ref, slack = R.step_ref(part, bqkv, kc, vc, 70, fmt)
    mut, mslack = R.step_ref(part, bqkv, kc, vc, 70, fmt, mutation=mutation)
    assert separated(ref, slack, mut, mslack, fmt)


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("mutation", R.PREFILL_MUTATIONS)
def test_prefill_mutations_are_visible_on_needles(mutation, fmt):
    G, T, E = 2, 130, 256
    qkv = R.prefill_needles(G, T, E, fmt, seed=3)
    ref, slack = R.prefill_ref(qkv, G, T, E, fmt)
    mut, mslack = R.prefill_ref(qkv, G, T, E, fmt, mutation=mutation)
    assert separated(ref, slack, mut, mslack, fmt)


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("mutation", R.LN_MUTATIONS)
def test_ln_mutations_are_visible(mutation, fmt):
    E, S = 128, 3
    x = R.ln_rows_input(8, E, seed=7)
    part = torch.randn(S, 8, E, generator=torch.Generator().manual_seed(8))
    part[:, 3] = 0                                        # (row 3 keeps its variance of ~1e-8)
    g, b = torch.rand(E, dtype=torch.float64) + 0.5, torch.randn(E, dtype=torch.float64)
    x_out = R.split_sum_f32(x, *part)
    ref, slack = R.ln_rows_ref(x_out, g, b, 1)
    xm = R.split_sum_f32(x, *part[:-1]) if mutation == "omit_last_partial" else None
    mut, mslack = R.ln_rows_ref(x_out, g, b, 1, mutation_x=xm, mutation=None if xm is not None else mutation)
    assert separated(ref, slack, mut, mslack, fmt)


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("mutation", ["tanh_gelu", "omit_one_partial"])
def test_gelu_mutations_are_visible(mutation, fmt):
    S, B, N = 3, 2, 512
    g = torch.Generator().manual_seed(9)
    part = torch.randn(S, B, N, generator=g)
    bias = torch.linspace(-4, 4, N)
    v = R.split_sum_f32(bias, *part)
    ref = R.gelu64(v)
    vm = R.split_sum_f32(bias, *part[:-1]) if mutation == "omit_one_partial" else v
    mut = R.gelu64(vm, "tanh_gelu" if mutation == "tanh_gelu" else None)
    assert separated(ref, R.gelu_slack(v, ref), mut, R.gelu_slack(vm, mut), fmt)
