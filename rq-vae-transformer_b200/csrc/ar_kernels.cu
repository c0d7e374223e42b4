// P3 building blocks, "exact" tier: fp32 activations, fp32 FFMA accumulate, weights fp32 (bit-exact-indices gate) or
// bf16 (storage only).  These are the correctness anchors for the wgmma weight-streaming kernels in
// ar_gemm_tc.cu: same interfaces, same epilogues.
//
// Reference sites (rqvae/models/rqtransformer/attentions.py unless noted):
//   linear_nt ......... nn.Linear everywhere: :69-71,:99 (q,k,v,proj), :117-122 (MLP, exact-erf GELU :34),
//                       transformers.py:64,67 (input_mlp/head_mlp), :94 (classifier)
//   layernorm ......... :113-114, transformers.py:91 (eps 1e-5)
//   attn_cached ....... :73-95 (KV append by torch.cat -> here an in-place write into a pre-allocated cache,
//                       scale folded into K :87, causal mask :89-91, softmax :92, att @ V :95)
//   embedding kernels . transformers.py:217-232 (body token = sum_d input_mlp(e_d) + pos_emb_hw, bias counted D
//                       times), :249-270 (head token = head_mlp(cumsum_d e) + pos_emb_d / spatial ctx + pos_emb_d[0])
#include "kernels.h"

namespace rqb {

// ------------------------------------------------------------------------------------------------ GEMM  Y = act(X W^T + b) (+R)
constexpr int GB_M = 64, GB_N = 64, GB_K = 16, G_THREADS = 256;

template <typename WT>
__device__ __forceinline__ float4 load_w4(const WT* p);
template <>
__device__ __forceinline__ float4 load_w4<float>(const float* p) { return *reinterpret_cast<const float4*>(p); }
template <>
__device__ __forceinline__ float4 load_w4<__nv_bfloat16>(const __nv_bfloat16* p) {
    uint2 raw = *reinterpret_cast<const uint2*>(p);
    __nv_bfloat162 a = *reinterpret_cast<__nv_bfloat162*>(&raw.x), b = *reinterpret_cast<__nv_bfloat162*>(&raw.y);
    float2 fa = __bfloat1622float2(a), fb = __bfloat1622float2(b);
    return make_float4(fa.x, fa.y, fb.x, fb.y);
}

// X [M,K] f32 (row stride ldx), W [N,K] WT, bias [N] f32 (nullable), R [M,N] f32 residual (nullable, ld = ldy),
// Y [M,N] f32.  K % 4 == 0.  act: 0 none, 1 exact GELU.
template <typename WT>
__global__ void __launch_bounds__(G_THREADS)
linear_nt_kernel(const float* __restrict__ X, int64_t ldx, const WT* __restrict__ W, const float* __restrict__ bias,
                 const float* R, float* Y, int64_t ldy, int M, int N, int K, int act) {
    __shared__ float As[GB_K][GB_M + 4];
    __shared__ float Ws[GB_K][GB_N + 4];
    const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
    const int m0 = blockIdx.y * GB_M, n0 = blockIdx.x * GB_N;
    const int lr = t >> 2, lk = (t & 3) * 4;        // loader: row lr, k offset lk
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] = 0.f;

    for (int k0 = 0; k0 < K; k0 += GB_K) {
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f), w = a;
        if (m0 + lr < M && k0 + lk < K) a = *reinterpret_cast<const float4*>(X + (int64_t)(m0 + lr) * ldx + k0 + lk);
        if (n0 + lr < N && k0 + lk < K) w = load_w4<WT>(W + (int64_t)(n0 + lr) * K + k0 + lk);
        As[lk + 0][lr] = a.x; As[lk + 1][lr] = a.y; As[lk + 2][lr] = a.z; As[lk + 3][lr] = a.w;
        Ws[lk + 0][lr] = w.x; Ws[lk + 1][lr] = w.y; Ws[lk + 2][lr] = w.z; Ws[lk + 3][lr] = w.w;
        __syncthreads();
#pragma unroll
        for (int k = 0; k < GB_K; k++) {
            float4 av = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
            float4 wv = *reinterpret_cast<const float4*>(&Ws[k][tx * 4]);
            float aa[4] = {av.x, av.y, av.z, av.w}, ww[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) acc[i][j] = fmaf(aa[i], ww[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; i++) {
        int m = m0 + ty * 4 + i;
        if (m >= M) continue;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            int n = n0 + tx * 4 + j;
            if (n >= N) continue;
            float v = acc[i][j] + (bias ? bias[n] : 0.f);
            if (act == 1) v = gelu_erf(v);
            if (R) v = R[(int64_t)m * ldy + n] + v;            // x = x + f(x)
            Y[(int64_t)m * ldy + n] = v;
        }
    }
}

int launch_linear(const float* X, int64_t ldx, const void* W, int wdtype, const float* bias, const float* R, float* Y,
                  int64_t ldy, int M, int N, int K, int act, cudaStream_t st) {
    if (M <= 0) return 0;
    if (K % 4 != 0) return fail(RQB200_EINVAL, "linear: K % 4 != 0");
    dim3 grid((unsigned)ceil_div(N, GB_N), (unsigned)ceil_div(M, GB_M));
    if (wdtype == RQB200_F32)
        linear_nt_kernel<float><<<grid, G_THREADS, 0, st>>>(X, ldx, (const float*)W, bias, R, Y, ldy, M, N, K, act);
    else if (wdtype == RQB200_BF16)
        linear_nt_kernel<__nv_bfloat16><<<grid, G_THREADS, 0, st>>>(X, ldx, (const __nv_bfloat16*)W, bias, R, Y, ldy, M, N, K, act);
    else
        return fail(RQB200_EINVAL, "linear: unsupported weight dtype");
    return check_launch("linear_nt");
}

// ------------------------------------------------------------------------------------------------ LayerNorm (eps 1e-5)
__global__ void __launch_bounds__(256) layernorm_kernel(const float* __restrict__ X, int64_t ldx, const float* __restrict__ g,
                                                        const float* __restrict__ b, float* __restrict__ Y, int64_t ldy, int E,
                                                        float eps) {
    __shared__ float red[33];
    const float* x = X + (int64_t)blockIdx.x * ldx;
    float* y = Y + (int64_t)blockIdx.x * ldy;
    float s = 0.f;
    for (int i = threadIdx.x; i < E; i += blockDim.x) s += x[i];
    const float mean = block_sum(s, red) / (float)E;
    float v = 0.f;
    for (int i = threadIdx.x; i < E; i += blockDim.x) { float d = x[i] - mean; v = fmaf(d, d, v); }
    const float var = block_sum(v, red) / (float)E;
    const float rstd = 1.0f / sqrtf(var + eps);
    for (int i = threadIdx.x; i < E; i += blockDim.x) y[i] = (x[i] - mean) * rstd * g[i] + b[i];
}

int launch_layernorm(const float* X, int64_t ldx, const float* g, const float* b, float* Y, int64_t ldy, int M, int E,
                     cudaStream_t st) {
    if (M <= 0) return 0;
    layernorm_kernel<<<M, 256, 0, st>>>(X, ldx, g, b, Y, ldy, E, 1e-5f);
    return check_launch("layernorm");
}

// ------------------------------------------------------------------------------------------------ cached causal attention
// qkv [B*Tn, 3E] rows m = b*Tn + tq, columns [query | key | value]; cache kc/vc [B][nh][Tmax][64] (this layer).
// Appends the Tn new K/V rows at T_past.. then, for each new token, softmax(q.(k/8)) V over keys 0..T_past+tq.
__global__ void __launch_bounds__(128) attn_cached_kernel(const float* __restrict__ qkv, float* __restrict__ kc,
                                                          float* __restrict__ vc, float* __restrict__ out, int Tn, int T_past,
                                                          int Tmax, int E, int nh) {
    extern __shared__ float sm[];
    float* sc = sm;                 // [T_past + Tn]
    float* qs = sm + (T_past + Tn); // [64]
    __shared__ float red[33];
    const int h = blockIdx.x, b = blockIdx.y, t = threadIdx.x, lane = t & 31, warp = t >> 5;
    float* kb = kc + ((int64_t)(b * nh + h) * Tmax) * 64;
    float* vb = vc + ((int64_t)(b * nh + h) * Tmax) * 64;
    for (int tq = 0; tq < Tn; tq++) {
        const float* row = qkv + (int64_t)(b * Tn + tq) * 3 * E + h * 64;
        if (t < 64) kb[(int64_t)(T_past + tq) * 64 + t] = row[E + t];
        else vb[(int64_t)(T_past + tq) * 64 + (t - 64)] = row[2 * E + (t - 64)];
    }
    __syncthreads();
    for (int tq = 0; tq < Tn; tq++) {
        const int T = T_past + tq + 1;
        const float* row = qkv + (int64_t)(b * Tn + tq) * 3 * E + h * 64;
        if (t < 64) qs[t] = row[t];
        __syncthreads();
        for (int j = warp; j < T; j += 4) {
            const float* kr = kb + (int64_t)j * 64;
            float p = qs[lane] * kr[lane];
            p = fmaf(qs[lane + 32], kr[lane + 32], p);
            p = warp_sum(p);
            if (lane == 0) sc[j] = p * 0.125f;            // == q . (k / sqrt(64)), attentions.py:87
        }
        __syncthreads();
        float m = -INFINITY;
        for (int j = t; j < T; j += 128) m = fmaxf(m, sc[j]);
        m = block_max(m, red);
        float s = 0.f;
        for (int j = t; j < T; j += 128) { float e = expf(sc[j] - m); sc[j] = e; s += e; }
        s = block_sum(s, red);
        __syncthreads();
        for (int j = t; j < T; j += 128) sc[j] = sc[j] / s;
        __syncthreads();
        if (t < 64) {
            float a = 0.f;
            for (int j = 0; j < T; j++) a = fmaf(sc[j], vb[(int64_t)j * 64 + t], a);
            out[(int64_t)(b * Tn + tq) * E + h * 64 + t] = a;
        }
        __syncthreads();
    }
}

int launch_attn_cached(const float* qkv, float* kc, float* vc, float* out, int B, int Tn, int T_past, int Tmax, int E,
                       int nh, cudaStream_t st) {
    if (E != nh * 64) return fail(RQB200_EINVAL, "attention: head dim must be 64");
    if (T_past + Tn > Tmax) return fail(RQB200_EINVAL, "attention: KV cache overflow");
    size_t smem = (size_t)(T_past + Tn + 64) * sizeof(float);
    attn_cached_kernel<<<dim3(nh, B), 128, smem, st>>>(qkv, kc, vc, out, Tn, T_past, Tmax, E, nh);
    return check_launch("attn_cached");
}

// ------------------------------------------------------------------------------------------------ embedding glue
// out[(b*J + (j-j0))*D + d, :] = codebook_d[codes[b, j, d], :]   for j in [j0, j0+J); codebook_d = cb + d * cb_dstride
// CV: j is a window position, read from the canvas through cv (kernels.h); else codes is [B, HW, D]
template <bool CV>
__global__ void code_emb_kernel(const int64_t* __restrict__ codes, const float* __restrict__ cb, int64_t cb_dstride, int HW, int D,
                                int K, int C, int j0, int J, float* __restrict__ out, CanvasMap cv) {
    int r = blockIdx.x;                         // over B*J*D
    int d = r % D, j = (r / D) % J, b = r / (D * J);
    int64_t k = codes[(CV ? cv.at(b, j0 + j) : (int64_t)b * HW + j0 + j) * D + d];
    k = k < 0 ? 0 : (k >= K ? K - 1 : k);
    const float* e = cb + d * cb_dstride + k * C;
    for (int c = threadIdx.x; c < C; c += blockDim.x) out[(int64_t)r * C + c] = e[c];
}
// body tokens: X[b, s0 + (j-j0), :] = ((l0 + l1) + l2) + ... + pos_hw[j]   with l_d = lin[(b*J + (j-j0))*D + d, :]
__global__ void body_token_kernel(const float* __restrict__ lin, const float* __restrict__ pos_hw, int D, int E, int j0, int J,
                                  int s0, int Tn, float* __restrict__ X) {
    int r = blockIdx.x;                         // over B*J
    int j = r % J, b = r / J;
    for (int e = threadIdx.x; e < E; e += blockDim.x) {
        float a = lin[((int64_t)r * D) * E + e];
        for (int d = 1; d < D; d++) a += lin[((int64_t)r * D + d) * E + e];
        X[((int64_t)b * Tn + s0 + j) * E + e] = a + pos_hw[(int64_t)(j0 + j) * E + e];
    }
}
// cond tokens: X[b, s, :] = cond_emb[cond[b,s]] + pos_emb_cond[s]   (cond == nullptr -> token 0, transformers.py:208-209)
__global__ void cond_token_kernel(const int64_t* __restrict__ cond, const float* __restrict__ cond_emb,
                                  const float* __restrict__ pos_cond, int cond_len, int vocab_cond, int E, int Tn,
                                  float* __restrict__ X) {
    int r = blockIdx.x;                         // over B*cond_len
    int s = r % cond_len, b = r / cond_len;
    int64_t c = cond ? cond[(int64_t)b * cond_len + s] : 0;
    c = c < 0 ? 0 : (c >= vocab_cond ? vocab_cond - 1 : c);
    for (int e = threadIdx.x; e < E; e += blockDim.x)
        X[((int64_t)b * Tn + s) * E + e] = cond_emb[c * E + e] + pos_cond[(int64_t)s * E + e];
}
// head input for depth d >= 1: out[b,:] = e_0 + e_1 + ... + e_{d-1} (sequential, torch.cumsum order); last_only: e_{d-1} alone
// (cumsum_depth_ctx = false, or the row of a token embedding table when cb is tok_emb).  CV: as code_emb_kernel
template <bool CV>
__global__ void head_cumsum_kernel(const int64_t* __restrict__ codes, const float* __restrict__ cb, int64_t cb_dstride, int HW, int D,
                                   int K, int C, int j, int d, int last_only, float* __restrict__ out, CanvasMap cv) {
    int b = blockIdx.x;
    const int i0 = last_only ? d - 1 : 0;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float a = 0.f;
        for (int i = i0; i < d; i++) {
            int64_t k = codes[(CV ? cv.at(b, j) : (int64_t)b * HW + j) * D + i];
            k = k < 0 ? 0 : (k >= K ? K - 1 : k);
            float e = cb[i * cb_dstride + k * C + c];
            a = (i == i0) ? e : a + e;
        }
        out[(int64_t)b * C + c] = a;
    }
}
// out[b,:] = in[b*ld_in ... ] + pos[:]   (row gather with stride: used for "last prefill token" and "+ pos_emb_d[d]")
__global__ void row_add_kernel(const float* __restrict__ in, int64_t in_row_stride, int64_t in_off, const float* __restrict__ pos,
                               int E, float* __restrict__ out) {
    int b = blockIdx.x;
    const float* x = in + (int64_t)b * in_row_stride + in_off;
    for (int e = threadIdx.x; e < E; e += blockDim.x) out[(int64_t)b * E + e] = x[e] + (pos ? pos[e] : 0.f);
}

int launch_code_emb(const int64_t* codes, const float* cb, int64_t cb_dstride, int B, int HW, int D, int K, int C, int j0, int J,
                    float* out, cudaStream_t st, const CanvasMap* cv) {
    if (B * J * D <= 0) return 0;
    if (cv)
        code_emb_kernel<true><<<B * J * D, 64, 0, st>>>(codes, cb, cb_dstride, HW, D, K, C, j0, J, out, *cv);
    else
        code_emb_kernel<false><<<B * J * D, 64, 0, st>>>(codes, cb, cb_dstride, HW, D, K, C, j0, J, out, CanvasMap{});
    return check_launch("code_emb");
}
int launch_body_token(const float* lin, const float* pos_hw, int B, int D, int E, int j0, int J, int s0, int Tn, float* X,
                      cudaStream_t st) {
    if (B * J <= 0) return 0;
    body_token_kernel<<<B * J, 256, 0, st>>>(lin, pos_hw, D, E, j0, J, s0, Tn, X);
    return check_launch("body_token");
}
int launch_cond_token(const int64_t* cond, const float* cond_emb, const float* pos_cond, int B, int cond_len, int vocab_cond,
                      int E, int Tn, float* X, cudaStream_t st) {
    cond_token_kernel<<<B * cond_len, 256, 0, st>>>(cond, cond_emb, pos_cond, cond_len, vocab_cond, E, Tn, X);
    return check_launch("cond_token");
}
int launch_head_cumsum(const int64_t* codes, const float* cb, int64_t cb_dstride, int B, int HW, int D, int K, int C, int j, int d,
                       float* out, cudaStream_t st, bool last_only, const CanvasMap* cv) {
    if (cv)
        head_cumsum_kernel<true><<<B, 64, 0, st>>>(codes, cb, cb_dstride, HW, D, K, C, j, d, last_only ? 1 : 0, out, *cv);
    else
        head_cumsum_kernel<false><<<B, 64, 0, st>>>(codes, cb, cb_dstride, HW, D, K, C, j, d, last_only ? 1 : 0, out, CanvasMap{});
    return check_launch("head_cumsum");
}
int launch_row_add(const float* in, int64_t in_row_stride, int64_t in_off, const float* pos, int B, int E, float* out,
                   cudaStream_t st) {
    row_add_kernel<<<B, 256, 0, st>>>(in, in_row_stride, in_off, pos, E, out);
    return check_launch("row_add");
}

}  // namespace rqb
