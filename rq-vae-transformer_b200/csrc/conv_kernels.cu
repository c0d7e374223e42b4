// P2 building blocks, "exact" tier (fp32 FFMA): NHWC implicit-GEMM convolution, GroupNorm(32)+SiLU, single-head
// spatial attention.  Correctness anchors for the wgmma implicit-GEMM path (conv_tc.cu).
//
// Reference sites (rqvae/models/rqvae/layers.py): Normalize :16-17 (GroupNorm 32 groups, eps 1e-6, affine),
// nonlinearity :11-13 (SiLU), ResnetBlock._forward :100-120 (3x3 s1 p1 convs, 1x1 nin_shortcut, x + h),
// Upsample :31-35 (nearest x2 then 3x3 -- here the x2 is folded into the conv's input indexing, the upsampled tensor
// is never materialised), Downsample :50-54 (F.pad (0,1,0,1) then 3x3 s2 p0 -- here implicit zero row/column),
// AttnBlock.forward :158-182 (1x1 q/k/v convs, bmm, * c^-0.5, softmax over keys, bmm, 1x1 proj_out, x + h).
// Layout: activations NHWC fp32 (channels contiguous -> the GEMM K axis is contiguous per tap), weights OHWI.
#include <algorithm>

#include "kernels.h"

namespace rqb {

constexpr int CB_M = 64, CB_N = 64, CB_K = 16, C_THREADS = 256;

template <typename WT>
__device__ __forceinline__ float w_at(const WT* p, int64_t i) { return to_f32<WT>(p[i]); }

// Epilogue forms of the conv body.  EPI_VAE: the VAE's form (one symmetric pad, output rows of Cout, optional residual R [M, Cout]).
// The plan forms (Inception, LPIPS, ResNet) take separate pad_h / pad_w (1x7, 7x1, 1x3, 3x1, 5x5 and 7x7 kernels) and write channels
// [yoff, yoff + Cout) of rows of ldy floats (a branch's slice of its block's concat buffer): EPI_RELU = ReLU(acc + bias); EPI_RES_RELU /
// EPI_RES_ID = act(acc + bias + R) with R (nullable) fp32 read at the output's own index (a ResNet block's identity), act ReLU or none.
enum ConvEpi { EPI_VAE = 0, EPI_RELU = 1, EPI_RES_RELU = 2, EPI_RES_ID = 3 };

template <typename WT, int EPI>
__device__ __forceinline__ void conv_igemm_body(const float* __restrict__ X, const WT* __restrict__ W, const float* __restrict__ bias,
                                                const float* R, float* Y, const ConvGeom& g) {
    constexpr bool INC = EPI != EPI_VAE;
    __shared__ float As[CB_K][CB_M + 4];
    __shared__ float Ws[CB_K][CB_N + 4];
    const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
    const int64_t M = (int64_t)g.B * g.Ho * g.Wo;
    const int N = g.Cout, K = g.KH * g.KW * g.Cin;
    const int64_t m0 = (int64_t)blockIdx.x * CB_M;
    const int n0 = blockIdx.y * CB_N;
    const int lr = t >> 2, lk = (t & 3) * 4;
    // this thread's A row: output pixel (b, oy, ox)
    const int64_t m = m0 + lr;
    const bool mvalid = m < M;
    int ox = 0, oy = 0, b = 0;
    if (mvalid) { ox = (int)(m % g.Wo); oy = (int)((m / g.Wo) % g.Ho); b = (int)(m / ((int64_t)g.Wo * g.Ho)); }
    const int Hv = g.upsample ? 2 * g.Hi : g.Hi, Wv = g.upsample ? 2 * g.Wi : g.Wi;   // virtual input extent
    const bool vec = (g.Cin % 4 == 0) && !g.in_nchw;

    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] = 0.f;

    for (int k0 = 0; k0 < K; k0 += CB_K) {
        float av[4] = {0.f, 0.f, 0.f, 0.f}, wv[4] = {0.f, 0.f, 0.f, 0.f};
        const int kk = k0 + lk;
        if (vec) {
            if (mvalid && kk < K) {
                int tap = kk / g.Cin, ci = kk % g.Cin;
                int ky = tap / g.KW, kx = tap % g.KW;
                int uy = oy * g.stride + ky - g.pad, ux = ox * g.stride + kx - (INC ? g.pad_w : g.pad);
                if (uy >= 0 && uy < Hv && ux >= 0 && ux < Wv) {
                    int iy = g.upsample ? (uy >> 1) : uy, ix = g.upsample ? (ux >> 1) : ux;
                    float4 v = *reinterpret_cast<const float4*>(X + (((int64_t)b * g.Hi + iy) * g.Wi + ix) * g.Cin + ci);
                    av[0] = v.x; av[1] = v.y; av[2] = v.z; av[3] = v.w;
                }
            }
        } else {
#pragma unroll
            for (int i = 0; i < 4; i++) {
                int k = kk + i;
                if (mvalid && k < K) {
                    int tap = k / g.Cin, ci = k % g.Cin;
                    int ky = tap / g.KW, kx = tap % g.KW;
                    int uy = oy * g.stride + ky - g.pad, ux = ox * g.stride + kx - (INC ? g.pad_w : g.pad);
                    if (uy >= 0 && uy < Hv && ux >= 0 && ux < Wv) {
                        int iy = g.upsample ? (uy >> 1) : uy, ix = g.upsample ? (ux >> 1) : ux;
                        av[i] = g.in_nchw ? X[(((int64_t)b * g.Cin + ci) * g.Hi + iy) * g.Wi + ix]
                                          : X[(((int64_t)b * g.Hi + iy) * g.Wi + ix) * g.Cin + ci];
                    }
                }
            }
        }
        if (n0 + lr < N) {
#pragma unroll
            for (int i = 0; i < 4; i++)
                if (kk + i < K) wv[i] = w_at<WT>(W, (int64_t)(n0 + lr) * K + kk + i);
        }
#pragma unroll
        for (int i = 0; i < 4; i++) { As[lk + i][lr] = av[i]; Ws[lk + i][lr] = wv[i]; }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < CB_K; k++) {
            float4 a4 = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
            float4 w4 = *reinterpret_cast<const float4*>(&Ws[k][tx * 4]);
            float aa[4] = {a4.x, a4.y, a4.z, a4.w}, ww[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) acc[i][j] = fmaf(aa[i], ww[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; i++) {
        int64_t mm = m0 + ty * 4 + i;
        if (mm >= M) continue;
        int oxx = (int)(mm % g.Wo), oyy = (int)((mm / g.Wo) % g.Ho), bb = (int)(mm / ((int64_t)g.Wo * g.Ho));
#pragma unroll
        for (int j = 0; j < 4; j++) {
            int n = n0 + tx * 4 + j;
            if (n >= N) continue;
            float v = acc[i][j] + (bias ? bias[n] : 0.f);
            if (EPI == EPI_RELU) {
                Y[mm * g.ldy + g.yoff + n] = fmaxf(v, 0.f);
                continue;
            }
            if (INC) {
                const int64_t o = mm * g.ldy + g.yoff + n;
                if (R) v = v + R[o];
                Y[o] = EPI == EPI_RES_RELU ? fmaxf(v, 0.f) : v;
                continue;
            }
            if (R) v = R[mm * N + n] + v;                                  // x + h  (layers.py:120,182)
            if (g.out_nchw) Y[(((int64_t)bb * N + n) * g.Ho + oyy) * g.Wo + oxx] = v;
            else Y[mm * N + n] = v;
        }
    }
}

// INC = false: the VAE's form; INC = true: the Inception and LPIPS plans' conv + bias + ReLU.  Separate instantiations, so each keeps its code.
template <typename WT, bool INC = false>
__global__ void __launch_bounds__(C_THREADS)
conv_igemm_kernel(const float* __restrict__ X, const WT* __restrict__ W, const float* __restrict__ bias, const float* R,
                  float* Y, ConvGeom g) {
    conv_igemm_body<WT, INC ? EPI_RELU : EPI_VAE>(X, W, bias, R, Y, g);
}

// the ResNet plan's residual forms: act(conv + bias [+ R]), fp32 weights
template <bool RELU>
__global__ void __launch_bounds__(C_THREADS)
conv_igemm_res_kernel(const float* __restrict__ X, const float* __restrict__ W, const float* __restrict__ bias, const float* R, float* Y,
                      ConvGeom g) {
    conv_igemm_body<float, RELU ? EPI_RES_RELU : EPI_RES_ID>(X, W, bias, R, Y, g);
}

ConvGeom vae_conv_geom(int B, int H, int W, int Cin, int Cout, int ks, int stride, int upsample, int in_nchw, int out_nchw) {
    ConvGeom g{};
    g.B = B; g.Hi = H; g.Wi = W; g.Cin = Cin; g.Cout = Cout; g.KH = g.KW = ks; g.stride = stride;
    g.upsample = upsample; g.in_nchw = in_nchw; g.out_nchw = out_nchw;
    g.pad = (ks == 3 && stride == 1) ? 1 : 0;
    g.Ho = (upsample ? 2 * H : H) / stride;
    g.Wo = (upsample ? 2 * W : W) / stride;
    return g;
}

int launch_conv(const float* X, const void* W, int wdtype, const float* bias, const float* R, float* Y, const ConvGeom& g,
                cudaStream_t st) {
    const int64_t M = (int64_t)g.B * g.Ho * g.Wo;
    if (M <= 0) return 0;
    dim3 grid((unsigned)ceil_div(M, CB_M), (unsigned)ceil_div(g.Cout, CB_N));
    if (wdtype == RQB200_F32)
        conv_igemm_kernel<float><<<grid, C_THREADS, 0, st>>>(X, (const float*)W, bias, R, Y, g);
    else if (wdtype == RQB200_F16)
        conv_igemm_kernel<__half><<<grid, C_THREADS, 0, st>>>(X, (const __half*)W, bias, R, Y, g);
    else if (wdtype == RQB200_BF16)
        conv_igemm_kernel<__nv_bfloat16><<<grid, C_THREADS, 0, st>>>(X, (const __nv_bfloat16*)W, bias, R, Y, g);
    else
        return fail(RQB200_EINVAL, "conv: unsupported weight dtype");
    return check_launch("conv_igemm");
}

// conv + bias + ReLU of the Inception engine (conv_igemm_kernel<float, true>): fp32 weights, NHWC input (or NCHW when g.in_nchw),
// output rows of g.ldy floats from channel g.yoff
int launch_conv_relu(const float* X, const float* W, const float* bias, float* Y, const ConvGeom& g, cudaStream_t st) {
    const int64_t M = (int64_t)g.B * g.Ho * g.Wo;
    if (M <= 0) return 0;
    dim3 grid((unsigned)ceil_div(M, CB_M), (unsigned)ceil_div(g.Cout, CB_N));
    conv_igemm_kernel<float, true><<<grid, C_THREADS, 0, st>>>(X, W, bias, nullptr, Y, g);
    return check_launch("conv_igemm_relu");
}

// the residual forms of the same conv (the ResNet engine): Y = act(conv + bias + R), R (nullable) fp32 rows of g.ldy floats read at the
// output's own index; act = ReLU when relu, else the identity
int launch_conv_res(const float* X, const float* W, const float* bias, const float* R, float* Y, const ConvGeom& g, bool relu,
                    cudaStream_t st) {
    const int64_t M = (int64_t)g.B * g.Ho * g.Wo;
    if (M <= 0) return 0;
    dim3 grid((unsigned)ceil_div(M, CB_M), (unsigned)ceil_div(g.Cout, CB_N));
    if (relu) conv_igemm_res_kernel<true><<<grid, C_THREADS, 0, st>>>(X, W, bias, R, Y, g);
    else conv_igemm_res_kernel<false><<<grid, C_THREADS, 0, st>>>(X, W, bias, R, Y, g);
    return check_launch("conv_igemm_res");
}

// ------------------------------------------------------------------------------------------------ GroupNorm(32) (+SiLU)
constexpr int GN_PIX = 256;       // pixels per CTA
constexpr int GN_G = 32;

// partial statistics: one (sum, sum of squares) pair per group and per chunk of 32 pixels (the conv epilogue's granularity; the
// stand-alone gn_stats_kernel uses every 8th slot's worth), then the finalised (mean, rstd) pairs
size_t groupnorm_ws_doubles(int B, int HW) { return (size_t)B * ceil_div(HW, 32) * GN_G * 2 + (size_t)B * GN_G * 2; }

// lane == group: a warp reads one pixel's C contiguous channels, lane l owns channels [l*cg, (l+1)*cg)
__global__ void __launch_bounds__(256) gn_stats_kernel(const float* __restrict__ X, double* __restrict__ part, int HW, int C) {
    __shared__ double sh[8][GN_G][2];
    const int b = blockIdx.y, chunk = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int cg = C / GN_G;
    const int p0 = chunk * GN_PIX, p1 = min(p0 + GN_PIX, HW);
    double s = 0.0, ss = 0.0;
    for (int p = p0 + warp; p < p1; p += 8) {
        const float* px = X + ((int64_t)b * HW + p) * C + lane * cg;
        float a = 0.f, a2 = 0.f;
        if ((cg & 3) == 0) {
            for (int i = 0; i < cg; i += 4) {
                float4 v = *reinterpret_cast<const float4*>(px + i);
                a += (v.x + v.y) + (v.z + v.w);
                a2 = fmaf(v.x, v.x, a2); a2 = fmaf(v.y, v.y, a2); a2 = fmaf(v.z, v.z, a2); a2 = fmaf(v.w, v.w, a2);
            }
        } else {
            for (int i = 0; i < cg; i++) { float v = px[i]; a += v; a2 = fmaf(v, v, a2); }
        }
        s += (double)a;
        ss += (double)a2;
    }
    sh[warp][lane][0] = s;
    sh[warp][lane][1] = ss;
    __syncthreads();
    if (warp == 0) {
        double ts = 0.0, tss = 0.0;
        for (int w = 0; w < 8; w++) { ts += sh[w][lane][0]; tss += sh[w][lane][1]; }
        double* o = part + (((int64_t)b * gridDim.x + chunk) * GN_G + lane) * 2;
        o[0] = ts;
        o[1] = tss;
    }
}

__global__ void __launch_bounds__(256) gn_apply_kernel(const float* __restrict__ X, const double* __restrict__ part,
                                                       const float* __restrict__ gamma, const float* __restrict__ beta,
                                                       float* __restrict__ Y, int HW, int C, float eps, int silu) {
    __shared__ float s_mean[GN_G], s_rstd[GN_G];
    const int b = blockIdx.y, chunk = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int cg = C / GN_G;
    if (warp == 0) {
        double ts = 0.0, tss = 0.0;
        for (unsigned c = 0; c < gridDim.x; c++) {
            const double* o = part + (((int64_t)b * gridDim.x + c) * GN_G + lane) * 2;
            ts += o[0];
            tss += o[1];
        }
        double n = (double)HW * cg, mean = ts / n, var = tss / n - mean * mean;
        if (var < 0.0) var = 0.0;
        s_mean[lane] = (float)mean;
        s_rstd[lane] = (float)(1.0 / sqrt(var + (double)eps));
    }
    __syncthreads();
    const float mean = s_mean[lane], rstd = s_rstd[lane];
    const int p0 = chunk * GN_PIX, p1 = min(p0 + GN_PIX, HW);
    for (int p = p0 + warp; p < p1; p += 8) {
        const int64_t base = ((int64_t)b * HW + p) * C + lane * cg;
        for (int i = 0; i < cg; i++) {
            int c = lane * cg + i;
            float scale = rstd * gamma[c];
            float shift = fmaf(-scale, mean, beta[c]);
            float v = fmaf(X[base + i], scale, shift);
            if (silu) v = v / (1.0f + expf(-v));
            Y[base + i] = v;
        }
    }
}

int launch_gn_stats(const float* X, double* stats_ws, int B, int HW, int C, cudaStream_t st) {
    if (C % GN_G != 0) return fail(RQB200_EINVAL, "groupnorm: C % 32 != 0");
    gn_stats_kernel<<<dim3((unsigned)ceil_div(HW, GN_PIX), B), 256, 0, st>>>(X, stats_ws, HW, C);
    return check_launch("gn_stats");
}

int launch_groupnorm_silu(const float* X, const float* gamma, const float* beta, float* Y, double* stats_ws, int B, int HW,
                          int C, int silu, cudaStream_t st) {
    if (C % GN_G != 0) return fail(RQB200_EINVAL, "groupnorm: C % 32 != 0");
    dim3 grid((unsigned)ceil_div(HW, GN_PIX), B);
    gn_stats_kernel<<<grid, 256, 0, st>>>(X, stats_ws, HW, C);
    RQB_TRY(check_launch("gn_stats"));
    gn_apply_kernel<<<grid, 256, 0, st>>>(X, stats_ws, gamma, beta, Y, HW, C, 1e-6f, silu);
    return check_launch("gn_apply");
}

// ------------------------------------------------------------------------------------------------ AttnBlock core
// qkv [B, HW, 3C] (q | k | v per pixel); out [B, HW, C].  One CTA per (query pixel, image).
__global__ void __launch_bounds__(256) vae_attn_kernel(const float* __restrict__ qkv, float* __restrict__ out, int HW, int C,
                                                       float scale) {
    extern __shared__ float sm[];
    float* qs = sm;          // [C]
    float* sc = sm + C;      // [HW]
    __shared__ float red[33];
    const int i = blockIdx.x, b = blockIdx.y, t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const float* base = qkv + (int64_t)b * HW * 3 * C;
    for (int c = t; c < C; c += 256) qs[c] = base[(int64_t)i * 3 * C + c];
    __syncthreads();
    for (int j = warp; j < HW; j += 8) {
        const float* kr = base + (int64_t)j * 3 * C + C;
        float a = 0.f;
        for (int c = lane; c < C; c += 32) a = fmaf(qs[c], kr[c], a);
        a = warp_sum(a);
        if (lane == 0) sc[j] = a * scale;                       // w_ = bmm(q,k) * c^-0.5   (layers.py:170-171)
    }
    __syncthreads();
    float m = -INFINITY;
    for (int j = t; j < HW; j += 256) m = fmaxf(m, sc[j]);
    m = block_max(m, red);
    float s = 0.f;
    for (int j = t; j < HW; j += 256) { float e = expf(sc[j] - m); sc[j] = e; s += e; }
    s = block_sum(s, red);
    __syncthreads();
    for (int j = t; j < HW; j += 256) sc[j] = sc[j] / s;
    __syncthreads();
    for (int c = t; c < C; c += 256) {
        float a = 0.f;
        for (int j = 0; j < HW; j++) a = fmaf(sc[j], base[(int64_t)j * 3 * C + 2 * C + c], a);
        out[((int64_t)b * HW + i) * C + c] = a;
    }
}

int launch_vae_attn(const float* qkv, float* out, int B, int HW, int C, cudaStream_t st) {
    // the dynamic [C + HW] floats must fit beside the kernel's static shared memory in the 48 KB a launch takes without an opt-in
    static const size_t max_dyn = [] {
        cudaFuncAttributes a{};
        if (cudaFuncGetAttributes(&a, vae_attn_kernel) != cudaSuccess) { cudaGetLastError(); return (size_t)0; }
        return std::min((size_t)a.maxDynamicSharedSizeBytes, 48 * 1024 - a.sharedSizeBytes);
    }();
    size_t smem = (size_t)(C + HW) * sizeof(float);
    if (smem > max_dyn) return fail(RQB200_EINVAL, "vae_attn: C + HW too large");
    float scale = (float)(1.0 / sqrt((double)C));                  // int(c) ** (-0.5) evaluated in double, then cast
    vae_attn_kernel<<<dim3(HW, B), 256, smem, st>>>(qkv, out, HW, C, scale);
    return check_launch("vae_attn");
}

}  // namespace rqb
