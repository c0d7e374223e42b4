// CLIP ViT image and text encoders (OpenAI's model definition, the reference's rqvae/metrics/clip_score.py) as a static layer plan.
//
// Vision: preprocessing (Pillow's 8-bit bicubic resize, centre crop, normalise) writes conv1's operand rows directly; conv1 (stride P,
// no bias) is one GEMM with K = 3 P^2 (padded to a multiple of 64 with zero columns); class token + positional embedding; ln_pre;
// L residual blocks (LN -> in_proj -> non-causal MHA -> out_proj + x, LN -> c_fc -> QuickGELU -> c_proj + x); ln_post on token 0;
// @ visual.proj.  Text: token_embedding + positional_embedding; L blocks with the causal mask; the row at tokens.argmax(-1);
// ln_final; @ text_projection.  Rows are token-major (row = t * G + g), as prefill_attn_flash_kernel reads them.
//
// Exact tier: fp32 FFMA everywhere (linear_nt_kernel, layernorm_kernel, clip_attn_f32_kernel).  Fast tier: fp16 operands on the GEMMs
// the AR engine's batched pass would pick (the persistent rows GEMM above 256 rows, else the weight streamer), fp32 accumulate,
// fp32 residual stream, LayerNorm and softmax; the pooled LayerNorm, both projections and the cosine are fp32 on both tiers.
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "kernels.h"

namespace rqb {

// ------------------------------------------------------------------------------------------------ preprocessing
// CLIP's Normalize constants, rounded to fp32 as torch.as_tensor(mean) rounds them
__constant__ float c_clip_mean[3] = {0.48145466f, 0.4578275f, 0.40821073f};
__constant__ float c_clip_std[3] = {0.26862954f, 0.26130258f, 0.27577711f};

// (pixel * 255).astype(np.uint8) on a clamped fp32 pixel: an fp32 multiply, then truncation
__device__ __forceinline__ int clip_u8(float x) { return (int)__fmul_rn(fminf(fmaxf(x, 0.f), 1.f), 255.f); }
// Pillow's clip8 of a fixed-point accumulator (22 fraction bits)
__device__ __forceinline__ int clip_px(int v) { return v >= (255 << 22) ? 255 : (v <= 0 ? 0 : (v >> 22)); }

// One resample axis restricted to the R output positions of the crop: for output i, taps [lo[i], lo[i] + n[i]) of the input with
// fixed-point weights k[i * ks + j].  ks == 0: no pass along this axis (the extent already equals R); output i reads input off + i.
struct ClipAxis {
    const int* lo;
    const int* n;
    const int* k;
    int ks, off;
};

// horizontal pass: x NCHW fp32 [B, 3, H, W] -> tmp uint8 [B, 3, H, R] (the crop's R columns of the horizontally resized image)
__global__ void __launch_bounds__(256) clip_resize_h_kernel(const float* __restrict__ x, uint8_t* __restrict__ tmp, int B, int H, int W, int R,
                                                             ClipAxis ax) {
    const int64_t total = (int64_t)B * 3 * H * R;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
        const int c = (int)(i % R);
        const int64_t row = i / R;                             // (b, ch, y)
        const float* src = x + row * W;
        int v;
        if (ax.ks == 0) {
            v = clip_u8(src[ax.off + c]);
        } else {
            int ss = 1 << 21;
            const int lo = ax.lo[c], n = ax.n[c];
            const int* k = ax.k + (int64_t)c * ax.ks;
            for (int j = 0; j < n; j++) ss += clip_u8(src[lo + j]) * k[j];
            v = clip_px(ss);
        }
        tmp[i] = (uint8_t)v;
    }
}

// vertical pass + ToTensor + Normalize: tmp [B, 3, H, R] -> u (optional uint8 [B, 3, R, R]), nchw (optional fp32 [B, 3, R, R]), and
// conv1's operand rows: patch p = (y / P) * (R / P) + x / P of image b is row p * B + b of rows [*, ld], column (ch * P + y % P) * P + x % P,
// fp32 (rows32) or fp16 (rows16)
__global__ void __launch_bounds__(256) clip_resize_v_kernel(const uint8_t* __restrict__ tmp, int B, int H, int R, ClipAxis ax, uint8_t* u8,
                                                             float* nchw, float* rows32, __half* rows16, int P, int ld) {
    const int64_t total = (int64_t)B * 3 * R * R;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
        const int xx = (int)(i % R), y = (int)((i / R) % R), ch = (int)((i / ((int64_t)R * R)) % 3);
        const int b = (int)(i / (3LL * R * R));
        const uint8_t* src = tmp + ((int64_t)b * 3 + ch) * H * R + xx;
        int v;
        if (ax.ks == 0) {
            v = src[(int64_t)(ax.off + y) * R];
        } else {
            int ss = 1 << 21;
            const int lo = ax.lo[y], n = ax.n[y];
            const int* k = ax.k + (int64_t)y * ax.ks;
            for (int j = 0; j < n; j++) ss += (int)src[(int64_t)(lo + j) * R] * k[j];
            v = clip_px(ss);
        }
        if (u8) u8[i] = (uint8_t)v;
        const float f = __fdiv_rn(__fsub_rn(__fdiv_rn((float)v, 255.f), c_clip_mean[ch]), c_clip_std[ch]);
        if (nchw) nchw[i] = f;
        if (rows32 || rows16) {
            const int g = R / P;
            const int64_t r = ((int64_t)(y / P) * g + xx / P) * B + b;
            const int col = (ch * P + y % P) * P + xx % P;
            if (rows32) rows32[r * ld + col] = f;
            else rows16[r * ld + col] = __float2half_rn(f);
        }
    }
}

// Pillow's precompute_coeffs + normalize_coeffs_8bpc (bicubic, a = -0.5, support 2) for in -> out, kept for the outputs
// [off, off + R): lo / n the taps, k the fixed-point weights (ks per output).  Returns ks.
static double pil_bicubic(double x) {
    const double a = -0.5;
    if (x < 0.0) x = -x;
    if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
    if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
    return 0.0;
}
static int pil_coeffs(int in, int out, int off, int R, std::vector<int>& lo, std::vector<int>& n, std::vector<int>& k) {
    const double scale = (double)in / out;
    const double filterscale = scale < 1.0 ? 1.0 : scale;
    const double support = 2.0 * filterscale;
    const int ks = (int)std::ceil(support) * 2 + 1;
    lo.assign(R, 0);
    n.assign(R, 0);
    k.assign((size_t)R * ks, 0);
    std::vector<double> w(ks);
    for (int i = 0; i < R; i++) {
        const int xx = off + i;
        const double center = (xx + 0.5) * scale;
        const double ss = 1.0 / filterscale;
        int xmin = (int)(center - support + 0.5);
        if (xmin < 0) xmin = 0;
        int xmax = (int)(center + support + 0.5);
        if (xmax > in) xmax = in;
        xmax -= xmin;
        double ww = 0.0;
        for (int x = 0; x < xmax; x++) {
            w[x] = pil_bicubic((x + xmin - center + 0.5) * ss);
            ww += w[x];
        }
        for (int x = 0; x < xmax; x++) {
            const double v = ww != 0.0 ? w[x] / ww : w[x];
            k[(size_t)i * ks + x] = v < 0 ? (int)(-0.5 + v * (1 << 22)) : (int)(0.5 + v * (1 << 22));
        }
        lo[i] = xmin;
        n[i] = xmax;
    }
    return ks;
}

// torchvision Resize(R) (the shorter side becomes R, the longer int(R * long / short)) then CenterCrop(R) (offset round-half-even
// of (n - R) / 2, as Python's round)
static void clip_geometry(int H, int W, int R, int* Hr, int* Wr, int* top, int* left) {
    if (W <= H) { *Wr = R; *Hr = (int)((double)R * H / W); }
    else { *Hr = R; *Wr = (int)((double)R * W / H); }
    *top = (int)std::nearbyint((*Hr - R) / 2.0);
    *left = (int)std::nearbyint((*Wr - R) / 2.0);
}

// ------------------------------------------------------------------------------------------------ small kernels
// x[t * G + g] = (t == 0 ? cls : x[t * G + g]) + pos[t]   (vision: class token + positional embedding; rows 1.. hold conv1's output)
__global__ void __launch_bounds__(256) clip_vis_embed_kernel(float* __restrict__ x, const float* __restrict__ cls, const float* __restrict__ pos,
                                                              int G, int T, int E) {
    const int64_t total = (int64_t)T * G * E;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
        const int e = (int)(i % E);
        const int t = (int)(i / ((int64_t)G * E));
        x[i] = (t == 0 ? cls[e] : x[i]) + pos[(int64_t)t * E + e];
    }
}

// x[t * N + n] = tok_emb[tokens[n, t]] + pos[t]; an id outside [0, V) gives NaN (the Python layer rejects them first)
__global__ void __launch_bounds__(256) clip_txt_embed_kernel(float* __restrict__ x, const int64_t* __restrict__ tokens, const float* __restrict__ emb,
                                                              const float* __restrict__ pos, int N, int T, int E, int V) {
    const int64_t total = (int64_t)T * N * E;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
        const int e = (int)(i % E);
        const int n = (int)((i / E) % N), t = (int)(i / ((int64_t)N * E));
        const int64_t id = tokens[(int64_t)n * T + t];
        x[i] = (id >= 0 && id < V) ? emb[id * E + e] + pos[(int64_t)t * E + e] : NAN;
    }
}

// out[n] = x[(argmax_t tokens[n, t]) * N + n] (the first maximum, as torch.argmax): one warp per caption
__global__ void __launch_bounds__(128) clip_eot_gather_kernel(const float* __restrict__ x, const int64_t* __restrict__ tokens, float* __restrict__ out,
                                                               int N, int T, int E) {
    const int n = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (n >= N) return;
    int64_t best = INT64_MIN;
    int at = 0;
    for (int t = lane; t < T; t += 32) {
        const int64_t v = tokens[(int64_t)n * T + t];
        if (v > best) { best = v; at = t; }
    }
    for (int o = 16; o > 0; o >>= 1) {
        const int64_t ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oa = __shfl_xor_sync(0xffffffffu, at, o);
        if (ob > best || (ob == best && oa < at)) { best = ob; at = oa; }
    }
    const float* src = x + ((int64_t)at * N + n) * E;
    for (int e = lane; e < E; e += 32) out[(int64_t)n * E + e] = src[e];
}

__global__ void __launch_bounds__(256) clip_quick_gelu_kernel(float* __restrict__ h, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) h[i] = quick_gelu(h[i]);
}

// Exact-tier attention, fp32 FFMA: qkv [T * G, 3E] (bias added, token-major), head dim 64, scale 1/8 on q; out [T * G, E].  One warp
// per (query, group, head), lane <-> dims (2 lane, 2 lane + 1); the row's scores sit in shared memory (T floats per warp).
__global__ void __launch_bounds__(128) clip_attn_f32_kernel(const float* __restrict__ qkv, float* __restrict__ out, int G, int T, int E,
                                                             int causal) {
    extern __shared__ float clip_sc[];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int nh = E / 64, g = blockIdx.y / nh, h = blockIdx.y % nh;
    const int t = blockIdx.x * 4 + w;
    if (t >= T) return;
    float* s = clip_sc + w * T;
    const int64_t ld = 3LL * E;
    const float* base = qkv + (int64_t)g * ld + h * 64 + 2 * lane;
    const float2 q = *reinterpret_cast<const float2*>(base + (int64_t)t * G * ld);
    const float qx = q.x * 0.125f, qy = q.y * 0.125f;
    const int nk = causal ? t + 1 : T;
    float mx = -INFINITY;
    int j = 0;
    for (; j + 4 <= nk; j += 4) {
        float d[4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const float2 k = *reinterpret_cast<const float2*>(base + (int64_t)(j + u) * G * ld + E);
            d[u] = fmaf(qy, k.y, qx * k.x);
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
            d[u] = warp_sum(d[u]);
            mx = fmaxf(mx, d[u]);
        }
        if (lane == 0) { s[j] = d[0]; s[j + 1] = d[1]; s[j + 2] = d[2]; s[j + 3] = d[3]; }
    }
    for (; j < nk; j++) {
        const float2 k = *reinterpret_cast<const float2*>(base + (int64_t)j * G * ld + E);
        const float d = warp_sum(fmaf(qy, k.y, qx * k.x));
        mx = fmaxf(mx, d);
        if (lane == 0) s[j] = d;
    }
    __syncwarp();
    float sum = 0.f;
    for (int i = lane; i < nk; i += 32) {
        const float e = expf(s[i] - mx);
        s[i] = e;
        sum += e;
    }
    sum = warp_sum(sum);
    __syncwarp();
    float ox = 0.f, oy = 0.f;
    for (int i = 0; i < nk; i++) {
        const float2 v = *reinterpret_cast<const float2*>(base + (int64_t)i * G * ld + 2 * E);
        ox = fmaf(s[i], v.x, ox);
        oy = fmaf(s[i], v.y, oy);
    }
    *reinterpret_cast<float2*>(out + ((int64_t)t * G + g) * E + h * 64 + 2 * lane) = make_float2(ox / sum, oy / sum);
}

int launch_clip_attn_f32(const float* qkv, float* out, int G, int T, int E, bool causal, cudaStream_t st) {
    if (E % 64 != 0 || T < 1 || G < 1) return fail(RQB200_EINVAL, "clip_attn: need E % 64 == 0, T >= 1, G >= 1");
    const size_t smem = (size_t)4 * T * sizeof(float);
    if (smem > 48 * 1024) return fail(RQB200_EINVAL, "clip_attn: T > 3072");
    clip_attn_f32_kernel<<<dim3((unsigned)ceil_div(T, 4), (unsigned)(G * (E / 64))), 128, smem, st>>>(qkv, out, G, T, E, causal ? 1 : 0);
    return check_launch("clip_attn_f32");
}

// F.cosine_similarity(a, b) per row: sum((a / max(|a|, eps)) * (b / max(|b|, eps))), eps 1e-8.  One warp per row.
__global__ void __launch_bounds__(128) clip_cosine_kernel(const float* __restrict__ a, const float* __restrict__ b, int n, int dim,
                                                           float* __restrict__ out) {
    const int r = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (r >= n) return;
    const float* x = a + (int64_t)r * dim;
    const float* y = b + (int64_t)r * dim;
    float sa = 0.f, sb = 0.f;
    for (int i = lane; i < dim; i += 32) { sa = fmaf(x[i], x[i], sa); sb = fmaf(y[i], y[i], sb); }
    const float na = fmaxf(sqrtf(warp_sum(sa)), 1e-8f), nb = fmaxf(sqrtf(warp_sum(sb)), 1e-8f);
    float d = 0.f;
    for (int i = lane; i < dim; i += 32) d = fmaf(__fdiv_rn(x[i], na), __fdiv_rn(y[i], nb), d);
    d = warp_sum(d);
    if (lane == 0) out[r] = d;
}

// ------------------------------------------------------------------------------------------------ the engine
// one linear layer: fp32 weight [N, K] and bias (the caller's tensors) and, fast tier, its fp16 copy behind a streamer tensor map
struct ClipLinear {
    const float* w = nullptr;
    const float* b = nullptr;
    int N = 0, K = 0;
    int64_t h_off = -1;            // fp16 copy at this element offset of the fp16 parameter region
    StreamedWeight sw;
};
struct ClipBlock {
    const float *ln1_w, *ln1_b, *ln2_w, *ln2_b;
    ClipLinear qkv, proj, fc, cproj;
};
struct ClipTower {
    std::string pre;               // "visual." or ""
    int width, layers, T;
    std::vector<ClipBlock> blocks;
    const float *lnf_w = nullptr, *lnf_b = nullptr;   // ln_post / ln_final
    const float* projT = nullptr;  // [embed, width] fp32 (params)
};

}  // namespace rqb

struct rqb200_clip {
    rqb200_clip_config cfg;
    bool fast = false;
    rqb::TensorTable t;
    rqb::ClipTower vis, txt;
    int Kp = 0;                    // conv1's K = 3 P^2, padded to a multiple of 64
    rqb::ClipLinear conv1;         // w = [width, Kp] fp32 in params (zero-padded), b = zeros
    int64_t f32_floats = 0, f16_elems = 0;
    bool finalized = false;
    int64_t last_launches = 0;
};

namespace rqb {

static int64_t clip_h_elems(const rqb200_clip* h) { return h->fast ? h->f16_elems : 0; }

// the parameter layout: fp32 [conv1 padded | conv1 zero bias | visual.proj^T | text_projection^T], then (fast) fp16 copies of every
// transformer GEMM weight and conv1
static void clip_plan(rqb200_clip* h) {
    const rqb200_clip_config& c = h->cfg;
    const int P = c.vision_patch;
    h->Kp = (int)ceil_div(3 * P * P, 64) * 64;
    int64_t f = 0, e = 0;
    h->conv1.N = c.vision_width; h->conv1.K = h->Kp;
    f = (int64_t)c.vision_width * h->Kp + c.vision_width + (int64_t)c.embed_dim * (c.vision_width + c.text_width);
    h->conv1.h_off = e;
    e += (int64_t)c.vision_width * h->Kp;
    auto tower = [&](ClipTower& tw, const char* pre, int width, int layers, int T) {
        tw.pre = pre; tw.width = width; tw.layers = layers; tw.T = T;
        tw.blocks.assign(layers, ClipBlock{});
        for (ClipBlock& b : tw.blocks) {
            ClipLinear* ls[4] = {&b.qkv, &b.proj, &b.fc, &b.cproj};
            const int NK[4][2] = {{3 * width, width}, {width, width}, {4 * width, width}, {width, 4 * width}};
            for (int i = 0; i < 4; i++) {
                ls[i]->N = NK[i][0]; ls[i]->K = NK[i][1]; ls[i]->h_off = e;
                e += (int64_t)NK[i][0] * NK[i][1];
            }
        }
    };
    const int g = c.vision_resolution / P;
    tower(h->vis, "visual.", c.vision_width, c.vision_layers, g * g + 1);
    tower(h->txt, "", c.text_width, c.text_layers, c.context_length);
    h->f32_floats = f;
    h->f16_elems = e;
}

__global__ void clip_pack_kernel(const float* __restrict__ src, int rows, int cols, int ld_dst, int transpose, float* dst32, __half* dst16) {
    const int64_t total = (int64_t)rows * cols;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
        const int r = (int)(i / cols), cc = (int)(i % cols);
        const float v = src[i];
        const int64_t o = transpose ? (int64_t)cc * ld_dst + r : (int64_t)r * ld_dst + cc;
        if (dst32) dst32[o] = v;
        if (dst16) dst16[o] = __float2half_rn(v);
    }
}
static int clip_pack(const float* src, int rows, int cols, int ld_dst, bool transpose, float* d32, __half* d16, cudaStream_t st) {
    clip_pack_kernel<<<grid_1d((int64_t)rows * cols), 256, 0, st>>>(src, rows, cols, ld_dst, transpose ? 1 : 0, d32, d16);
    return check_launch("clip_pack");
}

// buffers of one encoder call over G sequences of T tokens (M = T G rows; 16-bit buffers padded to whole 128-row tiles)
struct ClipBufs {
    float *X, *XN32, *QKV32, *ATT32, *H32, *pool, *rows32;
    h16 *XN, *QKV, *ATT, *H, *rows16;
    uint8_t* tmp;
    int* tabs;
};
static size_t clip_layout(const rqb200_clip* h, const ClipTower& tw, int G, int pre_rows, int pre_K, int64_t tmp_bytes, int tab_ints,
                          void* base, ClipBufs* b) {
    ClipBufs d;
    if (!b) b = &d;
    *b = ClipBufs{};                       // the other tier's buffers stay null: the kernels pick fp32 or fp16 rows by which is set
    Arena ar{(char*)base, base ? SIZE_MAX : 0};
    const int64_t M = (int64_t)tw.T * G, E = tw.width, Mp = ceil_div(M, 128) * 128;
    b->X = ar.take<float>(M * E);
    b->pool = ar.take<float>((int64_t)G * E);
    if (h->fast) {
        b->XN = ar.take<h16>(Mp * E);
        b->QKV = ar.take<h16>(Mp * 3 * E);
        b->ATT = ar.take<h16>(Mp * E);
        b->H = ar.take<h16>(Mp * 4 * E);
        if (pre_rows) b->rows16 = ar.take<h16>(ceil_div(pre_rows, 128) * 128 * pre_K);
    } else {
        b->XN32 = ar.take<float>(M * E);
        b->QKV32 = ar.take<float>(M * 3 * E);
        b->ATT32 = ar.take<float>(M * E);
        b->H32 = ar.take<float>(M * 4 * E);
        if (pre_rows) b->rows32 = ar.take<float>((int64_t)pre_rows * pre_K);
    }
    if (tmp_bytes) b->tmp = ar.take<uint8_t>(tmp_bytes);
    if (tab_ints) b->tabs = ar.take<int>(tab_ints);
    return ar.off + 256;
}

// one linear layer over M rows.  Exact: out32 = x32 W^T + b (+ res), act 2 = QuickGELU.  Fast: the GEMM linear_rows would pick (rows GEMM
// above 256 rows, else the weight streamer) with fp16 operands; out16 (act 0 or 2) or out32 (+ res, which may alias out32).
static int clip_linear(const rqb200_clip* h, const ClipLinear& L, int64_t M, const float* x32, const h16* x16, float* out32, h16* out16,
                       const float* res, int act, cudaStream_t st) {
    if (!h->fast) {
        RQB_TRY(launch_linear(x32, L.K, L.w, RQB200_F32, L.b, res, out32, L.N, (int)M, L.N, L.K, 0, st));
        if (act == 2) {
            clip_quick_gelu_kernel<<<grid_1d(M * L.N), 256, 0, st>>>(out32, M * L.N);
            RQB_TRY(check_launch("clip_quick_gelu"));
        }
        return 0;
    }
    if (M > 256) return launch_rows_gemm_tc(x16, L.sw.w16, L.b, res, out16 ? nullptr : out32, out16, act, 0, M, L.N, L.K, st);
    CUtensorMap tx;
    RQB_TRY(make_tmap_2d(&tx, x16, 1, (uint64_t)L.K, (uint64_t)M, (uint64_t)L.K * 2, 64, (uint32_t)gemm_tc_chunk_rows(L.sw, M)));
    GemmTcParams p = {};
    p.B = (int)M; p.splits = 1; p.fmt = 0; p.bias = L.b; p.bias_scale = 1.f;
    p.mode = out16 ? (act == 2 ? GT_H16_QGELU : GT_H16) : GT_F32;
    p.out = out16 ? (void*)out16 : (void*)out32;
    p.ld_out = L.N;
    p.residual = res;
    p.ld_res = L.N;
    return launch_gemm_tc(L.sw, tx, p, false, st);
}

// the residual blocks of one tower over G sequences (X holds the embedded, for vision ln_pre'd, rows)
static int clip_blocks(const rqb200_clip* h, const ClipTower& tw, const ClipBufs& b, int G, bool causal, cudaStream_t st) {
    const int E = tw.width, T = tw.T;
    const int64_t M = (int64_t)T * G;
    for (const ClipBlock& k : tw.blocks) {
        if (h->fast) {
            RQB_TRY(launch_ln_rows_f16(M, b.X, k.ln1_w, k.ln1_b, b.XN, E, st));
            RQB_TRY(clip_linear(h, k.qkv, M, nullptr, b.XN, nullptr, b.QKV, nullptr, 0, st));
            RQB_TRY(launch_attn_flash_f16(b.QKV, b.ATT, G, T, E, causal, st));
            RQB_TRY(clip_linear(h, k.proj, M, nullptr, b.ATT, b.X, nullptr, b.X, 0, st));
            RQB_TRY(launch_ln_rows_f16(M, b.X, k.ln2_w, k.ln2_b, b.XN, E, st));
            RQB_TRY(clip_linear(h, k.fc, M, nullptr, b.XN, nullptr, b.H, nullptr, 2, st));
            RQB_TRY(clip_linear(h, k.cproj, M, nullptr, b.H, b.X, nullptr, b.X, 0, st));
        } else {
            RQB_TRY(launch_layernorm(b.X, E, k.ln1_w, k.ln1_b, b.XN32, E, (int)M, E, st));
            RQB_TRY(clip_linear(h, k.qkv, M, b.XN32, nullptr, b.QKV32, nullptr, nullptr, 0, st));
            RQB_TRY(launch_clip_attn_f32(b.QKV32, b.ATT32, G, T, E, causal, st));
            RQB_TRY(clip_linear(h, k.proj, M, b.ATT32, nullptr, b.X, nullptr, b.X, 0, st));
            RQB_TRY(launch_layernorm(b.X, E, k.ln2_w, k.ln2_b, b.XN32, E, (int)M, E, st));
            RQB_TRY(clip_linear(h, k.fc, M, b.XN32, nullptr, b.H32, nullptr, nullptr, 2, st));
            RQB_TRY(clip_linear(h, k.cproj, M, b.H32, nullptr, b.X, nullptr, b.X, 0, st));
        }
    }
    return 0;
}

// the preprocessing tables of an H x W input: horizontal then vertical axis, and the temp buffer's bytes
struct ClipPrep {
    int Hr, Wr, top, left, ksh, ksv;
    std::vector<int> hlo, hn, hk, vlo, vn, vk;
    int tab_ints() const { return (int)(hlo.size() + hn.size() + hk.size() + vlo.size() + vn.size() + vk.size()); }
};
static void clip_prep(int H, int W, int R, ClipPrep* p) {
    clip_geometry(H, W, R, &p->Hr, &p->Wr, &p->top, &p->left);
    p->ksh = p->Wr != W ? pil_coeffs(W, p->Wr, p->left, R, p->hlo, p->hn, p->hk) : 0;
    p->ksv = p->Hr != H ? pil_coeffs(H, p->Hr, p->top, R, p->vlo, p->vn, p->vk) : 0;
}
// tables -> device (the workspace's int region), then the two passes
static int clip_preprocess(const ClipPrep& pp, const float* x, int B, int H, int W, int R, uint8_t* tmp, int* tabs, uint8_t* u8, float* nchw,
                           float* rows32, __half* rows16, int P, int ld, cudaStream_t st) {
    std::vector<int> all;
    for (const std::vector<int>* v : {&pp.hlo, &pp.hn, &pp.hk, &pp.vlo, &pp.vn, &pp.vk}) all.insert(all.end(), v->begin(), v->end());
    if (!all.empty()) RQB_CUDA(cudaMemcpyAsync(tabs, all.data(), all.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    // pageable source: cudaMemcpyAsync has staged it before returning, so `all` may go
    const int* q = tabs;
    ClipAxis ah{q, q + pp.hlo.size(), q + pp.hlo.size() + pp.hn.size(), pp.ksh, pp.left};
    q += pp.hlo.size() + pp.hn.size() + pp.hk.size();
    ClipAxis av{q, q + pp.vlo.size(), q + pp.vlo.size() + pp.vn.size(), pp.ksv, pp.top};
    clip_resize_h_kernel<<<grid_1d((int64_t)B * 3 * H * R), 256, 0, st>>>(x, tmp, B, H, W, R, ah);
    RQB_TRY(check_launch("clip_resize_h"));
    clip_resize_v_kernel<<<grid_1d((int64_t)B * 3 * R * R), 256, 0, st>>>(tmp, B, H, R, av, u8, nchw, rows32, rows16, P, ld);
    return check_launch("clip_resize_v");
}

// rows [t * G + g] of an already-normalised [G, 3, R, R] batch -> conv1 operand rows (no resize: an identity "resample")
__global__ void __launch_bounds__(256) clip_patch_rows_kernel(const float* __restrict__ x, int B, int R, int P, int ld, float* rows32,
                                                               __half* rows16) {
    const int64_t total = (int64_t)B * 3 * R * R;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
        const int xx = (int)(i % R), y = (int)((i / R) % R), ch = (int)((i / ((int64_t)R * R)) % 3);
        const int b = (int)(i / (3LL * R * R));
        const int64_t r = ((int64_t)(y / P) * (R / P) + xx / P) * B + b;
        const int col = (ch * P + y % P) * P + xx % P;
        if (rows32) rows32[r * ld + col] = x[i];
        else rows16[r * ld + col] = __float2half_rn(x[i]);
    }
}

}  // namespace rqb

extern "C" {

rqb200_clip* rqb200_clip_create(const rqb200_clip_config* cfg) {
    using namespace rqb;
    if (!cfg) { set_error("clip_create: null config"); return nullptr; }
    const rqb200_clip_config& c = *cfg;
    if (c.mode != RQB200_MODE_EXACT && c.mode != RQB200_MODE_FAST) { set_error("clip_create: mode must be RQB200_MODE_EXACT or RQB200_MODE_FAST"); return nullptr; }
    if (c.vision_width < 64 || c.vision_width % 64 || c.text_width < 64 || c.text_width % 64) {
        set_error("clip_create: vision and text widths must be positive multiples of 64 (head dim 64)");
        return nullptr;
    }
    if (c.mode == RQB200_MODE_FAST && (c.vision_width % 128 || c.text_width % 128)) {
        set_error("clip_create: the fast tier needs widths that are multiples of 128");
        return nullptr;
    }
    if (c.vision_layers < 1 || c.text_layers < 1 || c.vision_patch < 1 || c.vision_resolution < c.vision_patch ||
        c.vision_resolution % c.vision_patch || c.context_length < 1 || c.vocab_size < 1 || c.embed_dim < 1) {
        set_error("clip_create: bad geometry (layers >= 1, resolution a multiple of the patch, context, vocab and embed_dim >= 1)");
        return nullptr;
    }
    rqb200_clip* h = new rqb200_clip();
    h->cfg = c;
    h->fast = c.mode == RQB200_MODE_FAST;
    clip_plan(h);
    return h;
}
void rqb200_clip_destroy(rqb200_clip* h) { delete h; }

int rqb200_clip_set_tensor(rqb200_clip* h, const char* key, const void* ptr, int dtype, int64_t numel) {
    if (!h || !key || !ptr) return rqb::fail(RQB200_EINVAL, "clip_set_tensor: null argument");
    h->t.set(key, ptr, dtype, numel);
    h->finalized = false;
    return 0;
}

size_t rqb200_clip_params_bytes(const rqb200_clip* h) {
    return h ? (size_t)h->f32_floats * sizeof(float) + (size_t)rqb::clip_h_elems(h) * sizeof(__half) + 256 : 0;
}

int rqb200_clip_finalize(rqb200_clip* h, void* params, size_t params_bytes, void* stream) {
    using namespace rqb;
    if (!h) return fail(RQB200_EINVAL, "clip_finalize: null handle");
    h->finalized = false;
    const rqb200_clip_config& c = h->cfg;
    auto get = [h](const std::string& k, int64_t numel, const float** out) { return h->t.get_f32("clip_finalize", k, numel, out); };
    const int vw = c.vision_width, tw = c.text_width, P = c.vision_patch, D = c.embed_dim;
    const float *conv1 = nullptr, *cls = nullptr, *vpos = nullptr, *lnpre_w = nullptr, *lnpre_b = nullptr, *vproj = nullptr;
    const float *tok = nullptr, *tpos = nullptr, *tproj = nullptr;
    RQB_TRY(get("visual.conv1.weight", (int64_t)vw * 3 * P * P, &conv1));
    RQB_TRY(get("visual.class_embedding", vw, &cls));
    RQB_TRY(get("visual.positional_embedding", (int64_t)h->vis.T * vw, &vpos));
    RQB_TRY(get("visual.ln_pre.weight", vw, &lnpre_w));
    RQB_TRY(get("visual.ln_pre.bias", vw, &lnpre_b));
    for (ClipTower* T : {&h->vis, &h->txt}) {
        const int E = T->width;
        for (int l = 0; l < T->layers; l++) {
            ClipBlock& b = T->blocks[l];
            const std::string p = T->pre + "transformer.resblocks." + std::to_string(l) + ".";
            RQB_TRY(get(p + "ln_1.weight", E, &b.ln1_w));
            RQB_TRY(get(p + "ln_1.bias", E, &b.ln1_b));
            RQB_TRY(get(p + "attn.in_proj_weight", 3LL * E * E, &b.qkv.w));
            RQB_TRY(get(p + "attn.in_proj_bias", 3LL * E, &b.qkv.b));
            RQB_TRY(get(p + "attn.out_proj.weight", (int64_t)E * E, &b.proj.w));
            RQB_TRY(get(p + "attn.out_proj.bias", E, &b.proj.b));
            RQB_TRY(get(p + "ln_2.weight", E, &b.ln2_w));
            RQB_TRY(get(p + "ln_2.bias", E, &b.ln2_b));
            RQB_TRY(get(p + "mlp.c_fc.weight", 4LL * E * E, &b.fc.w));
            RQB_TRY(get(p + "mlp.c_fc.bias", 4LL * E, &b.fc.b));
            RQB_TRY(get(p + "mlp.c_proj.weight", 4LL * E * E, &b.cproj.w));
            RQB_TRY(get(p + "mlp.c_proj.bias", E, &b.cproj.b));
        }
    }
    RQB_TRY(get("visual.ln_post.weight", vw, &h->vis.lnf_w));
    RQB_TRY(get("visual.ln_post.bias", vw, &h->vis.lnf_b));
    RQB_TRY(get("visual.proj", (int64_t)vw * D, &vproj));
    RQB_TRY(get("token_embedding.weight", (int64_t)c.vocab_size * tw, &tok));
    RQB_TRY(get("positional_embedding", (int64_t)c.context_length * tw, &tpos));
    RQB_TRY(get("ln_final.weight", tw, &h->txt.lnf_w));
    RQB_TRY(get("ln_final.bias", tw, &h->txt.lnf_b));
    RQB_TRY(get("text_projection", (int64_t)tw * D, &tproj));
    if (!params) return fail(RQB200_EINVAL, "clip_finalize: null parameter buffer");
    if (params_bytes < rqb200_clip_params_bytes(h)) return fail(RQB200_EWORKSPACE, "clip_finalize: parameter buffer smaller than rqb200_clip_params_bytes");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "clip_finalize: no CUDA device");
    const cudaStream_t st = (cudaStream_t)stream;
    float* F = (float*)params;
    __half* Hh = h->fast ? (__half*)(((uintptr_t)(F + h->f32_floats) + 255) & ~(uintptr_t)255) : nullptr;
    float* conv1_p = F;
    float* zero_b = conv1_p + (int64_t)vw * h->Kp;
    float* vprojT = zero_b + vw;
    float* tprojT = vprojT + (int64_t)D * vw;
    RQB_CUDA(cudaMemsetAsync(conv1_p, 0, ((int64_t)vw * h->Kp + vw) * sizeof(float), st));
    RQB_TRY(clip_pack(conv1, vw, 3 * P * P, h->Kp, false, conv1_p, Hh ? Hh + h->conv1.h_off : nullptr, st));
    if (Hh) RQB_TRY(clip_pack(conv1_p, vw, h->Kp, h->Kp, false, nullptr, Hh + h->conv1.h_off, st));    // (the zero columns too)
    RQB_TRY(clip_pack(vproj, vw, D, vw, true, vprojT, nullptr, st));
    RQB_TRY(clip_pack(tproj, tw, D, tw, true, tprojT, nullptr, st));
    h->conv1.w = conv1_p;
    h->conv1.b = zero_b;
    h->vis.projT = vprojT;
    h->txt.projT = tprojT;
    std::vector<ClipLinear*> all = {&h->conv1};
    for (ClipTower* T : {&h->vis, &h->txt})
        for (ClipBlock& b : T->blocks)
            for (ClipLinear* L : {&b.qkv, &b.proj, &b.fc, &b.cproj}) all.push_back(L);
    if (Hh) {
        for (size_t i = 1; i < all.size(); i++) RQB_TRY(clip_pack(all[i]->w, all[i]->N, all[i]->K, all[i]->K, false, nullptr, Hh + all[i]->h_off, st));
        for (ClipLinear* L : all) RQB_TRY(make_streamed_weight(&L->sw, false, Hh + L->h_off, nullptr, L->N, L->K));
    }
    h->finalized = true;
    return 0;
}

static size_t clip_image_ws(const rqb200_clip* h, int B, int H, int W, int flags, rqb::ClipPrep* pp, void* base, rqb::ClipBufs* b) {
    using namespace rqb;
    const int R = h->cfg.vision_resolution, P = h->cfg.vision_patch, g = R / P;
    const bool prep = flags & RQB200_CLIP_PREPROCESS;
    ClipPrep local;
    if (!pp) pp = &local;
    int64_t tmp = 0;
    int tabs = 0;
    if (prep) {
        clip_prep(H, W, R, pp);
        tmp = (int64_t)B * 3 * H * R;
        tabs = pp->tab_ints();
    }
    return clip_layout(h, h->vis, B, B * g * g, h->Kp, tmp, tabs, base, b);
}

size_t rqb200_clip_workspace_bytes(rqb200_clip* h, int B, int H, int W, int flags) {
    if (!h || B <= 0 || H < 1 || W < 1) return 0;
    const int R = h->cfg.vision_resolution;
    if (!(flags & RQB200_CLIP_PREPROCESS) && (H != R || W != R)) return 0;
    return clip_image_ws(h, B, H, W, flags, nullptr, nullptr, nullptr);
}

size_t rqb200_clip_text_workspace_bytes(rqb200_clip* h, int N) {
    if (!h || N <= 0) return 0;
    return rqb::clip_layout(h, h->txt, N, 0, 0, 0, 0, nullptr, nullptr);
}

int rqb200_clip_encode_image(rqb200_clip* h, const float* x, int B, int H, int W, int flags, float* feat_out, void* ws, size_t ws_bytes,
                             void* stream) {
    using namespace rqb;
    if (!h || !x || !feat_out || !ws) return fail(RQB200_EINVAL, "clip_encode_image: null argument");
    if (!h->finalized) return fail(RQB200_ESTATE, "clip_encode_image: engine not finalised");
    const rqb200_clip_config& c = h->cfg;
    const int R = c.vision_resolution, P = c.vision_patch, E = c.vision_width, T = h->vis.T;
    if (B <= 0 || H < 1 || W < 1) return fail(RQB200_EINVAL, "clip_encode_image: B, H and W must be positive");
    const bool prep = flags & RQB200_CLIP_PREPROCESS;
    if (!prep && (H != R || W != R)) return fail(RQB200_EINVAL, "clip_encode_image: without RQB200_CLIP_PREPROCESS the input must be R x R");
    if ((int64_t)B * T > INT32_MAX / 4 || (int64_t)B * 3 * H * R > INT32_MAX) return fail(RQB200_EINVAL, "clip_encode_image: batch too large");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "clip_encode_image: no CUDA device");
    const cudaStream_t st = (cudaStream_t)stream;
    ClipPrep pp;
    ClipBufs b;
    if (clip_image_ws(h, B, H, W, flags, &pp, ws, &b) > ws_bytes)
        return fail(RQB200_EWORKSPACE, "clip_encode_image: workspace smaller than rqb200_clip_workspace_bytes");
    g_launches = 0;
    const int np = (R / P) * (R / P);
    if (h->fast) RQB_CUDA(cudaMemsetAsync(b.rows16, 0, (size_t)ceil_div((int64_t)B * np, 128) * 128 * h->Kp * 2, st));
    else if (h->Kp != 3 * P * P) RQB_CUDA(cudaMemsetAsync(b.rows32, 0, (size_t)B * np * h->Kp * 4, st));
    if (prep) RQB_TRY(clip_preprocess(pp, x, B, H, W, R, b.tmp, b.tabs, nullptr, nullptr, b.rows32, (__half*)b.rows16, P, h->Kp, st));
    else {
        clip_patch_rows_kernel<<<grid_1d((int64_t)B * 3 * R * R), 256, 0, st>>>(x, B, R, P, h->Kp, b.rows32, (__half*)b.rows16);
        RQB_TRY(check_launch("clip_patch_rows"));
    }
    // conv1 -> token rows 1.. (rows t * B + g), then class token + positional embedding, ln_pre (fp32, in place)
    RQB_TRY(clip_linear(h, h->conv1, (int64_t)B * np, b.rows32, b.rows16, b.X + (int64_t)B * E, nullptr, nullptr, 0, st));
    const float *cls = (const float*)h->t.find("visual.class_embedding")->ptr, *pos = (const float*)h->t.find("visual.positional_embedding")->ptr;
    clip_vis_embed_kernel<<<grid_1d((int64_t)B * T * E), 256, 0, st>>>(b.X, cls, pos, B, T, E);
    RQB_TRY(check_launch("clip_vis_embed"));
    RQB_TRY(launch_layernorm(b.X, E, (const float*)h->t.find("visual.ln_pre.weight")->ptr, (const float*)h->t.find("visual.ln_pre.bias")->ptr, b.X,
                             E, B * T, E, st));
    RQB_TRY(clip_blocks(h, h->vis, b, B, false, st));
    // token 0 of every image: rows 0 .. B - 1
    RQB_TRY(launch_layernorm(b.X, E, h->vis.lnf_w, h->vis.lnf_b, b.pool, E, B, E, st));
    RQB_TRY(launch_linear(b.pool, E, h->vis.projT, RQB200_F32, nullptr, nullptr, feat_out, c.embed_dim, B, c.embed_dim, E, 0, st));
    h->last_launches = g_launches;
    return 0;
}

int rqb200_clip_encode_text(rqb200_clip* h, const int64_t* tokens, int N, float* feat_out, void* ws, size_t ws_bytes, void* stream) {
    using namespace rqb;
    if (!h || !tokens || !feat_out || !ws) return fail(RQB200_EINVAL, "clip_encode_text: null argument");
    if (!h->finalized) return fail(RQB200_ESTATE, "clip_encode_text: engine not finalised");
    const rqb200_clip_config& c = h->cfg;
    const int E = c.text_width, T = c.context_length;
    if (N <= 0) return fail(RQB200_EINVAL, "clip_encode_text: N must be positive");
    if ((int64_t)N * T > INT32_MAX / 4) return fail(RQB200_EINVAL, "clip_encode_text: batch too large");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "clip_encode_text: no CUDA device");
    const cudaStream_t st = (cudaStream_t)stream;
    ClipBufs b;
    if (clip_layout(h, h->txt, N, 0, 0, 0, 0, ws, &b) > ws_bytes)
        return fail(RQB200_EWORKSPACE, "clip_encode_text: workspace smaller than rqb200_clip_text_workspace_bytes");
    g_launches = 0;
    clip_txt_embed_kernel<<<grid_1d((int64_t)N * T * E), 256, 0, st>>>(b.X, tokens, (const float*)h->t.find("token_embedding.weight")->ptr,
                                                                        (const float*)h->t.find("positional_embedding")->ptr, N, T, E, c.vocab_size);
    RQB_TRY(check_launch("clip_txt_embed"));
    RQB_TRY(clip_blocks(h, h->txt, b, N, true, st));
    float* gathered = h->fast ? (float*)b.XN : b.XN32;            // [N, E] fp32 scratch (XN holds at least 2 N T E bytes)
    clip_eot_gather_kernel<<<(unsigned)ceil_div(N, 4), 128, 0, st>>>(b.X, tokens, gathered, N, T, E);
    RQB_TRY(check_launch("clip_eot_gather"));
    RQB_TRY(launch_layernorm(gathered, E, h->txt.lnf_w, h->txt.lnf_b, b.pool, E, N, E, st));
    RQB_TRY(launch_linear(b.pool, E, h->txt.projT, RQB200_F32, nullptr, nullptr, feat_out, c.embed_dim, N, c.embed_dim, E, 0, st));
    h->last_launches = g_launches;
    return 0;
}

int rqb200_clip_cosine(const float* img_feat, const float* txt_feat, int n, int dim, float* out, void* stream) {
    using namespace rqb;
    if (!img_feat || !txt_feat || !out || n <= 0 || dim <= 0) return fail(RQB200_EINVAL, "clip_cosine: null argument or empty input");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "clip_cosine: no CUDA device");
    clip_cosine_kernel<<<(unsigned)ceil_div(n, 4), 128, 0, (cudaStream_t)stream>>>(img_feat, txt_feat, n, dim, out);
    return check_launch("clip_cosine");
}

int64_t rqb200_clip_last_launches(const rqb200_clip* h) { return h ? h->last_launches : 0; }

// ---- diagnostics
int rqb200_dbg_clip_preprocess(const float* x, int B, int H, int W, int R, uint8_t* u8_out, float* norm_out, void* stream) {
    using namespace rqb;
    if (!x || B <= 0 || H < 1 || W < 1 || R < 1) return fail(RQB200_EINVAL, "dbg_clip_preprocess: bad argument");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "dbg_clip_preprocess: no CUDA device");
    const cudaStream_t st = (cudaStream_t)stream;
    ClipPrep pp;
    clip_prep(H, W, R, &pp);
    uint8_t* tmp = nullptr;
    int* tabs = nullptr;
    RQB_CUDA(cudaMallocAsync((void**)&tmp, (size_t)B * 3 * H * R, st));
    RQB_CUDA(cudaMallocAsync((void**)&tabs, (size_t)std::max(pp.tab_ints(), 1) * sizeof(int), st));
    const int rc = clip_preprocess(pp, x, B, H, W, R, tmp, tabs, u8_out, norm_out, nullptr, nullptr, 1, 0, st);
    cudaFreeAsync(tmp, st);
    cudaFreeAsync(tabs, st);
    return rc;
}

// the host resize plan of an H x W input at resolution R: {Hr, Wr, top, left, horizontal taps per output (0: no pass), vertical taps}
int rqb200_clip_resize_plan(int H, int W, int R, int32_t* out6) {
    if (H < 1 || W < 1 || R < 1 || !out6) return rqb::fail(RQB200_EINVAL, "clip_resize_plan: bad argument");
    rqb::ClipPrep pp;
    rqb::clip_prep(H, W, R, &pp);
    const int v[6] = {pp.Hr, pp.Wr, pp.top, pp.left, pp.ksh, pp.ksv};
    memcpy(out6, v, sizeof(v));
    return 0;
}

int rqb200_dbg_clip_attn(const float* qkv, float* out, int G, int T, int E, int causal, void* stream) {
    if (!qkv || !out) return rqb::fail(RQB200_EINVAL, "dbg_clip_attn: null argument");
    return rqb::launch_clip_attn_f32(qkv, out, G, T, E, causal != 0, (cudaStream_t)stream);
}

int rqb200_dbg_clip_attn_flash(const void* qkv16, void* att16, int G, int T, int E, int causal, void* stream) {
    if (!qkv16 || !att16 || E % 64 != 0 || T < 1 || G < 1) return rqb::fail(RQB200_EINVAL, "dbg_clip_attn_flash: bad argument");
    return rqb::launch_attn_flash_f16((const rqb::h16*)qkv16, (rqb::h16*)att16, G, T, E, causal != 0, (cudaStream_t)stream);
}

}  // extern "C"
