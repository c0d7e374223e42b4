// LPIPS (rqvae/losses/vqgan/lpips.py: LPIPS over torchvision's VGG16 features[:30] and the five 1x1 `lin` heads) as a static layer
// plan.  Input and target run as ONE batch of 2n images (images [0, n) the inputs, [n, 2n) the targets), so the VGG runs once over
// 2n rows.  Two tiers: exact runs every conv on conv_igemm_kernel<float, true> (fp32 FFMA); fast runs every conv but conv1_1 (Cin = 3,
// fp32 FFMA on both tiers) on inc_conv_tc_kernel (split-fp16 operands, three products per k step).  Only the five tap convs
// (relu1_2 .. relu5_3) write fp32; on the fast tier every other conv writes the next conv's fp16 hi / lo operands only, and the pools
// read a tap's fp32 map and write those operands.  The head (normalize_tensor, squared difference, lin) runs in fp32 on both tiers; the
// spatial average is a fixed-order fp64 sum, so a pair's value does not depend on the batch around it.
#include <string>
#include <unordered_map>
#include <vector>

#include "kernels.h"

namespace rqb {

constexpr int LP_MIN_EXTENT = 16;                    // four 2x2 pools must leave relu5_3 at least 1 x 1
constexpr int LP_TAPS = 5;
constexpr int LP_CHNS[LP_TAPS] = {64, 128, 256, 512, 512};
constexpr size_t LP_CHUNK_BYTES = size_t(2) << 30;   // a call's workspace covers at most this many bytes of pairs; larger batches
                                                     // run in chunks of as many pairs as fit
constexpr float LP_EPS = 1e-10f;                     // normalize_tensor's eps

// ------------------------------------------------------------------------------------------------ kernels
// x0, x1 NCHW [n, 3, H, W] -> y NHWC [2n, H, W, 3]: images [0, n) from x0, [n, 2n) from x1, each (x - shift[c]) / scale[c] (ScalingLayer,
// a correctly rounded fp32 division as torch's)
__global__ void lpips_input_kernel(const float* __restrict__ x0, const float* __restrict__ x1, const float* __restrict__ shift,
                                   const float* __restrict__ scale, float* __restrict__ y, int n, int H, int W) {
    const int64_t hw = (int64_t)H * W, total = 2 * (int64_t)n * hw * 3;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % 3);
        const int64_t q = (i / 3) % hw, b = i / 3 / hw;
        const float v = b < n ? x0[(b * 3 + c) * hw + q] : x1[((b - n) * 3 + c) * hw + q];
        y[i] = __fdiv_rn(v - shift[c], scale[c]);
    }
}

// 2x2 stride-2 max pool (F.max_pool2d(2, 2): floor extents, an odd last row / column dropped) of X NHWC [N, H, W, C] (C % 4 == 0) into
// Y [N, H/2, W/2, C] fp32 and / or its fp16 hi / lo split (Yhi = fp16(v), Ylo = fp16(v - Yhi)), each nullable
__global__ void lpips_pool_kernel(const float* __restrict__ X, float* __restrict__ Y, __half* __restrict__ Yhi, __half* __restrict__ Ylo,
                                  int N, int H, int W, int C) {
    const int Ho = H / 2, Wo = W / 2, C4 = C / 4;
    const int64_t total = (int64_t)N * Ho * Wo * C4;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % C4) * 4;
        const int64_t m = i / C4;
        const int ox = (int)(m % Wo), oy = (int)((m / Wo) % Ho);
        const int64_t b = m / ((int64_t)Wo * Ho);
        const float* p = X + ((b * H + 2 * oy) * W + 2 * ox) * C + c;
        const int64_t row = (int64_t)W * C;
        const float4 a = *reinterpret_cast<const float4*>(p), bq = *reinterpret_cast<const float4*>(p + C);
        const float4 cq = *reinterpret_cast<const float4*>(p + row), d = *reinterpret_cast<const float4*>(p + row + C);
        const float v[4] = {fmaxf(fmaxf(a.x, bq.x), fmaxf(cq.x, d.x)), fmaxf(fmaxf(a.y, bq.y), fmaxf(cq.y, d.y)),
                            fmaxf(fmaxf(a.z, bq.z), fmaxf(cq.z, d.z)), fmaxf(fmaxf(a.w, bq.w), fmaxf(cq.w, d.w))};
        const int64_t o = m * C + c;
        if (Y) *reinterpret_cast<float4*>(Y + o) = make_float4(v[0], v[1], v[2], v[3]);
        if (Yhi) {
            const __half2 h0 = __floats2half2_rn(v[0], v[1]), h1 = __floats2half2_rn(v[2], v[3]);
            const float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
            const __half2 l0 = __floats2half2_rn(v[0] - f0.x, v[1] - f0.y), l1 = __floats2half2_rn(v[2] - f1.x, v[3] - f1.y);
            reinterpret_cast<__half2*>(Yhi + o)[0] = h0;
            reinterpret_cast<__half2*>(Yhi + o)[1] = h1;
            reinterpret_cast<__half2*>(Ylo + o)[0] = l0;
            reinterpret_cast<__half2*>(Ylo + o)[1] = l1;
        }
    }
}

// One warp per pixel q of pair b: F NHWC [2n, hw, C] holds image b (the input) and image b + n (the target).  d[b * hw + q] =
// sum_c w[c] (a_c / (|a| + eps) - t_c / (|t| + eps))^2: normalize_tensor, the squared difference and lin's 1x1 conv.  Two passes over
// the channels (the norms, then the weighted differences), never the expanded square, which cancels for a close pair.  An all-zero
// pixel normalises to 0.  Swapping a and t gives the same bits.
__global__ void lpips_head_kernel(const float* __restrict__ F, const float* __restrict__ w, float* __restrict__ d, int n, int hw, int C) {
    const int lane = threadIdx.x & 31;
    const int64_t npix = (int64_t)n * hw, other = npix * C;
    const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t p = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5); p < npix; p += nwarps) {
        const float* a = F + p * C;
        const float* t = a + other;
        float sa = 0.f, st = 0.f;
        for (int c = lane; c < C; c += 32) {
            const float va = a[c], vt = t[c];
            sa = fmaf(va, va, sa);
            st = fmaf(vt, vt, st);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            sa += __shfl_xor_sync(0xffffffffu, sa, o);
            st += __shfl_xor_sync(0xffffffffu, st, o);
        }
        const float na = sqrtf(sa) + LP_EPS, nt = sqrtf(st) + LP_EPS;
        float s = 0.f;
        for (int c = lane; c < C; c += 32) {
            const float df = __fdiv_rn(a[c], na) - __fdiv_rn(t[c], nt);
            s = fmaf(w[c], df * df, s);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) d[p] = s;
    }
}

// spatial_average of tap k, one CTA per pair b, in fp64 and a fixed order (no atomics): tapmean[b * 5 + k] = mean of d[b * hw ..
// b * hw + hw); layer_out[b * 5 + k] (nullable) its fp32 value; at k == 4, val[b] = the five taps' sum.  Taps 0..3 were written by
// earlier launches on the same stream.
constexpr int LP_MEAN_THREADS = 256;
__global__ void __launch_bounds__(LP_MEAN_THREADS) lpips_mean_kernel(const float* __restrict__ d, int hw, int k, double* __restrict__ tapmean,
                                                                     float* __restrict__ layer_out, float* __restrict__ val) {
    __shared__ double red[LP_MEAN_THREADS];
    const int b = blockIdx.x, t = threadIdx.x;
    const float* p = d + (int64_t)b * hw;
    double s = 0.0;
    for (int q = t; q < hw; q += LP_MEAN_THREADS) s += (double)p[q];
    red[t] = s;
    __syncthreads();
    for (int h = LP_MEAN_THREADS / 2; h > 0; h >>= 1) {
        if (t < h) red[t] += red[t + h];
        __syncthreads();
    }
    if (t == 0) {
        const double m = red[0] / (double)hw;
        tapmean[b * LP_TAPS + k] = m;
        if (layer_out) layer_out[(int64_t)b * LP_TAPS + k] = (float)m;
        if (k == LP_TAPS - 1) {
            double v = 0.0;
            for (int j = 0; j < LP_TAPS; j++) v += tapmean[b * LP_TAPS + j];
            val[b] = (float)v;
        }
    }
}

// finalize: a conv weight OIHW [Cout, Cin, 3, 3] -> OHWI fp32 (wo) and, on the fast tier, its split-fp16 halves
__global__ void lpips_pack_kernel(const float* __restrict__ w, float* __restrict__ wo, __half* __restrict__ whi, __half* __restrict__ wlo,
                                  int Cout, int Cin) {
    const int64_t total = (int64_t)Cout * 9 * Cin;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int ci = (int)(i % Cin), tap = (int)((i / Cin) % 9);
        const int64_t o = i / Cin / 9;
        const float f = w[(o * Cin + ci) * 9 + tap];
        wo[i] = f;
        if (whi) {
            const __half h = __float2half_rn(f);
            whi[i] = h;
            wlo[i] = __float2half_rn(f - __half2float(h));
        }
    }
}

static unsigned lp_grid(int64_t n) { return (unsigned)std::min<int64_t>(std::max<int64_t>(ceil_div(n, 256), 1), 8192); }

int launch_lpips_input(const float* x0, const float* x1, const float* shift, const float* scale, float* y, int n, int H, int W,
                       cudaStream_t st) {
    lpips_input_kernel<<<lp_grid(2 * (int64_t)n * H * W * 3), 256, 0, st>>>(x0, x1, shift, scale, y, n, H, W);
    return check_launch("lpips_input");
}
int launch_lpips_pool(const float* X, float* Y, __half* Yhi, __half* Ylo, int N, int H, int W, int C, cudaStream_t st) {
    lpips_pool_kernel<<<lp_grid((int64_t)N * (H / 2) * (W / 2) * (C / 4)), 256, 0, st>>>(X, Y, Yhi, Ylo, N, H, W, C);
    return check_launch("lpips_pool");
}
int launch_lpips_head(const float* F, const float* w, float* d, int n, int hw, int C, cudaStream_t st) {
    const int64_t blocks = std::min<int64_t>(ceil_div((int64_t)n * hw, 8), 16384);
    lpips_head_kernel<<<(unsigned)blocks, 256, 0, st>>>(F, w, d, n, hw, C);
    return check_launch("lpips_head");
}
int launch_lpips_mean(const float* d, int n, int hw, int k, double* tapmean, float* layer_out, float* val, cudaStream_t st) {
    lpips_mean_kernel<<<n, LP_MEAN_THREADS, 0, st>>>(d, hw, k, tapmean, layer_out, val);
    return check_launch("lpips_mean");
}

// ------------------------------------------------------------------------------------------------ layer plan
struct LpTensor {
    const void* ptr;
    int dtype;
    int64_t numel;
};
// one 3x3 pad-1 conv + bias + ReLU of vgg16.features: its OHWI weight and bias at w_off / b_off (floats) of the parameter buffer
struct LpConv {
    std::string name;           // "net.slice<s>.<index>"
    int cin, cout;
    bool tap;                   // relu1_2 .. relu5_3: writes the fp32 map the head and the next pool read
    int64_t w_off, b_off;
};

}  // namespace rqb

struct rqb200_lpips {
    rqb200_lpips_config cfg;
    std::unordered_map<std::string, rqb::LpTensor> t;
    std::vector<rqb::LpConv> convs;               // plan order
    int64_t lin_off[rqb::LP_TAPS];                // lin{k}'s weight [C_k]
    int64_t shift_off = 0, scale_off = 0;         // ScalingLayer's buffers [3]
    int64_t params_floats = 0;
    bool fast = false;                            // RQB200_MODE_FAST
    const float* params = nullptr;                // finalize: fp32, then (fast) the fp16 hi and lo copies at the same element offsets
    const __half* params_hi = nullptr;
    const __half* params_lo = nullptr;
    bool finalized = false;
    int64_t last_launches = 0;
};

namespace rqb {

static void lp_plan(rqb200_lpips* h) {
    // features index of each conv, by slice (the ReLUs and pools between them hold no parameters)
    static const int idx[13] = {0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28};
    static const int slice[13] = {1, 1, 2, 2, 3, 3, 3, 4, 4, 4, 5, 5, 5};
    static const int cout[13] = {64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512};
    auto take = [h](int64_t n) {
        const int64_t o = h->params_floats;
        h->params_floats = (int64_t)align_up((size_t)(o + n), 64);
        return o;
    };
    int cin = 3;
    for (int i = 0; i < 13; i++) {
        LpConv c{"net.slice" + std::to_string(slice[i]) + "." + std::to_string(idx[i]), cin, cout[i], i == 12 || slice[i] != slice[i + 1], 0, 0};
        c.w_off = take((int64_t)c.cout * 9 * c.cin);
        c.b_off = take(c.cout);
        h->convs.push_back(c);
        cin = cout[i];
    }
    for (int k = 0; k < LP_TAPS; k++) h->lin_off[k] = take(LP_CHNS[k]);
    h->shift_off = take(3);
    h->scale_off = take(3);
}

// per pair: two staged images; exact: two fp32 activation buffers per image, fast: one plus two fp16 hi / lo operand pairs; the head's
// per-pixel values of the largest tap; the five tap means
static int64_t lp_max_act(int H, int W) { return (int64_t)H * W * 64; }   // relu1_2 (every later map is smaller)
static size_t lp_pair_bytes(int H, int W, bool fast) {
    const size_t ma = (size_t)lp_max_act(H, W), hw = (size_t)H * W;
    return 2 * (hw * 3 + (fast ? 1 : 2) * ma) * sizeof(float) + (fast ? 2 * 4 * ma * sizeof(__half) : 0) + hw * sizeof(float) +
           LP_TAPS * sizeof(double);
}
static int lp_chunk(int B, int H, int W, bool fast) {
    const int64_t fit = std::max<int64_t>(1, (int64_t)(LP_CHUNK_BYTES / lp_pair_bytes(H, W, fast)));
    return (int)std::min<int64_t>(B, fit);
}
struct LpBufs {
    float* x0 = nullptr;          // staged input [2n, H, W, 3]
    float* f[2] = {nullptr, nullptr};
    __half* hi[2] = {nullptr, nullptr};
    __half* lo[2] = {nullptr, nullptr};
    float* d = nullptr;           // head values [n, hw]
    double* tapmean = nullptr;    // [n, 5]
};
static size_t lp_layout(int n, int H, int W, bool fast, void* base, size_t cap, LpBufs* o) {
    Arena ar(base, cap);
    const size_t ma = (size_t)lp_max_act(H, W), hw = (size_t)H * W;
    LpBufs b;
    b.x0 = ar.take<float>(2 * (size_t)n * hw * 3);
    for (int i = 0; i < (fast ? 1 : 2); i++) b.f[i] = ar.take<float>(2 * (size_t)n * ma);
    if (fast)
        for (int i = 0; i < 2; i++) {
            b.hi[i] = ar.take<__half>(2 * (size_t)n * ma);
            b.lo[i] = ar.take<__half>(2 * (size_t)n * ma);
        }
    b.d = ar.take<float>((size_t)n * hw);
    b.tapmean = ar.take<double>((size_t)n * LP_TAPS);
    if (o) *o = b;
    return ar.off + 256;
}

// one chunk of n pairs: x0 / x1 NCHW [n, 3, H, W] -> layer_out [n, 5] (nullable), val [n]
static int lp_run(rqb200_lpips* h, const LpBufs& bf, const float* x0, const float* x1, int n, int H, int W, float* layer_out, float* val,
                  cudaStream_t st) {
    const float* P = h->params;
    const int N = 2 * n;
    RQB_TRY(launch_lpips_input(x0, x1, P + h->shift_off, P + h->scale_off, bf.x0, n, H, W, st));
    const float* in = bf.x0;      // the current fp32 map (exact tier; the staged input and the taps on both tiers)
    int cs = 0;                   // fast tier: the slot holding the next conv's fp16 operands
    int tap = 0;
    for (size_t i = 0; i < h->convs.size(); i++) {
        const LpConv& c = h->convs[i];
        float* out = h->fast ? bf.f[0] : (in == bf.f[0] ? bf.f[1] : bf.f[0]);
        if (c.cin == 3 || !h->fast) {
            ConvGeom g{};
            g.B = N; g.Hi = H; g.Wi = W; g.Cin = c.cin; g.Ho = H; g.Wo = W; g.Cout = c.cout; g.KH = 3; g.KW = 3; g.stride = 1;
            g.pad = 1; g.pad_w = 1; g.ldy = c.cout; g.yoff = 0;
            RQB_TRY(launch_conv_relu(in, P + c.w_off, P + c.b_off, out, g, st));
            // fast tier: conv1_1's output becomes the next conv's operand
            if (h->fast) RQB_TRY(launch_cast_f16(out, bf.hi[0], bf.lo[0], N, H, W, c.cout, 0, st));
            cs = 0;
        } else {
            const int os = 1 - cs;
            RQB_TRY(launch_inc_conv_tc(bf.hi[cs], bf.lo[cs], h->params_hi + c.w_off, h->params_lo + c.w_off, P + c.b_off,
                                       c.tap ? out : nullptr, c.tap ? nullptr : bf.hi[os], c.tap ? nullptr : bf.lo[os], N, H, W, c.cin,
                                       c.cout, 3, 3, 1, 1, 1, c.cout, 0, st));
            cs = os;
        }
        in = out;
        if (!c.tap) continue;
        RQB_TRY(launch_lpips_head(in, P + h->lin_off[tap], bf.d, n, H * W, c.cout, st));
        RQB_TRY(launch_lpips_mean(bf.d, n, H * W, tap, bf.tapmean, layer_out, val, st));
        if (tap + 1 < LP_TAPS) {
            float* pout = h->fast ? nullptr : (in == bf.f[0] ? bf.f[1] : bf.f[0]);
            RQB_TRY(launch_lpips_pool(in, pout, h->fast ? bf.hi[0] : nullptr, h->fast ? bf.lo[0] : nullptr, N, H, W, c.cout, st));
            in = pout;
            cs = 0;
            H /= 2;
            W /= 2;
        }
        tap++;
    }
    return 0;
}

}  // namespace rqb

extern "C" {

rqb200_lpips* rqb200_lpips_create(const rqb200_lpips_config* cfg) {
    if (!cfg || (cfg->mode != RQB200_MODE_EXACT && cfg->mode != RQB200_MODE_FAST)) {
        rqb::set_error("lpips_create: mode must be RQB200_MODE_EXACT or RQB200_MODE_FAST");
        return nullptr;
    }
    rqb200_lpips* h = new rqb200_lpips();
    h->cfg = *cfg;
    h->fast = cfg->mode == RQB200_MODE_FAST;
    rqb::lp_plan(h);
    return h;
}
void rqb200_lpips_destroy(rqb200_lpips* h) { delete h; }

int rqb200_lpips_set_tensor(rqb200_lpips* h, const char* key, const void* ptr, int dtype, int64_t numel) {
    if (!h || !key || !ptr) return rqb::fail(RQB200_EINVAL, "lpips_set_tensor: null argument");
    h->t[key] = rqb::LpTensor{ptr, dtype, numel};
    h->finalized = false;
    return 0;
}

size_t rqb200_lpips_params_bytes(const rqb200_lpips* h) {
    return h ? (size_t)h->params_floats * (sizeof(float) + (h->fast ? 2 * sizeof(__half) : 0)) : 0;
}

int rqb200_lpips_finalize(rqb200_lpips* h, void* params, size_t params_bytes, void* stream) {
    using namespace rqb;
    if (!h) return fail(RQB200_EINVAL, "lpips_finalize: null handle");
    h->finalized = false;
    auto get = [&](const std::string& k, int64_t numel, const LpTensor** out) -> int {
        auto it = h->t.find(k);
        if (it == h->t.end()) return fail(RQB200_ESTATE, "lpips_finalize: tensor " + k + " (missing)");
        if (it->second.numel != numel) return fail(RQB200_ESTATE, "lpips_finalize: tensor " + k + " (wrong size)");
        if (it->second.dtype != RQB200_F32) return fail(RQB200_EINVAL, "lpips_finalize: tensor " + k + " must be fp32");
        *out = &it->second;
        return 0;
    };
    std::vector<const LpTensor*> ts(h->convs.size() * 2);
    for (size_t i = 0; i < h->convs.size(); i++) {
        const LpConv& c = h->convs[i];
        RQB_TRY(get(c.name + ".weight", (int64_t)c.cout * c.cin * 9, &ts[2 * i]));
        RQB_TRY(get(c.name + ".bias", c.cout, &ts[2 * i + 1]));
    }
    const LpTensor* lin[LP_TAPS];
    for (int k = 0; k < LP_TAPS; k++) {
        // lin<k>.model.1.weight with the Dropout in front (use_dropout=True), lin<k>.model.0.weight without
        const std::string p = "lin" + std::to_string(k) + ".model.";
        RQB_TRY(get(h->t.count(p + "1.weight") ? p + "1.weight" : p + "0.weight", LP_CHNS[k], &lin[k]));
    }
    const LpTensor *shift, *scale;
    RQB_TRY(get("scaling_layer.shift", 3, &shift));
    RQB_TRY(get("scaling_layer.scale", 3, &scale));
    if (!params) return fail(RQB200_EINVAL, "lpips_finalize: null parameter buffer");
    if (params_bytes < rqb200_lpips_params_bytes(h))
        return fail(RQB200_EWORKSPACE, "lpips_finalize: parameter buffer smaller than rqb200_lpips_params_bytes");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "lpips_finalize: no CUDA device");
    const cudaStream_t st = (cudaStream_t)stream;
    float* P = (float*)params;
    __half* Ph = h->fast ? (__half*)(P + h->params_floats) : nullptr;
    __half* Pl = h->fast ? Ph + h->params_floats : nullptr;
    auto copy = [&](float* dst, const LpTensor* s) -> int {
        RQB_CUDA(cudaMemcpyAsync(dst, s->ptr, (size_t)s->numel * sizeof(float), cudaMemcpyDeviceToDevice, st));
        return 0;
    };
    for (size_t i = 0; i < h->convs.size(); i++) {
        const LpConv& c = h->convs[i];
        lpips_pack_kernel<<<lp_grid((int64_t)c.cout * 9 * c.cin), 256, 0, st>>>((const float*)ts[2 * i]->ptr, P + c.w_off,
                                                                             Ph ? Ph + c.w_off : nullptr, Pl ? Pl + c.w_off : nullptr,
                                                                             c.cout, c.cin);
        RQB_TRY(check_launch("lpips_pack"));
        RQB_TRY(copy(P + c.b_off, ts[2 * i + 1]));
    }
    for (int k = 0; k < LP_TAPS; k++) RQB_TRY(copy(P + h->lin_off[k], lin[k]));
    RQB_TRY(copy(P + h->shift_off, shift));
    RQB_TRY(copy(P + h->scale_off, scale));
    h->params = P;
    h->params_hi = Ph;
    h->params_lo = Pl;
    h->finalized = true;
    return 0;
}

size_t rqb200_lpips_workspace_bytes(rqb200_lpips* h, int B, int H, int W) {
    using namespace rqb;
    if (!h || B <= 0 || H < LP_MIN_EXTENT || W < LP_MIN_EXTENT) return 0;
    return lp_layout(lp_chunk(B, H, W, h->fast), H, W, h->fast, nullptr, 0, nullptr);
}

int rqb200_lpips_forward(rqb200_lpips* h, const float* x0, const float* x1, int B, int H, int W, float* layer_out, float* val_out,
                         void* workspace, size_t workspace_bytes, void* stream) {
    using namespace rqb;
    if (!h || !x0 || !x1 || !val_out || !workspace) return fail(RQB200_EINVAL, "lpips_forward: null argument");
    if (!h->finalized) return fail(RQB200_ESTATE, "lpips_forward: engine not finalised");
    if (B <= 0 || H < LP_MIN_EXTENT || W < LP_MIN_EXTENT)
        return fail(RQB200_EINVAL, "lpips_forward: need B >= 1 and H, W >= 16");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "lpips_forward: no CUDA device");
    const cudaStream_t st = (cudaStream_t)stream;
    const int chunk = lp_chunk(B, H, W, h->fast);
    LpBufs bf;
    if (lp_layout(chunk, H, W, h->fast, workspace, workspace_bytes, &bf) > workspace_bytes)
        return fail(RQB200_EWORKSPACE, "lpips_forward: workspace smaller than rqb200_lpips_workspace_bytes");
    g_launches = 0;
    const int64_t img = (int64_t)3 * H * W;
    int rc = 0;
    for (int b0 = 0; b0 < B && rc == 0; b0 += chunk) {
        const int n = std::min(chunk, B - b0);
        rc = lp_run(h, bf, x0 + b0 * img, x1 + b0 * img, n, H, W, layer_out ? layer_out + (int64_t)b0 * LP_TAPS : nullptr, val_out + b0, st);
    }
    h->last_launches = g_launches;
    return rc;
}

int64_t rqb200_lpips_last_launches(const rqb200_lpips* h) { return h ? h->last_launches : 0; }

// ---- diagnostic entry points (tests/test_gpu_lpips.py): one launch of each LPIPS kernel through its launcher

int rqb200_dbg_lpips_input(const float* x0, const float* x1, const float* shift, const float* scale, float* y, int n, int H, int W,
                           void* stream) {
    using namespace rqb;
    if (n < 1 || H < 1 || W < 1 || !x0 || !x1 || !shift || !scale || !y)
        return fail(RQB200_EINVAL, "dbg_lpips_input: need n, H, W >= 1 and every pointer");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "dbg_lpips_input: no CUDA device");
    return launch_lpips_input(x0, x1, shift, scale, y, n, H, W, (cudaStream_t)stream);
}

int rqb200_dbg_lpips_pool(const float* X, float* Y, void* Yhi, void* Ylo, int N, int H, int W, int C, void* stream) {
    using namespace rqb;
    if (N < 1 || H < 2 || W < 2 || C < 4 || C % 4 || !X || (!Y && !Yhi) || (!Yhi) != (!Ylo))
        return fail(RQB200_EINVAL, "dbg_lpips_pool: need N >= 1, H, W >= 2, C % 4 == 0, an output and hi / lo both or neither");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "dbg_lpips_pool: no CUDA device");
    return launch_lpips_pool(X, Y, (__half*)Yhi, (__half*)Ylo, N, H, W, C, (cudaStream_t)stream);
}

int rqb200_dbg_lpips_head(const float* F, const float* w, float* d, int n, int hw, int C, void* stream) {
    using namespace rqb;
    if (n < 1 || hw < 1 || C < 1 || !F || !w || !d) return fail(RQB200_EINVAL, "dbg_lpips_head: need n, hw, C >= 1 and every pointer");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "dbg_lpips_head: no CUDA device");
    return launch_lpips_head(F, w, d, n, hw, C, (cudaStream_t)stream);
}

int rqb200_dbg_lpips_mean(const float* d, int n, int hw, int k, double* tapmean, float* layer_out, float* val, void* stream) {
    using namespace rqb;
    if (n < 1 || hw < 1 || k < 0 || k >= LP_TAPS || !d || !tapmean || (k == LP_TAPS - 1 && !val))
        return fail(RQB200_EINVAL, "dbg_lpips_mean: need n, hw >= 1, 0 <= k < 5, d, tapmean and (k == 4) val");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "dbg_lpips_mean: no CUDA device");
    return launch_lpips_mean(d, n, hw, k, tapmean, layer_out, val, (cudaStream_t)stream);
}
}
