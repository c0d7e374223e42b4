// The FID Inception-v3 (rqvae/metrics/inception.py: InceptionV3 over fid_inception_v3, the pytorch-fid port of TensorFlow's
// 2015-12-05 graph) as a static layer plan with each BatchNorm folded into its conv, so each BasicConv2d is one conv + bias + ReLU
// launch.  Two tiers: exact runs every conv on conv_igemm_kernel<float, true> (fp32 FFMA); fast runs every conv but Conv2d_1a_3x3
// (Cin = 3, as the VAE's conv_in) on inc_conv_tc_kernel (conv_tc.cu: wgmma, split-fp16 operands, three products per k step), whose
// epilogue writes the next conv's fp16 hi / lo operands beside the fp32 map.
//
// Layer names are the reference's InceptionV3 state_dict keys: blocks.0.{0,1,2} = Conv2d_1a_3x3 / 2a / 2b, blocks.1.{0,1} =
// Conv2d_3b_1x1 / 4a, blocks.2.{0..7} = Mixed_5b..5d (FIDInceptionA), Mixed_6a (torchvision's InceptionB), Mixed_6b..6e
// (FIDInceptionC), blocks.3.{0,1,2} = Mixed_7a (InceptionD), Mixed_7b (FIDInceptionE_1), Mixed_7c (FIDInceptionE_2), and fc.
// Differences in execution, not arithmetic: activations are NHWC fp32; every branch writes straight into its channel slice of
// the block's output (torch.cat is never a copy); the bilinear resize, 2x - 1 and NCHW -> NHWC are one pass.
#include <vector>

#include "kernels.h"

namespace rqb {

constexpr int INC_RES = 299;                       // F.interpolate(size=(299, 299)) of resize_input
constexpr int INC_MIN_EXTENT = 75;                 // smallest H, W every layer accepts (Mixed_7a's stride-2 3x3 needs 3 pixels)
constexpr double INC_BN_EPS = 1e-3;                // BasicConv2d's BatchNorm2d(eps=0.001)
constexpr int INC_FEAT = 2048, INC_CLASSES = 1008;

// ------------------------------------------------------------------------------------------------ kernels
// x NCHW [B, 3, H, W] -> y NHWC [B, Ho, Wo, 3]: F.interpolate(mode='bilinear', align_corners=False) to Ho x Wo when resize (ATen's
// upsample_bilinear2d: src = scale (dst + 0.5) - 0.5 clamped at 0, scale = in / out, evaluated here in fp64), then 2 v - 1 when
// normalize
__global__ void inc_input_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int H, int W, int Ho, int Wo, int resize,
                                 int normalize) {
    const int64_t n = (int64_t)B * Ho * Wo * 3;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % 3);
        const int ox = (int)((i / 3) % Wo), oy = (int)((i / 3 / Wo) % Ho), b = (int)(i / 3 / Wo / Ho);
        const float* p = x + ((int64_t)b * 3 + c) * H * W;
        float v;
        if (resize) {
            // coordinates and weights in fp64: in fp32 a source coordinate near 512 is off by up to 3e-5 of a pixel, which moves a
            // noisy image's resized values by as much
            const double sh = (double)H / Ho, sw = (double)W / Wo;
            const double fy = fmax(sh * (oy + 0.5) - 0.5, 0.0), fx = fmax(sw * (ox + 0.5) - 0.5, 0.0);
            const int y0 = (int)fy, x0 = (int)fx;
            const int dy = y0 < H - 1 ? 1 : 0, dx = x0 < W - 1 ? 1 : 0;
            const double ly1 = fy - y0, lx1 = fx - x0, ly0 = 1.0 - ly1, lx0 = 1.0 - lx1;
            const float* r0 = p + (int64_t)y0 * W + x0;
            const float* r1 = r0 + (int64_t)dy * W;
            v = (float)(ly0 * (lx0 * r0[0] + lx1 * r0[dx]) + ly1 * (lx0 * r1[0] + lx1 * r1[dx]));
        } else {
            v = p[(int64_t)oy * W + ox];
        }
        if (normalize) v = 2.f * v - 1.f;
        y[i] = v;
    }
}

// 3x3 pooling of X NHWC [B, H, W, C] into channels [yoff, yoff + C) of rows of ldy floats.  mode 0: max (padding acts as -inf,
// F.max_pool2d); mode 1: average over the window's pixels inside the map (F.avg_pool2d(count_include_pad=False))
__global__ void inc_pool_kernel(const float* __restrict__ X, float* __restrict__ Y, int B, int H, int W, int C, int Ho, int Wo,
                                int stride, int pad, int mode, int ldy, int yoff, __half* __restrict__ Yhi, __half* __restrict__ Ylo) {
    const int64_t n = (int64_t)B * Ho * Wo * C;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const int64_t m = i / C;
        const int ox = (int)(m % Wo), oy = (int)((m / Wo) % Ho), b = (int)(m / Wo / Ho);
        float acc = mode == 0 ? -INFINITY : 0.f;
        int cnt = 0;
        for (int ky = 0; ky < 3; ky++) {
            const int iy = oy * stride - pad + ky;
            if (iy < 0 || iy >= H) continue;
            for (int kx = 0; kx < 3; kx++) {
                const int ix = ox * stride - pad + kx;
                if (ix < 0 || ix >= W) continue;
                const float v = X[(((int64_t)b * H + iy) * W + ix) * C + c];
                acc = mode == 0 ? fmaxf(acc, v) : acc + v;
                cnt++;
            }
        }
        const float v = mode == 0 ? acc : acc / (float)cnt;
        Y[m * ldy + yoff + c] = v;
        if (Yhi) split_f16(v, Yhi[m * ldy + yoff + c], Ylo[m * ldy + yoff + c]);   // fast tier: the next conv's operand halves too
    }
}

// global average pool: X NHWC [B, HW, C] -> Y [B, C]
__global__ void inc_gap_kernel(const float* __restrict__ X, float* __restrict__ Y, int HW, int C) {
    const int b = blockIdx.y, c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    const float* p = X + (int64_t)b * HW * C + c;
    float s = 0.f;
    for (int q = 0; q < HW; q++) s += p[(int64_t)q * C];
    Y[(int64_t)b * C + c] = s / (float)HW;
}

// NHWC [B, HW, C] -> NCHW [B, C, HW] (the reference's block outputs)
__global__ void inc_to_nchw_kernel(const float* __restrict__ X, float* __restrict__ Y, int B, int HW, int C) {
    const int64_t n = (int64_t)B * HW * C;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int q = (int)(i % HW);
        const int64_t bc = i / HW;
        const int c = (int)(bc % C), b = (int)(bc / C);
        Y[i] = X[((int64_t)b * HW + q) * C + c];
    }
}

int launch_inc_input(const float* x, float* y, int B, int H, int W, int resize, int normalize, cudaStream_t st) {
    const int Ho = resize ? INC_RES : H, Wo = resize ? INC_RES : W;
    inc_input_kernel<<<grid_1d((int64_t)B * Ho * Wo * 3), 256, 0, st>>>(x, y, B, H, W, Ho, Wo, resize, normalize);
    return check_launch("inc_input");
}
int launch_inc_pool(const float* X, float* Y, int B, int H, int W, int C, int stride, int pad, int mode, int ldy, int yoff,
                    cudaStream_t st, __half* Yhi = nullptr, __half* Ylo = nullptr) {
    const int Ho = (H + 2 * pad - 3) / stride + 1, Wo = (W + 2 * pad - 3) / stride + 1;
    inc_pool_kernel<<<grid_1d((int64_t)B * Ho * Wo * C), 256, 0, st>>>(X, Y, B, H, W, C, Ho, Wo, stride, pad, mode, ldy, yoff, Yhi, Ylo);
    return check_launch(mode == 0 ? "inc_maxpool" : "inc_avgpool");
}
int launch_inc_gap(const float* X, float* Y, int B, int HW, int C, cudaStream_t st) {
    inc_gap_kernel<<<dim3((unsigned)ceil_div(C, 256), B), 256, 0, st>>>(X, Y, HW, C);
    return check_launch("inc_gap");
}

// ------------------------------------------------------------------------------------------------ layer plan
// one BasicConv2d: its folded OHWI weight and bias live at w_off / b_off (floats) of the folded-parameter buffer
struct IncConv {
    std::string name;
    int cin, cout, kh, kw;
    int64_t w_off, b_off;
};

}  // namespace rqb

struct rqb200_inception {
    rqb200_inception_config cfg;
    rqb::TensorTable t;
    std::vector<rqb::IncConv> convs;              // plan order
    std::unordered_map<std::string, int> conv_at;
    rqb::SplitParams par;                         // the folded weights and biases (bound at finalize)
    bool fast = false;                            // RQB200_MODE_FAST
    bool finalized = false;
    int64_t last_launches = 0;
};

namespace rqb {

// One walk of the plan serves three purposes: collecting the convs (create), measuring the largest activation of an extent (dry),
// and launching.  Buffers: x0 the staged input, a / b the block inputs and outputs (ping-pong), t1 / t2 the branches' temporaries.
struct IncRun {
    rqb200_inception* h;
    cudaStream_t st;
    int B;
    int mode;                         // 0 collect, 1 dry, 2 launch
    float *a = nullptr, *b = nullptr, *t1 = nullptr, *t2 = nullptr, *feat = nullptr;
    __half* hi[4] = {nullptr, nullptr, nullptr, nullptr};   // fast tier: the fp16 hi / lo operands of a, b, t1, t2
    __half* lo[4] = {nullptr, nullptr, nullptr, nullptr};
    int64_t max_act = 0;              // floats per image
    // the caller's NCHW buffers for blocks 0-2 (null: not wanted), written from image out_b0 on
    float* out_nchw[3] = {nullptr, nullptr, nullptr};
    int64_t out_b0 = 0;

    void note(int64_t hw, int64_t c) { if (hw * c > max_act) max_act = hw * c; }
    // the fp16 operand buffers of one of a, b, t1, t2 (fast tier), else -1
    int slot(const float* p) const {
        const float* bufs[4] = {a, b, t1, t2};
        for (int i = 0; i < 4; i++) if (p == bufs[i]) return i;
        return -1;
    }

    // BasicConv2d name: x NHWC [B, H, W, Cin] -> y rows of ldy floats from channel yoff; (H, W) becomes the output extent
    int conv(const std::string& name, const float* x, int& H, int& W, int Cin, float* y, int ldy, int yoff, int Cout, int kh, int kw,
             int ph, int pw, int stride) {
        const ConvGeom g = conv_geom(B, H, W, Cin, Cout, kh, kw, ph, pw, stride, ldy, yoff);
        note((int64_t)g.Ho * g.Wo, ldy);
        if (mode == 0) {
            const int64_t w_off = h->par.take((int64_t)Cout * kh * kw * Cin);
            h->conv_at[name] = (int)h->convs.size();
            h->convs.push_back(IncConv{name, Cin, Cout, kh, kw, w_off, h->par.take(Cout)});
        }
        if (mode == 2) {
            // Conv2d_1a_3x3 reads the staged fp32 input (no fp16 operand): fp32 FFMA on both tiers
            const IncConv& c = h->convs[h->conv_at.at(name)];
            const int sx = slot(x), sy = slot(y);
            RQB_TRY(launch_plan_conv(h->fast, h->par, c.w_off, c.b_off, x, sx >= 0 ? hi[sx] : nullptr, sx >= 0 ? lo[sx] : nullptr, y, hi[sy],
                                     lo[sy], g, st));
        }
        H = g.Ho;
        W = g.Wo;
        return 0;
    }
    int conv1(const std::string& name, const float* x, int H, int W, int Cin, float* y, int ldy, int yoff, int Cout) {
        return conv(name, x, H, W, Cin, y, ldy, yoff, Cout, 1, 1, 0, 0, 1);
    }
    // same-size conv (stride 1, "same" padding) of a kh x kw kernel
    int convs(const std::string& name, const float* x, int H, int W, int Cin, float* y, int ldy, int yoff, int Cout, int kh, int kw) {
        return conv(name, x, H, W, Cin, y, ldy, yoff, Cout, kh, kw, kh / 2, kw / 2, 1);
    }
    int pool(const float* x, int& H, int& W, int C, float* y, int ldy, int yoff, int stride, int pad, int max) {
        const int Ho = (H + 2 * pad - 3) / stride + 1, Wo = (W + 2 * pad - 3) / stride + 1;
        note((int64_t)Ho * Wo, ldy);
        if (mode == 2) {
            const int sy = slot(y);
            RQB_TRY(launch_inc_pool(x, y, B, H, W, C, stride, pad, max ? 0 : 1, ldy, yoff, st, h->fast ? hi[sy] : nullptr,
                                    h->fast ? lo[sy] : nullptr));
        }
        H = Ho;
        W = Wo;
        return 0;
    }

    // block k's output y NHWC [B, H, W, C] into the caller's NCHW buffer, if wanted
    int emit(int k, const float* y, int H, int W, int C) {
        if (mode != 2 || !out_nchw[k]) return 0;
        const int64_t hw = (int64_t)H * W;
        inc_to_nchw_kernel<<<grid_1d(B * hw * C), 256, 0, st>>>(y, out_nchw[k] + out_b0 * hw * C, B, (int)hw, C);
        return check_launch("inc_to_nchw");
    }

    // FIDInceptionA: [branch1x1 64 | branch5x5 64 | branch3x3dbl 96 | branch_pool pf]
    int block_a(const std::string& p, const float* x, int H, int W, int Cin, int pf, float* y) {
        const int ld = 224 + pf;
        RQB_TRY(conv1(p + ".branch1x1", x, H, W, Cin, y, ld, 0, 64));
        RQB_TRY(conv1(p + ".branch5x5_1", x, H, W, Cin, t1, 48, 0, 48));
        RQB_TRY(convs(p + ".branch5x5_2", t1, H, W, 48, y, ld, 64, 64, 5, 5));
        RQB_TRY(conv1(p + ".branch3x3dbl_1", x, H, W, Cin, t1, 64, 0, 64));
        RQB_TRY(convs(p + ".branch3x3dbl_2", t1, H, W, 64, t2, 96, 0, 96, 3, 3));
        RQB_TRY(convs(p + ".branch3x3dbl_3", t2, H, W, 96, y, ld, 128, 96, 3, 3));
        int h2 = H, w2 = W;
        RQB_TRY(pool(x, h2, w2, Cin, t1, Cin, 0, 1, 1, 0));
        return conv1(p + ".branch_pool", t1, H, W, Cin, y, ld, 224, pf);
    }
    // torchvision InceptionB (Mixed_6a): [branch3x3 384 | branch3x3dbl 96 | max pool Cin], all stride 2
    int block_b(const std::string& p, const float* x, int& H, int& W, int Cin, float* y) {
        const int ld = 480 + Cin;
        int ho = H, wo = W, h1 = H, w1 = W;
        RQB_TRY(conv(p + ".branch3x3", x, ho, wo, Cin, y, ld, 0, 384, 3, 3, 0, 0, 2));
        RQB_TRY(conv1(p + ".branch3x3dbl_1", x, H, W, Cin, t1, 64, 0, 64));
        RQB_TRY(convs(p + ".branch3x3dbl_2", t1, H, W, 64, t2, 96, 0, 96, 3, 3));
        RQB_TRY(conv(p + ".branch3x3dbl_3", t2, h1, w1, 96, y, ld, 384, 96, 3, 3, 0, 0, 2));
        RQB_TRY(pool(x, H, W, Cin, y, ld, 480, 2, 0, 1));
        return 0;
    }
    // FIDInceptionC: [branch1x1 192 | branch7x7 192 | branch7x7dbl 192 | branch_pool 192]
    int block_c(const std::string& p, const float* x, int H, int W, int c7, float* y) {
        const int C = 768;
        RQB_TRY(conv1(p + ".branch1x1", x, H, W, C, y, C, 0, 192));
        RQB_TRY(conv1(p + ".branch7x7_1", x, H, W, C, t1, c7, 0, c7));
        RQB_TRY(convs(p + ".branch7x7_2", t1, H, W, c7, t2, c7, 0, c7, 1, 7));
        RQB_TRY(convs(p + ".branch7x7_3", t2, H, W, c7, y, C, 192, 192, 7, 1));
        RQB_TRY(conv1(p + ".branch7x7dbl_1", x, H, W, C, t1, c7, 0, c7));
        RQB_TRY(convs(p + ".branch7x7dbl_2", t1, H, W, c7, t2, c7, 0, c7, 7, 1));
        RQB_TRY(convs(p + ".branch7x7dbl_3", t2, H, W, c7, t1, c7, 0, c7, 1, 7));
        RQB_TRY(convs(p + ".branch7x7dbl_4", t1, H, W, c7, t2, c7, 0, c7, 7, 1));
        RQB_TRY(convs(p + ".branch7x7dbl_5", t2, H, W, c7, y, C, 384, 192, 1, 7));
        int h2 = H, w2 = W;
        RQB_TRY(pool(x, h2, w2, C, t1, C, 0, 1, 1, 0));
        return conv1(p + ".branch_pool", t1, H, W, C, y, C, 576, 192);
    }
    // torchvision InceptionD (Mixed_7a): [branch3x3 320 | branch7x7x3 192 | max pool 768], all stride 2
    int block_d(const std::string& p, const float* x, int& H, int& W, float* y) {
        const int C = 768, ld = 1280;
        int h1 = H, w1 = W, h2 = H, w2 = W;
        RQB_TRY(conv1(p + ".branch3x3_1", x, H, W, C, t1, 192, 0, 192));
        RQB_TRY(conv(p + ".branch3x3_2", t1, h1, w1, 192, y, ld, 0, 320, 3, 3, 0, 0, 2));
        RQB_TRY(conv1(p + ".branch7x7x3_1", x, H, W, C, t1, 192, 0, 192));
        RQB_TRY(convs(p + ".branch7x7x3_2", t1, H, W, 192, t2, 192, 0, 192, 1, 7));
        RQB_TRY(convs(p + ".branch7x7x3_3", t2, H, W, 192, t1, 192, 0, 192, 7, 1));
        RQB_TRY(conv(p + ".branch7x7x3_4", t1, h2, w2, 192, y, ld, 320, 192, 3, 3, 0, 0, 2));
        RQB_TRY(pool(x, H, W, C, y, ld, 512, 2, 0, 1));
        return 0;
    }
    // FIDInceptionE_1 (avg pool) / E_2 (max pool): [branch1x1 320 | branch3x3 2 x 384 | branch3x3dbl 2 x 384 | branch_pool 192]
    int block_e(const std::string& p, const float* x, int H, int W, int Cin, int max_pool, float* y) {
        const int ld = 2048;
        RQB_TRY(conv1(p + ".branch1x1", x, H, W, Cin, y, ld, 0, 320));
        RQB_TRY(conv1(p + ".branch3x3_1", x, H, W, Cin, t1, 384, 0, 384));
        RQB_TRY(convs(p + ".branch3x3_2a", t1, H, W, 384, y, ld, 320, 384, 1, 3));
        RQB_TRY(convs(p + ".branch3x3_2b", t1, H, W, 384, y, ld, 704, 384, 3, 1));
        RQB_TRY(conv1(p + ".branch3x3dbl_1", x, H, W, Cin, t1, 448, 0, 448));
        RQB_TRY(convs(p + ".branch3x3dbl_2", t1, H, W, 448, t2, 384, 0, 384, 3, 3));
        RQB_TRY(convs(p + ".branch3x3dbl_3a", t2, H, W, 384, y, ld, 1088, 384, 1, 3));
        RQB_TRY(convs(p + ".branch3x3dbl_3b", t2, H, W, 384, y, ld, 1472, 384, 3, 1));
        int h2 = H, w2 = W;
        RQB_TRY(pool(x, h2, w2, Cin, t1, Cin, 0, 1, 1, max_pool));
        return conv1(p + ".branch_pool", t1, H, W, Cin, y, ld, 1856, 192);
    }

    // the network from the staged NHWC input x0 [B, H, W, 3] through block h->cfg.last_block; block 3 ends in feat [B, 2048]
    int walk(const float* x0, int H, int W) {
        const int last = h->cfg.last_block;
        float* A = a;
        float* Bf = b;
        note((int64_t)H * W, 3);
        RQB_TRY(conv("blocks.0.0", x0, H, W, 3, t1, 32, 0, 32, 3, 3, 0, 0, 2));
        RQB_TRY(conv("blocks.0.1", t1, H, W, 32, t2, 32, 0, 32, 3, 3, 0, 0, 1));
        RQB_TRY(conv("blocks.0.2", t2, H, W, 32, t1, 64, 0, 64, 3, 3, 1, 1, 1));
        RQB_TRY(pool(t1, H, W, 64, A, 64, 0, 2, 0, 1));
        RQB_TRY(emit(0, A, H, W, 64));
        if (last < 1) return 0;
        RQB_TRY(conv1("blocks.1.0", A, H, W, 64, t1, 80, 0, 80));
        RQB_TRY(conv("blocks.1.1", t1, H, W, 80, t2, 192, 0, 192, 3, 3, 0, 0, 1));
        RQB_TRY(pool(t2, H, W, 192, Bf, 192, 0, 2, 0, 1));
        RQB_TRY(emit(1, Bf, H, W, 192));
        if (last < 2) return 0;
        RQB_TRY(block_a("blocks.2.0", Bf, H, W, 192, 32, A));
        RQB_TRY(block_a("blocks.2.1", A, H, W, 256, 64, Bf));
        RQB_TRY(block_a("blocks.2.2", Bf, H, W, 288, 64, A));
        RQB_TRY(block_b("blocks.2.3", A, H, W, 288, Bf));
        RQB_TRY(block_c("blocks.2.4", Bf, H, W, 128, A));
        RQB_TRY(block_c("blocks.2.5", A, H, W, 160, Bf));
        RQB_TRY(block_c("blocks.2.6", Bf, H, W, 160, A));
        RQB_TRY(block_c("blocks.2.7", A, H, W, 192, Bf));
        RQB_TRY(emit(2, Bf, H, W, 768));
        if (last < 3) return 0;
        RQB_TRY(block_d("blocks.3.0", Bf, H, W, A));
        RQB_TRY(block_e("blocks.3.1", A, H, W, 1280, 0, Bf));
        RQB_TRY(block_e("blocks.3.2", Bf, H, W, 2048, 1, A));
        if (mode == 2) RQB_TRY(launch_inc_gap(A, feat, B, H * W, INC_FEAT, st));
        return 0;
    }
};

// the extent the network sees: 299 x 299 when resizing, else the input's own
static void staged_extent(int H, int W, int flags, int* Hs, int* Ws) {
    *Hs = (flags & RQB200_INC_RESIZE) ? INC_RES : H;
    *Ws = (flags & RQB200_INC_RESIZE) ? INC_RES : W;
}
static int64_t inc_max_act(rqb200_inception* h, int Hs, int Ws) {
    IncRun d{h, nullptr, 1, 1};
    d.walk(nullptr, Hs, Ws);
    return d.max_act;
}
// per image: the staged input, four fp32 activation buffers and the pooled features; the fast tier's eight fp16 operand buffers
static size_t inc_image_bytes(int Hs, int Ws, int64_t max_act, bool fast) {
    return ((size_t)Hs * Ws * 3 + 4 * (size_t)max_act + INC_FEAT) * sizeof(float) + (fast ? 8 * (size_t)max_act * sizeof(__half) : 0);
}
static size_t inc_layout(int n, int Hs, int Ws, int64_t max_act, bool fast, void* base, size_t cap, float** x0, IncRun* run) {
    Arena ar(base, cap);
    float* p = ar.take<float>((size_t)n * Hs * Ws * 3);
    if (x0) *x0 = p;
    float* bufs[4];
    for (int i = 0; i < 4; i++) bufs[i] = ar.take<float>((size_t)n * max_act);
    float* feat = ar.take<float>((size_t)n * INC_FEAT);
    if (run) {
        run->a = bufs[0]; run->b = bufs[1]; run->t1 = bufs[2]; run->t2 = bufs[3]; run->feat = feat;
    }
    if (fast)
        for (int i = 0; i < 4; i++) {
            __half* ph = ar.take<__half>((size_t)n * max_act);
            __half* pl = ar.take<__half>((size_t)n * max_act);
            if (run) { run->hi[i] = ph; run->lo[i] = pl; }
        }
    return ar.off + 256;
}

}  // namespace rqb

extern "C" {

rqb200_inception* rqb200_inception_create(const rqb200_inception_config* cfg) {
    if (!cfg || cfg->last_block < 0 || cfg->last_block > 3) { rqb::set_error("inception_create: last_block must be 0..3"); return nullptr; }
    if (cfg->mode != RQB200_MODE_EXACT && cfg->mode != RQB200_MODE_FAST) {
        rqb::set_error("inception_create: mode must be RQB200_MODE_EXACT or RQB200_MODE_FAST");
        return nullptr;
    }
    rqb200_inception* h = new rqb200_inception();
    h->cfg = *cfg;
    h->fast = cfg->mode == RQB200_MODE_FAST;
    rqb::IncRun c{h, nullptr, 1, 0};
    c.walk(nullptr, rqb::INC_RES, rqb::INC_RES);
    return h;
}
void rqb200_inception_destroy(rqb200_inception* h) { delete h; }

int rqb200_inception_set_tensor(rqb200_inception* h, const char* key, const void* ptr, int dtype, int64_t numel) {
    if (!h || !key || !ptr) return rqb::fail(RQB200_EINVAL, "inception_set_tensor: null argument");
    h->t.set(key, ptr, dtype, numel);
    h->finalized = false;
    return 0;
}

size_t rqb200_inception_params_bytes(const rqb200_inception* h) {
    return h ? h->par.bytes(h->fast) : 0;
}

int rqb200_inception_finalize(rqb200_inception* h, void* params, size_t params_bytes, void* stream) {
    using namespace rqb;
    if (!h) return fail(RQB200_EINVAL, "inception_finalize: null handle");
    h->finalized = false;
    const char* who = "inception_finalize";
    std::vector<const float*> ts(h->convs.size() * 5);
    for (size_t i = 0; i < h->convs.size(); i++) {
        const IncConv& c = h->convs[i];
        RQB_TRY(h->t.get_f32(who, c.name + ".conv.weight", (int64_t)c.cout * c.cin * c.kh * c.kw, &ts[i * 5]));
        static const char* bn[4] = {".bn.weight", ".bn.bias", ".bn.running_mean", ".bn.running_var"};
        for (int j = 0; j < 4; j++) RQB_TRY(h->t.get_f32(who, c.name + bn[j], c.cout, &ts[i * 5 + 1 + j]));
    }
    if (h->cfg.last_block == 3) {
        const float* d;
        RQB_TRY(h->t.get_f32(who, "fc.weight", (int64_t)INC_CLASSES * INC_FEAT, &d));
        RQB_TRY(h->t.get_f32(who, "fc.bias", INC_CLASSES, &d));
    }
    if (!params) return fail(RQB200_EINVAL, "inception_finalize: null parameter buffer");
    if (params_bytes < rqb200_inception_params_bytes(h))
        return fail(RQB200_EWORKSPACE, "inception_finalize: parameter buffer smaller than rqb200_inception_params_bytes");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "inception_finalize: no CUDA device");
    h->par.bind(params, h->fast);
    for (size_t i = 0; i < h->convs.size(); i++) {       // each BatchNorm folded into its conv
        const IncConv& c = h->convs[i];
        RQB_TRY(launch_conv_prep(ts[i * 5], nullptr, &ts[i * 5 + 1], INC_BN_EPS, h->par, c.w_off, c.b_off, c.cout, c.cin, c.kh, c.kw,
                                 (cudaStream_t)stream));
    }
    h->finalized = true;
    return 0;
}

size_t rqb200_inception_workspace_bytes(rqb200_inception* h, int B, int H, int W, int flags) {
    using namespace rqb;
    if (!h || B <= 0 || H < 1 || W < 1) return 0;
    int Hs, Ws;
    staged_extent(H, W, flags, &Hs, &Ws);
    if (Hs < INC_MIN_EXTENT || Ws < INC_MIN_EXTENT) return 0;
    const int64_t ma = inc_max_act(h, Hs, Ws);
    return inc_layout(chunk_items(B, inc_image_bytes(Hs, Ws, ma, h->fast)), Hs, Ws, ma, h->fast, nullptr, 0, nullptr, nullptr);
}

int rqb200_inception_forward(rqb200_inception* h, const float* x, int B, int H, int W, int flags, float* out0, float* out1, float* out2,
                             float* out3, float* logits, void* workspace, size_t workspace_bytes, void* stream) {
    using namespace rqb;
    if (!h || !x || !workspace) return fail(RQB200_EINVAL, "inception_forward: null argument");
    if (!h->finalized) return fail(RQB200_ESTATE, "inception_forward: engine not finalised");
    if (B <= 0 || H < 1 || W < 1) return fail(RQB200_EINVAL, "inception_forward: B, H and W must be positive");
    int Hs, Ws;
    staged_extent(H, W, flags, &Hs, &Ws);
    if (Hs < INC_MIN_EXTENT || Ws < INC_MIN_EXTENT)
        return fail(RQB200_EINVAL, "inception_forward: without resizing, H and W must be at least 75");
    float* outs[4] = {out0, out1, out2, out3};
    for (int k = 0; k < 4; k++) {
        const bool want = (flags >> (2 + k)) & 1;
        if (want && !outs[k]) return fail(RQB200_EINVAL, "inception_forward: block output " + std::to_string(k) + " requested without a buffer");
        if (want && k > h->cfg.last_block) return fail(RQB200_EINVAL, "inception_forward: block " + std::to_string(k) + " is past the engine's last block");
        if (!want) outs[k] = nullptr;
    }
    const bool want_logits = flags & RQB200_INC_LOGITS;
    if (want_logits && (!logits || h->cfg.last_block != 3))
        return fail(RQB200_EINVAL, "inception_forward: logits need a buffer and an engine through block 3");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "inception_forward: no CUDA device");
    const cudaStream_t st = (cudaStream_t)stream;
    const int64_t ma = inc_max_act(h, Hs, Ws);
    const int chunk = chunk_items(B, inc_image_bytes(Hs, Ws, ma, h->fast));
    IncRun run{h, st, chunk, 2};
    for (int k = 0; k < 3; k++) run.out_nchw[k] = outs[k];
    float* x0 = nullptr;
    if (inc_layout(chunk, Hs, Ws, ma, h->fast, workspace, workspace_bytes, &x0, &run) > workspace_bytes)
        return fail(RQB200_EWORKSPACE, "inception_forward: workspace smaller than rqb200_inception_workspace_bytes");
    g_launches = 0;
    const float* fc_w = want_logits ? (const float*)h->t.find("fc.weight")->ptr : nullptr;
    const float* fc_b = want_logits ? (const float*)h->t.find("fc.bias")->ptr : nullptr;
    int rc = 0;
    for (int b0 = 0; b0 < B && rc == 0; b0 += chunk) {
        const int n = std::min(chunk, B - b0);
        run.B = n;
        rc = launch_inc_input(x + (int64_t)b0 * 3 * H * W, x0, n, H, W, (flags & RQB200_INC_RESIZE) != 0, (flags & RQB200_INC_NORMALIZE) != 0, st);
        run.out_b0 = b0;
        if (rc == 0) rc = run.walk(x0, Hs, Ws);
        if (rc == 0 && outs[3]) {
            const cudaError_t e = cudaMemcpyAsync(outs[3] + (int64_t)b0 * INC_FEAT, run.feat, (size_t)n * INC_FEAT * sizeof(float),
                                                  cudaMemcpyDeviceToDevice, st);
            if (e != cudaSuccess) rc = fail(RQB200_ECUDA, std::string("inception_forward: feature copy: ") + cudaGetErrorString(e));
        }
        if (rc == 0 && want_logits)
            rc = launch_linear(run.feat, INC_FEAT, fc_w, RQB200_F32, fc_b, nullptr, logits + (int64_t)b0 * INC_CLASSES, INC_CLASSES, n,
                               INC_CLASSES, INC_FEAT, 0, st);
    }
    h->last_launches = g_launches;
    return rc;
}

int64_t rqb200_inception_last_launches(const rqb200_inception* h) { return h ? h->last_launches : 0; }

// ---- diagnostic entry points (tests/test_gpu_inception.py): one launch of each Inception kernel through its launcher

int rqb200_dbg_inception_conv(const float* X, const float* Wt, const float* bias, float* out, int B, int H, int W, int Cin, int Cout,
                              int kh, int kw, int pad_h, int pad_w, int stride, int ldy, int yoff, void* stream) {
    using namespace rqb;
    if (B < 1 || Cin < 1 || Cout < 1 || kh < 1 || kw < 1 || pad_h < 0 || pad_w < 0 || stride < 1 || yoff < 0 || ldy < yoff + Cout)
        return fail(RQB200_EINVAL, "dbg_inception_conv: need B, Cin, Cout, kh, kw, stride >= 1, pads >= 0, ldy >= yoff + Cout");
    if (H + 2 * pad_h < kh || W + 2 * pad_w < kw) return fail(RQB200_EINVAL, "dbg_inception_conv: kernel larger than the padded input");
    if (!X || !Wt || !bias || !out) return fail(RQB200_EINVAL, "dbg_inception_conv: null argument");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "dbg_inception_conv: no CUDA device");
    return launch_conv_relu(X, Wt, bias, out, conv_geom(B, H, W, Cin, Cout, kh, kw, pad_h, pad_w, stride, ldy, yoff), (cudaStream_t)stream);
}

int rqb200_dbg_inception_conv_tc(const void* X16, const void* X16lo, const void* W16, const void* W16lo, const float* bias, float* out,
                                 void* out_hi, void* out_lo, int B, int H, int W, int Cin, int Cout, int kh, int kw, int pad_h, int pad_w,
                                 int stride, int ldy, int yoff, void* stream) {
    using namespace rqb;
    if (B < 1 || Cin < 1 || Cout < 1 || kh < 1 || kw < 1 || H + 2 * pad_h < kh || W + 2 * pad_w < kw)
        return fail(RQB200_EINVAL, "dbg_inception_conv_tc: need B, Cin, Cout, kh, kw >= 1 and a kernel inside the padded input");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "dbg_inception_conv_tc: no CUDA device");
    return launch_inc_conv_tc(X16, X16lo, W16, W16lo, bias, out, out_hi, out_lo, B, H, W, Cin, Cout, kh, kw, pad_h, pad_w, stride, ldy, yoff,
                              (cudaStream_t)stream);
}

int rqb200_dbg_inception_input(const float* x, float* y, int B, int H, int W, int resize, int normalize, void* stream) {
    using namespace rqb;
    if (B < 1 || H < 1 || W < 1 || !x || !y) return fail(RQB200_EINVAL, "dbg_inception_input: need B, H, W >= 1 and both pointers");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "dbg_inception_input: no CUDA device");
    return launch_inc_input(x, y, B, H, W, resize != 0, normalize != 0, (cudaStream_t)stream);
}

int rqb200_dbg_inception_pool(int mode, const float* X, float* Y, int B, int H, int W, int C, int stride, int pad, int ldy, int yoff,
                              void* stream) {
    using namespace rqb;
    if ((mode != 0 && mode != 1) || B < 1 || C < 1 || stride < 1 || pad < 0 || pad > 1 || H + 2 * pad < 3 || W + 2 * pad < 3 ||
        yoff < 0 || ldy < yoff + C || !X || !Y)
        return fail(RQB200_EINVAL, "dbg_inception_pool: need mode 0 | 1, pad 0 | 1, a 3x3 window inside the padded map, ldy >= yoff + C");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "dbg_inception_pool: no CUDA device");
    return launch_inc_pool(X, Y, B, H, W, C, stride, pad, mode, ldy, yoff, (cudaStream_t)stream);
}

int rqb200_dbg_inception_gap(const float* X, float* Y, int B, int HW, int C, void* stream) {
    using namespace rqb;
    if (B < 1 || HW < 1 || C < 1 || !X || !Y) return fail(RQB200_EINVAL, "dbg_inception_gap: need B, HW, C >= 1 and both pointers");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "dbg_inception_gap: no CUDA device");
    return launch_inc_gap(X, Y, B, HW, C, (cudaStream_t)stream);
}
}
