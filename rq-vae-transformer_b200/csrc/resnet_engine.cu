// torchvision's resnet101 (rqvae/metrics/resnet.py: ResNet101, the v1.5 Bottleneck with the stride on its 3x3) as a static layer plan,
// the classifier of class-conditional rejection sampling.  Every BatchNorm is folded into its conv in fp64 (conv_prep_kernel, eps 1e-5),
// so each conv + bn is one launch.  Two tiers: exact runs every conv on conv_igemm_kernel (fp32 FFMA); fast runs every conv but the Cin = 3
// stem conv1 on inc_conv_tc_kernel (wgmma, split-fp16 operands, three products per k step).  The residual stream stays fp32 on both
// tiers: a bottleneck's conv3 adds the block input (or its downsample conv's output, which has no ReLU) before its ReLU in the conv
// epilogue, and writes the block output as fp32 (the next block's identity) and, on the fast tier, as the next conv1's fp16 hi / lo
// operands.  On the fast tier conv1 and conv2 of a block write only those operands, and the stem's max pool writes them beside its fp32
// map, so no cast pass runs anywhere in the network.
//
// Layer names are torchvision's state_dict keys: conv1 / bn1, layer{1..4}.{i}.conv{1,2,3} / bn{1,2,3}, layer{1..4}.0.downsample.{0,1},
// fc.  Activations are NHWC fp32.  The optional centre crop, the ImageNet normalisation and NCHW -> NHWC are one pass.
#include <vector>

#include "kernels.h"

namespace rqb {

constexpr int RN_MIN_EXTENT = 32;                  // the smallest H, W (after the crop) the engine takes: layer4 sees 1 x 1
constexpr double RN_BN_EPS = 1e-5;                 // nn.BatchNorm2d's default
constexpr int RN_FEAT = 2048, RN_CLASSES = 1000;
constexpr int RN_BLOCKS[4] = {3, 4, 23, 3};        // resnet101's Bottleneck counts per layer

// ------------------------------------------------------------------------------------------------ kernels
// x NCHW [B, 3, H, W] -> y NHWC [B, Hc, Wc, 3]: the Hc x Wc window at (top, left), then transforms.Normalize with ImageNet's mean and
// std: (v - mean[c]) / std[c] in fp32, a subtraction and then a correctly rounded division, as torch computes it
__global__ void resnet_input_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int H, int W, int Hc, int Wc, int top,
                                    int left) {
    const int64_t n = (int64_t)B * Hc * Wc * 3;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % 3);
        const int ox = (int)((i / 3) % Wc), oy = (int)((i / 3 / Wc) % Hc), b = (int)(i / 3 / Wc / Hc);
        const float v = x[(((int64_t)b * 3 + c) * H + oy + top) * W + ox + left];
        const float mean = c == 0 ? 0.485f : (c == 1 ? 0.456f : 0.406f);
        const float sd = c == 0 ? 0.229f : (c == 1 ? 0.224f : 0.225f);
        y[i] = __fdiv_rn(__fsub_rn(v, mean), sd);
    }
}

// torchvision CenterCrop's offset of a c-wide window in n: int(round((n - c) / 2)), Python's round (half to even)
static int crop_offset(int n, int c) {
    const int d = n - c, q = d / 2;
    return (d % 2 == 0 || q % 2 == 0) ? q : q + 1;
}

int launch_resnet_input(const float* x, float* y, int B, int H, int W, int crop, cudaStream_t st) {
    const int Hc = crop ? crop : H, Wc = crop ? crop : W;
    const int top = crop ? crop_offset(H, crop) : 0, left = crop ? crop_offset(W, crop) : 0;
    resnet_input_kernel<<<grid_1d((int64_t)B * Hc * Wc * 3), 256, 0, st>>>(x, y, B, H, W, Hc, Wc, top, left);
    return check_launch("resnet_input");
}

// ------------------------------------------------------------------------------------------------ layer plan
// one conv + BatchNorm: the conv weight under `name`.weight, the BatchNorm under `bn`.{weight,bias,running_mean,running_var}; the folded
// OHWI weight and bias live at w_off / b_off (floats) of the parameter buffer
struct RnConv {
    std::string name, bn;
    int cin, cout, k;
    int64_t w_off, b_off;
};

}  // namespace rqb

struct rqb200_resnet {
    rqb200_resnet_config cfg;
    rqb::TensorTable t;
    std::vector<rqb::RnConv> convs;               // plan order
    rqb::SplitParams par;                         // the folded weights and biases (bound at finalize)
    bool fast = false;                            // RQB200_MODE_FAST
    bool finalized = false;
    int64_t last_launches = 0;
};

namespace rqb {

// buffer slots of a walk: the block input / output (ping-pong), the bottleneck's two temporaries, the downsample output and the staged
// input.  The first four have fp16 hi / lo operand twins on the fast tier.
enum RnSlot { RN_A = 0, RN_B = 1, RN_T1 = 2, RN_T2 = 3, RN_DS = 4, RN_X0 = 5 };

// One walk of the plan serves three purposes: collecting the convs (create), measuring the largest activation of an extent (dry),
// and launching
struct RnRun {
    rqb200_resnet* h;
    cudaStream_t st;
    int B;
    int mode;                         // 0 collect, 1 dry, 2 launch
    float* f[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    __half* hi[4] = {nullptr, nullptr, nullptr, nullptr};
    __half* lo[4] = {nullptr, nullptr, nullptr, nullptr};
    float* feat = nullptr;            // the pooled features [B, 2048]
    int64_t max_act = 0;              // floats per image
    size_t next = 0;                  // launch: the plan index of the next conv

    void note(int64_t hw, int64_t c) { if (hw * c > max_act) max_act = hw * c; }

    // conv `name` + BatchNorm `bn` of a k x k kernel (pad, stride) from slot x [B, H, W, Cin] into slot y [B, Ho, Wo, Cout]; (H, W)
    // becomes the output extent.  res: the slot added before the activation, or -1; relu: ReLU, else the identity.  f32 / half: which
    // forms of the output the next layers read (half only matters on the fast tier)
    int conv(const std::string& name, const std::string& bn, int x, int& H, int& W, int Cin, int y, int Cout, int k, int stride, int pad,
             int res, bool relu, bool f32, bool half) {
        const ConvGeom g = conv_geom(B, H, W, Cin, Cout, k, k, pad, pad, stride, Cout, 0);
        note((int64_t)g.Ho * g.Wo, Cout);
        if (mode == 0) {
            const int64_t w_off = h->par.take((int64_t)Cout * k * k * Cin);
            h->convs.push_back(RnConv{name, bn, Cin, Cout, k, w_off, h->par.take(Cout)});
        }
        if (mode == 2) {
            const RnConv& c = h->convs[next++];
            const bool fast = h->fast;
            // the stem conv reads the staged fp32 input (no fp16 operand): fp32 FFMA on both tiers
            const __half* xh = fast && x < 4 ? hi[x] : nullptr;
            const __half* xl = fast && x < 4 ? lo[x] : nullptr;
            const bool tc = xh != nullptr;
            RQB_TRY(launch_plan_conv(fast, h->par, c.w_off, c.b_off, f[x], xh, xl, (f32 || !tc) ? f[y] : nullptr,
                                     fast && half && y < 4 ? hi[y] : nullptr, fast && half && y < 4 ? lo[y] : nullptr, g, st,
                                     res >= 0 ? f[res] : nullptr, relu));
        }
        H = g.Ho;
        W = g.Wo;
        return 0;
    }

    // the network from the staged NHWC input [B, H, W, 3] to the pooled features
    int walk(int H, int W) {
        const bool fast = h->fast;
        RQB_TRY(conv("conv1", "bn1", RN_X0, H, W, 3, RN_T1, 64, 7, 2, 3, -1, true, true, false));
        // maxpool 3x3 / 2, pad 1 (padding acts as -inf); on the fast tier it also writes layer1's fp16 operands
        const int Hp = (H + 2 - 3) / 2 + 1, Wp = (W + 2 - 3) / 2 + 1;
        note((int64_t)Hp * Wp, 64);
        if (mode == 2)
            RQB_TRY(launch_inc_pool(f[RN_T1], f[RN_A], B, H, W, 64, 2, 1, 0, 64, 0, st, fast ? hi[RN_A] : nullptr, fast ? lo[RN_A] : nullptr));
        H = Hp;
        W = Wp;
        int x = RN_A, C = 64;
        for (int L = 0; L < 4; L++) {
            const int width = 64 << L;
            for (int i = 0; i < RN_BLOCKS[L]; i++) {
                const std::string p = "layer" + std::to_string(L + 1) + "." + std::to_string(i) + ".";
                const int stride = (i == 0 && L > 0) ? 2 : 1, y = x == RN_A ? RN_B : RN_A;
                int h1 = H, w1 = W;
                RQB_TRY(conv(p + "conv1", p + "bn1", x, h1, w1, C, RN_T1, width, 1, 1, 0, -1, true, !fast, true));
                RQB_TRY(conv(p + "conv2", p + "bn2", RN_T1, h1, w1, width, RN_T2, width, 3, stride, 1, -1, true, !fast, true));
                int res = x;
                if (i == 0) {
                    int hd = H, wd = W;
                    RQB_TRY(conv(p + "downsample.0", p + "downsample.1", x, hd, wd, C, RN_DS, 4 * width, 1, stride, 0, -1, false, true, false));
                    res = RN_DS;
                }
                RQB_TRY(conv(p + "conv3", p + "bn3", RN_T2, h1, w1, width, y, 4 * width, 1, 1, 0, res, true, true, true));
                H = h1;
                W = w1;
                C = 4 * width;
                x = y;
            }
        }
        if (mode == 2) RQB_TRY(launch_inc_gap(f[x], feat, B, H * W, RN_FEAT, st));
        return 0;
    }
};

static int64_t rn_max_act(rqb200_resnet* h, int Hs, int Ws) {
    RnRun d{h, nullptr, 1, 1};
    d.walk(Hs, Ws);
    return d.max_act;
}
// per image: the staged input, five fp32 activation buffers and the pooled features; the fast tier's eight fp16 operand buffers
static size_t rn_image_bytes(int Hs, int Ws, int64_t max_act, bool fast) {
    return ((size_t)Hs * Ws * 3 + 5 * (size_t)max_act + RN_FEAT) * sizeof(float) + (fast ? 8 * (size_t)max_act * sizeof(__half) : 0);
}
static size_t rn_layout(int n, int Hs, int Ws, int64_t max_act, bool fast, void* base, size_t cap, RnRun* run) {
    Arena ar(base, cap);
    float* x0 = ar.take<float>((size_t)n * Hs * Ws * 3);
    float* bufs[5];
    for (int i = 0; i < 5; i++) bufs[i] = ar.take<float>((size_t)n * max_act);
    float* feat = ar.take<float>((size_t)n * RN_FEAT);
    if (run) {
        for (int i = 0; i < 5; i++) run->f[i] = bufs[i];
        run->f[RN_X0] = x0;
        run->feat = feat;
    }
    if (fast)
        for (int i = 0; i < 4; i++) {
            __half* ph = ar.take<__half>((size_t)n * max_act);
            __half* pl = ar.take<__half>((size_t)n * max_act);
            if (run) { run->hi[i] = ph; run->lo[i] = pl; }
        }
    return ar.off + 256;
}

// the extent the network sees: crop x crop, or the input's own; false when the engine does not take it
static bool rn_extent(int H, int W, int flags, int* Hs, int* Ws) {
    const int crop = flags >> 8;
    if (crop < 0 || (crop > 0 && (crop > H || crop > W))) return false;
    *Hs = crop ? crop : H;
    *Ws = crop ? crop : W;
    return *Hs >= RN_MIN_EXTENT && *Ws >= RN_MIN_EXTENT;
}

}  // namespace rqb

extern "C" {

rqb200_resnet* rqb200_resnet_create(const rqb200_resnet_config* cfg) {
    if (!cfg || (cfg->mode != RQB200_MODE_EXACT && cfg->mode != RQB200_MODE_FAST)) {
        rqb::set_error("resnet_create: mode must be RQB200_MODE_EXACT or RQB200_MODE_FAST");
        return nullptr;
    }
    rqb200_resnet* h = new rqb200_resnet();
    h->cfg = *cfg;
    h->fast = cfg->mode == RQB200_MODE_FAST;
    rqb::RnRun c{h, nullptr, 1, 0};
    c.walk(224, 224);
    return h;
}
void rqb200_resnet_destroy(rqb200_resnet* h) { delete h; }

int rqb200_resnet_set_tensor(rqb200_resnet* h, const char* key, const void* ptr, int dtype, int64_t numel) {
    if (!h || !key || !ptr) return rqb::fail(RQB200_EINVAL, "resnet_set_tensor: null argument");
    h->t.set(key, ptr, dtype, numel);
    h->finalized = false;
    return 0;
}

size_t rqb200_resnet_params_bytes(const rqb200_resnet* h) { return h ? h->par.bytes(h->fast) : 0; }

int rqb200_resnet_finalize(rqb200_resnet* h, void* params, size_t params_bytes, void* stream) {
    using namespace rqb;
    if (!h) return fail(RQB200_EINVAL, "resnet_finalize: null handle");
    h->finalized = false;
    const char* who = "resnet_finalize";
    std::vector<const float*> ts(h->convs.size() * 5);
    for (size_t i = 0; i < h->convs.size(); i++) {
        const RnConv& c = h->convs[i];
        RQB_TRY(h->t.get_f32(who, c.name + ".weight", (int64_t)c.cout * c.cin * c.k * c.k, &ts[i * 5]));
        static const char* bn[4] = {".weight", ".bias", ".running_mean", ".running_var"};
        for (int j = 0; j < 4; j++) RQB_TRY(h->t.get_f32(who, c.bn + bn[j], c.cout, &ts[i * 5 + 1 + j]));
    }
    const float* d;
    RQB_TRY(h->t.get_f32(who, "fc.weight", (int64_t)RN_CLASSES * RN_FEAT, &d));
    RQB_TRY(h->t.get_f32(who, "fc.bias", RN_CLASSES, &d));
    if (!params) return fail(RQB200_EINVAL, "resnet_finalize: null parameter buffer");
    if (params_bytes < rqb200_resnet_params_bytes(h))
        return fail(RQB200_EWORKSPACE, "resnet_finalize: parameter buffer smaller than rqb200_resnet_params_bytes");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "resnet_finalize: no CUDA device");
    h->par.bind(params, h->fast);
    for (size_t i = 0; i < h->convs.size(); i++) {       // each BatchNorm folded into its conv
        const RnConv& c = h->convs[i];
        RQB_TRY(launch_conv_prep(ts[i * 5], nullptr, &ts[i * 5 + 1], RN_BN_EPS, h->par, c.w_off, c.b_off, c.cout, c.cin, c.k, c.k,
                                 (cudaStream_t)stream));
    }
    h->finalized = true;
    return 0;
}

size_t rqb200_resnet_workspace_bytes(rqb200_resnet* h, int B, int H, int W, int flags) {
    using namespace rqb;
    int Hs, Ws;
    if (!h || B <= 0 || !rn_extent(H, W, flags, &Hs, &Ws)) return 0;
    const int64_t ma = rn_max_act(h, Hs, Ws);
    return rn_layout(chunk_items(B, rn_image_bytes(Hs, Ws, ma, h->fast)), Hs, Ws, ma, h->fast, nullptr, 0, nullptr);
}

int rqb200_resnet_forward(rqb200_resnet* h, const float* x, int B, int H, int W, int flags, float* logits, float* features, void* workspace,
                          size_t workspace_bytes, void* stream) {
    using namespace rqb;
    if (!h || !x || !logits || !workspace) return fail(RQB200_EINVAL, "resnet_forward: null argument");
    if (!h->finalized) return fail(RQB200_ESTATE, "resnet_forward: engine not finalised");
    int Hs, Ws;
    if (B <= 0 || !rn_extent(H, W, flags, &Hs, &Ws))
        return fail(RQB200_EINVAL, "resnet_forward: need B >= 1, a crop no larger than H and W, and an extent of at least 32 x 32");
    if ((flags & RQB200_RESNET_FEATURES) && !features) return fail(RQB200_EINVAL, "resnet_forward: features requested without a buffer");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "resnet_forward: no CUDA device");
    const cudaStream_t st = (cudaStream_t)stream;
    const int64_t ma = rn_max_act(h, Hs, Ws);
    const int chunk = chunk_items(B, rn_image_bytes(Hs, Ws, ma, h->fast));
    RnRun run{h, st, chunk, 2};
    if (rn_layout(chunk, Hs, Ws, ma, h->fast, workspace, workspace_bytes, &run) > workspace_bytes)
        return fail(RQB200_EWORKSPACE, "resnet_forward: workspace smaller than rqb200_resnet_workspace_bytes");
    g_launches = 0;
    const float* fc_w = (const float*)h->t.find("fc.weight")->ptr;
    const float* fc_b = (const float*)h->t.find("fc.bias")->ptr;
    int rc = 0;
    for (int b0 = 0; b0 < B && rc == 0; b0 += chunk) {
        const int n = std::min(chunk, B - b0);
        run.B = n;
        run.next = 0;
        rc = launch_resnet_input(x + (int64_t)b0 * 3 * H * W, run.f[RN_X0], n, H, W, flags >> 8, st);
        if (rc == 0) rc = run.walk(Hs, Ws);
        if (rc == 0 && (flags & RQB200_RESNET_FEATURES)) {
            const cudaError_t e = cudaMemcpyAsync(features + (int64_t)b0 * RN_FEAT, run.feat, (size_t)n * RN_FEAT * sizeof(float),
                                                  cudaMemcpyDeviceToDevice, st);
            if (e != cudaSuccess) rc = fail(RQB200_ECUDA, std::string("resnet_forward: feature copy: ") + cudaGetErrorString(e));
        }
        if (rc == 0)
            rc = launch_linear(run.feat, RN_FEAT, fc_w, RQB200_F32, fc_b, nullptr, logits + (int64_t)b0 * RN_CLASSES, RN_CLASSES, n, RN_CLASSES,
                               RN_FEAT, 0, st);
    }
    h->last_launches = g_launches;
    return rc;
}

int64_t rqb200_resnet_last_launches(const rqb200_resnet* h) { return h ? h->last_launches : 0; }

// ---- diagnostic entry points (tests/test_gpu_resnet.py): the input kernel and the residual forms of both conv kernels

int rqb200_dbg_resnet_input(const float* x, float* y, int B, int H, int W, int crop, void* stream) {
    using namespace rqb;
    if (B < 1 || H < 1 || W < 1 || crop < 0 || crop > H || crop > W || !x || !y)
        return fail(RQB200_EINVAL, "dbg_resnet_input: need B, H, W >= 1, 0 <= crop <= H, W and both pointers");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "dbg_resnet_input: no CUDA device");
    return launch_resnet_input(x, y, B, H, W, crop, (cudaStream_t)stream);
}

int rqb200_dbg_resnet_conv(const float* X, const float* Wt, const float* bias, const float* residual, float* out, int B, int H, int W, int Cin,
                           int Cout, int k, int pad, int stride, int ldy, int yoff, int relu, void* stream) {
    using namespace rqb;
    if (B < 1 || Cin < 1 || Cout < 1 || k < 1 || pad < 0 || stride < 1 || yoff < 0 || ldy < yoff + Cout || H + 2 * pad < k ||
        W + 2 * pad < k || !X || !Wt || !bias || !out)
        return fail(RQB200_EINVAL, "dbg_resnet_conv: need B, Cin, Cout, k, stride >= 1, pad >= 0, ldy >= yoff + Cout, a kernel inside "
                                   "the padded input and every pointer but the residual");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "dbg_resnet_conv: no CUDA device");
    return launch_conv_res(X, Wt, bias, residual, out, conv_geom(B, H, W, Cin, Cout, k, k, pad, pad, stride, ldy, yoff), relu != 0,
                           (cudaStream_t)stream);
}

int rqb200_dbg_resnet_conv_tc(const void* X16, const void* X16lo, const void* W16, const void* W16lo, const float* bias, const float* residual,
                              float* out, void* out_hi, void* out_lo, int B, int H, int W, int Cin, int Cout, int k, int pad, int stride,
                              int ldy, int yoff, int relu, void* stream) {
    using namespace rqb;
    if (B < 1 || Cin < 1 || Cout < 1 || k < 1 || pad < 0 || H + 2 * pad < k || W + 2 * pad < k)
        return fail(RQB200_EINVAL, "dbg_resnet_conv_tc: need B, Cin, Cout, k >= 1, pad >= 0 and a kernel inside the padded input");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "dbg_resnet_conv_tc: no CUDA device");
    return launch_inc_conv_tc(X16, X16lo, W16, W16lo, bias, out, out_hi, out_lo, B, H, W, Cin, Cout, k, k, pad, pad, stride, ldy, yoff,
                              (cudaStream_t)stream, relu ? 1 : 2, residual);
}
}
