// What the layer-plan engines share: the tensor table behind rqb200_<engine>_set_tensor (VAE, Inception, CLIP, LPIPS), and the
// conv-weight preparation and per-conv tier choice of the Inception and LPIPS plans.
#include "kernels.h"

namespace rqb {

const PlanTensor* TensorTable::find(const std::string& key) const {
    auto it = t.find(key);
    return it == t.end() ? nullptr : &it->second;
}

int TensorTable::get_f32(const char* who, const std::string& key, int64_t numel, const float** out) const {
    const PlanTensor* p = find(key);
    if (!p) return fail(RQB200_ESTATE, std::string(who) + ": tensor " + key + " (missing)");
    if (p->numel != numel) return fail(RQB200_ESTATE, std::string(who) + ": tensor " + key + " (wrong size)");
    if (p->dtype != RQB200_F32) return fail(RQB200_EINVAL, std::string(who) + ": tensor " + key + " must be fp32");
    *out = (const float*)p->ptr;
    return 0;
}

__global__ void conv_prep_kernel(const float* __restrict__ w, const float* __restrict__ bias, const float* __restrict__ gamma,
                                 const float* __restrict__ beta, const float* __restrict__ mean, const float* __restrict__ var, double eps,
                                 float* __restrict__ wo, float* __restrict__ bo, __half* __restrict__ whi, __half* __restrict__ wlo, int Cout,
                                 int Cin, int KH, int KW) {
    const int64_t n = (int64_t)Cout * KH * KW * Cin;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int ci = (int)(i % Cin);
        const int kx = (int)((i / Cin) % KW), ky = (int)((i / Cin / KW) % KH), o = (int)(i / Cin / KW / KH);
        const float v = w[(((int64_t)o * Cin + ci) * KH + ky) * KW + kx];
        const float f = gamma ? (float)((double)v * ((double)gamma[o] / sqrt((double)var[o] + eps))) : v;
        wo[i] = f;
        if (whi) split_f16(f, whi[i], wlo[i]);
        if (i < Cout) {
            if (gamma) {
                const double so = (double)gamma[i] / sqrt((double)var[i] + eps);
                bo[i] = (float)((double)beta[i] - (double)mean[i] * so);
            } else {
                bo[i] = bias[i];
            }
        }
    }
}

int launch_conv_prep(const float* w, const float* bias, const float* const* bn, double bn_eps, const SplitParams& P, int64_t w_off,
                     int64_t b_off, int Cout, int Cin, int KH, int KW, cudaStream_t st) {
    conv_prep_kernel<<<grid_1d((int64_t)Cout * KH * KW * Cin), 256, 0, st>>>(
        w, bias, bn ? bn[0] : nullptr, bn ? bn[1] : nullptr, bn ? bn[2] : nullptr, bn ? bn[3] : nullptr, bn_eps, P.f32 + w_off, P.f32 + b_off,
        P.hi ? P.hi + w_off : nullptr, P.lo ? P.lo + w_off : nullptr, Cout, Cin, KH, KW);
    return check_launch("conv_prep");
}

int launch_plan_conv(bool fast, const SplitParams& P, int64_t w_off, int64_t b_off, const float* x, const __half* x_hi,
                     const __half* x_lo, float* y, __half* y_hi, __half* y_lo, const ConvGeom& g, cudaStream_t st) {
    if (fast && x_hi)
        return launch_inc_conv_tc(x_hi, x_lo, P.hi + w_off, P.lo + w_off, P.f32 + b_off, y, y_hi, y_lo, g.B, g.Hi, g.Wi, g.Cin, g.Cout, g.KH,
                                  g.KW, g.pad, g.pad_w, g.stride, g.ldy, g.yoff, st);
    RQB_TRY(launch_conv_relu(x, P.f32 + w_off, P.f32 + b_off, y, g, st));
    return fast ? launch_cast_f16(y, y_hi, y_lo, g.B, g.Ho, g.Wo, g.ldy, 0, st) : 0;
}

}  // namespace rqb
