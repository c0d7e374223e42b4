// P2 host orchestration -- RQVAE.encode / decode / decode_code as a static layer plan over the kernels in
// conv_kernels.cu (exact tier) / conv_tc.cu (fast tier).
//
// Mirrors rqvae/models/rqvae/rqvae.py:80-109 and modules.py (Encoder.forward :73-98, Decoder.forward :171-202);
// layer names are the reference's state_dict keys (SURVEY.md A.3/A.4) so a checkpoint loads unchanged.
// Differences in execution, not arithmetic: activations stay NHWC end to end (the reference permutes NHWC<->NCHW at
// rqvae.py:82,86), the nearest-x2 upsample and the (0,1,0,1) pad are folded into conv indexing, q/k/v 1x1 convs run as
// one Cout=3C GEMM, and the whole batch is decoded in one pass (the reference's callers decode image by image).
#include <string>
#include <unordered_map>
#include <vector>

#include "kernels.h"

struct VTensor {
    const void* ptr;
    int dtype;
    int64_t numel;
};

struct rqb200_vae {
    rqb200_vae_config cfg;
    std::unordered_map<std::string, VTensor> t;
    bool finalized = false;
    bool fast_ok = false;     // FAST mode and every decoder channel count is a multiple of 128
    bool split = false;       // split-fp16 (3 products per conv): "<key>.weight_lo" tensors registered
    bool enc_fast = false;    // the encoder's convs were registered in fp16 as well: encode on the wgmma path
    bool gn_fuse = true;      // conv epilogues emit the next GroupNorm's partial statistics (mode bit RQB200_VAE_NO_GN_FUSE clears it)
    int64_t last_launches = 0;
    int64_t max_act = 0;      // max H*W*C per image over all activations
    int64_t max_gn_hw = 0;
    rqb::RqTables codebooks{};   // decode_code's embedding tables, resolved by finalize from "codebook" or "codebook.<d>"
};

namespace rqb {

struct VaeRun {
    rqb200_vae* h;
    cudaStream_t st;
    int B;
    bool dry;                 // dry run: only check tensors / measure buffer sizes
    float* buf[4];
    double* gn_ws;
    std::string missing;
    __half* h16[2] = {nullptr, nullptr};      // fast tier: fp16 conv operands (GN output / cast / upsampled cast)
    __half* l16[2] = {nullptr, nullptr};      // their fp16 'lo' halves (split-fp16 products); null -> single product
    bool fast = false;

    // ---- fast tier helpers (wgmma implicit GEMM; decoder only, C % 128 == 0 everywhere)
    // want_stats: the output feeds a GroupNorm next -> its epilogue emits the GroupNorm partial statistics (no gn_stats pass)
    const float* stats_buf = nullptr;         // conv output whose statistics sit in gn_ws
    int stats_chunks = 0;
    int conv_f(const std::string& name, const __half* in16, float* out, const float* resid, int Hh, int Ww, int Cin, int Cout,
               int ks, int out_nchw, int stride = 1, bool want_stats = false) {
        const VTensor* w = get(name + ".weight", (int64_t)Cout * ks * ks * Cin);
        const VTensor* b = get(name + ".bias", Cout);
        note_act((int64_t)Hh * Ww, Cout);
        if (dry || !w || !b) return 0;
        if (w->dtype != RQB200_F16) return fail(RQB200_ESTATE, "vae fast tier: conv weights must be fp16: " + name);
        const __half* in_lo = nullptr;
        const void* w_lo = nullptr;
        if (h->split) {
            const VTensor* wl = get(name + ".weight_lo", (int64_t)Cout * ks * ks * Cin);
            if (!wl) return 0;
            w_lo = wl->ptr;
            in_lo = in16 == h16[0] ? l16[0] : l16[1];
        }
        const bool fuse = want_stats && h->gn_fuse && !out_nchw && conv_tc_gn_fusable(Hh, Ww, Cout, ks, stride);
        stats_buf = fuse ? out : nullptr;
        stats_chunks = fuse ? Hh * Ww / 32 : 0;
        return launch_conv_tc(in16, w->ptr, in_lo, w_lo, (const float*)b->ptr, resid, out, B, Hh, Ww, Cin, Cout, ks, out_nchw, st, stride,
                              fuse ? gn_ws : nullptr);
    }
    int gn_f(const std::string& name, const float* in, __half* out16, int HW, int C, int silu) {
        const VTensor* g = get(name + ".weight", C);
        const VTensor* b = get(name + ".bias", C);
        if (HW > h->max_gn_hw) h->max_gn_hw = HW;
        if (dry || !g || !b) return 0;
        const int fused = (in == stats_buf) ? stats_chunks : 0;
        stats_buf = nullptr;
        return launch_groupnorm_f16(in, (const float*)g->ptr, (const float*)b->ptr, out16, out16 == h16[0] ? l16[0] : l16[1], gn_ws, B, HW, C, silu, st,
                                    fused);
    }
    int resblock_f(const std::string& p, int cur, int Hh, int Ww, int Cin, int Cout, int* rc) {
        int a = (cur + 1) & 3, b = (cur + 2) & 3, c = (cur + 3) & 3;
        (void)a;
        *rc = gn_f(p + ".norm1", buf[cur], h16[0], Hh * Ww, Cin, 1); if (*rc) return cur;
        *rc = conv_f(p + ".conv1", h16[0], buf[b], nullptr, Hh, Ww, Cin, Cout, 3, 0, 1, true); if (*rc) return cur;
        *rc = gn_f(p + ".norm2", buf[b], h16[0], Hh * Ww, Cout, 1); if (*rc) return cur;
        const float* res = buf[cur];
        if (Cin != Cout) {
            if (!dry) { *rc = launch_cast_f16(buf[cur], h16[1], l16[1], B, Hh, Ww, Cin, 0, st); if (*rc) return cur; }
            *rc = conv_f(p + ".nin_shortcut", h16[1], buf[c], nullptr, Hh, Ww, Cin, Cout, 1, 0); if (*rc) return cur;
            res = buf[c];
        }
        *rc = conv_f(p + ".conv2", h16[0], buf[b], res, Hh, Ww, Cout, Cout, 3, 0, 1, true);
        return b;
    }
    int attnblock_f(const std::string& p, int cur, int Hh, int Ww, int C, int* rc) {
        int a = (cur + 1) & 3, b = (cur + 2) & 3, c = (cur + 3) & 3;
        *rc = gn_f(p + ".norm", buf[cur], h16[0], Hh * Ww, C, 0); if (*rc) return cur;
        *rc = conv_f(p + ".qkv", h16[0], buf[b], nullptr, Hh, Ww, C, 3 * C, 1, 0); if (*rc) return cur;
        if (!dry && missing.empty()) {
            *rc = launch_vae_attn(buf[b], buf[a], B, Hh * Ww, C, st); if (*rc) return cur;
            *rc = launch_cast_f16(buf[a], h16[0], l16[0], B, Hh, Ww, C, 0, st); if (*rc) return cur;
        }
        *rc = conv_f(p + ".proj_out", h16[0], buf[c], buf[cur], Hh, Ww, C, C, 1, 0, 1, true);
        return c;
    }
    int decode_fast(const float* z, float* out) {
        const rqb200_vae_config& c = h->cfg;
        const int nl = c.n_levels, nb = c.num_res_blocks;
        int res = c.resolution >> (nl - 1), rc = 0;
        int ch = c.ch * c.ch_mult[nl - 1];
        int cur = 0;
        if (!dry) { rc = launch_cast_f16(z, h16[0], l16[0], B, res, res, c.embed_dim, 0, st); if (rc) return rc; }
        rc = conv_f("post_quant_conv", h16[0], buf[1], nullptr, res, res, c.embed_dim, c.z_channels, 1, 0); if (rc) return rc;
        if (!dry) { rc = launch_cast_f16(buf[1], h16[0], l16[0], B, res, res, c.z_channels, 0, st); if (rc) return rc; }
        rc = conv_f("decoder.conv_in", h16[0], buf[0], nullptr, res, res, c.z_channels, ch, 3, 0, 1, true); if (rc) return rc;
        cur = resblock_f("decoder.mid.block_1", cur, res, res, ch, ch, &rc); if (rc) return rc;
        cur = attnblock_f("decoder.mid.attn_1", cur, res, res, ch, &rc); if (rc) return rc;
        cur = resblock_f("decoder.mid.block_2", cur, res, res, ch, ch, &rc); if (rc) return rc;
        for (int lvl = nl - 1; lvl >= 0; lvl--) {
            int cout = c.ch * c.ch_mult[lvl];
            for (int b = 0; b <= nb; b++) {
                std::string p = "decoder.up." + std::to_string(lvl);
                cur = resblock_f(p + ".block." + std::to_string(b), cur, res, res, ch, cout, &rc); if (rc) return rc;
                ch = cout;
                if (has_attn(res)) { cur = attnblock_f(p + ".attn." + std::to_string(b), cur, res, res, ch, &rc); if (rc) return rc; }
            }
            if (lvl != 0) {
                int nxt = (cur + 1) & 3;
                if (!dry) { rc = launch_cast_f16(buf[cur], h16[1], l16[1], B, res, res, ch, 1, st); if (rc) return rc; }   // x2 nearest, fp16
                rc = conv_f("decoder.up." + std::to_string(lvl) + ".upsample.conv", h16[1], buf[nxt], nullptr, 2 * res, 2 * res, ch, ch, 3, 0, 1, true);
                if (rc) return rc;
                cur = nxt;
                res *= 2;
            }
        }
        rc = gn_f("decoder.norm_out", buf[cur], h16[0], res * res, ch, 1); if (rc) return rc;
        return conv_f("decoder.conv_out", h16[0], out, nullptr, res, res, ch, c.out_ch, 3, 1);
    }

    const VTensor* get(const std::string& k, int64_t numel) {
        auto it = h->t.find(k);
        if (it == h->t.end() || it->second.numel != numel) {
            if (missing.empty()) missing = k + (it == h->t.end() ? " (missing)" : " (wrong size)");
            return nullptr;
        }
        return &it->second;
    }
    void note_act(int64_t hw, int64_t c) { if (hw * c > h->max_act) h->max_act = hw * c; }

    int conv(const std::string& name, const float* in, float* out, const float* resid, int Hi, int Wi, int Cin, int Cout,
             int ks, int stride, int upsample, int in_nchw, int out_nchw) {
        ConvGeom g;
        g.B = B; g.Hi = Hi; g.Wi = Wi; g.Cin = Cin; g.Cout = Cout; g.KH = g.KW = ks; g.stride = stride;
        g.upsample = upsample; g.in_nchw = in_nchw; g.out_nchw = out_nchw;
        g.pad = (ks == 3 && stride == 1) ? 1 : 0;
        int Hv = upsample ? 2 * Hi : Hi, Wv = upsample ? 2 * Wi : Wi;
        g.Ho = stride == 2 ? Hv / 2 : Hv;
        g.Wo = stride == 2 ? Wv / 2 : Wv;
        const VTensor* w = get(name + ".weight", (int64_t)Cout * ks * ks * Cin);
        const VTensor* b = get(name + ".bias", Cout);
        note_act((int64_t)g.Ho * g.Wo, Cout);
        if (dry || !w || !b) return 0;
        return launch_conv(in, w->ptr, w->dtype, (const float*)b->ptr, resid, out, g, st);
    }
    int gn(const std::string& name, const float* in, float* out, int HW, int C, int silu) {
        const VTensor* g = get(name + ".weight", C);
        const VTensor* b = get(name + ".bias", C);
        if (HW > h->max_gn_hw) h->max_gn_hw = HW;
        note_act(HW, C);
        if (dry || !g || !b) return 0;
        return launch_groupnorm_silu(in, (const float*)g->ptr, (const float*)b->ptr, out, gn_ws, B, HW, C, silu, st);
    }
    // buffers: cur = index of the live activation; returns new cur
    int resblock(const std::string& p, int cur, int Hh, int Ww, int Cin, int Cout, int* rc) {
        int a = (cur + 1) & 3, b = (cur + 2) & 3, c = (cur + 3) & 3;
        *rc = gn(p + ".norm1", buf[cur], buf[a], Hh * Ww, Cin, 1); if (*rc) return cur;
        *rc = conv(p + ".conv1", buf[a], buf[b], nullptr, Hh, Ww, Cin, Cout, 3, 1, 0, 0, 0); if (*rc) return cur;
        *rc = gn(p + ".norm2", buf[b], buf[a], Hh * Ww, Cout, 1); if (*rc) return cur;
        const float* res = buf[cur];
        if (Cin != Cout) {
            *rc = conv(p + ".nin_shortcut", buf[cur], buf[c], nullptr, Hh, Ww, Cin, Cout, 1, 1, 0, 0, 0); if (*rc) return cur;
            res = buf[c];
        }
        *rc = conv(p + ".conv2", buf[a], buf[b], res, Hh, Ww, Cout, Cout, 3, 1, 0, 0, 0);
        return b;
    }
    int attnblock(const std::string& p, int cur, int Hh, int Ww, int C, int* rc) {
        int a = (cur + 1) & 3, b = (cur + 2) & 3, c = (cur + 3) & 3;
        *rc = gn(p + ".norm", buf[cur], buf[a], Hh * Ww, C, 0); if (*rc) return cur;
        // fused q|k|v 1x1 conv: key "<p>.qkv" registered by the host binding ([3C,1,1,C] / [3C])
        *rc = conv(p + ".qkv", buf[a], buf[b], nullptr, Hh, Ww, C, 3 * C, 1, 1, 0, 0, 0); if (*rc) return cur;
        if (!dry && missing.empty()) { *rc = launch_vae_attn(buf[b], buf[a], B, Hh * Ww, C, st); if (*rc) return cur; }
        *rc = conv(p + ".proj_out", buf[a], buf[c], buf[cur], Hh, Ww, C, C, 1, 1, 0, 0, 0);
        return c;
    }
    bool has_attn(int res) const {
        for (int i = 0; i < h->cfg.n_attn_res; i++) if (h->cfg.attn_resolutions[i] == res) return true;
        return false;
    }

    // Decoder.forward (modules.py:171-202) preceded by post_quant_conv (rqvae.py:87).  z NHWC [B,r,r,embed_dim].
    int decode(const float* z, float* out) {
        if (fast) return decode_fast(z, out);
        const rqb200_vae_config& c = h->cfg;
        const int nl = c.n_levels, nb = c.num_res_blocks;
        int res = c.resolution >> (nl - 1), rc = 0;
        int ch = c.ch * c.ch_mult[nl - 1];
        int cur = 0;
        rc = conv("post_quant_conv", z, buf[1], nullptr, res, res, c.embed_dim, c.z_channels, 1, 1, 0, 0, 0); if (rc) return rc;
        rc = conv("decoder.conv_in", buf[1], buf[0], nullptr, res, res, c.z_channels, ch, 3, 1, 0, 0, 0); if (rc) return rc;
        cur = resblock("decoder.mid.block_1", cur, res, res, ch, ch, &rc); if (rc) return rc;
        cur = attnblock("decoder.mid.attn_1", cur, res, res, ch, &rc); if (rc) return rc;
        cur = resblock("decoder.mid.block_2", cur, res, res, ch, ch, &rc); if (rc) return rc;
        for (int lvl = nl - 1; lvl >= 0; lvl--) {
            int cout = c.ch * c.ch_mult[lvl];
            for (int b = 0; b <= nb; b++) {
                std::string p = "decoder.up." + std::to_string(lvl);
                cur = resblock(p + ".block." + std::to_string(b), cur, res, res, ch, cout, &rc); if (rc) return rc;
                ch = cout;
                if (has_attn(res)) { cur = attnblock(p + ".attn." + std::to_string(b), cur, res, res, ch, &rc); if (rc) return rc; }
            }
            if (lvl != 0) {
                int nxt = (cur + 1) & 3;
                rc = conv("decoder.up." + std::to_string(lvl) + ".upsample.conv", buf[cur], buf[nxt], nullptr, res, res, ch, ch, 3, 1, 1, 0, 0);
                if (rc) return rc;
                cur = nxt;
                res *= 2;
            }
        }
        int a = (cur + 1) & 3;
        rc = gn("decoder.norm_out", buf[cur], buf[a], res * res, ch, 1); if (rc) return rc;
        return conv("decoder.conv_out", buf[a], out, nullptr, res, res, ch, c.out_ch, 3, 1, 0, 0, 1);
    }

    // fast-tier encoder: every conv but conv_in on the wgmma path through the decoder's building blocks, the five stride-2
    // Downsample convs included (tensor map with element stride 2); conv_in (Cin = 3, NCHW fp32 input, 0.3 % of the encoder's
    // flops) stays on the fp32 FFMA kernel
    int encode_fast(const float* x, float* z_e) {
        const rqb200_vae_config& c = h->cfg;
        const int nl = c.n_levels, nb = c.num_res_blocks;
        int res = c.resolution, rc = 0, ch = c.ch, cur = 0;
        rc = conv("encoder.conv_in", x, buf[0], nullptr, res, res, c.in_channels, ch, 3, 1, 0, 1, 0); if (rc) return rc;
        for (int lvl = 0; lvl < nl; lvl++) {
            int cout = c.ch * c.ch_mult[lvl];
            std::string p = "encoder.down." + std::to_string(lvl);
            for (int b = 0; b < nb; b++) {
                cur = resblock_f(p + ".block." + std::to_string(b), cur, res, res, ch, cout, &rc); if (rc) return rc;
                ch = cout;
                if (has_attn(res)) { cur = attnblock_f(p + ".attn." + std::to_string(b), cur, res, res, ch, &rc); if (rc) return rc; }
            }
            if (lvl != nl - 1) {
                int nxt = (cur + 1) & 3;
                // Downsample (layers.py:50-57): pad (0,1,0,1) + 3x3 stride 2 = the same implicit GEMM through a tensor map that
                // samples every other pixel; the one-pixel right/bottom pad is its out-of-bounds fill
                if (!dry) { rc = launch_cast_f16(buf[cur], h16[1], l16[1], B, res, res, ch, 0, st); if (rc) return rc; }
                rc = conv_f(p + ".downsample.conv", h16[1], buf[nxt], nullptr, res / 2, res / 2, ch, ch, 3, 0, 2, true); if (rc) return rc;
                cur = nxt;
                res /= 2;
            }
        }
        cur = resblock_f("encoder.mid.block_1", cur, res, res, ch, ch, &rc); if (rc) return rc;
        cur = attnblock_f("encoder.mid.attn_1", cur, res, res, ch, &rc); if (rc) return rc;
        cur = resblock_f("encoder.mid.block_2", cur, res, res, ch, ch, &rc); if (rc) return rc;
        int b2 = (cur + 2) & 3;
        rc = gn_f("encoder.norm_out", buf[cur], h16[0], res * res, ch, 1); if (rc) return rc;
        rc = conv_f("encoder.conv_out", h16[0], buf[b2], nullptr, res, res, ch, c.z_channels, 3, 0); if (rc) return rc;
        if (!dry) { rc = launch_cast_f16(buf[b2], h16[0], l16[0], B, res, res, c.z_channels, 0, st); if (rc) return rc; }
        return conv_f("quant_conv", h16[0], z_e, nullptr, res, res, c.z_channels, c.embed_dim, 1, 0);
    }

    // Encoder.forward (modules.py:73-98) followed by quant_conv (rqvae.py:82).  x NCHW -> z_e NHWC.
    int encode(const float* x, float* z_e) {
        if (fast && h->enc_fast) return encode_fast(x, z_e);
        const rqb200_vae_config& c = h->cfg;
        const int nl = c.n_levels, nb = c.num_res_blocks;
        int res = c.resolution, rc = 0, ch = c.ch, cur = 0;
        rc = conv("encoder.conv_in", x, buf[0], nullptr, res, res, c.in_channels, ch, 3, 1, 0, 1, 0); if (rc) return rc;
        for (int lvl = 0; lvl < nl; lvl++) {
            int cout = c.ch * c.ch_mult[lvl];
            std::string p = "encoder.down." + std::to_string(lvl);
            for (int b = 0; b < nb; b++) {
                cur = resblock(p + ".block." + std::to_string(b), cur, res, res, ch, cout, &rc); if (rc) return rc;
                ch = cout;
                if (has_attn(res)) { cur = attnblock(p + ".attn." + std::to_string(b), cur, res, res, ch, &rc); if (rc) return rc; }
            }
            if (lvl != nl - 1) {
                int nxt = (cur + 1) & 3;
                rc = conv(p + ".downsample.conv", buf[cur], buf[nxt], nullptr, res, res, ch, ch, 3, 2, 0, 0, 0); if (rc) return rc;
                cur = nxt;
                res /= 2;
            }
        }
        cur = resblock("encoder.mid.block_1", cur, res, res, ch, ch, &rc); if (rc) return rc;
        cur = attnblock("encoder.mid.attn_1", cur, res, res, ch, &rc); if (rc) return rc;
        cur = resblock("encoder.mid.block_2", cur, res, res, ch, ch, &rc); if (rc) return rc;
        int a = (cur + 1) & 3, b2 = (cur + 2) & 3;
        rc = gn("encoder.norm_out", buf[cur], buf[a], res * res, ch, 1); if (rc) return rc;
        rc = conv("encoder.conv_out", buf[a], buf[b2], nullptr, res, res, ch, c.z_channels, 3, 1, 0, 0, 0); if (rc) return rc;
        return conv("quant_conv", buf[b2], z_e, nullptr, res, res, c.z_channels, c.embed_dim, 1, 1, 0, 0, 0);
    }
};

static size_t vae_layout(const rqb200_vae* h, int B, void* base, size_t cap, VaeRun* run) {
    Arena a(base, cap);
    for (int i = 0; i < 4; i++) {
        float* p = a.take<float>((size_t)B * h->max_act);
        if (run) run->buf[i] = p;
    }
    double* g = a.take<double>(groupnorm_ws_doubles(B, (int)h->max_gn_hw));
    if (run) run->gn_ws = g;
    const rqb200_vae_config& c = h->cfg;
    int r = c.resolution >> (c.n_levels - 1);
    float* zq = a.take<float>((size_t)B * r * r * c.embed_dim);      // decode_code staging
    (void)zq;
    for (int i = 0; i < 2; i++) {
        __half* p16 = a.take<__half>((size_t)B * h->max_act);
        if (run) run->h16[i] = p16;
    }
    if (h->split)
        for (int i = 0; i < 2; i++) {
            __half* p16 = a.take<__half>((size_t)B * h->max_act);
            if (run) run->l16[i] = p16;
        }
    return a.off + 256;
}

static float* vae_zq_buffer(const rqb200_vae* h, int B, void* base, size_t cap) {
    Arena a(base, cap);
    for (int i = 0; i < 4; i++) a.take<float>((size_t)B * h->max_act);
    a.take<double>(groupnorm_ws_doubles(B, (int)h->max_gn_hw));
    const rqb200_vae_config& c = h->cfg;
    int r = c.resolution >> (c.n_levels - 1);
    return a.take<float>((size_t)B * r * r * c.embed_dim);
}

}  // namespace rqb

extern "C" {

rqb200_vae* rqb200_vae_create(const rqb200_vae_config* cfg) {
    if (!cfg || cfg->n_levels < 1 || cfg->n_levels > 8 || cfg->n_attn_res > 8) { rqb::set_error("vae_create: bad config"); return nullptr; }
    rqb200_vae* h = new rqb200_vae();
    h->cfg = *cfg;
    return h;
}
void rqb200_vae_destroy(rqb200_vae* h) { delete h; }

int rqb200_vae_set_tensor(rqb200_vae* h, const char* key, const void* ptr, int dtype, int64_t numel) {
    if (!h || !key || !ptr) return rqb::fail(RQB200_EINVAL, "vae_set_tensor: null argument");
    h->t[key] = VTensor{ptr, dtype, numel};
    h->finalized = false;
    return 0;
}

int rqb200_vae_finalize(rqb200_vae* h) {
    if (!h) return rqb::fail(RQB200_EINVAL, "vae_finalize: null handle");
    rqb::VaeRun run{h, nullptr, 1, true, {nullptr, nullptr, nullptr, nullptr}, nullptr, ""};
    h->max_act = 0;
    h->max_gn_hw = 0;
    {
        const rqb200_vae_config& c = h->cfg;
        int r = c.resolution >> (c.n_levels - 1);
        bool ok = (c.mode & 0xff) == RQB200_MODE_FAST && c.ch % 128 == 0 && c.z_channels % 128 == 0 && c.embed_dim % 128 == 0 &&
                  c.out_ch == 3 && r > 0 && (r & (r - 1)) == 0;
        h->fast_ok = ok;
        h->gn_fuse = !(c.mode & RQB200_VAE_NO_GN_FUSE);
        h->split = ok && h->t.find("decoder.conv_in.weight_lo") != h->t.end();
    }
    {
        auto it = h->t.find("encoder.conv_out.weight");
        h->enc_fast = h->fast_ok && it != h->t.end() && it->second.dtype == RQB200_F16;
    }
    run.fast = h->fast_ok;
    run.decode(nullptr, nullptr);
    run.fast = h->fast_ok && h->enc_fast;
    run.encode(nullptr, nullptr);
    if (!run.missing.empty()) return rqb::fail(RQB200_ESTATE, "vae_finalize: tensor " + run.missing);
    {
        const rqb200_vae_config& c = h->cfg;
        const bool shared = h->t.count("codebook") != 0, per_depth = h->t.count("codebook.0") != 0;
        if (!shared && !per_depth) return rqb::fail(RQB200_ESTATE, "vae_finalize: tensor codebook (missing)");
        if (shared && per_depth) return rqb::fail(RQB200_EINVAL, "vae_finalize: both codebook and codebook.<d> registered");
        if (per_depth && (c.depth < 1 || c.depth > rqb::RQ_MAX_TABLES))
            return rqb::fail(RQB200_EINVAL, "vae_finalize: per-depth codebooks need depth 1..16");
        const float* ptrs[rqb::RQ_MAX_TABLES];
        int32_t ks[rqb::RQ_MAX_TABLES];
        const int n = shared ? 1 : c.depth;
        for (int d = 0; d < n; d++) {
            auto it = h->t.find(shared ? std::string("codebook") : "codebook." + std::to_string(d));
            if (it == h->t.end()) return rqb::fail(RQB200_ESTATE, "vae_finalize: tensor codebook." + std::to_string(d) + " (missing)");
            ptrs[d] = (const float*)it->second.ptr;
            ks[d] = shared ? c.codebook_size : (int32_t)(it->second.numel / c.embed_dim);
            if (!shared && (int64_t)ks[d] * c.embed_dim != it->second.numel)
                return rqb::fail(RQB200_EINVAL, "vae_finalize: codebook." + std::to_string(d) + " is not [K, embed_dim]");
        }
        RQB_TRY(rqb::make_rq_tables(&h->codebooks, ptrs, ks, n));
    }
    h->finalized = true;
    return 0;
}

size_t rqb200_vae_workspace_bytes(const rqb200_vae* h, int B) {
    if (!h || !h->finalized || B <= 0) return 0;
    return rqb::vae_layout(h, B, nullptr, 0, nullptr);
}

static int vae_prepare(rqb200_vae* h, int B, void* ws, size_t ws_bytes, void* stream, rqb::VaeRun* run) {
    if (!h || !ws) return rqb::fail(RQB200_EINVAL, "vae: null argument");
    if (!h->finalized) return rqb::fail(RQB200_ESTATE, "vae: engine not finalised");
    if (B <= 0) return rqb::fail(RQB200_EINVAL, "vae: B must be > 0");
    if (rqb200_device_count() <= 0) return rqb::fail(RQB200_ENODEV, "vae: no CUDA device");
    *run = rqb::VaeRun{h, (cudaStream_t)stream, B, false, {nullptr, nullptr, nullptr, nullptr}, nullptr, ""};
    run->fast = h->fast_ok;
    size_t need = rqb::vae_layout(h, B, ws, ws_bytes, run);
    if (need > ws_bytes) return rqb::fail(RQB200_EWORKSPACE, "vae: workspace too small");
    rqb::g_launches = 0;
    return 0;
}

int rqb200_vae_decode(rqb200_vae* h, const float* z_q, int B, float* out, void* workspace, size_t workspace_bytes,
                      void* stream) {
    rqb::VaeRun run;
    RQB_TRY(vae_prepare(h, B, workspace, workspace_bytes, stream, &run));
    int rc = run.decode(z_q, out);
    h->last_launches = rqb::g_launches;
    return rc;
}

int rqb200_vae_decode_code(rqb200_vae* h, const int64_t* codes, int B, float* out, void* workspace,
                           size_t workspace_bytes, void* stream) {
    rqb::VaeRun run;
    RQB_TRY(vae_prepare(h, B, workspace, workspace_bytes, stream, &run));
    const rqb200_vae_config& c = h->cfg;
    int r = c.resolution >> (c.n_levels - 1);
    float* zq = rqb::vae_zq_buffer(h, B, workspace, workspace_bytes);
    RQB_TRY(rqb::launch_rq_embed(codes, h->codebooks, (int64_t)B * r * r, c.depth, c.embed_dim, zq, true, (cudaStream_t)stream));
    int rc = run.decode(zq, out);
    h->last_launches = rqb::g_launches;
    return rc;
}

int rqb200_vae_encode(rqb200_vae* h, const float* x, int B, float* z_e, void* workspace, size_t workspace_bytes,
                      void* stream) {
    rqb::VaeRun run;
    RQB_TRY(vae_prepare(h, B, workspace, workspace_bytes, stream, &run));
    run.fast = h->fast_ok && h->enc_fast;   // default: exact-tier kernels for the whole encoder; see encode_fast
    int rc = run.encode(x, z_e);
    h->last_launches = rqb::g_launches;
    return rc;
}
int64_t rqb200_vae_last_launches(const rqb200_vae* h) { return h ? h->last_launches : 0; }
}
