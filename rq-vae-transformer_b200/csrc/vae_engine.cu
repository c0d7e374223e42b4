// P2 host orchestration -- RQVAE.encode / decode / decode_code as a static layer plan over the kernels in
// conv_kernels.cu (exact tier) / conv_tc.cu (fast tier).
//
// Mirrors rqvae/models/rqvae/rqvae.py:80-109 and modules.py (Encoder.forward :73-98, Decoder.forward :171-202);
// layer names are the reference's state_dict keys (SURVEY.md A.3/A.4) so a checkpoint loads unchanged.
// Differences in execution, not arithmetic: activations stay NHWC end to end (the reference permutes NHWC<->NCHW at
// rqvae.py:82,86), the nearest-x2 upsample and the (0,1,0,1) pad are folded into conv indexing, q/k/v 1x1 convs run as
// one Cout=3C GEMM, and the whole batch is decoded in one pass (the reference's callers decode image by image).
#include <vector>

#include "kernels.h"

struct rqb200_vae {
    rqb200_vae_config cfg;
    rqb::TensorTable t;
    bool finalized = false;
    bool fast_ok = false;     // FAST mode and every decoder channel count is a multiple of 128
    bool enc_fast = false;    // the encoder's convs were registered in fp16 as well: encode on the wgmma path
    bool gn_fuse = true;      // conv epilogues emit the next GroupNorm's partial statistics (mode bit RQB200_VAE_NO_GN_FUSE clears it)
    int64_t last_launches = 0;
    // the activation sizes of the last pixel extent a workspace was laid out for (vae_layout's dry walk, cached)
    mutable int ext_h = 0, ext_w = 0;
    mutable int64_t ext_act = 0, ext_gn_hw = 0;
    rqb::RqTables codebooks{};   // decode_code's embedding tables, resolved by finalize from "codebook" or "codebook.<d>"
};

namespace rqb {

// What a conv reads: an fp32 activation for the exact-tier kernel, which folds the nearest x2 upsample and an NCHW layout into
// its indexing, or, for the wgmma kernel, the fp16 hi/lo copy in h16[slot] / l16[slot], already upsampled by the cast.
struct Operand {
    const float* x;
    int slot;                 // -1: the fp32 activation x
    int upsample;
    int nchw;
};

// One walk per network serves both tiers: the tier lives in operand / norm / conv, each of which branches on `fast`.  The
// exact tier runs every conv and GroupNorm on the fp32 FFMA kernels; the fast tier (fast_ok: every channel count a multiple of
// 128) runs them on the wgmma implicit GEMM with split-fp16 operands: each wgmma conv needs "<key>.weight_lo" beside its weight.
struct VaeRun {
    rqb200_vae* h;
    cudaStream_t st;
    int B;
    bool dry;                 // dry run: only check tensors / measure buffer sizes
    float* buf[4];
    double* gn_ws;
    std::string missing;
    __half* h16[2] = {nullptr, nullptr};      // fp16 conv operands (GN output / cast / upsampled cast)
    __half* l16[2] = {nullptr, nullptr};      // their fp16 'lo' halves (split-fp16 products)
    float* zq = nullptr;                      // decode_code's staging buffer for the embedded codes
    bool fast = false;                        // the walk's tier, set by decode / encode

    // fast tier: a conv whose output feeds a GroupNorm emits that GroupNorm's partial statistics from its epilogue
    const float* stats_buf = nullptr;         // conv output whose statistics sit in gn_ws
    int stats_chunks = 0;
    // what a dry walk measures for the workspace
    int64_t max_act = 0;                      // max H*W*C per image over all activations
    int64_t max_gn_hw = 0;

    const PlanTensor* get(const std::string& k, int64_t numel) {
        const PlanTensor* p = h->t.find(k);
        if (!p || p->numel != numel) {
            if (missing.empty()) missing = k + (!p ? " (missing)" : " (wrong size)");
            return nullptr;
        }
        return p;
    }
    void note_act(int64_t hw, int64_t c) { if (hw * c > max_act) max_act = hw * c; }

    // x as a conv operand: itself on the exact tier; on the fast tier its fp16 copy, cast into slot (x2 nearest upsampled if asked)
    int operand(const float* x, int H, int W, int C, int slot, int upsample, Operand* o) {
        *o = fast ? Operand{nullptr, slot, upsample, 0} : Operand{x, -1, upsample, 0};
        if (!fast || dry) return 0;
        return launch_cast_f16(x, h16[slot], l16[slot], B, H, W, C, upsample, st);
    }
    // GroupNorm (+ SiLU) of in: into out on the exact tier, into slot 0 on the fast tier (from fused statistics where the
    // producing conv emitted them)
    int norm(const std::string& name, const float* in, float* out, int HW, int C, int silu, Operand* o) {
        const PlanTensor* g = get(name + ".weight", C);
        const PlanTensor* b = get(name + ".bias", C);
        if (HW > max_gn_hw) max_gn_hw = HW;
        note_act(HW, C);
        *o = fast ? Operand{nullptr, 0, 0, 0} : Operand{out, -1, 0, 0};
        if (dry || !g || !b) return 0;
        if (!fast) return launch_groupnorm_silu(in, (const float*)g->ptr, (const float*)b->ptr, out, gn_ws, B, HW, C, silu, st);
        const int fused = (in == stats_buf) ? stats_chunks : 0;
        stats_buf = nullptr;
        return launch_groupnorm_f16(in, (const float*)g->ptr, (const float*)b->ptr, h16[0], l16[0], gn_ws, B, HW, C, silu, st, fused);
    }
    // H, W: the operand's extent before its upsample; a stride-2 conv is the Downsample's (0,1,0,1) pad + 3x3 conv
    // (layers.py:50-57), which the wgmma kernel runs through a tensor map that samples every other pixel.  feeds_gn: the output
    // goes to a GroupNorm next, so the wgmma epilogue emits its partial statistics.
    int conv(const std::string& name, const Operand& in, float* out, const float* resid, int H, int W, int Cin, int Cout, int ks,
             int stride, bool feeds_gn, int out_nchw) {
        const ConvGeom g = vae_conv_geom(B, H, W, Cin, Cout, ks, stride, in.upsample, in.nchw, out_nchw);
        const int Ho = g.Ho, Wo = g.Wo;
        const int64_t wn = (int64_t)Cout * ks * ks * Cin;
        const PlanTensor* w = get(name + ".weight", wn);
        const PlanTensor* b = get(name + ".bias", Cout);
        const PlanTensor* wl = in.slot < 0 ? nullptr : get(name + ".weight_lo", wn);
        note_act((int64_t)Ho * Wo, Cout);
        if (dry || !w || !b) return 0;
        if (in.slot < 0) return launch_conv(in.x, w->ptr, w->dtype, (const float*)b->ptr, resid, out, g, st);
        if (!wl) return 0;
        if (w->dtype != RQB200_F16 || wl->dtype != RQB200_F16)
            return fail(RQB200_ESTATE, "vae fast tier: conv weights and their lo halves must be fp16: " + name);
        const bool fuse = feeds_gn && h->gn_fuse && !out_nchw && conv_tc_gn_fusable(Ho, Wo, Cout, ks, stride);
        stats_buf = fuse ? out : nullptr;
        stats_chunks = fuse ? Ho * Wo / 32 : 0;
        return launch_conv_tc(h16[in.slot], w->ptr, l16[in.slot], wl->ptr, (const float*)b->ptr, resid, out, B, Ho, Wo, Cin, Cout, ks, out_nchw, st,
                              stride, fuse ? gn_ws : nullptr);
    }

    // buffers: cur = index of the live activation, advanced past the block
    int resblock(const std::string& p, int& cur, int H, int W, int Cin, int Cout) {
        const int a = (cur + 1) & 3, b = (cur + 2) & 3, c = (cur + 3) & 3;
        Operand x;
        RQB_TRY(norm(p + ".norm1", buf[cur], buf[a], H * W, Cin, 1, &x));
        RQB_TRY(conv(p + ".conv1", x, buf[b], nullptr, H, W, Cin, Cout, 3, 1, true, 0));
        RQB_TRY(norm(p + ".norm2", buf[b], buf[a], H * W, Cout, 1, &x));
        const float* res = buf[cur];
        if (Cin != Cout) {
            Operand s;
            RQB_TRY(operand(buf[cur], H, W, Cin, 1, 0, &s));
            RQB_TRY(conv(p + ".nin_shortcut", s, buf[c], nullptr, H, W, Cin, Cout, 1, 1, false, 0));
            res = buf[c];
        }
        RQB_TRY(conv(p + ".conv2", x, buf[b], res, H, W, Cout, Cout, 3, 1, true, 0));
        cur = b;
        return 0;
    }
    int attnblock(const std::string& p, int& cur, int H, int W, int C) {
        const int a = (cur + 1) & 3, b = (cur + 2) & 3, c = (cur + 3) & 3;
        Operand x;
        RQB_TRY(norm(p + ".norm", buf[cur], buf[a], H * W, C, 0, &x));
        // fused q|k|v 1x1 conv: key "<p>.qkv" registered by the host binding ([3C,1,1,C] / [3C])
        RQB_TRY(conv(p + ".qkv", x, buf[b], nullptr, H, W, C, 3 * C, 1, 1, false, 0));
        // the fast tier runs maps past 1024 tokens on the tensor-core kernel; up to 1024 (every shipped VAE at its configured
        // resolution) both tiers keep the fp32 kernel
        if (!dry && missing.empty())
            RQB_TRY(fast && H * W > 1024 ? launch_vae_attn_tc(buf[b], buf[a], B, H * W, C, st) : launch_vae_attn(buf[b], buf[a], B, H * W, C, st));
        RQB_TRY(operand(buf[a], H, W, C, 0, 0, &x));
        RQB_TRY(conv(p + ".proj_out", x, buf[c], buf[cur], H, W, C, C, 1, 1, true, 0));
        cur = c;
        return 0;
    }
    // which levels carry an AttnBlock follows the CONFIGURED resolution ladder (the reference's Encoder / Decoder decide it at
    // construction from ddconfig["resolution"], modules.py:29-50,117-160), whatever extent the call walks
    bool has_attn(int cres) const {
        for (int i = 0; i < h->cfg.n_attn_res; i++) if (h->cfg.attn_resolutions[i] == cres) return true;
        return false;
    }

    // Decoder.forward (modules.py:171-202) preceded by post_quant_conv (rqvae.py:87).  z NHWC [B,H,W,embed_dim], H x W the latent
    // extent; out NCHW [B,out_ch,H f,W f].  cres: the level's resolution in the configured ladder.
    int decode(const float* z, float* out, int H, int W) {
        fast = h->fast_ok;
        const rqb200_vae_config& c = h->cfg;
        const int nl = c.n_levels, nb = c.num_res_blocks;
        int cres = c.resolution >> (nl - 1), ch = c.ch * c.ch_mult[nl - 1], cur = 0;
        Operand x;
        RQB_TRY(operand(z, H, W, c.embed_dim, 0, 0, &x));
        RQB_TRY(conv("post_quant_conv", x, buf[1], nullptr, H, W, c.embed_dim, c.z_channels, 1, 1, false, 0));
        RQB_TRY(operand(buf[1], H, W, c.z_channels, 0, 0, &x));
        RQB_TRY(conv("decoder.conv_in", x, buf[0], nullptr, H, W, c.z_channels, ch, 3, 1, true, 0));
        RQB_TRY(resblock("decoder.mid.block_1", cur, H, W, ch, ch));
        RQB_TRY(attnblock("decoder.mid.attn_1", cur, H, W, ch));
        RQB_TRY(resblock("decoder.mid.block_2", cur, H, W, ch, ch));
        for (int lvl = nl - 1; lvl >= 0; lvl--) {
            const int cout = c.ch * c.ch_mult[lvl];
            const std::string p = "decoder.up." + std::to_string(lvl);
            for (int b = 0; b <= nb; b++) {
                RQB_TRY(resblock(p + ".block." + std::to_string(b), cur, H, W, ch, cout));
                ch = cout;
                if (has_attn(cres)) RQB_TRY(attnblock(p + ".attn." + std::to_string(b), cur, H, W, ch));
            }
            if (lvl != 0) {
                const int nxt = (cur + 1) & 3;
                RQB_TRY(operand(buf[cur], H, W, ch, 1, 1, &x));
                RQB_TRY(conv(p + ".upsample.conv", x, buf[nxt], nullptr, H, W, ch, ch, 3, 1, true, 0));
                cur = nxt;
                cres *= 2;
                H *= 2;
                W *= 2;
            }
        }
        RQB_TRY(norm("decoder.norm_out", buf[cur], buf[(cur + 1) & 3], H * W, ch, 1, &x));
        return conv("decoder.conv_out", x, out, nullptr, H, W, ch, c.out_ch, 3, 1, false, 1);
    }

    // Encoder.forward (modules.py:73-98) followed by quant_conv (rqvae.py:82).  x NCHW [B,in_channels,H,W] -> z_e NHWC
    // [B,H/f,W/f,embed_dim].  The fast tier needs the encoder's convs registered in fp16 (enc_fast); conv_in (Cin = 3, NCHW fp32
    // input, 0.3 % of the encoder's flops) runs the fp32 FFMA kernel on both tiers.
    int encode(const float* x, float* z_e, int H, int W) {
        fast = h->fast_ok && h->enc_fast;
        const rqb200_vae_config& c = h->cfg;
        const int nl = c.n_levels, nb = c.num_res_blocks;
        int cres = c.resolution, ch = c.ch, cur = 0;
        RQB_TRY(conv("encoder.conv_in", Operand{x, -1, 0, 1}, buf[0], nullptr, H, W, c.in_channels, ch, 3, 1, false, 0));
        Operand o;
        for (int lvl = 0; lvl < nl; lvl++) {
            const int cout = c.ch * c.ch_mult[lvl];
            const std::string p = "encoder.down." + std::to_string(lvl);
            for (int b = 0; b < nb; b++) {
                RQB_TRY(resblock(p + ".block." + std::to_string(b), cur, H, W, ch, cout));
                ch = cout;
                if (has_attn(cres)) RQB_TRY(attnblock(p + ".attn." + std::to_string(b), cur, H, W, ch));
            }
            if (lvl != nl - 1) {
                const int nxt = (cur + 1) & 3;
                RQB_TRY(operand(buf[cur], H, W, ch, 1, 0, &o));
                RQB_TRY(conv(p + ".downsample.conv", o, buf[nxt], nullptr, H, W, ch, ch, 3, 2, true, 0));
                cur = nxt;
                cres /= 2;
                H /= 2;
                W /= 2;
            }
        }
        RQB_TRY(resblock("encoder.mid.block_1", cur, H, W, ch, ch));
        RQB_TRY(attnblock("encoder.mid.attn_1", cur, H, W, ch));
        RQB_TRY(resblock("encoder.mid.block_2", cur, H, W, ch, ch));
        float* zc = buf[(cur + 2) & 3];
        RQB_TRY(norm("encoder.norm_out", buf[cur], buf[(cur + 1) & 3], H * W, ch, 1, &o));
        RQB_TRY(conv("encoder.conv_out", o, zc, nullptr, H, W, ch, c.z_channels, 3, 1, false, 0));
        RQB_TRY(operand(zc, H, W, c.z_channels, 0, 0, &o));
        return conv("quant_conv", o, z_e, nullptr, H, W, c.z_channels, c.embed_dim, 1, 1, false, 0);
    }
};

// the downsampling factor f = 2^(n_levels - 1): an image's H and W must be positive multiples of it
static int vae_factor(const rqb200_vae* h) { return 1 << (h->cfg.n_levels - 1); }
static bool vae_extent_ok(const rqb200_vae* h, int H, int W) {
    const int f = vae_factor(h);
    return H > 0 && W > 0 && H % f == 0 && W % f == 0;
}

// the workspace of a call on B images of H x W pixels: the activation sizes come from a dry walk of both networks at that extent;
// decode_code's zq staging stays at the configured latent grid
static size_t vae_layout(const rqb200_vae* h, int B, int H, int W, void* base, size_t cap, VaeRun* run) {
    if (H != h->ext_h || W != h->ext_w) {
        VaeRun d{const_cast<rqb200_vae*>(h), nullptr, 1, true, {nullptr, nullptr, nullptr, nullptr}, nullptr, ""};
        const int f = vae_factor(h);
        d.decode(nullptr, nullptr, H / f, W / f);
        d.encode(nullptr, nullptr, H, W);
        h->ext_h = H;
        h->ext_w = W;
        h->ext_act = d.max_act;
        h->ext_gn_hw = d.max_gn_hw;
    }
    const int64_t max_act = h->ext_act;
    Arena a(base, cap);
    for (int i = 0; i < 4; i++) {
        float* p = a.take<float>((size_t)B * max_act);
        if (run) run->buf[i] = p;
    }
    double* g = a.take<double>(groupnorm_ws_doubles(B, (int)h->ext_gn_hw));
    if (run) run->gn_ws = g;
    const rqb200_vae_config& c = h->cfg;
    int r = c.resolution >> (c.n_levels - 1);
    float* zq = a.take<float>((size_t)B * r * r * c.embed_dim);
    if (run) run->zq = zq;
    for (int i = 0; i < 2; i++) {
        __half* p16 = a.take<__half>((size_t)B * max_act);
        if (run) run->h16[i] = p16;
    }
    if (h->fast_ok)
        for (int i = 0; i < 2; i++) {
            __half* p16 = a.take<__half>((size_t)B * max_act);
            if (run) run->l16[i] = p16;
        }
    return a.off + 256;
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
    h->t.set(key, ptr, dtype, numel);
    h->finalized = false;
    return 0;
}

int rqb200_vae_finalize(rqb200_vae* h) {
    if (!h) return rqb::fail(RQB200_EINVAL, "vae_finalize: null handle");
    rqb::VaeRun run{h, nullptr, 1, true, {nullptr, nullptr, nullptr, nullptr}, nullptr, ""};
    h->ext_h = h->ext_w = 0;
    {
        const rqb200_vae_config& c = h->cfg;
        if (c.resolution < 1 || c.resolution % rqb::vae_factor(h))
            return rqb::fail(RQB200_EINVAL, "vae_finalize: resolution must be a positive multiple of 2^(n_levels - 1)");
        bool ok = (c.mode & 0xff) == RQB200_MODE_FAST && c.ch % 128 == 0 && c.z_channels % 128 == 0 && c.embed_dim % 128 == 0 &&
                  c.out_ch == 3;
        h->fast_ok = ok;
        h->gn_fuse = !(c.mode & RQB200_VAE_NO_GN_FUSE);
    }
    {
        const rqb::PlanTensor* w = h->t.find("encoder.conv_out.weight");
        h->enc_fast = h->fast_ok && w && w->dtype == RQB200_F16;
    }
    const int R = h->cfg.resolution, f = rqb::vae_factor(h);
    run.decode(nullptr, nullptr, R / f, R / f);
    run.encode(nullptr, nullptr, R, R);
    if (!run.missing.empty()) return rqb::fail(RQB200_ESTATE, "vae_finalize: tensor " + run.missing);
    {
        const rqb200_vae_config& c = h->cfg;
        const bool shared = h->t.find("codebook") != nullptr, per_depth = h->t.find("codebook.0") != nullptr;
        if (!shared && !per_depth) return rqb::fail(RQB200_ESTATE, "vae_finalize: tensor codebook (missing)");
        if (shared && per_depth) return rqb::fail(RQB200_EINVAL, "vae_finalize: both codebook and codebook.<d> registered");
        if (per_depth && (c.depth < 1 || c.depth > rqb::RQ_MAX_TABLES))
            return rqb::fail(RQB200_EINVAL, "vae_finalize: per-depth codebooks need depth 1..16");
        const float* ptrs[rqb::RQ_MAX_TABLES];
        int32_t ks[rqb::RQ_MAX_TABLES];
        const int n = shared ? 1 : c.depth;
        for (int d = 0; d < n; d++) {
            const rqb::PlanTensor* cb = h->t.find(shared ? std::string("codebook") : "codebook." + std::to_string(d));
            if (!cb) return rqb::fail(RQB200_ESTATE, "vae_finalize: tensor codebook." + std::to_string(d) + " (missing)");
            ptrs[d] = (const float*)cb->ptr;
            ks[d] = shared ? c.codebook_size : (int32_t)(cb->numel / c.embed_dim);
            if (!shared && (int64_t)ks[d] * c.embed_dim != cb->numel)
                return rqb::fail(RQB200_EINVAL, "vae_finalize: codebook." + std::to_string(d) + " is not [K, embed_dim]");
        }
        RQB_TRY(rqb::make_rq_tables(&h->codebooks, ptrs, ks, n));
    }
    h->finalized = true;
    return 0;
}

size_t rqb200_vae_workspace_bytes(const rqb200_vae* h, int B) {
    if (!h || !h->finalized || B <= 0) return 0;
    return rqb::vae_layout(h, B, h->cfg.resolution, h->cfg.resolution, nullptr, 0, nullptr);
}

size_t rqb200_vae_workspace_bytes_hw(const rqb200_vae* h, int B, int H, int W) {
    if (!h || !h->finalized || B <= 0 || !rqb::vae_extent_ok(h, H, W)) return 0;
    return rqb::vae_layout(h, B, H, W, nullptr, 0, nullptr);
}

// H, W: the call's pixel extent
static int vae_prepare(rqb200_vae* h, int B, int H, int W, void* ws, size_t ws_bytes, void* stream, rqb::VaeRun* run) {
    if (!h || !ws) return rqb::fail(RQB200_EINVAL, "vae: null argument");
    if (!h->finalized) return rqb::fail(RQB200_ESTATE, "vae: engine not finalised");
    if (B <= 0) return rqb::fail(RQB200_EINVAL, "vae: B must be > 0");
    if (!rqb::vae_extent_ok(h, H, W))
        return rqb::fail(RQB200_EINVAL, "vae: H and W must be positive multiples of 2^(n_levels - 1) = " + std::to_string(rqb::vae_factor(h)));
    if (rqb200_device_count() <= 0) return rqb::fail(RQB200_ENODEV, "vae: no CUDA device");
    *run = rqb::VaeRun{h, (cudaStream_t)stream, B, false, {nullptr, nullptr, nullptr, nullptr}, nullptr, ""};
    size_t need = rqb::vae_layout(h, B, H, W, ws, ws_bytes, run);
    if (need > ws_bytes) return rqb::fail(RQB200_EWORKSPACE, "vae: workspace too small");
    rqb::g_launches = 0;
    return 0;
}

int rqb200_vae_decode_hw(rqb200_vae* h, const float* z_q, int B, int hl, int wl, float* out, void* workspace, size_t workspace_bytes,
                         void* stream) {
    if (!h) return rqb::fail(RQB200_EINVAL, "vae: null argument");
    if (hl <= 0 || wl <= 0) return rqb::fail(RQB200_EINVAL, "vae_decode: the latent extent must be positive");
    const int f = rqb::vae_factor(h);
    if ((int64_t)hl * f > (1 << 20) || (int64_t)wl * f > (1 << 20)) return rqb::fail(RQB200_EINVAL, "vae_decode: latent extent too large");
    rqb::VaeRun run;
    RQB_TRY(vae_prepare(h, B, hl * f, wl * f, workspace, workspace_bytes, stream, &run));
    int rc = run.decode(z_q, out, hl, wl);
    h->last_launches = rqb::g_launches;
    return rc;
}

int rqb200_vae_decode(rqb200_vae* h, const float* z_q, int B, float* out, void* workspace, size_t workspace_bytes,
                      void* stream) {
    if (!h) return rqb::fail(RQB200_EINVAL, "vae: null argument");
    const int r = h->cfg.resolution / rqb::vae_factor(h);
    return rqb200_vae_decode_hw(h, z_q, B, r, r, out, workspace, workspace_bytes, stream);
}

int rqb200_vae_decode_code(rqb200_vae* h, const int64_t* codes, int B, float* out, void* workspace,
                           size_t workspace_bytes, void* stream) {
    if (!h) return rqb::fail(RQB200_EINVAL, "vae: null argument");
    rqb::VaeRun run;
    const rqb200_vae_config& c = h->cfg;
    RQB_TRY(vae_prepare(h, B, c.resolution, c.resolution, workspace, workspace_bytes, stream, &run));
    int r = c.resolution >> (c.n_levels - 1);
    RQB_TRY(rqb::launch_rq_embed(codes, h->codebooks, (int64_t)B * r * r, c.depth, c.embed_dim, run.zq, true, (cudaStream_t)stream));
    int rc = run.decode(run.zq, out, r, r);
    h->last_launches = rqb::g_launches;
    return rc;
}

int rqb200_vae_encode_hw(rqb200_vae* h, const float* x, int B, int H, int W, float* z_e, void* workspace, size_t workspace_bytes,
                         void* stream) {
    rqb::VaeRun run;
    RQB_TRY(vae_prepare(h, B, H, W, workspace, workspace_bytes, stream, &run));
    int rc = run.encode(x, z_e, H, W);
    h->last_launches = rqb::g_launches;
    return rc;
}

int rqb200_vae_encode(rqb200_vae* h, const float* x, int B, float* z_e, void* workspace, size_t workspace_bytes,
                      void* stream) {
    if (!h) return rqb::fail(RQB200_EINVAL, "vae: null argument");
    return rqb200_vae_encode_hw(h, x, B, h->cfg.resolution, h->cfg.resolution, z_e, workspace, workspace_bytes, stream);
}
int64_t rqb200_vae_last_launches(const rqb200_vae* h) { return h ? h->last_launches : 0; }

// ---- diagnostic entry points (tests/test_gpu_vae_kernels.py): one launch of a kernel between the VAE's convs, or of the exact tier's
// conv, through the launcher the engine calls

int rqb200_dbg_vae_conv(const float* X, const void* Wt, int wdtype, const float* bias, const float* residual, float* out, int B, int H,
                        int W, int Cin, int Cout, int ks, int stride, int upsample, int in_nchw, int out_nchw, void* stream) {
    using namespace rqb;
    if (B < 1 || H < 1 || W < 1 || Cin < 1 || Cout < 1 || (ks != 1 && ks != 3) || (stride != 1 && stride != 2) || (upsample && stride != 1))
        return fail(RQB200_EINVAL, "dbg_vae_conv: need B, H, W, Cin, Cout >= 1, ks 1 | 3, stride 1 | 2, no upsample with stride 2");
    if (!X || !Wt || !out || (residual && out_nchw)) return fail(RQB200_EINVAL, "dbg_vae_conv: null argument, or a residual with NCHW output");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "dbg_vae_conv: no CUDA device");
    const ConvGeom g = vae_conv_geom(B, H, W, Cin, Cout, ks, stride, upsample != 0, in_nchw != 0, out_nchw != 0);
    return launch_conv(X, Wt, wdtype, bias, residual, out, g, (cudaStream_t)stream);
}

int rqb200_dbg_groupnorm(int form, const float* X, const float* gamma, const float* beta, float* Y, void* Y16, void* Y16lo,
                         double* stats_ws, int64_t ws_doubles, int B, int HW, int C, int silu, void* stream) {
    using namespace rqb;
    if (form < 0 || form > 2 || B < 1 || HW < 1 || C < 32 || C % 32 || (form > 0 && C % 128) || (form == 2 && HW % 32))
        return fail(RQB200_EINVAL, "dbg_groupnorm: need form 0..2, B, HW >= 1, C % 32 == 0 (forms 1, 2: C % 128 == 0; form 2: HW % 32 == 0)");
    if (!X || !gamma || !beta || !stats_ws || (form == 0 ? !Y : !Y16))
        return fail(RQB200_EINVAL, "dbg_groupnorm: null argument");
    if (ws_doubles < 0 || (size_t)ws_doubles < groupnorm_ws_doubles(B, HW))
        return fail(RQB200_EWORKSPACE, "dbg_groupnorm: statistics workspace smaller than groupnorm_ws_doubles(B, HW)");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "dbg_groupnorm: no CUDA device");
    const cudaStream_t st = (cudaStream_t)stream;
    if (form == 0) return launch_groupnorm_silu(X, gamma, beta, Y, stats_ws, B, HW, C, silu != 0, st);
    return launch_groupnorm_f16(X, gamma, beta, Y16, Y16lo, stats_ws, B, HW, C, silu != 0, st, form == 2 ? HW / 32 : 0);
}

int rqb200_dbg_cast_f16(const float* X, void* Y16, void* Y16lo, int B, int H, int W, int C, int upsample, void* stream) {
    using namespace rqb;
    if (B < 1 || H < 1 || W < 1 || C < 4) return fail(RQB200_EINVAL, "dbg_cast_f16: need B, H, W >= 1, C >= 4");
    if (!X || !Y16) return fail(RQB200_EINVAL, "dbg_cast_f16: null argument");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "dbg_cast_f16: no CUDA device");
    return launch_cast_f16(X, Y16, Y16lo, B, H, W, C, upsample != 0, (cudaStream_t)stream);
}

int rqb200_dbg_vae_attn(const float* qkv, float* out, int B, int HW, int C, void* stream) {
    using namespace rqb;
    if (B < 1 || HW < 1 || C < 1) return fail(RQB200_EINVAL, "dbg_vae_attn: need B, HW, C >= 1");
    if (!qkv || !out) return fail(RQB200_EINVAL, "dbg_vae_attn: null argument");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "dbg_vae_attn: no CUDA device");
    return launch_vae_attn(qkv, out, B, HW, C, (cudaStream_t)stream);
}

int rqb200_dbg_vae_attn_tc(const float* qkv, float* out, int B, int HW, int C, void* stream) {
    using namespace rqb;
    if (B < 1 || HW < 1 || C < 1) return fail(RQB200_EINVAL, "dbg_vae_attn_tc: need B, HW, C >= 1");
    if (!qkv || !out) return fail(RQB200_EINVAL, "dbg_vae_attn_tc: null argument");
    if (C != 128 && C != 256 && C != 384 && C != 512) return fail(RQB200_EINVAL, "dbg_vae_attn_tc: C must be 128, 256, 384 or 512");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "dbg_vae_attn_tc: no CUDA device");
    return launch_vae_attn_tc(qkv, out, B, HW, C, (cudaStream_t)stream);
}
}
