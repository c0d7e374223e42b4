// P3 host orchestration -- RQTransformer.sample as one device-side loop (no host sync, no per-token Python).
//
// Mirrors rqvae/models/rqtransformer/transformers.py: sample :294-369 (raster (h,w,d) order, start_loc resume),
// cached_forward :190-287 (body step once per spatial position, head step per depth, classifier), init_cache :289-292.
// What is deliberately different from the reference's execution (not from its arithmetic):
//   * KV caches are pre-allocated [layer][B][nh][Tmax][64] and appended in place (reference: torch.cat per step/layer);
//   * only the NEW position's code embeddings are computed each step (reference re-embeds the whole prefix twice per
//     token, transformers.py:217-220,249-255 -- row-wise identical values);
//   * the sampled code is written on the device and consumed by the next step's kernels; nothing returns to the host.
#include <algorithm>
#include <cstddef>
#include <cstring>
#include <vector>

#include "kernels.h"

struct rqb200_ar {
    rqb200_ar_config cfg;
    rqb200_ar_weights w;
    std::vector<rqb200_block_weights> body, head;
    int64_t last_launches = 0;
    rqb::ArFast* fast = nullptr;
    // rqb200_ar_step: the workspace / batch of the stepped sequence and its next token ((pos_h*W + pos_w)*D + d), -1 when none
    const void* step_ws = nullptr;
    int step_B = 0;
    int64_t step_next = -1;
};

namespace rqb {

struct ArWs {
    float *X, *XN, *QKV, *ATT, *H, *CTX, *TOK, *EMB, *LIN, *LOGITS;
    float *kc_body, *vc_body, *kc_head, *vc_head;
    int64_t* CODES;              // [B, HW, D] rqb200_ar_step's copy of the caller's codes
};

static size_t ar_layout(const rqb200_ar_config& c, int B, void* base, size_t cap, ArWs* ws) {
    Arena a(base, cap);
    const int64_t E = c.embed_dim, HW = (int64_t)c.H * c.W, Tb = c.cond_len + HW, D = c.D;
    const int64_t Mmax = (int64_t)B * Tb;                 // worst-case prefill (start_loc resume)
    float* X = a.take<float>(Mmax * E);
    float* XN = a.take<float>(Mmax * E);
    float* QKV = a.take<float>(Mmax * 3 * E);
    float* ATT = a.take<float>(Mmax * E);
    float* H = a.take<float>(Mmax * 4 * E);
    float* CTX = a.take<float>((int64_t)B * E);
    float* TOK = a.take<float>((int64_t)B * E);
    float* EMB = a.take<float>((int64_t)B * HW * D * c.code_dim);
    float* LIN = a.take<float>((int64_t)B * HW * D * E);
    float* LOGITS = a.take<float>((int64_t)B * c.vocab);
    const int64_t per_body = (int64_t)B * c.n_head * Tb * 64, per_head = (int64_t)B * c.n_head * D * 64;
    float* kcb = a.take<float>(per_body * c.n_body);
    float* vcb = a.take<float>(per_body * c.n_body);
    float* kch = a.take<float>(per_head * c.n_head_layers);
    float* vch = a.take<float>(per_head * c.n_head_layers);
    int64_t* codes = a.take<int64_t>((int64_t)B * HW * D);
    if (ws) *ws = ArWs{X, XN, QKV, ATT, H, CTX, TOK, EMB, LIN, LOGITS, kcb, vcb, kch, vch, codes};
    return a.off + 256;
}

// one transformer stack over M = B*Tn rows held in ws.X (in place).  attentions.py:134-142 per block.
static int run_stack(const rqb200_ar* h, const std::vector<rqb200_block_weights>& blocks, ArWs& ws, int B, int Tn, int T_past,
                     int Tmax, float* kc, float* vc, cudaStream_t st) {
    const rqb200_ar_config& c = h->cfg;
    const int E = c.embed_dim, M = B * Tn, wd = c.weight_dtype;
    const int64_t per = (int64_t)B * c.n_head * Tmax * 64;
    for (size_t l = 0; l < blocks.size(); l++) {
        const rqb200_block_weights& bw = blocks[l];
        RQB_TRY(launch_layernorm(ws.X, E, bw.ln1_w, bw.ln1_b, ws.XN, E, M, E, st));
        RQB_TRY(launch_linear(ws.XN, E, bw.wqkv, wd, bw.bqkv, nullptr, ws.QKV, 3 * E, M, 3 * E, E, 0, st));
        RQB_TRY(launch_attn_cached(ws.QKV, kc + per * l, vc + per * l, ws.ATT, B, Tn, T_past, Tmax, E, c.n_head, st));
        RQB_TRY(launch_linear(ws.ATT, E, bw.wproj, wd, bw.bproj, ws.X, ws.X, E, M, E, E, 0, st));
        RQB_TRY(launch_layernorm(ws.X, E, bw.ln2_w, bw.ln2_b, ws.XN, E, M, E, st));
        RQB_TRY(launch_linear(ws.XN, E, bw.w1, wd, bw.b1, nullptr, ws.H, 4 * E, M, 4 * E, E, 1, st));
        RQB_TRY(launch_linear(ws.H, 4 * E, bw.w2, wd, bw.b2, ws.X, ws.X, E, M, E, 4 * E, 0, st));
    }
    return 0;
}

// ws.LIN[(b*J + j)*D + d, :] = the body input embedding of code d at position j0 + j: input_mlp(e_d) (transformers.py:219-220), or
// the tok_emb row of the code (:222, EMB_TOK_INPUT).  cv (nullable): the positions are window positions of a canvas (kernels.h); this
// and the functions below pass it to the code gathers.
static int body_inputs(const rqb200_ar* h, const int64_t* codes, int B, int j0, int J, ArWs& ws, cudaStream_t st, const CanvasMap* cv) {
    const rqb200_ar_config& c = h->cfg;
    const rqb200_ar_weights& w = h->w;
    const int E = c.embed_dim, D = c.D, HW = c.H * c.W, C = c.code_dim, K = c.codebook_size;
    if (c.embed_variant & RQB200_EMB_TOK_INPUT)
        return launch_code_emb(codes, w.tok_emb, (c.embed_variant & RQB200_EMB_TUPLE) ? (int64_t)c.vocab * E : 0, B, HW, D, c.vocab, E,
                               j0, J, ws.LIN, st, cv);
    RQB_TRY(launch_code_emb(codes, w.codebook, c.codebook_per_depth ? (int64_t)K * C : 0, B, HW, D, K, C, j0, J, ws.EMB, st, cv));
    return launch_linear(ws.EMB, C, w.w_in, c.weight_dtype, w.b_in, nullptr, ws.LIN, E, B * J * D, E, C, 0, st);
}

// RQB200_E4M3: every weight the fast tier streams needs its fp32 row scales and a 16-byte aligned packed stream (the tiles arrive by
// bulk copies).  nullptr when they do, else the reason.
static const char* check_e4m3_weights(const rqb200_ar_config& c, const rqb200_ar_weights& w) {
    auto bad = [](const void* q, const float* s) { return q != nullptr && (s == nullptr || (reinterpret_cast<uintptr_t>(q) & 15) != 0); };
    for (int st = 0; st < 2; st++) {
        const rqb200_block_weights* bl = st == 0 ? w.body : w.head;
        const int n = st == 0 ? c.n_body : c.n_head_layers;
        for (int l = 0; l < n; l++)
            if (bad(bl[l].wqkv, bl[l].sqkv) || bad(bl[l].wproj, bl[l].sproj) || bad(bl[l].w1, bl[l].s1) || bad(bl[l].w2, bl[l].s2) ||
                !bl[l].wqkv || !bl[l].wproj || !bl[l].w1 || !bl[l].w2)
                return st == 0 ? "ar_create: E4M3 body block weights need their row scales (sqkv/sproj/s1/s2) and 16-byte aligned packed tiles"
                               : "ar_create: E4M3 head block weights need their row scales (sqkv/sproj/s1/s2) and 16-byte aligned packed tiles";
    }
    if (bad(w.w_in, w.s_in)) return "ar_create: E4M3 w_in needs s_in and 16-byte aligned packed tiles";
    if (bad(w.w_head, w.s_head)) return "ar_create: E4M3 w_head needs s_head and 16-byte aligned packed tiles";
    if (bad(w.w_cls, w.s_cls)) return "ar_create: E4M3 w_cls needs s_cls and 16-byte aligned packed tiles";
    if (bad(w.w_ccls, w.s_ccls)) return "ar_create: E4M3 w_ccls needs s_ccls and 16-byte aligned packed tiles";
    return nullptr;
}

// prefill: tokens [cond (cl) | xs_emb[0 .. idx0-1]] through the body (transformers.py:224-239); ws.CTX = the last token's output
static int prefill_prefix(const rqb200_ar* h, const int64_t* codes, const int64_t* cond, int B, int idx0, ArWs& ws, cudaStream_t st,
                          const CanvasMap* cv = nullptr) {
    const rqb200_ar_config& c = h->cfg;
    const rqb200_ar_weights& w = h->w;
    const int E = c.embed_dim, D = c.D, cl = c.cond_len, Tb = cl + c.H * c.W;
    const int Tn0 = cl + idx0;
    RQB_TRY(launch_cond_token(cond, w.cond_emb, w.pos_emb_cond, B, cl, c.vocab_cond, E, Tn0, ws.X, st));
    if (idx0 > 0) {
        RQB_TRY(body_inputs(h, codes, B, 0, idx0, ws, st, cv));
        RQB_TRY(launch_body_token(ws.LIN, w.pos_emb_hw, B, D, E, 0, idx0, cl, Tn0, ws.X, st));
    }
    RQB_TRY(run_stack(h, h->body, ws, B, Tn0, 0, Tb, ws.kc_body, ws.vc_body, st));
    return launch_row_add(ws.X, (int64_t)Tn0 * E, (int64_t)(Tn0 - 1) * E, nullptr, B, E, ws.CTX, st);   // latents[:, -1]
}

// decode step of the body on the token of position idx-1 (transformers.py:240-242); ws.CTX = its output
static int body_step(const rqb200_ar* h, const int64_t* codes, int B, int idx, ArWs& ws, cudaStream_t st, const CanvasMap* cv = nullptr) {
    const rqb200_ar_config& c = h->cfg;
    const int E = c.embed_dim, cl = c.cond_len, Tb = cl + c.H * c.W;
    RQB_TRY(body_inputs(h, codes, B, idx - 1, 1, ws, st, cv));
    RQB_TRY(launch_body_token(ws.LIN, h->w.pos_emb_hw, B, c.D, E, idx - 1, 1, 0, 1, ws.X, st));
    RQB_TRY(run_stack(h, h->body, ws, B, 1, cl + idx - 1, Tb, ws.kc_body, ws.vc_body, st));
    RQB_CUDA(cudaMemcpyAsync(ws.CTX, ws.X, (size_t)B * E * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return 0;
}

// head depth d of position idx: its token, the head stack (cache rows [0, d) from the earlier depths) and the classifier -> lg [B,V]
static int head_depth(const rqb200_ar* h, const int64_t* codes, int B, int idx, int d, ArWs& ws, float* lg, cudaStream_t st,
                      const CanvasMap* cv = nullptr) {
    const rqb200_ar_config& c = h->cfg;
    const rqb200_ar_weights& w = h->w;
    const int E = c.embed_dim, D = c.D, HW = c.H * c.W, C = c.code_dim, V = c.vocab, K = c.codebook_size, wd = c.weight_dtype;
    const int64_t cbs = c.codebook_per_depth ? (int64_t)K * C : 0;     // floats between depth d's codebook and depth d+1's
    const int ev = c.embed_variant;
    const int64_t tes = (ev & RQB200_EMB_TUPLE) ? (int64_t)V * E : 0;  // floats between depth d's token table and depth d+1's
    const size_t wsz = wd == RQB200_F32 ? 4 : 2;
    if (d == 0) {
        RQB_TRY(launch_row_add(ws.CTX, E, 0, w.pos_emb_d, B, E, ws.X, st));                         // ctx + pos_emb_d[0]
    } else if (ev & RQB200_EMB_TOK_HEAD) {
        RQB_TRY(launch_head_cumsum(codes, w.tok_emb, tes, B, HW, D, V, E, idx, d, ws.TOK, st, true, cv));  // tok_emb(code_{d-1})
        RQB_TRY(launch_row_add(ws.TOK, E, 0, w.pos_emb_d + (int64_t)d * E, B, E, ws.X, st));
    } else {
        // head_mlp(cumsum_{i<d} e_i), or head_mlp(e_{d-1}) without cumsum_depth_ctx
        RQB_TRY(launch_head_cumsum(codes, w.codebook, cbs, B, HW, D, K, C, idx, d, ws.EMB, st, (ev & RQB200_EMB_NO_CUMSUM) != 0, cv));
        RQB_TRY(launch_linear(ws.EMB, C, w.w_head, wd, w.b_head, nullptr, ws.TOK, E, B, E, C, 0, st));
        RQB_TRY(launch_row_add(ws.TOK, E, 0, w.pos_emb_d + (int64_t)d * E, B, E, ws.X, st));
    }
    RQB_TRY(run_stack(h, h->head, ws, B, 1, d, D, ws.kc_head, ws.vc_head, st));                   // head cache restarts at d==0
    RQB_TRY(launch_layernorm(ws.X, E, w.cls_ln_w, w.cls_ln_b, ws.XN, E, B, E, st));
    // one shared classifier, or depth d's [V,E] slice of the per-depth stack (BatchLinear, transformers.py:278-283)
    const int64_t cd = (ev & RQB200_EMB_CLS_PER_DEPTH) ? d : 0;
    return launch_linear(ws.XN, E, (const char*)w.w_cls + cd * V * E * wsz, wd, w.b_cls + cd * V, nullptr, lg, V, B, V, E, 0, st);
}

// positions [idx0, idx_end) of the raster; resume != 0: no prefill, continue on the caches / context left in this workspace.
// cfg_n > 0: classifier-free guidance over B = 2 cfg_n rows [cond | uncond] with scale cfg_s (the sampler forms the guided logits).
// keep / sampled: the masked-sample plan of the fast tier (kernels.h), with one body step per appended code token.
// Ht x Wt: the canvas (H x W: the grid).  Positions are canvas positions; a canvas is walked in segments as on the fast tier
// (ar_fast_sample): a new window origin restarts the body with a prefill of the window's prefix.
// B >= 1 and a span within the raster: rqb200_ar_sample_span checks them, ar_log_prob_impl forms them.
static int ar_sample_impl(rqb200_ar* h, const int64_t* partial, const int64_t* cond, int B, int idx0, int idx_end, int resume,
                          float temperature, const int32_t* top_k, const float* top_p, const float* noise,
                          int64_t noise_stride, float* logits_out, const int64_t* force, int64_t* out, void* wsp,
                          size_t ws_bytes, cudaStream_t st, int cfg_n, float cfg_s, const uint8_t* keep, const uint8_t* sampled,
                          int Ht, int Wt) {
    const rqb200_ar_config& c = h->cfg;
    const int D = c.D, V = c.vocab;
    const int64_t row = (int64_t)Ht * Wt * D;         // codes per batch row
    CanvasMap cm{c.W, Wt, 0, Ht * Wt};
    const CanvasMap* cv = (Ht != c.H || Wt != c.W) ? &cm : nullptr;
    ArWs ws;
    size_t need = ar_layout(c, B, wsp, ws_bytes, &ws);
    if (need > ws_bytes) return fail(RQB200_EWORKSPACE, "ar_sample: workspace too small");
    const int64_t code_bytes = (int64_t)B * row * sizeof(int64_t);
    if (!resume && out != partial) RQB_CUDA(cudaMemcpyAsync(out, partial, code_bytes, cudaMemcpyDeviceToDevice, st));   // xs = partial_sample.clone()
    if (idx0 >= idx_end) return 0;

    int prev = resume ? plan_prev(sampled, idx0) : -1;     // the last sampled position before this span; none: prefill at the first
    int prev_p = -1;                                        // its window position
    if (prev >= 0) win_locate(prev, c.H, c.W, Wt, Ht, &cm.org, &prev_p);
    for (int idx = idx0; idx < idx_end; idx++) {
        if (!plan_sampled(sampled, idx)) continue;
        int org, p;
        win_locate(idx, c.H, c.W, Wt, Ht, &org, &p);
        if (prev < 0 || org != cm.org) {
            cm.org = org;
            RQB_TRY(prefill_prefix(h, out, cond, B, p, ws, st, cv));
        } else {
            for (int j = prev_p + 1; j <= p; j++) RQB_TRY(body_step(h, out, B, j, ws, st, cv));   // decode steps on positions prev_p .. p-1
        }
        for (int d = 0; d < D; d++) {
            const int64_t step = (int64_t)(idx - idx0) * D + d;
            float* lg = logits_out ? logits_out + step * (int64_t)B * V : ws.LOGITS;
            RQB_TRY(head_depth(h, out, B, p, d, ws, lg, st, cv));
            const float* q = noise ? noise + step * noise_stride : nullptr;
            const int64_t off = cm.at(0, p) * D + d;
            RQB_TRY(launch_sample(lg, q, B, V, temperature, top_k[d], top_p[d], out + off, force ? force + off : nullptr, row, st, 1, cfg_n,
                                  cfg_s, keep ? keep + off : nullptr));
        }
        prev = idx; prev_p = p;
    }
    return 0;
}

// rqb200_ar_step on the exact tier: the launches of ar_sample_impl, split at the depth boundary, on the workspace's copy of the
// caller's codes (ws.CODES) and without the sampler
static int ar_step_impl(rqb200_ar* h, const int64_t* xs, int64_t xs_stride, const int64_t* cond, int B, int idx, int d, int restart,
                        float* logits_out, void* wsp, size_t ws_bytes, cudaStream_t st) {
    const rqb200_ar_config& c = h->cfg;
    const int D = c.D, HW = c.H * c.W;
    ArWs ws;
    if (ar_layout(c, B, wsp, ws_bytes, &ws) > ws_bytes) return fail(RQB200_EWORKSPACE, "ar_step: workspace too small");
    // the codes this step consumes (as in ar_fast_step)
    const int64_t lo = restart ? 0 : (d == 0 ? (int64_t)(idx - 1) * D : (int64_t)idx * D);
    const int64_t hi = d == 0 ? (int64_t)idx * D : (int64_t)idx * D + d;
    if (hi > lo)
        RQB_CUDA(cudaMemcpy2DAsync(ws.CODES + lo, (size_t)HW * D * sizeof(int64_t), xs + lo, (size_t)xs_stride * sizeof(int64_t),
                                   (size_t)(hi - lo) * sizeof(int64_t), (size_t)B, cudaMemcpyDeviceToDevice, st));
    if (restart)
        RQB_TRY(prefill_prefix(h, ws.CODES, cond, B, idx, ws, st));
    else if (d == 0)
        RQB_TRY(body_step(h, ws.CODES, B, idx, ws, st));
    return head_depth(h, ws.CODES, B, idx, d, ws, logits_out, st);
}

// rqb200_ar_log_prob on the exact tier: the teacher-forced replay of ar_sample_impl over spans of positions whose logits fit one
// bounded span buffer (each span resumes on the state the previous one left).  Per span: the targets gathered in the logits' row
// order (token step, b), one reduction over all its rows into a [steps][B] buffer, and one strided copy per depth into logp_out.
constexpr int64_t EXACT_LOGPROB_SPAN_BYTES = (int64_t)64 << 20;

static int64_t lp_span_positions(const rqb200_ar_config& c, int B) {
    const int64_t per_pos = (int64_t)c.D * B * c.vocab * (int64_t)sizeof(float);
    return std::max<int64_t>(1, std::min<int64_t>((int64_t)c.H * c.W, EXACT_LOGPROB_SPAN_BYTES / per_pos));
}
struct LpSpan {
    float* logits;               // [P*D][B][V] the span's logits, token-major in raster order
    int64_t* tgt;                // [P*D][B] their targets
    float* lp;                   // [P*D][B] their log-probs
};
static size_t lp_layout(const rqb200_ar_config& c, int B, void* base, size_t cap, ArWs* ws, LpSpan* sp) {
    Arena a(base, cap);
    a.off = ar_layout(c, B, base, cap, ws);
    const int64_t rows = lp_span_positions(c, B) * c.D * B;
    LpSpan s;
    s.logits = a.take<float>(rows * c.vocab);
    s.tgt = a.take<int64_t>(rows);
    s.lp = a.take<float>(rows);
    if (sp) *sp = s;
    return a.off + 256;
}

static int ar_log_prob_impl(rqb200_ar* h, const int64_t* codes, const int64_t* cond, int B, float* logp_out, void* wsp, size_t ws_bytes,
                            cudaStream_t st) {
    const rqb200_ar_config& c = h->cfg;
    const int D = c.D, HW = c.H * c.W, V = c.vocab;
    if (B <= 0) return fail(RQB200_EINVAL, "ar_log_prob: B must be > 0");
    ArWs ws;
    LpSpan sp;
    if (lp_layout(c, B, wsp, ws_bytes, &ws, &sp) > ws_bytes) return fail(RQB200_EWORKSPACE, "ar_log_prob: workspace too small");
    const std::vector<int32_t> top_k(D, V);          // (the sampler writes the forced code; its settings are moot)
    const std::vector<float> top_p(D, 1.f);
    const int64_t P = lp_span_positions(c, B), HWD = (int64_t)HW * D;
    for (int p0 = 0; p0 < HW; p0 += (int)P) {
        const int p1 = (int)std::min<int64_t>(p0 + P, HW), n_pos = p1 - p0, steps = n_pos * D;
        RQB_TRY(ar_sample_impl(h, codes, cond, B, p0, p1, p0 > 0, 1.f, top_k.data(), top_p.data(), nullptr, 0, sp.logits, codes, ws.CODES,
                               wsp, ws_bytes, st, 0, 0.f, nullptr, nullptr, c.H, c.W));
        // row (step, b), step = (idx - p0)*D + d  <-  codes[b][p0*D + step]
        RQB_TRY(launch_gather_targets(codes, 1, steps, B, 0, 1, HWD, (int64_t)p0 * D, sp.tgt, st));
        RQB_TRY(launch_logprob_rows(sp.logits, V, V, (int64_t)steps * B, sp.tgt, 1, sp.lp, st));
        // depth d: rows (idx, d) of the span, D*B floats apart  ->  logp_out[d][p0 .. p1)[B]
        for (int d = 0; d < D; d++)
            RQB_CUDA(cudaMemcpy2DAsync(logp_out + ((int64_t)d * HW + p0) * B, (size_t)B * sizeof(float), sp.lp + (int64_t)d * B,
                                       (size_t)D * B * sizeof(float), (size_t)B * sizeof(float), (size_t)n_pos, cudaMemcpyDeviceToDevice,
                                       st));
    }
    return 0;
}

}  // namespace rqb

extern "C" {

rqb200_ar* rqb200_ar_create(const rqb200_ar_config* cfg, const rqb200_ar_weights* w) {
    if (!cfg || !w) { rqb::set_error("ar_create: null argument"); return nullptr; }
    if (cfg->embed_dim != cfg->n_head * 64) { rqb::set_error("ar_create: embed_dim must be n_head*64"); return nullptr; }
    if (cfg->embed_dim % 64 || cfg->code_dim % 4 || cfg->vocab > 16384 || cfg->cond_len < 1 || cfg->D < 1 ||
        (cfg->codebook_per_depth != 0 && cfg->codebook_per_depth != 1)) {
        rqb::set_error("ar_create: unsupported shape");
        return nullptr;
    }
    if (cfg->weight_dtype != RQB200_F32 && cfg->weight_dtype != RQB200_BF16 && cfg->weight_dtype != RQB200_F16 &&
        cfg->weight_dtype != RQB200_E4M3) {
        rqb::set_error("ar_create: weight dtype");
        return nullptr;
    }
    const bool e4m3 = cfg->weight_dtype == RQB200_E4M3;
    if (e4m3 && cfg->mode != RQB200_MODE_FAST) { rqb::set_error("ar_create: E4M3 weights are a fast-tier format (mode RQB200_MODE_FAST)"); return nullptr; }
    {
        const int ev = cfg->embed_variant;
        const bool tok_in = ev & RQB200_EMB_TOK_INPUT, tok_head = ev & RQB200_EMB_TOK_HEAD;
        const char* bad = nullptr;
        if (ev & ~(RQB200_EMB_TOK_INPUT | RQB200_EMB_TOK_HEAD | RQB200_EMB_NO_CUMSUM | RQB200_EMB_TUPLE | RQB200_EMB_CLS_PER_DEPTH))
            bad = "ar_create: unknown embed_variant bits";
        else if ((tok_in || tok_head) && !w->tok_emb) bad = "ar_create: embed_variant needs tok_emb";
        else if ((!tok_in && !w->w_in) || (!tok_head && cfg->D > 1 && !w->w_head)) bad = "ar_create: embed_variant needs w_in / w_head";
        else if (!(tok_in && tok_head) && !w->codebook) bad = "ar_create: embed_variant needs the RQ-VAE codebook";
        else if (!w->w_cls || !w->b_cls) bad = "ar_create: classifier missing";
        if (bad) { rqb::set_error(bad); return nullptr; }
    }
    if (e4m3) {
        const char* bad = rqb::check_e4m3_weights(*cfg, *w);
        if (bad) { rqb::set_error(bad); return nullptr; }
    }
    rqb200_ar* h = new rqb200_ar();
    h->cfg = *cfg;
    // the scale fields trail the struct: read them only for E4M3 (a caller built against the older struct ends before them)
    h->w = rqb200_ar_weights{};
    std::memcpy(&h->w, w, e4m3 ? sizeof(rqb200_ar_weights) : offsetof(rqb200_ar_weights, s_in));
    h->body.assign(w->body, w->body + cfg->n_body);
    h->head.assign(w->head, w->head + cfg->n_head_layers);
    if (!e4m3)
        for (auto* v : {&h->body, &h->head})
            for (rqb200_block_weights& b : *v) b.sqkv = b.sproj = b.s1 = b.s2 = nullptr;
    h->w.body = h->body.data();
    h->w.head = h->head.data();
    if (cfg->mode == RQB200_MODE_FAST) {
        if (cfg->weight_dtype == RQB200_F32) { rqb::set_error("ar_create: fast tier needs fp16, bf16 or E4M3 weights"); delete h; return nullptr; }
        h->fast = rqb::ar_fast_create(h->cfg, h->w, h->body.data(), h->head.data());
        if (!h->fast) { delete h; return nullptr; }
    }
    return h;
}
void rqb200_ar_destroy(rqb200_ar* h) {
    if (h && h->fast) rqb::ar_fast_destroy(h->fast);
    delete h;
}
size_t rqb200_ar_workspace_bytes(const rqb200_ar* h, int B) {
    if (!h || B <= 0) return 0;
    if (h->fast) return rqb::ar_fast_workspace_bytes(h->fast, B);
    return rqb::ar_layout(h->cfg, B, nullptr, 0, nullptr);
}
// The only way into the sampling loop and the one place its arguments are checked, before any CUDA call; the tiers check only their
// own batch and workspace limits.  cfg_n = 0 unguided, else guided over B = 2 cfg_n rows; keep / sampled_host null: every token sampled
int rqb200_ar_sample_span(rqb200_ar* h, const int64_t* partial, const int64_t* cond, int B, int idx_begin, int idx_end, int resume,
                          float temperature, const int32_t* top_k_host, const float* top_p_host, const float* noise,
                          int64_t noise_stride, float* logits_out, const int64_t* force_codes, int64_t* out_codes,
                          void* workspace, size_t workspace_bytes, void* stream, const uint8_t* keep, const uint8_t* sampled_host,
                          int cfg_n, float cfg_scale, int canvas_h, int canvas_w) {
    if (!h || (!partial && !resume) || !out_codes || !top_k_host || !top_p_host || !workspace)
        return rqb::fail(RQB200_EINVAL, "ar_sample: null argument");
    if (B < 1) return rqb::fail(RQB200_EINVAL, "ar_sample: B must be > 0");
    if (cfg_n < 0 || (cfg_n > 0 && B != 2 * cfg_n))
        return rqb::fail(RQB200_EINVAL, "ar_sample: cfg_n must be 0, or n >= 1 with B = 2n rows (n conditional, then n unconditional)");
    if (canvas_h < h->cfg.H || canvas_w < h->cfg.W)
        return rqb::fail(RQB200_EINVAL, "ar_sample: the canvas must be at least the model's grid (canvas_h >= H, canvas_w >= W)");
    if ((int64_t)canvas_h * canvas_w * h->cfg.D > RQB200_CANVAS_MAX_CODES)
        return rqb::fail(RQB200_EINVAL, "ar_sample: canvas_h * canvas_w * D must be at most RQB200_CANVAS_MAX_CODES (2^31 - 1)");
    if (idx_begin < 0 || idx_end > canvas_h * canvas_w || idx_begin > idx_end)
        return rqb::fail(RQB200_EINVAL, "ar_sample: bad position span");
    if (sampled_host && !resume)
        for (int p = 0; p < idx_begin; p++)
            if (sampled_host[p]) return rqb::fail(RQB200_EINVAL, "ar_sample: sampled_host must be 0 before the call's first position");
    if (rqb200_device_count() <= 0) return rqb::fail(RQB200_ENODEV, "ar_sample: no CUDA device");
    if (h->cfg.weight_dtype != RQB200_F32 && !h->fast) return rqb::fail(RQB200_EINVAL, "ar_sample: 16-bit weights need the fast tier");
    const float cfg_s = cfg_n > 0 ? cfg_scale : 0.f;
    h->step_next = -1;                   // sampling reuses the caches a stepped sequence keeps: that sequence ends here
    rqb::g_launches = 0;
    int rc;
    if (h->fast)
        rc = rqb::ar_fast_sample(h->fast, partial, cond, B, idx_begin, idx_end, resume, temperature, top_k_host, top_p_host, noise,
                                 noise_stride, logits_out, force_codes, out_codes, workspace, workspace_bytes, (cudaStream_t)stream,
                                 cfg_n, cfg_s, keep, sampled_host, canvas_h, canvas_w);
    else
        rc = rqb::ar_sample_impl(h, partial, cond, B, idx_begin, idx_end, resume, temperature, top_k_host, top_p_host, noise,
                                 noise_stride, logits_out, force_codes, out_codes, workspace, workspace_bytes, (cudaStream_t)stream,
                                 cfg_n, cfg_s, keep, sampled_host, canvas_h, canvas_w);
    h->last_launches = rqb::g_launches;
    return rc;
}
int rqb200_ar_step(rqb200_ar* h, const int64_t* xs, int64_t xs_batch_stride, const int64_t* cond, int B, int pos_h, int pos_w,
                   int d, int restart, float* logits_out, void* workspace, size_t workspace_bytes, void* stream) {
    if (!h || !xs || !logits_out || !workspace) return rqb::fail(RQB200_EINVAL, "ar_step: null argument");
    const rqb200_ar_config& c = h->cfg;
    if (B <= 0) return rqb::fail(RQB200_EINVAL, "ar_step: B must be > 0");
    if (pos_h < 0 || pos_h >= c.H || pos_w < 0 || pos_w >= c.W || d < 0 || d >= c.D)
        return rqb::fail(RQB200_EINVAL, "ar_step: position (h, w, d) out of range");
    if (restart && d != 0) return rqb::fail(RQB200_EINVAL, "ar_step: a restart begins a position: d must be 0");
    const int idx = pos_h * c.W + pos_w;
    const int64_t token = (int64_t)idx * c.D + d;
    const int64_t reads = d > 0 ? token : (int64_t)idx * c.D;      // codes of each batch row this step reads: [0, reads) at most
    if (xs_batch_stride < reads) return rqb::fail(RQB200_EINVAL, "ar_step: xs_batch_stride is shorter than the codes this step reads");
    if (!restart && (h->step_ws != workspace || h->step_B != B || h->step_next != token))
        return rqb::fail(RQB200_ESTATE, "ar_step: not the token after the previous step on this workspace and batch (restart the sequence)");
    if (rqb200_device_count() <= 0) return rqb::fail(RQB200_ENODEV, "ar_step: no CUDA device");
    if (c.weight_dtype != RQB200_F32 && !h->fast) return rqb::fail(RQB200_EINVAL, "ar_step: 16-bit weights need the fast tier");
    h->step_next = -1;
    rqb::g_launches = 0;
    int rc;
    if (h->fast)
        rc = rqb::ar_fast_step(h->fast, xs, xs_batch_stride, cond, B, idx, d, restart, logits_out, workspace, workspace_bytes,
                               (cudaStream_t)stream);
    else
        rc = rqb::ar_step_impl(h, xs, xs_batch_stride, cond, B, idx, d, restart, logits_out, workspace, workspace_bytes,
                               (cudaStream_t)stream);
    h->last_launches = rqb::g_launches;
    if (rc == 0) {
        h->step_ws = workspace;
        h->step_B = B;
        h->step_next = token + 1;
    }
    return rc;
}
size_t rqb200_ar_forward_workspace_bytes(const rqb200_ar* h, int B) {
    if (!h || !h->fast || B <= 0) return 0;
    return rqb::ar_fast_forward_workspace_bytes(h->fast, B);
}
int rqb200_ar_forward(rqb200_ar* h, const int64_t* codes, const int64_t* cond, int B, float* logits_out, float* cond_logits_out,
                      void* workspace, size_t workspace_bytes, void* stream) {
    if (!h || !codes || !logits_out || !workspace) return rqb::fail(RQB200_EINVAL, "ar_forward: null argument");
    if (rqb200_device_count() <= 0) return rqb::fail(RQB200_ENODEV, "ar_forward: no CUDA device");
    if (!h->fast) return rqb::fail(RQB200_EINVAL, "ar_forward: the batched forward is a fast-tier path (exact tier: teacher-forced rqb200_ar_sample_span)");
    rqb::g_launches = 0;
    int rc = rqb::ar_fast_forward(h->fast, codes, cond, B, logits_out, cond_logits_out, workspace, workspace_bytes, (cudaStream_t)stream);
    h->last_launches = rqb::g_launches;
    return rc;
}
size_t rqb200_ar_log_prob_workspace_bytes(const rqb200_ar* h, int B) {
    if (!h || B <= 0) return 0;
    if (h->fast) return rqb::ar_fast_log_prob_workspace_bytes(h->fast, B);
    return rqb::lp_layout(h->cfg, B, nullptr, 0, nullptr, nullptr);
}
int rqb200_ar_log_prob(rqb200_ar* h, const int64_t* codes, const int64_t* cond, int B, float* logp_out, float* cond_logp_out,
                       void* workspace, size_t workspace_bytes, void* stream) {
    if (!h || !codes || !logp_out || !workspace) return rqb::fail(RQB200_EINVAL, "ar_log_prob: null argument");
    if (rqb200_device_count() <= 0) return rqb::fail(RQB200_ENODEV, "ar_log_prob: no CUDA device");
    if (!h->fast && cond_logp_out) return rqb::fail(RQB200_EINVAL, "ar_log_prob: cond log-probs come from the fast tier's cond classifier");
    if (h->cfg.weight_dtype != RQB200_F32 && !h->fast) return rqb::fail(RQB200_EINVAL, "ar_log_prob: 16-bit weights need the fast tier");
    rqb::g_launches = 0;
    int rc;
    if (h->fast) {
        rc = rqb::ar_fast_log_prob(h->fast, codes, cond, B, logp_out, cond_logp_out, workspace, workspace_bytes, (cudaStream_t)stream);
    } else {
        h->step_next = -1;               // the replay runs on the kind of workspace a stepped sequence keeps its caches in: that sequence ends
        rc = rqb::ar_log_prob_impl(h, codes, cond, B, logp_out, workspace, workspace_bytes, (cudaStream_t)stream);
    }
    h->last_launches = rqb::g_launches;
    return rc;
}
int rqb200_ar_trace(rqb200_ar* h, long long* out_host, int cap_launches, char* names, int names_cap) {
    if (!h || !h->fast || !out_host) return 0;
    cudaDeviceSynchronize();
    return rqb::ar_fast_trace(h->fast, out_host, cap_launches, names, names_cap);
}
int64_t rqb200_ar_last_launches(const rqb200_ar* h) { return h ? h->last_launches : 0; }
}
