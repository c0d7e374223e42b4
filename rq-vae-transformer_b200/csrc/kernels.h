// internal launch prototypes (host side) shared by the engine translation units
#pragma once
#include <cuda.h>

#include <string>
#include <unordered_map>

#include "common.cuh"

namespace rqb {
// The codebooks of one RQ search / embedding launch, passed by value.  n == 1: one [K,C] table serves every depth (a shared
// codebook); n == D: depth d uses table d ([K_d,C], shared_codebook=False).
constexpr int RQ_MAX_TABLES = 16;
struct RqTables {
    const float* cb[RQ_MAX_TABLES];
    int K[RQ_MAX_TABLES];
    int n;
    __host__ __device__ __forceinline__ int of(int depth) const { return n == 1 ? 0 : depth; }
};
// host arrays of n device pointers / sizes -> RqTables; fails unless 1 <= n <= RQ_MAX_TABLES, every K > 0 and no pointer is null
int make_rq_tables(RqTables* out, const float* const* cb_host, const int32_t* K_host, int n);

// Sliding-window sampling of a code map larger than the model's grid (rqb200_ar_sample_span with a canvas): the token at canvas
// position (i, j) is sampled as the model's token (i - r0, j - c0) of the grid-sized window with origin (r0, c0) = (win_origin(i, H, Ht),
// win_origin(j, W, Wt)).  The window's position p (raster order in the H x W grid) lies at canvas position org + (p / gw) * cw + p % gw
// of its batch row, org = r0 * cw + c0; a batch row holds chw canvas positions.  Kernels that gather codes take it as a template switch:
// their grid instantiation addresses [B, H*W, D] exactly as before.
struct CanvasMap {
    int gw;         // the model grid's width W
    int cw;         // the canvas width Wt
    int org;        // the window's origin, r0 * Wt + c0
    int chw;        // canvas positions per batch row, Ht * Wt
    __host__ __device__ __forceinline__ int64_t at(int64_t b, int p) const { return b * chw + org + (p / gw) * cw + p % gw; }
};
// the window origin along one axis: the window of n cells that centres coordinate i (floor(n/2) cells before it), clamped to [0, nt - n]
inline int win_origin(int i, int n, int nt) {
    const int r = i - n / 2;
    return r < 0 ? 0 : (r > nt - n ? nt - n : r);
}
// canvas position idx (raster order in Ht x Wt) -> its window's origin org and its position p inside the window
inline void win_locate(int idx, int H, int W, int Wt, int Ht, int* org, int* p) {
    const int i = idx / Wt, j = idx % Wt, r0 = win_origin(i, H, Ht), c0 = win_origin(j, W, Wt);
    *org = r0 * Wt + c0;
    *p = (i - r0) * W + (j - c0);
}

// rq_search.cu
int launch_rq_quantize(const float* x, const RqTables& tabs, int64_t N, int C, int D, int64_t* codes, float* quant_list,
                       float* resid_out, cudaStream_t st, int form = 0);
// rq_search2.cu -- 8x8 register tile, codebook streamed in 32-channel slabs, 2-CTA clusters splitting the codebook (the default form)
bool rq_quantize2_supported(int64_t N, const RqTables& tabs, int C);
int launch_rq_quantize2(const float* x, const RqTables& tabs, int64_t N, int C, int D, int64_t* codes, float* quant_list,
                        float* resid_out, cudaStream_t st);
int launch_rq_embed(const int64_t* codes, const RqTables& tabs, int64_t N, int D, int C, float* out, bool sum, cudaStream_t st);
// sampler.cu
int launch_sample(const float* logits, const float* q, int B, int V, float temperature, int top_k, float top_p,
                  int64_t* out_idx, const int64_t* force, int64_t out_stride, cudaStream_t st, int algo = 1, int cfg_n = 0,
                  float cfg_s = 0.f, const uint8_t* keep = nullptr);
// logprob.cu -- out[r] = lg[r*ld + t] - logsumexp(lg[r*ld .. r*ld + V)), t = tgt[r*tgt_stride]; NaN when t is outside [0, V)
int launch_logprob_rows(const float* lg, int64_t ld, int V, int64_t rows, const int64_t* tgt, int64_t tgt_stride, float* out,
                        cudaStream_t st);
// dst[(a*A2 + c)*G + g] = src[off + a*sa + c*sc + g*sg] for a < A1, c < A2, g < G
int launch_gather_targets(const int64_t* src, int A1, int A2, int G, int64_t sa, int64_t sc, int64_t sg, int64_t off, int64_t* dst,
                          cudaStream_t st);
// ar_kernels.cu
int launch_linear(const float* X, int64_t ldx, const void* W, int wdtype, const float* bias, const float* R, float* Y,
                  int64_t ldy, int M, int N, int K, int act, cudaStream_t st);
int launch_layernorm(const float* X, int64_t ldx, const float* g, const float* b, float* Y, int64_t ldy, int M, int E,
                     cudaStream_t st);
int launch_attn_cached(const float* qkv, float* kc, float* vc, float* out, int B, int Tn, int T_past, int Tmax, int E,
                       int nh, cudaStream_t st);
// cb_dstride: floats between depth d's table and depth d+1's (0: one shared [K,C] table; K*C: a [D,K,C] per-depth stack)
int launch_code_emb(const int64_t* codes, const float* cb, int64_t cb_dstride, int B, int HW, int D, int K, int C, int j0, int J,
                    float* out, cudaStream_t st, const CanvasMap* cv = nullptr);
int launch_body_token(const float* lin, const float* pos_hw, int B, int D, int E, int j0, int J, int s0, int Tn, float* X,
                      cudaStream_t st);
int launch_cond_token(const int64_t* cond, const float* cond_emb, const float* pos_cond, int B, int cond_len, int vocab_cond,
                      int E, int Tn, float* X, cudaStream_t st);
// last_only: code d-1 alone instead of the sum over codes 0..d-1
int launch_head_cumsum(const int64_t* codes, const float* cb, int64_t cb_dstride, int B, int HW, int D, int K, int C, int j, int d,
                       float* out, cudaStream_t st, bool last_only = false, const CanvasMap* cv = nullptr);
int launch_row_add(const float* in, int64_t in_row_stride, int64_t in_off, const float* pos, int B, int E, float* out,
                   cudaStream_t st);
// conv_kernels.cu
struct ConvGeom {
    int B, Hi, Wi, Cin;      // input NHWC (before the optional fused nearest x2 upsample)
    int Ho, Wo, Cout;        // output
    int KH, KW, stride;      // 3x3 / 1x1 ; stride 1|2
    int pad;                 // symmetric zero pad of the (possibly upsampled) input; stride-2 convs use pad=0 + implicit
                             // bottom/right zero row/col (F.pad (0,1,0,1), layers.py:52-54)
    int upsample;            // 1: the conv reads nearest-x2-upsampled input (layers.py:31-35)
    int out_nchw;            // 1: write [B,Cout,Ho,Wo] (final conv_out)
    int in_nchw;             // 1: read [B,Cin,Hi,Wi] (encoder conv_in)
    // launch_conv_relu only (the Inception engine): pad is the top/bottom pad and pad_w the left/right one; the output pixel m's
    // channel n goes to Y[m * ldy + yoff + n]
    int pad_w;
    int ldy, yoff;
};
// the geometry of one conv of the Inception and LPIPS layer plans (launch_conv_relu / launch_plan_conv): x NHWC [B, H, W, Cin], a kh x kw
// kernel with pads ph (top / bottom) and pw (left / right), output rows of ldy floats from channel yoff
inline ConvGeom conv_geom(int B, int H, int W, int Cin, int Cout, int kh, int kw, int ph, int pw, int stride, int ldy, int yoff) {
    ConvGeom g{};
    g.B = B; g.Hi = H; g.Wi = W; g.Cin = Cin; g.Cout = Cout; g.KH = kh; g.KW = kw; g.stride = stride; g.pad = ph; g.pad_w = pw;
    g.Ho = (H + 2 * ph - kh) / stride + 1;
    g.Wo = (W + 2 * pw - kw) / stride + 1;
    g.ldy = ldy;
    g.yoff = yoff;
    return g;
}
// the geometry of one conv of the VAE layer plan (vae_engine.cu): H, W the input extent before the optional nearest x2 upsample;
// Ho, Wo = the (upsampled) extent / stride; pad 1 for a 3x3 stride-1 conv, else 0 (stride 2: the Downsample's implicit (0,1,0,1))
ConvGeom vae_conv_geom(int B, int H, int W, int Cin, int Cout, int ks, int stride, int upsample, int in_nchw, int out_nchw);
int launch_conv(const float* X, const void* W, int wdtype, const float* bias, const float* R, float* Y, const ConvGeom& g,
                cudaStream_t st);
int launch_conv_relu(const float* X, const float* W, const float* bias, float* Y, const ConvGeom& g, cudaStream_t st);
// the ResNet plan's residual forms of launch_conv_relu: Y = act(conv + bias + R), R (nullable) fp32 rows of g.ldy floats read at the
// output's own index, act ReLU when relu, else the identity
int launch_conv_res(const float* X, const float* W, const float* bias, const float* R, float* Y, const ConvGeom& g, bool relu,
                    cudaStream_t st);
int launch_groupnorm_silu(const float* X, const float* gamma, const float* beta, float* Y, double* stats_ws, int B, int HW,
                          int C, int silu, cudaStream_t st);
int launch_vae_attn(const float* qkv, float* out, int B, int HW, int C, cudaStream_t st);
// vae_attn_tc.cu -- the same attention on the tensor cores (fp16 operands, fp32 softmax and accumulators), C = 128 | 256 | 384 | 512
int launch_vae_attn_tc(const float* qkv, float* out, int B, int HW, int C, cudaStream_t st);
size_t groupnorm_ws_doubles(int B, int HW);
int launch_gn_stats(const float* X, double* stats_ws, int B, int HW, int C, cudaStream_t st);
// conv_tc.cu -- wgmma implicit-GEMM conv (fast tier), the large-M rows GEMM on the same kernel, and the fp16 operand producers
bool conv_tc_supported(int H, int W, int Cin, int Cout, int ks, int stride, int in_nchw, int out_nchw);
int launch_conv_tc(const void* X16, const void* W16, const void* X16lo, const void* W16lo, const float* bias,
                   const float* residual, float* out, int B, int H, int W, int Cin, int Cout, int ks, int out_nchw,
                   cudaStream_t st, int stride = 1, double* gn_part = nullptr);
bool conv_tc_gn_fusable(int H, int W, int Cout, int ks, int stride);
// the Inception engine's fast-tier conv (conv_tc.cu, inc_conv_tc_kernel): X NHWC [B, Hi, Wi, Cin] fp16 hi + lo, W OHWI [Cout, KH, KW, Cin]
// fp16 hi + lo, out[pix * ldy + yoff + n] = ReLU(conv + bias) as fp32 (out) and / or fp16 hi + lo (out_hi, out_lo).  epi 1 / 2 (the
// ResNet plan, inc_conv_tc_res_kernel): act(conv + bias + residual) with act ReLU / the identity; residual (nullable) fp32 rows of ldy
// floats read at the output's own index.
int launch_inc_conv_tc(const void* X16, const void* X16lo, const void* W16, const void* W16lo, const float* bias, float* out,
                       void* out_hi, void* out_lo, int B, int Hi, int Wi, int Cin, int Cout, int KH, int KW, int pad_h, int pad_w,
                       int stride, int ldy, int yoff, cudaStream_t st, int epi = 0, const float* residual = nullptr);
int launch_rows_gemm_tc(const void* X16, const void* W16, const float* bias, const float* residual, float* out_f32, void* out_16,
                        int gelu, int fmt, int64_t M, int N_out, int K, cudaStream_t st);
int launch_groupnorm_f16(const float* X, const float* gamma, const float* beta, void* Y16, void* Y16lo, double* stats_ws, int B,
                         int HW, int C, int silu, cudaStream_t st, int fused_chunks = 0);
int launch_cast_f16(const float* X, void* Y16, void* Y16lo, int B, int H, int W, int C, int upsample, cudaStream_t st);
int make_tmap_4d_nhwc(CUtensorMap* out, const void* base, uint64_t C, uint64_t W, uint64_t H, uint64_t B, uint32_t box_c,
                      uint32_t box_w, uint32_t box_h, uint32_t box_b, uint32_t stride = 1);

// plan.cu -- what the layer-plan engines (VAE, Inception, CLIP, LPIPS) share
// The caller's tensors of one engine by state_dict key (rqb200_<engine>_set_tensor); the engine reads them at finalize
struct PlanTensor {
    const void* ptr;
    int dtype;
    int64_t numel;
};
struct TensorTable {
    std::unordered_map<std::string, PlanTensor> t;
    void set(const char* key, const void* ptr, int dtype, int64_t numel) { t[key] = PlanTensor{ptr, dtype, numel}; }
    const PlanTensor* find(const std::string& key) const;      // null when the key was never set
    // *out = the fp32 data of key, registered with numel elements; else fails with "<who>: tensor <key> (missing)" / "(wrong size)"
    // (RQB200_ESTATE) or "must be fp32" (RQB200_EINVAL)
    int get_f32(const char* who, const std::string& key, int64_t numel, const float** out) const;
};
// The parameter buffer of the Inception and LPIPS engines: `floats` fp32 values, then on the fast tier their fp16 hi and lo halves
// (split_f16) at the same element offsets.  Each region a plan takes starts at a multiple of 64 floats.
struct SplitParams {
    int64_t floats = 0;
    float* f32 = nullptr;           // bind()
    __half* hi = nullptr;           // null on the exact tier
    __half* lo = nullptr;
    int64_t take(int64_t n) {
        const int64_t o = floats;
        floats = (int64_t)align_up((size_t)(o + n), 64);
        return o;
    }
    size_t bytes(bool fast) const { return (size_t)floats * (sizeof(float) + (fast ? 2 * sizeof(__half) : 0)); }
    void bind(void* params, bool fast) {
        f32 = (float*)params;
        hi = fast ? (__half*)(f32 + floats) : nullptr;
        lo = fast ? hi + floats : nullptr;
    }
};
// finalize of one plan conv: w OIHW [Cout, Cin, KH, KW] -> P.f32 + w_off OHWI and, on the fast tier (P.hi set), its split-fp16 halves
// at the same offset; the bias -> P.f32 + b_off.  bn = {gamma, beta, running_mean, running_var} (nullable): the BatchNorm after the
// conv, folded in fp64 (s = gamma / sqrt(var + bn_eps), w' = w s, b' = beta - mean s); without it w and bias are stored unchanged.
int launch_conv_prep(const float* w, const float* bias, const float* const* bn, double bn_eps, const SplitParams& P, int64_t w_off,
                     int64_t b_off, int Cout, int Cin, int KH, int KW, cudaStream_t st);
// One plan conv + bias + ReLU, weights at w_off / bias at b_off of P.  The fast tier with the input's fp16 hi / lo operands (x_hi set)
// runs inc_conv_tc_kernel, writing y (fp32) and / or y_hi / y_lo (either nullable); otherwise the fp32 FFMA kernel reads x and
// writes y, and on the fast tier y's rows are then cast into y_hi / y_lo (when y_hi is set) for the next conv.
// The residual forms (the ResNet plan): relu = false or a residual (fp32 rows of g.ldy floats at the output's index) compute
// act(conv + bias [+ residual]) on the same two kernels' residual instantiations.
int launch_plan_conv(bool fast, const SplitParams& P, int64_t w_off, int64_t b_off, const float* x, const __half* x_hi,
                     const __half* x_lo, float* y, __half* y_hi, __half* y_lo, const ConvGeom& g, cudaStream_t st,
                     const float* residual = nullptr, bool relu = true);

// inception_engine.cu, shared with the ResNet plan.  3x3 pool of X NHWC [B, H, W, C] with stride and pad into channels [yoff, yoff + C)
// of rows of ldy floats: mode 0 max (padding acts as -inf), mode 1 average over the pixels inside the map; Yhi / Ylo (nullable): the
// values' fp16 hi / lo halves at the same index too
int launch_inc_pool(const float* X, float* Y, int B, int H, int W, int C, int stride, int pad, int mode, int ldy, int yoff,
                    cudaStream_t st, __half* Yhi = nullptr, __half* Ylo = nullptr);
// global average pool: X NHWC [B, HW, C] -> Y [B, C]
int launch_inc_gap(const float* X, float* Y, int B, int HW, int C, cudaStream_t st);

// gemm_tc.cu -- wgmma weight-streaming GEMM (fast tier)
// GT_H16_QGELU: QuickGELU x * sigmoid(1.702 x) (CLIP's MLP) instead of the exact GELU; 16-bit weights, splits == 1
enum GemmTcMode { GT_F32 = 0, GT_H16 = 1, GT_H16_GELU = 2, GT_PARTIAL = 3, GT_H16_QGELU = 4 };
struct GemmTcParams {
    int N_out, K, B, splits, mode;   // B = activation rows (batch rows of the cached step, or B*T tokens of a prefill / forward pass)
    int fmt;                      // 16-bit operand / output format: 0 = fp16 (the reference's autocast class), 1 = bf16
    const float* bias;            // [N_out] (nullable); added as bias * bias_scale
    float bias_scale;
    // GT_F32 only: out = acc + bias + residual[(row0 * res_row_stride) + b * ld_res + n], row0 = res_row_ptr ? *res_row_ptr : 0
    // (ld_res = 0 broadcasts one row -- positional embeddings)
    const float* residual;
    int64_t ld_res, res_row_stride;
    const int* res_row_ptr;
    int res_div;                  // > 1: activation row b reads residual row b / res_div (token-major prefill rows share a positional row)
    void* out;                    // [B, ld_out] f32 / 16-bit
    int64_t ld_out;
    float* partial;               // GT_PARTIAL: [splits][B][N_out] f32 (no bias)
    long long* trace;             // diagnostics, nullable: 4 globaltimer stamps of CTA 0 (entry, dependency resolved, accumulator ready, done)
};
// One weight [N_out, K] of the streamer: 16-bit (fp16 or bf16, the activations' GemmTcParams.fmt) behind its TMA tensor map, or E4M3
// packed in 128 x 64 fragment-order tiles (rqvae._native.pack_fp8_tiles) with one fp32 scale per output row, which takes fp16
// activations only.
struct StreamedWeight {
    int N_out = 0, K = 0;
    const void* w16 = nullptr;          // 16-bit [N_out, K]; null for E4M3
    CUtensorMap tm;                     // of w16
    const uint8_t* q8 = nullptr;        // E4M3 tiles
    const float* s8 = nullptr;          // E4M3 row scales [N_out]
    bool e4m3() const { return w16 == nullptr; }
};
// e4m3: w = the packed tiles (16 B aligned) and scale their row scales (non-null); else w = the 16-bit matrix and scale unused
int make_streamed_weight(StreamedWeight* out, bool e4m3, const void* w, const float* scale, int N_out, int K);
// activation rows per row chunk (gridDim.y) of a launch over `rows` rows: the box height of the activation tensor map.  At most 256,
// and 128 for E4M3 weights (BN = 256 would need both A fragment sets beside 128 accumulators per thread).
inline int gemm_tc_chunk_rows(const StreamedWeight& w, int64_t rows) {
    return rows <= 16 ? 16 : rows <= 32 ? 32 : rows <= 64 ? 64 : (rows <= 128 || w.e4m3()) ? 128 : 256;
}
// D = W X over the p.B activation rows behind tmX; p.N_out and p.K are the weight's
int launch_gemm_tc(const StreamedWeight& w, const CUtensorMap& tmX, GemmTcParams p, bool pdl, cudaStream_t st);
int make_tmap_2d(CUtensorMap* out, const void* base, int elem_bytes_log2, uint64_t inner, uint64_t outer,
                 uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_outer);

// ar_fast.cu / sampler.cu -- device-resident per-call state of the fast AR tier
struct StepState {
    int s;          // body sequence index of the token being processed (= cached body keys before it)
    int idx;        // spatial position whose codes are being sampled
    int step;       // tokens sampled so far in this call (indexes noise / logits_out); 0 in a single-token step
    int cfg_n;      // classifier-free guidance: images n of a guided call over 2n rows [cond | uncond]; 0 unguided
    const int64_t* cond;      // [B, cond_len] or null
    int64_t* codes;           // [B, HW, D] working copy (xs)
    const int64_t* force;     // teacher forcing or null
    const float* noise;       // [n_tok][B][V] or null
    float* logits_out;        // [n_tok][B][V] or null
    int64_t noise_stride;
    float temperature;
    float cfg_scale;          // guidance scale s (cfg_n > 0)
    const uint8_t* keep;      // [B, HW, D] nonzero: the token keeps the code `codes` was initialised with (the sampler writes nothing); or null
    int top_k[8];
    float top_p[8];
    CanvasMap cv;             // sliding-window sampling: where the window of the current segment lies in `codes` (canvas graphs only)
};

// The position plan of a masked sample (rqb200_ar_sample_span): sampled[p] != 0 when some row samples some depth of position p;
// sampled == NULL samples every position.  Only sampled positions run the head stack, classifier and sampler; the body consumes the
// code tokens of the positions between two sampled ones right before the later one's head (positions after the last sampled one
// are never consumed).
inline bool plan_sampled(const uint8_t* sampled, int p) { return sampled == nullptr || sampled[p] != 0; }
// the last sampled position before p, or -1
inline int plan_prev(const uint8_t* sampled, int p) {
    for (int i = p - 1; i >= 0; i--)
        if (plan_sampled(sampled, i)) return i;
    return -1;
}
// canvas: the sampler writes the canvas position of stt->idx through stt->cv (the canvas graphs), else position stt->idx of [B, HW, D]
int launch_sample_dyn(const float* logits, const StepState* stt, int d, int B, int V, int HW, int D, cudaStream_t st, bool pdl,
                      bool canvas = false);

// ar_fast.cu, for the CLIP engine: prefill_attn_flash_kernel over G groups of T tokens (qkv token-major [T*G, 3E] fp16, bias added;
// head dim 64; causal or not) -> att [T*G, E] fp16; LayerNorm (eps 1e-5) of fp32 rows x [rows, E] -> xn fp16 (E % 4 == 0)
int launch_attn_flash_f16(const h16* qkv, h16* att, int G, int T, int E, bool causal, cudaStream_t st);
int launch_ln_rows_f16(int64_t rows, const float* x, const float* g, const float* be, h16* xn, int E, cudaStream_t st);

struct ArFast;
ArFast* ar_fast_create(const rqb200_ar_config& cfg, const rqb200_ar_weights& w, const rqb200_block_weights* body,
                       const rqb200_block_weights* head);
void ar_fast_destroy(ArFast* f);
size_t ar_fast_workspace_bytes(const ArFast* f, int B);
// positions [idx_begin, idx_end) of the raster; resume != 0: continue on the KV state the previous call left in this workspace.
// cfg_n > 0: classifier-free guidance over B = 2 cfg_n rows [cond | uncond] with scale cfg_s.  keep / sampled: the masked-sample
// plan (null: every token sampled).  Ht x Wt: the canvas (H x W: the grid).  Arguments already checked by rqb200_ar_sample_span, except
// B <= 256 and the workspace size.
int ar_fast_sample(ArFast* f, const int64_t* partial, const int64_t* cond, int B, int idx_begin, int idx_end, int resume,
                   float temperature, const int32_t* top_k, const float* top_p, const float* noise, int64_t noise_stride,
                   float* logits_out, const int64_t* force, int64_t* out, void* wsp, size_t ws_bytes, cudaStream_t st, int cfg_n,
                   float cfg_s, const uint8_t* keep, const uint8_t* sampled, int Ht, int Wt);
// the logits of ONE token (idx, d) into logits_out [B,V] (rqb200_ar_step; arguments already checked by the caller)
int ar_fast_step(ArFast* f, const int64_t* xs, int64_t xs_stride, const int64_t* cond, int B, int idx, int d, int restart,
                 float* logits_out, void* wsp, size_t ws_bytes, cudaStream_t st);
size_t ar_fast_forward_workspace_bytes(const ArFast* f, int B);
int ar_fast_forward(ArFast* f, const int64_t* codes, const int64_t* cond, int B, float* logits_out, float* cond_logits_out, void* wsp,
                    size_t ws_bytes, cudaStream_t st);
size_t ar_fast_log_prob_workspace_bytes(const ArFast* f, int B);
int ar_fast_log_prob(ArFast* f, const int64_t* codes, const int64_t* cond, int B, float* logp_out, float* cond_logp_out, void* wsp,
                     size_t ws_bytes, cudaStream_t st);
// diagnostics: copies the stage trace of the last replays to the host (RQB200 ar_config.trace); returns the number of launches traced
int ar_fast_trace(ArFast* f, long long* out_host, int cap_launches, char* names, int names_cap);
}  // namespace rqb
