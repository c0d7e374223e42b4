/*
 * rqb200 -- C ABI of the H100-native RQ-VAE / RQ-Transformer sampling engine (sm_90a).
 *
 * The reference (kakaobrain/rq-vae-transformer @ 341395e) is pure Python/PyTorch and has no plugin / FFI
 * registry; its boundary for this path is the Python class surface of `rqvae.models` (SURVEY.md section 8b).  Each
 * entry point below replaces the *library calls* behind one reference method and is what a ctypes binding in
 * the reference's own classes would call (INTEGRATION.md shows those stubs).  Conventions:
 *   - plain pointers and sizes only; every `const T*` / `T*` tensor argument is a DEVICE pointer unless the
 *     name ends in `_host`; row-major, contiguous; `stream` is a cudaStream_t passed as void*.
 *   - return 0 on success, a negative RQB200_E* code otherwise; `rqb200_last_error()` gives the message.
 *   - entry points never allocate device memory and never synchronise the device; scratch space is a caller
 *     supplied workspace whose size is reported by the matching `*_workspace_bytes` query.
 *   - there is NO CPU fallback: without a CUDA device every compute entry point returns RQB200_ENODEV.
 */
#ifndef RQB200_H
#define RQB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RQB200_OK 0
#define RQB200_EINVAL (-1)   /* bad argument / unsupported shape            */
#define RQB200_ECUDA (-2)    /* a CUDA runtime call or kernel launch failed */
#define RQB200_ENODEV (-3)   /* no CUDA device                               */
#define RQB200_EWORKSPACE (-4) /* workspace too small                        */
#define RQB200_ESTATE (-5)   /* engine not finalised / tensor missing        */

#define RQB200_F32 0
#define RQB200_BF16 1
#define RQB200_F16 2
/* FP8 weights (fast tier only): every streamed weight ([N,K] row-major in the other formats) is given as its E4M3 values q packed in
 * 128 x 64 tiles of 8 KB in wgmma A-fragment order (rqvae._native.pack_fp8_tiles), 16-byte aligned, plus one fp32 scale per output
 * row (the s* fields below); the weight is q * s.  Activations and the KV cache are fp16. */
#define RQB200_E4M3 3

/* arithmetic modes (DESIGN.md "two modes") */
#define RQB200_MODE_EXACT 0  /* fp32 weights + fp32 FFMA: the bit-exact-indices gate                    */
#define RQB200_MODE_FAST 1   /* fp16 (default) or bf16 operands on wgmma, fp32 accumulate: throughput  */

/* rqb200_ar_config.flags (fast tier; scheduling only -- none of them changes a result bit, except SEQUENTIAL_PREFILL's
 * summation order) */
#define RQB200_AR_NO_GRAPH 1            /* launch kernel by kernel instead of replaying CUDA graphs                        */
#define RQB200_AR_NO_PDL 2              /* plain stream order instead of programmatic dependent launch                     */
#define RQB200_AR_TRACE 4               /* record 4 globaltimer stamps per launch (rqb200_ar_trace)                        */
#define RQB200_AR_SEQUENTIAL_PREFILL 32 /* prefill the prefix token by token with the single-step graph (the prefill oracle) */

const char* rqb200_last_error(void);
int rqb200_version(void);
int rqb200_device_count(void);

/* ------------------------------------------------------------------------------------------------ P1
 * RQBottleneck.quantize  (rqvae/models/rqvae/quantizations.py:237-271; VQEmbedding.compute_distances :43-62,
 * find_nearest_embedding :64-69, embed :144-146).  x [N,C] f32, codebook [K,C] f32 (weight[:-1], no padding row).
 * codes [N,D] int64.  quant_list (nullable) [D,N,C] f32 = the D cumulative aggregates (quant_list[i] of the
 * reference).  residual_out (nullable) [N,C] f32 = x - quant_list[D-1].  C must be 256 (quantizations.py:181). */
int rqb200_rq_quantize(const float* x, const float* codebook, int64_t N, int K, int C, int D, int64_t* codes,
                       float* quant_list, float* residual_out, void* stream);
/* The same search with one codebook per depth (RQBottleneck(shared_codebook=False)): depth d searches and subtracts with
 * codebooks_host[d] [K_host[d],C] f32.  codebooks_host / K_host are HOST arrays of D entries, D <= 16; the K_d may differ. */
int rqb200_rq_quantize_depthwise(const float* x, const float* const* codebooks_host, const int32_t* K_host, int64_t N, int C, int D,
                                 int64_t* codes, float* quant_list, float* residual_out, void* stream);

/* One depth of RQBottleneck.get_soft_codes (quantizations.py:371-399): residual [N,C] f32 -> soft_out [N,K] = softmax(-d/temp) with
 * d = VQEmbedding.compute_distances (:43-62); logits_out (nullable) [N,K] = -d/temp (what the stochastic variant samples from). */
int rqb200_rq_soft_codes(const float* residual, const float* codebook, int64_t N, int K, int C, float temp, float* soft_out,
                         float* logits_out, void* stream);

/* RQBottleneck.embed_code (quantizations.py:297-311): out[n,:] = sum_d codebook[codes[n,d],:]  (order d=0..D-1). */
int rqb200_rq_embed_sum(const int64_t* codes, const float* codebook, int64_t N, int D, int K, int C, float* out,
                        void* stream);
/* RQBottleneck.embed_code_with_depth (quantizations.py:313-334): out[n,d,:] = codebook[codes[n,d],:]. */
int rqb200_rq_embed_depth(const int64_t* codes, const float* codebook, int64_t N, int D, int K, int C, float* out,
                          void* stream);
/* embed_code / embed_code_with_depth with one codebook per depth: code d is looked up in codebooks_host[d] [K_host[d],C]
 * (HOST arrays of D entries, D <= 16). */
int rqb200_rq_embed_sum_depthwise(const int64_t* codes, const float* const* codebooks_host, const int32_t* K_host, int64_t N, int D,
                                  int C, float* out, void* stream);
int rqb200_rq_embed_depth_depthwise(const int64_t* codes, const float* const* codebooks_host, const int32_t* K_host, int64_t N,
                                    int D, int C, float* out, void* stream);

/* ------------------------------------------------------------------------------------------------ sampler
 * sample_from_logits (rqvae/utils/utils.py:82-123; top_k_logits :60-64, top_p_probs :67-79).  logits [B,V] f32.
 * q (nullable) [B,V] f32 Exp(1) noise: torch.multinomial(probs,1) == argmax(probs/q) (SURVEY.md finding 7);
 * NULL means q == 1 (arg-max of the filtered distribution).  top_k <= 0 or >= V disables top-k; top_p >= 1
 * takes the reference's p = 1.0 branch.  out_idx [B] int64.  V <= 16384.  No host sync (the reference's NaN
 * check syncs; here NaN -> -inf is done on the device). */
int rqb200_sample_logits(const float* logits, const float* q, int B, int V, float temperature, int top_k,
                         float top_p, int64_t* out_idx, void* stream);

/* ------------------------------------------------------------------------------------------------ P3
 * RQTransformer (rqvae/models/rqtransformer/transformers.py) -- cached AR sampling. */
typedef struct rqb200_block_weights {
    const void *wqkv, *wproj, *w1, *w2;            /* [3E,E] (rows: query|key|value), [E,E], [4E,E], [E,4E]; weight dtype */
    const float *bqkv, *bproj, *b1, *b2;           /* f32 biases */
    const float *ln1_w, *ln1_b, *ln2_w, *ln2_b;    /* f32 */
    /* RQB200_E4M3 only (ignored otherwise): fp32 row scales of wqkv, wproj, w1, w2 -- [3E], [E], [4E], [E].  ABI 106 appended these
     * four pointers, so arrays of this struct built against an older header have the wrong stride: rebuild them. */
    const float *sqkv, *sproj, *s1, *s2;
} rqb200_block_weights;

typedef struct rqb200_ar_config {
    int32_t embed_dim, n_head, n_body, n_head_layers;  /* E, heads (E/heads must be 64), body / head depth   */
    int32_t vocab, H, W, D;                             /* V and block_size                                    */
    int32_t vocab_cond, cond_len;                       /* cond_emb rows, block_size_cond (>=1)                */
    int32_t code_dim, codebook_size;                    /* C (=256) and K of the RQ-VAE codebook               */
    int32_t mode;                                       /* RQB200_MODE_*                                       */
    int32_t weight_dtype;                               /* RQB200_F32 (exact); RQB200_F16, RQB200_BF16 or RQB200_E4M3 (fast) */
    int32_t flags;                                      /* fast tier: RQB200_AR_* flags                         */
    int32_t split_qkv, split_proj, split_fc1, split_fc2; /* fast tier: split-K factors, 0 = fill the SMs        */
    int32_t codebook_per_depth;                         /* 0: w.codebook is [K,C]; 1: [D,K,C], depth d's table at d*K*C */
    int32_t embed_variant;                              /* RQB200_EMB_* bits; 0 = the shipped family (see below)  */
} rqb200_ar_config;

/* rqb200_ar_config.embed_variant: where the body / head tokens come from and which classifier serves depth d
 * (RQTransformerConfig's input_emb_vqvae, head_emb_vqvae, cumsum_depth_ctx, shared_tok_emb, shared_cls_emb; transformers.py:63-99).
 * 0 is the shipped family: body token = sum_d input_mlp(e_d) + pos_emb_hw, head token d = head_mlp(sum_{i<d} e_i) + pos_emb_d[d],
 * one [V,E] classifier, e_i = the RQ-VAE codebook row of code i. */
#define RQB200_EMB_TOK_INPUT 1        /* input_emb_vqvae = false: body token = sum_d tok_emb(code_d) + pos_emb_hw (no w_in / b_in)     */
#define RQB200_EMB_TOK_HEAD 2         /* head_emb_vqvae = false: head token d = tok_emb(code_{d-1}) + pos_emb_d[d] (no w_head / b_head) */
#define RQB200_EMB_NO_CUMSUM 4        /* cumsum_depth_ctx = false (with head_mlp): head token d = head_mlp(e_{d-1}) + pos_emb_d[d]      */
#define RQB200_EMB_TUPLE 8            /* shared_tok_emb = false: tok_emb is [D*V,E], code d of depth d at row d*V + code (TupleEmbedding) */
#define RQB200_EMB_CLS_PER_DEPTH 16   /* shared_cls_emb = false: w_cls [D,V,E], b_cls [D,V]; depth d uses slice d (BatchLinear)       */

typedef struct rqb200_ar_weights {
    const float *pos_emb_cond, *pos_emb_hw, *pos_emb_d;  /* [cond_len,E], [H*W,E], [D,E] f32                    */
    const float* cond_emb;                                /* [vocab_cond,E] f32                                  */
    const void *w_in, *w_head, *w_cls;                    /* [E,C], [E,C], [V,E] ([D,V,E] with EMB_CLS_PER_DEPTH); weight dtype;
                                                             w_in / w_head NULL when EMB_TOK_INPUT / EMB_TOK_HEAD replace them */
    const float *b_in, *b_head, *b_cls;                   /* b_cls [V] or [D,V]                                  */
    const float *cls_ln_w, *cls_ln_b;
    const float* codebook;                                /* [K,C] or [D,K,C] f32 (model_aux.get_code_emb_with_depth); NULL when
                                                             both EMB_TOK_INPUT and EMB_TOK_HEAD are set */
    const rqb200_block_weights* body;                     /* host array [n_body]                                 */
    const rqb200_block_weights* head;                     /* host array [n_head_layers]                          */
    /* optional (cond_len > 1): cond_classifier (transformers.py:100-104) -- only rqb200_ar_forward's cond_logits use it */
    const void* w_ccls;                                   /* [Vc,E], Vc = vocab_cond rounded up to 128 (zero rows); weight dtype; NULL when absent */
    const float *b_ccls, *ccls_ln_w, *ccls_ln_b;
    const float* tok_emb;                                 /* [V,E] or [D*V,E] (EMB_TUPLE) f32; NULL unless EMB_TOK_INPUT or EMB_TOK_HEAD */
    /* RQB200_E4M3 only: fp32 row scales of w_in [E], w_head [E], w_cls ([V], or [D,V] with EMB_CLS_PER_DEPTH: depth d's packed [V,E]
     * slice starts at byte d*V*E of w_cls) and w_ccls [Vc] (the zero padding rows: s = 1, q = 0).  Read only when weight_dtype is
     * RQB200_E4M3, so a caller built against the struct without them is never read past its end. */
    const float *s_in, *s_head, *s_cls, *s_ccls;
} rqb200_ar_weights;

typedef struct rqb200_ar rqb200_ar;

/* Both tiers: embed_dim == 64 * n_head, n_head_layers >= 0 (0: a head-less model, each depth's token goes straight to the
 * classifier).  Fast tier (RQB200_MODE_FAST) also: cond_len + H*W <= 2048 (a 32x32 grid behind up to 1024 prefix tokens),
 * n_body >= 1, E % 128 == 0, V % 128 == 0, code_dim % 64 == 0, D <= 8, E <= 4608.  RQB200_E4M3 weights: fast tier only, every
 * present weight needs its scales and a 16-byte aligned packed stream.  NULL on failure (rqb200_last_error). */
rqb200_ar* rqb200_ar_create(const rqb200_ar_config* cfg, const rqb200_ar_weights* w);
void rqb200_ar_destroy(rqb200_ar* h);
size_t rqb200_ar_workspace_bytes(const rqb200_ar* h, int B);

/* RQTransformer.sample (transformers.py:294-369) with cached_forward (:190-287) and sample_from_logits fused into one device-side
 * loop (no host sync per token), over the positions [idx_begin, idx_end) of the raster.
 *   partial [B,H,W,D] int64 (the prefix before idx_begin is used), cond [B,cond_len] int64 or NULL (zeros),
 *   top_k_host[D] / top_p_host[D]: per-depth settings (HOST arrays, already clamped like :314-330),
 *   noise (nullable): per-token Exp(1) draws, token t (= the t-th (h,w,d) of this span in raster order) at
 *   noise + t*noise_stride, each [B,V] f32; NULL -> q = 1,
 *   logits_out (nullable) [n_tokens,B,V] f32 receives every step's logits (teacher-forcing / parity tests),
 *   force_codes (nullable) [B,H,W,D] int64: teacher forcing -- logits are computed and (optionally) dumped but
 *   the code written back is force_codes' (so the step-parity protocol of SURVEY.md 8c can be run),
 *   out_codes [B,H,W,D] int64.
 * resume == 0: a new call; sample(start_loc=(h, w)) is idx_begin = h*W + w, idx_end = H*W (prefix prefill from `partial`).
 * resume != 0: continues on the KV / context state the previous call left in the SAME workspace (no prefill; `partial` is
 * ignored, out_codes must be the buffer of the previous call).  noise / logits_out are indexed from the first token of THIS
 * span.  Lets a caller draw the per-token noise in bounded chunks.
 * Classifier-free guidance: cfg_n = 0 is unguided (cfg_scale ignored); cfg_n = n >= 1 needs B = 2n rows.  partial, cond,
 * out_codes, force_codes and logits_out are then laid out [n conditional rows | n unconditional rows]; noise is per image,
 * [n_tok][n][V] (noise_stride apart per token).  At every token both branches produce logits c and u, and the sampler draws
 * image b's code from l = u + cfg_scale * (c - u) in fp32 (three rounded operations, no FMA), then temperature, top-k and top-p
 * as unguided, with noise row b; the code is written to rows b and n + b, and both branches consume it from the next token on.
 * Teacher forcing copies every row's own forced code.  logits_out receives the raw logits of all 2n rows.
 * Masked completion samples only the tokens the caller does not keep (keep == sampled_host == NULL: every token sampled):
 *   keep (nullable, device) uint8 [B, H*W, D], rows laid out like out_codes (guided: the image's mask in both branch rows): nonzero keeps
 *     the token -- out_codes holds partial's code there (it was initialised from partial) and the sampler writes nothing, teacher
 *     forcing included.
 *   sampled_host (nullable, host) uint8 [H*W], the same array for every span of a call: nonzero where some row samples some depth of
 *     the position.  Only those positions run the head stack, classifier and sampler; a position marked 0 is kept whole, whatever keep
 *     says.  It must be 0 before the call's first position (start_loc).  NULL marks every position.
 * Every token of a span still takes its noise row and logits_out slot (indexed from the span's first token, as above); the logits_out
 * rows of skipped positions are left untouched.  The body consumes the code tokens of the positions between two sampled positions a < b
 * right before b's head: on the fast tier in one batched pass at sequence offset cond_len + a when b - a is at least a few tokens
 * (token by token with RQB200_AR_SEQUENTIAL_PREFILL), on the exact tier token by token.  That grouping depends on sampled_host alone, so
 * a call split into spans gives the codes of one span bit for bit.
 * Sliding-window sampling of a canvas larger than the grid: canvas_h x canvas_w = Ht x Wt with Ht >= H, Wt >= W (H x W: the
 *   grid, today's call).  partial, force_codes and out_codes are then [B, Ht, Wt, D], keep [B, Ht*Wt, D], sampled_host [Ht*Wt], and
 *   idx_begin / idx_end and the noise / logits_out token indices count canvas positions in raster order.  The token at canvas (i, j, d)
 *   is sampled as the model's token (i - r0, j - c0, d) of the H x W window with origin
 *       r0 = clamp(i - floor(H/2), 0, Ht - H),   c0 = clamp(j - floor(W/2), 0, Wt - W),
 *   seeing the cond prefix, the window's positions before it in window raster order (read from the canvas as it stands) and its own
 *   depths < d -- nothing outside its window.  Consecutive sampled positions with one origin continue one KV cache (one segment); a new
 *   origin restarts the body with a prefill of the window's prefix.  The workspace is the grid's (rqb200_ar_workspace_bytes).
 *   canvas_h * canvas_w * D must not exceed RQB200_CANVAS_MAX_CODES.
 * Fast tier: B <= 256 rows per call (a guided call: n <= 128 images).  The null pointers, B, cfg_n, the canvas, the span and
 * sampled_host are checked before any CUDA call.  ABI 113 appended keep .. cfg_scale and ABI 117 canvas_h and canvas_w: a caller built
 * against an older header must pass them (the grid's H and W for today's call). */
#define RQB200_CANVAS_MAX_CODES 2147483647LL   /* canvas_h * canvas_w * D: canvas positions and offsets are 32-bit */
int rqb200_ar_sample_span(rqb200_ar* h, const int64_t* partial, const int64_t* cond, int B, int idx_begin, int idx_end, int resume,
                          float temperature, const int32_t* top_k_host, const float* top_p_host, const float* noise,
                          int64_t noise_stride, float* logits_out, const int64_t* force_codes, int64_t* out_codes,
                          void* workspace, size_t workspace_bytes, void* stream, const uint8_t* keep, const uint8_t* sampled_host,
                          int cfg_n, float cfg_scale, int canvas_h, int canvas_w);
/* RQTransformer.cached_forward (transformers.py:190-287): the logits of ONE token (h, w, d) into logits_out [B,V] f32.
 *   xs: the caller's code map, int64, batch row b at xs + b*xs_batch_stride, positions in raster order, D codes each
 *       (only the codes this step consumes are read: position idx-1 when d == 0, codes 0..d-1 of position idx when d > 0;
 *       idx = pos_h*W + pos_w);
 *   restart != 0: a new sequence -- d must be 0; prefill cond + positions [0, idx) from xs (batched prefill as in
 *       rqb200_ar_sample_span), then head depth 0;
 *   restart == 0: continue on the KV / context state the previous step left in the SAME workspace; (h,w,d) must be the
 *       token after the previous step's, else RQB200_ESTATE.  A rqb200_ar_sample_span call on the handle ends the sequence.
 * The launches are those of the sampling loop (split-K factors included) minus the sampler: under teacher forcing the logits
 * equal rqb200_ar_sample_span's logits_out bit for bit.  Fast tier: B <= 256 per call.  Arguments are checked before any CUDA
 * call. */
int rqb200_ar_step(rqb200_ar* h, const int64_t* xs, int64_t xs_batch_stride, const int64_t* cond, int B, int pos_h, int pos_w,
                   int d, int restart, float* logits_out, void* workspace, size_t workspace_bytes, void* stream);
/* RQTransformer.forward (transformers.py:113-188): teacher-forced logits of complete code maps, all positions at once (fast tier:
 * M = B*T row GEMMs on wgmma + causal attention; exact tier: returns RQB200_EINVAL -- use rqb200_ar_sample_span with force_codes and
 * logits_out, the sequential replay).  codes [B,H,W,D] int64, cond [B,cond_len] or NULL.
 * logits_out [D][H*W][B][V] f32 (token-major: logits of (b, pos, d) at ((d*H*W + pos)*B + b)*V); cond_logits_out (nullable,
 * cond_len > 1 and w_ccls given) [cond_len-1][B][Vc] f32 with Vc = vocab_cond rounded up to a multiple of 128. */
size_t rqb200_ar_forward_workspace_bytes(const rqb200_ar* h, int B);
int rqb200_ar_forward(rqb200_ar* h, const int64_t* codes, const int64_t* cond, int B, float* logits_out, float* cond_logits_out,
                      void* workspace, size_t workspace_bytes, void* stream);
/* Teacher-forced log-likelihoods of complete code maps (RQTransformer.forward's logits, log-softmaxed and gathered at the codes), without
 * materialising the logits.  Arguments as rqb200_ar_forward.  logp_out [D][H*W][B] f32 (token-major like rqb200_ar_forward's logits):
 * log p(code (b, pos, d) | its prefix) at (d*H*W + pos)*B + b; cond_logp_out (nullable; fast tier, cond_len > 1, cond and w_ccls given)
 * [cond_len-1][B] f32: log p(cond[b][s+1]) under the cond classifier's logits of body token s, over the vocab_cond real classes.
 * Fast tier: the forward's passes, then the classifier in fixed chunks of rows, each chunk's logits (the forward's GEMM for those rows:
 * the forward's values) reduced in a bounded fp32 buffer of the workspace.  Exact tier: the teacher-forced replay of
 * rqb200_ar_sample_span in spans of positions whose logits fit a bounded buffer.  A code outside [0, vocab) gives NaN for its entry;
 * each entry depends on its own row's logits only, deterministically. */
size_t rqb200_ar_log_prob_workspace_bytes(const rqb200_ar* h, int B);
int rqb200_ar_log_prob(rqb200_ar* h, const int64_t* codes, const int64_t* cond, int B, float* logp_out, float* cond_logp_out,
                       void* workspace, size_t workspace_bytes, void* stream);
/* fast tier with RQB200_AR_TRACE: copies 4 globaltimer stamps (ns: entry, dependency resolved, accumulator ready / mid, done) per
 * launch slot of the last graph replays to out_host[cap_launches][4] and the slot names ('\n'-separated) to names; returns the
 * number of slots (0 when tracing is off).  Synchronises the device. */
int rqb200_ar_trace(rqb200_ar* h, long long* out_host, int cap_launches, char* names, int names_cap);
/* number of kernels the last rqb200_ar_sample_span / _step / _forward call launched (bench.py's gpu_launches) */
int64_t rqb200_ar_last_launches(const rqb200_ar* h);

/* ------------------------------------------------------------------------------------------------ P2
 * RQVAE encode / decode (rqvae/models/rqvae/rqvae.py:80-109; modules.py:73-98,171-202; layers.py). */
/* OR-ed into rqb200_vae_config.mode (fast tier; diagnostics): GroupNorm statistics by the stand-alone gn_stats pass instead of the
 * producing conv's epilogue */
#define RQB200_VAE_NO_GN_FUSE 0x100
typedef struct rqb200_vae_config {
    int32_t ch, n_levels, ch_mult[8], num_res_blocks;
    int32_t n_attn_res, attn_resolutions[8];
    int32_t resolution, z_channels, embed_dim, in_channels, out_ch;
    int32_t codebook_size, depth;     /* K, D */
    int32_t mode;                     /* RQB200_MODE_*: EXACT = f32 conv weights, FAST = f16 conv weights; | RQB200_VAE_* flags */
} rqb200_vae_config;

typedef struct rqb200_vae rqb200_vae;

rqb200_vae* rqb200_vae_create(const rqb200_vae_config* cfg);
void rqb200_vae_destroy(rqb200_vae* h);
/* register one tensor under its reference state_dict key (SURVEY.md A.3).  Conv weights must be passed
 * re-laid-out as [Cout,KH,KW,Cin] (OHWI) in the engine's weight dtype; everything else f32 as stored.  The RQ codebook is
 * either "codebook" ([K,C], shared by every depth) or "codebook.0" .. "codebook.<D-1>" (one [K_d,C] table per depth,
 * K_d = numel / embed_dim); finalize requires exactly one of the two. */
int rqb200_vae_set_tensor(rqb200_vae* h, const char* key, const void* ptr, int dtype, int64_t numel);
/* resolves every layer of encoder+decoder against the registered tensors; fails listing the first missing key */
int rqb200_vae_finalize(rqb200_vae* h);
size_t rqb200_vae_workspace_bytes(const rqb200_vae* h, int B);
/* RQVAE.decode (rqvae.py:85-89): z_q [B,h,w,embed_dim] f32 NHWC -> out [B,out_ch,R,R] f32 NCHW */
int rqb200_vae_decode(rqb200_vae* h, const float* z_q, int B, float* out, void* workspace, size_t workspace_bytes,
                      void* stream);
/* RQVAE.decode_code (rqvae.py:105-109): codes [B,h,w,D] int64 -> out NCHW */
int rqb200_vae_decode_code(rqb200_vae* h, const int64_t* codes, int B, float* out, void* workspace,
                           size_t workspace_bytes, void* stream);
/* RQVAE.encode (rqvae.py:80-83): x [B,in_channels,R,R] f32 NCHW -> z_e [B,h,w,embed_dim] f32 NHWC */
int rqb200_vae_encode(rqb200_vae* h, const float* x, int B, float* z_e, void* workspace, size_t workspace_bytes,
                      void* stream);
int64_t rqb200_vae_last_launches(const rqb200_vae* h);
/* Any image size (the reference's RQ-VAE is fully convolutional): the same calls on B images of H x W pixels, H and W positive
 * multiples of f = 2^(n_levels - 1) (RQB200_EINVAL otherwise; the workspace query returns 0).  Which levels carry an AttnBlock
 * follows the configured resolution ladder, as in the reference.  The calls above are these at H = W = resolution. */
size_t rqb200_vae_workspace_bytes_hw(const rqb200_vae* h, int B, int H, int W);
/* x [B,in_channels,H,W] f32 NCHW -> z_e [B,H/f,W/f,embed_dim] f32 NHWC */
int rqb200_vae_encode_hw(rqb200_vae* h, const float* x, int B, int H, int W, float* z_e, void* workspace, size_t workspace_bytes,
                         void* stream);
/* z_q [B,hl,wl,embed_dim] f32 NHWC (hl, wl the latent extent) -> out [B,out_ch,hl f,wl f] f32 NCHW; its workspace is
 * rqb200_vae_workspace_bytes_hw(h, B, hl f, wl f) */
int rqb200_vae_decode_hw(rqb200_vae* h, const float* z_q, int B, int hl, int wl, float* out, void* workspace, size_t workspace_bytes,
                         void* stream);

/* ------------------------------------------------------------------------------------------------ FID Inception-v3
 * InceptionV3 (rqvae/metrics/inception.py, use_fid_inception=True): the pytorch-fid Inception-v3 behind FID, as a static layer plan
 * (csrc/inception_engine.cu).  Tensors are registered under the reference's InceptionV3 state_dict keys as they are (fp32, device):
 * "<layer>.conv.weight" OIHW and "<layer>.bn.{weight,bias,running_mean,running_var}" for every BasicConv2d of blocks 0..last_block,
 * plus "fc.weight" [1008, 2048] / "fc.bias" when last_block == 3.  rqb200_inception_finalize names the first missing or mis-sized
 * key, then folds each BatchNorm (eps 0.001) into its conv in fp64 on `stream`, into the caller's parameter buffer of
 * rqb200_inception_params_bytes(h) bytes, which must stay alive and unchanged while the engine is used.  Two tiers:
 * RQB200_MODE_EXACT runs every conv on fp32 FFMA; RQB200_MODE_FAST runs every conv but Conv2d_1a_3x3 (Cin = 3, fp32 FFMA on both
 * tiers) on the wgmma implicit GEMM with split-fp16 operands (three fp16 products per k step, fp32 accumulate).  ABI 116 added
 * this section. */
typedef struct rqb200_inception rqb200_inception;
typedef struct {
    int32_t last_block; /* 0..3: the deepest block the engine holds (InceptionV3's max(output_blocks)) */
    int32_t mode;       /* RQB200_MODE_EXACT or RQB200_MODE_FAST */
} rqb200_inception_config;

/* rqb200_inception_forward flags */
#define RQB200_INC_RESIZE 1      /* bilinear resize (align_corners=False) to 299 x 299 first; else H, W >= 75 */
#define RQB200_INC_NORMALIZE 2   /* x -> 2 x - 1 */
#define RQB200_INC_OUT0 4        /* write block 0's output (64 channels) to out0; OUT1 = 8, OUT2 = 16 (192, 768 channels) */
#define RQB200_INC_OUT1 8
#define RQB200_INC_OUT2 16
#define RQB200_INC_OUT3 32       /* write the pooled features [B, 2048] to out3 */
#define RQB200_INC_LOGITS 64     /* write fc's logits [B, 1008] to logits (last_block == 3) */

rqb200_inception* rqb200_inception_create(const rqb200_inception_config* cfg);
void rqb200_inception_destroy(rqb200_inception* h);
int rqb200_inception_set_tensor(rqb200_inception* h, const char* key, const void* ptr, int dtype, int64_t numel);
size_t rqb200_inception_params_bytes(const rqb200_inception* h);
int rqb200_inception_finalize(rqb200_inception* h, void* params, size_t params_bytes, void* stream);
/* the workspace of rqb200_inception_forward on B images of H x W with these flags; 0 for an extent the network does not take.  A
 * batch whose activations exceed 2 GiB runs in chunks of as many images as fit, so the workspace stops growing with B there. */
size_t rqb200_inception_workspace_bytes(rqb200_inception* h, int B, int H, int W, int flags);
/* x NCHW [B, 3, H, W] f32 in [0, 1] (the reference's input).  Block k's output, NCHW [B, C_k, h_k, w_k] (C = 64, 192, 768), goes to
 * out_k when flags has RQB200_INC_OUT<k>; out3 [B, 2048] and logits [B, 1008] likewise.  An image's outputs do not depend on the other
 * images of the batch. */
int rqb200_inception_forward(rqb200_inception* h, const float* x, int B, int H, int W, int flags, float* out0, float* out1, float* out2,
                             float* out3, float* logits, void* workspace, size_t workspace_bytes, void* stream);
int64_t rqb200_inception_last_launches(const rqb200_inception* h);

/* ------------------------------------------------------------------------------------------------ CLIP ViT
 * OpenAI's CLIP ViT image and text encoders (the model behind the reference's rqvae/metrics/clip_score.py) as a static layer plan
 * (csrc/clip_engine.cu).  Tensors are registered under OpenAI's state_dict keys as they are (fp32, device): visual.conv1.weight,
 * visual.class_embedding, visual.positional_embedding, visual.ln_pre.*, visual.transformer.resblocks.N.{ln_1, attn.in_proj_*,
 * attn.out_proj.*, ln_2, mlp.c_fc.*, mlp.c_proj.*}, visual.ln_post.*, visual.proj, token_embedding.weight, positional_embedding,
 * transformer.resblocks.N.*, ln_final.*, text_projection.  rqb200_clip_finalize names the first missing or mis-sized key, then packs
 * conv1 (K padded to a multiple of 64), the transposed projections and, on the fast tier, fp16 copies of every GEMM weight into the
 * caller's buffer of rqb200_clip_params_bytes(h) bytes, which must stay alive and unchanged (as must the registered tensors) while
 * the engine is used.  Heads = width / 64.  RQB200_MODE_EXACT: fp32 FFMA throughout.  RQB200_MODE_FAST: fp16 operands on the wgmma
 * GEMMs (fp32 accumulate), fp32 residual stream, LayerNorm and softmax; widths must be multiples of 128.  ABI 118 added this section. */
typedef struct rqb200_clip rqb200_clip;
typedef struct {
    int32_t vision_width, vision_layers, vision_patch, vision_resolution;
    int32_t text_width, text_layers, context_length, vocab_size;
    int32_t embed_dim;
    int32_t mode;       /* RQB200_MODE_EXACT or RQB200_MODE_FAST */
} rqb200_clip_config;

/* rqb200_clip_encode_image flags */
#define RQB200_CLIP_PREPROCESS 1   /* x = NCHW pixels in [0, 1] at any H x W: (x * 255) truncated to uint8 (inputs clamped to [0, 1] first),
                                    * Pillow's bicubic resize of the shorter side to R, centre crop R x R, (u / 255 - mean) / std;
                                    * bit-exact to the PIL / torchvision route.  Else x = an already-normalised [B, 3, R, R] batch. */

rqb200_clip* rqb200_clip_create(const rqb200_clip_config* cfg);
void rqb200_clip_destroy(rqb200_clip* h);
int rqb200_clip_set_tensor(rqb200_clip* h, const char* key, const void* ptr, int dtype, int64_t numel);
size_t rqb200_clip_params_bytes(const rqb200_clip* h);
int rqb200_clip_finalize(rqb200_clip* h, void* params, size_t params_bytes, void* stream);
/* workspaces of one encode call; 0 for an input the call refuses */
size_t rqb200_clip_workspace_bytes(rqb200_clip* h, int B, int H, int W, int flags);
size_t rqb200_clip_text_workspace_bytes(rqb200_clip* h, int N);
/* image features [B, embed_dim] fp32 of x (see RQB200_CLIP_PREPROCESS) */
int rqb200_clip_encode_image(rqb200_clip* h, const float* x, int B, int H, int W, int flags, float* feat_out, void* workspace,
                             size_t workspace_bytes, void* stream);
/* text features [N, embed_dim] fp32 of tokens [N, context_length] int64 (ids in [0, vocab_size)), pooled at tokens.argmax(-1) */
int rqb200_clip_encode_text(rqb200_clip* h, const int64_t* tokens, int N, float* feat_out, void* workspace, size_t workspace_bytes,
                            void* stream);
/* out[i] = F.cosine_similarity(img_feat[i], txt_feat[i]) (eps 1e-8) for n rows of dim floats */
int rqb200_clip_cosine(const float* img_feat, const float* txt_feat, int n, int dim, float* out, void* stream);
int64_t rqb200_clip_last_launches(const rqb200_clip* h);
/* the host resize plan of an H x W input at resolution R: out6 = {resized H, resized W, crop top, crop left, horizontal taps per
 * output pixel (0: that pass is skipped), vertical taps} */
int rqb200_clip_resize_plan(int H, int W, int R, int32_t* out6);

/* ------------------------------------------------------------------------------------------------ diagnostics
 * Single-kernel entry points used by tests/ and bench.py's roofline leg; not part of the reference-facing surface.
 * rqb200_dbg_gemm_tc: one launch of the wgmma weight-streaming GEMM (csrc/gemm_tc.cu):
 *   out[b, n] = act(sum_k W[n,k] X[b,k] + bias[n]) (+ residual[b,n]);  W [N_out,K], X [B,K] both 16-bit: fmt 0 = fp16, 1 = bf16;
 *   act (16-bit output only): gelu 0 none, 1 exact GELU, 2 QuickGELU x * sigmoid(1.702 x) (16-bit weights; ABI 118);
 *   partial != NULL: partial [splits,B,N_out] f32 receives the per-split sums instead (no bias / act / residual; B <= 256).
 *   B > 256 (splits == 1) runs as row chunks of 256 (the batched-prefill / teacher-forced-forward shape). */
/* rqb200_dbg_clip_preprocess: the CLIP preprocessing of x [B, 3, H, W] at resolution R: u8_out [B, 3, R, R] the uint8 crop, norm_out
 * [B, 3, R, R] fp32 the normalised tensor (either nullable).  rqb200_dbg_clip_attn: the exact tier's fp32 attention, qkv [T * G, 3E]
 * token-major -> out [T * G, E]; rqb200_dbg_clip_attn_flash: the fast tier's (prefill_attn_flash_kernel, fp16).  causal 0 / 1. */
int rqb200_dbg_clip_preprocess(const float* x, int B, int H, int W, int R, uint8_t* u8_out, float* norm_out, void* stream);
int rqb200_dbg_clip_attn(const float* qkv, float* out, int G, int T, int E, int causal, void* stream);
int rqb200_dbg_clip_attn_flash(const void* qkv16, void* att16, int G, int T, int E, int causal, void* stream);
int rqb200_dbg_gemm_tc(const void* W16, const void* X16, const float* bias, const float* residual, void* out,
                       int out_is_16, int gelu, float* partial, int N_out, int K, int B, int splits, int fmt, void* stream);
/* rqb200_dbg_gemm_tc_fp8: the same GEMM with FP8 (E4M3) weights and fp16 activations:
 *   out[b, n] = act(scale[n] * sum_k q[n,k] X[b,k] + bias[n]) (+ residual[b,n]);  partial != NULL: scale[n] * the per-split sums.
 *   W8_packed: q [N_out,K] (float8_e4m3fn) rearranged into 128 x 64 tiles of 8 KB in wgmma A-fragment order, 16-byte aligned
 *   (rqvae._native.pack_fp8_tiles); scale [N_out] f32.  X16 [B,K] fp16, 16-bit outputs fp16.  B > 128 (splits == 1) runs as row
 *   chunks of 128. */
int rqb200_dbg_gemm_tc_fp8(const void* W8_packed, const float* scale, const void* X16, const float* bias, const float* residual,
                           void* out, int out_is_16, int gelu, float* partial, int N_out, int K, int B, int splits, void* stream);
/* rqb200_dbg_gemm_tc_epi: one launch of the same GEMM with the epilogue options the AR engine passes (its w_in / w_head launches):
 *   W: 16-bit [N_out,K] (fmt 0 fp16, 1 bf16) when scale == NULL, else packed E4M3 tiles with row scales scale [N_out] (fmt 0).
 *   acc[b, n] = sum_k W[n,k] X[b,k] (times scale[n]); mode 0: out f32 [B,N_out] = acc + bias[n] * bias_scale + residual[row0 *
 *   res_row_stride + r * ld_res + n] with r = b / res_div (res_div > 1) or b, row0 = *res_row_ptr (a device int) or 0 when
 *   res_row_ptr == NULL (residual nullable; ld_res = 0 broadcasts one row); mode 1: acc + bias * bias_scale rounded to 16 bits; mode 2:
 *   gelu_erf of it; mode 3: partial [splits,B,N_out] f32 = the per-split accumulators (B <= 256).  Modes 0-2 take splits == 1. */
int rqb200_dbg_gemm_tc_epi(const void* W, const float* scale, const void* X16, int mode, const float* bias, float bias_scale,
                           const float* residual, int64_t ld_res, int res_div, const int* res_row_ptr, int64_t res_row_stride,
                           void* out, float* partial, int N_out, int K, int B, int splits, int fmt, void* stream);

/* rqb200_dbg_rq_quantize: rqb200_rq_quantize with the kernel form forced: 1 = csrc/rq_search.cu (2x4 register tile), 2 =
 * csrc/rq_search2.cu (8x8 register tile, 2-CTA clusters splitting the codebook; fails with RQB200_EINVAL for shapes it does not
 * take), 0 = what rqb200_rq_quantize picks.  Both forms are bit-identical (tests/test_gpu_parity.py). */
int rqb200_dbg_rq_quantize(int form, const float* x, const float* codebook, int64_t N, int K, int C, int D, int64_t* codes,
                           float* quant_list, float* residual_out, void* stream);
/* rqb200_rq_quantize_depthwise with the kernel form forced (form 2 takes every K_d <= 16384).  Both forms are bit-identical. */
int rqb200_dbg_rq_quantize_depthwise(int form, const float* x, const float* const* codebooks_host, const int32_t* K_host, int64_t N,
                                     int C, int D, int64_t* codes, float* quant_list, float* residual_out, void* stream);
/* rqb200_dbg_sample_logits: rqb200_sample_logits with the top-k threshold search forced: 0 = 8-pass radix select, 1 = bucket
 * select (the default).  Identical indices. */
int rqb200_dbg_sample_logits(int algo, const float* logits, const float* q, int B, int V, float temperature, int top_k,
                             float top_p, int64_t* out_idx, void* stream);

/* rqb200_dbg_conv_tc: one launch of the wgmma implicit-GEMM conv (csrc/conv_tc.cu): X NHWC fp16 [B,H,W,Cin], W OHWI fp16
 * [Cout,ks,ks,Cin], stride 1 "same" padding, out f32 NHWC (+bias, +residual; Cout % 16 == 0) or NCHW when out_nchw (+bias only:
 * a residual is refused with RQB200_EINVAL).  X16lo / W16lo (both
 * required, RQB200_EINVAL when either is NULL): the fp16 "lo" halves (value - fp16(value)) for the split-fp16 products, three
 * per conv.  Operands are fp16 only: out_nchw bit 1 (bf16) is refused with RQB200_EINVAL.  Every refusal comes before any CUDA
 * call.  out_nchw bits 8..: stride (2: the Downsample conv, H, W the output extent). */
int rqb200_dbg_conv_tc(const void* X16, const void* W16, const void* X16lo, const void* W16lo, const float* bias,
                       const float* residual, float* out, int B, int H, int W, int Cin, int Cout, int ks, int out_nchw,
                       void* stream);

/* rqb200_dbg_conv_tc_gn: rqb200_dbg_conv_tc (NHWC output only) whose epilogue also writes the GroupNorm(32) partial statistics
 * of its output: gn_part[((b * (H*W/32) + chunk) * 32 + group) * 2 + {0: sum, 1: sum of squares}] as fp64, the chunks of one
 * (image, group) summing to the group's totals. */
int rqb200_dbg_conv_tc_gn(const void* X16, const void* W16, const void* X16lo, const void* W16lo, const float* bias,
                          const float* residual, float* out, double* gn_part, int B, int H, int W, int Cin, int Cout, int ks,
                          int out_nchw, void* stream);

/* rqb200_dbg_rows_gemm: the large-M GEMM of the batched prefill / forward passes (csrc/conv_tc.cu launch_rows_gemm_tc: persistent
 * 128 x BN tiles, wgmma): out[m,n] = act(sum_k X[m,k] W[n,k] + bias[n]) (+ residual[m,n]).  X [ceil(M/128)*128, K] and
 * W [N_out,K] 16-bit (fmt 0 fp16 / 1 bf16); exactly one of out_f32 / out_16; gelu (0 none, 1 exact GELU,
 * 2 QuickGELU since ABI 118) applies to out_16 only. */
int rqb200_dbg_rows_gemm(const void* X16, const void* W16, const float* bias, const float* residual, float* out_f32, void* out_16,
                         int gelu, int fmt, int64_t M, int N_out, int K, void* stream);

/* rqb200_dbg_log_prob_rows: one launch of the reduction behind rqb200_ar_log_prob (csrc/logprob.cu): for each of `rows` rows of
 * logits [rows, ld] f32 (V <= ld valid columns), out[r] = logits[r, t] - logsumexp(logits[r, 0..V)) with t = targets[r] (int64); NaN
 * when t is outside [0, V).  Nothing outside a row's V columns is read. */
int rqb200_dbg_log_prob_rows(const float* logits, int64_t ld, int V, int64_t rows, const int64_t* targets, float* out, void* stream);

/* The fast AR tier's non-GEMM kernels (csrc/ar_fast.cu), one launch each through the launcher the engine calls (its form choice
 * included).  16-bit tensors are fp16 (fmt 0) or bf16 (fmt 1); nh = E / 64 heads of 64 dims; a KV cache is [B or G][nh][Tmax][64].
 * rqb200_dbg_attn_step: one step attention over B rows.  q, k, v [B, nh, 64] = fp32 (bqkv + part[0] + ... + part[S-1]) in that order,
 *   rounded to 16 bits (bqkv [3E] f32; part [S, B, 3E] f32, rows query|key|value); k, v are written at cache row t of kc / vc; att [B, E]
 *   = softmax(q k^T / 8) v over the cached rows [0, t) and the new token.  t is *t_dev (a device int32, the body graph's path) when
 *   t_dev != NULL, else t_host.  form 1 = attn_fast_kernel, 2 = attn_fast2_kernel (RQB200_EINVAL unless Tmax <= 321), 0 = the form the
 *   engine runs for this Tmax (2 for 16 <= Tmax <= 321, else 1).  Tmax <= 2048. */
int rqb200_dbg_attn_step(int form, const float* part, int S, const float* bqkv, void* kc, void* vc, void* att, int B, int E, int Tmax,
                         const int* t_dev, int t_host, int fmt, void* stream);
/* rqb200_dbg_prefill_attn: the causal attention of a batched pass over G groups of T <= 2048 tokens: qkv [T*G, 3E] 16-bit, token-major
 *   (row of token t of group g = t*G + g; query|key|value); att [T*G, E].  kc / vc (both or neither, T <= Tmax) receive the cache rows
 *   [0, T) of every (group, head), nothing else.  The kernel is chosen by T as in the engine: a warp per (group, head) for T <= 4 and
 *   T <= 8, 64 x 64 tiles with an online softmax above. */
int rqb200_dbg_prefill_attn(const void* qkv, void* kc, void* vc, void* att, int G, int T, int E, int Tmax, int fmt, void* stream);
/* rqb200_dbg_append_attn: the same attention for T new tokens at sequence offset T0 (the fast tier's append of a run of kept positions
 *   to the body cache): qkv / att as above for the new tokens; new token t (sequence token T0 + t) sees the cache rows [0, T0) of kc / vc
 *   and the new tokens 0 .. t, and its k / v are written at cache row T0 + t.  Cache rows outside [T0, T0 + T) are read (below T0) or
 *   untouched.  kc, vc required; T0 + T <= Tmax <= 2048.  T0 > 0: the 64 x 64 tiled kernel for every T; T0 = 0 is
 *   rqb200_dbg_prefill_attn's launch. */
int rqb200_dbg_append_attn(const void* qkv, void* kc, void* vc, void* att, int G, int T0, int T, int E, int Tmax, int fmt, void* stream);
/* rqb200_dbg_ln: LayerNorm (eps 1e-5) of `rows` rows of E <= 4608 (E % 128 == 0) f32: x_out (nullable) = x_in + bias + part[0] + ...
 *   + part[S-1] + extra, summed in fp32 in that order (x_in / bias / extra nullable, bias / extra one [E] row for all rows; part [S, rows,
 *   E]); xn (nullable; g, b [E]) = 16-bit LN(x).  x_in == x_out is allowed.  form 1: ln_reduce_kernel (the step's LN1 / LN2 form, one CTA
 *   per row); form 2: ln_rows_kernel (the batched passes', a warp per row, rows grid-strided); form 0: the batched passes' choice by the
 *   row count (form 1 below 512 rows, else form 2).  Forms 0 and 2 need x_in and take no part or bias. */
int rqb200_dbg_ln(int form, const float* x_in, const float* part, int S, const float* bias, const float* extra, float* x_out, const float* g,
                  const float* b, void* xn, int64_t rows, int E, int fmt, void* stream);
/* rqb200_dbg_act_reduce: h [B, N] 16-bit = gelu_erf(fp32 (bias + part[0] + ... + part[S-1])) with bias [N], part [S, B, N] f32;
 *   N % 4 == 0. */
int rqb200_dbg_act_reduce(const float* part, int S, const float* bias, void* h, int B, int N, int fmt, void* stream);

/* The VAE engine's kernels between the convs, and the exact tier's conv (csrc/conv_kernels.cu, csrc/conv_tc.cu), one launch each
 * through the launcher the engine calls.  Activations are NHWC f32 unless stated.
 * rqb200_dbg_vae_conv: the fp32 FFMA implicit-GEMM conv of the exact tier (and of the encoder's conv_in on both tiers), with the
 *   engine's geometry rule: X [B, H, W, Cin] (NCHW [B, Cin, H, W] when in_nchw), Wt OHWI [Cout, ks, ks, Cin] in wdtype (RQB200_F32,
 *   RQB200_F16 or RQB200_BF16), ks 1 or 3.  upsample: the conv reads the nearest x2 upsample of X; stride 2 (no upsample): the
 *   Downsample's F.pad (0, 1, 0, 1) then a 3x3 stride-2 conv.  Output extent Ho = (upsample ? 2H : H) / stride (Wo alike), padding 1
 *   for 3x3 stride 1, else 0.  out [B, Ho, Wo, Cout] (NCHW [B, Cout, Ho, Wo] when out_nchw) = conv + bias (nullable) + residual
 *   (nullable, [B, Ho, Wo, Cout]; not with out_nchw). */
int rqb200_dbg_vae_conv(const float* X, const void* Wt, int wdtype, const float* bias, const float* residual, float* out, int B, int H,
                        int W, int Cin, int Cout, int ks, int stride, int upsample, int in_nchw, int out_nchw, void* stream);
/* rqb200_dbg_groupnorm: GroupNorm(32, eps 1e-6) of X [B, HW, C] (C % 32 == 0), then SiLU when silu, with gamma / beta [C] f32.
 *   form 0: the exact tier (gn_stats_kernel + gn_apply_kernel) into Y [B, HW, C] f32.
 *   form 1: the fast tier with stand-alone statistics (gn_stats_kernel, gn_finalize_kernel, gn_apply_f16_kernel) into the fp16 conv
 *   operand Y16 [B, HW, C] and, when Y16lo != NULL, its lo half (value - fp16(value), rounded to fp16).  C % 128 == 0.
 *   form 2: as form 1 from the partial statistics a conv epilogue left in stats_ws (rqb200_dbg_conv_tc_gn on X with gn_part =
 *   stats_ws): HW / 32 chunks per image, HW % 32 == 0.
 *   stats_ws holds ws_doubles doubles, at least B * ceil(HW / 32) * 64 + B * 64 (RQB200_EWORKSPACE otherwise); its contents after
 *   the call are unspecified. */
int rqb200_dbg_groupnorm(int form, const float* X, const float* gamma, const float* beta, float* Y, void* Y16, void* Y16lo,
                         double* stats_ws, int64_t ws_doubles, int B, int HW, int C, int silu, void* stream);
/* rqb200_dbg_cast_f16: the fast tier's conv operand of X [B, H, W, C] (C % 4 == 0): Y16 = fp16(X) and, when Y16lo != NULL,
 *   Y16lo = fp16(X - Y16); upsample: of the nearest x2 upsample of X, [B, 2H, 2W, C]. */
int rqb200_dbg_cast_f16(const float* X, void* Y16, void* Y16lo, int B, int H, int W, int C, int upsample, void* stream);
/* rqb200_dbg_vae_attn: the core of the VAE's AttnBlock: qkv [B, HW, 3C] (q | k | v per pixel) -> out [B, HW, C] = softmax over the HW
 *   keys of (q k^T * float(1 / sqrt(C))) v, single head.  RQB200_EINVAL, with nothing launched, when the C + HW floats of the query
 *   and its scores do not fit in shared memory beside the kernel's static shared memory within 48 KB (C + HW > about 12000). */
int rqb200_dbg_vae_attn(const float* qkv, float* out, int B, int HW, int C, void* stream);
/* rqb200_dbg_vae_attn_tc: the same attention on the tensor-core kernel the fast tier runs on maps past 1024 tokens (fp16 operands,
 *   fp32 scores, softmax and accumulators; no shared-memory limit on HW).  C must be 128, 256, 384 or 512 (RQB200_EINVAL). */
int rqb200_dbg_vae_attn_tc(const float* qkv, float* out, int B, int HW, int C, void* stream);

/* The Inception engine's kernels (csrc/inception_engine.cu), one launch each through the launcher the engine calls.  Maps are NHWC f32.
 * rqb200_dbg_inception_conv: conv + bias + ReLU of X [B, H, W, Cin] with Wt OHWI [Cout, kh, kw, Cin] f32 (BatchNorm already folded),
 *   zero padding pad_h rows above and below, pad_w columns left and right, stride `stride`; output pixel m's channel n goes to
 *   out[m * ldy + yoff + n] (nothing else is written), Ho = (H + 2 pad_h - kh) / stride + 1, Wo alike. */
int rqb200_dbg_inception_conv(const float* X, const float* Wt, const float* bias, float* out, int B, int H, int W, int Cin, int Cout,
                              int kh, int kw, int pad_h, int pad_w, int stride, int ldy, int yoff, void* stream);
/* rqb200_dbg_inception_conv_tc: the fast tier's conv (csrc/conv_tc.cu inc_conv_tc_kernel) with the same geometry and output placement:
 *   X16 / X16lo NHWC [B, H, W, Cin] fp16 hi / lo, W16 / W16lo OHWI [Cout, kh, kw, Cin] fp16 hi / lo, Cin % 8 == 0, Cout, ldy and yoff
 *   multiples of 16, stride 1 or 2; ReLU(A_hi W_hi + A_lo W_hi + A_hi W_lo + bias) to out (fp32, nullable) and its fp16 hi / lo to
 *   out_hi / out_lo (both or neither), at out[m * ldy + yoff + n]. */
int rqb200_dbg_inception_conv_tc(const void* X16, const void* X16lo, const void* W16, const void* W16lo, const float* bias, float* out,
                                 void* out_hi, void* out_lo, int B, int H, int W, int Cin, int Cout, int kh, int kw, int pad_h, int pad_w,
                                 int stride, int ldy, int yoff, void* stream);
/* rqb200_dbg_inception_input: x NCHW [B, 3, H, W] -> y NHWC [B, 299, 299, 3] (resize) or [B, H, W, 3], then 2 v - 1 when normalize. */
int rqb200_dbg_inception_input(const float* x, float* y, int B, int H, int W, int resize, int normalize, void* stream);
/* rqb200_dbg_inception_pool: 3x3 pool of X [B, H, W, C] with stride and pad (0 | 1) into channels [yoff, yoff + C) of rows of ldy
 *   floats; mode 0 max (padding acts as -inf), 1 average over the in-map pixels (count_include_pad=False). */
int rqb200_dbg_inception_pool(int mode, const float* X, float* Y, int B, int H, int W, int C, int stride, int pad, int ldy, int yoff,
                              void* stream);
/* rqb200_dbg_inception_gap: Y [B, C] = the mean of X [B, HW, C] over HW. */
int rqb200_dbg_inception_gap(const float* X, float* Y, int B, int HW, int C, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* RQB200_H */
