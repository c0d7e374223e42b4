// P1 -- residual-quantisation nearest-codeword search, fused over all D depths in ONE launch.
//
// Replaces (reference, rqvae/models/rqvae/quantizations.py): VQEmbedding.compute_distances :43-62 (addmm),
// find_nearest_embedding :64-69 (argmin, first index wins ties), embed :144-146 (gather) and the depth loop of
// RQBottleneck.quantize :237-271 (r -= q ; agg += q ; clone) -- 4x(addmm+argmin+gather) + 3 elementwise passes + the
// materialised [N,K] distance matrix become one kernel whose only HBM traffic is x in, codes/aggregates out.
//
// Layout / schedule (DESIGN.md "P1"): one CTA owns TN=32 residual vectors for the whole depth loop; they live in
// shared memory (padded pitch) and never go back to HBM between depths.  The K x 256 fp32 codebook (16 MB at
// K=16384: L2 resident, not SMEM resident) is streamed through a 2-stage shared-memory ring of TK=64-row tiles by
// TMA bulk copies (cp.async.bulk + mbarrier complete_tx; one 1 KB copy per codeword row so that rows land on a
// padded 1040 B pitch -> conflict-free 128-bit LDS).  The prefetch of the next tile -- including the first tile of
// the NEXT depth, which does not depend on this depth's argmin -- is always in flight while the FFMA micro-kernel
// (2 vectors x 4 codewords per thread, float4 along C) runs.  Distances are ||x||^2 + ||e||^2 - 2 x.e in fp32 exactly
// as the reference forms them; argmin keeps the first index on ties (strict < inside a thread visiting k in
// increasing order, (dist,idx)-lexicographic shuffles across threads).  Bound: FP32 FFMA (2*N*K*C*D flop), not HBM
// (SURVEY.md finding 4); the HBM figure is reported as well because the north star asks for it.
#include <cstdlib>

#include "kernels.h"

namespace rqb {

constexpr int RQ_C = 256;        // code embedding dim (quantizations.py:181)
constexpr int RQ_TN = 32;        // residual vectors per CTA
constexpr int RQ_TK = 64;        // codewords per tile
constexpr int RQ_PITCH = 260;    // floats per smem row (1040 B: 16 B aligned, breaks the 1 KB bank period)
constexpr int RQ_THREADS = 256;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE;\n"
        "bra WAIT_LOOP;\n"
        "DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

struct RqSmem {
    float resid[RQ_TN][RQ_PITCH];
    float tile[2][RQ_TK][RQ_PITCH];
    float en[2][RQ_TK];
    float xn[RQ_TN];
    int win[RQ_TN];
    uint64_t bar[2];
};

__global__ void __launch_bounds__(RQ_THREADS, 1)
rq_quantize_kernel(const float* __restrict__ x, const RqTables tabs, int64_t N, int D, int64_t* __restrict__ codes,
                   float* __restrict__ quant_list, float* __restrict__ resid_out) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    RqSmem& s = *reinterpret_cast<RqSmem*>(smem_raw);
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int tx = t & 15, ty = t >> 4;
    const int64_t n0 = (int64_t)blockIdx.x * RQ_TN;
    const int nvalid = (int)min((int64_t)RQ_TN, N - n0);

    if (t == 0) {
        mbar_init(&s.bar[0], 1);
        mbar_init(&s.bar[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // residual tile <- x (zero padded)
    for (int i = t; i < RQ_TN * (RQ_C / 4); i += RQ_THREADS) {
        int v = i / (RQ_C / 4), c4 = i % (RQ_C / 4);
        float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
        if (v < nvalid) val = *reinterpret_cast<const float4*>(x + (n0 + v) * RQ_C + c4 * 4);
        *reinterpret_cast<float4*>(&s.resid[v][c4 * 4]) = val;
    }
    __syncthreads();

    auto issue = [&](int depth, int tl, int slot) {   // warp 0 only: stream tile tl of depth's codebook into ring slot `slot`
        const int ti = tabs.of(depth);
        const float* cb = tabs.cb[ti];
        int k0 = tl * RQ_TK, rows = min(RQ_TK, tabs.K[ti] - k0);
        if (lane == 0) mbar_expect_tx(&s.bar[slot], (uint32_t)rows * RQ_C * 4);
        __syncwarp();
        for (int r = lane; r < rows; r += 32)
            bulk_g2s(&s.tile[slot][r][0], cb + (int64_t)(k0 + r) * RQ_C, RQ_C * 4, &s.bar[slot]);
    };

    auto norms_x = [&]() {       // ||r||^2 per vector: warp w -> vectors 4w..4w+3
#pragma unroll
        for (int i = 0; i < 4; i++) {
            int v = warp * 4 + i;
            float a = 0.f;
#pragma unroll
            for (int c = lane; c < RQ_C; c += 32) a = fmaf(s.resid[v][c], s.resid[v][c], a);
            a = warp_sum(a);
            if (lane == 0) s.xn[v] = a;
        }
    };

    if (warp == 0) issue(0, 0, 0);
    norms_x();
    float agg[RQ_TN];            // thread t owns channel t of every vector's aggregate
#pragma unroll
    for (int v = 0; v < RQ_TN; v++) agg[v] = 0.f;
    __syncthreads();

    float best_d[2] = {INFINITY, INFINITY};
    int best_k[2] = {0x7fffffff, 0x7fffffff};
    uint32_t phase[2] = {0u, 0u};
    const int v0 = ty * 2;

    // tiles are visited depth by depth; each depth has its own table and tile count
    for (int it = 0, depth = 0, tl = 0; depth < D; it++) {
        const int slot = it & 1;
        const int ti = tabs.of(depth), K = tabs.K[ti], ntiles = (K + RQ_TK - 1) / RQ_TK;
        const float* cb = tabs.cb[ti];
        if (warp == 0) {          // the next tile; the next depth's first tile does not depend on this depth's argmin
            if (tl + 1 < ntiles) issue(depth, tl + 1, slot ^ 1);
            else if (depth + 1 < D) issue(depth + 1, 0, slot ^ 1);
        }
        mbar_wait(&s.bar[slot], phase[slot]);
        phase[slot] ^= 1u;
        const int k0 = tl * RQ_TK, rows = min(RQ_TK, K - k0);
        {   // ||e||^2 of this tile: 4 lanes per codeword row
            int r = t >> 2, part = t & 3;
            float a = 0.f;
            if (r < rows) {
                const float* row = &s.tile[slot][r][part * 64];
#pragma unroll 16
                for (int c = 0; c < 64; c++) a = fmaf(row[c], row[c], a);
            }
            a += __shfl_xor_sync(0xffffffffu, a, 1);
            a += __shfl_xor_sync(0xffffffffu, a, 2);
            if (part == 0) s.en[slot][r] = a;
        }
        float acc[2][4];
#pragma unroll
        for (int i = 0; i < 2; i++)
#pragma unroll
            for (int j = 0; j < 4; j++) acc[i][j] = 0.f;
#pragma unroll 4
        for (int c4 = 0; c4 < RQ_C / 4; c4++) {
            float4 r4[2], e4[4];
#pragma unroll
            for (int i = 0; i < 2; i++) r4[i] = *reinterpret_cast<const float4*>(&s.resid[v0 + i][c4 * 4]);
#pragma unroll
            for (int j = 0; j < 4; j++) e4[j] = *reinterpret_cast<const float4*>(&s.tile[slot][tx + 16 * j][c4 * 4]);
#pragma unroll
            for (int i = 0; i < 2; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    acc[i][j] = fmaf(r4[i].x, e4[j].x, acc[i][j]);
                    acc[i][j] = fmaf(r4[i].y, e4[j].y, acc[i][j]);
                    acc[i][j] = fmaf(r4[i].z, e4[j].z, acc[i][j]);
                    acc[i][j] = fmaf(r4[i].w, e4[j].w, acc[i][j]);
                }
        }
        __syncthreads();   // en[] visible
#pragma unroll
        for (int j = 0; j < 4; j++) {
            int kk = tx + 16 * j;
            if (kk < rows) {
                float en = s.en[slot][kk];
#pragma unroll
                for (int i = 0; i < 2; i++) {
                    float dist = fmaf(-2.0f, acc[i][j], s.xn[v0 + i] + en);   // (xn + en) + (-2)*(x.e), quantizations.py:55-60
                    if (dist < best_d[i]) { best_d[i] = dist; best_k[i] = k0 + kk; }
                }
            }
        }
        __syncthreads();   // every thread is done with ring slot `slot` (and en[slot]) -> may be refilled at it+1

        if (tl == ntiles - 1) {   // ---- end of one depth: argmin across the 16 tx lanes, then residual update
#pragma unroll
            for (int i = 0; i < 2; i++) {
#pragma unroll
                for (int o = 8; o > 0; o >>= 1) {
                    float od = __shfl_xor_sync(0xffffffffu, best_d[i], o);
                    int ok = __shfl_xor_sync(0xffffffffu, best_k[i], o);
                    if (od < best_d[i] || (od == best_d[i] && ok < best_k[i])) { best_d[i] = od; best_k[i] = ok; }
                }
                if (tx == 0) {
                    int kw = best_k[i] == 0x7fffffff ? 0 : best_k[i];   // all-NaN row: torch.argmin would return a NaN slot; we pin 0
                    s.win[v0 + i] = kw;
                    if (v0 + i < nvalid) codes[(n0 + v0 + i) * D + depth] = (int64_t)kw;
                }
                best_d[i] = INFINITY;
                best_k[i] = 0x7fffffff;
            }
            __syncthreads();
#pragma unroll
            for (int v = 0; v < RQ_TN; v++) {
                float q = __ldg(cb + (int64_t)s.win[v] * RQ_C + t);
                s.resid[v][t] -= q;                                         // residual_feature.sub_(quant)   :264
                agg[v] += q;                                                // aggregated_quants.add_(quant)  :265
                if (quant_list != nullptr && v < nvalid)
                    quant_list[((int64_t)depth * N + n0 + v) * RQ_C + t] = agg[v];   // quant_list.append(agg.clone()) :267
            }
            __syncthreads();
            if (depth + 1 < D) norms_x();
            __syncthreads();
            depth++;
            tl = 0;
        } else {
            tl++;
        }
    }
    if (resid_out != nullptr) {
        for (int v = 0; v < nvalid; v++) resid_out[(n0 + v) * RQ_C + t] = s.resid[v][t];
    }
}

template <bool SUM>
__global__ void rq_embed_kernel(const int64_t* __restrict__ codes, const RqTables tabs, int64_t N, int D, int C,
                                float* __restrict__ out) {
    // one CTA (C/4 threads, float4 each) per vector; SUM: cat(D rows).sum(-2) in depth order (quantizations.py:308).
    // Depth d reads table tabs.of(d).
    int64_t n = blockIdx.x;
    int c4 = threadIdx.x;
    if (c4 * 4 >= C) return;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int d = 0; d < D; d++) {
        const int ti = tabs.of(d), K = tabs.K[ti];
        int64_t k = codes[n * D + d];
        k = k < 0 ? 0 : (k >= K ? K - 1 : k);
        float4 e = __ldg(reinterpret_cast<const float4*>(tabs.cb[ti] + k * C) + c4);
        if (SUM) {
            acc.x += e.x; acc.y += e.y; acc.z += e.z; acc.w += e.w;
        } else {
            reinterpret_cast<float4*>(out + (n * D + d) * C)[c4] = e;
        }
    }
    if (SUM) reinterpret_cast<float4*>(out + n * C)[c4] = acc;
}

// RQBottleneck.get_soft_codes' inner step (quantizations.py:381-383): for every residual vector r, all K distances
// d_k = (||r||^2 + ||e_k||^2) - 2 r.e_k (the reference's addmm form) and soft = softmax(-d / temp) over the codebook.
// Not a hot path (stage-2 soft targets): one CTA per vector, warp <-> codeword (coalesced 1 KB row reads out of L2), the K
// negated-scaled distances staged in shared memory for the softmax.  logits_out (nullable) receives -d/temp itself (the
// stochastic variant draws argmax(softmax(logits)/q) from it with rqb200_sample_logits).
__global__ void __launch_bounds__(256)
rq_soft_kernel(const float* __restrict__ r, const float* __restrict__ cb, int K, int C, float inv_temp, float* __restrict__ soft,
               float* __restrict__ logits_out) {
    extern __shared__ float rs_smem[];          // r[C] | z[K]
    __shared__ float red[33];
    float* rv = rs_smem;
    float* z = rs_smem + C;
    const int n = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
    float rn = 0.f;
    for (int c = t; c < C; c += 256) {
        const float v = r[(int64_t)n * C + c];
        rv[c] = v;
        rn = fmaf(v, v, rn);
    }
    rn = block_sum(rn, red);                     // ||r||^2 (all threads)
    __syncthreads();
    for (int k = warp; k < K; k += 8) {
        const float* e = cb + (int64_t)k * C;
        float dot = 0.f, en = 0.f;
        for (int c = lane * 4; c < C; c += 128) {
            const float4 ev = *reinterpret_cast<const float4*>(e + c);
            const float4 xv = *reinterpret_cast<const float4*>(rv + c);
            dot = fmaf(xv.x, ev.x, dot); dot = fmaf(xv.y, ev.y, dot); dot = fmaf(xv.z, ev.z, dot); dot = fmaf(xv.w, ev.w, dot);
            en = fmaf(ev.x, ev.x, en); en = fmaf(ev.y, ev.y, en); en = fmaf(ev.z, ev.z, en); en = fmaf(ev.w, ev.w, en);
        }
        dot = warp_sum(dot);
        en = warp_sum(en);
        if (lane == 0) z[k] = -(fmaf(-2.0f, dot, rn + en)) * inv_temp;
    }
    __syncthreads();
    float m = -INFINITY;
    for (int k = t; k < K; k += 256) m = fmaxf(m, z[k]);
    m = block_max(m, red);
    float sum = 0.f;
    for (int k = t; k < K; k += 256) sum += expf(z[k] - m);
    sum = block_sum(sum, red);
    const float inv = 1.0f / sum;
    for (int k = t; k < K; k += 256) {
        const float zk = z[k];
        soft[(int64_t)n * K + k] = expf(zk - m) * inv;
        if (logits_out) logits_out[(int64_t)n * K + k] = zk;
    }
}

int launch_rq_soft(const float* r, const float* cb, int64_t N, int K, int C, float temp, float* soft, float* logits_out,
                   cudaStream_t st) {
    if (N < 0 || K <= 0 || C <= 0 || C % 4 != 0 || !(temp > 0.f)) return fail(RQB200_EINVAL, "rq_soft_codes: bad shape / temperature");
    if (N == 0) return 0;
    const size_t smem = (size_t)(C + K) * sizeof(float);
    if (smem > 200 * 1024) return fail(RQB200_EINVAL, "rq_soft_codes: codebook too large for the shared-memory staging (K + C <= 51200)");
    RQB_ENSURE_SMEM(200 * 1024, rq_soft_kernel);
    rq_soft_kernel<<<(unsigned)N, 256, smem, st>>>(r, cb, K, C, 1.0f / temp, soft, logits_out);
    return check_launch("rq_soft_codes");
}

int make_rq_tables(RqTables* out, const float* const* cb_host, const int32_t* K_host, int n) {
    if (!cb_host || !K_host || n < 1 || n > RQ_MAX_TABLES) return fail(RQB200_EINVAL, "rq tables: need 1..16 tables");
    *out = RqTables{};
    out->n = n;
    for (int i = 0; i < n; i++) {
        if (!cb_host[i] || K_host[i] <= 0) return fail(RQB200_EINVAL, "rq tables: null table or K <= 0");
        out->cb[i] = cb_host[i];
        out->K[i] = K_host[i];
    }
    return 0;
}

int launch_rq_embed(const int64_t* codes, const RqTables& tabs, int64_t N, int D, int C, float* out, bool sum, cudaStream_t st) {
    if (C % 4 != 0 || C > 4096 || N < 0 || D <= 0) return fail(RQB200_EINVAL, "rq_embed: bad shape");
    if (tabs.n != 1 && tabs.n != D) return fail(RQB200_EINVAL, "rq_embed: need one table or one per depth");
    if (N == 0) return 0;
    if (sum)
        rq_embed_kernel<true><<<(unsigned)N, C / 4, 0, st>>>(codes, tabs, N, D, C, out);
    else
        rq_embed_kernel<false><<<(unsigned)N, C / 4, 0, st>>>(codes, tabs, N, D, C, out);
    return check_launch("rq_embed");
}

// form: 0 = pick (the 8x8-register-tile cluster kernel of rq_search2.cu whenever the shape allows: 3.7 vs 7.6 ms at N = 4096,
// K = 16384; bit-identical results), 1 = this file's 2x4-tile kernel, 2 = rq_search2.cu or fail
int launch_rq_quantize(const float* x, const RqTables& tabs, int64_t N, int C, int D, int64_t* codes, float* quant_list,
                       float* resid_out, cudaStream_t st, int form) {
    if (C != RQ_C) return fail(RQB200_EINVAL, "rq_quantize: C must be 256");
    if (N < 0 || D <= 0) return fail(RQB200_EINVAL, "rq_quantize: bad shape");
    if (tabs.n != 1 && tabs.n != D) return fail(RQB200_EINVAL, "rq_quantize: need one codebook or one per depth");
    if (N == 0) return 0;   // empty input: nothing to do (reference returns empty tensors)
    if (form != 1 && rq_quantize2_supported(N, tabs, C)) return launch_rq_quantize2(x, tabs, N, C, D, codes, quant_list, resid_out, st);
    if (form == 2) return fail(RQB200_EINVAL, "rq_quantize: shape not supported by the cluster kernel");
    RQB_ENSURE_SMEM(sizeof(RqSmem), rq_quantize_kernel);
    unsigned grid = (unsigned)ceil_div(N, RQ_TN);
    rq_quantize_kernel<<<grid, RQ_THREADS, sizeof(RqSmem), st>>>(x, tabs, N, D, codes, quant_list, resid_out);
    return check_launch("rq_quantize");
}

}  // namespace rqb

static int rq_quantize_entry(int form, const float* x, const float* const* cb_host, const int32_t* K_host, int n, int64_t N, int C,
                             int D, int64_t* codes, float* quant_list, float* residual_out, void* stream) {
    rqb::RqTables tabs;
    RQB_TRY(rqb::make_rq_tables(&tabs, cb_host, K_host, n));
    return rqb::launch_rq_quantize(x, tabs, N, C, D, codes, quant_list, residual_out, (cudaStream_t)stream, form);
}
static int rq_embed_entry(const int64_t* codes, const float* const* cb_host, const int32_t* K_host, int n, int64_t N, int D, int C,
                          float* out, bool sum, void* stream) {
    rqb::RqTables tabs;
    RQB_TRY(rqb::make_rq_tables(&tabs, cb_host, K_host, n));
    return rqb::launch_rq_embed(codes, tabs, N, D, C, out, sum, (cudaStream_t)stream);
}

extern "C" {
int rqb200_rq_quantize(const float* x, const float* codebook, int64_t N, int K, int C, int D, int64_t* codes,
                       float* quant_list, float* residual_out, void* stream) {
    return rq_quantize_entry(0, x, &codebook, &K, 1, N, C, D, codes, quant_list, residual_out, stream);
}
int rqb200_rq_quantize_depthwise(const float* x, const float* const* codebooks_host, const int32_t* K_host, int64_t N, int C, int D,
                                 int64_t* codes, float* quant_list, float* residual_out, void* stream) {
    return rq_quantize_entry(0, x, codebooks_host, K_host, D, N, C, D, codes, quant_list, residual_out, stream);
}
int rqb200_dbg_rq_quantize(int form, const float* x, const float* codebook, int64_t N, int K, int C, int D, int64_t* codes,
                           float* quant_list, float* residual_out, void* stream) {
    return rq_quantize_entry(form, x, &codebook, &K, 1, N, C, D, codes, quant_list, residual_out, stream);
}
int rqb200_dbg_rq_quantize_depthwise(int form, const float* x, const float* const* codebooks_host, const int32_t* K_host, int64_t N,
                                     int C, int D, int64_t* codes, float* quant_list, float* residual_out, void* stream) {
    return rq_quantize_entry(form, x, codebooks_host, K_host, D, N, C, D, codes, quant_list, residual_out, stream);
}
int rqb200_rq_soft_codes(const float* residual, const float* codebook, int64_t N, int K, int C, float temp, float* soft_out,
                         float* logits_out, void* stream) {
    return rqb::launch_rq_soft(residual, codebook, N, K, C, temp, soft_out, logits_out, (cudaStream_t)stream);
}
int rqb200_rq_embed_sum(const int64_t* codes, const float* codebook, int64_t N, int D, int K, int C, float* out,
                        void* stream) {
    return rq_embed_entry(codes, &codebook, &K, 1, N, D, C, out, true, stream);
}
int rqb200_rq_embed_depth(const int64_t* codes, const float* codebook, int64_t N, int D, int K, int C, float* out,
                          void* stream) {
    return rq_embed_entry(codes, &codebook, &K, 1, N, D, C, out, false, stream);
}
int rqb200_rq_embed_sum_depthwise(const int64_t* codes, const float* const* codebooks_host, const int32_t* K_host, int64_t N, int D,
                                  int C, float* out, void* stream) {
    return rq_embed_entry(codes, codebooks_host, K_host, D, N, D, C, out, true, stream);
}
int rqb200_rq_embed_depth_depthwise(const int64_t* codes, const float* const* codebooks_host, const int32_t* K_host, int64_t N,
                                    int D, int C, float* out, void* stream) {
    return rq_embed_entry(codes, codebooks_host, K_host, D, N, D, C, out, false, stream);
}
}
