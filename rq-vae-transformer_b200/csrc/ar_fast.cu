// P3 "fast" tier -- the cached AR step as a PDL-chained, CUDA-graph-replayed sequence of sm_90a kernels.
//
// Same semantics as ar_engine.cu's exact tier (reference: transformers.py:190-369, attentions.py:60-142), different
// arithmetic class: 16-bit weights / activations / KV cache on wgmma (gemm_tc.cu) -- fp16 by default, the reference's own
// autocast class (transformers.py:114,206; main_sampling_fid.py:216), bf16 on request -- fp32 accumulation, fp32 residual
// stream, fp32 LayerNorm / softmax / sampler.  RQB200_E4M3: E4M3 weights with fp32 row scales on the weight streamer's E4M3 form
// (gemm_tc_kernel<BN, GT_E4M3>) in every GEMM, fp16 activations / KV cache; everything else as with fp16.
//
// One transformer block on the single new token of every batch row (M = batch rows):
//
//     ln_reduce  x += bias_prev + sum_s partial_prev[s] ; xn = LN(x)     <- fused split-K reduction + residual
//     gemm_tc    qkv partials = Wqkv . xn                                 (split-K, 144 CTAs)
//     attn_fast  q,k,v = sum partials + bias ; append k,v to the cache ; softmax(q k^T/8) v -> att
//     gemm_tc    proj partials = Wproj . att
//     ln_reduce  x += bproj + sum partials ; xn = LN2(x)
//     gemm_tc    fc1 partials ; act_reduce h = gelu(sum + b1)
//     gemm_tc    fc2 partials = W2 . h
//
// Every launch is one all-to-all exchange between the SMs; the step is bound by the latency of these dependent exchanges before
// it is bound by HBM.  Forms with fewer LAUNCHES but the same number of EXCHANGES (a persistent megakernel with grid barriers,
// split-K reduced inside the GEMM behind an arrival counter) pay the same per exchange and are not kept in the tree.
//
// Every kernel starts with griddepcontrol.launch_dependents and reads upstream data only after griddepcontrol.wait, so
// the NEXT kernel's prologue -- for the GEMMs: filling the shared-memory ring with weight tiles -- overlaps this one.
// Position-dependent scalars (sequence index, spatial index, token counter) live in a device-side StepState that the
// last kernel of each graph advances, so a handful of captured graphs (cond-token body step, code-token body step, head
// steps + sampling; for rqb200_ar_step one head depth without sampling) are replayed for all positions without host involvement.
//
// The prefix (cond tokens, and on a start_loc resume the code tokens before it) is prefilled in ONE pass of M = B*T row
// GEMMs + a causal attention kernel that writes the KV cache (reference: transformers.py:237-239, attentions.py:60-104 with
// Tnew > 1); the token-by-token replay of the single-step graph remains available (flag) and is the prefill's oracle.  A masked
// sample (keep / sampled) runs the head graph at sampled positions only and appends each run of kept positions' code tokens to the
// body cache with the same batched pass at the run's sequence offset.
#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "kernels.h"
#include "tc_common.cuh"

namespace rqb {

// diagnostic stage trace: 4 globaltimer stamps per launch written by CTA 0 (entry, dependency resolved, mid, done)
#define TR_IN(tr)  do { if ((tr) != nullptr && blockIdx.x == 0 && threadIdx.x == 0) (tr)[0] = tc::gtimer(); } while (0)
#define TR_DEP(tr) do { if ((tr) != nullptr && blockIdx.x == 0 && threadIdx.x == 0) (tr)[1] = tc::gtimer(); } while (0)
#define TR_OUT(tr) do { if ((tr) != nullptr && blockIdx.x == 0 && threadIdx.x == 0) { (tr)[2] = tc::gtimer(); (tr)[3] = (tr)[2]; } } while (0)

// ------------------------------------------------------------------------------------------------ kernels
// The per-block small vectors (biases, LayerNorm parameters: ~80 KB per block, read once per token) are DRAM misses -- 2.8 GB of
// weights and the KV cache pass through L2 between two uses -- and each sits on a stage's critical path.  LN1 of block l therefore
// asks L2 for block l+1's.
struct PrefetchList {
    const void* p[8];
    uint32_t bytes[8];
    int n;
};

// x_out = x_in + bias + sum_s partial[s] (+ extra row) ; xn = LayerNorm(x_out) in 16-bit.  One CTA per row.
// (instantiated as <384, 3> only)
template <int THREADS, int NCH>
__global__ void __launch_bounds__(THREADS)
ln_reduce_kernel(const float* __restrict__ x_in, const float* __restrict__ partial, int S, const float* __restrict__ bias,
                 const float* __restrict__ extra, float* __restrict__ x_out, const float* __restrict__ g,
                 const float* __restrict__ be, h16* __restrict__ xn, int B, int E, int bf, long long* tr, PrefetchList pf) {
    // each thread owns up to NCH float4 chunks of the row (E <= THREADS*4*NCH); every load is issued before the first dependent add and
    // the row stays in registers between the statistics and the normalisation
    __shared__ float red[33];
    tc::pdl_launch_dependents();
    TR_IN(tr);
    if (blockIdx.x == 0 && threadIdx.x < pf.n) tc::bulk_prefetch_l2(pf.p[threadIdx.x], pf.bytes[threadIdx.x]);   // (parameters: no dependency)
    tc::pdl_wait();
    TR_DEP(tr);
    const int b = blockIdx.x;
    const int E4 = E >> 2;
    const int S12 = S < 12 ? S : 12;
    float4 v[NCH], gg[NCH], bb[NCH];
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < NCH; k++) {
        const int e4 = threadIdx.x + k * THREADS;
        v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (e4 < E4) {
            float4 pr[12];
            if (xn) { gg[k] = reinterpret_cast<const float4*>(g)[e4]; bb[k] = reinterpret_cast<const float4*>(be)[e4]; }
#pragma unroll
            for (int i = 0; i < 12; i++)
                if (i < S12) pr[i] = reinterpret_cast<const float4*>(partial + ((int64_t)i * B + b) * E)[e4];
            if (x_in) v[k] = reinterpret_cast<const float4*>(x_in + (int64_t)b * E)[e4];
            if (bias) { float4 t = reinterpret_cast<const float4*>(bias)[e4]; v[k].x += t.x; v[k].y += t.y; v[k].z += t.z; v[k].w += t.w; }
#pragma unroll
            for (int i = 0; i < 12; i++)
                if (i < S12) { v[k].x += pr[i].x; v[k].y += pr[i].y; v[k].z += pr[i].z; v[k].w += pr[i].w; }
            for (int i = 12; i < S; i++) {
                float4 p0 = reinterpret_cast<const float4*>(partial + ((int64_t)i * B + b) * E)[e4];
                v[k].x += p0.x; v[k].y += p0.y; v[k].z += p0.z; v[k].w += p0.w;
            }
            if (extra) { float4 t = reinterpret_cast<const float4*>(extra)[e4]; v[k].x += t.x; v[k].y += t.y; v[k].z += t.z; v[k].w += t.w; }
            if (x_out) reinterpret_cast<float4*>(x_out + (int64_t)b * E)[e4] = v[k];
            s += (v[k].x + v[k].y) + (v[k].z + v[k].w);
        }
    }
    if (xn) {
        const float mean = block_sum(s, red) / (float)E;
        if (tr != nullptr && blockIdx.x == 0 && threadIdx.x == 0) tr[2] = tc::gtimer();      // every load has landed, first reduction done
        float q = 0.f;
#pragma unroll
        for (int k = 0; k < NCH; k++)
            if (threadIdx.x + k * THREADS < E4) {
                const float d0 = v[k].x - mean, d1 = v[k].y - mean, d2 = v[k].z - mean, d3 = v[k].w - mean;
                q = fmaf(d0, d0, q); q = fmaf(d1, d1, q); q = fmaf(d2, d2, q); q = fmaf(d3, d3, q);
            }
        const float rstd = rsqrtf(block_sum(q, red) / (float)E + 1e-5f);
#pragma unroll
        for (int k = 0; k < NCH; k++) {
            const int e4 = threadIdx.x + k * THREADS;
            if (e4 < E4) {
                uint2 pk;
                pk.x = pack_h16x2((v[k].x - mean) * rstd * gg[k].x + bb[k].x, (v[k].y - mean) * rstd * gg[k].y + bb[k].y, bf);
                pk.y = pack_h16x2((v[k].z - mean) * rstd * gg[k].z + bb[k].z, (v[k].w - mean) * rstd * gg[k].w + bb[k].w, bf);
                reinterpret_cast<uint2*>(xn + (int64_t)b * E)[e4] = pk;
            }
        }
        if (tr != nullptr && blockIdx.x == 0 && threadIdx.x == 0) tr[3] = tc::gtimer();
    } else {
        TR_OUT(tr);
    }
}

// The batched passes' LayerNorm (prefill / teacher-forced forward: thousands of rows, no split-K partials): one WARP per row, the
// row in registers between the statistics and the normalisation, rows grid-strided over 8-warp CTAs.  (ln_reduce_kernel's
// one-384-thread-CTA-per-row form is built for 64 rows on 64 SMs; on 4096+ rows it ran at a tenth of the HBM rate.)
// x_out (nullable) = x_in (+ extra row); xn (nullable) = LayerNorm(x) in 16-bit.  NV = float4 chunks per lane (E <= 128 * NV).
template <int NV>
__global__ void __launch_bounds__(256)
ln_rows_kernel(const float* __restrict__ x_in, const float* __restrict__ extra, float* __restrict__ x_out, const float* __restrict__ g,
               const float* __restrict__ be, h16* __restrict__ xn, int64_t M, int E, int bf) {
    tc::pdl_launch_dependents();
    tc::pdl_wait();
    const int lane = threadIdx.x & 31;
    const int E4 = E >> 2;
    for (int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5); row < M; row += (int64_t)gridDim.x * 8) {
        const float4* xr = reinterpret_cast<const float4*>(x_in + row * E);
        float4 v[NV];
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < NV; k++) {
            const int e4 = lane + 32 * k;
            v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (e4 < E4) v[k] = xr[e4];
        }
#pragma unroll
        for (int k = 0; k < NV; k++) {
            const int e4 = lane + 32 * k;
            if (e4 < E4) {
                if (extra) { const float4 t = reinterpret_cast<const float4*>(extra)[e4]; v[k].x += t.x; v[k].y += t.y; v[k].z += t.z; v[k].w += t.w; }
                if (x_out) reinterpret_cast<float4*>(x_out + row * E)[e4] = v[k];
                s += (v[k].x + v[k].y) + (v[k].z + v[k].w);
            }
        }
        if (xn) {
            const float mean = warp_sum(s) / (float)E;
            float q = 0.f;
#pragma unroll
            for (int k = 0; k < NV; k++)
                if (lane + 32 * k < E4) {
                    const float d0 = v[k].x - mean, d1 = v[k].y - mean, d2 = v[k].z - mean, d3 = v[k].w - mean;
                    q = fmaf(d0, d0, q); q = fmaf(d1, d1, q); q = fmaf(d2, d2, q); q = fmaf(d3, d3, q);
                }
            const float rstd = rsqrtf(warp_sum(q) / (float)E + 1e-5f);
#pragma unroll
            for (int k = 0; k < NV; k++) {
                const int e4 = lane + 32 * k;
                if (e4 < E4) {
                    const float4 gg = reinterpret_cast<const float4*>(g)[e4], bb = reinterpret_cast<const float4*>(be)[e4];
                    uint2 pk;
                    pk.x = pack_h16x2((v[k].x - mean) * rstd * gg.x + bb.x, (v[k].y - mean) * rstd * gg.y + bb.y, bf);
                    pk.y = pack_h16x2((v[k].z - mean) * rstd * gg.z + bb.z, (v[k].w - mean) * rstd * gg.w + bb.w, bf);
                    reinterpret_cast<uint2*>(xn + row * E)[e4] = pk;
                }
            }
        }
    }
}

// h = 16-bit(gelu(sum_s partial[s] + bias))   (only when fc1 runs split-K); 4 elements per thread, all partial loads in flight
__global__ void __launch_bounds__(256)
act_reduce_kernel(const float* __restrict__ partial, int S, const float* __restrict__ bias, h16* __restrict__ h, int B, int N, int bf,
                  long long* tr) {
    tc::pdl_launch_dependents();
    TR_IN(tr);
    tc::pdl_wait();
    TR_DEP(tr);
    const int64_t total4 = (int64_t)B * N / 4;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total4; i += (int64_t)gridDim.x * 256) {
        const int n = (int)((i * 4) % N);
        float4 pr[4];
#pragma unroll
        for (int s = 0; s < 4; s++)
            if (s < S) pr[s] = __ldcg(reinterpret_cast<const float4*>(partial + (int64_t)s * B * N) + i);
        float4 v = *reinterpret_cast<const float4*>(bias + n);
#pragma unroll
        for (int s = 0; s < 4; s++)
            if (s < S) { v.x += pr[s].x; v.y += pr[s].y; v.z += pr[s].z; v.w += pr[s].w; }
        for (int s = 4; s < S; s++) {
            float4 p = __ldcg(reinterpret_cast<const float4*>(partial + (int64_t)s * B * N) + i);
            v.x += p.x; v.y += p.y; v.z += p.z; v.w += p.w;
        }
        float r[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int k = 0; k < 4; k++) r[k] = gelu_erf(r[k]);
        uint2 pk;
        pk.x = pack_h16x2(r[0], r[1], bf);
        pk.y = pack_h16x2(r[2], r[3], bf);
        *reinterpret_cast<uint2*>(h + i * 4) = pk;
    }
    TR_OUT(tr);
}

// one warp per (b, head): reduce the split-K qkv partials (+bias), append k,v at row t of the 16-bit cache, attend.
// lane <-> dims (2*lane, 2*lane+1) for q/k/v/out everywhere: every cache row is read as ONE coalesced 128 B line per warp
// instruction (a lane-per-key row read costs 8x the L1 wavefronts); the per-key dot products are finished with a 31-shuffle
// transpose-reduce per 32 keys, after which lane j holds the score of key j.  Up to 64 K rows / 64 V rows are in flight at once
// and the V rows are requested before the softmax arithmetic.  T <= FAST_MAXT: the scores take 16 * T B of dynamic shared memory
// (32 KB at 2048, under the 48 KB default).
// (The cached rows are not read into registers ahead of griddepcontrol.wait: that is a race in the head graph, where the producer of row d-1 is a kernel of the SAME graph that a chain of
// small launches does not keep from still being in flight.)
constexpr int FAST_MAXT = 2048;          // the fast tier's longest body sequence, cond_len + H*W (a 32x32 grid behind a 1024-token prefix)

// pv[u] = this lane's partial dot product for key u (u < 32); returns the full dot product of key `lane`
__device__ __forceinline__ float af_transpose_reduce(float (&pv)[32], int lane) {
#pragma unroll
    for (int S = 16; S >= 1; S >>= 1) {
        const bool up = (lane & S) != 0;
#pragma unroll
        for (int i = 0; i < S; i++) {
            const float send = up ? pv[i] : pv[i + S];
            const float keep = up ? pv[i + S] : pv[i];
            pv[i] = keep + __shfl_xor_sync(0xffffffffu, send, S);
        }
    }
    return pv[0];
}

__global__ void __launch_bounds__(128)
attn_fast_kernel(const float* __restrict__ part, int S, const float* __restrict__ bqkv, h16* __restrict__ kc, h16* __restrict__ vc,
                 h16* __restrict__ att, int B, int E, int nh, int Tmax, const int* __restrict__ t_ptr, int t_host, int bf,
                 long long* tr) {
    extern __shared__ float af_smem[];              // ps[4][tp]
    const int tp = (Tmax + 31) & ~31;
    const int lane = threadIdx.x & 31, wq = threadIdx.x >> 5;
    float* ps = af_smem + wq * tp;
    tc::pdl_launch_dependents();
    TR_IN(tr);
    tc::pdl_wait();
    TR_DEP(tr);
    const int bh = blockIdx.x * 4 + wq;
    if (bh < B * nh) {
    const int b = bh / nh, h = bh % nh;
    const int t = t_ptr ? *t_ptr : t_host;
    h16* kb = kc + ((int64_t)(b * nh + h) * Tmax) * 64;
    h16* vb = vc + ((int64_t)(b * nh + h) * Tmax) * 64;
    const int c = h * 64 + 2 * lane;
    float2 q = make_float2(bqkv[c], bqkv[c + 1]);
    float2 k = make_float2(bqkv[E + c], bqkv[E + c + 1]);
    float2 v = make_float2(bqkv[2 * E + c], bqkv[2 * E + c + 1]);
#pragma unroll 4
    for (int s = 0; s < S; s++) {
        const float* p = part + ((int64_t)s * B + b) * 3 * E;
        float2 a = *reinterpret_cast<const float2*>(p + c);
        float2 bb = *reinterpret_cast<const float2*>(p + E + c);
        float2 cc = *reinterpret_cast<const float2*>(p + 2 * E + c);
        q.x += a.x; q.y += a.y; k.x += bb.x; k.y += bb.y; v.x += cc.x; v.y += cc.y;
    }
    const uint32_t k2 = pack_h16x2(k.x, k.y, bf), v2 = pack_h16x2(v.x, v.y, bf);
    *reinterpret_cast<uint32_t*>(kb + (int64_t)t * 64 + 2 * lane) = k2;
    *reinterpret_cast<uint32_t*>(vb + (int64_t)t * 64 + 2 * lane) = v2;
    // use the 16-bit-rounded q/k/v everywhere (what a later step reads back from the cache)
    const float2 qf = unpack_h16x2(pack_h16x2(q.x, q.y, bf), bf), kf = unpack_h16x2(k2, bf), vf = unpack_h16x2(v2, bf);
    const float s_new = warp_sum(qf.x * kf.x + qf.y * kf.y) * 0.125f;
    float m = s_new;
    for (int j0 = 0; j0 < t; j0 += 64) {          // scores of the cached rows: 64 coalesced row reads in flight
        uint32_t kr[64];
#pragma unroll
        for (int u = 0; u < 64; u++)
            kr[u] = (j0 + u < t) ? *reinterpret_cast<const uint32_t*>(kb + (int64_t)(j0 + u) * 64 + 2 * lane) : 0u;
#pragma unroll
        for (int half = 0; half < 2; half++) {
            if (j0 + half * 32 < t) {                                  // (warp-uniform)
                float pv[32];
#pragma unroll
                for (int u = 0; u < 32; u++) {
                    const float2 kk = unpack_h16x2(kr[half * 32 + u], bf);
                    pv[u] = fmaf(qf.y, kk.y, qf.x * kk.x);
                }
                const float sc = af_transpose_reduce(pv, lane) * 0.125f;
                const int j = j0 + half * 32 + lane;
                if (j < t) {
                    ps[j] = sc;
                    m = fmaxf(m, sc);
                }
            }
        }
    }
    // the V rows do not depend on the scores: the first 64 are requested before the softmax arithmetic
    uint32_t raw[64];
#pragma unroll
    for (int u = 0; u < 64; u++)
        raw[u] = (u < t) ? *reinterpret_cast<const uint32_t*>(vb + (int64_t)u * 64 + 2 * lane) : 0u;
    m = warp_max(m);
    if (tr != nullptr && blockIdx.x == 0 && threadIdx.x == 0) tr[2] = tc::gtimer();      // scores done
    float sum = 0.f;
    for (int j = lane; j < t; j += 32) {
        float e = __expf(ps[j] - m);
        ps[j] = e;
        sum += e;
    }
    const float e_new = __expf(s_new - m);
    sum = warp_sum(sum) + e_new;
    __syncwarp();
    const float inv = 1.0f / sum;
    float2 o = make_float2(e_new * vf.x, e_new * vf.y);
    for (int j0 = 0; j0 < t; j0 += 64) {                  // (rows added in cache order)
        if (j0 > 0) {
#pragma unroll
            for (int u = 0; u < 64; u++)
                raw[u] = (j0 + u < t) ? *reinterpret_cast<const uint32_t*>(vb + (int64_t)(j0 + u) * 64 + 2 * lane) : 0u;
        }
#pragma unroll
        for (int u = 0; u < 64; u++)
            if (j0 + u < t) {
                const float2 vv = unpack_h16x2(raw[u], bf);
                o.x = fmaf(ps[j0 + u], vv.x, o.x);
                o.y = fmaf(ps[j0 + u], vv.y, o.y);
            }
    }
    *reinterpret_cast<uint32_t*>(att + (int64_t)b * E + c) = pack_h16x2(o.x * inv, o.y * inv, bf);
    }
    if (tr != nullptr && blockIdx.x == 0 && threadIdx.x == 0) tr[3] = tc::gtimer();
}

// Four warps per (b, head) -- the body stack's form.  The cached K / V rows [0, t) are staged in shared memory by cp.async (16 B
// per request, every request of the CTA in flight at once, issued right after the dependency resolves and overlapped with the
// q/k/v split-K reduction): the whole KV read of a step is ONE memory round trip instead of two (K, then V) serialised per 64 rows
// in one warp's registers.  Rows are 128 B with the 16 B chunks XOR-swizzled by (row & 7): conflict-free for the score pass
// (a lane pair per row, 4 chunks each) and for the output pass (a warp per row, lane <-> dims (2*lane, 2*lane+1)).
// Softmax statistics go through shared memory; warp w adds the rows j = w (mod 4) in cache order and the four partial outputs
// are summed in warp order -> run-to-run deterministic.  q/k/v bits as in attn_fast_kernel (same reduction order).
// 11 CTAs per SM (40 registers, 19.6 KB at 64 rows): the 1536 (b, head) pairs of the 1.4B model at B = 64 are one wave.
constexpr int AF2_MAXROWS = 320;
static size_t attn2_smem(int rows) { return (size_t)rows * 256 + ((size_t)rows + 64 * 3 + 4 * 64 + 8) * sizeof(float); }
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__global__ void __launch_bounds__(128, 11)
attn_fast2_kernel(const float* __restrict__ part, int S, const float* __restrict__ bqkv, h16* __restrict__ kc, h16* __restrict__ vc,
                  h16* __restrict__ att, int B, int E, int nh, int Tmax, int rows, const int* __restrict__ t_ptr, int t_host, int bf,
                  long long* tr) {
    extern __shared__ __align__(128) uint8_t af2_smem[];
    uint8_t* Ks = af2_smem;                                   // [rows][128 B], chunk c of row j at ((c ^ (j & 7)) << 4)
    uint8_t* Vs = Ks + (size_t)rows * 128;
    float* ps = reinterpret_cast<float*>(Vs + (size_t)rows * 128);   // scores, then exp(score - max)
    float* qs = ps + rows;                // q, k_new, v_new (16-bit-rounded), 64 floats each
    float* kn = qs + 64;
    float* vn = kn + 64;
    float* ov = vn + 64;                  // [4][64] partial outputs
    float* red = ov + 256;                // [0..3] warp maxima, [4..7] warp sums
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    tc::pdl_launch_dependents();
    TR_IN(tr);
    tc::pdl_wait();
    TR_DEP(tr);
    const int b = blockIdx.x / nh, h = blockIdx.x % nh;
    const int t = t_ptr ? *t_ptr : t_host;
    h16* kb = kc + ((int64_t)(b * nh + h) * Tmax) * 64;
    h16* vb = vc + ((int64_t)(b * nh + h) * Tmax) * 64;
    {
        const uint32_t ks = tc::smem_u32(Ks), vs = tc::smem_u32(Vs);
        for (int i = threadIdx.x; i < t * 8; i += 128) {
            const int j = i >> 3, c = i & 7;
            const uint32_t off = (uint32_t)j * 128u + (uint32_t)((c ^ (j & 7)) << 4);
            cp_async16(ks + off, kb + (int64_t)j * 64 + c * 8);
            cp_async16(vs + off, vb + (int64_t)j * 64 + c * 8);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    // ---- q / k / v of the new token: warp 0 -> q, warp 1 -> k, warp 2 -> v (value = bias + p0 + p1 + ..., split order)
    if (w < 3) {
        const int c = h * 64 + 2 * lane;
        float2 a = make_float2(bqkv[w * E + c], bqkv[w * E + c + 1]);
#pragma unroll 4
        for (int s = 0; s < S; s++) {
            const float2 pp = *reinterpret_cast<const float2*>(part + ((int64_t)s * B + b) * 3 * E + w * E + c);
            a.x += pp.x; a.y += pp.y;
        }
        const uint32_t a2 = pack_h16x2(a.x, a.y, bf);
        const float2 af = unpack_h16x2(a2, bf);
        float* dst = w == 0 ? qs : (w == 1 ? kn : vn);
        dst[2 * lane] = af.x;
        dst[2 * lane + 1] = af.y;
        if (w == 1) *reinterpret_cast<uint32_t*>(kb + (int64_t)t * 64 + 2 * lane) = a2;
        if (w == 2) *reinterpret_cast<uint32_t*>(vb + (int64_t)t * 64 + 2 * lane) = a2;
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    const float s_new = warp_sum(qs[2 * lane] * kn[2 * lane] + qs[2 * lane + 1] * kn[2 * lane + 1]) * 0.125f;
    float m = -INFINITY;
    {
        const int half = threadIdx.x & 1;
        for (int j0 = 0; j0 < t; j0 += 64) {
            const int j = j0 + (threadIdx.x >> 1);
            float acc = 0.f;
            if (j < t) {
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    const int c = half * 4 + i;
                    const uint4 k4 = *reinterpret_cast<const uint4*>(Ks + (size_t)j * 128 + ((c ^ (j & 7)) << 4));
                    const float4 qa = *reinterpret_cast<const float4*>(qs + c * 8), qb = *reinterpret_cast<const float4*>(qs + c * 8 + 4);
                    float2 kk = unpack_h16x2(k4.x, bf);
                    acc = fmaf(qa.x, kk.x, acc); acc = fmaf(qa.y, kk.y, acc);
                    kk = unpack_h16x2(k4.y, bf);
                    acc = fmaf(qa.z, kk.x, acc); acc = fmaf(qa.w, kk.y, acc);
                    kk = unpack_h16x2(k4.z, bf);
                    acc = fmaf(qb.x, kk.x, acc); acc = fmaf(qb.y, kk.y, acc);
                    kk = unpack_h16x2(k4.w, bf);
                    acc = fmaf(qb.z, kk.x, acc); acc = fmaf(qb.w, kk.y, acc);
                }
            }
            acc += __shfl_xor_sync(0xffffffffu, acc, 1);
            acc *= 0.125f;
            if (j < t) {
                if (half == 0) ps[j] = acc;
                m = fmaxf(m, acc);
            }
        }
    }
    m = warp_max(m);
    if (lane == 0) red[w] = m;
    __syncthreads();
    m = fmaxf(fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3])), s_new);
    if (tr != nullptr && blockIdx.x == 0 && threadIdx.x == 0) tr[2] = tc::gtimer();      // scores done
    float sum = 0.f;
    for (int j = threadIdx.x; j < t; j += 128) {
        const float e = __expf(ps[j] - m);
        ps[j] = e;
        sum += e;
    }
    sum = warp_sum(sum);
    if (lane == 0) red[4 + w] = sum;
    __syncthreads();
    const float e_new = __expf(s_new - m);
    const float inv = 1.0f / ((((red[4] + red[5]) + red[6]) + red[7]) + e_new);
    float2 o = w == 0 ? make_float2(e_new * vn[2 * lane], e_new * vn[2 * lane + 1]) : make_float2(0.f, 0.f);
    for (int j = w; j < t; j += 4) {
        const uint32_t v2 = *reinterpret_cast<const uint32_t*>(Vs + (size_t)j * 128 + (((lane >> 2) ^ (j & 7)) << 4) + ((lane & 3) << 2));
        const float2 vv = unpack_h16x2(v2, bf);
        const float pj = ps[j];
        o.x = fmaf(pj, vv.x, o.x);
        o.y = fmaf(pj, vv.y, o.y);
    }
    ov[w * 64 + 2 * lane] = o.x;
    ov[w * 64 + 2 * lane + 1] = o.y;
    __syncthreads();
    if (w == 0) {
        const float ox = ((ov[2 * lane] + ov[64 + 2 * lane]) + ov[128 + 2 * lane]) + ov[192 + 2 * lane];
        const float oy = ((ov[2 * lane + 1] + ov[64 + 2 * lane + 1]) + ov[128 + 2 * lane + 1]) + ov[192 + 2 * lane + 1];
        *reinterpret_cast<uint32_t*>(att + (int64_t)b * E + h * 64 + 2 * lane) = pack_h16x2(ox * inv, oy * inv, bf);
    }
    if (tr != nullptr && blockIdx.x == 0 && threadIdx.x == 0) tr[3] = tc::gtimer();
}

// Warp-level tensor-core pieces of prefill_attn_flash_kernel: mma.sync.m16n8k16 (fp32 accumulate) and ldmatrix.x4 (plain, .trans).
template <bool BF>
__device__ __forceinline__ void pa_mma(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    if (BF)
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    else
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void pa_ldsm4(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void pa_ldsm4_t(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
constexpr int PM_ROW = 144;                           // bytes per staged row (64 x 16-bit + 16 B pad)
// Causal attention of T new tokens at sequence offset T0 in one launch (batched prefill, T0 = 0; an append to the KV cache, T0 > 0;
// teacher-forced forward, T0 = 0 and no cache) for groups of more than 8 tokens.
// qkv [M, 3E] 16-bit (bias already added by the GEMM epilogue), row of (group g, new token t) = t * G + g (token-major: the rows of one
// token are contiguous, like the single-step buffers).  New token t is sequence token T0 + t and sees keys [0, T0 + t]: keys < T0 are
// the cache rows [g][head][key][64] of kc / vc (written by earlier launches; no CTA of this one writes them), keys >= T0 are qkv's rows.
// One CTA per (query tile of 64 new tokens, group, head), query tiles launched heaviest (last) first; each of the four warps owns 16
// query rows.  K / V are read in 64-key tiles of the whole sequence (a tile may straddle T0) double-buffered through cp.async (144 B
// rows: conflict-free ldmatrix); per tile S = Q K^T on mma.sync (fp32 accumulate), the causal mask on the tiles that hold keys past
// some query row, an online softmax (running row max and sum in fp32, O rescaled between tiles), the probabilities repacked as 16-bit
// A fragments (the m16n8 accumulator pair of two adjacent key tiles IS the m16k16 A fragment) and O += P V with V through
// ldmatrix.trans.  Key tiles are visited in a fixed order: run-to-run deterministic.  When kc != NULL the CTA of query tile i writes
// the cache rows T0 + t of its tile's new tokens t (every new row exactly once).  At T0 = 0 every tile but the diagonal one is
// unmasked, as in the plain prefill.
// CAUSAL == false (the CLIP vision tower; T0 = 0, no cache): every query sees keys [0, T0 + T); the key tile that holds the last key
// masks the zero-filled rows past it explicitly (causality no longer does).
template <bool BF, bool CAUSAL = true>
__global__ void __launch_bounds__(128)
prefill_attn_flash_kernel(const h16* __restrict__ qkv, h16* __restrict__ kc, h16* __restrict__ vc, h16* __restrict__ att, int G, int T, int E,
                          int nh, int Tmax, int T0) {
    __shared__ __align__(16) uint8_t sm[5 * 64 * PM_ROW];         // Q | K[2] | V[2]
    uint8_t* Qs = sm;
    tc::pdl_launch_dependents();
    tc::pdl_wait();
    const int n_pairs = G * nh;
    const int qt = (T + 63) / 64 - 1 - (int)(blockIdx.x / n_pairs);  // heaviest query tile first
    const int pair = (int)(blockIdx.x % n_pairs);
    const int g = pair / nh, h = pair % nh;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int64_t crow0 = ((int64_t)g * nh + h) * Tmax;        // this (group, head)'s cache rows
    // tile `kt` of matrix `mat` (0 Q: new tokens; 1 K, 2 V: sequence keys, < T0 from the cache) -> dst; rows beyond the last token are
    // zeros (their scores are masked, but P V must not see NaN)
    auto load_tile = [&](int mat, int kt, uint8_t* dst) {
        const int base = mat == 0 ? 0 : T0;               // sequence index of qkv row 0 in this tile's coordinates
        for (int i = threadIdx.x; i < 64 * 8; i += 128) {
            const int r = i >> 3, c = i & 7, t = kt * 64 + r - base;
            uint8_t* d = dst + r * PM_ROW + c * 16;
            if (t < 0)
                cp_async16(tc::smem_u32(d), (mat == 1 ? kc : vc) + (crow0 + kt * 64 + r) * 64 + c * 8);
            else if (t < T)
                cp_async16(tc::smem_u32(d), qkv + ((int64_t)t * G + g) * 3 * E + mat * E + h * 64 + c * 8);
            else
                *reinterpret_cast<uint4*>(d) = make_uint4(0u, 0u, 0u, 0u);
        }
    };
    load_tile(0, qt, Qs);
    load_tile(1, 0, sm + 64 * PM_ROW);
    load_tile(2, 0, sm + 3 * 64 * PM_ROW);
    asm volatile("cp.async.commit_group;" ::: "memory");
    if (kc != nullptr) {                                  // this query tile's K / V rows -> the cache
        for (int i = threadIdx.x; i < 2 * 64 * 8; i += 128) {
            const int mat = 1 + (i >> 9), r = (i >> 3) & 63, c = i & 7, t = qt * 64 + r;
            if (t < T)
                *reinterpret_cast<uint4*>((mat == 1 ? kc : vc) + (crow0 + T0 + t) * 64 + c * 8) =
                    *reinterpret_cast<const uint4*>(qkv + ((int64_t)t * G + g) * 3 * E + mat * E + h * 64 + c * 8);
        }
    }
    const int r0 = qt * 64 + 16 * w + (lane >> 2), r1 = r0 + 8;          // new-token rows; sequence rows T0 + r0, T0 + r1
    const int q0 = T0 + r0, q1 = T0 + r1;
    // the last key tile of this query tile: the one holding its last real query's key (rows past T see keys up to it, never beyond)
    const int kt_last = CAUSAL ? (T0 + min(qt * 64 + 63, T - 1)) >> 6 : (T0 + T - 1) >> 6;
    uint32_t qa[4][4];
    float oacc[8][4];
#pragma unroll
    for (int j = 0; j < 8; j++) { oacc[j][0] = oacc[j][1] = oacc[j][2] = oacc[j][3] = 0.f; }
    float m0 = -INFINITY, m1 = -INFINITY, s0 = 0.f, s1 = 0.f;      // running max; this lane's share of the running sum
    for (int kt = 0; kt <= kt_last; kt++) {
        if (kt < kt_last) {                               // prefetch the next key tile into the other buffer
            load_tile(1, kt + 1, sm + (1 + ((kt + 1) & 1)) * 64 * PM_ROW);
            load_tile(2, kt + 1, sm + (3 + ((kt + 1) & 1)) * 64 * PM_ROW);
            asm volatile("cp.async.commit_group;" ::: "memory");
            asm volatile("cp.async.wait_group 1;" ::: "memory");
        } else {
            asm volatile("cp.async.wait_group 0;" ::: "memory");
        }
        __syncthreads();
        const uint32_t ks = tc::smem_u32(sm + (1 + (kt & 1)) * 64 * PM_ROW), vs = tc::smem_u32(sm + (3 + (kt & 1)) * 64 * PM_ROW);
        if (kt == 0) {
#pragma unroll
            for (int kk = 0; kk < 4; kk++)
                pa_ldsm4(qa[kk], tc::smem_u32(Qs) + (uint32_t)((16 * w + (lane & 15)) * PM_ROW + kk * 32 + (lane >> 4) * 16));
        }
        // ---- S = Q K^T for this warp's 16 query rows x 64 keys
        float sacc[8][4];
#pragma unroll
        for (int j = 0; j < 8; j++) { sacc[j][0] = sacc[j][1] = sacc[j][2] = sacc[j][3] = 0.f; }
#pragma unroll
        for (int kk = 0; kk < 4; kk++) {
#pragma unroll
            for (int jp = 0; jp < 4; jp++) {
                uint32_t b[4];
                pa_ldsm4(b, ks + (uint32_t)((16 * jp + (lane & 7) + ((lane >> 4) << 3)) * PM_ROW + kk * 32 + ((lane >> 3) & 1) * 16));
                pa_mma<BF>(sacc[2 * jp], qa[kk], b[0], b[1]);
                pa_mma<BF>(sacc[2 * jp + 1], qa[kk], b[2], b[3]);
            }
        }
        // ---- scale (+ causal mask where the tile holds keys past this tile's first query row), new row maxima
        const bool masked = CAUSAL ? kt * 64 + 63 > T0 + qt * 64 : kt * 64 + 63 >= T0 + T;
        // the last key a row sees: its own sequence index (causal), else the last token
        const int lim0 = CAUSAL ? q0 : T0 + T - 1, lim1 = CAUSAL ? q1 : T0 + T - 1;
        float t0 = m0, t1 = m1;
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const int c0 = kt * 64 + 8 * j + (lane & 3) * 2;
            sacc[j][0] = (!masked || c0 <= lim0) ? sacc[j][0] * 0.125f : -INFINITY;
            sacc[j][1] = (!masked || c0 + 1 <= lim0) ? sacc[j][1] * 0.125f : -INFINITY;
            sacc[j][2] = (!masked || c0 <= lim1) ? sacc[j][2] * 0.125f : -INFINITY;
            sacc[j][3] = (!masked || c0 + 1 <= lim1) ? sacc[j][3] * 0.125f : -INFINITY;
            t0 = fmaxf(t0, fmaxf(sacc[j][0], sacc[j][1]));
            t1 = fmaxf(t1, fmaxf(sacc[j][2], sacc[j][3]));
        }
        t0 = fmaxf(t0, __shfl_xor_sync(0xffffffffu, t0, 1)); t0 = fmaxf(t0, __shfl_xor_sync(0xffffffffu, t0, 2));
        t1 = fmaxf(t1, __shfl_xor_sync(0xffffffffu, t1, 1)); t1 = fmaxf(t1, __shfl_xor_sync(0xffffffffu, t1, 2));
        // Key 0 is in tile 0 and every row sees it, so t0 / t1 are finite from the first tile on (alpha of the first tile is 0).  A
        // later tile may be fully masked for some rows (an append's query tile straddles two key tiles): their max stays, alpha is 1
        // and every exp(-inf - m) is 0 -- zero weight, no NaN.
        const float a0 = __expf(m0 - t0), a1 = __expf(m1 - t1);
        m0 = t0;
        m1 = t1;
        s0 *= a0;
        s1 *= a1;
#pragma unroll
        for (int j = 0; j < 8; j++) { oacc[j][0] *= a0; oacc[j][1] *= a0; oacc[j][2] *= a1; oacc[j][3] *= a1; }
        uint32_t pa[4][4];
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const float e0 = __expf(sacc[j][0] - m0), e1 = __expf(sacc[j][1] - m0), e2 = __expf(sacc[j][2] - m1), e3 = __expf(sacc[j][3] - m1);
            s0 += e0 + e1;
            s1 += e2 + e3;
            pa[j >> 1][(j & 1) * 2] = pack_h16x2(e0, e1, BF ? 1 : 0);
            pa[j >> 1][(j & 1) * 2 + 1] = pack_h16x2(e2, e3, BF ? 1 : 0);
        }
        // ---- O += P V
#pragma unroll
        for (int kk = 0; kk < 4; kk++) {
#pragma unroll
            for (int jp = 0; jp < 4; jp++) {
                uint32_t b[4];
                pa_ldsm4_t(b, vs + (uint32_t)((16 * kk + (lane & 7) + ((lane >> 3) & 1) * 8) * PM_ROW + (2 * jp + (lane >> 4)) * 16));
                pa_mma<BF>(oacc[2 * jp], pa[kk], b[0], b[1]);
                pa_mma<BF>(oacc[2 * jp + 1], pa[kk], b[2], b[3]);
            }
        }
        __syncthreads();                                  // (this buffer is refilled by the next iteration's prefetch)
    }
    s0 += __shfl_xor_sync(0xffffffffu, s0, 1); s0 += __shfl_xor_sync(0xffffffffu, s0, 2);
    s1 += __shfl_xor_sync(0xffffffffu, s1, 1); s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
    const float i0 = 1.0f / s0, i1 = 1.0f / s1;
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const int d = 8 * j + (lane & 3) * 2;
        if (r0 < T) *reinterpret_cast<uint32_t*>(att + ((int64_t)r0 * G + g) * E + h * 64 + d) = pack_h16x2(oacc[j][0] * i0, oacc[j][1] * i0, BF ? 1 : 0);
        if (r1 < T) *reinterpret_cast<uint32_t*>(att + ((int64_t)r1 * G + g) * E + h * 64 + d) = pack_h16x2(oacc[j][2] * i1, oacc[j][3] * i1, BF ? 1 : 0);
    }
}

// The same causal attention for groups of at most 8 tokens (the head stack of the teacher-forced forward: D tokens per (position,
// batch row), ~10^5 (group, head) pairs): one WARP per pair, everything in registers, lane <-> dims (2*lane, 2*lane+1), scores by
// warp reductions.
template <int TMAXS>
__global__ void __launch_bounds__(128)
prefill_attn_small_kernel(const h16* __restrict__ qkv, h16* __restrict__ kc, h16* __restrict__ vc, h16* __restrict__ att, int G, int T, int E,
                          int nh, int Tmax, int bf) {
    tc::pdl_launch_dependents();
    tc::pdl_wait();
    const int lane = threadIdx.x & 31;
    const int64_t pair = (int64_t)blockIdx.x * 4 + (threadIdx.x >> 5);
    if (pair >= (int64_t)G * nh) return;
    const int g = (int)(pair / nh), h = (int)(pair % nh);
    float2 q[TMAXS], k[TMAXS], v[TMAXS];
#pragma unroll
    for (int t = 0; t < TMAXS; t++)
        if (t < T) {
            const h16* row = qkv + ((int64_t)t * G + g) * 3 * E + h * 64 + 2 * lane;
            const uint32_t q2 = *reinterpret_cast<const uint32_t*>(row), k2 = *reinterpret_cast<const uint32_t*>(row + E),
                           v2 = *reinterpret_cast<const uint32_t*>(row + 2 * E);
            q[t] = unpack_h16x2(q2, bf); k[t] = unpack_h16x2(k2, bf); v[t] = unpack_h16x2(v2, bf);
            if (kc) {
                *reinterpret_cast<uint32_t*>(kc + (((int64_t)g * nh + h) * Tmax + t) * 64 + 2 * lane) = k2;
                *reinterpret_cast<uint32_t*>(vc + (((int64_t)g * nh + h) * Tmax + t) * 64 + 2 * lane) = v2;
            }
        }
#pragma unroll
    for (int t = 0; t < TMAXS; t++)
        if (t < T) {
            float sc[TMAXS];
            float m = -INFINITY;
#pragma unroll
            for (int j = 0; j < TMAXS; j++)
                if (j <= t) {
                    sc[j] = warp_sum(fmaf(q[t].y, k[j].y, q[t].x * k[j].x)) * 0.125f;
                    m = fmaxf(m, sc[j]);
                }
            float sum = 0.f;
            float2 o = make_float2(0.f, 0.f);
#pragma unroll
            for (int j = 0; j < TMAXS; j++)
                if (j <= t) {
                    const float e = __expf(sc[j] - m);
                    sum += e;
                    o.x = fmaf(e, v[j].x, o.x);
                    o.y = fmaf(e, v[j].y, o.y);
                }
            const float inv = 1.0f / sum;
            *reinterpret_cast<uint32_t*>(att + ((int64_t)t * G + g) * E + h * 64 + 2 * lane) = pack_h16x2(o.x * inv, o.y * inv, bf);
        }
}

// token sources --------------------------------------------------------------------------------------------------
// cond token s: x[b,:] = cond_emb[cond[b,s]] + pos_emb_cond[s]                      (transformers.py:224)
// grid (B, n_tokens): token s = stt->s + blockIdx.y, written to row blockIdx.y * B + b
__global__ void __launch_bounds__(256)
cond_tok_kernel(const StepState* __restrict__ stt, const float* __restrict__ cond_emb, const float* __restrict__ pos_cond,
                int cond_len, int vocab_cond, int E, float* __restrict__ x) {
    tc::pdl_launch_dependents();
    tc::pdl_wait();
    const int b = blockIdx.x, s = stt->s + blockIdx.y, B = gridDim.x;
    int64_t c = stt->cond ? stt->cond[(int64_t)b * cond_len + s] : 0;
    c = c < 0 ? 0 : (c >= vocab_cond ? vocab_cond - 1 : c);
    float* xr = x + ((int64_t)blockIdx.y * B + b) * E;
    for (int e = threadIdx.x; e < E; e += 256) xr[e] = cond_emb[c * E + e] + pos_cond[(int64_t)s * E + e];
}
// summed code embeddings in 16-bit: mode 0 -> all D codes of position idx-1 (body input), mode d>=1 -> codes 0..d-1 of
// position idx (head input, cumsum)                                              (transformers.py:219-225, 250-255)
// mode < 0 (prefill / forward): grid (B, n_pos); the first -mode codes of position blockIdx.y + pos0, written to row blockIdx.y * B + b
// code i is looked up in cb + i * cb_dstride (0: one shared codebook; K*C: per-depth codebooks stacked [D,K,C]).
// last_only: code nd-1 alone instead of codes 0..nd-1 (cumsum_depth_ctx = false: the head input of depth d is e_{d-1}, :250-255).
// stt is not __restrict__: the previous kernel writes it, and a read-only (non-coherent) load may be scheduled above pdl_wait().
// CV: the positions are window positions, read from the canvas through stt->cv (kernels.h); else stt->codes is [B, HW, D].
template <bool CV>
__global__ void __launch_bounds__(64)
code_sum_kernel(const StepState* stt, const float* __restrict__ cb, int64_t cb_dstride, int HW, int D, int K, int C,
                int mode, int pos0, h16* __restrict__ out, int bf, int last_only) {
    tc::pdl_launch_dependents();
    tc::pdl_wait();
    const int b = blockIdx.x, B = gridDim.x;
    const int pos = mode < 0 ? pos0 + blockIdx.y : (mode == 0 ? stt->idx - 1 : stt->idx);
    const int nd = mode == 0 ? D : (mode < 0 ? -mode : mode);
    h16* o = out + ((int64_t)blockIdx.y * B + b) * C;
    for (int c = threadIdx.x; c < C; c += 64) {
        float a = 0.f;
        for (int i = last_only ? nd - 1 : 0; i < nd; i++) {
            int64_t k = stt->codes[(CV ? stt->cv.at(b, pos) : (int64_t)b * HW + pos) * D + i];
            k = k < 0 ? 0 : (k >= K ? K - 1 : k);
            a += cb[i * cb_dstride + k * C + c];
        }
        o[c] = pack_h16(a, bf);
    }
}
static int64_t cb_dstride(const rqb200_ar_config& c) { return c.codebook_per_depth ? (int64_t)c.codebook_size * c.code_dim : 0; }

// token embeddings straight into the fp32 residual stream (input_emb_vqvae / head_emb_vqvae = false, transformers.py:222,257):
//   out[row, :] = ((tok_d0[k_d0] + tok_d0+1[k_d0+1]) + ...) + pos[p * pos_stride]      over the codes d0 .. d0+nd-1 of position p,
// tok_i = tok + i * tok_dstride (0: one shared [V,E] table; V*E: the TupleEmbedding's per-depth blocks).  The position:
//   where 0: stt->idx - 1 (the body step's token),  1: stt->idx (a head step's token),  2: pos0 + blockIdx.y (batched rows),
// row = blockIdx.y * B + b (token-major, like code_sum_kernel).  The body token sums all D codes with pos = pos_emb_hw (pos_stride E);
// the head token of depth d is code d-1 alone with pos = pos_emb_d + d*E (pos_stride 0).  E % 4 == 0.
// stt is not __restrict__ (see code_sum_kernel).  CV: as code_sum_kernel.
template <bool CV>
__global__ void __launch_bounds__(128)
tok_gather_kernel(const StepState* stt, const float* __restrict__ tok, int64_t tok_dstride, int HW, int D, int V, int E, int d0, int nd,
                  int where, int pos0, const float* __restrict__ pos, int64_t pos_stride, float* __restrict__ out) {
    tc::pdl_launch_dependents();
    tc::pdl_wait();
    const int b = blockIdx.x, B = gridDim.x;
    const int p = where == 2 ? pos0 + blockIdx.y : (where == 0 ? stt->idx - 1 : stt->idx);
    const int64_t* kr = stt->codes + (CV ? stt->cv.at(b, p) : (int64_t)b * HW + p) * D;
    int64_t rows[8];
#pragma unroll
    for (int i = 0; i < 8; i++)
        if (i < nd) {
            int64_t k = kr[d0 + i];
            k = k < 0 ? 0 : (k >= V ? V - 1 : k);
            rows[i] = (d0 + i) * tok_dstride + k * E;
        }
    const float4* pr = reinterpret_cast<const float4*>(pos + (int64_t)p * pos_stride);
    float4* o = reinterpret_cast<float4*>(out + ((int64_t)blockIdx.y * B + b) * E);
    for (int e4 = threadIdx.x; e4 < E / 4; e4 += 128) {
        float4 a = reinterpret_cast<const float4*>(tok + rows[0])[e4];
#pragma unroll
        for (int i = 1; i < 8; i++)
            if (i < nd) {
                const float4 t = reinterpret_cast<const float4*>(tok + rows[i])[e4];
                a.x += t.x; a.y += t.y; a.z += t.z; a.w += t.w;
            }
        const float4 q = pr[e4];
        a.x += q.x; a.y += q.y; a.z += q.z; a.w += q.w;
        o[e4] = a;
    }
}
static int64_t tok_dstride(const rqb200_ar_config& c) { return (c.embed_variant & RQB200_EMB_TUPLE) ? (int64_t)c.vocab * c.embed_dim : 0; }
// bookkeeping: which graph just ran decides what advances
__global__ void advance_kernel(StepState* stt, int ds, int didx, int dstep) {
    tc::pdl_launch_dependents();
    tc::pdl_wait();
    if (threadIdx.x == 0) { stt->s += ds; stt->idx += didx; stt->step += dstep; }
}
__global__ void __launch_bounds__(256) logits_copy_kernel(const StepState* __restrict__ stt, const float* __restrict__ lg, int d,
                                                          int64_t n) {
    tc::pdl_launch_dependents();
    tc::pdl_wait();
    if (!stt->logits_out) return;
    float* dst = stt->logits_out + (int64_t)(stt->step + d) * n;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) dst[i] = lg[i];
}

// a new segment of a canvas: the body sequence restarts (s = idx = 0) on the window at canvas offset org
__global__ void segment_kernel(StepState* stt, int org) {
    tc::pdl_launch_dependents();
    tc::pdl_wait();
    if (threadIdx.x == 0) { stt->s = 0; stt->idx = 0; stt->cv.org = org; }
}

// keep_pos != 0: a resumed span keeps the position counters the previous span left behind
__global__ void init_state_kernel(StepState* dst, StepState v, int keep_pos) {
    if (threadIdx.x == 0) {
        if (keep_pos) { v.s = dst->s; v.idx = dst->idx; }
        *dst = v;
    }
}

// Single-token step (rqb200_ar_step): the codes [lo, hi) of every batch row (flat index pos * D + depth) from the caller's xs
// (row b at xs + b * xs_stride) into the engine's code buffer, and the step's counters into the StepState, so that the captured
// graphs replay unchanged.  restart: the whole StepState is v (prefill from position 0); else s / idx / logits_out only.  One CTA per
// batch row.  The caller's pointers reach the graphs only through the StepState (logits_out) or not at all (xs is read here).
__global__ void __launch_bounds__(128)
step_ingest_kernel(StepState* stt, StepState v, int restart, const int64_t* __restrict__ xs, int64_t xs_stride, int64_t lo, int64_t hi,
                   int64_t row_codes) {
    tc::pdl_launch_dependents();
    tc::pdl_wait();
    const int b = blockIdx.x;
    for (int64_t i = lo + threadIdx.x; i < hi; i += 128) v.codes[(int64_t)b * row_codes + i] = xs[(int64_t)b * xs_stride + i];
    if (b == 0 && threadIdx.x == 0) {
        if (restart) {
            *stt = v;
        } else {
            stt->s = v.s; stt->idx = v.idx; stt->step = 0; stt->logits_out = v.logits_out;
        }
    }
}

// ------------------------------------------------------------------------------------------------ engine
// Every weight is a StreamedWeight in the engine's format (16-bit, or E4M3 with RQB200_E4M3); only linear_rows() tells the two apart.
struct FastLayer {
    StreamedWeight qkv, proj, fc1, fc2;
};

// G_HEAD_STEP + d: head depth d alone with its logits copied out (rqb200_ar_step), d < 8.  G_CODE_CV .. G_HEAD_LOGITS_CV: G_CODE ..
// G_HEAD_LOGITS on a canvas (their gathers and sampler address the window through StepState::cv); they share their grid twins' trace
// slots, so the trace buffer keeps G_COUNT graphs' worth.
enum { G_COND = 0, G_CODE = 1, G_HEAD = 2, G_HEAD_LOGITS = 3, G_HEAD_STEP = 4, G_COUNT = G_HEAD_STEP + 8,
       G_CODE_CV = G_COUNT, G_HEAD_CV, G_HEAD_LOGITS_CV, G_ALL };
static int grid_twin(int which) { return which < G_COUNT ? which : which - G_CODE_CV + G_CODE; }

struct ArFast {
    rqb200_ar_config cfg;
    rqb200_ar_weights w;
    std::vector<rqb200_block_weights> body, head;
    std::vector<FastLayer> lbody, lhead;
    StreamedWeight w_in, w_head, w_cls, w_ccls;
    StreamedWeight w_cls_d[8];           // RQB200_EMB_CLS_PER_DEPTH: depth d's [V,E] slice of w_cls
    int bf = 0;                          // 16-bit activation format: 0 fp16, 1 bf16
    bool fp8 = false;                    // RQB200_E4M3 weights (fp16 activations)
    // per (workspace, B) state
    void* ws_base = nullptr;
    int B = 0;
    CUtensorMap tx_xn, tx_att, tx_h, tx_s;
    cudaGraphExec_t graphs[G_ALL] = {};
    int64_t n_nodes[G_ALL] = {};       // kernels recorded in each graph (for the launch counter)
    cudaStream_t cap_stream = nullptr;   // capture never happens on the caller's stream (it may be the legacy default stream)
    // launch options (cfg.flags), set by ar_fast_create and never changed afterwards.  use_pdl and trace are the single-token chain's;
    // a batched pass states each launch's PDL attribute at the launch and is never traced.
    bool use_graph = true, use_pdl = true, batched_prefill = true;
    bool trace = false;                  // diagnostic stage trace (RQB200_AR_TRACE)
    int split_qkv = 4, split_proj = 12, split_fc1 = 1, split_fc2 = 12;
    int n_sm = 0;
    mutable long long* tr_base = nullptr;
    mutable int tr_next = 0;
    mutable std::vector<std::string> tr_names;
    int tr_graph_base[G_COUNT + 1] = {};
};

constexpr int TR_PER_GRAPH = 1024;                 // trace slots owned by each graph
constexpr int TR_CAP = TR_PER_GRAPH * G_COUNT;     // launches per trace buffer

struct FastWs {
    StepState* state;
    long long* trace;
    int64_t* CODES;              // [B, HW, D] the single-token step's copy of the caller's codes (sampling writes its own `out`)
    float *XB, *XH, *P, *LOGITS;
    h16 *XN, *ATT, *Hh, *S;
    h16 *kc_body, *vc_body, *kc_head, *vc_head;
    // batched prefill (M = B * T rows, token-major)
    int64_t Mmax;
    float* PX;                   // [Mmax, E] residual stream
    h16 *PXN, *PQKV, *PATT, *PH, *PS;
};

static int pick_split(int n_tiles, int nkb, int want, int n_sm) {
    int s = want > 0 ? want : n_sm / n_tiles;
    if (s < 1) s = 1;
    if (s > nkb) s = nkb;
    return s;
}

static long long* tr_slot(const ArFast& f, const char* name) {
    if (!f.trace || !f.tr_base || f.tr_next >= TR_CAP) return nullptr;
    if ((int)f.tr_names.size() <= f.tr_next) f.tr_names.resize(f.tr_next + 1);
    f.tr_names[f.tr_next] = name;
    return f.tr_base + 4 * (int64_t)(f.tr_next++);
}

static int prefill_tmax(const rqb200_ar_config& c) { return c.cond_len + c.H * c.W - 1; }

static size_t fast_layout(const ArFast& f, int B, void* base, size_t cap, FastWs* ws) {
    const rqb200_ar_config& c = f.cfg;
    Arena a(base, cap);
    const int64_t E = c.embed_dim, HW = (int64_t)c.H * c.W, Tb = c.cond_len + HW;
    FastWs w;
    w.state = a.take<StepState>(1);
    w.trace = a.take<long long>(4 * TR_CAP);
    w.CODES = a.take<int64_t>((int64_t)B * HW * c.D);
    w.XB = a.take<float>(B * E);
    w.XH = a.take<float>(B * E);
    int maxs = std::max(std::max(f.split_qkv * 3, f.split_proj), std::max(f.split_fc2, f.split_fc1 * 4));
    w.P = a.take<float>((int64_t)maxs * B * E);
    w.LOGITS = a.take<float>((int64_t)B * c.vocab);
    w.XN = a.take<h16>(B * E);
    w.ATT = a.take<h16>(B * E);
    w.Hh = a.take<h16>(B * 4 * E);
    w.S = a.take<h16>((int64_t)B * c.code_dim);
    const int64_t per_body = (int64_t)B * c.n_head * Tb * 64, per_head = (int64_t)B * c.n_head * c.D * 64;
    w.kc_body = a.take<h16>(per_body * c.n_body);
    w.vc_body = a.take<h16>(per_body * c.n_body);
    w.kc_head = a.take<h16>(per_head * c.n_head_layers);
    w.vc_head = a.take<h16>(per_head * c.n_head_layers);
    w.Mmax = f.batched_prefill ? (int64_t)B * prefill_tmax(c) : 0;
    const int64_t Mp = w.Mmax ? w.Mmax + 128 : 0;          // (the rows GEMM reads whole 128-row tiles)
    w.PX = a.take<float>(Mp * E);
    w.PXN = a.take<h16>(Mp * E);
    w.PQKV = a.take<h16>(Mp * 3 * E);
    w.PATT = a.take<h16>(Mp * E);
    w.PH = a.take<h16>(Mp * 4 * E);
    w.PS = a.take<h16>(w.Mmax * c.code_dim);
    if (ws) *ws = w;
    return a.off + 256;
}

// the weight streamer on one engine weight over the p.B activation rows behind tx; p carries the split, the mode and the epilogue, the
// weight and the engine give the rest
static int gemm_w(const ArFast& f, const StreamedWeight& w, const CUtensorMap& tx, GemmTcParams p, bool pdl, cudaStream_t st) {
    p.fmt = f.bf; p.ld_out = w.N_out;
    return launch_gemm_tc(w, tx, p, pdl, st);
}

// ---- the single-token chain's launchers: PDL attribute from f.use_pdl, one trace slot each
static int gemm(const ArFast& f, const char* name, const StreamedWeight& w, const CUtensorMap& tx, int B, int splits, int mode, const float* bias,
                float bias_scale, void* out, float* partial, const float* residual, int64_t ld_res, const int* res_row_ptr,
                int64_t res_row_stride, cudaStream_t st) {
    GemmTcParams p = {};
    p.B = B; p.splits = splits; p.mode = mode;
    p.bias = bias; p.bias_scale = bias_scale; p.out = out; p.partial = partial;
    p.residual = residual; p.ld_res = ld_res; p.res_row_ptr = res_row_ptr; p.res_row_stride = res_row_stride;
    p.trace = tr_slot(f, name);
    return gemm_w(f, w, tx, p, f.use_pdl, st);
}

// ---- the single-token chain's non-GEMM launchers, functions of plain arguments: the engine and the rqb200_dbg_* entry points at the
// end of this file call the same functions, so a kernel-level test runs the engine's own dispatch.  nh = E / 64 heads.

// ln_reduce_kernel over `rows` rows (one CTA each): x_out = x_in + bias + sum_s partial[s] + extra ; xn = LN(x_out)
static int ln(int rows, const float* x_in, const float* partial, int S, const float* bias, const float* extra, float* x_out, const float* g,
              const float* be, h16* xn, int E, int bf, bool pdl, long long* tr, const PrefetchList& pf, cudaStream_t st) {
    return launch_pdl(ln_reduce_kernel<384, 3>, dim3((unsigned)rows), dim3(384), (size_t)0, st, pdl, x_in, partial, S, bias, extra, x_out,
                      g, be, xn, rows, E, bf, tr, pf);
}

// the step attention form a cache of Tmax rows runs: 2 = attn_fast2_kernel (the body stack: four warps per (b, head), cached rows
// staged in shared memory), 1 = attn_fast_kernel (head stacks, and body stacks past AF2_MAXROWS cached rows)
static int attn_form(int Tmax) { return Tmax >= 16 && Tmax - 1 <= AF2_MAXROWS ? 2 : 1; }

// one step attention over B rows: q/k/v = bqkv + sum of the S split-K partials part [S][B][3E], k/v appended at cache row t (t_ptr, a
// device int, or t_host), att [B, E] = softmax(q k^T / 8) v.  form 0: attn_form(Tmax).
static int attn(int form, const float* part, int S, const float* bqkv, h16* kc, h16* vc, h16* att, int B, int E, int Tmax, const int* t_ptr,
                int t_host, int bf, bool pdl, long long* tr, cudaStream_t st) {
    const int nh = E / 64;
    if (form == 0) form = attn_form(Tmax);
    if (form == 2) {
        const int rows = (Tmax - 1 + 7) & ~7;                        // cached rows a step can read (row t is the new token); 32 B-aligned float arrays behind them
        RQB_ENSURE_SMEM(attn2_smem(AF2_MAXROWS), attn_fast2_kernel);
        {   // 11 CTAs x 19.6 KB need the largest shared-memory carve-out (L1 is not used by this kernel)
            static std::atomic<uint64_t> carve{0};
            int dev = 0;
            RQB_CUDA(cudaGetDevice(&dev));
            if (!(carve.load(std::memory_order_acquire) & (1ull << (dev & 63)))) {
                RQB_CUDA(cudaFuncSetAttribute(attn_fast2_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
                carve.fetch_or(1ull << (dev & 63), std::memory_order_release);
            }
        }
        return launch_pdl(attn_fast2_kernel, dim3((unsigned)(B * nh)), dim3(128), attn2_smem(rows), st, pdl, part, S, bqkv, kc, vc, att, B, E,
                          nh, Tmax, rows, t_ptr, t_host, bf, tr);
    }
    const size_t smem = (size_t)(4 * ((Tmax + 31) & ~31)) * sizeof(float);
    return launch_pdl(attn_fast_kernel, dim3((unsigned)ceil_div(B * nh, 4)), dim3(128), smem, st, pdl, part, S, bqkv, kc, vc, att, B, E, nh,
                      Tmax, t_ptr, t_host, bf, tr);
}

// h [B, N] = 16-bit(gelu(bias + sum of the S split-K partials partial [S][B][N]))
static int act_reduce(const float* partial, int S, const float* bias, h16* h, int B, int N, int bf, bool pdl, long long* tr, cudaStream_t st) {
    return launch_pdl(act_reduce_kernel, dim3((unsigned)std::min<int64_t>(ceil_div((int64_t)B * N / 4, 256), 1184)), dim3(256), (size_t)0, st,
                      pdl, partial, S, bias, h, B, N, bf, tr);
}

// one transformer stack on the single new token of every batch row; x lives in `x` (fp32); residual additions are deferred
// into the next ln_reduce.
// fin_g / fin_b (nullable): a LayerNorm applied to the stack's output rows -> ws.XN (the classifier's), fused with whatever
// launch finishes x.
static int fast_stack(const ArFast& f, const std::vector<rqb200_block_weights>& blocks, const std::vector<FastLayer>& maps,
                      FastWs& ws, float* x, const float* pending_extra, const float* x_src, h16* kc, h16* vc, int Tmax,
                      const int* t_ptr, int t_host, const float* fin_g, const float* fin_b, cudaStream_t st) {
    const rqb200_ar_config& c = f.cfg;
    const int E = c.embed_dim, B = f.B;
    const int64_t per = (int64_t)B * c.n_head * Tmax * 64;
    const float* nof = nullptr;
    for (size_t l = 0; l < blocks.size(); l++) {
        const rqb200_block_weights& bw = blocks[l];
        const bool first = l == 0;
        // LN1 (+ pending fc2 reduction of the previous block)
        const bool pend = l > 0;
        PrefetchList pf = {};
        if (l + 1 < blocks.size()) {
            const rqb200_block_weights& nx = blocks[l + 1];
            const void* ptrs[8] = {nx.ln1_w, nx.ln1_b, nx.bqkv, nx.bproj, nx.ln2_w, nx.ln2_b, nx.b1, bw.b2};
            const uint32_t words[8] = {(uint32_t)E, (uint32_t)E, (uint32_t)(3 * E), (uint32_t)E, (uint32_t)E, (uint32_t)E, (uint32_t)(4 * E),
                                       (uint32_t)E};
            for (int i = 0; i < 8; i++) { pf.p[i] = ptrs[i]; pf.bytes[i] = words[i] * 4u; }
            pf.n = 8;
        }
        RQB_TRY(ln(B, first ? x_src : x, pend ? ws.P : nof, pend ? f.split_fc2 : 0, pend ? blocks[l - 1].b2 : nof, first ? pending_extra : nof,
                   x, bw.ln1_w, bw.ln1_b, ws.XN, E, f.bf, f.use_pdl, tr_slot(f, "ln1"), pf, st));
        RQB_TRY(gemm(f, "qkv", maps[l].qkv, f.tx_xn, B, f.split_qkv, GT_PARTIAL, nullptr, 1.f, nullptr, ws.P, nullptr, 0, nullptr, 0, st));
        RQB_TRY(attn(0, ws.P, f.split_qkv, bw.bqkv, kc + per * l, vc + per * l, ws.ATT, B, E, Tmax, t_ptr, t_host, f.bf, f.use_pdl,
                     tr_slot(f, "attn"), st));
        RQB_TRY(gemm(f, "proj", maps[l].proj, f.tx_att, B, f.split_proj, GT_PARTIAL, nullptr, 1.f, nullptr, ws.P, nullptr, 0, nullptr, 0, st));
        RQB_TRY(ln(B, x, ws.P, f.split_proj, bw.bproj, nof, x, bw.ln2_w, bw.ln2_b, ws.XN, E, f.bf, f.use_pdl, tr_slot(f, "ln2"), PrefetchList{},
                   st));
        if (f.split_fc1 == 1) {
            RQB_TRY(gemm(f, "fc1", maps[l].fc1, f.tx_xn, B, 1, GT_H16_GELU, bw.b1, 1.f, ws.Hh, nullptr, nullptr, 0, nullptr, 0, st));
        } else {
            RQB_TRY(gemm(f, "fc1", maps[l].fc1, f.tx_xn, B, f.split_fc1, GT_PARTIAL, nullptr, 1.f, nullptr, ws.P, nullptr, 0, nullptr, 0, st));
            RQB_TRY(act_reduce(ws.P, f.split_fc1, bw.b1, ws.Hh, B, 4 * E, f.bf, f.use_pdl, tr_slot(f, "act_reduce"), st));
        }
        RQB_TRY(gemm(f, "fc2", maps[l].fc2, f.tx_h, B, f.split_fc2, GT_PARTIAL, nullptr, 1.f, nullptr, ws.P, nullptr, 0, nullptr, 0, st));
    }
    // fold the last block's pending fc2 reduction into x (x is final on return) -- and the caller's LayerNorm, if any.  An empty
    // stack (a head-less model) only forms its input token x = x_src + pending_extra.
    if (blocks.empty())
        RQB_TRY(ln(B, x_src, nof, 0, nof, pending_extra, x, fin_g, fin_b, fin_g ? ws.XN : nullptr, E, f.bf, f.use_pdl, tr_slot(f, "finalize"),
                   PrefetchList{}, st));
    else
        RQB_TRY(ln(B, x, ws.P, f.split_fc2, blocks.back().b2, nof, x, fin_g, fin_b, fin_g ? ws.XN : nullptr, E, f.bf, f.use_pdl,
                   tr_slot(f, "finalize"), PrefetchList{}, st));
    return 0;
}

static int record_body(ArFast& f, FastWs& ws, bool cond_token, bool cv, cudaStream_t st) {
    const rqb200_ar_config& c = f.cfg;
    const rqb200_ar_weights& w = f.w;
    const int E = c.embed_dim, B = f.B, HW = c.H * c.W, Tb = c.cond_len + HW;
    if (cond_token) {
        RQB_TRY(launch_pdl(cond_tok_kernel, dim3(B, 1), dim3(256), (size_t)0, st, f.use_pdl, (const StepState*)ws.state, w.cond_emb,
                           w.pos_emb_cond, c.cond_len, c.vocab_cond, E, ws.XB));
    } else if (c.embed_variant & RQB200_EMB_TOK_INPUT) {
        // x = sum_d tok_emb(code_d) + pos_emb_hw[idx-1]           (transformers.py:222,225)
        RQB_TRY(launch_pdl(cv ? tok_gather_kernel<true> : tok_gather_kernel<false>, dim3(B, 1), dim3(128), (size_t)0, st, f.use_pdl,
                           (const StepState*)ws.state, w.tok_emb, tok_dstride(c), HW, c.D, c.vocab, E, 0, c.D, 0, 0, w.pos_emb_hw, (int64_t)E,
                           ws.XB));
    } else {
        RQB_TRY(launch_pdl(cv ? code_sum_kernel<true> : code_sum_kernel<false>, dim3(B, 1), dim3(64), (size_t)0, st, f.use_pdl,
                           (const StepState*)ws.state, w.codebook, cb_dstride(c), HW, c.D, c.codebook_size, c.code_dim, 0, 0, ws.S, f.bf, 0));
        // x = W_in (sum_d e_d) + D b_in + pos_emb_hw[idx-1]       (bias counted D times, transformers.py:220,225)
        RQB_TRY(gemm(f, "w_in", f.w_in, f.tx_s, B, 1, GT_F32, w.b_in, (float)c.D, ws.XB, nullptr, w.pos_emb_hw - E /* row idx-1 */, 0,
                     &ws.state->idx, E, st));
    }
    RQB_TRY(fast_stack(f, f.body, f.lbody, ws, ws.XB, nullptr, ws.XB, ws.kc_body, ws.vc_body, Tb, &ws.state->s, 0, nullptr, nullptr, st));
    RQB_TRY(launch_pdl(advance_kernel, dim3(1), dim3(32), (size_t)0, st, f.use_pdl, ws.state, 1, 0, 0));
    return 0;
}

// head depth d of the position stt->idx: its token, the head stack (cache rows [0, d) from the earlier depths of this position) and
// the classifier -> ws.LOGITS
static int record_head_depth(ArFast& f, FastWs& ws, int d, bool cv, cudaStream_t st) {
    const rqb200_ar_config& c = f.cfg;
    const rqb200_ar_weights& w = f.w;
    const int E = c.embed_dim, B = f.B, HW = c.H * c.W, D = c.D, V = c.vocab;
    if (d == 0) {
        // token = spatial ctx (body output) + pos_emb_d[0]                                   (transformers.py:259-270)
        RQB_TRY(fast_stack(f, f.head, f.lhead, ws, ws.XH, w.pos_emb_d, ws.XB, ws.kc_head, ws.vc_head, D, nullptr, 0, w.cls_ln_w,
                           w.cls_ln_b, st));
    } else {
        if (c.embed_variant & RQB200_EMB_TOK_HEAD) {
            // token = tok_emb(code_{d-1}) + pos_emb_d[d]                                    (transformers.py:257,267)
            RQB_TRY(launch_pdl(cv ? tok_gather_kernel<true> : tok_gather_kernel<false>, dim3(B, 1), dim3(128), (size_t)0, st, f.use_pdl,
                               (const StepState*)ws.state, w.tok_emb, tok_dstride(c), HW, D, c.vocab, E, d - 1, 1, 1, 0, w.pos_emb_d + (int64_t)d * E, (int64_t)0,
                               ws.XH));
        } else {
            // token = head_mlp(sum_{i<d} e_i, or e_{d-1} alone) + pos_emb_d[d]              (transformers.py:250-255,267)
            RQB_TRY(launch_pdl(cv ? code_sum_kernel<true> : code_sum_kernel<false>, dim3(B, 1), dim3(64), (size_t)0, st, f.use_pdl,
                               (const StepState*)ws.state, w.codebook, cb_dstride(c), HW, D, c.codebook_size, c.code_dim, d, 0, ws.S, f.bf,
                               (c.embed_variant & RQB200_EMB_NO_CUMSUM) ? 1 : 0));
            RQB_TRY(gemm(f, "w_head", f.w_head, f.tx_s, B, 1, GT_F32, w.b_head, 1.f, ws.XH, nullptr,
                         w.pos_emb_d + (int64_t)d * E, 0, nullptr, 0, st));
        }
        RQB_TRY(fast_stack(f, f.head, f.lhead, ws, ws.XH, nullptr, ws.XH, ws.kc_head, ws.vc_head, D, nullptr, d, w.cls_ln_w,
                           w.cls_ln_b, st));
    }
    // classifier: LN(x) (fused into the stack's last launch) -> logits                       (transformers.py:278-285)
    // per-depth classifiers (BatchLinear): depth d's [V,E] slice and bias row
    const bool pd = c.embed_variant & RQB200_EMB_CLS_PER_DEPTH;
    RQB_TRY(gemm(f, "cls", pd ? f.w_cls_d[d] : f.w_cls, f.tx_xn, B, 1, GT_F32, w.b_cls + (pd ? (int64_t)d * V : 0), 1.f,
                 ws.LOGITS, nullptr, nullptr, 0, nullptr, 0, st));
    return 0;
}

static int record_head(ArFast& f, FastWs& ws, bool with_logits, bool cv, cudaStream_t st) {
    const rqb200_ar_config& c = f.cfg;
    const int B = f.B, HW = c.H * c.W, D = c.D, V = c.vocab;
    for (int d = 0; d < D; d++) {
        RQB_TRY(record_head_depth(f, ws, d, cv, st));
        if (with_logits)
            RQB_TRY(launch_pdl(logits_copy_kernel, dim3(64), dim3(256), (size_t)0, st, f.use_pdl, (const StepState*)ws.state,
                               (const float*)ws.LOGITS, d, (int64_t)B * V));
        RQB_TRY(launch_sample_dyn(ws.LOGITS, ws.state, d, B, V, HW, D, st, f.use_pdl, cv));
    }
    RQB_TRY(launch_pdl(advance_kernel, dim3(1), dim3(32), (size_t)0, st, f.use_pdl, ws.state, 0, 1, D));
    return 0;
}

// the single-token step's head graph: depth d only, its logits to stt->logits_out (stt->step == 0), no sampler; the code of depth d
// comes from the caller at the next step.  Launch for launch the depth-d part of record_head: the same logits, bit for bit.
static int record_head_step(ArFast& f, FastWs& ws, int d, cudaStream_t st) {
    RQB_TRY(record_head_depth(f, ws, d, false, st));
    RQB_TRY(launch_pdl(logits_copy_kernel, dim3(64), dim3(256), (size_t)0, st, f.use_pdl, (const StepState*)ws.state,
                       (const float*)ws.LOGITS, 0, (int64_t)f.B * f.cfg.vocab));
    if (d == f.cfg.D - 1) RQB_TRY(launch_pdl(advance_kernel, dim3(1), dim3(32), (size_t)0, st, f.use_pdl, ws.state, 0, 1, 0));
    return 0;
}

static int record(ArFast& f, FastWs& ws, int which, cudaStream_t st) {
    f.tr_base = ws.trace;
    f.tr_next = f.tr_graph_base[grid_twin(which)];
    const bool cv = which >= G_COUNT;
    const int kind = grid_twin(which);
    int rc = kind == G_COND ? record_body(f, ws, true, false, st) : kind == G_CODE ? record_body(f, ws, false, cv, st)
           : kind >= G_HEAD_STEP ? record_head_step(f, ws, kind - G_HEAD_STEP, st)
                                 : record_head(f, ws, kind == G_HEAD_LOGITS, cv, st);
    // trace slots: every graph owns TR_PER_GRAPH of the buffer
    return rc;
}

static int capture(ArFast& f, FastWs& ws, int which, cudaGraphExec_t* out) {
    cudaGraph_t g = nullptr;
    if (!f.cap_stream) RQB_CUDA(cudaStreamCreateWithFlags(&f.cap_stream, cudaStreamNonBlocking));
    cudaStream_t st = f.cap_stream;
    RQB_CUDA(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
    const int64_t before = g_launches;
    int rc = record(f, ws, which, st);
    f.n_nodes[which] = g_launches - before;
    g_launches = before;                   // recording is not launching
    cudaError_t e = cudaStreamEndCapture(st, &g);
    if (rc) { if (g) cudaGraphDestroy(g); return rc; }
    if (e != cudaSuccess) return fail(RQB200_ECUDA, std::string("graph capture failed: ") + cudaGetErrorString(e));
    e = cudaGraphInstantiate(out, g, 0);
    cudaGraphDestroy(g);
    if (e != cudaSuccess) return fail(RQB200_ECUDA, std::string("graph instantiate failed: ") + cudaGetErrorString(e));
    return 0;
}

static void drop_graphs(ArFast& f) {
    for (int i = 0; i < G_ALL; i++) {
        if (f.graphs[i]) cudaGraphExecDestroy(f.graphs[i]);
        f.graphs[i] = nullptr;
    }
}

ArFast* ar_fast_create(const rqb200_ar_config& cfg, const rqb200_ar_weights& w, const rqb200_block_weights* body_p,
                       const rqb200_block_weights* head_p) {
    std::vector<rqb200_block_weights> body(body_p, body_p + cfg.n_body), head(head_p, head_p + cfg.n_head_layers);
    const int E = cfg.embed_dim;
    if (E % 128 != 0 || cfg.vocab % 128 != 0 || cfg.code_dim % 64 != 0 || cfg.D > 8 || cfg.cond_len + cfg.H * cfg.W > FAST_MAXT || E > 4608) {
        set_error("ar fast tier: need E % 128 == 0, V % 128 == 0, code_dim % 64 == 0, D <= 8, cond_len + H*W <= 2048, E <= 4608");
        return nullptr;
    }
    if (cfg.n_body < 1) {
        set_error("ar fast tier: need at least one body layer (n_body >= 1)");
        return nullptr;
    }
    ArFast* f = new ArFast();
    f->cfg = cfg; f->w = w; f->body = body; f->head = head;
    f->bf = cfg.weight_dtype == RQB200_BF16 ? 1 : 0;
    f->fp8 = cfg.weight_dtype == RQB200_E4M3;
    f->use_graph = !(cfg.flags & RQB200_AR_NO_GRAPH);
    f->use_pdl = !(cfg.flags & RQB200_AR_NO_PDL);
    f->trace = (cfg.flags & RQB200_AR_TRACE) != 0;
    f->batched_prefill = !(cfg.flags & RQB200_AR_SEQUENTIAL_PREFILL);
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&f->n_sm, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
        f->n_sm < 1) {
        set_error("ar fast tier: cannot read the device's SM count (the split-K factors are planned for it)");
        delete f;
        return nullptr;
    }
    const int nkbE = E / 64;
    f->split_qkv = pick_split(3 * E / 128, nkbE, cfg.split_qkv, f->n_sm);
    f->split_proj = pick_split(E / 128, nkbE, cfg.split_proj, f->n_sm);
    f->split_fc1 = pick_split(4 * E / 128, nkbE, cfg.split_fc1, f->n_sm);
    f->split_fc2 = pick_split(E / 128, 4 * nkbE, cfg.split_fc2, f->n_sm);
    auto make_w = [&](StreamedWeight* out, const void* wt, const float* s, int N_out, int K) {
        return make_streamed_weight(out, f->fp8, wt, s, N_out, K);
    };
    auto mk = [&](const std::vector<rqb200_block_weights>& bl, std::vector<FastLayer>& out) -> int {
        out.resize(bl.size());
        for (size_t l = 0; l < bl.size(); l++) {
            RQB_TRY(make_w(&out[l].qkv, bl[l].wqkv, bl[l].sqkv, 3 * E, E));
            RQB_TRY(make_w(&out[l].proj, bl[l].wproj, bl[l].sproj, E, E));
            RQB_TRY(make_w(&out[l].fc1, bl[l].w1, bl[l].s1, 4 * E, E));
            RQB_TRY(make_w(&out[l].fc2, bl[l].w2, bl[l].s2, E, 4 * E));
        }
        return 0;
    };
    int rc = mk(body, f->lbody);
    if (!rc) rc = mk(head, f->lhead);
    if (!rc && w.w_in) rc = make_w(&f->w_in, w.w_in, w.s_in, E, cfg.code_dim);
    if (!rc && w.w_head) rc = make_w(&f->w_head, w.w_head, w.s_head, E, cfg.code_dim);
    if (!rc) rc = make_w(&f->w_cls, w.w_cls, w.s_cls, cfg.vocab, E);
    if (cfg.embed_variant & RQB200_EMB_CLS_PER_DEPTH)       // depth d's [V,E] slice: V*E weight bytes per depth (2 per element in 16 bits)
        for (int d = 0; d < cfg.D && !rc; d++)
            rc = make_w(&f->w_cls_d[d], (const char*)w.w_cls + (size_t)d * cfg.vocab * E * (f->fp8 ? 1 : 2),
                        f->fp8 ? w.s_cls + (size_t)d * cfg.vocab : nullptr, cfg.vocab, E);
    if (!rc && w.w_ccls) rc = make_w(&f->w_ccls, w.w_ccls, w.s_ccls, (cfg.vocab_cond + 127) / 128 * 128, E);
    if (rc) { delete f; return nullptr; }
    for (int i = 0; i <= G_COUNT; i++) f->tr_graph_base[i] = i * (TR_CAP / G_COUNT);
    return f;
}

void ar_fast_destroy(ArFast* f) {
    if (!f) return;
    drop_graphs(*f);
    if (f->cap_stream) cudaStreamDestroy(f->cap_stream);
    delete f;
}

size_t ar_fast_workspace_bytes(const ArFast* f, int B) { return fast_layout(*f, B, nullptr, 0, nullptr); }

// ---- batched passes (prefill, teacher-forced forward): M = G * T token rows, token-major (row = t * G + g), through one stack.
struct BatchBufs {
    float* X;                    // [M, E] residual stream (in / out)
    h16 *XN, *QKV, *ATT, *H;     // [M,E], [M,3E], [M,E], [M,4E] scratch
};

// The epilogue of one linear layer of a batched pass, in the weight streamer's terms: out = acc + bias, to 16 bits (GT_H16, GT_H16_GELU) or,
// after adding activation row b's residual row b * ld_res, to fp32 (GT_F32).
static GemmTcParams epilogue(int mode, const float* bias, void* out, const float* residual = nullptr, int64_t ld_res = 0) {
    GemmTcParams p = {};
    p.splits = 1; p.mode = mode; p.bias = bias; p.bias_scale = 1.f; p.out = out; p.residual = residual; p.ld_res = ld_res;
    return p;
}

// One linear layer of a batched pass: the weight w over the M activation rows x [M, w.K], with the epilogue p.  The one place that picks
// the GEMM:
//   weights with a 16-bit copy, M_launch > 256: the persistent rows GEMM (conv_tc.cu: 128 x 256 tiles, operand loads overlapped with the epilogue,
//   like the next tile); it has no PDL attribute;
//   M_launch <= 256, and E4M3 weights at every M: the weight streamer (E4M3: 128-row chunks, faster than the fp16 rows GEMM at the
//   forward's shapes) over a tensor map of x, with the PDL attribute `pdl`.
// M_launch = M, except for a chunk of a launch the forward makes over M_launch rows (log_prob's classifier chunks): both GEMMs compute
// each output row from its own activation row alone, so the GEMM the forward picks gives the chunk the forward's logits bit for bit.
// streamer_only: never the rows GEMM.  For w_in / w_head, whose epilogues (bias_scale, a broadcast residual, res_div) the rows GEMM
// does not have, and for the cond classifier, whose logits have always been the streamer's (the rows GEMM sums in another order).
static int linear_rows(const ArFast& f, const StreamedWeight& w, const h16* x, int64_t M, int64_t M_launch, bool streamer_only, GemmTcParams p,
                       bool pdl, cudaStream_t st) {
    if (!streamer_only && !w.e4m3() && M_launch > 256) {
        const bool f32 = p.mode == GT_F32;
        return launch_rows_gemm_tc(x, w.w16, p.bias, p.residual, f32 ? (float*)p.out : nullptr, f32 ? nullptr : p.out, p.mode == GT_H16_GELU,
                                   f.bf, M, w.N_out, w.K, st);
    }
    CUtensorMap tx;
    RQB_TRY(make_tmap_2d(&tx, x, 1, w.K, M, (uint64_t)w.K * 2, 64, gemm_tc_chunk_rows(w, M)));
    p.B = (int)M;
    return gemm_w(f, w, tx, p, pdl, st);
}

// LayerNorm over the rows of a batched pass: x_out (nullable) = x_in + extra (nullable), xn (nullable) = LN(x_out).  512 rows and more: a
// warp per row, launched with the PDL attribute; fewer: ln_reduce_kernel with nothing to reduce, launched without.  The two kernels
// sum in different orders, so the threshold is part of the results.
// The warp-per-row form alone (ln_rows_kernel<NV>, the smallest NV with E <= 128 * NV), rows grid-strided over at most 8 CTAs per SM.
static int ln_rows_warp(int64_t rows, const float* x_in, const float* extra, float* x_out, const float* g, const float* be, h16* xn, int E,
                        int bf, int n_sm, cudaStream_t st) {
    const dim3 grid((unsigned)std::min<int64_t>(ceil_div(rows, 8), (int64_t)n_sm * 8));
    const int nv = ceil_div(E, 128);
#define RQB_LN_ROWS(NV) launch_pdl(ln_rows_kernel<NV>, grid, dim3(256), (size_t)0, st, true, x_in, extra, x_out, g, be, xn, rows, E, bf)
    if (nv <= 8) return RQB_LN_ROWS(8);
    if (nv <= 12) return RQB_LN_ROWS(12);
    if (nv <= 20) return RQB_LN_ROWS(20);
    return RQB_LN_ROWS(36);
#undef RQB_LN_ROWS
}
static int ln_rows(int64_t rows, const float* x_in, const float* extra, float* x_out, const float* g, const float* be, h16* xn, int E, int bf,
                   int n_sm, cudaStream_t st) {
    if (rows < 512) {
        const float* nof = nullptr;
        return ln((int)rows, x_in, nof, 0, nof, extra, x_out, g, be, xn, E, bf, false, nullptr, PrefetchList{}, st);
    }
    return ln_rows_warp(rows, x_in, extra, x_out, g, be, xn, E, bf, n_sm, st);
}

// Causal attention of a batched pass over G groups of T new tokens at sequence offset T0 (qkv token-major [T*G, 3E], bias added; keys
// before T0 from the cache), the cache rows [T0, T0 + T) of every (group, head) written when kc != NULL: at T0 = 0 a warp per (group,
// head) for T <= 8, 64-query tiles over 64-key tiles otherwise.
static int prefill_attn(const h16* qkv, h16* kc, h16* vc, h16* att, int G, int T, int E, int Tmax, int bf, bool pdl, cudaStream_t st,
                        int T0 = 0) {
    const int nh = E / 64;
    if (T0 == 0 && T <= 4)                                       // tiny groups (the forward's head stack): a warp per (group, head)
        return launch_pdl(prefill_attn_small_kernel<4>, dim3((unsigned)ceil_div((int64_t)G * nh, 4)), dim3(128), (size_t)0, st, pdl, qkv, kc,
                          vc, att, G, T, E, nh, Tmax, bf);
    if (T0 == 0 && T <= 8)
        return launch_pdl(prefill_attn_small_kernel<8>, dim3((unsigned)ceil_div((int64_t)G * nh, 4)), dim3(128), (size_t)0, st, pdl, qkv, kc,
                          vc, att, G, T, E, nh, Tmax, bf);
    const dim3 grid((unsigned)((int64_t)ceil_div(T, 64) * G * nh));     // 64-query tiles over 64-key tiles, online softmax
    if (bf) return launch_pdl(prefill_attn_flash_kernel<true>, grid, dim3(128), (size_t)0, st, pdl, qkv, kc, vc, att, G, T, E, nh, Tmax, T0);
    return launch_pdl(prefill_attn_flash_kernel<false>, grid, dim3(128), (size_t)0, st, pdl, qkv, kc, vc, att, G, T, E, nh, Tmax, T0);
}

// The CLIP engine's pieces of the batched pass (fp16, no KV cache): the tiled attention over G groups of T tokens, causal (text) or
// not (vision), and the warp-per-row LayerNorm to fp16 at every row count.
int launch_attn_flash_f16(const h16* qkv, h16* att, int G, int T, int E, bool causal, cudaStream_t st) {
    const dim3 grid((unsigned)((int64_t)ceil_div(T, 64) * G * (E / 64)));
    if (causal) return launch_pdl(prefill_attn_flash_kernel<false>, grid, dim3(128), (size_t)0, st, false, qkv, (h16*)nullptr,
                                  (h16*)nullptr, att, G, T, E, E / 64, 0, 0);
    return launch_pdl(prefill_attn_flash_kernel<false, false>, grid, dim3(128), (size_t)0, st, false, qkv, (h16*)nullptr, (h16*)nullptr,
                      att, G, T, E, E / 64, 0, 0);
}
int launch_ln_rows_f16(int64_t rows, const float* x, const float* g, const float* be, h16* xn, int E, cudaStream_t st) {
    int dev = 0, n_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
    return ln_rows_warp(rows, x, nullptr, nullptr, g, be, xn, E, 0, n_sm > 0 ? n_sm : 132, st);
}

// T new tokens of G groups at sequence offset T0 through one stack; cache rows [T0, T0 + T) written when kc != NULL (T0 > 0 needs kc)
static int stack_batched(const ArFast& f, const std::vector<rqb200_block_weights>& blocks, const std::vector<FastLayer>& maps,
                         const BatchBufs& bb, int G, int T, h16* kc, h16* vc, int64_t kv_per_layer, int Tmax, cudaStream_t st, int T0 = 0) {
    const rqb200_ar_config& c = f.cfg;
    const int E = c.embed_dim;
    const int64_t M = (int64_t)G * T;
    if (M > (int64_t)1 << 30 || T > FAST_MAXT) return fail(RQB200_EINVAL, "ar fast tier: batched pass too large");
    const bool pdl = true;               // the pass is a PDL chain too: a launch's set-up overlaps its predecessor's tail
    const float* nof = nullptr;
    for (size_t l = 0; l < blocks.size(); l++) {
        const rqb200_block_weights& bw = blocks[l];
        RQB_TRY(ln_rows(M, bb.X, nof, nullptr, bw.ln1_w, bw.ln1_b, bb.XN, E, f.bf, f.n_sm, st));
        RQB_TRY(linear_rows(f, maps[l].qkv, bb.XN, M, M, false, epilogue(GT_H16, bw.bqkv, bb.QKV), pdl, st));
        h16* kcl = kc ? kc + kv_per_layer * l : nullptr;
        h16* vcl = vc ? vc + kv_per_layer * l : nullptr;
        RQB_TRY(prefill_attn(bb.QKV, kcl, vcl, bb.ATT, G, T, E, Tmax, f.bf, pdl, st, T0));
        RQB_TRY(linear_rows(f, maps[l].proj, bb.ATT, M, M, false, epilogue(GT_F32, bw.bproj, bb.X, bb.X, E), pdl, st));
        RQB_TRY(ln_rows(M, bb.X, nof, nullptr, bw.ln2_w, bw.ln2_b, bb.XN, E, f.bf, f.n_sm, st));
        RQB_TRY(linear_rows(f, maps[l].fc1, bb.XN, M, M, false, epilogue(GT_H16_GELU, bw.b1, bb.H), pdl, st));
        RQB_TRY(linear_rows(f, maps[l].fc2, bb.H, M, M, false, epilogue(GT_F32, bw.b2, bb.X, bb.X, E), pdl, st));
    }
    return 0;
}

// body input tokens [T0, T0 + T) of every batch row into X (token-major, token T0 + r in rows r * B ..): token s < cond_len is a cond
// token (transformers.py:224), token s >= cond_len carries the summed input embeddings of the codes of position s - cond_len (:219-225).
// The cond tokens' kernel reads their index from state->s, which must equal T0.
// cv: the code tokens are window positions, gathered from the canvas through state->cv.
static int body_tokens_batched(const ArFast& f, const StepState* state, float* X, h16* S, int B, int T, cudaStream_t st, int T0 = 0,
                               bool cv = false) {
    const rqb200_ar_config& c = f.cfg;
    const rqb200_ar_weights& w = f.w;
    const int E = c.embed_dim, HW = c.H * c.W, cl = c.cond_len;
    const int n_cond = std::max(0, std::min(T0 + T, cl) - T0);
    if (n_cond > 0)
        RQB_TRY(launch_pdl(cond_tok_kernel, dim3(B, n_cond), dim3(256), (size_t)0, st, false, state, w.cond_emb, w.pos_emb_cond, cl,
                           c.vocab_cond, E, X));
    const int n_code = T - n_cond, pos0 = T0 + n_cond - cl;     // code tokens of positions pos0 .. pos0 + n_code - 1
    float* Xc = X + (int64_t)n_cond * B * E;
    if (n_code > 0 && (c.embed_variant & RQB200_EMB_TOK_INPUT)) {
        // row (j, b) = sum_d tok_emb(code_d of position j) + pos_emb_hw[j]                   (:222,225)
        RQB_TRY(launch_pdl(cv ? tok_gather_kernel<true> : tok_gather_kernel<false>, dim3(B, n_code), dim3(128), (size_t)0, st, false, state,
                           w.tok_emb, tok_dstride(c), HW, c.D, c.vocab, E, 0, c.D, 2, pos0, w.pos_emb_hw, (int64_t)E, Xc));
    } else if (n_code > 0) {
        RQB_TRY(launch_pdl(cv ? code_sum_kernel<true> : code_sum_kernel<false>, dim3(B, n_code), dim3(64), (size_t)0, st, false, state,
                           w.codebook, cb_dstride(c), HW, c.D, c.codebook_size, c.code_dim, -c.D, pos0, S, f.bf, 0));
        const int64_t Mc = (int64_t)B * n_code;
        GemmTcParams e = epilogue(GT_F32, w.b_in, Xc, w.pos_emb_hw + (int64_t)pos0 * E, E);
        e.bias_scale = (float)c.D;       // (the bias is counted D times, as in the single-token step)
        e.res_div = B;                   // row (j, b) gets pos_emb_hw[j]
        RQB_TRY(linear_rows(f, f.w_in, S, Mc, Mc, true, e, false, st));
    }
    return 0;
}

// ---- batched body pass: body tokens [T0, T0 + T) of every batch row in one pass, on the KV cache rows [0, T0) earlier passes or steps
// left (state.s == T0).  Leaves ws.XB = the last token's output rows, the KV cache rows [T0, T0 + T) written, state.s = T0 + T.  The
// prefill is T0 = 0; an append of a run of kept positions' code tokens to the cache is T0 > 0.
static int body_batched(const ArFast& f, FastWs& ws, int T0, int T, cudaStream_t st, bool cv = false) {
    const rqb200_ar_config& c = f.cfg;
    const int E = c.embed_dim, B = f.B, HW = c.H * c.W, cl = c.cond_len, Tb = cl + HW;
    const int64_t M = (int64_t)B * T;
    if (M > ws.Mmax || T0 + T > Tb) return fail(RQB200_EINVAL, "ar fast tier: too many tokens for the batched body pass");
    RQB_TRY(body_tokens_batched(f, ws.state, ws.PX, ws.PS, B, T, st, T0, cv));
    BatchBufs bb = {ws.PX, ws.PXN, ws.PQKV, ws.PATT, ws.PH};
    RQB_TRY(stack_batched(f, f.body, f.lbody, bb, B, T, ws.kc_body, ws.vc_body, (int64_t)B * c.n_head * Tb * 64, Tb, st, T0));
    RQB_CUDA(cudaMemcpyAsync(ws.XB, ws.PX + (int64_t)(T - 1) * B * E, (size_t)B * E * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return launch_pdl(advance_kernel, dim3(1), dim3(32), (size_t)0, st, false, ws.state, T, 0, 0);
}

// ---- teacher-forced forward (transformers.py:113-188): all H*W*D logits of given code maps in a handful of large-M GEMM passes.
// Body: T = cond_len + H*W - 1 tokens per batch row (M = B*T rows); head: for every (position, batch row) a group of D tokens
// [spatial ctx + pos_d[0], head_mlp(cumsum_{i<d} e_i) + pos_d[d]] (M = D * H*W * B rows, causal attention inside each group).
// logits_out [D][H*W][B][V] f32 (token-major; the host permutes), cond_logits_out (nullable) [cond_len-1][B][vocab_cond rounded
// up to a multiple of 128] (the cond classifier's weight / bias rows are zero-padded to that size by the caller).
struct FwdWs {
    StepState* state;
    float *BX, *HX;
    h16 *XN, *QKV, *ATT, *H, *S;
};
static size_t forward_layout(const ArFast& f, int B, void* base, size_t cap, FwdWs* out) {
    const rqb200_ar_config& c = f.cfg;
    Arena a(base, cap);
    const int64_t E = c.embed_dim, HW = (int64_t)c.H * c.W, Tb = c.cond_len + HW - 1;
    const int64_t Mb = B * Tb, Mh = (int64_t)c.D * HW * B, Mm = std::max(Mb, Mh) + 128;   // (+128: whole-tile reads of the rows GEMM)
    FwdWs w;
    w.state = a.take<StepState>(1);
    w.BX = a.take<float>(Mb * E);
    w.HX = a.take<float>(Mh * E);
    w.XN = a.take<h16>(Mm * E);
    w.QKV = a.take<h16>(Mm * 3 * E);
    w.ATT = a.take<h16>(Mm * E);
    w.H = a.take<h16>(Mm * 4 * E);
    w.S = a.take<h16>(HW * B * c.code_dim);
    if (out) *out = w;
    return a.off + 256;
}
size_t ar_fast_forward_workspace_bytes(const ArFast* f, int B) { return forward_layout(*f, B, nullptr, 0, nullptr); }

// The passes the forward and the log-likelihood share: body tokens and body stack (ws.BX); with_cond: the cond classifier's LayerNorm
// of the first (cond_len-1)*B body rows into ws.XN, then cond_cls(Mc) runs its GEMMs on them (before the head reuses ws.XN); head
// tokens, head stack and the classifier's LayerNorm: ws.XN [D*H*W*B, E], row (d*H*W + pos)*B + b.
template <class CondCls>
static int forward_passes(const ArFast& f, const FwdWs& ws, const int64_t* codes, const int64_t* cond, int B, bool with_cond,
                          CondCls&& cond_cls, cudaStream_t st) {
    const rqb200_ar_config& c = f.cfg;
    const rqb200_ar_weights& w = f.w;
    const int E = c.embed_dim, D = c.D, HW = c.H * c.W, cl = c.cond_len, V = c.vocab, Tb = cl + HW - 1;
    StepState h = {};
    h.cond = cond; h.codes = const_cast<int64_t*>(codes);
    RQB_TRY(launch_pdl(init_state_kernel, dim3(1), dim3(32), (size_t)0, st, false, ws.state, h, 0));
    const float* nof = nullptr;
    const int G = HW * B;                                  // head groups, g = pos * B + b
    const int64_t Mh = (int64_t)D * G;
    // body
    RQB_TRY(body_tokens_batched(f, ws.state, ws.BX, ws.S, B, Tb, st));
    BatchBufs bb = {ws.BX, ws.XN, ws.QKV, ws.ATT, ws.H};
    RQB_TRY(stack_batched(f, f.body, f.lbody, bb, B, Tb, nullptr, nullptr, 0, Tb, st));
    if (with_cond) {                                        // cond_classifier(latents[:, :cond_len-1])        (:153-156)
        const int64_t Mc = (int64_t)(cl - 1) * B;
        RQB_TRY(ln_rows(Mc, ws.BX, nof, nullptr, w.ccls_ln_w, w.ccls_ln_b, ws.XN, E, f.bf, f.n_sm, st));
        RQB_TRY(cond_cls(Mc));
    }
    // head tokens: d = 0 rows = spatial ctx (body rows of tokens cond_len-1 ..) + pos_emb_d[0]; d >= 1 rows = head_mlp(cumsum)
    RQB_TRY(ln_rows(G, ws.BX + (int64_t)(cl - 1) * B * E, w.pos_emb_d, ws.HX, nof, nof, nullptr, E, f.bf, f.n_sm, st));
    for (int d = 1; d < D; d++) {
        if (c.embed_variant & RQB200_EMB_TOK_HEAD) {        // tok_emb(code_{d-1}) + pos_emb_d[d]        (:164,177)
            RQB_TRY(launch_pdl(tok_gather_kernel<false>, dim3(B, HW), dim3(128), (size_t)0, st, false, (const StepState*)ws.state, w.tok_emb,
                               tok_dstride(c), HW, D, V, E, d - 1, 1, 2, 0, w.pos_emb_d + (int64_t)d * E, (int64_t)0,
                               ws.HX + (int64_t)d * G * E));
            continue;
        }
        RQB_TRY(launch_pdl(code_sum_kernel<false>, dim3(B, HW), dim3(64), (size_t)0, st, false, (const StepState*)ws.state, w.codebook,
                           cb_dstride(c), HW, D, c.codebook_size, c.code_dim, -d, 0, ws.S, f.bf,
                           (c.embed_variant & RQB200_EMB_NO_CUMSUM) ? 1 : 0));
        RQB_TRY(linear_rows(f, f.w_head, ws.S, G, G, true,
                            epilogue(GT_F32, w.b_head, ws.HX + (int64_t)d * G * E, w.pos_emb_d + (int64_t)d * E, 0 /* one row for all */), false, st));
    }
    BatchBufs hb = {ws.HX, ws.XN, ws.QKV, ws.ATT, ws.H};
    RQB_TRY(stack_batched(f, f.head, f.lhead, hb, G, D, nullptr, nullptr, 0, D, st));
    // classifier LayerNorm                                                                         (:181-183)
    return ln_rows(Mh, ws.HX, nof, nullptr, w.cls_ln_w, w.cls_ln_b, ws.XN, E, f.bf, f.n_sm, st);
}

// The classifier launches of the forward: one over all D*H*W*B rows of ws.XN, or (per-depth classifiers) one per depth over that
// depth's slice of H*W*B rows.  cls(weight, bias, slice, rows) runs one of them.  (The rows GEMM reads whole 128-row tiles -- past a
// slice into the next depth's rows, past the last one into forward_layout's +128 -- and stores only the slice's rows.)
template <class Cls>
static int for_each_cls_slice(const ArFast& f, int B, Cls&& cls) {
    const rqb200_ar_config& c = f.cfg;
    const bool pd = c.embed_variant & RQB200_EMB_CLS_PER_DEPTH;
    const int64_t Ms = (int64_t)(pd ? 1 : c.D) * c.H * c.W * B;
    for (int d = 0; d < (pd ? c.D : 1); d++) RQB_TRY(cls(pd ? f.w_cls_d[d] : f.w_cls, f.w.b_cls + (int64_t)d * c.vocab, d, Ms));
    return 0;
}

int ar_fast_forward(ArFast* fp, const int64_t* codes, const int64_t* cond, int B, float* logits_out, float* cond_logits_out, void* wsp,
                    size_t ws_bytes, cudaStream_t st) {
    const ArFast& f = *fp;
    const rqb200_ar_config& c = f.cfg;
    const rqb200_ar_weights& w = f.w;
    const int V = c.vocab;
    if (B < 1) return fail(RQB200_EINVAL, "ar_forward: B must be > 0");
    if (cond_logits_out && (c.cond_len < 2 || !w.w_ccls)) return fail(RQB200_EINVAL, "ar_forward: cond logits need cond_len > 1 and a cond classifier");
    FwdWs ws;
    if (forward_layout(f, B, wsp, ws_bytes, &ws) > ws_bytes) return fail(RQB200_EWORKSPACE, "ar_forward: workspace too small");
    RQB_TRY(forward_passes(f, ws, codes, cond, B, cond_logits_out != nullptr, [&](int64_t Mc) {
        return linear_rows(f, f.w_ccls, ws.XN, Mc, Mc, true, epilogue(GT_F32, w.b_ccls, cond_logits_out), false, st);
    }, st));
    return for_each_cls_slice(f, B, [&](const StreamedWeight& fw, const float* bias, int d, int64_t Ms) {
        return linear_rows(f, fw, ws.XN + (int64_t)d * Ms * c.embed_dim, Ms, Ms, false, epilogue(GT_F32, bias, logits_out + (int64_t)d * Ms * V),
                           false, st);
    });
}

// ---- teacher-forced log-likelihood: the forward's passes, then the classifier in chunks of LOGPROB_CHUNK rows into one fp32 chunk
// buffer, each chunk reduced to log p(target) by logprob_rows_kernel -- the [D*H*W*B, V] logits never exist.  Chunks never straddle
// two depths' slices of per-depth classifiers, and each uses the GEMM the forward uses for its slice (linear_rows), so the log-probs are
// those of the forward's logits.  512 rows: at V = 16384 a 32 MB chunk that stays in the H100's 50 MB L2 between the GEMM's stores
// and the reduction's loads (the chunk sweep is in DESIGN.md section 4).
constexpr int64_t LOGPROB_CHUNK = 512;

struct LpWs {
    FwdWs fwd;
    float* CHUNK;                // [LOGPROB_CHUNK, max(V, cond classifier rows)] f32
    int64_t* TGT;                // [D*H*W*B] targets in the logits' row order, then [(cond_len-1)*B] cond targets
};
static size_t log_prob_layout(const ArFast& f, int B, void* base, size_t cap, LpWs* out) {
    const rqb200_ar_config& c = f.cfg;
    Arena a(base, cap);
    a.off = forward_layout(f, B, base, cap, out ? &out->fwd : nullptr);
    const int64_t vcp = (c.vocab_cond + 127) / 128 * 128, Mh = (int64_t)c.D * c.H * c.W * B, Mc = (int64_t)(c.cond_len - 1) * B;
    float* chunk = a.take<float>(LOGPROB_CHUNK * std::max<int64_t>(c.vocab, f.w.w_ccls ? vcp : 0));
    int64_t* tgt = a.take<int64_t>(Mh + Mc);
    if (out) { out->CHUNK = chunk; out->TGT = tgt; }
    return a.off + 256;
}
size_t ar_fast_log_prob_workspace_bytes(const ArFast* f, int B) { return log_prob_layout(*f, B, nullptr, 0, nullptr); }

int ar_fast_log_prob(ArFast* fp, const int64_t* codes, const int64_t* cond, int B, float* logp_out, float* cond_logp_out, void* wsp,
                     size_t ws_bytes, cudaStream_t st) {
    const ArFast& f = *fp;
    const rqb200_ar_config& c = f.cfg;
    const rqb200_ar_weights& w = f.w;
    const int E = c.embed_dim, D = c.D, HW = c.H * c.W, V = c.vocab, cl = c.cond_len;
    if (B < 1) return fail(RQB200_EINVAL, "ar_log_prob: B must be > 0");
    if (cond_logp_out && (cl < 2 || !w.w_ccls || !cond)) return fail(RQB200_EINVAL, "ar_log_prob: cond log-probs need cond_len > 1, cond and a cond classifier");
    LpWs ws;
    if (log_prob_layout(f, B, wsp, ws_bytes, &ws) > ws_bytes) return fail(RQB200_EWORKSPACE, "ar_log_prob: workspace too small");
    const int64_t Mh = (int64_t)D * HW * B;
    // targets in the logits' row order: row (d*HW + pos)*B + b <- codes[b][pos][d]; cond row s*B + b <- cond[b][s+1]
    RQB_TRY(launch_gather_targets(codes, D, HW, B, 1, D, (int64_t)HW * D, 0, ws.TGT, st));
    if (cond_logp_out) RQB_TRY(launch_gather_targets(cond, 1, cl - 1, B, 0, 1, cl, 1, ws.TGT + Mh, st));
    RQB_TRY(forward_passes(f, ws.fwd, codes, cond, B, cond_logp_out != nullptr, [&](int64_t Mc) {
        for (int64_t r0 = 0; r0 < Mc; r0 += LOGPROB_CHUNK) {
            const int64_t n = std::min(LOGPROB_CHUNK, Mc - r0);
            RQB_TRY(linear_rows(f, f.w_ccls, ws.fwd.XN + r0 * E, n, Mc, true, epilogue(GT_F32, w.b_ccls, ws.CHUNK), false, st));
            // over the vocab_cond real columns: the zero padding rows' logits (0) are no class
            RQB_TRY(launch_logprob_rows(ws.CHUNK, f.w_ccls.N_out, c.vocab_cond, n, ws.TGT + Mh + r0, 1, cond_logp_out + r0, st));
        }
        return 0;
    }, st));
    return for_each_cls_slice(f, B, [&](const StreamedWeight& fw, const float* bias, int d, int64_t Ms) {
        for (int64_t r0 = 0; r0 < Ms; r0 += LOGPROB_CHUNK) {
            const int64_t n = std::min(LOGPROB_CHUNK, Ms - r0), row = (int64_t)d * Ms + r0;
            RQB_TRY(linear_rows(f, fw, ws.fwd.XN + row * E, n, Ms, false, epilogue(GT_F32, bias, ws.CHUNK), false, st));
            RQB_TRY(launch_logprob_rows(ws.CHUNK, V, V, n, ws.TGT + row, 1, logp_out + row, st));
        }
        return 0;
    });
}

// (re)binds the activation tensor maps + graphs to the workspace wsp at batch B
static int bind(ArFast& f, const FastWs& ws, void* wsp, int B) {
    const rqb200_ar_config& c = f.cfg;
    const int E = c.embed_dim;
    drop_graphs(f);
    f.ws_base = nullptr;
    const uint32_t bn = gemm_tc_chunk_rows(f.w_cls, B);      // (every weight of the engine has the classifier's format)
    RQB_TRY(make_tmap_2d(&f.tx_xn, ws.XN, 1, E, B, (uint64_t)E * 2, 64, bn));
    RQB_TRY(make_tmap_2d(&f.tx_att, ws.ATT, 1, E, B, (uint64_t)E * 2, 64, bn));
    RQB_TRY(make_tmap_2d(&f.tx_h, ws.Hh, 1, 4 * E, B, (uint64_t)E * 8, 64, bn));
    RQB_TRY(make_tmap_2d(&f.tx_s, ws.S, 1, c.code_dim, B, (uint64_t)c.code_dim * 2, 64, bn));
    f.ws_base = wsp;
    f.B = B;
    return 0;
}

// one captured graph (captured on first use), or its launches recorded straight onto the stream (RQB200_AR_NO_GRAPH)
static int run_graph(ArFast& f, FastWs& ws, int which, cudaStream_t st) {
    if (!f.use_graph) return record(f, ws, which, st);
    if (!f.graphs[which]) RQB_TRY(capture(f, ws, which, &f.graphs[which]));
    RQB_CUDA(cudaGraphLaunch(f.graphs[which], st));
    g_launches += f.n_nodes[which];      // kernels executed by this replay
    return 0;
}

// prefill: cond tokens, then (start_loc resume) the code tokens of positions < idx_begin (transformers.py:237-239), from a StepState
// with s = idx = 0.  Leaves state.idx = idx_begin, state.s = cond_len + idx_begin, ws.XB = the last prefix token's output rows.
// cv: the positions are those of the canvas window state.cv (code_graph is then G_CODE_CV).
static int prefill_prefix(ArFast& f, FastWs& ws, int idx_begin, cudaStream_t st, bool cv = false) {
    const int T0 = f.cfg.cond_len + idx_begin;
    const int code_graph = cv ? G_CODE_CV : G_CODE;
    if (f.batched_prefill && T0 >= 4 && (int64_t)f.B * T0 <= ws.Mmax) {
        RQB_TRY(body_batched(f, ws, 0, T0, st, cv));
        // state.idx must equal idx_begin for the first head graph
        if (idx_begin > 0) RQB_TRY(launch_pdl(advance_kernel, dim3(1), dim3(32), (size_t)0, st, false, ws.state, 0, idx_begin, 0));
    } else {
        // one cached step each -- causal, so identical to the batched form
        for (int s = 0; s < f.cfg.cond_len; s++) RQB_TRY(run_graph(f, ws, G_COND, st));
        // state.idx must equal (position whose codes feed the body) + 1 while replaying the code-token graph
        for (int j = 1; j <= idx_begin; j++) {
            RQB_TRY(launch_pdl(advance_kernel, dim3(1), dim3(32), (size_t)0, st, false, ws.state, 0, 1, 0));
            RQB_TRY(run_graph(f, ws, code_graph, st));
        }
    }
    return 0;
}

// Runs of kept positions shorter than this many code tokens are appended to the body cache by replaying the single-token body graph
// once per token; longer runs take one batched body pass (body_batched at T0 > 0).  scripts/bench_keep.py --sweep, in1400m B = 64 on
// an H100 80GB HBM3 at 700 W, runs of exactly k: batched / token by token = 1.03 at k = 5, 0.90 at k = 6, 0.68 at k = 8.
constexpr int APPEND_BATCHED_MIN = 6;

// A canvas larger than the grid is walked in segments: consecutive sampled positions whose windows share an origin continue one KV
// cache (the window positions between them are appended as kept code tokens, as on the grid); a new origin restarts the body sequence
// with a prefill of the window's prefix.  On the grid every origin is 0: one segment, the grid graphs, the launches of a grid call.
int ar_fast_sample(ArFast* f, const int64_t* partial, const int64_t* cond, int B, int idx_begin, int idx_end, int resume,
                   float temperature, const int32_t* top_k, const float* top_p, const float* noise, int64_t noise_stride,
                   float* logits_out, const int64_t* force, int64_t* out, void* wsp, size_t ws_bytes, cudaStream_t st, int cfg_n,
                   float cfg_s, const uint8_t* keep, const uint8_t* sampled, int Ht, int Wt) {
    const rqb200_ar_config& c = f->cfg;
    const int D = c.D, cl = c.cond_len;
    const bool cv = Ht != c.H || Wt != c.W;
    if (B > 256) return fail(RQB200_EINVAL, "ar fast tier: batch must be in [1,256] per call");
    FastWs ws;
    size_t need = fast_layout(*f, B, wsp, ws_bytes, &ws);
    if (need > ws_bytes) return fail(RQB200_EWORKSPACE, "ar_sample: workspace too small");
    if (!resume && out != partial)
        RQB_CUDA(cudaMemcpyAsync(out, partial, (size_t)B * Ht * Wt * D * sizeof(int64_t), cudaMemcpyDeviceToDevice, st));
    int first = idx_begin;                            // the span's first sampled position
    while (first < idx_end && !plan_sampled(sampled, first)) first++;
    if (first >= idx_end) return 0;                   // nothing to sample: `out` holds partial
    // prev: the last sampled position of the call before this span (its code tokens are the body's next input); none: the prefill runs
    // at the first sampled position
    int prev = resume ? plan_prev(sampled, idx_begin) : -1;
    if (f->ws_base != wsp || f->B != B) {
        if (prev >= 0) return fail(RQB200_ESTATE, "ar_sample: resume on a workspace / batch the engine is not bound to");
        RQB_TRY(bind(*f, ws, wsp, B));
    }
    // the current segment's window origin and the window position of prev (on the grid: 0 and prev)
    int cur_org = 0, prev_p = -1;
    win_locate(prev >= 0 ? prev : first, c.H, c.W, Wt, Ht, &cur_org, &prev_p);
    if (prev < 0) prev_p = -1;
    StepState h = {};
    h.s = 0; h.idx = 0; h.step = 0;
    h.cond = cond; h.codes = out; h.force = force; h.noise = noise; h.logits_out = logits_out; h.noise_stride = noise_stride;
    h.temperature = temperature;
    h.cfg_n = cfg_n; h.cfg_scale = cfg_s;        // (the head graphs' samplers read them: no recapture between guided and unguided calls)
    h.keep = keep;
    for (int d = 0; d < D; d++) { h.top_k[d] = top_k[d]; h.top_p[d] = top_p[d]; }
    h.cv = CanvasMap{c.W, Wt, cur_org, Ht * Wt};
    RQB_TRY(launch_pdl(init_state_kernel, dim3(1), dim3(32), (size_t)0, st, false, ws.state, h, prev >= 0 ? 1 : 0));
    if (f->trace && prev < 0) RQB_CUDA(cudaMemsetAsync(ws.trace, 0, (size_t)4 * TR_CAP * sizeof(long long), st));
    const int head_graph = logits_out ? (cv ? G_HEAD_LOGITS_CV : G_HEAD_LOGITS) : (cv ? G_HEAD_CV : G_HEAD);
    const int code_graph = cv ? G_CODE_CV : G_CODE;
    // the host's copy of state.idx / state.step: a head graph leaves idx one past its (window) position; step counts the span's canvas
    // tokens, sampled or not, so that noise and logits_out stay indexed by token
    int cur_idx = prev >= 0 ? prev_p + 1 : 0, cur_step = 0;
    auto advance_to = [&](int idx, int step) -> int {
        if (idx == cur_idx && step == cur_step) return 0;
        RQB_TRY(launch_pdl(advance_kernel, dim3(1), dim3(32), (size_t)0, st, false, ws.state, 0, idx - cur_idx, step - cur_step));
        cur_idx = idx; cur_step = step;
        return 0;
    };
    for (int b = first; b < idx_end; b++) {
        if (!plan_sampled(sampled, b)) continue;
        int org, p;
        win_locate(b, c.H, c.W, Wt, Ht, &org, &p);
        if (prev >= 0 && org != cur_org) {                                 // a new window: its body sequence starts over
            RQB_TRY(launch_pdl(segment_kernel, dim3(1), dim3(32), (size_t)0, st, false, ws.state, org));
            cur_org = org; cur_idx = 0;
            prev = -1;
        }
        if (prev < 0) {
            RQB_TRY(prefill_prefix(*f, ws, p, st, cv));                    // cond tokens and window positions [0, p); state.idx = p
            cur_idx = p;
        } else if (f->batched_prefill && p - prev_p >= APPEND_BATCHED_MIN && (int64_t)B * (p - prev_p) <= ws.Mmax) {
            RQB_TRY(body_batched(*f, ws, cl + prev_p, p - prev_p, st, cv)); // the code tokens of window positions [prev_p, p) in one pass
        } else {
            for (int j = prev_p; j < p; j++) {                             // one body step each (state.idx == j + 1: position j)
                RQB_TRY(advance_to(j + 1, cur_step));
                RQB_TRY(run_graph(*f, ws, code_graph, st));
            }
        }
        RQB_TRY(advance_to(p, (b - idx_begin) * D));
        RQB_TRY(run_graph(*f, ws, head_graph, st));                        // D head steps + sampling; advances idx, step
        cur_idx = p + 1; cur_step += D;
        prev = b; prev_p = p;
    }
    return 0;
}

int ar_fast_step(ArFast* f, const int64_t* xs, int64_t xs_stride, const int64_t* cond, int B, int idx, int d, int restart,
                 float* logits_out, void* wsp, size_t ws_bytes, cudaStream_t st) {
    const rqb200_ar_config& c = f->cfg;
    const int D = c.D, HW = c.H * c.W, cl = c.cond_len;
    if (B < 1 || B > 256) return fail(RQB200_EINVAL, "ar fast tier: batch must be in [1,256] per call");
    FastWs ws;
    if (fast_layout(*f, B, wsp, ws_bytes, &ws) > ws_bytes) return fail(RQB200_EWORKSPACE, "ar_step: workspace too small");
    if (f->ws_base != wsp || f->B != B) {
        if (!restart) return fail(RQB200_ESTATE, "ar_step: continuing on a workspace / batch the engine is not bound to");
        RQB_TRY(bind(*f, ws, wsp, B));
    }
    // the codes this step consumes: restart -> positions [0, idx) for the prefill; d == 0 -> position idx-1 for the body step;
    // d > 0 -> codes 0 .. d-1 of position idx for the head token
    const int64_t lo = restart ? 0 : (d == 0 ? (int64_t)(idx - 1) * D : (int64_t)idx * D);
    const int64_t hi = d == 0 ? (int64_t)idx * D : (int64_t)idx * D + d;
    StepState v = {};
    v.cond = cond; v.codes = ws.CODES; v.logits_out = logits_out;
    v.s = restart ? 0 : (d == 0 ? cl + idx - 1 : cl + idx);   // body keys cached before the token the next body step appends
    v.idx = restart ? 0 : idx;                                  // (a restart's prefill advances idx itself, as in ar_fast_sample)
    RQB_TRY(launch_pdl(step_ingest_kernel, dim3(B), dim3(128), (size_t)0, st, false, ws.state, v, restart, xs, xs_stride, lo, hi,
                       (int64_t)HW * D));
    if (restart) {
        if (f->trace) RQB_CUDA(cudaMemsetAsync(ws.trace, 0, (size_t)4 * TR_CAP * sizeof(long long), st));
        RQB_TRY(prefill_prefix(*f, ws, idx, st));
    } else if (d == 0) {
        RQB_TRY(run_graph(*f, ws, G_CODE, st));                  // body step on the codes of position idx-1
    }
    return run_graph(*f, ws, G_HEAD_STEP + d, st);
}

int ar_fast_trace(ArFast* f, long long* out_host, int cap_launches, char* names, int names_cap) {
    if (!f || !f->trace || !f->tr_base) return 0;
    const int n = std::min(cap_launches, TR_CAP);
    if (cudaMemcpy(out_host, f->tr_base, (size_t)n * 4 * sizeof(long long), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
    std::string all;
    for (int i = 0; i < n; i++) {
        all += i < (int)f->tr_names.size() ? f->tr_names[i] : "";
        all += '\n';
    }
    if (names && names_cap > 0) {
        const size_t k = std::min(all.size(), (size_t)names_cap - 1);
        memcpy(names, all.data(), k);
        names[k] = 0;
    }
    return n;
}

}  // namespace rqb

// ---- diagnostic entry points (tests/test_gpu_ar_kernels.py): one launch of a step or batched-pass kernel through the launcher the
// engine calls, without the PDL attribute and the trace

extern "C" int rqb200_dbg_attn_step(int form, const float* part, int S, const float* bqkv, void* kc, void* vc, void* att, int B, int E, int Tmax,
                                    const int* t_dev, int t_host, int fmt, void* stream) {
    using namespace rqb;
    if (form < 0 || form > 2 || fmt < 0 || fmt > 1 || B < 1 || S < 0 || E < 64 || E % 64 || Tmax < 1 || Tmax > FAST_MAXT)
        return fail(RQB200_EINVAL, "dbg_attn_step: need form 0..2, fmt 0..1, B >= 1, S >= 0, E % 64 == 0, 1 <= Tmax <= 2048");
    if (!bqkv || !kc || !vc || !att || (S > 0 && !part)) return fail(RQB200_EINVAL, "dbg_attn_step: null argument");
    if (!t_dev && (t_host < 0 || t_host >= Tmax)) return fail(RQB200_EINVAL, "dbg_attn_step: t outside [0, Tmax)");
    if (form == 2 && Tmax - 1 > AF2_MAXROWS) return fail(RQB200_EINVAL, "dbg_attn_step: form 2 takes at most 320 cached rows (Tmax <= 321)");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "dbg_attn_step: no CUDA device");
    return attn(form, part, S, bqkv, (h16*)kc, (h16*)vc, (h16*)att, B, E, Tmax, t_dev, t_host, fmt, false, nullptr, (cudaStream_t)stream);
}

extern "C" int rqb200_dbg_prefill_attn(const void* qkv, void* kc, void* vc, void* att, int G, int T, int E, int Tmax, int fmt, void* stream) {
    using namespace rqb;
    if (fmt < 0 || fmt > 1 || G < 1 || T < 1 || T > FAST_MAXT || E < 64 || E % 64 || (int64_t)ceil_div(T, 64) * G * (E / 64) > INT32_MAX)
        return fail(RQB200_EINVAL, "dbg_prefill_attn: need fmt 0..1, G >= 1, 1 <= T <= 2048, E % 64 == 0");
    if (!qkv || !att || !kc != !vc) return fail(RQB200_EINVAL, "dbg_prefill_attn: null qkv / att, or only one of kc / vc");
    if (kc && T > Tmax) return fail(RQB200_EINVAL, "dbg_prefill_attn: T > Tmax");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "dbg_prefill_attn: no CUDA device");
    return prefill_attn((const h16*)qkv, (h16*)kc, (h16*)vc, (h16*)att, G, T, E, Tmax, fmt, false, (cudaStream_t)stream);
}

extern "C" int rqb200_dbg_append_attn(const void* qkv, void* kc, void* vc, void* att, int G, int T0, int T, int E, int Tmax, int fmt,
                                      void* stream) {
    using namespace rqb;
    if (fmt < 0 || fmt > 1 || G < 1 || T < 1 || T0 < 0 || E < 64 || E % 64 || Tmax > FAST_MAXT || T0 + T > Tmax ||
        (int64_t)ceil_div(T, 64) * G * (E / 64) > INT32_MAX)
        return fail(RQB200_EINVAL, "dbg_append_attn: need fmt 0..1, G >= 1, T >= 1, T0 >= 0, T0 + T <= Tmax <= 2048, E % 64 == 0");
    if (!qkv || !att || !kc || !vc) return fail(RQB200_EINVAL, "dbg_append_attn: null argument");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "dbg_append_attn: no CUDA device");
    return prefill_attn((const h16*)qkv, (h16*)kc, (h16*)vc, (h16*)att, G, T, E, Tmax, fmt, false, (cudaStream_t)stream, T0);
}

extern "C" int rqb200_dbg_ln(int form, const float* x_in, const float* partial, int S, const float* bias, const float* extra, float* x_out,
                             const float* g, const float* b, void* xn, int64_t rows, int E, int fmt, void* stream) {
    using namespace rqb;
    if (form < 0 || form > 2 || fmt < 0 || fmt > 1 || rows < 1 || rows > INT32_MAX || S < 0 || E < 128 || E % 128 || E > 4608)
        return fail(RQB200_EINVAL, "dbg_ln: need form 0..2, fmt 0..1, 1 <= rows < 2^31, S >= 0, E % 128 == 0, E <= 4608");
    if ((S > 0 && !partial) || (xn && (!g || !b))) return fail(RQB200_EINVAL, "dbg_ln: null partial, or xn without g / b");
    if (form != 1 && (S > 0 || partial || bias || !x_in))
        return fail(RQB200_EINVAL, "dbg_ln: forms 0 and 2 (the batched passes' LayerNorm) take x_in and no partials or bias");
    int dev = 0, n_sm = 0;
    if (rqb200_device_count() <= 0 || cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
        return fail(RQB200_ENODEV, "dbg_ln: no CUDA device");
    const cudaStream_t st = (cudaStream_t)stream;
    if (form == 1) return ln((int)rows, x_in, partial, S, bias, extra, x_out, g, b, (h16*)xn, E, fmt, false, nullptr, PrefetchList{}, st);
    if (form == 2) return ln_rows_warp(rows, x_in, extra, x_out, g, b, (h16*)xn, E, fmt, n_sm, st);
    return ln_rows(rows, x_in, extra, x_out, g, b, (h16*)xn, E, fmt, n_sm, st);
}

extern "C" int rqb200_dbg_act_reduce(const float* partial, int S, const float* bias, void* h, int B, int N, int fmt, void* stream) {
    using namespace rqb;
    if (fmt < 0 || fmt > 1 || S < 0 || B < 1 || N < 4 || N % 4)
        return fail(RQB200_EINVAL, "dbg_act_reduce: need fmt 0..1, S >= 0, B >= 1, N % 4 == 0");
    if (!bias || !h || (S > 0 && !partial)) return fail(RQB200_EINVAL, "dbg_act_reduce: null argument");
    if (rqb200_device_count() <= 0) return fail(RQB200_ENODEV, "dbg_act_reduce: no CUDA device");
    return act_reduce(partial, S, bias, (h16*)h, B, N, fmt, false, nullptr, (cudaStream_t)stream);
}
