// P1, second form of the fused residual-quantisation search.
//
// Why: the 2x4 register tile of rq_quantize_kernel is bound by shared-memory wavefronts (6 LDS.128 = 24 wavefronts per 32 FFMA
// instructions).  Balance needs F >= 16 L per thread, i.e. an 8x8
// register tile (16 LDS.128 per 256 FFMA), which needs a CTA tile of 64 vectors x 256 codewords for 8 warps; the 1 KB codeword
// rows then no longer fit the shared memory whole, so the codebook is streamed in 32-channel slabs (TMA 2-D boxes of 256 rows x
// 128 B, SWIZZLE_128B -> conflict-free 128-bit reads) while the 64 accumulators of a thread stay live over the 8 slabs of a
// codeword block.  64 vectors per CTA would leave N=4096 with 64 CTAs for 132 SMs, so two CTAs of a cluster share one group of
// vectors and split the CODEBOOK; after every depth they exchange their 64 (distance, index) candidates through distributed
// shared memory and both apply the same residual update.
//
// Arithmetic is kept operation-for-operation identical to rq_quantize_kernel (csrc/rq_search.cu): the dot product of a
// (vector, codeword) pair accumulates channels 0..255 in order in one fp32 chain, ||e||^2 and ||r||^2 use the same partial-sum
// trees, dist = fmaf(-2, x.e, ||r||^2 + ||e||^2), argmin is the lexicographic minimum of (dist, index), the residual and the
// aggregate are updated by the same sequence of fp32 subtractions / additions  ==> bit-identical codes and aggregates, so the
// first kernel (pinned to the reference's golden vectors) is this one's oracle on the GPU.
// Reference: rqvae/models/rqvae/quantizations.py:43-69 (distances, argmin), :237-271 (depth loop).
#include "kernels.h"
#include "tc_common.cuh"

namespace rqb {

constexpr int R2_C = 256;          // channels
constexpr int R2_TN = 64;          // vectors per cluster (both CTAs hold a copy of their residuals)
constexpr int R2_KB = 256;         // codewords per accumulation block
constexpr int R2_CC = 32;          // channels per slab (128 B rows)
constexpr int R2_NCH = R2_C / R2_CC;
constexpr int R2_STAGES = 3;
constexpr int R2_STAGE_BYTES = R2_KB * R2_CC * 4;     // 32 KB
constexpr int R2_PITCH = 260;
constexpr int R2_MAXEN = 8192;     // codewords per CTA whose ||e||^2 fit the shared table  (every K_d <= 16384)
constexpr int R2_CONSUMERS = 256;
constexpr int R2_THREADS = R2_CONSUMERS;      // 8 warps = 2 per scheduler partition: the 8x8 tile needs ~200 registers per thread

struct Rq2Smem {
    float resid[R2_TN][R2_PITCH];
    float en[R2_MAXEN];
    float xn[R2_TN];
    float wbest_d[4][R2_TN];
    int wbest_k[4][R2_TN];
    float rc_d[2][R2_TN];          // candidates pushed by the peer CTA (double-buffered by depth parity)
    int rc_k[2][R2_TN];
    int win[R2_TN];
    uint64_t full[R2_STAGES], empty[R2_STAGES], peer_bar[2];
};

__device__ __forceinline__ void r2_consumer_sync() { __syncthreads(); }
__device__ __forceinline__ void r2_cluster_sync() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t r2_mapa(uint32_t local_addr, uint32_t rank) {
    uint32_t ra;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(local_addr), "r"(rank));
    return ra;
}
__device__ __forceinline__ void r2_st_remote_f32(uint32_t addr, float v) {
    asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory");
}
__device__ __forceinline__ void r2_st_remote_s32(uint32_t addr, int v) {
    asm volatile("st.shared::cluster.s32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ void r2_arrive_remote(uint32_t bar_addr) {
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(bar_addr) : "memory");
}
__device__ __forceinline__ void r2_wait_cluster(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "R2_WAIT:\n"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%0], %1;\n"
        "@p bra R2_DONE;\n"
        "bra R2_WAIT;\n"
        "R2_DONE:\n"
        "}\n" ::"r"(tc::smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// one TMA descriptor per codebook table (RqTables order)
struct Rq2Maps {
    CUtensorMap m[RQ_MAX_TABLES];
};

__device__ __forceinline__ bool r2_before(float d, int k, float od, int ok) {   // (od, ok) < (d, k) lexicographically
    return od < d || (od == d && ok < k);
}

__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(R2_THREADS, 1)
rq_quantize2_kernel(const __grid_constant__ Rq2Maps tms, const RqTables tabs, const float* __restrict__ x, int64_t N, int D,
                    int64_t* __restrict__ codes, float* __restrict__ quant_list, float* __restrict__ resid_out) {
    extern __shared__ uint8_t smem_raw[];
    // 1024 B alignment (swizzle atom) by an OFFSET into the shared array: keeps the pointers in the shared address space, so the
    // hot loop compiles to LDS.128 and not to generic LD
    uint8_t* ring = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);
    Rq2Smem& s = *reinterpret_cast<Rq2Smem*>(ring + R2_STAGES * R2_STAGE_BYTES);

    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const uint32_t rank = blockIdx.x & 1u;                       // cluster = 2 consecutive CTAs along x
    const int64_t n0 = (int64_t)(blockIdx.x >> 1) * R2_TN;
    const int nvalid = (int)min((int64_t)R2_TN, N - n0);
    // the codebook split of depth d: this CTA's codeword blocks [blk0, blk0 + nb) of table tabs.of(d)
    auto split = [&](int d, int& blk0, int& nb) {
        const int nblk = (tabs.K[tabs.of(d)] + R2_KB - 1) / R2_KB;
        const int nb0 = (nblk + 1) / 2;
        blk0 = rank == 0 ? 0 : nb0;
        nb = rank == 0 ? nb0 : nblk - nb0;
    };

    if (t == 0) {
        for (int i = 0; i < R2_STAGES; i++) { tc::mbar_init(&s.full[i], 1); tc::mbar_init(&s.empty[i], 8); }
        tc::mbar_init(&s.peer_bar[0], R2_TN);
        tc::mbar_init(&s.peer_bar[1], R2_TN);
        tc::fence_barrier_init();
        for (int i = 0; i < tabs.n; i++) tc::prefetch_tmap(&tms.m[i]);
    }
    __syncthreads();
    r2_cluster_sync();                                           // the peer's barriers exist before anything is pushed to them

    // producer duty: lane 0 of warp 0 keeps R2_STAGES - 1 slabs in flight; before chunk `it` it (re)fills the slot chunk it-1 used,
    // which blocks it only while another warp is still reading that slot (warp 0 is never more than one chunk ahead of the slowest)
    // slabs are streamed depth by depth; thread 0 keeps a cursor (pd, pb, pcc) = (depth, block, slab) of the next slab to issue
    int total = 0;
    for (int d = 0; d < D; d++) {
        int b0, n;
        split(d, b0, n);
        total += n * R2_NCH;
    }
    int pd = 0, pb = 0, pcc = 0, p_blk0, p_nb;
    split(0, p_blk0, p_nb);
    auto issue = [&](int nx) {
        while (p_nb == 0) split(++pd, p_blk0, p_nb);             // a depth whose table leaves this CTA no block
        const int st = nx % R2_STAGES;
        tc::mbar_wait(&s.empty[st], ((nx / R2_STAGES) & 1) ^ 1);
        tc::mbar_expect_tx(&s.full[st], R2_STAGE_BYTES);
        tc::tma_load_2d(ring + st * R2_STAGE_BYTES, &tms.m[tabs.of(pd)], &s.full[st], pcc * R2_CC, (p_blk0 + pb) * R2_KB,
                        tc::L2_EVICT_LAST);
        if (++pcc == R2_NCH) {
            pcc = 0;
            if (++pb == p_nb) { pb = 0; if (++pd < D) split(pd, p_blk0, p_nb); }
        }
    };
    if (t == 0)
        for (int nx = 0; nx < R2_STAGES - 1 && nx < total; nx++) issue(nx);
    {
        // ---------------------------------------------------------------- consumers (8 warps)
        const int wv = warp >> 2, wk = warp & 3, lv = lane >> 3, lk = lane & 7;
        const int vb = wv * 32 + lv * 8;                         // this thread's 8 vectors: vb + i
        // residual tile <- x (zero padded)
        for (int i = t; i < R2_TN * (R2_C / 4); i += R2_CONSUMERS) {
            const int v = i / (R2_C / 4), c4 = i % (R2_C / 4);
            float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
            if (v < nvalid) val = *reinterpret_cast<const float4*>(x + (n0 + v) * R2_C + c4 * 4);
            *reinterpret_cast<float4*>(&s.resid[v][c4 * 4]) = val;
        }
        // ||e||^2 of this CTA's codewords of depth d's table, the partial-sum tree of rq_quantize_kernel: 4 lanes x 64 sequential
        // fmaf, (p0+p1)+(p2+p3)
        auto fill_en = [&](int d) {
            int blk0, nb;
            split(d, blk0, nb);
            const int ti = tabs.of(d), kbase = blk0 * R2_KB;
            const float* cb = tabs.cb[ti];
            const int nk = min(nb * R2_KB, tabs.K[ti] - kbase);
            const int part = t & 3;
            for (int r0 = 0; r0 < nk; r0 += R2_CONSUMERS / 4) {
                const int r = r0 + (t >> 2);
                float a = 0.f;
                if (r < nk) {
                    const float4* row = reinterpret_cast<const float4*>(cb + (int64_t)(kbase + r) * R2_C + part * 64);
                    float4 w[16];
#pragma unroll
                    for (int c = 0; c < 16; c++) w[c] = __ldg(row + c);
#pragma unroll
                    for (int c = 0; c < 16; c++) {
                        a = fmaf(w[c].x, w[c].x, a); a = fmaf(w[c].y, w[c].y, a);
                        a = fmaf(w[c].z, w[c].z, a); a = fmaf(w[c].w, w[c].w, a);
                    }
                }
                a += __shfl_xor_sync(0xffffffffu, a, 1);
                a += __shfl_xor_sync(0xffffffffu, a, 2);
                if (part == 0 && r < nk) s.en[r] = a;
            }
        };
        fill_en(0);
        r2_consumer_sync();
        auto norms_x = [&]() {       // ||r||^2 per vector: lane sums channels lane, lane+32, ... then the xor butterfly (as rq_search.cu)
#pragma unroll
            for (int i = 0; i < 8; i++) {
                const int v = warp * 8 + i;
                float a = 0.f;
#pragma unroll
                for (int c = lane; c < R2_C; c += 32) a = fmaf(s.resid[v][c], s.resid[v][c], a);
                a = warp_sum(a);
                if (lane == 0) s.xn[v] = a;
            }
        };
        norms_x();
        r2_consumer_sync();

        float best_d[8];
        int best_k[8];
#pragma unroll
        for (int i = 0; i < 8; i++) { best_d[i] = INFINITY; best_k[i] = 0x7fffffff; }
        int it = 0;
        for (int depth = 0; depth < D; depth++) {
            const int ti = tabs.of(depth), K = tabs.K[ti];
            const float* cb = tabs.cb[ti];
            int blk0, nb;
            split(depth, blk0, nb);
            const int kbase = blk0 * R2_KB;
            for (int b = 0; b < nb; b++) {
                float acc[8][8];
#pragma unroll
                for (int i = 0; i < 8; i++)
#pragma unroll
                    for (int j = 0; j < 8; j++) acc[i][j] = 0.f;
#pragma unroll 1
                for (int cc = 0; cc < R2_NCH; cc++, it++) {
                    const int st = it % R2_STAGES;
                    if (t == 0 && it + R2_STAGES - 1 < total) issue(it + R2_STAGES - 1);
                    __syncwarp();
                    tc::mbar_wait(&s.full[st], (it / R2_STAGES) & 1);
                    const uint8_t* slab = ring + st * R2_STAGE_BYTES + (wk * 64 + lk) * 128;     // row of codeword j: + j * 8 * 128
#pragma unroll 2
                    for (int c4 = 0; c4 < R2_CC / 4; c4++) {
                        float4 r4[8], e4[8];
#pragma unroll
                        for (int i = 0; i < 8; i++) r4[i] = *reinterpret_cast<const float4*>(&s.resid[vb + i][cc * R2_CC + c4 * 4]);
#pragma unroll
                        for (int j = 0; j < 8; j++)      // SWIZZLE_128B: 16-byte chunk c4 of row r sits at chunk c4 ^ (r & 7); r & 7 == lk
                            e4[j] = *reinterpret_cast<const float4*>(slab + j * 1024 + ((c4 ^ lk) << 4));
#pragma unroll
                        for (int i = 0; i < 8; i++)
#pragma unroll
                            for (int j = 0; j < 8; j++) {
                                acc[i][j] = fmaf(r4[i].x, e4[j].x, acc[i][j]);
                                acc[i][j] = fmaf(r4[i].y, e4[j].y, acc[i][j]);
                                acc[i][j] = fmaf(r4[i].z, e4[j].z, acc[i][j]);
                                acc[i][j] = fmaf(r4[i].w, e4[j].w, acc[i][j]);
                            }
                    }
                    __syncwarp();
                    if (lane == 0) tc::mbar_arrive(&s.empty[st]);
                }
                // distances of this block, codewords in increasing index per thread (strict < keeps the first on ties)
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    const int kloc = b * R2_KB + wk * 64 + lk + 8 * j;       // index within this CTA's codewords
                    const int kk = kbase + kloc;
                    if (kk < K) {
                        const float en = s.en[kloc];
#pragma unroll
                        for (int i = 0; i < 8; i++) {
                            const float dist = fmaf(-2.0f, acc[i][j], s.xn[vb + i] + en);
                            if (dist < best_d[i]) { best_d[i] = dist; best_k[i] = kk; }
                        }
                    }
                }
            }
            // ---- end of one depth: argmin over the 8 lk lanes, the 4 wk warps, the 2 CTAs; then the residual update
#pragma unroll
            for (int i = 0; i < 8; i++) {
#pragma unroll
                for (int o = 4; o > 0; o >>= 1) {
                    const float od = __shfl_xor_sync(0xffffffffu, best_d[i], o);
                    const int ok = __shfl_xor_sync(0xffffffffu, best_k[i], o);
                    if (r2_before(best_d[i], best_k[i], od, ok)) { best_d[i] = od; best_k[i] = ok; }
                }
                if (lk == 0) { s.wbest_d[wk][vb + i] = best_d[i]; s.wbest_k[wk][vb + i] = best_k[i]; }
                best_d[i] = INFINITY;
                best_k[i] = 0x7fffffff;
            }
            r2_consumer_sync();
            const int par = depth & 1;
            if (t < R2_TN) {
                float d = s.wbest_d[0][t];
                int k = s.wbest_k[0][t];
#pragma unroll
                for (int w = 1; w < 4; w++) {
                    const float od = s.wbest_d[w][t];
                    const int ok = s.wbest_k[w][t];
                    if (r2_before(d, k, od, ok)) { d = od; k = ok; }
                }
                // push this CTA's candidate to the peer, then wait for the peer's
                const uint32_t peer = rank ^ 1u;
                r2_st_remote_f32(r2_mapa(tc::smem_u32(&s.rc_d[par][t]), peer), d);
                r2_st_remote_s32(r2_mapa(tc::smem_u32(&s.rc_k[par][t]), peer), k);
                r2_arrive_remote(r2_mapa(tc::smem_u32(&s.peer_bar[par]), peer));
                r2_wait_cluster(&s.peer_bar[par], (uint32_t)((depth >> 1) & 1));
                const float od = s.rc_d[par][t];
                const int ok = s.rc_k[par][t];
                if (r2_before(d, k, od, ok)) { d = od; k = ok; }
                const int kw = k == 0x7fffffff ? 0 : k;      // all-NaN row: pinned to 0 like rq_quantize_kernel
                s.win[t] = kw;
                if (rank == 0 && t < nvalid) codes[(n0 + t) * D + depth] = (int64_t)kw;
            }
            r2_consumer_sync();
            for (int v = 0; v < R2_TN; v++) {                    // thread t <-> channel t
                const float q = __ldg(cb + (int64_t)s.win[v] * R2_C + t);
                s.resid[v][t] -= q;                                          // residual_feature.sub_(quant)   :264
                if (quant_list != nullptr && rank == 0 && v < nvalid) {
                    // aggregated_quants.add_(quant) :265 -- the running sum is re-read from the previous depth's slice (written by
                    // this thread): 0 + q0, (q0) + q1, ... the same fp32 additions as a register accumulator
                    const float prev = depth > 0 ? quant_list[((int64_t)(depth - 1) * N + n0 + v) * R2_C + t] : 0.f;
                    quant_list[((int64_t)depth * N + n0 + v) * R2_C + t] = prev + q;
                }
            }
            r2_consumer_sync();
            if (depth + 1 < D) {
                // a new table: refill ||e||^2 (en[] is no longer read: every thread passed the syncs since this depth's distances)
                if (tabs.of(depth + 1) != ti) fill_en(depth + 1);
                norms_x();
            }
            r2_consumer_sync();
        }
        if (resid_out != nullptr && rank == 0)
            for (int v = 0; v < nvalid; v++) resid_out[(n0 + v) * R2_C + t] = s.resid[v][t];
    }
    __syncwarp();
    r2_cluster_sync();                                           // nobody leaves while the peer may still push into this CTA
}

bool rq_quantize2_supported(int64_t N, const RqTables& tabs, int C) {
    if (C != R2_C || N <= 0) return false;
    for (int i = 0; i < tabs.n; i++)
        if (tabs.K[i] > 2 * R2_MAXEN) return false;
    return true;
}

int launch_rq_quantize2(const float* x, const RqTables& tabs, int64_t N, int C, int D, int64_t* codes, float* quant_list,
                        float* resid_out, cudaStream_t st) {
    if (!rq_quantize2_supported(N, tabs, C)) return fail(RQB200_EINVAL, "rq_quantize2: need C == 256 and every K <= 16384");
    Rq2Maps tms{};
    for (int i = 0; i < tabs.n; i++)
        RQB_TRY(make_tmap_2d(&tms.m[i], tabs.cb[i], 2, (uint64_t)R2_C, (uint64_t)tabs.K[i], (uint64_t)R2_C * 4, R2_CC, R2_KB));
    const size_t smem = (size_t)R2_STAGES * R2_STAGE_BYTES + sizeof(Rq2Smem) + 1024;
    RQB_ENSURE_SMEM(smem, rq_quantize2_kernel);
    const unsigned grid = 2u * (unsigned)ceil_div(N, R2_TN);
    rq_quantize2_kernel<<<grid, R2_THREADS, smem, st>>>(tms, tabs, x, N, D, codes, quant_list, resid_out);
    return check_launch("rq_quantize2");
}

}  // namespace rqb
