// Fast tier: the VAE's spatial attention (AttnBlock core, layers.py:158-182) on the tensor cores, for maps past 1024 tokens.
//
// Same contract as launch_vae_attn (conv_kernels.cu): qkv [B, HW, 3C] fp32 (q | k | v per pixel) -> out [B, HW, C] fp32 =
// softmax_j(q_i k_j * s) v_j with s = float(1 / sqrt(double C)).  One head of dimension C (128 | 256 | 384 | 512), any HW >= 1, no
// workspace: the [HW, HW] scores are never formed.
//
// Flash form: one CTA per (64-query tile, image) walks the keys in tiles of 32 with an online softmax (running row maximum m and
// sum l, the output rescaled by exp(m_old - m_new) whenever the maximum moves).  Operands are fp16, rounded from the fp32 qkv in
// shared memory; products run on mma.sync m16n8k16 with fp32 accumulation; scores, softmax and the output accumulator are fp32.
// The fp32 K and V tiles come in by cp.async into one fp32 staging buffer, each one's load running under the previous phase's
// MMAs (V_t under the S phase, K_t+1 under the PV phase), and are rounded to the fp16 operand tile from there.  Per key tile:
//   S phase   K tile -> fp16; warp w forms S[16 (w % 4) .. +16, 16 (w / 4) .. +16] = Q K^T over all C, scaled, into fp32 smem
//   softmax   4 threads per query row: tile maximum, new running maximum, P = exp(S - m) as fp16, l and the rescale factor
//   PV phase  V tile -> fp16; warp w rescales and accumulates O[16 (w % 4) .. +16, (w / 4) C / 2 .. +C / 2] += P V: the C / 2
//             columns of a warp's 16 rows are its C / 4 accumulator registers per thread (128 at C = 512)
// The last key tile and query tile are partial: keys past HW score -inf and are staged as zero rows; query rows past HW are not
// stored.
#include "kernels.h"

namespace rqb {

constexpr int AT_BQ = 64, AT_BK = 32, AT_THREADS = 256;
constexpr int AT_SLD = AT_BK + 1;          // fp32 score row (floats)
constexpr int AT_PLD = AT_BK + 8;          // fp16 probability row (halves): 80 B, eight rows on distinct 16 B bank groups

template <int C>
struct AttnTcSmem {
    static constexpr int LD = C + 8;                                  // fp16 operand row (halves): 16 B off a 128 B multiple
    static constexpr int Q = 0;
    static constexpr int KV = Q + AT_BQ * LD * 2;
    static constexpr int S = KV + AT_BK * LD * 2;
    static constexpr int P = S + AT_BQ * AT_SLD * 4;
    static constexpr int STATS = P + AT_BQ * AT_PLD * 2;              // m, l, alpha per query row
    static constexpr int F = STATS + 3 * AT_BQ * 4;                   // fp32 staging of the next K or V tile [AT_BK][C]
    static constexpr int BYTES = F + AT_BK * C * 4;
};

__device__ __forceinline__ void at_ldsm_x4(uint32_t (&r)[4], const void* p) {
    const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void at_ldsm_x4_t(uint32_t (&r)[4], const void* p) {
    const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
// D (+)= A B, m16n8k16, fp16 operands, fp32 accumulators
__device__ __forceinline__ void at_mma(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// rows [r0, r0 + R) of one third of qkv (column offset off) -> fp16 smem [R][C + 8]; rows at or past HW are zero
template <int C, int R>
__device__ __forceinline__ void at_stage(__half* dst, const float* __restrict__ src, int r0, int HW, int off) {
    constexpr int C4 = C / 4, N4 = R * C4;
    static_assert(N4 % (4 * AT_THREADS) == 0, "at_stage: whole unrolled rounds");
#pragma unroll 1
    for (int i0 = threadIdx.x; i0 < N4; i0 += 4 * AT_THREADS) {
        float4 v[4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int i = i0 + u * AT_THREADS, r = i / C4, c4 = i % C4;
            v[u] = r0 + r < HW ? __ldg(reinterpret_cast<const float4*>(src + (int64_t)(r0 + r) * 3 * C + off) + c4)
                               : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int i = i0 + u * AT_THREADS, r = i / C4, c4 = i % C4;
            __half2 h[2] = {__floats2half2_rn(v[u].x, v[u].y), __floats2half2_rn(v[u].z, v[u].w)};
            *reinterpret_cast<uint2*>(dst + r * (C + 8) + 4 * c4) = *reinterpret_cast<uint2*>(h);
        }
    }
}

// cp.async of the fp32 rows [r0, r0 + AT_BK) of one third of qkv (column offset off) into F [AT_BK][C]; rows at or past HW are
// zero-filled (source size 0)
template <int C>
__device__ __forceinline__ void at_issue(float* F, const float* __restrict__ src, int r0, int HW, int off) {
    constexpr int C4 = C / 4, N4 = AT_BK * C4;
#pragma unroll 4
    for (int i = threadIdx.x; i < N4; i += AT_THREADS) {
        const int r = i / C4, c4 = i % C4;
        const bool in = r0 + r < HW;
        const float* g = in ? src + (int64_t)(r0 + r) * 3 * C + off + 4 * c4 : src;
        const uint32_t d = (uint32_t)__cvta_generic_to_shared(F + 4 * i);
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(g), "r"(in ? 16 : 0) : "memory");
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
}
__device__ __forceinline__ void at_wait() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// F [AT_BK][C] fp32 -> fp16 [AT_BK][C + 8]
template <int C>
__device__ __forceinline__ void at_round(__half* dst, const float* F) {
    constexpr int C4 = C / 4, N4 = AT_BK * C4;
#pragma unroll 4
    for (int i = threadIdx.x; i < N4; i += AT_THREADS) {
        const float4 v = *reinterpret_cast<const float4*>(F + 4 * i);
        __half2 h[2] = {__floats2half2_rn(v.x, v.y), __floats2half2_rn(v.z, v.w)};
        *reinterpret_cast<uint2*>(dst + (i / C4) * (C + 8) + 4 * (i % C4)) = *reinterpret_cast<uint2*>(h);
    }
}

template <int C>
__global__ void __launch_bounds__(AT_THREADS, 1) vae_attn_tc_kernel(const float* __restrict__ qkv, float* __restrict__ out, int HW,
                                                                    float scale) {
    using L = AttnTcSmem<C>;
    constexpr int LD = L::LD, NT = C / 16;                           // NT: n8 tiles of a warp's C / 2 output columns
    extern __shared__ __align__(16) uint8_t at_smem[];
    __half* Qs = reinterpret_cast<__half*>(at_smem + L::Q);
    __half* KVs = reinterpret_cast<__half*>(at_smem + L::KV);
    float* Ss = reinterpret_cast<float*>(at_smem + L::S);
    __half* Ps = reinterpret_cast<__half*>(at_smem + L::P);
    float* Ms = reinterpret_cast<float*>(at_smem + L::STATS);
    float* Ls = Ms + AT_BQ;
    float* As = Ls + AT_BQ;
    float* F = reinterpret_cast<float*>(at_smem + L::F);

    const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
    const int q0 = blockIdx.x * AT_BQ, b = blockIdx.y;
    const float* base = qkv + (int64_t)b * HW * 3 * C;
    const int rg = warp & 3;                                         // this warp's 16 query rows
    // ldmatrix row addresses: A fragments (rows 0-15, k 0 / 8), B fragments of two n8 tiles from [n][k] (K) and [k][n] (V) storage
    const int a_row = (lane & 7) + ((lane >> 3) & 1) * 8, a_col = (lane >> 4) * 8;
    const int bk_row = (lane & 7) + (lane >> 4) * 8, bk_col = ((lane >> 3) & 1) * 8;
    const int bv_row = (lane & 7) + ((lane >> 3) & 1) * 8, bv_col = (lane >> 4) * 8;

    at_issue<C>(F, base, 0, HW, C);                                 // K tile 0 loads while Q is staged
    at_stage<C, AT_BQ>(Qs, base, q0, HW, 0);
    if (t < AT_BQ) { Ms[t] = -INFINITY; Ls[t] = 0.f; }

    float o[NT][4];
#pragma unroll
    for (int i = 0; i < NT; i++) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;

    for (int k0 = 0; k0 < HW; k0 += AT_BK) {
        at_wait();
        __syncthreads();                                             // K tile in F; the previous PV phase is done with KVs and Ps
        at_round<C>(KVs, F);
        __syncthreads();
        at_issue<C>(F, base, k0, HW, 2 * C);                        // V tile, under the S phase
        {   // ---- S phase
            const int cg = warp >> 2;
            float s[2][4] = {};
#pragma unroll 4
            for (int kk = 0; kk < C; kk += 16) {
                uint32_t a[4], bb[4];
                at_ldsm_x4(a, Qs + (16 * rg + a_row) * LD + kk + a_col);
                at_ldsm_x4(bb, KVs + (16 * cg + bk_row) * LD + kk + bk_col);
                at_mma(s[0], a, bb[0], bb[1]);
                at_mma(s[1], a, bb[2], bb[3]);
            }
#pragma unroll
            for (int j = 0; j < 2; j++)
#pragma unroll
                for (int e = 0; e < 4; e++) {
                    const int r = 16 * rg + (lane >> 2) + 8 * (e >> 1), c = 16 * cg + 8 * j + 2 * (lane & 3) + (e & 1);
                    Ss[r * AT_SLD + c] = k0 + c < HW ? s[j][e] * scale : -INFINITY;
                }
        }
        __syncthreads();
        {   // ---- online softmax: row t / 4, columns 8 (t % 4) .. +8
            const int r = t >> 2, c0 = 8 * (t & 3);
            const float m_old = Ms[r];
            float v[8], mx = -INFINITY;
#pragma unroll
            for (int i = 0; i < 8; i++) { v[i] = Ss[r * AT_SLD + c0 + i]; mx = fmaxf(mx, v[i]); }
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            const float m_new = fmaxf(m_old, mx);                    // finite: key k0 < HW is in every tile
            float sum = 0.f;
            __half2 p2[4];
#pragma unroll
            for (int i = 0; i < 8; i += 2) {
                const float e0 = expf(v[i] - m_new), e1 = expf(v[i + 1] - m_new);
                sum += e0 + e1;
                p2[i / 2] = __floats2half2_rn(e0, e1);
            }
            *reinterpret_cast<uint4*>(Ps + r * AT_PLD + c0) = *reinterpret_cast<uint4*>(p2);
            sum += __shfl_xor_sync(0xffffffffu, sum, 1);
            sum += __shfl_xor_sync(0xffffffffu, sum, 2);
            __syncwarp();
            if ((t & 3) == 0) {
                const float alpha = expf(m_old - m_new);             // 0 on the first tile (m_old = -inf)
                Ms[r] = m_new;
                Ls[r] = fmaf(Ls[r], alpha, sum);
                As[r] = alpha;
            }
        }
        at_wait();
        __syncthreads();                                             // V tile in F; the S phase is done with KVs
        at_round<C>(KVs, F);
        __syncthreads();
        if (k0 + AT_BK < HW) at_issue<C>(F, base, k0 + AT_BK, HW, C);   // next K tile, under the PV phase
        {   // ---- PV phase
            const int c_lo = (warp >> 2) * (C / 2);
            const float al0 = As[16 * rg + (lane >> 2)], al1 = As[16 * rg + (lane >> 2) + 8];
#pragma unroll
            for (int i = 0; i < NT; i++) { o[i][0] *= al0; o[i][1] *= al0; o[i][2] *= al1; o[i][3] *= al1; }
#pragma unroll
            for (int kk = 0; kk < AT_BK; kk += 16) {
                uint32_t a[4];
                at_ldsm_x4(a, Ps + (16 * rg + a_row) * AT_PLD + kk + a_col);
#pragma unroll
                for (int i = 0; i < NT; i += 2) {
                    uint32_t bb[4];
                    at_ldsm_x4_t(bb, KVs + (kk + bv_row) * LD + c_lo + 8 * i + bv_col);
                    at_mma(o[i], a, bb[0], bb[1]);
                    at_mma(o[i + 1], a, bb[2], bb[3]);
                }
            }
        }
    }
    // ---- out = O / l (Ls final: the last softmax phase precedes the last barrier)
    const int c_lo = (warp >> 2) * (C / 2);
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const int r = 16 * rg + (lane >> 2) + 8 * h;
        if (q0 + r >= HW) continue;
        const float inv = 1.f / Ls[r];
        float* orow = out + ((int64_t)b * HW + q0 + r) * C + c_lo + 2 * (lane & 3);
#pragma unroll
        for (int i = 0; i < NT; i++)
            *reinterpret_cast<float2*>(orow + 8 * i) = make_float2(o[i][2 * h] * inv, o[i][2 * h + 1] * inv);
    }
}

template <int C>
static int launch_vae_attn_tc_t(const float* qkv, float* out, int B, int HW, cudaStream_t st) {
    constexpr int smem = AttnTcSmem<C>::BYTES;
    static_assert(smem <= 227 * 1024, "vae_attn_tc: shared memory budget");
    RQB_ENSURE_SMEM(smem, vae_attn_tc_kernel<C>);
    const float scale = (float)(1.0 / sqrt((double)C));           // int(c) ** (-0.5) evaluated in double, then cast
    vae_attn_tc_kernel<C><<<dim3((unsigned)ceil_div(HW, AT_BQ), B), AT_THREADS, smem, st>>>(qkv, out, HW, scale);
    return check_launch("vae_attn_tc");
}

int launch_vae_attn_tc(const float* qkv, float* out, int B, int HW, int C, cudaStream_t st) {
    if (B < 1 || HW < 1) return fail(RQB200_EINVAL, "vae_attn_tc: need B, HW >= 1");
    if (B > 65535) return fail(RQB200_EINVAL, "vae_attn_tc: B > 65535");
    switch (C) {
        case 128: return launch_vae_attn_tc_t<128>(qkv, out, B, HW, st);
        case 256: return launch_vae_attn_tc_t<256>(qkv, out, B, HW, st);
        case 384: return launch_vae_attn_tc_t<384>(qkv, out, B, HW, st);
        case 512: return launch_vae_attn_tc_t<512>(qkv, out, B, HW, st);
        default: return fail(RQB200_EINVAL, "vae_attn_tc: C must be 128, 256, 384 or 512");
    }
}

}  // namespace rqb
