// P2 "fast" tier -- NHWC implicit-GEMM convolution on wgmma tensor cores (split-fp16 operands, fp32 accumulate in registers).
//
// Replaces cuDNN's conv behind ResnetBlock / AttnBlock / Upsample / conv_in / conv_out of the decoder (reference:
// rqvae/models/rqvae/layers.py:100-120,158-182,31-35; modules.py:171-202).  The reference's own GPU path runs these convs
// with TF32 allowed (10-bit mantissa).  Every conv takes both operands as fp16 hi + lo pairs and forms three products per k
// step (see ct_mma_kblock): fp32-class products on the fp16 tensor pipe.
//
//   D[pixel, cout] = sum_{tap, cin} A[pixel + tap, cin] * W[cout, tap, cin]
//
//   M = 128 output pixels per tile: a TW x TH x NB box of the NHWC activation tensor (NB > 1 images per tile when the
//       feature map is smaller than 128 pixels).  Out-of-range rows/columns of a TMA box are zero-filled by the TMA unit,
//       which IS the conv's zero padding; no im2col buffer.
//   N = BN output channels (16 | 64 | 128 | 256), K = taps x Cin walked in 64-channel slabs (one 128 B swizzled row per pixel).
//
// Three kernels share the layout and the epilogue:
//   conv3x3_wreg_kernel  3x3 stride-1 convs with Cout % 128 == 0, the GEMM transposed: 128 output channels on the wgmma M side
//                      with the weight fragments in registers, 256 output pixels on N (see the comment above the kernel).
//   conv3x3_tc_kernel  the other 3x3 stride-1 convs (conv_out, Cout = 3; Cout = 64).  Input-stationary within a channel slab: ONE
//                      TMA box brings the 8 x TH x NB tile plus its one-pixel halo, and the nine taps read it as shifted wgmma
//                      operands; only the weight slabs stream through the ring (see the comment above the kernel).
//   conv_tc_kernel     1x1 convs, the encoder's stride-2 convs and the rows GEMM: one activation box and one weight slab per
//                      (tap, slab) k block.  The rows GEMM (launch_rows_gemm_tc) is the only caller of its single-product
//                      forms (PASSES == 1) and of bf16 operands (ConvTcParams.fmt == 1).
//
// Persistent CTAs (grid = #SMs) loop over (pixel tile, cout tile) pairs; warp 8 = TMA producer, warps 0-7 = two consumer
// warpgroups, each issuing wgmma m64nBNk16 for 64 of the tile's 128 pixels and then running the epilogue (registers -> shared
// staging -> +bias (+residual) -> fp32 NHWC / NCHW stores).  The producer runs ahead across tiles, so the next tile's operands
// load while this tile's epilogue runs.
#include <cstdlib>

#include "kernels.h"
#include "tc_common.cuh"

namespace rqb {

struct ConvTcParams {
    int B, H, W, Cin, Cout;        // H,W: OUTPUT extent; the input is H*stride x W*stride
    int ks;                        // 1 or 3
    int stride;                    // 3x3 stride 1: "same" zero padding (conv3x3_tc_kernel); 2: no left/top pad, one zero column/row
                                   // on the right/bottom (F.pad(0,1,0,1) + stride-2 conv, layers.py:50-57) -- both are the tensor
                                   // map's out-of-bounds fill
    int TW, TH, NB;                // tile box, TW*TH*NB == 128
    int tiles_x, tiles_y, tiles_b, n_tiles_n;
    const float* bias;
    const float* residual;         // [B,H,W,Cout] f32 or null
    float* out;                    // NHWC f32, or NCHW f32 when out_nchw
    int out_nchw;
    // "rows GEMM" use of the same kernel (launch_rows_gemm_tc: a 1x1 conv over M token rows viewed as 16x8-pixel images):
    void* out16;                   // non-null: 16-bit NHWC output (fmt) instead of `out`, optionally through GELU
    int gelu, fmt;                 // fmt: 16-bit operand / output format of the rows GEMM, 0 fp16, 1 bf16; every conv is 0 (fp16)
    int64_t m_rows;                // > 0: only pixels (rows) below m_rows are stored
    // GroupNorm(32) statistics of the OUTPUT (bias / residual included), for the GroupNorm that consumes it next (layers.py:16-17,
    // 100-120): every epilogue warp (32 pixels of one image) writes (sum, sum of squares) per group as fp64 to
    // gn_part[((b * gn_chunks + chunk) * 32 + group) * 2] -- the partial layout gn_finalize_kernel reduces.  NULL: off.
    double* gn_part;
    int gn_chunks;                 // H * W / 32
};

constexpr int CT_THREADS = 288;            // warps 0-7: two consumer warpgroups (64 tile rows each), warp 8: TMA producer
constexpr int CT_A_BYTES = 128 * 64 * 2;

// PASSES == 3 (every conv): split-fp16 ("fp16x3") -- both operands are carried as hi + lo fp16 pairs and the accumulator receives
// A_hi W_hi + A_lo W_hi + A_hi W_lo (the dropped A_lo W_lo term is ~2^-22 relative): fp32-class products on the fp16 tensor pipe,
// which is what keeps 60 chained convs inside the 1e-3 pixel tolerance.  PASSES == 1: the rows GEMM's single 16-bit product.
// GroupNorm partial statistics of one 16-channel chunk of a warp's 32 pixels: NV = 2 * (16 / CG) values (the sums, then the sums
// of squares, of the chunk's 16 / CG groups) are formed per thread and reduced over the 32 lanes with a transpose-reduce
// (log2(NV) halving steps, then plain butterfly steps): NV + 1 shuffles of depth 5 instead of 5 * NV.  On return `tot` is the total
// of value index `vidx` and `writer` marks the one lane per value that stores it.
template <int CG>
__device__ __forceinline__ void gn_chunk_stats(const float (&wv)[16], bool valid, int lane, float& tot, int& vidx, bool& writer) {
    constexpr int NG = 16 / CG, NV = 2 * NG;
    float vals[NV];
#pragma unroll
    for (int g = 0; g < NG; g++) {
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int i = 0; i < CG; i++) {
            const float x = valid ? wv[g * CG + i] : 0.f;
            s1 += x;
            s2 = fmaf(x, x, s2);
        }
        vals[g] = s1;
        vals[NG + g] = s2;
    }
    int n = NV;
    vidx = 0;
    int keep_mask = 31;                         // lanes that end up holding identical totals differ only in these bits
#pragma unroll
    for (int S = 16; S >= 1; S >>= 1) {
        if (n > 1) {
            const int half = n >> 1;
            const bool up = (lane & S) != 0;
#pragma unroll
            for (int i = 0; i < NV / 2; i++)
                if (i < half) {
                    const float send = up ? vals[i] : vals[i + half];
                    const float keep = up ? vals[i + half] : vals[i];
                    vals[i] = keep + __shfl_xor_sync(0xffffffffu, send, S);
                }
            vidx += up ? half : 0;
            keep_mask &= ~S;
            n = half;
        } else {
            vals[0] += __shfl_xor_sync(0xffffffffu, vals[0], S);
        }
    }
    tot = vals[0];
    writer = (lane & keep_mask) == 0;
}

// Epilogue of one thread: tile row r (one output pixel), output channels [n0, n0 + 16) in v.  Warp q of the four that share a column
// half holds the tile's pixels [32 q, 32 q + 32) -- the layout the GroupNorm partial statistics are formed over.  OUT16: the rows
// GEMM's 16-bit output is possible (conv_tc_kernel); the 3x3 kernels never have it.  QG: that output's activation is QuickGELU
// (x * sigmoid(1.702 x), the CLIP engine's c_fc) rather than p.gelu's exact GELU.
template <bool OUT16, bool QG = false>
__device__ __forceinline__ void ct_epilogue16(const ConvTcParams& p, const float (&v)[16], int n0, int q, int lane, int tx, int ty, int tb,
                                              int b, int y, int x, int64_t pix, bool valid) {
    if (n0 >= p.Cout) return;                                           // (warp-uniform)
    if (p.out_nchw) {
        if (!valid) return;
#pragma unroll
        for (int i = 0; i < 16; i++) {
            const int n = n0 + i;
            if (n < p.Cout) p.out[(((int64_t)b * p.Cout + n) * p.H + y) * p.W + x] = v[i] + p.bias[n];
        }
    } else if (OUT16 && p.out16 != nullptr) {
        if (!valid) return;
        float w[16];
#pragma unroll
        for (int i = 0; i < 16; i += 4) {
            const float4 bb = *reinterpret_cast<const float4*>(p.bias + n0 + i);
            w[i] = v[i] + bb.x; w[i + 1] = v[i + 1] + bb.y; w[i + 2] = v[i + 2] + bb.z; w[i + 3] = v[i + 3] + bb.w;
        }
        if (QG) {
#pragma unroll
            for (int i = 0; i < 16; i++) w[i] = quick_gelu(w[i]);
        } else if (p.gelu) {
#pragma unroll
            for (int i = 0; i < 16; i++) w[i] = gelu_erf(w[i]);
        }
        uint4 pk[2];
        uint32_t* pw = reinterpret_cast<uint32_t*>(pk);
#pragma unroll
        for (int i = 0; i < 8; i++) pw[i] = pack_h16x2(w[2 * i], w[2 * i + 1], p.fmt);
        uint4* o16 = reinterpret_cast<uint4*>(reinterpret_cast<h16*>(p.out16) + pix * p.Cout + n0);
        o16[0] = pk[0];
        o16[1] = pk[1];
    } else {
        float* o = p.out + pix * p.Cout + n0;
        const float* rs = p.residual ? p.residual + pix * p.Cout + n0 : nullptr;
        float wv[16];
#pragma unroll
        for (int i = 0; i < 16; i += 4) {
            float4 bb = *reinterpret_cast<const float4*>(p.bias + n0 + i);
            float4 w = make_float4(v[i] + bb.x, v[i + 1] + bb.y, v[i + 2] + bb.z, v[i + 3] + bb.w);
            if (rs && valid) {
                float4 rr = *reinterpret_cast<const float4*>(rs + i);
                w.x += rr.x; w.y += rr.y; w.z += rr.z; w.w += rr.w;
            }
            if (valid) *reinterpret_cast<float4*>(o + i) = w;
            wv[i] = w.x; wv[i + 1] = w.y; wv[i + 2] = w.z; wv[i + 3] = w.w;
        }
        if (p.gn_part != nullptr) {
            // this warp's 32 pixels belong to one image (TW*TH >= 32, checked by the host); cg = 4 | 8 | 16 channels
            const int cg = p.Cout >> 5;
            const int wpi = (p.TW * p.TH) >> 5;                      // warps (32-pixel chunks) per image within a tile
            const int chunk = (ty * p.tiles_x + tx) * wpi + (q % wpi);
            const int bw = tb * p.NB + (q * 32) / (p.TW * p.TH);      // image of this warp
            float tot;
            int vidx;
            bool writer;
            if (cg == 4) gn_chunk_stats<4>(wv, valid, lane, tot, vidx, writer);
            else if (cg == 8) gn_chunk_stats<8>(wv, valid, lane, tot, vidx, writer);
            else gn_chunk_stats<16>(wv, valid, lane, tot, vidx, writer);
            const int ngr = 16 / cg;
            if (writer && bw < p.B)                                    // vidx < ngr: sum of group vidx; else sum of squares
                p.gn_part[(((int64_t)bw * p.gn_chunks + chunk) * 32 + (n0 / cg + (vidx % ngr))) * 2 + (vidx / ngr)] = (double)tot;
        }
    }
}

template <int BN, int FMT, int PASSES>
__device__ __forceinline__ void ct_mma_kblock(float (&acc)[BN / 2], uint32_t a, uint32_t b, bool first) {
    constexpr int B_BYTES = BN * 64 * 2;
    if (PASSES == 3) {                              // small terms first, the dominant product last
#pragma unroll
        for (int j = 0; j < 4; j++)
            tc::Wgmma<BN, FMT>::mma(acc, tc::gmma_desc_k128(a + CT_A_BYTES + j * 32), tc::gmma_desc_k128(b + j * 32),
                                    (!first || j > 0) ? 1u : 0u);
#pragma unroll
        for (int j = 0; j < 4; j++)
            tc::Wgmma<BN, FMT>::mma(acc, tc::gmma_desc_k128(a + j * 32), tc::gmma_desc_k128(b + B_BYTES + j * 32), 1u);
    }
#pragma unroll
    for (int j = 0; j < 4; j++)
        tc::Wgmma<BN, FMT>::mma(acc, tc::gmma_desc_k128(a + j * 32), tc::gmma_desc_k128(b + j * 32),
                                (PASSES == 3 || !first || j > 0) ? 1u : 0u);
}

template <int BN, int STAGES, int PASSES, bool QG = false>
__global__ void __launch_bounds__(CT_THREADS, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmAlo, const __grid_constant__ CUtensorMap tmBlo, ConvTcParams p) {
    constexpr int B_BYTES = BN * 64 * 2;
    constexpr int NOPS = PASSES == 3 ? 2 : 1;
    constexpr int STAGE_BYTES = NOPS * (CT_A_BYTES + B_BYTES);
    constexpr int OFF_B = NOPS * CT_A_BYTES;                 // [A_hi | A_lo | B_hi | B_lo]
    constexpr int CW = BN < 32 ? BN : 32;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    float* stage = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES);        // [128][CW + 4] epilogue staging
    uint64_t* full = reinterpret_cast<uint64_t*>(stage + 128 * (CW + 4));
    uint64_t* empty = full + STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int cslabs = p.Cin / 64;
    const int nkb = p.ks * p.ks * cslabs;
    const int sx = p.stride;
    const int m_tiles = p.tiles_x * p.tiles_y * p.tiles_b;
    const int total = m_tiles * p.n_tiles_n;

    if (warp == 8 && lane == 0) {
        tc::prefetch_tmap(&tmA);
        tc::prefetch_tmap(&tmB);
        // empty[s]: one arrival per consumer warp once its warpgroup's MMAs of that slot have completed
        for (int s = 0; s < STAGES; s++) { tc::mbar_init(&full[s], 1); tc::mbar_init(&empty[s], 8); }
        tc::fence_barrier_init();
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            // ---- TMA producer: runs ahead across tiles, so the next tile's operands load during this tile's epilogue
            uint32_t it = 0;                                   // running k-block counter across tiles
            for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
                const int nt = tile % p.n_tiles_n, mt = tile / p.n_tiles_n;
                const int tx = mt % p.tiles_x, ty = (mt / p.tiles_x) % p.tiles_y, tb = mt / (p.tiles_x * p.tiles_y);
                const int x0 = tx * p.TW, y0 = ty * p.TH, b0 = tb * p.NB;
                for (int kb = 0; kb < nkb; kb++, it++) {
                    const int s = it % STAGES;
                    tc::mbar_wait(&empty[s], ((it / STAGES) & 1) ^ 1);
                    const int tap = kb / cslabs, c0 = (kb % cslabs) * 64;
                    const int ky = tap / p.ks, kx = tap % p.ks;
                    tc::mbar_expect_tx(&full[s], STAGE_BYTES);
                    uint8_t* st = smem + s * STAGE_BYTES;
                    tc::tma_load_4d(st, &tmA, &full[s], c0, x0 * sx + kx, y0 * sx + ky, b0, tc::L2_EVICT_NORMAL);
                    tc::tma_load_2d(st + OFF_B, &tmB, &full[s], tap * p.Cin + c0, nt * BN, tc::L2_EVICT_LAST);
                    if (PASSES == 3) {
                        tc::tma_load_4d(st + CT_A_BYTES, &tmAlo, &full[s], c0, x0 * sx + kx, y0 * sx + ky, b0, tc::L2_EVICT_NORMAL);
                        tc::tma_load_2d(st + OFF_B + B_BYTES, &tmBlo, &full[s], tap * p.Cin + c0, nt * BN, tc::L2_EVICT_LAST);
                    }
                }
            }
        }
        return;
    }

    // ---- consumer warpgroups 0, 1: tile rows (pixels) [64 wg, 64 wg + 64) x BN output channels; one k block in flight
    const int wg = warp >> 2, t = threadIdx.x;
    const int r = t & 127;                                           // epilogue: row of the tile
    const int rx = r % p.TW, ry = (r / p.TW) % p.TH, rb = r / (p.TW * p.TH);
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; i++) acc[i] = 0.f;
    uint32_t it = 0;
    for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
        for (int kb = 0; kb < nkb; kb++, it++) {
            const int s = it % STAGES;
            tc::mbar_wait(&full[s], (it / STAGES) & 1);
            const uint32_t a = tc::smem_u32(smem + s * STAGE_BYTES) + wg * (64 * 128), b = tc::smem_u32(smem + s * STAGE_BYTES + OFF_B);
            tc::wgmma_fence();
            if (p.fmt) ct_mma_kblock<BN, 1, PASSES>(acc, a, b, kb == 0);
            else ct_mma_kblock<BN, 0, PASSES>(acc, a, b, kb == 0);
            tc::wgmma_commit();
            tc::wgmma_wait<1>();
            if (kb > 0 && lane == 0) tc::mbar_arrive(&empty[(it - 1) % STAGES]);
        }
        tc::wgmma_wait<0>();
        tc::acc_fence(acc);
        if (lane == 0) tc::mbar_arrive(&empty[(it - 1) % STAGES]);

        const int nt = tile % p.n_tiles_n, mt = tile / p.n_tiles_n;
        const int tx = mt % p.tiles_x, ty = (mt / p.tiles_x) % p.tiles_y, tb = mt / (p.tiles_x * p.tiles_y);
        const int x = tx * p.TW + rx, y = ty * p.TH + ry, b = tb * p.NB + rb;
        const int64_t pix = ((int64_t)b * p.H + y) * p.W + x;
        const bool valid = (x < p.W) && (y < p.H) && (b < p.B) && (p.m_rows == 0 || pix < p.m_rows);
        tc::drain_acc<BN, CW, 0>(acc, stage, wg, t, [&p, t, nt, tx, ty, tb, b, y, x, pix, valid](const float (&v)[16], int, int c) {
            ct_epilogue16<true, QG>(p, v, nt * BN + c, (t >> 5) & 3, t & 31, tx, ty, tb, b, y, x, pix, valid);
        });
    }
}

template <int BN, int STAGES, int PASSES, bool QG = false>
static int launch_conv_tc_t(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmAlo, const CUtensorMap& tmBlo,
                            const ConvTcParams& p, int n_sm, cudaStream_t st) {
    constexpr size_t smem = (size_t)STAGES * (PASSES == 3 ? 2 : 1) * (CT_A_BYTES + BN * 128) + 128 * ((BN < 32 ? BN : 32) + 4) * 4 + 1024 + 256;
    static_assert(smem <= 227 * 1024, "conv_tc: shared memory budget");
    RQB_ENSURE_SMEM(smem, conv_tc_kernel<BN, STAGES, PASSES, QG>);
    const int total = p.tiles_x * p.tiles_y * p.tiles_b * p.n_tiles_n;
    const int grid = total < n_sm ? total : n_sm;
    conv_tc_kernel<BN, STAGES, PASSES, QG><<<grid, CT_THREADS, smem, st>>>(tmA, tmB, tmAlo, tmBlo, p);
    return check_launch("conv_tc");
}

// ------------------------------------------------------------------------------------------------ 3x3 stride-1 convs
// The output tile is 8 pixels wide (TW = 8) and TH = 16 rows (TH = 8 and NB = 2 images below 16 rows), so each wgmma core-matrix
// group -- 8 rows of 128 B -- is one output row.  Per 64-channel slab ONE TMA box loads the (TW + 2) x (TH + 2) x NB input
// pixels the tile's nine taps touch, at (x0 - 1, y0 - 1): halo pixel (b, hy, hx) sits at ((b (TH + 2) + hy) 10 + hx) 128 B.
// Tap (dy, dx) of output row oy is then the same smem image read from pixel ((oy + dy) 10 + dx), with a uniform 1280 B group
// stride (SBO): a shifted descriptor, no reload.  Only the weight slabs [BN x 64] of the nine taps stream through the ring.
// k order: slab-major, tap-minor.
//
// L2 -> smem bytes per 64-channel slab and 128-pixel tile (hi + lo operands), conv_out (BN = 16, Cout = 3): 46 KB halo + 9 x 4 KB
// weights -> 85 flop/B of wgmma work, against 21 for per-tap A + W reloads.
constexpr int C3_HALO_BYTES = 10 * 10 * 2 * 128;   // per operand; the largest box (TH = 8, NB = 2: 200 pixels; TH = 16: 180)

template <int BN>
__device__ __forceinline__ void c3_mma_kblock(float (&acc)[BN / 2], uint32_t a, uint32_t b, bool first) {
    constexpr int B_BYTES = BN * 64 * 2;
    constexpr uint32_t SBO = 10 * 128;                 // one halo row per core-matrix group
    // split-fp16: small terms first, the dominant product last
#pragma unroll
    for (int j = 0; j < 4; j++)
        tc::Wgmma<BN, 0>::mma(acc, tc::gmma_desc_k128(a + C3_HALO_BYTES + j * 32, SBO), tc::gmma_desc_k128(b + j * 32),
                              (!first || j > 0) ? 1u : 0u);
#pragma unroll
    for (int j = 0; j < 4; j++)
        tc::Wgmma<BN, 0>::mma(acc, tc::gmma_desc_k128(a + j * 32, SBO), tc::gmma_desc_k128(b + B_BYTES + j * 32), 1u);
#pragma unroll
    for (int j = 0; j < 4; j++)
        tc::Wgmma<BN, 0>::mma(acc, tc::gmma_desc_k128(a + j * 32, SBO), tc::gmma_desc_k128(b + j * 32), 1u);
}

// TMA producer of both 3x3 kernels (one thread): per 64-channel slab ONE halo box (hi + lo) into the next of two halo slots,
// per tap one [BM x 64] weight slab (hi + lo) into the STAGES-deep ring.  Runs ahead across tiles, so the next tile's operands
// load during this tile's epilogue.  Halo slot: [X_hi | X_lo], HALO_BYTES apart; weight stage: [W_hi | W_lo], BM x 128 B apart.
template <int BM, int STAGES, int SLOT_BYTES, int HALO_BYTES>
__device__ __forceinline__ void c3_produce(const CUtensorMap* tmA, const CUtensorMap* tmB, const CUtensorMap* tmAlo, const CUtensorMap* tmBlo,
                                           const ConvTcParams& p, uint8_t* smem, uint8_t* wst, uint64_t* full, uint64_t* empty,
                                           uint64_t* hfull, uint64_t* hempty) {
    constexpr int NOPS = 2;
    constexpr int B_BYTES = BM * 64 * 2;
    constexpr int STAGE_BYTES = NOPS * B_BYTES;
    const int cslabs = p.Cin / 64;
    const int total = p.tiles_x * p.tiles_y * p.tiles_b * p.n_tiles_n;
    const uint32_t halo_tx = NOPS * 10 * (p.TH + 2) * p.NB * 128;
    uint32_t it = 0, hit = 0;                          // running weight-stage / halo counters across tiles
    for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
        const int nt = tile % p.n_tiles_n, mt = tile / p.n_tiles_n;
        const int tx = mt % p.tiles_x, ty = (mt / p.tiles_x) % p.tiles_y, tb = mt / (p.tiles_x * p.tiles_y);
        const int x0 = tx * 8, y0 = ty * p.TH, b0 = tb * p.NB;
        for (int sl = 0; sl < cslabs; sl++, hit++) {
            const int c0 = sl * 64;
            for (int tap = 0; tap < 9; tap++, it++) {
                const int s = it % STAGES;
                tc::mbar_wait(&empty[s], ((it / STAGES) & 1) ^ 1);
                tc::mbar_expect_tx(&full[s], STAGE_BYTES);
                uint8_t* w = wst + s * STAGE_BYTES;
                tc::tma_load_2d(w, tmB, &full[s], tap * p.Cin + c0, nt * BM, tc::L2_EVICT_LAST);
                tc::tma_load_2d(w + B_BYTES, tmBlo, &full[s], tap * p.Cin + c0, nt * BM, tc::L2_EVICT_LAST);
                if (tap == 0) {                        // the slab's first weights go out before the wait for a halo slot
                    const int h = hit % 2;
                    tc::mbar_wait(&hempty[h], ((hit / 2) & 1) ^ 1);
                    tc::mbar_expect_tx(&hfull[h], halo_tx);
                    uint8_t* a = smem + h * SLOT_BYTES;
                    tc::tma_load_4d(a, tmA, &hfull[h], c0, x0 - 1, y0 - 1, b0, tc::L2_EVICT_NORMAL);
                    tc::tma_load_4d(a + HALO_BYTES, tmAlo, &hfull[h], c0, x0 - 1, y0 - 1, b0, tc::L2_EVICT_NORMAL);
                }
            }
        }
    }
}

// Two halo slots (the next slab's halo loads during this slab's taps) and STAGES weight stages.
// smem: [halo slot: A_hi | A_lo] x 2, [B_hi | B_lo] x STAGES, epilogue staging, barriers.
template <int BN, int STAGES>
__global__ void __launch_bounds__(CT_THREADS, 1)
conv3x3_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ CUtensorMap tmAlo, const __grid_constant__ CUtensorMap tmBlo, ConvTcParams p) {
    constexpr int B_BYTES = BN * 64 * 2;
    constexpr int NOPS = 2;
    constexpr int HSLOTS = 2;
    constexpr int SLOT_BYTES = NOPS * C3_HALO_BYTES;
    constexpr int STAGE_BYTES = NOPS * B_BYTES;
    constexpr int CW = BN < 32 ? BN : 32;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* wst = smem + HSLOTS * SLOT_BYTES;
    float* stage = reinterpret_cast<float*>(wst + STAGES * STAGE_BYTES);           // [128][CW + 4] epilogue staging
    uint64_t* full = reinterpret_cast<uint64_t*>(stage + 128 * (CW + 4));
    uint64_t* empty = full + STAGES;
    uint64_t* hfull = empty + STAGES;
    uint64_t* hempty = hfull + HSLOTS;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int cslabs = p.Cin / 64;
    const int m_tiles = p.tiles_x * p.tiles_y * p.tiles_b;
    const int total = m_tiles * p.n_tiles_n;

    if (warp == 8 && lane == 0) {
        tc::prefetch_tmap(&tmA);
        tc::prefetch_tmap(&tmB);
        // empty[s] / hempty[h]: one arrival per consumer warp once its warpgroup's MMAs reading that buffer have completed
        for (int s = 0; s < STAGES; s++) { tc::mbar_init(&full[s], 1); tc::mbar_init(&empty[s], 8); }
        for (int h = 0; h < HSLOTS; h++) { tc::mbar_init(&hfull[h], 1); tc::mbar_init(&hempty[h], 8); }
        tc::fence_barrier_init();
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) c3_produce<BN, STAGES, SLOT_BYTES, C3_HALO_BYTES>(&tmA, &tmB, &tmAlo, &tmBlo, p, smem, wst, full, empty, hfull, hempty);
        return;
    }

    // ---- consumer warpgroups 0, 1: tile rows [64 wg, 64 wg + 64) = output rows [8 wg, 8 wg + 8) of the tile, all in one image
    const int wg = warp >> 2, t = threadIdx.x;
    const int r = t & 127;                                           // epilogue: row of the tile
    const int rx = r % 8, ry = (r / 8) % p.TH, rb = r / (8 * p.TH);
    const uint32_t a_wg = (uint32_t)(((8 * wg / p.TH) * (p.TH + 2) + (8 * wg) % p.TH) * 10 * 128);   // tap (0, 0) of row 8 wg
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; i++) acc[i] = 0.f;
    uint32_t it = 0, hit = 0;
    for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
        for (int sl = 0; sl < cslabs; sl++, hit++) {
            const int h = hit % HSLOTS;
            tc::mbar_wait(&hfull[h], (hit / HSLOTS) & 1);
            const uint32_t a0 = tc::smem_u32(smem + h * SLOT_BYTES) + a_wg;
            for (int tap = 0; tap < 9; tap++, it++) {
                const int s = it % STAGES;
                tc::mbar_wait(&full[s], (it / STAGES) & 1);
                const uint32_t a = a0 + ((tap / 3) * 10 + tap % 3) * 128, b = tc::smem_u32(wst + s * STAGE_BYTES);
                const bool first = sl == 0 && tap == 0;
                tc::wgmma_fence();
                c3_mma_kblock<BN>(acc, a, b, first);
                tc::wgmma_commit();
                tc::wgmma_wait<1>();
                if (!first && lane == 0) {                   // the previous k block's MMAs are complete: free what only it read
                    tc::mbar_arrive(&empty[(it - 1) % STAGES]);
                    if (tap == 0) tc::mbar_arrive(&hempty[(hit - 1) % HSLOTS]);
                }
            }
        }
        tc::wgmma_wait<0>();
        tc::acc_fence(acc);
        if (lane == 0) {
            tc::mbar_arrive(&empty[(it - 1) % STAGES]);
            tc::mbar_arrive(&hempty[(hit - 1) % HSLOTS]);
        }

        const int nt = tile % p.n_tiles_n, mt = tile / p.n_tiles_n;
        const int tx = mt % p.tiles_x, ty = (mt / p.tiles_x) % p.tiles_y, tb = mt / (p.tiles_x * p.tiles_y);
        const int x = tx * 8 + rx, y = ty * p.TH + ry, b = tb * p.NB + rb;
        const int64_t pix = ((int64_t)b * p.H + y) * p.W + x;
        const bool valid = (x < p.W) && (y < p.H) && (b < p.B);
        tc::drain_acc<BN, CW, 0>(acc, stage, wg, t, [&p, t, nt, tx, ty, tb, b, y, x, pix, valid](const float (&v)[16], int, int c) {
            ct_epilogue16<false>(p, v, nt * BN + c, (t >> 5) & 3, t & 31, tx, ty, tb, b, y, x, pix, valid);
        });
    }
}

template <int BN, int STAGES>
static int launch_conv3x3_tc_t(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmAlo, const CUtensorMap& tmBlo,
                               const ConvTcParams& p, int n_sm, cudaStream_t st) {
    constexpr int NOPS = 2;
    constexpr size_t smem = (size_t)2 * NOPS * C3_HALO_BYTES + (size_t)STAGES * NOPS * BN * 128 +
                            128 * ((BN < 32 ? BN : 32) + 4) * 4 + 1024 + 256;
    static_assert(smem <= 227 * 1024, "conv3x3_tc: shared memory budget");
    RQB_ENSURE_SMEM(smem, conv3x3_tc_kernel<BN, STAGES>);
    const int total = p.tiles_x * p.tiles_y * p.tiles_b * p.n_tiles_n;
    const int grid = total < n_sm ? total : n_sm;
    conv3x3_tc_kernel<BN, STAGES><<<grid, CT_THREADS, smem, st>>>(tmA, tmB, tmAlo, tmBlo, p);
    return check_launch("conv3x3_tc");
}

// ------------------------------------------------------------------------------------------------ 3x3 stride-1 convs, Cout % 128 == 0
// The GEMM transposed: D[cout, pixel] = sum_{slab, tap, c} W[cout, tap, c] X[pixel + tap, c].
//   M = 128 output channels per tile, 64 per consumer warpgroup.  Each warpgroup ldmatrix-es its W_hi / W_lo fragments of a tap
//       out of the weight ring and issues register-A wgmma, so the weights cross shared memory once per tap, not once per product.
//   N = the tile's output pixels in the shared-memory operand: 8 wide x TH rows of NB images (TH = 32 on maps of 32 rows or more:
//       N = 256; TH = 16: 128; TH = 8, NB = 2: 2 x 64), one wgmma per image.  The halo trick of conv3x3_tc_kernel is unchanged:
//       one core-matrix group is one 8-pixel output row, 1280 B apart, a tap is a start-address shift, and the TMA's
//       out-of-bounds fill is the zero padding.
// Split-fp16 products per k16: W_hi X_lo, W_lo X_hi, W_hi X_hi -- only X is read from shared memory, ~64 B/clk of operand reads at
// the fp16 rate against ~94 for the pixel-major SS form.  k order (slab-major, tap-minor) and the small-terms-first order of
// conv3x3_tc_kernel are kept.
// smem at TH = 32: two halo slots of 2 x 43 KB, ONE 32 KB weight stage, a 16.5 KB epilogue staging buffer and 2 KB of
// GroupNorm partial sums = 223 KB.
// The single weight stage is enough because a warpgroup holds two taps' fragments in registers: the producer refills the stage
// as soon as both warpgroups have loaded tap t, while tap t - 1's and tap t's MMAs run.
template <int TH, int NB>
struct C3wTile {
    static constexpr int NI = 8 * TH;                                          // pixels per wgmma: TH rows of one image
    static constexpr int NP = NI * NB;                                         // pixels per tile
    static constexpr int HALO = (10 * (TH + 2) * NB * 128 + 1023) / 1024 * 1024;   // bytes per halo operand (1024 B aligned)
};
constexpr int C3W_SP = 128 + 4;                    // epilogue staging row (one pixel, 128 output channels) in floats
// warps 0-7: two consumer warpgroups, warp 8: TMA producer; warps 9-11 idle.  A whole producer warpgroup lets setmaxnreg move its
// registers to the consumers (128 accumulators + two taps' fragments per thread): ptxas sizes a wgmma kernel's register budget
// in warpgroups, so 288 threads would leave 168 registers per thread, as 384 do.  setmaxnreg.inc waits until the CTA's pool (the
// 168 x 384 registers it was launched with) can grant the increase, so the split must fit that pool.
constexpr int C3W_THREADS = 384, C3W_REGS_CONSUMER = 240, C3W_REGS_PRODUCER = 24;
static_assert(256 * C3W_REGS_CONSUMER + 128 * C3W_REGS_PRODUCER <= 168 * C3W_THREADS, "conv3x3_wreg: register split exceeds the pool");

template <int TH, int NB>
__device__ __forceinline__ void c3w_mma_kblock(float (&acc)[C3wTile<TH, NB>::NP / 2], const uint32_t (&fh)[4][4],
                                               const uint32_t (&fl)[4][4], uint32_t x, bool first) {
    constexpr int NI = C3wTile<TH, NB>::NI, HALO = C3wTile<TH, NB>::HALO;
    constexpr uint32_t SBO = 10 * 128, IMG = (TH + 2) * 10 * 128;
    auto mma = [&acc](const uint32_t (&a)[4], uint32_t xa, uint32_t accumulate) {
#pragma unroll
        for (int b = 0; b < NB; b++)
            tc::WgmmaRA<NI>::mma(*reinterpret_cast<float(*)[NI / 2]>(&acc[b * (NI / 2)]), a, tc::gmma_desc_k128(xa + b * IMG, SBO),
                                 accumulate);
    };
    // split-fp16: small terms first, the dominant product last
#pragma unroll
    for (int j = 0; j < 4; j++) mma(fh[j], x + HALO + j * 32, (!first || j > 0) ? 1u : 0u);
#pragma unroll
    for (int j = 0; j < 4; j++) mma(fl[j], x + j * 32, 1u);
#pragma unroll
    for (int j = 0; j < 4; j++) mma(fh[j], x + j * 32, 1u);
}

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}

// smem: [halo slot: X_hi | X_lo] x 2, [W_hi | W_lo] x STAGES (128 rows x 128 B each, SWIZZLE_128B), epilogue staging, barriers.
template <int TH, int NB, int STAGES>
__global__ void __launch_bounds__(C3W_THREADS, 1)
conv3x3_wreg_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                    const __grid_constant__ CUtensorMap tmAlo, const __grid_constant__ CUtensorMap tmBlo, ConvTcParams p) {
    using T = C3wTile<TH, NB>;
    constexpr int NOPS = 2;
    constexpr int SLOT_BYTES = NOPS * T::HALO;
    constexpr int B_BYTES = 128 * 128;
    constexpr int STAGE_BYTES = NOPS * B_BYTES;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* wst = smem + 2 * SLOT_BYTES;
    float* stage = reinterpret_cast<float*>(wst + STAGES * STAGE_BYTES);          // [32 pixels][C3W_SP]
    float2* gnred = reinterpret_cast<float2*>(stage + 32 * C3W_SP);               // [8 warps][32 lanes] GroupNorm partial sums
    uint64_t* full = reinterpret_cast<uint64_t*>(gnred + 256);
    uint64_t* empty = full + STAGES;
    uint64_t* hfull = empty + STAGES;
    uint64_t* hempty = hfull + 2;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nkb = 9 * (p.Cin / 64);
    const int total = p.tiles_x * p.tiles_y * p.tiles_b * p.n_tiles_n;

    if (warp == 8 && lane == 0) {
        tc::prefetch_tmap(&tmA);
        tc::prefetch_tmap(&tmB);
        // empty[s] / hempty[h]: one arrival per consumer warp -- empty once its fragments are in registers, hempty once its
        // warpgroup's MMAs reading the halo have completed
        for (int s = 0; s < STAGES; s++) { tc::mbar_init(&full[s], 1); tc::mbar_init(&empty[s], 8); }
        for (int h = 0; h < 2; h++) { tc::mbar_init(&hfull[h], 1); tc::mbar_init(&hempty[h], 8); }
        tc::fence_barrier_init();
    }
    __syncthreads();

    if (warp >= 8) {
        tc::setmaxnreg_dec<C3W_REGS_PRODUCER>();
        if (warp == 8 && lane == 0)
            c3_produce<128, STAGES, SLOT_BYTES, T::HALO>(&tmA, &tmB, &tmAlo, &tmBlo, p, smem, wst, full, empty, hfull, hempty);
        return;
    }
    tc::setmaxnreg_inc<C3W_REGS_CONSUMER>();

    // ---- consumer warpgroups 0, 1: output channels [64 wg, 64 wg + 64) of the tile, all NP pixels
    const int wg = warp >> 2;
    // ldmatrix.x4 of the m64k16 A fragment: lane l addresses row 16 (warp % 4) + l % 8 + 8 ((l / 8) % 2) of this warpgroup's 64,
    // 16 B chunk l / 16 + 2 j (k16 step j) of the 128 B swizzled row, stored at chunk (l / 16 + 2 j) ^ (row % 8) -- the byte
    // offset of step j is lofs ^ 32 j (stages are 1024 B aligned)
    const uint32_t lofs = (64 * wg + 16 * (warp & 3) + (lane & 7) + 8 * ((lane >> 3) & 1)) * 128 + (((lane >> 4) ^ (lane & 7)) << 4);
    const uint32_t halo0 = tc::smem_u32(smem), wst0 = tc::smem_u32(wst);

    float acc[T::NP / 2];
#pragma unroll
    for (int i = 0; i < T::NP / 2; i++) acc[i] = 0.f;
    uint32_t frag[2][2][4][4];                          // [tap parity][hi, lo][k16 step][register]
    uint32_t it = 0, hit = 0;
    // one k block (tap): fragments of tap kb into frag[F] (their previous reader, tap kb - 2, has completed), MMAs issued, then
    // wait until tap kb - 1 has completed
    auto kblock = [&](int kb, uint32_t (&fr)[2][4][4]) {
        const int tap = kb % 9;
        if (tap == 0) tc::mbar_wait(&hfull[hit % 2], (hit / 2) & 1);
        const int s = it % STAGES;
        tc::mbar_wait(&full[s], (it / STAGES) & 1);
        const uint32_t w = wst0 + s * STAGE_BYTES + lofs;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            ldsm_x4(fr[0][j], w ^ (32 * j));
            ldsm_x4(fr[1][j], (w + B_BYTES) ^ (32 * j));
        }
        const uint32_t x = halo0 + (hit % 2) * SLOT_BYTES + ((tap / 3) * 10 + tap % 3) * 128;
        tc::wgmma_fence();
        c3w_mma_kblock<TH, NB>(acc, fr[0], fr[1], x, kb == 0);
        tc::wgmma_commit();
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(&empty[s]);       // the wgmmas above have read the fragments: the stage is free
        tc::wgmma_wait<1>();
        if (tap == 0 && kb > 0 && lane == 0) tc::mbar_arrive(&hempty[(hit - 1) % 2]);   // the previous slab's last tap is complete
        it++;
        if (tap == 8) hit++;
    };
    for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
        for (int kb = 0; kb < nkb; kb += 2) {
            kblock(kb, frag[0]);
            if (kb + 1 < nkb) kblock(kb + 1, frag[1]);
        }
        tc::wgmma_wait<0>();
        tc::acc_fence(acc);
        if (lane == 0) tc::mbar_arrive(&hempty[(hit - 1) % 2]);

        // ---- epilogue, 32 pixels at a time through the staging buffer: consumer warp w (0..7) <-> pixels w, w + 8, w + 16, w + 24 of
        // the chunk, lane <-> output channels [4 lane, 4 lane + 4), so every warp access to the output and the residual is one pixel's
        // 512 contiguous bytes.  The chunks are the 32-pixel sets the GroupNorm partial statistics are formed over.
        const int nt = tile % p.n_tiles_n, mt = tile / p.n_tiles_n;
        const int tx = mt % p.tiles_x, ty = (mt / p.tiles_x) % p.tiles_y, tb = mt / (p.tiles_x * p.tiles_y);
        const int srow = 2 * (lane & 3), scol = 64 * wg + 16 * (warp & 3) + (lane >> 2);
        const int n0 = nt * 128 + 4 * lane;
#pragma unroll
        for (int c = 0; c < T::NP / 32; c++) {
#pragma unroll
            for (int jj = 0; jj < 4; jj++)
#pragma unroll
                for (int i = 0; i < 4; i++)
                    stage[(8 * jj + srow + (i & 1)) * C3W_SP + scol + 8 * (i >> 1)] = acc[4 * (4 * c + jj) + i];
            tc::bar_sync(1, 256);
            // pixel 8 r + warp of the chunk: x = tx * 8 + warp, output row y0 + r of image b (TH % 4 == 0: one image per chunk)
            const int x = tx * 8 + warp, y0 = ty * TH + (4 * c) % TH, b = tb * NB + (4 * c) / TH;
            const int64_t off = (((int64_t)b * p.H + y0) * p.W + x) * p.Cout + n0;
            const int rs = p.W * p.Cout;                     // one output row
            const float4 bb = *reinterpret_cast<const float4*>(p.bias + n0);
            float4 v[4];
            unsigned valid = 0;
#pragma unroll
            for (int r = 0; r < 4; r++) {
                if (x < p.W && y0 + r < p.H && b < p.B) valid |= 1u << r;
                const float4 q = *reinterpret_cast<const float4*>(stage + (8 * r + warp) * C3W_SP + 4 * lane);
                v[r] = make_float4(q.x + bb.x, q.y + bb.y, q.z + bb.z, q.w + bb.w);
            }
            if (p.out_nchw) {
                const int64_t cs = (int64_t)p.H * p.W;
#pragma unroll
                for (int r = 0; r < 4; r++)
                    if (valid >> r & 1) {
                        float* o = p.out + (((int64_t)b * p.Cout + n0) * p.H + y0 + r) * p.W + x;
                        o[0] = v[r].x; o[cs] = v[r].y; o[2 * cs] = v[r].z; o[3 * cs] = v[r].w;
                    }
            } else {
                if (p.residual) {
#pragma unroll
                    for (int r = 0; r < 4; r++)
                        if (valid >> r & 1) {
                            const float4 rr = *reinterpret_cast<const float4*>(p.residual + off + r * rs);
                            v[r].x += rr.x; v[r].y += rr.y; v[r].z += rr.z; v[r].w += rr.w;
                        }
                }
#pragma unroll
                for (int r = 0; r < 4; r++)
                    if (valid >> r & 1) *reinterpret_cast<float4*>(p.out + off + r * rs) = v[r];
            }
            const int cl = p.Cout >> 7;                      // lanes per GroupNorm(32) group: cg = Cout / 32 = 4 cl channels
            if (p.gn_part != nullptr) {
                float s1 = 0.f, s2 = 0.f;
#pragma unroll
                for (int r = 0; r < 4; r++)
                    if (valid >> r & 1) {
                        s1 += (v[r].x + v[r].y) + (v[r].z + v[r].w);
                        s2 += fmaf(v[r].x, v[r].x, v[r].y * v[r].y) + fmaf(v[r].z, v[r].z, v[r].w * v[r].w);
                    }
                for (int m = 1; m < cl; m <<= 1) {
                    s1 += __shfl_xor_sync(0xffffffffu, s1, m);
                    s2 += __shfl_xor_sync(0xffffffffu, s2, m);
                }
                gnred[warp * 32 + lane] = make_float2(s1, s2);
            }
            tc::bar_sync(1, 256);
            if (p.gn_part != nullptr && warp == 0 && (lane & (cl - 1)) == 0) {     // one lane per group sums the 8 warps' pixels
                float s1 = 0.f, s2 = 0.f;
#pragma unroll
                for (int w = 0; w < 8; w++) {
                    const float2 q = gnred[w * 32 + lane];
                    s1 += q.x;
                    s2 += q.y;
                }
                const int chunk = (ty * p.tiles_x + tx) * (TH / 4) + c % (TH / 4);
                double* o = p.gn_part + (((int64_t)b * p.gn_chunks + chunk) * 32 + n0 / (4 * cl)) * 2;
                if (b < p.B) { o[0] = (double)s1; o[1] = (double)s2; }
            }
        }
    }
}

template <int TH, int NB, int STAGES>
static int launch_conv3x3_wreg_t(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmAlo, const CUtensorMap& tmBlo,
                                 const ConvTcParams& p, int n_sm, cudaStream_t st) {
    constexpr int NOPS = 2;
    constexpr size_t smem = (size_t)2 * NOPS * C3wTile<TH, NB>::HALO + (size_t)STAGES * NOPS * 128 * 128 + 32 * C3W_SP * 4 + 256 * 8 + 1024 + 256;
    static_assert(smem <= 227 * 1024, "conv3x3_wreg: shared memory budget");
    RQB_ENSURE_SMEM(smem, conv3x3_wreg_kernel<TH, NB, STAGES>);
    const int total = p.tiles_x * p.tiles_y * p.tiles_b * p.n_tiles_n;
    const int grid = total < n_sm ? total : n_sm;
    conv3x3_wreg_kernel<TH, NB, STAGES><<<grid, C3W_THREADS, smem, st>>>(tmA, tmB, tmAlo, tmBlo, p);
    return check_launch("conv3x3_wreg");
}

static int sm_count() {
    static int n = 0;
    if (!n) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        if (n <= 0) n = 132;
    }
    return n;
}

bool conv_tc_supported(int H, int W, int Cin, int Cout, int ks, int stride, int in_nchw, int out_nchw) {
    if ((stride != 1 && !(stride == 2 && ks == 3)) || in_nchw || (ks != 1 && ks != 3)) return false;
    if (Cin % 64 != 0) return false;
    if (Cout != 3 && Cout % 128 != 0 && Cout != 64) return false;
    if (!out_nchw && Cout % 16 != 0) return false;       // the NHWC epilogue reads bias / residual and stores 16 channels at a time
    return H > 0 && W > 0;
}

// output tile of one CTA, TW x TH x NB pixels.  3x3 stride 1, 8 pixels wide: Cout % 128 == 0 (conv3x3_wreg_kernel) 32 rows
// (256 pixels), 16 rows, or 8 rows of NB = 2 images below 16 rows; other Cout (conv3x3_tc_kernel) 16 rows, or 8 rows of NB = 2
// images below 16 rows.  Else (conv_tc_kernel) 128 pixels: TW and TH the powers of two at or above W and H, capped at 16 and
// 128 / TW.  Maps narrower or lower than the tile, or not a multiple of it, leave the out-of-range part of it unstored; the TMA
// box reads zeros there.
static bool conv3x3_wreg(int Cout, int ks, int stride) { return ks == 3 && stride == 1 && Cout % 128 == 0; }

static void conv_tile(int H, int W, int Cout, int ks, int stride, int& TW, int& TH, int& NB) {
    if (ks == 3 && stride == 1) {
        TW = 8;
        TH = conv3x3_wreg(Cout, ks, stride) && H >= 32 ? 32 : (H > 8 ? 16 : 8);
        NB = TH == 8 ? 2 : 1;
    } else {
        auto pow2_ceil = [](int v) { int p = 1; while (p < v) p *= 2; return p; };
        TW = pow2_ceil(W < 16 ? W : 16);
        TH = pow2_ceil(H < 128 / TW ? H : 128 / TW);
        NB = 128 / (TW * TH);
    }
}

// the epilogue can emit the output's GroupNorm(32) partial statistics when the tiles cover the map exactly, every epilogue warp's
// 32 pixels lie in one image and a 16-channel chunk holds whole groups
bool conv_tc_gn_fusable(int H, int W, int Cout, int ks, int stride) {
    int TW, TH, NB;
    conv_tile(H, W, Cout, ks, stride, TW, TH, NB);
    const int cg = Cout / 32;
    return Cout % 32 == 0 && (cg == 4 || cg == 8 || cg == 16) && W % TW == 0 && H % TH == 0 && TW * TH >= 32 && (H * W) % 32 == 0;
}

// X: NHWC fp16 [B,H*stride,W*stride,Cin]; Wt: [Cout, ks, ks, Cin] fp16; out fp32 [B,H,W,Cout].  X16lo / W16lo (required): their
// fp16 lo halves, for the split-fp16 products.  H, W are the OUTPUT extent.
int launch_conv_tc(const void* X16, const void* W16, const void* X16lo, const void* W16lo, const float* bias,
                   const float* residual, float* out, int B, int H, int W, int Cin, int Cout, int ks, int out_nchw,
                   cudaStream_t st, int stride, double* gn_part) {
    if (X16lo == nullptr || W16lo == nullptr) return fail(RQB200_EINVAL, "conv_tc: the lo halves X16lo and W16lo are required");
    // the NHWC epilogue moves 16 channels per access (past the end of `out` unless Cout % 16 == 0); the NCHW one adds no residual
    if (!out_nchw && Cout % 16 != 0) return fail(RQB200_EINVAL, "conv_tc: an NHWC output needs Cout % 16 == 0");
    if (out_nchw && residual != nullptr) return fail(RQB200_EINVAL, "conv_tc: an NCHW output takes no residual");
    ConvTcParams p = {};
    p.B = B; p.H = H; p.W = W; p.Cin = Cin; p.Cout = Cout; p.ks = ks; p.stride = stride;
    conv_tile(H, W, Cout, ks, stride, p.TW, p.TH, p.NB);
    const bool c3 = ks == 3 && stride == 1;
    p.tiles_x = (int)ceil_div(W, p.TW); p.tiles_y = (int)ceil_div(H, p.TH); p.tiles_b = (int)ceil_div(B, p.NB);
    // 3x3: 128 output channels per tile (conv3x3_wreg_kernel), or 16 | 64 (conv3x3_tc_kernel)
    const int BN = Cout <= 16 ? 16 : (Cout % 256 == 0 && !c3 ? 256 : (Cout % 128 == 0 ? 128 : 64));
    p.n_tiles_n = (int)ceil_div(Cout, BN);
    p.bias = bias; p.residual = residual; p.out = out; p.out_nchw = out_nchw;
    if (gn_part != nullptr) {
        if (!conv_tc_gn_fusable(H, W, Cout, ks, stride) || out_nchw)
            return fail(RQB200_EINVAL, "conv_tc: GroupNorm statistics cannot be fused for this shape");
        p.gn_part = gn_part;
        p.gn_chunks = H * W / 32;
    }
    CUtensorMap tmA, tmB, tmAlo, tmBlo;
    RQB_TRY(make_tmap_2d(&tmB, W16, 1, (uint64_t)ks * ks * Cin, (uint64_t)Cout, (uint64_t)ks * ks * Cin * 2, 64, (uint32_t)BN));
    RQB_TRY(make_tmap_2d(&tmBlo, W16lo, 1, (uint64_t)ks * ks * Cin, (uint64_t)Cout, (uint64_t)ks * ks * Cin * 2, 64, (uint32_t)BN));
    const int n_sm = sm_count();
    if (c3) {
        // the halo box: the tile plus one pixel on every side
        RQB_TRY(make_tmap_4d_nhwc(&tmA, X16, (uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)B, 64, (uint32_t)p.TW + 2,
                                  (uint32_t)p.TH + 2, (uint32_t)p.NB, 1));
        RQB_TRY(make_tmap_4d_nhwc(&tmAlo, X16lo, (uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)B, 64, (uint32_t)p.TW + 2,
                                  (uint32_t)p.TH + 2, (uint32_t)p.NB, 1));
        if (conv3x3_wreg(Cout, ks, stride)) {
            if (p.TH == 32) return launch_conv3x3_wreg_t<32, 1, 1>(tmA, tmB, tmAlo, tmBlo, p, n_sm, st);
            if (p.TH == 16) return launch_conv3x3_wreg_t<16, 1, 3>(tmA, tmB, tmAlo, tmBlo, p, n_sm, st);
            return launch_conv3x3_wreg_t<8, 2, 3>(tmA, tmB, tmAlo, tmBlo, p, n_sm, st);
        }
        return BN == 16 ? launch_conv3x3_tc_t<16, 8>(tmA, tmB, tmAlo, tmBlo, p, n_sm, st)
                        : launch_conv3x3_tc_t<64, 4>(tmA, tmB, tmAlo, tmBlo, p, n_sm, st);
    }
    RQB_TRY(make_tmap_4d_nhwc(&tmA, X16, (uint64_t)Cin, (uint64_t)W * stride, (uint64_t)H * stride, (uint64_t)B, 64, (uint32_t)p.TW,
                              (uint32_t)p.TH, (uint32_t)p.NB, (uint32_t)stride));
    RQB_TRY(make_tmap_4d_nhwc(&tmAlo, X16lo, (uint64_t)Cin, (uint64_t)W * stride, (uint64_t)H * stride, (uint64_t)B, 64,
                              (uint32_t)p.TW, (uint32_t)p.TH, (uint32_t)p.NB, (uint32_t)stride));
    switch (BN) {
        case 16: return launch_conv_tc_t<16, 5, 3>(tmA, tmB, tmAlo, tmBlo, p, n_sm, st);
        case 64: return launch_conv_tc_t<64, 4, 3>(tmA, tmB, tmAlo, tmBlo, p, n_sm, st);
        case 128: return launch_conv_tc_t<128, 3, 3>(tmA, tmB, tmAlo, tmBlo, p, n_sm, st);
        default: return launch_conv_tc_t<256, 2, 3>(tmA, tmB, tmAlo, tmBlo, p, n_sm, st);
    }
}

// Rows GEMM through the persistent conv kernel: out[m, n] = act(sum_k X[m,k] W[n,k] + bias[n]) (+ residual[m,n]) for M token rows
// -- a 1x1 "conv" over ceil(M/128) images of 16x8 pixels.  The batched prefill / teacher-forced forward passes of the AR tier
// (csrc/ar_fast.cu) use it for M > 256: persistent CTAs, 128 x BN tiles, operand loads of the next tile overlapped with
// this tile's epilogue -- what gemm_tc_kernel (a weight streamer built for M <= 256) does not have.
// gelu: 0 none, 1 exact GELU, 2 QuickGELU (16-bit output only).
// X [M_alloc, K] 16-bit with M_alloc >= ceil(M/128)*128 rows readable; exactly one of out_f32 / out_16 non-null;
// residual (f32, may alias out_f32) only with out_f32.  N_out % 128 == 0, K % 64 == 0.
int launch_rows_gemm_tc(const void* X16, const void* W16, const float* bias, const float* residual, float* out_f32, void* out_16,
                        int gelu, int fmt, int64_t M, int N_out, int K, cudaStream_t st) {
    if (N_out % 128 != 0 || K % 64 != 0 || M < 1 || (out_f32 == nullptr) == (out_16 == nullptr) || bias == nullptr)
        return fail(RQB200_EINVAL, "rows_gemm_tc: need N_out % 128 == 0, K % 64 == 0, a bias and exactly one output");
    ConvTcParams p = {};
    p.B = (int)ceil_div(M, 128); p.H = 8; p.W = 16; p.Cin = K; p.Cout = N_out; p.ks = 1; p.stride = 1;
    p.TW = 16; p.TH = 8; p.NB = 1;
    p.tiles_x = 1; p.tiles_y = 1; p.tiles_b = p.B;
    const int BN = N_out % 256 == 0 ? 256 : 128;
    p.n_tiles_n = N_out / BN;
    p.bias = bias; p.residual = residual; p.out = out_f32; p.out_nchw = 0;
    p.out16 = out_16; p.gelu = gelu; p.fmt = fmt; p.m_rows = M;
    CUtensorMap tmA, tmB;
    RQB_TRY(make_tmap_4d_nhwc(&tmA, X16, (uint64_t)K, 16, 8, (uint64_t)p.B, 64, 16, 8, 1, 1));
    RQB_TRY(make_tmap_2d(&tmB, W16, 1, (uint64_t)K, (uint64_t)N_out, (uint64_t)K * 2, 64, (uint32_t)BN));
    const int n_sm = sm_count();
    if (gelu == 2) {
        if (BN == 256) return launch_conv_tc_t<256, 4, 1, true>(tmA, tmB, tmA, tmB, p, n_sm, st);
        return launch_conv_tc_t<128, 6, 1, true>(tmA, tmB, tmA, tmB, p, n_sm, st);
    }
    if (BN == 256) return launch_conv_tc_t<256, 4, 1>(tmA, tmB, tmA, tmB, p, n_sm, st);
    return launch_conv_tc_t<128, 6, 1>(tmA, tmB, tmA, tmB, p, n_sm, st);
}

// ------------------------------------------------------------------------------------------------ Inception convs (fast tier)
// The Inception engine's convs on conv_tc_kernel's layout, generalised: any KH x KW with separate top/bottom and left/right zero
// padding (the tap's box starts at x * stride + kx - pad_w, y * stride + ky - pad_h; TMA zero-fills every box element at a negative
// or past-the-end coordinate, which IS the padding, also with the element stride 2 of a padded stride-2 conv, whose box can start at
// -1), stride-2 convs, and Cin % 8 == 0 rather than % 64: the activation's
// tensor map has the true channel extent Cin, so the last 64-channel slab's channels past Cin are zero-filled in A and multiply the
// next tap's weights (or the weight map's own zero fill) to zero.  That keeps the activations unpadded, so the engine's concat
// buffers stay exactly the reference's channel layout.  Epilogue: bias + ReLU, stored at channel yoff of rows of ldy as fp32 and
// as the next conv's fp16 hi / lo operands (no cast pass between convs).
struct IncTcParams {
    int B, H, W, Cin, Cout;        // H, W: OUTPUT extent
    int KH, KW, pad_h, pad_w, stride;
    int TW, TH, NB;
    int tiles_x, tiles_y, tiles_b, n_tiles_n;
    const float* bias;
    float* out;                    // fp32 [B, H, W, ldy] or null
    __half* out_hi;                // fp16 hi / lo of the same values, [B, H, W, ldy], or null
    __half* out_lo;
    int ldy, yoff;
    const float* residual;         // residual forms only: fp32 [B, H, W, ldy] read at the output's own index, or null
};

// EPI: 0 = ReLU(acc + bias) (the Inception and LPIPS plans); 1 / 2 = act(acc + bias [+ residual]) with act ReLU / the identity (the
// ResNet plan's bottleneck conv3 and downsample convs)
template <int BN, int STAGES, int EPI>
__device__ __forceinline__ void inc_conv_tc_body(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmAlo,
                                                 const CUtensorMap& tmBlo, const IncTcParams& p) {
    constexpr int B_BYTES = BN * 64 * 2;
    constexpr int STAGE_BYTES = 2 * (CT_A_BYTES + B_BYTES);
    constexpr int OFF_B = 2 * CT_A_BYTES;                    // [A_hi | A_lo | B_hi | B_lo]
    constexpr int CW = BN < 32 ? BN : 32;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    float* stage = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES);
    uint64_t* full = reinterpret_cast<uint64_t*>(stage + 128 * (CW + 4));
    uint64_t* empty = full + STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int cslabs = (p.Cin + 63) / 64;
    const int nkb = p.KH * p.KW * cslabs;
    const int sx = p.stride;
    const int m_tiles = p.tiles_x * p.tiles_y * p.tiles_b;
    const int total = m_tiles * p.n_tiles_n;

    if (warp == 8 && lane == 0) {
        tc::prefetch_tmap(&tmA);
        tc::prefetch_tmap(&tmB);
        for (int s = 0; s < STAGES; s++) { tc::mbar_init(&full[s], 1); tc::mbar_init(&empty[s], 8); }
        tc::fence_barrier_init();
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            uint32_t it = 0;
            for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
                const int nt = tile % p.n_tiles_n, mt = tile / p.n_tiles_n;
                const int tx = mt % p.tiles_x, ty = (mt / p.tiles_x) % p.tiles_y, tb = mt / (p.tiles_x * p.tiles_y);
                const int x0 = tx * p.TW, y0 = ty * p.TH, b0 = tb * p.NB;
                for (int kb = 0; kb < nkb; kb++, it++) {
                    const int s = it % STAGES;
                    tc::mbar_wait(&empty[s], ((it / STAGES) & 1) ^ 1);
                    const int tap = kb / cslabs, c0 = (kb % cslabs) * 64;
                    const int ky = tap / p.KW, kx = tap % p.KW;
                    const int ix = x0 * sx + kx - p.pad_w, iy = y0 * sx + ky - p.pad_h;
                    tc::mbar_expect_tx(&full[s], STAGE_BYTES);
                    uint8_t* st = smem + s * STAGE_BYTES;
                    tc::tma_load_4d(st, &tmA, &full[s], c0, ix, iy, b0, tc::L2_EVICT_NORMAL);
                    tc::tma_load_4d(st + CT_A_BYTES, &tmAlo, &full[s], c0, ix, iy, b0, tc::L2_EVICT_NORMAL);
                    tc::tma_load_2d(st + OFF_B, &tmB, &full[s], tap * p.Cin + c0, nt * BN, tc::L2_EVICT_LAST);
                    tc::tma_load_2d(st + OFF_B + B_BYTES, &tmBlo, &full[s], tap * p.Cin + c0, nt * BN, tc::L2_EVICT_LAST);
                }
            }
        }
        return;
    }

    const int wg = warp >> 2, t = threadIdx.x;
    const int r = t & 127;
    const int rx = r % p.TW, ry = (r / p.TW) % p.TH, rb = r / (p.TW * p.TH);
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; i++) acc[i] = 0.f;
    uint32_t it = 0;
    for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
        for (int kb = 0; kb < nkb; kb++, it++) {
            const int s = it % STAGES;
            tc::mbar_wait(&full[s], (it / STAGES) & 1);
            const uint32_t a = tc::smem_u32(smem + s * STAGE_BYTES) + wg * (64 * 128), b = tc::smem_u32(smem + s * STAGE_BYTES + OFF_B);
            tc::wgmma_fence();
            ct_mma_kblock<BN, 0, 3>(acc, a, b, kb == 0);
            tc::wgmma_commit();
            tc::wgmma_wait<1>();
            if (kb > 0 && lane == 0) tc::mbar_arrive(&empty[(it - 1) % STAGES]);
        }
        tc::wgmma_wait<0>();
        tc::acc_fence(acc);
        if (lane == 0) tc::mbar_arrive(&empty[(it - 1) % STAGES]);

        const int nt = tile % p.n_tiles_n, mt = tile / p.n_tiles_n;
        const int tx = mt % p.tiles_x, ty = (mt / p.tiles_x) % p.tiles_y, tb = mt / (p.tiles_x * p.tiles_y);
        const int x = tx * p.TW + rx, y = ty * p.TH + ry, b = tb * p.NB + rb;
        const int64_t pix = ((int64_t)b * p.H + y) * p.W + x;
        const bool valid = (x < p.W) && (y < p.H) && (b < p.B);
        tc::drain_acc<BN, CW, 0>(acc, stage, wg, t, [&p, nt, pix, valid](const float (&v)[16], int, int c) {
            const int n0 = nt * BN + c;
            if (n0 >= p.Cout || !valid) return;                     // Cout % 16 == 0: a 16-channel chunk is all in or all out
            float w[16];
            const int64_t o = pix * p.ldy + p.yoff + n0;
            if (EPI == 0) {
#pragma unroll
                for (int i = 0; i < 16; i += 4) {
                    const float4 bb = *reinterpret_cast<const float4*>(p.bias + n0 + i);
                    w[i] = fmaxf(v[i] + bb.x, 0.f); w[i + 1] = fmaxf(v[i + 1] + bb.y, 0.f);
                    w[i + 2] = fmaxf(v[i + 2] + bb.z, 0.f); w[i + 3] = fmaxf(v[i + 3] + bb.w, 0.f);
                }
            } else {
#pragma unroll
                for (int i = 0; i < 16; i += 4) {
                    const float4 bb = *reinterpret_cast<const float4*>(p.bias + n0 + i);
                    w[i] = v[i] + bb.x; w[i + 1] = v[i + 1] + bb.y; w[i + 2] = v[i + 2] + bb.z; w[i + 3] = v[i + 3] + bb.w;
                    if (p.residual) {
                        const float4 rr = *reinterpret_cast<const float4*>(p.residual + o + i);
                        w[i] += rr.x; w[i + 1] += rr.y; w[i + 2] += rr.z; w[i + 3] += rr.w;
                    }
                    if (EPI == 1) {
                        w[i] = fmaxf(w[i], 0.f); w[i + 1] = fmaxf(w[i + 1], 0.f); w[i + 2] = fmaxf(w[i + 2], 0.f); w[i + 3] = fmaxf(w[i + 3], 0.f);
                    }
                }
            }
            if (p.out) {
#pragma unroll
                for (int i = 0; i < 16; i += 4) *reinterpret_cast<float4*>(p.out + o + i) = make_float4(w[i], w[i + 1], w[i + 2], w[i + 3]);
            }
            if (p.out_hi) {
                uint32_t hi[8], lo[8];
#pragma unroll
                for (int i = 0; i < 8; i++) {
                    __half2 h, l;
                    split_f16x2(w[2 * i], w[2 * i + 1], h, l);
                    hi[i] = *reinterpret_cast<const uint32_t*>(&h);
                    lo[i] = *reinterpret_cast<const uint32_t*>(&l);
                }
                uint4* dh = reinterpret_cast<uint4*>(p.out_hi + o);
                dh[0] = make_uint4(hi[0], hi[1], hi[2], hi[3]);
                dh[1] = make_uint4(hi[4], hi[5], hi[6], hi[7]);
                uint4* dl = reinterpret_cast<uint4*>(p.out_lo + o);
                dl[0] = make_uint4(lo[0], lo[1], lo[2], lo[3]);
                dl[1] = make_uint4(lo[4], lo[5], lo[6], lo[7]);
            }
        });
    }
}

template <int BN, int STAGES>
__global__ void __launch_bounds__(CT_THREADS, 1)
inc_conv_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                   const __grid_constant__ CUtensorMap tmAlo, const __grid_constant__ CUtensorMap tmBlo, IncTcParams p) {
    inc_conv_tc_body<BN, STAGES, 0>(tmA, tmB, tmAlo, tmBlo, p);
}

// the residual forms (the ResNet plan): act(conv + bias [+ p.residual]), act ReLU when RELU, else the identity
template <int BN, int STAGES, bool RELU>
__global__ void __launch_bounds__(CT_THREADS, 1)
inc_conv_tc_res_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                       const __grid_constant__ CUtensorMap tmAlo, const __grid_constant__ CUtensorMap tmBlo, IncTcParams p) {
    inc_conv_tc_body<BN, STAGES, RELU ? 1 : 2>(tmA, tmB, tmAlo, tmBlo, p);
}

template <int BN, int STAGES>
static int launch_inc_conv_tc_t(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmAlo, const CUtensorMap& tmBlo,
                                const IncTcParams& p, int n_sm, cudaStream_t st) {
    constexpr size_t smem = (size_t)STAGES * 2 * (CT_A_BYTES + BN * 128) + 128 * ((BN < 32 ? BN : 32) + 4) * 4 + 1024 + 256;
    static_assert(smem <= 227 * 1024, "inc_conv_tc: shared memory budget");
    RQB_ENSURE_SMEM(smem, inc_conv_tc_kernel<BN, STAGES>);
    const int total = p.tiles_x * p.tiles_y * p.tiles_b * p.n_tiles_n;
    inc_conv_tc_kernel<BN, STAGES><<<total < n_sm ? total : n_sm, CT_THREADS, smem, st>>>(tmA, tmB, tmAlo, tmBlo, p);
    return check_launch("inc_conv_tc");
}

template <int BN, int STAGES, bool RELU>
static int launch_inc_conv_tc_res_t(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmAlo, const CUtensorMap& tmBlo,
                                    const IncTcParams& p, int n_sm, cudaStream_t st) {
    constexpr size_t smem = (size_t)STAGES * 2 * (CT_A_BYTES + BN * 128) + 128 * ((BN < 32 ? BN : 32) + 4) * 4 + 1024 + 256;
    static_assert(smem <= 227 * 1024, "inc_conv_tc: shared memory budget");
    RQB_ENSURE_SMEM(smem, (inc_conv_tc_res_kernel<BN, STAGES, RELU>));
    const int total = p.tiles_x * p.tiles_y * p.tiles_b * p.n_tiles_n;
    inc_conv_tc_res_kernel<BN, STAGES, RELU><<<total < n_sm ? total : n_sm, CT_THREADS, smem, st>>>(tmA, tmB, tmAlo, tmBlo, p);
    return check_launch("inc_conv_tc_res");
}

int launch_inc_conv_tc(const void* X16, const void* X16lo, const void* W16, const void* W16lo, const float* bias, float* out,
                       void* out_hi, void* out_lo, int B, int Hi, int Wi, int Cin, int Cout, int KH, int KW, int pad_h, int pad_w,
                       int stride, int ldy, int yoff, cudaStream_t st, int epi, const float* residual) {
    if (epi < 0 || epi > 2 || (residual && epi == 0))
        return fail(RQB200_EINVAL, "inc_conv_tc: epilogue must be 0 (ReLU), 1 (residual + ReLU) or 2 (residual, no ReLU)");
    if (!X16 || !X16lo || !W16 || !W16lo || !bias || (!out && !out_hi) || (out_hi && !out_lo))
        return fail(RQB200_EINVAL, "inc_conv_tc: need both operand halves, a bias and an fp32 or an fp16 hi + lo output");
    if (Cin % 8 || Cout % 16 || ldy % 16 || yoff % 16 || yoff + Cout > ldy || (stride != 1 && stride != 2) || KH < 1 || KW < 1 ||
        pad_h < 0 || pad_w < 0)
        return fail(RQB200_EINVAL, "inc_conv_tc: need Cin % 8 == 0, Cout, ldy, yoff % 16 == 0, yoff + Cout <= ldy, stride 1 | 2");
    IncTcParams p = {};
    p.B = B; p.Cin = Cin; p.Cout = Cout; p.KH = KH; p.KW = KW; p.pad_h = pad_h; p.pad_w = pad_w; p.stride = stride;
    p.H = (Hi + 2 * pad_h - KH) / stride + 1;
    p.W = (Wi + 2 * pad_w - KW) / stride + 1;
    if (B < 1 || p.H < 1 || p.W < 1) return fail(RQB200_EINVAL, "inc_conv_tc: empty output");
    auto pow2_ceil = [](int v) { int q = 1; while (q < v) q *= 2; return q; };
    p.TW = pow2_ceil(p.W < 16 ? p.W : 16);
    p.TH = pow2_ceil(p.H < 128 / p.TW ? p.H : 128 / p.TW);
    p.NB = 128 / (p.TW * p.TH);
    p.tiles_x = (int)ceil_div(p.W, p.TW); p.tiles_y = (int)ceil_div(p.H, p.TH); p.tiles_b = (int)ceil_div(B, p.NB);
    const int BN = Cout >= 128 ? 128 : 64;
    p.n_tiles_n = (int)ceil_div(Cout, BN);
    p.bias = bias; p.out = out; p.out_hi = (__half*)out_hi; p.out_lo = (__half*)out_lo; p.ldy = ldy; p.yoff = yoff; p.residual = residual;
    const uint64_t K = (uint64_t)KH * KW * Cin;
    CUtensorMap tmA, tmB, tmAlo, tmBlo;
    RQB_TRY(make_tmap_2d(&tmB, W16, 1, K, (uint64_t)Cout, K * 2, 64, (uint32_t)BN));
    RQB_TRY(make_tmap_2d(&tmBlo, W16lo, 1, K, (uint64_t)Cout, K * 2, 64, (uint32_t)BN));
    RQB_TRY(make_tmap_4d_nhwc(&tmA, X16, (uint64_t)Cin, (uint64_t)Wi, (uint64_t)Hi, (uint64_t)B, 64, (uint32_t)p.TW, (uint32_t)p.TH,
                              (uint32_t)p.NB, (uint32_t)stride));
    RQB_TRY(make_tmap_4d_nhwc(&tmAlo, X16lo, (uint64_t)Cin, (uint64_t)Wi, (uint64_t)Hi, (uint64_t)B, 64, (uint32_t)p.TW, (uint32_t)p.TH,
                              (uint32_t)p.NB, (uint32_t)stride));
    const int n_sm = sm_count();
    if (epi == 1)
        return BN == 128 ? launch_inc_conv_tc_res_t<128, 3, true>(tmA, tmB, tmAlo, tmBlo, p, n_sm, st)
                         : launch_inc_conv_tc_res_t<64, 4, true>(tmA, tmB, tmAlo, tmBlo, p, n_sm, st);
    if (epi == 2)
        return BN == 128 ? launch_inc_conv_tc_res_t<128, 3, false>(tmA, tmB, tmAlo, tmBlo, p, n_sm, st)
                         : launch_inc_conv_tc_res_t<64, 4, false>(tmA, tmB, tmAlo, tmBlo, p, n_sm, st);
    return BN == 128 ? launch_inc_conv_tc_t<128, 3>(tmA, tmB, tmAlo, tmBlo, p, n_sm, st)
                     : launch_inc_conv_tc_t<64, 4>(tmA, tmB, tmAlo, tmBlo, p, n_sm, st);
}

// ------------------------------------------------------------------------------------------------ fp16 operand producers
// 4 fp32 values -> fp16 hi (+ optional fp16 lo = value - hi)
__device__ __forceinline__ void store_split4(__half* hi, __half* lo, const float (&v)[4]) {
    __half2 h0 = __floats2half2_rn(v[0], v[1]), h1 = __floats2half2_rn(v[2], v[3]);
    uint2 pk;
    pk.x = *reinterpret_cast<uint32_t*>(&h0);
    pk.y = *reinterpret_cast<uint32_t*>(&h1);
    *reinterpret_cast<uint2*>(hi) = pk;
    if (lo) {
        float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
        __half2 l0 = __floats2half2_rn(v[0] - f0.x, v[1] - f0.y), l1 = __floats2half2_rn(v[2] - f1.x, v[3] - f1.y);
        pk.x = *reinterpret_cast<uint32_t*>(&l0);
        pk.y = *reinterpret_cast<uint32_t*>(&l1);
        *reinterpret_cast<uint2*>(lo) = pk;
    }
}

// one warp per (image, group): reduce the per-chunk fp64 partial sums once (instead of once per apply CTA); fixed order
__global__ void gn_finalize_kernel(double* __restrict__ part, int B, int nchunks, double n, double eps) {
    const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (i >= B * 32) return;
    const int b = i / 32, g = i % 32;
    double ts = 0.0, tss = 0.0;
    for (int c = lane; c < nchunks; c += 32) {
        const double* o = part + (((int64_t)b * nchunks + c) * 32 + g) * 2;
        ts += o[0];
        tss += o[1];
    }
    ts = warp_sum_d(ts);
    tss = warp_sum_d(tss);
    if (lane != 0) return;
    double mean = ts / n, var = tss / n - mean * mean;
    if (var < 0.0) var = 0.0;
    double* fin = part + (int64_t)B * nchunks * 64 + (int64_t)i * 2;
    fin[0] = mean;
    fin[1] = 1.0 / sqrt(var + eps);
}

// GroupNorm apply (+SiLU) from the fp64 partial statistics of gn_stats_kernel, writing the fp16 NHWC conv operand
__global__ void __launch_bounds__(256) gn_apply_f16_kernel(const float* __restrict__ X, const double* __restrict__ part,
                                                           const float* __restrict__ gamma, const float* __restrict__ beta,
                                                           __half* __restrict__ Y, __half* __restrict__ Ylo, int HW, int C,
                                                           float eps, int silu, int nchunks) {
    __shared__ float s_mean[32], s_rstd[32];
    const int b = blockIdx.y;
    const int cg = C / 32;
    if (threadIdx.x < 32) {                                        // finalised by gn_finalize_kernel: (mean, rstd) per (b, group)
        const double* fin = part + (int64_t)gridDim.y * nchunks * 64 + ((int64_t)b * 32 + threadIdx.x) * 2;
        s_mean[threadIdx.x] = (float)fin[0];
        s_rstd[threadIdx.x] = (float)fin[1];
    }
    __syncthreads();
    (void)eps;
    // thread <-> 8 consecutive channels (two float4 loads, one 16 B store per output tensor); 32-bit indexing per image
    const int c8n = C / 8;
    const unsigned total8 = (unsigned)HW * (unsigned)c8n;
    const float* Xb = X + (int64_t)b * HW * C;
    __half* Yb = Y + (int64_t)b * HW * C;
    __half* Lb = Ylo ? Ylo + (int64_t)b * HW * C : nullptr;
    for (unsigned i = blockIdx.x * 256u + threadIdx.x; i < total8; i += gridDim.x * 256u) {
        const int c = (int)(i % (unsigned)c8n) * 8;
        const float4 x0 = __ldcs(reinterpret_cast<const float4*>(Xb + (size_t)i * 8));
        const float4 x1 = __ldcs(reinterpret_cast<const float4*>(Xb + (size_t)i * 8 + 4));
        const float4 ga0 = *reinterpret_cast<const float4*>(gamma + c), ga1 = *reinterpret_cast<const float4*>(gamma + c + 4);
        const float4 be0 = *reinterpret_cast<const float4*>(beta + c), be1 = *reinterpret_cast<const float4*>(beta + c + 4);
        const int g0 = c / cg, g1 = (c + 4) / cg;                 // cg % 4 == 0 -> each half shares a group
        const float m0 = s_mean[g0], r0 = s_rstd[g0], m1 = s_mean[g1], r1 = s_rstd[g1];
        float v[8] = {(x0.x - m0) * r0 * ga0.x + be0.x, (x0.y - m0) * r0 * ga0.y + be0.y, (x0.z - m0) * r0 * ga0.z + be0.z,
                      (x0.w - m0) * r0 * ga0.w + be0.w, (x1.x - m1) * r1 * ga1.x + be1.x, (x1.y - m1) * r1 * ga1.y + be1.y,
                      (x1.z - m1) * r1 * ga1.z + be1.z, (x1.w - m1) * r1 * ga1.w + be1.w};
        if (silu) {
#pragma unroll
            for (int k = 0; k < 8; k++) v[k] = v[k] / (1.0f + __expf(-v[k]));
        }
        __half2 h[4], l[4];
#pragma unroll
        for (int k = 0; k < 4; k++) split_f16x2(v[2 * k], v[2 * k + 1], h[k], l[k]);
        *reinterpret_cast<uint4*>(Yb + (size_t)i * 8) = *reinterpret_cast<uint4*>(h);
        if (Lb) *reinterpret_cast<uint4*>(Lb + (size_t)i * 8) = *reinterpret_cast<uint4*>(l);
    }
}

// fp32 NHWC -> fp16 NHWC, optionally nearest x2 upsampled (layers.py:31-35 folded into the operand producer)
__global__ void __launch_bounds__(256) cast_f16_kernel(const float* __restrict__ X, __half* __restrict__ Y, __half* __restrict__ Ylo,
                                                       int B, int H, int W, int C, int upsample) {
    const int c4n = C / 4;
    const int Ho = upsample ? 2 * H : H, Wo = upsample ? 2 * W : W;
    const int64_t total4 = (int64_t)B * Ho * Wo * c4n;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total4; i += (int64_t)gridDim.x * 256) {
        const int c4 = (int)(i % c4n);
        int64_t pix = i / c4n;
        const int ox = (int)(pix % Wo), oy = (int)((pix / Wo) % Ho), b = (int)(pix / ((int64_t)Wo * Ho));
        const int ix = upsample ? ox >> 1 : ox, iy = upsample ? oy >> 1 : oy;
        const float4 x = *reinterpret_cast<const float4*>(X + (((int64_t)b * H + iy) * W + ix) * C + c4 * 4);
        const float v[4] = {x.x, x.y, x.z, x.w};
        store_split4(Y + i * 4, Ylo ? Ylo + i * 4 : nullptr, v);
    }
}

// fused_chunks > 0: the partial statistics were already written by the producing conv's epilogue (fused_chunks = HW / 32 partials
// per image and group); otherwise gn_stats_kernel computes them (HW / 256 partials)
int launch_groupnorm_f16(const float* X, const float* gamma, const float* beta, void* Y16, void* Y16lo, double* stats_ws, int B,
                         int HW, int C, int silu, cudaStream_t st, int fused_chunks) {
    if (C % 128 != 0) return fail(RQB200_EINVAL, "groupnorm_f16: C % 128 != 0");
    const int nchunks = fused_chunks > 0 ? fused_chunks : (int)ceil_div(HW, 256);
    if (fused_chunks <= 0) RQB_TRY(launch_gn_stats(X, stats_ws, B, HW, C, st));
    gn_finalize_kernel<<<(unsigned)ceil_div(B * 32 * 32, 128), 128, 0, st>>>(stats_ws, B, nchunks, (double)HW * (C / 32), 1e-6);
    RQB_TRY(check_launch("gn_finalize"));
    int gx = (int)std::min<int64_t>(ceil_div((int64_t)HW * C / 8, 256), 1024);
    gn_apply_f16_kernel<<<dim3(gx, B), 256, 0, st>>>(X, stats_ws, gamma, beta, (__half*)Y16, (__half*)Y16lo, HW, C, 1e-6f, silu, nchunks);
    return check_launch("gn_apply_f16");
}

int launch_cast_f16(const float* X, void* Y16, void* Y16lo, int B, int H, int W, int C, int upsample, cudaStream_t st) {
    if (C % 4 != 0) return fail(RQB200_EINVAL, "cast_f16: C % 4 != 0");
    int64_t total4 = (int64_t)B * H * W * C / 4 * (upsample ? 4 : 1);
    int gx = (int)std::min<int64_t>(ceil_div(total4, 256), sm_count() * 16);
    cast_f16_kernel<<<gx, 256, 0, st>>>(X, (__half*)Y16, (__half*)Y16lo, B, H, W, C, upsample);
    return check_launch("cast_f16");
}

}  // namespace rqb

// diagnostic entry point: one conv through the wgmma path (tests/test_gpu_tc.py, tests/test_gpu_conv3x3.py)
// out_nchw bit 0: NCHW output; bit 1 (bf16 operands) is refused: the convs take fp16 only; bits 8.. : stride (0/1 -> 1, 2 -> the
// Downsample conv; then H, W are the OUTPUT extent)
extern "C" int rqb200_dbg_conv_tc(const void* X16, const void* W16, const void* X16lo, const void* W16lo, const float* bias,
                                  const float* residual, float* out, int B, int H, int W, int Cin, int Cout, int ks, int out_nchw,
                                  void* stream) {
    return rqb200_dbg_conv_tc_gn(X16, W16, X16lo, W16lo, bias, residual, out, nullptr, B, H, W, Cin, Cout, ks, out_nchw, stream);
}

// diagnostic entry point: one conv with the GroupNorm(32) partial statistics of its output emitted by the epilogue
// (tests/test_gpu_conv3x3.py, tests/test_gpu_vae_kernels.py); gn_part holds B * (H * W / 32) * 32 * 2 doubles, or is null (no
// statistics).  out_nchw bits as above (NCHW is rejected with gn_part).
extern "C" int rqb200_dbg_conv_tc_gn(const void* X16, const void* W16, const void* X16lo, const void* W16lo, const float* bias,
                                     const float* residual, float* out, double* gn_part, int B, int H, int W, int Cin, int Cout, int ks,
                                     int out_nchw, void* stream) {
    const int stride = (out_nchw >> 8) > 1 ? (out_nchw >> 8) : 1;
    if (!rqb::conv_tc_supported(H, W, Cin, Cout, ks, stride, 0, out_nchw & 1)) return rqb::fail(RQB200_EINVAL, "conv_tc: unsupported shape");
    if (out_nchw & 2) return rqb::fail(RQB200_EINVAL, "conv_tc: bf16 operands are not supported (fp16 only)");
    return rqb::launch_conv_tc(X16, W16, X16lo, W16lo, bias, residual, out, B, H, W, Cin, Cout, ks, out_nchw & 1, (cudaStream_t)stream,
                               stride, gn_part);
}

// diagnostic entry point: the rows GEMM (tests/test_gpu_tc.py).  X must have ceil(M/128)*128 readable rows.
extern "C" int rqb200_dbg_rows_gemm(const void* X16, const void* W16, const float* bias, const float* residual, float* out_f32,
                                    void* out_16, int gelu, int fmt, int64_t M, int N_out, int K, void* stream) {
    return rqb::launch_rows_gemm_tc(X16, W16, bias, residual, out_f32, out_16, gelu, fmt, M, N_out, K, (cudaStream_t)stream);
}
