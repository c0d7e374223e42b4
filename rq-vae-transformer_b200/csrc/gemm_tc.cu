// P3 "fast" tier workhorse -- weight-streaming skinny GEMM on wgmma tensor cores.
//
//   D[n, b] = sum_k W[n, k] * X[b, k]            W: [N_out, K] (nn.Linear layout), X: [B, K], both fp16 or both bf16
//                                                (GemmTcParams.fmt; the reference's amp class is fp16), or E4M3 W with row
//                                                scales and fp16 X (GtFormat<GT_E4M3>), D fp32 in registers
//
// Replaces every nn.Linear of the cached AR step (reference: attentions.py:69-71,99,117-122; transformers.py:94) at
// M = batch rows.  At B <= 256 these GEMMs are HBM-bound on the *weights* (SURVEY.md finding 5), so the kernel is laid
// out as a weight streamer with the operands SWAPPED: the weight tile is the wgmma "A" operand (M = 128 output features
// per CTA, 64 per consumer warpgroup, K-major -- exactly the [out,in] row-major layout checkpoints already have, no transpose), the activations are
// the "B" operand (N = batch padded to 16).  Two consumer warpgroups issue wgmma (m64nBNk16 each, fp32 register accumulators);
// weights and activations arrive through TMA (SWIZZLE_128B, 64-element K slabs) into a STAGES-deep mbarrier ring.
//
// Programmatic dependent launch: weight tiles do not depend on the previous kernel, so the producer warp fills the ring
// with weights BEFORE griddepcontrol.wait; only the activation loads, the epilogue's residual reads and all stores wait
// for the upstream kernel.  Back-to-back kernels of the per-token chain thereby keep HBM busy across kernel boundaries.
//
// Split-K (blockIdx.x = tile * splits + split) spreads the N_out/128 tiles of the narrow GEMMs (proj, fc2: 12 tiles at
// E = 1536) over all 132 SMs; partial tiles go to an fp32 workspace [split][B][N_out] and are summed in a FIXED order by
// the consumer kernel (ln_reduce / attn_fast / act_reduce) -> deterministic, no atomics.
//
// More activation rows than one wgmma N (256) -- batched prefill, teacher-forced forward -- run as gridDim.y row chunks of BN.
#include "kernels.h"
#include "tc_common.cuh"
#include <cudaTypedefs.h>
#include <cstdlib>

namespace rqb {

static int get_encode_fn(PFN_cuTensorMapEncodeTiled_v12000* fn) {
    static PFN_cuTensorMapEncodeTiled_v12000 cached = nullptr;
    if (!cached) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
        if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !p)
            return fail(RQB200_ECUDA, "cuTensorMapEncodeTiled entry point not available");
        cached = (PFN_cuTensorMapEncodeTiled_v12000)p;
    }
    *fn = cached;
    return 0;
}

int make_tmap_2d(CUtensorMap* out, const void* base, int elem_bytes_log2, uint64_t inner, uint64_t outer,
                 uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_outer) {
    PFN_cuTensorMapEncodeTiled_v12000 enc;
    RQB_TRY(get_encode_fn(&enc));
    cuuint64_t dims[2] = {inner, outer};
    cuuint64_t strides[1] = {row_stride_bytes};
    cuuint32_t box[2] = {box_inner, box_outer};
    cuuint32_t estr[2] = {1, 1};
    CUtensorMapDataType dt = elem_bytes_log2 == 1 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    CUresult r = enc(out, dt, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(RQB200_ECUDA, "cuTensorMapEncodeTiled(2d) failed: " + std::to_string((int)r));
    return 0;
}

// stride > 1: the box samples every `stride`-th pixel along W and H (a strided conv's input pixels for one filter tap): boxDim is
// the traversed extent, the unit loads boxDim / elementStride elements
int make_tmap_4d_nhwc(CUtensorMap* out, const void* base, uint64_t C, uint64_t W, uint64_t H, uint64_t B, uint32_t box_c,
                      uint32_t box_w, uint32_t box_h, uint32_t box_b, uint32_t stride) {
    PFN_cuTensorMapEncodeTiled_v12000 enc;
    RQB_TRY(get_encode_fn(&enc));
    cuuint64_t dims[4] = {C, W, H, B};
    cuuint64_t strides[3] = {C * 2, W * C * 2, H * W * C * 2};
    cuuint32_t box[4] = {box_c, box_w * stride, box_h * stride, box_b};
    cuuint32_t estr[4] = {1, stride, stride, 1};
    CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(RQB200_ECUDA, "cuTensorMapEncodeTiled(4d) failed: " + std::to_string((int)r));
    return 0;
}

constexpr int GT_THREADS = 288;             // warps 0-7: two consumer warpgroups (64 output features each), warp 8: TMA producer

// Epilogue of one thread for 16 accumulator columns [col0, col0 + 16) = activation rows m0 + col of output feature n.
template <int MODE, bool FULL>
__device__ __forceinline__ void gt_epilogue_cols(const GemmTcParams& p, const float* v, bool nvalid, float bias, const float* res,
                                                 int64_t res_ld, int rdiv, float* out_f, h16* out_h, int64_t ld, int m0, int nb,
                                                 int col0) {
    if (!nvalid) return;
#pragma unroll
    for (int i = 0; i < 16; i++) {
        const int col = col0 + i;                                    // activation row m0 + col
        if (FULL || col < nb) {
            float x = v[i];
            if (MODE != GT_PARTIAL) x += bias;
            if (MODE == GT_F32 && res != nullptr) x += res[(rdiv ? (int64_t)((m0 + col) / rdiv) : (int64_t)(m0 + col)) * res_ld];
            if (MODE == GT_PARTIAL || MODE == GT_F32) out_f[(int64_t)col * ld] = x;
            else if (MODE == GT_H16) out_h[(int64_t)col * ld] = pack_h16(x, p.fmt);
            else if (MODE == GT_H16_GELU) out_h[(int64_t)col * ld] = pack_h16(gelu_erf(x), p.fmt);
            else out_h[(int64_t)col * ld] = pack_h16(quick_gelu(x), p.fmt);
        }
    }
}

// Epilogue of one thread: output feature n, accumulator columns [col0, col0 + 16) staged in shared memory (v), for the activation rows
// m0 .. m0 + nb - 1.  The mode is a template parameter, row addresses are base + constant * stride, and the row bound is checked
// only for ragged chunks.
template <int MODE>
__device__ __forceinline__ void gt_epilogue(const GemmTcParams& p, const float* v, int n, int split, int m0, int nb, int col0) {
    const bool nvalid = n < p.N_out;
    const float bias = (MODE != GT_PARTIAL && p.bias != nullptr && nvalid) ? p.bias[n] * p.bias_scale : 0.f;
    const float* res = nullptr;
    int64_t res_ld = 0;
    if (MODE == GT_F32 && p.residual != nullptr && nvalid) {
        res = p.residual + (p.res_row_ptr ? (int64_t)(*p.res_row_ptr) * p.res_row_stride : 0) + n;
        res_ld = p.ld_res;
    }
    const int rdiv = p.res_div > 1 ? p.res_div : 0;                 // 0: residual row == activation row
    float* out_f = nullptr;
    h16* out_h = nullptr;
    int64_t ld = 0;
    if (MODE == GT_PARTIAL) {
        out_f = p.partial + ((int64_t)split * p.B + m0) * p.N_out + n;
        ld = p.N_out;
    } else if (MODE == GT_F32) {
        out_f = reinterpret_cast<float*>(p.out) + (int64_t)m0 * p.ld_out + n;
        ld = p.ld_out;
    } else {
        out_h = reinterpret_cast<h16*>(p.out) + (int64_t)m0 * p.ld_out + n;
        ld = p.ld_out;
    }
    if (col0 + 16 <= nb) gt_epilogue_cols<MODE, true>(p, v, nvalid, bias, res, res_ld, rdiv, out_f, out_h, ld, m0, nb, col0);
    else if (col0 < nb) gt_epilogue_cols<MODE, false>(p, v, nvalid, bias, res, res_ld, rdiv, out_f, out_h, ld, m0, nb, col0);
}

template <int BN, int FMT>
__device__ __forceinline__ void gt_mma_kblock(float (&acc)[BN / 2], uint32_t a, uint32_t b, bool first) {
#pragma unroll
    for (int j = 0; j < 4; j++)
        tc::Wgmma<BN, FMT>::mma(acc, tc::gmma_desc_k128(a + j * 32), tc::gmma_desc_k128(b + j * 32), (!first || j > 0) ? 1u : 0u);
}

// ---------------------------------------------------------------- weight formats
//
// What the weight format decides: the weight bytes of a ring stage, the ring depth, how the producer loads the weight tile of the
// i-th k block of a CTA's slice (row tile, k blocks from kb0) into a stage, how a consumer warpgroup multiplies one 64-k block, and
// the row scale applied before the epilogue.
enum GtWeightFormat { GT_W16 = 0, GT_E4M3 = 1 };
template <int WF>
struct GtFormat;

// 16-bit weights (fp16 or bf16, as the activations: p.fmt): a 128 x 64 tile through the tensor map, the wgmma's descriptor A operand.
template <>
struct GtFormat<GT_W16> {
    using Arg = CUtensorMap;
    static constexpr int A_BYTES = 128 * 64 * 2;
    // the deepest ring that fits (one CTA per SM, the whole K slice of a split prefetched ahead of the upstream kernel)
    __host__ __device__ static constexpr int stages(int bn) { return bn <= 64 ? 8 : bn == 128 ? 6 : 4; }
    struct Frag {};
    struct Scale {};
    struct Slice { const CUtensorMap* tm; int tile, kb0; };
    __device__ static void prefetch(const Arg& w) { tc::prefetch_tmap(&w); }
    __device__ static Slice slice(const Arg& w, int tile, int, int kb0) { return {&w, tile, kb0}; }
    __device__ static void load(const Slice& w, uint8_t* dst, uint64_t* bar, int i, uint64_t hint) {
        tc::tma_load_2d(dst, w.tm, bar, (w.kb0 + i) * 64, w.tile * 128, hint);
    }
    template <int BN>
    __device__ static void kblock(float (&acc)[BN / 2], Frag&, uint8_t* stage, int wg, int t, int fmt, bool first) {
        const uint32_t a = tc::smem_u32(stage) + wg * (64 * 128), b = tc::smem_u32(stage + A_BYTES);
        tc::wgmma_fence();
        if (fmt) gt_mma_kblock<BN, 1>(acc, a, b, first);
        else gt_mma_kblock<BN, 0>(acc, a, b, first);
    }
    __device__ static Scale row_scale(const Arg&, int, int, int, int) { return {}; }
    template <int R>
    __device__ static void scale(float (&)[R], Scale) {}
};

// FP8 (E4M3) weights, fp16 activations:
//
//   D[n, b] = s[n] * sum_k q[n, k] * X[b, k]       q: E4M3, one fp32 scale per output row; X fp16
//
// Half the weight bytes.  wgmma has no mixed e4m3 x f16 form, so the weight tile is the REGISTER A operand: every consumer thread
// loads its bytes from shared memory, widens them with cvt.rn.f16x2.e4m3x2 (exact: every E4M3 value is an fp16 value) and issues
// the register-A m64nBNk16 f16 wgmma against the activations' descriptor.
//
// Packed weights (rqvae._native.pack_fp8_tiles): tile (row block T, k block kb) is 8 KB at ((T * K/64) + kb) * 8192, laid out
// [warpgroup 2][half 2][thread 128][16 B]; the 16 bytes of (half h, thread t) are the A fragments of k16 steps 2h and 2h + 1,
// 8 bytes each, byte e = element e of the fragment (WgmmaRA: register e / 2, lower byte = lower half).  A thread's k block is
// two 16 B shared loads, consecutive threads on consecutive 16 B (conflict-free), and a tile arrives by one bulk copy.
// The scale multiplies the accumulator before the common epilogue (bias, residual, GELU, partial sums): x = s[n] acc + bias.
struct GtE4m3Tiles {
    const uint8_t* q;
    const float* s;
};

__device__ __forceinline__ uint32_t e4m3x2_to_f16x2(uint32_t v) {
    uint32_t r;
    asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(r) : "h"((unsigned short)v));
    return r;
}

__device__ __forceinline__ void lds128(uint32_t (&v)[4], uint32_t addr) {
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3]) : "r"(addr) : "memory");
}

template <>
struct GtFormat<GT_E4M3> {
    using Arg = GtE4m3Tiles;
    static constexpr int A_BYTES = 128 * 64;
    // the freed half of every stage deepens the ring
    __host__ __device__ static constexpr int stages(int bn) { return bn <= 32 ? 16 : bn == 64 ? 12 : 8; }
    // the A fragments of the four k16 steps of one k block
    using Frag = uint32_t[4][4];
    struct Scale { float lo, hi; };
    using Slice = const uint8_t*;
    __device__ static void prefetch(const Arg&) {}
    __device__ static Slice slice(const Arg& w, int tile, int nkb_total, int kb0) { return w.q + ((size_t)tile * nkb_total + kb0) * A_BYTES; }
    __device__ static void load(Slice w, uint8_t* dst, uint64_t* bar, int i, uint64_t hint) {
        tc::bulk_load(dst, w + (size_t)i * A_BYTES, A_BYTES, bar, hint);
    }
    // widen this thread's 32 weight bytes into the four k16 A fragments, then issue the four wgmmas.  `a` must not be the fragment
    // set of the (possibly still running) previous block.
    template <int BN>
    __device__ static void kblock(float (&acc)[BN / 2], Frag& a, uint8_t* stage, int wg, int t, int, bool first) {
        const uint32_t st0 = tc::smem_u32(stage), wt = st0 + wg * 4096 + (t & 127) * 16, b = st0 + A_BYTES;
        uint32_t lo[4], hi[4];
        lds128(lo, wt);
        lds128(hi, wt + 2048);
        const uint32_t w[8] = {lo[0], lo[1], lo[2], lo[3], hi[0], hi[1], hi[2], hi[3]};
#pragma unroll
        for (int kk = 0; kk < 4; kk++) {
            a[kk][0] = e4m3x2_to_f16x2(w[2 * kk]);
            a[kk][1] = e4m3x2_to_f16x2(w[2 * kk] >> 16);
            a[kk][2] = e4m3x2_to_f16x2(w[2 * kk + 1]);
            a[kk][3] = e4m3x2_to_f16x2(w[2 * kk + 1] >> 16);
        }
        tc::wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; kk++) tc::WgmmaRA<BN>::mma(acc, a[kk], tc::gmma_desc_k128(b + kk * 32), (!first || kk > 0) ? 1u : 0u);
    }
    // the scales of this thread's accumulator rows: d[4 j + i] is output feature frow + 8 (i / 2)
    __device__ static Scale row_scale(const Arg& w, int tile, int wg, int warp, int lane) {
        const int frow = tile * 128 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
        return {__ldg(w.s + frow), __ldg(w.s + frow + 8)};
    }
    template <int R>
    __device__ static void scale(float (&acc)[R], Scale s) {
#pragma unroll
        for (int j = 0; j < R / 4; j++) {
            acc[4 * j] *= s.lo; acc[4 * j + 1] *= s.lo;
            acc[4 * j + 2] *= s.hi; acc[4 * j + 3] *= s.hi;
        }
    }
};

// ---------------------------------------------------------------- the streamer
// QG: the 16-bit activation epilogue applies QuickGELU (GT_H16_QGELU) instead of the exact GELU; every other mode is the same code
template <int BN, int WF, bool QG = false>
__global__ void __launch_bounds__(GT_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ typename GtFormat<WF>::Arg W, const __grid_constant__ CUtensorMap tmX, GemmTcParams p) {
    using F = GtFormat<WF>;
    constexpr int STAGES = F::stages(BN);
    constexpr int B_BYTES = BN * 64 * 2;
    constexpr int STAGE_BYTES = F::A_BYTES + B_BYTES;
    constexpr int CW = BN < 32 ? BN : 32;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    float* stage = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES);          // [128][CW + 4] epilogue staging
    uint64_t* full = reinterpret_cast<uint64_t*>(stage + 128 * (CW + 4));
    uint64_t* xfull = full + STAGES;              // activations land on their own barrier (weights: full[])
    uint64_t* empty = xfull + STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tile = blockIdx.x / p.splits, split = blockIdx.x % p.splits;
    const int m0 = blockIdx.y * BN;                  // first activation row of this CTA's chunk
    const int nkb_total = p.K / 64;
    const int kb0 = (int)((int64_t)nkb_total * split / p.splits), kb1 = (int)((int64_t)nkb_total * (split + 1) / p.splits);
    const int nkb = kb1 - kb0;
    const bool tr = p.trace != nullptr && blockIdx.x == 0 && blockIdx.y == 0;

    tc::pdl_launch_dependents();             // let the next kernel of the chain start its own weight prefetch
    if (warp == 8 && lane == 0) {
        if (tr) p.trace[0] = tc::gtimer();
        F::prefetch(W);
        tc::prefetch_tmap(&tmX);
        // empty[s]: one arrival per consumer warp once its warpgroup's MMAs of that slot have completed
        for (int s = 0; s < STAGES; s++) { tc::mbar_init(&full[s], 1); tc::mbar_init(&xfull[s], 1); tc::mbar_init(&empty[s], 8); }
        tc::fence_barrier_init();
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            // ---- TMA producer.  Weights first (independent of the upstream kernel), then wait, then activations.
            const int pre = nkb < STAGES ? nkb : STAGES;
            const typename F::Slice wsl = F::slice(W, tile, nkb_total, kb0);
            // streamed once (M <= 256: evict first) or shared by every row chunk of a large-M launch (keep in L2)
            const uint64_t w_hint = gridDim.y > 1 ? tc::L2_EVICT_LAST : tc::L2_EVICT_FIRST;
            for (int i = 0; i < pre; i++) {
                tc::mbar_expect_tx(&full[i], F::A_BYTES);
                F::load(wsl, smem + i * STAGE_BYTES, &full[i], i, w_hint);
            }
            tc::pdl_wait();
            if (tr) p.trace[1] = tc::gtimer();
            for (int i = 0; i < pre; i++) {
                tc::mbar_expect_tx(&xfull[i], B_BYTES);
                tc::tma_load_2d(smem + i * STAGE_BYTES + F::A_BYTES, &tmX, &xfull[i], (kb0 + i) * 64, m0, tc::L2_EVICT_LAST);
            }
            for (int i = pre; i < nkb; i++) {
                const int s = i % STAGES;
                tc::mbar_wait(&empty[s], ((i / STAGES) & 1) ^ 1);
                tc::mbar_expect_tx(&full[s], F::A_BYTES);
                F::load(wsl, smem + s * STAGE_BYTES, &full[s], i, w_hint);
                tc::mbar_expect_tx(&xfull[s], B_BYTES);
                tc::tma_load_2d(smem + s * STAGE_BYTES + F::A_BYTES, &tmX, &xfull[s], (kb0 + i) * 64, m0, tc::L2_EVICT_LAST);
            }
        }
        return;
    }

    // ---- consumer warpgroups 0, 1: weight rows [64 wg, 64 wg + 64) of the tile x all BN activation columns, k in 16-wide steps.
    //      One k block stays in flight: the slot of block i - 1 is released once block i has been issued and i - 1 has completed.
    const int wg = warp >> 2, t = threadIdx.x;
    const typename F::Scale rs = F::row_scale(W, tile, wg, warp, lane);
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; i++) acc[i] = 0.f;
    auto kblock = [&](int i, typename F::Frag& a) {
        const int s = i % STAGES;
        tc::mbar_wait(&full[s], (i / STAGES) & 1);
        tc::mbar_wait(&xfull[s], (i / STAGES) & 1);
        F::template kblock<BN>(acc, a, smem + s * STAGE_BYTES, wg, t, p.fmt, i == 0);
        tc::wgmma_commit();
        tc::wgmma_wait<1>();
        if (i > 0 && lane == 0) tc::mbar_arrive(&empty[(i - 1) % STAGES]);
    };
    if constexpr (WF == GT_E4M3) {
        // register-A fragments: two sets alternate, so that the block in flight keeps its A registers
        typename F::Frag fa, fb;
        int i = 0;
        for (; i + 1 < nkb; i += 2) {
            kblock(i, fa);
            kblock(i + 1, fb);
        }
        if (i < nkb) kblock(i, fa);
    } else {
        // (the same step as kblock, written out: through the lambda, ptxas allocates the BN <= 32 kernels' registers differently)
        typename F::Frag none;
        for (int i = 0; i < nkb; i++) {
            const int s = i % STAGES;
            tc::mbar_wait(&full[s], (i / STAGES) & 1);
            tc::mbar_wait(&xfull[s], (i / STAGES) & 1);
            F::template kblock<BN>(acc, none, smem + s * STAGE_BYTES, wg, t, p.fmt, i == 0);
            tc::wgmma_commit();
            tc::wgmma_wait<1>();
            if (i > 0 && lane == 0) tc::mbar_arrive(&empty[(i - 1) % STAGES]);
        }
    }
    tc::wgmma_wait<0>();
    tc::acc_fence(acc);
    if (nkb > 0 && lane == 0) tc::mbar_arrive(&empty[(nkb - 1) % STAGES]);
    F::scale(acc, rs);

    tc::pdl_wait();
    if (tr && t == 0) p.trace[2] = tc::gtimer();
    const int nb = (p.B - m0) < BN ? (p.B - m0) : BN;          // valid activation rows of this chunk
    const int n_base = tile * 128;
    // (values captured by copy: captured by reference, the 16-bit kernels' SASS differs from the drain's former hand-written form)
    tc::drain_acc<BN, CW, 0>(acc, stage, wg, t, [&p, n_base, split, m0, nb](const float (&v)[16], int r, int col0) {
        const int n = n_base + r;
        switch (p.mode) {
            case GT_PARTIAL: gt_epilogue<GT_PARTIAL>(p, v, n, split, m0, nb, col0); break;
            case GT_F32: gt_epilogue<GT_F32>(p, v, n, split, m0, nb, col0); break;
            case GT_H16: gt_epilogue<GT_H16>(p, v, n, split, m0, nb, col0); break;
            default: gt_epilogue<QG ? GT_H16_QGELU : GT_H16_GELU>(p, v, n, split, m0, nb, col0); break;
        }
    });
    if (tr && t == 0) p.trace[3] = tc::gtimer();
}

template <int BN, int WF, bool QG = false>
static int launch_gemm_tc_t(const typename GtFormat<WF>::Arg& w, const CUtensorMap& tmX, const GemmTcParams& p, bool pdl,
                            cudaStream_t st) {
    using F = GtFormat<WF>;
    constexpr size_t smem = (size_t)F::stages(BN) * (F::A_BYTES + BN * 128) + 128 * ((BN < 32 ? BN : 32) + 4) * 4 + 1024 + 512;
    static_assert(smem <= 227 * 1024, "gemm_tc: shared memory budget");
    RQB_ENSURE_SMEM(smem, gemm_tc_kernel<BN, WF, QG>);
    return launch_pdl(gemm_tc_kernel<BN, WF, QG>, dim3((unsigned)(ceil_div(p.N_out, 128) * p.splits), (unsigned)ceil_div(p.B, BN)),
                      dim3(GT_THREADS), smem, st, pdl, w, tmX, p);
}

template <int WF>
static int launch_gemm_tc_bn(const typename GtFormat<WF>::Arg& w, const CUtensorMap& tmX, const GemmTcParams& p, int bn, bool pdl,
                             cudaStream_t st) {
    switch (bn) {
        case 16: return launch_gemm_tc_t<16, WF>(w, tmX, p, pdl, st);
        case 32: return launch_gemm_tc_t<32, WF>(w, tmX, p, pdl, st);
        case 64: return launch_gemm_tc_t<64, WF>(w, tmX, p, pdl, st);
        case 128: return launch_gemm_tc_t<128, WF>(w, tmX, p, pdl, st);
        default: return launch_gemm_tc_t<(WF == GT_E4M3 ? 128 : 256), WF>(w, tmX, p, pdl, st);      // (256 rows: 16-bit weights only)
    }
}

// GT_H16_QGELU (the CLIP engine's c_fc): 16-bit weights only
static int launch_gemm_tc_qgelu(const CUtensorMap& w, const CUtensorMap& tmX, const GemmTcParams& p, int bn, bool pdl, cudaStream_t st) {
    switch (bn) {
        case 16: return launch_gemm_tc_t<16, GT_W16, true>(w, tmX, p, pdl, st);
        case 32: return launch_gemm_tc_t<32, GT_W16, true>(w, tmX, p, pdl, st);
        case 64: return launch_gemm_tc_t<64, GT_W16, true>(w, tmX, p, pdl, st);
        case 128: return launch_gemm_tc_t<128, GT_W16, true>(w, tmX, p, pdl, st);
        default: return launch_gemm_tc_t<256, GT_W16, true>(w, tmX, p, pdl, st);
    }
}

int make_streamed_weight(StreamedWeight* out, bool e4m3, const void* w, const float* scale, int N_out, int K) {
    *out = StreamedWeight{};
    out->N_out = N_out;
    out->K = K;
    if (e4m3) {
        if (w == nullptr || scale == nullptr || (reinterpret_cast<uintptr_t>(w) & 15) != 0)
            return fail(RQB200_EINVAL, "gemm_tc: packed E4M3 weights must be 16-byte aligned, scales non-null");
        out->q8 = static_cast<const uint8_t*>(w);
        out->s8 = scale;
        return 0;
    }
    out->w16 = w;
    // row-major [N_out, K] 16-bit, box = 64 k x 128 rows
    return make_tmap_2d(&out->tm, w, 1, (uint64_t)K, (uint64_t)N_out, (uint64_t)K * 2, 64, 128);
}

int launch_gemm_tc(const StreamedWeight& w, const CUtensorMap& tmX, GemmTcParams p, bool pdl, cudaStream_t st) {
    p.N_out = w.N_out;
    p.K = w.K;
    if (p.K % 64 != 0 || p.N_out % 128 != 0) return fail(RQB200_EINVAL, "gemm_tc: need K % 64 == 0 and N_out % 128 == 0");
    if (p.B < 1) return fail(RQB200_EINVAL, "gemm_tc: no activation rows");
    if (p.splits < 1 || p.splits > p.K / 64) return fail(RQB200_EINVAL, "gemm_tc: bad split count");
    if (w.e4m3() && p.fmt != 0) return fail(RQB200_EINVAL, "gemm_tc: E4M3 weights take fp16 activations only");
    if (p.fmt != 0 && p.fmt != 1) return fail(RQB200_EINVAL, "gemm_tc: fmt must be 0 (fp16) or 1 (bf16)");
    if (p.B > 256 && p.mode == GT_PARTIAL) return fail(RQB200_EINVAL, "gemm_tc: split-K takes at most 256 activation rows");
    if (p.mode != GT_PARTIAL && p.splits != 1) return fail(RQB200_EINVAL, "gemm_tc: direct epilogues need splits == 1");
    const int bn = gemm_tc_chunk_rows(w, p.B);
    if (ceil_div(p.B, bn) > 65535) return fail(RQB200_EINVAL, "gemm_tc: more than 65535 row chunks");
    if (p.mode == GT_H16_QGELU) {
        if (w.e4m3()) return fail(RQB200_EINVAL, "gemm_tc: the QuickGELU epilogue takes 16-bit weights only");
        return launch_gemm_tc_qgelu(w.tm, tmX, p, bn, pdl, st);
    }
    if (w.e4m3()) return launch_gemm_tc_bn<GT_E4M3>(GtE4m3Tiles{w.q8, w.s8}, tmX, p, bn, pdl, st);
    return launch_gemm_tc_bn<GT_W16>(w.tm, tmX, p, bn, pdl, st);
}

}  // namespace rqb

// ---- diagnostic entry points (tests/test_gpu_tc.py, tests/test_gpu_fp8.py, tests/test_gpu_tc_kernels.py, bench.py's roofline leg): one
// GEMM through the streamer

// the GEMM over B activation rows X16 [B, K] fp16 / bf16 with the epilogue the arguments select
static int dbg_gemm_tc(const rqb::StreamedWeight& w, const void* X16, const float* bias, const float* residual, void* out, int out_is_16,
                       int gelu, float* partial, int B, int splits, int fmt, void* stream) {
    using namespace rqb;
    CUtensorMap tx;
    RQB_TRY(make_tmap_2d(&tx, X16, 1, (uint64_t)w.K, (uint64_t)B, (uint64_t)w.K * 2, 64, (uint32_t)gemm_tc_chunk_rows(w, B)));
    GemmTcParams p = {};
    p.B = B; p.splits = splits; p.fmt = fmt;
    p.bias = bias; p.bias_scale = 1.f; p.residual = residual; p.ld_res = w.N_out; p.out = out; p.ld_out = w.N_out; p.partial = partial;
    p.mode = (splits > 1 || partial != nullptr) ? GT_PARTIAL
                                                 : (out_is_16 ? (gelu == 2 ? GT_H16_QGELU : gelu ? GT_H16_GELU : GT_H16) : GT_F32);
    if (p.mode == GT_PARTIAL && partial == nullptr) return fail(RQB200_EINVAL, "dbg_gemm_tc: splits > 1 needs a partial buffer");
    return launch_gemm_tc(w, tx, p, false, (cudaStream_t)stream);
}

extern "C" int rqb200_dbg_gemm_tc(const void* W16, const void* X16, const float* bias, const float* residual, void* out,
                                  int out_is_16, int gelu, float* partial, int N_out, int K, int B, int splits, int fmt,
                                  void* stream) {
    rqb::StreamedWeight w;
    RQB_TRY(rqb::make_streamed_weight(&w, false, W16, nullptr, N_out, K));
    return dbg_gemm_tc(w, X16, bias, residual, out, out_is_16, gelu, partial, B, splits, fmt, stream);
}

extern "C" int rqb200_dbg_gemm_tc_fp8(const void* W8_packed, const float* scale, const void* X16, const float* bias,
                                      const float* residual, void* out, int out_is_16, int gelu, float* partial, int N_out, int K, int B,
                                      int splits, void* stream) {
    rqb::StreamedWeight w;
    RQB_TRY(rqb::make_streamed_weight(&w, true, W8_packed, scale, N_out, K));
    return dbg_gemm_tc(w, X16, bias, residual, out, out_is_16, gelu, partial, B, splits, 0, stream);
}

// the streamer with every epilogue option the AR engine uses (w_in's bias_scale and broadcast / indexed position rows, res_div of the
// batched w_in), through the same launcher as the engine's GEMMs
extern "C" int rqb200_dbg_gemm_tc_epi(const void* W, const float* scale, const void* X16, int mode, const float* bias, float bias_scale,
                                      const float* residual, int64_t ld_res, int res_div, const int* res_row_ptr, int64_t res_row_stride,
                                      void* out, float* partial, int N_out, int K, int B, int splits, int fmt, void* stream) {
    using namespace rqb;
    if (mode < GT_F32 || mode > GT_PARTIAL) return fail(RQB200_EINVAL, "dbg_gemm_tc_epi: mode must be 0..3");
    if ((mode == GT_PARTIAL) != (partial != nullptr)) return fail(RQB200_EINVAL, "dbg_gemm_tc_epi: a partial buffer exactly in mode 3");
    StreamedWeight w;
    RQB_TRY(make_streamed_weight(&w, scale != nullptr, W, scale, N_out, K));
    if (B < 1) return fail(RQB200_EINVAL, "gemm_tc: no activation rows");
    CUtensorMap tx;
    RQB_TRY(make_tmap_2d(&tx, X16, 1, (uint64_t)w.K, (uint64_t)B, (uint64_t)w.K * 2, 64, (uint32_t)gemm_tc_chunk_rows(w, B)));
    GemmTcParams p = {};
    p.B = B; p.splits = splits; p.mode = mode; p.fmt = fmt;
    p.bias = bias; p.bias_scale = bias_scale;
    p.residual = residual; p.ld_res = ld_res; p.res_div = res_div; p.res_row_ptr = res_row_ptr; p.res_row_stride = res_row_stride;
    p.out = out; p.ld_out = N_out; p.partial = partial;
    return launch_gemm_tc(w, tx, p, false, (cudaStream_t)stream);
}
