// sm_90a primitives written as inline PTX: mbarrier, TMA (cp.async.bulk.tensor), wgmma (fence / commit / wait, shared-memory
// matrix descriptors; the mma_async wrappers themselves are in wgmma.cuh), PDL (griddepcontrol).  Bit layouts follow the PTX
// ISA wgmma matrix-descriptor table.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "wgmma.cuh"

namespace rqb {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "LAB_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE;\n"
        "bra LAB_WAIT;\n"
        "DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}

// ---------------------------------------------------------------- TMA
constexpr uint64_t L2_EVICT_NORMAL = 0x1000000000000000ull;
constexpr uint64_t L2_EVICT_FIRST = 0x12F0000000000000ull;
constexpr uint64_t L2_EVICT_LAST = 0x14F0000000000000ull;

__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, uint64_t hint) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5;"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(hint)
        : "memory");
}
// contiguous global -> shared copy through the TMA unit (bytes % 16 == 0, both ends 16 B aligned), completing on `bar`
__device__ __forceinline__ void bulk_load(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint64_t hint) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(smem_u32(bar)), "l"(hint)
        : "memory");
}
// L2-only prefetch of a contiguous global range (bytes % 16 == 0, 16 B aligned)
__device__ __forceinline__ void bulk_prefetch_l2(const void* p, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3,
                                            uint64_t hint) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4, %5, %6}], [%2], %7;"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "l"(hint)
        : "memory");
}

// nanosecond wall clock shared by all SMs (diagnostic stage traces)
__device__ __forceinline__ long long gtimer() {
    long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// ---------------------------------------------------------------- PDL
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ---------------------------------------------------------------- wgmma (warpgroup MMA)
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across an in-flight wgmma
template <int R>
__device__ __forceinline__ void acc_fence(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; i++) asm volatile("" : "+f"(d[i])::"memory");
}
// hand registers from one warpgroup to another (all warps of the warpgroup execute it; the kernel's budget must cover the total)
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
// named barrier over the `n` threads of the consumer warpgroups (id 0 is __syncthreads)
__device__ __forceinline__ void bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// K-major operand tile in shared memory, rows of 128 B (64 x 16-bit) written by TMA with SWIZZLE_128B, 8-row groups
// 1024 B apart: start_address[0,14) = addr>>4, LBO[16,30) unused for swizzled K-major, SBO[32,46) = 1024>>4,
// base_offset[49,52) = 0, layout_type[62,64) = 1 (SWIZZLE_128B).  Tile base must be 1024 B aligned; stepping along
// K inside the 128 B row = adding the byte offset to the start address (hardware applies the XOR swizzle).
// sbo != 1024: the 8-row groups are `sbo` bytes apart (a multiple of 128) -- conv3x3_tc_kernel reads one output row of a halo
// tile per group.  The XOR swizzle is a function of the absolute shared-memory address, as in the TMA write, so a group may
// start at any 128 B row of a 1024 B-aligned TMA box.
__device__ __forceinline__ uint64_t gmma_desc_k128(uint32_t smem_addr, uint32_t sbo = 1024) {
    uint64_t d = (uint64_t)((smem_addr >> 4) & 0x3FFFu);
    d |= (uint64_t)1 << 16;                    // LBO = 1 (ignored)
    d |= (uint64_t)((sbo >> 4) & 0x3FFFu) << 32;   // SBO
    d |= (uint64_t)1 << 62;                    // SWIZZLE_128B
    return d;
}

// Register accumulator of one consumer warpgroup (64 rows x N columns, wgmma D fragment) -> a row-major staging buffer in shared
// memory holding columns [c0, c0 + CW) of the 128-row tile (two warpgroups): stage[row * (CW + 4) + col - c0].  The epilogue then
// reads it back as "one thread <-> one row, 16 consecutive columns".
template <int N, int CW, int C0>
__device__ __forceinline__ void stage_acc(const float (&d)[N / 2], float* stage, int wg, int t) {
    constexpr int SP = CW + 4;
    const int w = (t >> 5) & 3, l = t & 31;
    const int row = wg * 64 + w * 16 + (l >> 2);
#pragma unroll
    for (int j = C0 / 8; j < (C0 + CW) / 8; j++) {
        const int col = 8 * j + 2 * (l & 3) - C0;
        *reinterpret_cast<float2*>(stage + row * SP + col) = make_float2(d[4 * j], d[4 * j + 1]);
        *reinterpret_cast<float2*>(stage + (row + 8) * SP + col) = make_float2(d[4 * j + 2], d[4 * j + 3]);
    }
}

// The epilogue of the two consumer warpgroups (256 threads, named barrier 1): accumulator columns [C0, N) in chunks of CW through the
// staging buffer.  Per chunk, consumer thread t passes tile row t % 128, columns [c, c + 16) with c = C0 + 16 (t / 128) < C0 + CW, to
// epi(v, row, c).
template <int N, int CW, int C0, typename Epi>
__device__ __forceinline__ void drain_acc(const float (&acc)[N / 2], float* stage, int wg, int t, const Epi& epi) {
    if constexpr (C0 < N) {
        stage_acc<N, CW, C0>(acc, stage, wg, t);
        bar_sync(1, 256);
        const int r = t & 127, h = t >> 7;
        if (h * 16 < CW) {
            float v[16];
            const float4* src = reinterpret_cast<const float4*>(stage + r * (CW + 4) + h * 16);
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const float4 x = src[i];
                v[4 * i] = x.x; v[4 * i + 1] = x.y; v[4 * i + 2] = x.z; v[4 * i + 3] = x.w;
            }
            epi(v, r, C0 + h * 16);
        }
        bar_sync(1, 256);
        drain_acc<N, CW, C0 + CW>(acc, stage, wg, t, epi);
    }
}

}  // namespace tc

// host: cuTensorMapEncodeTiled through the runtime's driver entry point (no link-time libcuda dependency)
int make_tmap_2d(CUtensorMap* out, const void* base, int elem_bytes_log2 /*1 = 16-bit*/, uint64_t inner, uint64_t outer,
                 uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_outer);
int make_tmap_4d_nhwc(CUtensorMap* out, const void* base, uint64_t C, uint64_t W, uint64_t H, uint64_t B, uint32_t box_c,
                      uint32_t box_w, uint32_t box_h, uint32_t box_b, uint32_t stride);

}  // namespace rqb
