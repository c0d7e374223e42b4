// Diagnostic micro-benchmark (not on any product path): how fast does ONE SM pull L2-resident data into shared memory?
//
// The stage trace of the cached AR step (RQB200_TRACE=1) shows a GEMM's "dependency resolved -> accumulator ready" time growing
// with the activation boxes it loads (64 rows x 128 B, SWIZZLE_128B tensor-map load).  This kernel measures the candidates for
// that load on all SMs at once:
//   mode 0  cp.async.bulk.tensor.2d boxes of `rows` x 128 B out of a row-major [rows_total, row_bytes] tensor (what gemm_tc does)
//   mode 1  cp.async.bulk (1-D) copies of rows*128 contiguous bytes (what a pre-swizzled, tile-major operand would allow)
// Every CTA issues `depth` loads back to back into distinct shared-memory slots, waits for all of them, and repeats `iters` times.
// Result: bytes per clock per SM (clock64 around the loop of CTA 0) and the wall time.
#include "kernels.h"
#include "tc_common.cuh"

namespace rqb {

__global__ void __launch_bounds__(128)
dbg_tma_kernel(const __grid_constant__ CUtensorMap tm, const char* __restrict__ src, int mode, int rows, int depth, int iters,
               int boxes_total, long long* out_cycles) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    __shared__ uint64_t bar;
    const int box_bytes = rows * 128;
    if (threadIdx.x == 0) {
        tc::prefetch_tmap(&tm);
        tc::mbar_init(&bar, 1);
        tc::fence_barrier_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const long long t0 = clock64();
        uint32_t phase = 0;
        for (int it = 0; it < iters; it++) {
            tc::mbar_expect_tx(&bar, (uint32_t)(depth * box_bytes));
            for (int d = 0; d < depth; d++) {
                // every CTA walks the same small set of boxes (like the split-K CTAs of one GEMM reading the same activations)
                const int box = (it * depth + d) % boxes_total;
                if (mode == 0) {
                    tc::tma_load_2d(smem + d * box_bytes, &tm, &bar, (box % 8) * 64, (box / 8) * rows, tc::L2_EVICT_LAST);
                } else {
                    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                                 ::"r"(tc::smem_u32(smem + d * box_bytes)), "l"(src + (size_t)box * box_bytes), "r"(box_bytes),
                                 "r"(tc::smem_u32(&bar)) : "memory");
                }
            }
            tc::mbar_wait(&bar, phase);
            phase ^= 1;
        }
        if (blockIdx.x == 0) out_cycles[0] = clock64() - t0;
    }
}

}  // namespace rqb

// buffer: >= boxes_total * rows * 128 bytes of device memory (16-bit elements, row-major [boxes_total/8 * rows, 512] for mode 0).
// Returns bytes per clock per SM in *bytes_per_clk and microseconds per iteration in *us_per_iter.
extern "C" int rqb200_dbg_tma_rate(int mode, int rows, int depth, int iters, int boxes_total, const void* buffer, int ctas,
                                   float* bytes_per_clk, float* us_per_iter) {
    using namespace rqb;
    if (rows < 8 || rows > 256 || depth < 1 || depth * rows * 128 > 200 * 1024 || iters < 1 || boxes_total < 8 || boxes_total % 8)
        return fail(RQB200_EINVAL, "dbg_tma_rate: bad arguments");
    CUtensorMap tm;
    // mode 0 view: [boxes_total/8 * rows] rows of 512 elements (1 KB); a box = 64 elements (128 B) x `rows` rows
    RQB_TRY(make_tmap_2d(&tm, buffer, 1, 512, (uint64_t)(boxes_total / 8) * rows, 1024, 64, (uint32_t)rows));
    const size_t smem = (size_t)depth * rows * 128 + 1024;
    RQB_ENSURE_SMEM(201 * 1024, dbg_tma_kernel);
    long long* cyc = nullptr;
    RQB_CUDA(cudaMalloc(&cyc, sizeof(long long)));
    cudaStream_t st;
    RQB_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    cudaEvent_t e0, e1;
    RQB_CUDA(cudaEventCreate(&e0));
    RQB_CUDA(cudaEventCreate(&e1));
    dbg_tma_kernel<<<ctas, 128, smem, st>>>(tm, (const char*)buffer, mode, rows, depth, iters, boxes_total, cyc);   // warm-up (L2 fill)
    RQB_CUDA(cudaEventRecord(e0, st));
    dbg_tma_kernel<<<ctas, 128, smem, st>>>(tm, (const char*)buffer, mode, rows, depth, iters, boxes_total, cyc);
    RQB_CUDA(cudaEventRecord(e1, st));
    RQB_CUDA(cudaStreamSynchronize(st));
    RQB_CUDA(cudaGetLastError());
    float ms = 0.f;
    RQB_CUDA(cudaEventElapsedTime(&ms, e0, e1));
    long long h = 0;
    RQB_CUDA(cudaMemcpy(&h, cyc, sizeof(h), cudaMemcpyDeviceToHost));
    cudaFree(cyc);
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    cudaStreamDestroy(st);
    if (bytes_per_clk) *bytes_per_clk = (float)((double)iters * depth * rows * 128 / (double)(h > 0 ? h : 1));
    if (us_per_iter) *us_per_iter = ms * 1000.f / (float)iters;
    return 0;
}
