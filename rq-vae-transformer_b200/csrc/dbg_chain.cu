// Diagnostic micro-benchmark (not on any product path): what does ONE dependent stage cost on this GPU?
//
// The cached AR step (csrc/ar_fast.cu) is a chain of ~530 dependent stages per spatial position; DESIGN.md section 8 shows it is
// bound by stage latency, not by HBM.  This file measures the floor of such a stage in the forms the engine could take:
//   mode 0  PDL chain of empty kernels inside a CUDA graph                       (launch + drain + griddepcontrol only)
//   mode 1  PDL chain, every CTA reads 16 KB written by ANOTHER CTA of the previous kernel and writes 16 KB (L2 round trip)
//   mode 2  one persistent kernel, the same data flow, stages separated by a grid-wide barrier (release/acquire counter)
//   mode 3  one persistent kernel, the same data flow, every CTA waits only for the epoch flags of the `fan` CTAs it reads from
//   mode 4  mode 1 with all of a thread's loads in flight before its first store (threads * 8 float4 >= 16 KB)
// Result: microseconds per stage.  tests/test_gpu_tc.py only checks that it runs.
#include "kernels.h"
#include "tc_common.cuh"

namespace rqb {

constexpr int CH_WORDS = 4096;          // floats per CTA per stage (16 KB)

__device__ __forceinline__ void chain_stage_work(const float* __restrict__ in, float* __restrict__ out, int src_cta, int fan, int ctas) {
    // read 16 KB spread over `fan` producer CTAs' chunks, add one, write this CTA's chunk
    const int per = CH_WORDS / 4 / fan;                  // float4 per producer
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int i = threadIdx.x; i < CH_WORDS / 4; i += blockDim.x) {
        const int pr = (src_cta + i / per) % ctas;
        const float4 v = __ldcg(reinterpret_cast<const float4*>(in + (size_t)pr * CH_WORDS) + i);
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        __stcg(reinterpret_cast<float4*>(out + (size_t)blockIdx.x * CH_WORDS) + i, make_float4(v.x + 1.f, v.y, v.z, v.w));
    }
    if (acc.x == -1.f) out[0] = acc.y;                    // keep the loads alive
}

// the same data flow with every load of a thread in flight before its first store (one round trip per stage instead of one per
// loop iteration): the floor of a well-formed stage
__device__ __forceinline__ void chain_stage_work_mlp(const float* __restrict__ in, float* __restrict__ out, int src_cta, int fan, int ctas) {
    const int per = CH_WORDS / 4 / fan;
    float4 v[8];
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const int i = threadIdx.x + k * blockDim.x;
        if (i < CH_WORDS / 4) {
            const int pr = (src_cta + i / per) % ctas;
            v[k] = __ldcg(reinterpret_cast<const float4*>(in + (size_t)pr * CH_WORDS) + i);
        }
    }
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const int i = threadIdx.x + k * blockDim.x;
        if (i < CH_WORDS / 4)
            __stcg(reinterpret_cast<float4*>(out + (size_t)blockIdx.x * CH_WORDS) + i, make_float4(v[k].x + 1.f, v[k].y, v[k].z, v[k].w));
    }
}

__global__ void chain_pdl_kernel(const float* in, float* out, int work, int fan) {
    // (dynamic shared memory is requested by the launch only to control how many CTAs fit on an SM; it is never touched)
    tc::pdl_launch_dependents();
    tc::pdl_wait();
    if (work == 1) chain_stage_work(in, out, (blockIdx.x * 7 + 1) % gridDim.x, fan, gridDim.x);
    else if (work == 4) chain_stage_work_mlp(in, out, (blockIdx.x * 7 + 1) % gridDim.x, fan, gridDim.x);
}

__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void red_release_add(unsigned* p, unsigned v) {
    asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void st_release(unsigned* p, unsigned v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// mode 2 / 3.  bar[0]: barrier counter (monotonic), flags[c]: last stage CTA c has published.  Mode 3 leaves the WAR hazard of
// the ping-pong buffers open on purpose (a fast CTA may overwrite a chunk a slow one still reads): only the timing matters here.
__global__ void chain_persistent_kernel(float* a, float* b, int n_stages, int fan, int use_flags, unsigned* bar, unsigned* flags) {
    const int ctas = gridDim.x;
    const int src = (blockIdx.x * 7 + 1) % ctas;
    for (int s = 0; s < n_stages; s++) {
        const float* in = (s & 1) ? b : a;
        float* out = (s & 1) ? a : b;
        if (s > 0) {
            if (use_flags) {
                // wait for the `fan` producers this CTA reads from (thread i < fan polls producer i)
                if (threadIdx.x < fan) {
                    const unsigned* f = flags + (src + threadIdx.x) % ctas;
                    while (ld_acquire(f) < (unsigned)s) {}
                }
            } else if (threadIdx.x == 0) {
                while (ld_acquire(bar) < (unsigned)(s * ctas)) {}
            }
            __syncthreads();
        }
        chain_stage_work(in, out, src, fan, ctas);
        __syncthreads();                                  // all of this CTA's stores issued ...
        if (threadIdx.x == 0) {
            __threadfence();                              // ... and ordered before the signal
            if (use_flags) st_release(flags + blockIdx.x, (unsigned)(s + 1));
            else red_release_add(bar, 1u);
        }
    }
}

// chain2: what part of a dependent stage is the READ of freshly written data, what part the WRITE + completion flush?
//   variant bit 0: every CTA reads `words` floats written by another CTA (all loads of a thread in flight, 16 x 16 B at a time)
//   variant bit 1: every CTA writes `words` floats (after its loads have all returned: the stores carry their sum)
//   variant bit 2: the reads go to a buffer nobody writes during the run (clean lines) instead of the previous stage's output
//   variant bit 3: (with bit 1) the writes are scattered line by line over the whole buffer: a consumer's region has many writers
__global__ void chain2_kernel(const float* __restrict__ in, float* __restrict__ out, int words, int variant) {
    tc::pdl_launch_dependents();
    tc::pdl_wait();
    const int n4 = words >> 2;
    const int src = (blockIdx.x * 7 + 1) % gridDim.x;
    float4 acc = make_float4(1.f, 0.f, 0.f, 0.f);
    if (variant & 1) {
        const float4* p = reinterpret_cast<const float4*>(in + (size_t)src * words);
        for (int i0 = 0; i0 < n4; i0 += 16 * blockDim.x) {
            float4 v[16];
#pragma unroll
            for (int k = 0; k < 16; k++) {
                const int i = i0 + threadIdx.x + k * blockDim.x;
                v[k] = i < n4 ? __ldcg(p + i) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int k = 0; k < 16; k++) { acc.x += v[k].x; acc.y += v[k].y; acc.z += v[k].z; acc.w += v[k].w; }
        }
    }
    if ((variant & 10) == 10) {
        // bit 3: scattered writes -- 128 B line l of this CTA goes to line (l * ctas + cta): every 16 KB region a consumer reads was
        // written by many different CTAs (the split-K partial planes / activation rows of the real chain)
        for (int i = threadIdx.x; i < n4; i += blockDim.x) {
            const size_t line = (size_t)(i >> 3) * gridDim.x + blockIdx.x;
            __stcg(reinterpret_cast<float4*>(out) + line * 8 + (i & 7), acc);
        }
    } else if (variant & 2) {
        float4* q = reinterpret_cast<float4*>(out + (size_t)blockIdx.x * words);
        for (int i = threadIdx.x; i < n4; i += blockDim.x) __stcg(q + i, acc);
    } else if (acc.x == -1.f) {
        out[0] = acc.y;
    }
}

}  // namespace rqb

extern "C" int rqb200_dbg_chain(int mode, int n_stages, int ctas, int threads, int smem_bytes, int fan, int reps, void* workspace,
                                size_t workspace_bytes, float* us_per_stage) {
    using namespace rqb;
    if (mode < 0 || mode > 4 || n_stages < 1 || ctas < 1 || threads < 32 || threads > 1024 || fan < 1 || fan > 32 || reps < 1 ||
        (CH_WORDS / 4) % fan != 0)
        return fail(RQB200_EINVAL, "dbg_chain: bad arguments");
    const size_t need = (size_t)2 * ctas * CH_WORDS * sizeof(float) + 4096 + (size_t)ctas * 4;
    if (workspace_bytes < need) return fail(RQB200_EINVAL, "dbg_chain: workspace too small");
    float* a = reinterpret_cast<float*>(workspace);
    float* b = a + (size_t)ctas * CH_WORDS;
    unsigned* bar = reinterpret_cast<unsigned*>(b + (size_t)ctas * CH_WORDS);
    unsigned* flags = bar + 1024;
    cudaStream_t st;
    RQB_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    RQB_CUDA(cudaMemsetAsync(workspace, 0, need, st));
    cudaEvent_t e0, e1;
    RQB_CUDA(cudaEventCreate(&e0));
    RQB_CUDA(cudaEventCreate(&e1));
    float ms = 0.f;
    if (mode <= 1 || mode == 4) {
        if (smem_bytes > 48 * 1024)
            RQB_CUDA(cudaFuncSetAttribute(chain_pdl_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
        cudaGraph_t g = nullptr;
        cudaGraphExec_t ge = nullptr;
        RQB_CUDA(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
        for (int s = 0; s < n_stages; s++) {
            cudaLaunchConfig_t cfg = {};
            cfg.gridDim = dim3((unsigned)ctas);
            cfg.blockDim = dim3((unsigned)threads);
            cfg.dynamicSmemBytes = (size_t)smem_bytes;
            cfg.stream = st;
            cudaLaunchAttribute at[1];
            at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
            at[0].val.programmaticStreamSerializationAllowed = 1;
            cfg.attrs = at;
            cfg.numAttrs = 1;
            cudaError_t e = cudaLaunchKernelEx(&cfg, chain_pdl_kernel, (const float*)((s & 1) ? b : a), (s & 1) ? a : b, mode, fan);
            if (e != cudaSuccess) {
                cudaStreamEndCapture(st, &g);
                return fail(RQB200_ECUDA, std::string("dbg_chain launch: ") + cudaGetErrorString(e));
            }
        }
        RQB_CUDA(cudaStreamEndCapture(st, &g));
        RQB_CUDA(cudaGraphInstantiate(&ge, g, 0));
        RQB_CUDA(cudaGraphLaunch(ge, st));                 // warm-up
        RQB_CUDA(cudaEventRecord(e0, st));
        for (int r = 0; r < reps; r++) RQB_CUDA(cudaGraphLaunch(ge, st));
        RQB_CUDA(cudaEventRecord(e1, st));
        RQB_CUDA(cudaStreamSynchronize(st));
        RQB_CUDA(cudaEventElapsedTime(&ms, e0, e1));
        cudaGraphExecDestroy(ge);
        cudaGraphDestroy(g);
    } else {
        int dev = 0, n_sm = 0, occ = 0;
        RQB_CUDA(cudaGetDevice(&dev));
        RQB_CUDA(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
        if (smem_bytes > 48 * 1024)
            RQB_CUDA(cudaFuncSetAttribute(chain_persistent_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
        RQB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, chain_persistent_kernel, threads, (size_t)smem_bytes));
        if ((int64_t)occ * n_sm < ctas) return fail(RQB200_EINVAL, "dbg_chain: persistent grid would not be co-resident");
        for (int r = 0; r < reps + 1; r++) {
            RQB_CUDA(cudaMemsetAsync(bar, 0, 4096 + (size_t)ctas * 4, st));
            if (r == 1) RQB_CUDA(cudaEventRecord(e0, st));
            chain_persistent_kernel<<<ctas, threads, (size_t)smem_bytes, st>>>(a, b, n_stages, fan, mode == 3 ? 1 : 0, bar, flags);
            RQB_CUDA(cudaGetLastError());
        }
        RQB_CUDA(cudaEventRecord(e1, st));
        RQB_CUDA(cudaStreamSynchronize(st));
        RQB_CUDA(cudaEventElapsedTime(&ms, e0, e1));
    }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    cudaStreamDestroy(st);
    if (us_per_stage) *us_per_stage = ms * 1000.f / ((float)n_stages * (float)reps);
    return 0;
}

extern "C" int rqb200_dbg_chain2(int variant, int words, int n_stages, int ctas, int threads, int smem_bytes, int reps, void* workspace,
                                 size_t workspace_bytes, float* us_per_stage) {
    using namespace rqb;
    if (variant < 0 || variant > 15 || words < 4 || (words & 3) || n_stages < 1 || ctas < 1 || threads < 32 || threads > 1024 || reps < 1)
        return fail(RQB200_EINVAL, "dbg_chain2: bad arguments");
    const size_t buf = (size_t)ctas * words * sizeof(float);
    if (workspace_bytes < 3 * buf) return fail(RQB200_EINVAL, "dbg_chain2: workspace too small");
    float* a = reinterpret_cast<float*>(workspace);
    float* b = a + (size_t)ctas * words;
    float* c = b + (size_t)ctas * words;
    cudaStream_t st;
    RQB_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    RQB_CUDA(cudaMemsetAsync(workspace, 0, 3 * buf, st));
    if (smem_bytes > 48 * 1024) RQB_CUDA(cudaFuncSetAttribute(chain2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
    cudaGraph_t g = nullptr;
    cudaGraphExec_t ge = nullptr;
    RQB_CUDA(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
    for (int s = 0; s < n_stages; s++) {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3((unsigned)ctas);
        cfg.blockDim = dim3((unsigned)threads);
        cfg.dynamicSmemBytes = (size_t)smem_bytes;
        cfg.stream = st;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        at[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = at;
        cfg.numAttrs = 1;
        const float* in = (variant & 4) ? c : ((s & 1) ? b : a);
        cudaError_t e = cudaLaunchKernelEx(&cfg, chain2_kernel, in, (s & 1) ? a : b, words, variant);
        if (e != cudaSuccess) {
            cudaStreamEndCapture(st, &g);
            return fail(RQB200_ECUDA, std::string("dbg_chain2 launch: ") + cudaGetErrorString(e));
        }
    }
    RQB_CUDA(cudaStreamEndCapture(st, &g));
    RQB_CUDA(cudaGraphInstantiate(&ge, g, 0));
    RQB_CUDA(cudaGraphLaunch(ge, st));
    cudaEvent_t e0, e1;
    RQB_CUDA(cudaEventCreate(&e0));
    RQB_CUDA(cudaEventCreate(&e1));
    RQB_CUDA(cudaEventRecord(e0, st));
    for (int r = 0; r < reps; r++) RQB_CUDA(cudaGraphLaunch(ge, st));
    RQB_CUDA(cudaEventRecord(e1, st));
    RQB_CUDA(cudaStreamSynchronize(st));
    float ms = 0.f;
    RQB_CUDA(cudaEventElapsedTime(&ms, e0, e1));
    cudaGraphExecDestroy(ge);
    cudaGraphDestroy(g);
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    cudaStreamDestroy(st);
    if (us_per_stage) *us_per_stage = ms * 1000.f / ((float)n_stages * (float)reps);
    return 0;
}
