// Row-wise log-softmax gather: log p = l[t] - logsumexp(l[0..V)) for fp32 logit rows, the reduction behind rqb200_ar_log_prob.
// One CTA per row reads the row once (16-byte loads when the row allows them), keeps an online (max, sum of exp) pair per thread in
// fp32 and combines the 256 pairs in a fixed order, so a row's result depends on that row alone -- not on the rows launched with it,
// the batch or the chunk -- and is the same from run to run.
#include <math.h>

#include <algorithm>

#include "kernels.h"

namespace rqb {

constexpr int LP_THREADS = 256;

// (m, s) <- the pair of the union of (m, s) and (m2, s2); m = -inf marks an empty pair
__device__ __forceinline__ void lse_merge(float& m, float& s, float m2, float s2) {
    const float M = fmaxf(m, m2);
    if (M == -INFINITY) return;
    s = s * expf(m - M) + s2 * expf(m2 - M);
    m = M;
}

__device__ __forceinline__ void lse_add4(float& m, float& s, float4 v) {
    const float mx = fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w));
    if (mx == -INFINITY) return;
    if (mx > m) {
        s *= expf(m - mx);
        m = mx;
    }
    s += (expf(v.x - m) + expf(v.y - m)) + (expf(v.z - m) + expf(v.w - m));
}

__device__ __forceinline__ void lse_add1(float& m, float& s, float x) {
    if (x == -INFINITY) return;
    if (x > m) {
        s = s * expf(m - x) + 1.f;
        m = x;
    } else {
        s += expf(x - m);
    }
}

// row r: logits lg + r*ld (V valid columns), target tgt[r*tgt_stride], result out[r].  vec: lg and ld allow 16-byte loads.
__global__ void __launch_bounds__(LP_THREADS) logprob_rows_kernel(const float* __restrict__ lg, int64_t ld, int V,
                                                                   const int64_t* __restrict__ tgt, int64_t tgt_stride,
                                                                   float* __restrict__ out, int vec) {
    __shared__ float sm[LP_THREADS / 32], ss[LP_THREADS / 32];
    const int64_t row = blockIdx.x;
    const float* x = lg + row * ld;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    float m = -INFINITY, s = 0.f;
    int tail = 0;
    if (vec) {
        const float4* x4 = reinterpret_cast<const float4*>(x);
        const int n4 = V >> 2;
        for (int i = tid; i < n4; i += LP_THREADS) lse_add4(m, s, __ldcs(x4 + i));
        tail = n4 << 2;
    }
    for (int i = tail + tid; i < V; i += LP_THREADS) lse_add1(m, s, __ldcs(x + i));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
        lse_merge(m, s, m2, s2);
    }
    if (lane == 0) { sm[warp] = m; ss[warp] = s; }
    __syncthreads();
    if (tid == 0) {
        float M = sm[0], S = ss[0];
        for (int w = 1; w < LP_THREADS / 32; w++) lse_merge(M, S, sm[w], ss[w]);
        const int64_t t = tgt[row * tgt_stride];
        out[row] = (t >= 0 && t < V) ? x[t] - (M + logf(S)) : __int_as_float(0x7fc00000);
    }
}

int launch_logprob_rows(const float* lg, int64_t ld, int V, int64_t rows, const int64_t* tgt, int64_t tgt_stride, float* out,
                        cudaStream_t st) {
    if (rows <= 0) return 0;
    if (V < 1 || ld < V || rows > 0x7fffffff) return fail(RQB200_EINVAL, "log_prob_rows: need 1 <= V <= ld and rows < 2^31");
    const int vec = (reinterpret_cast<uintptr_t>(lg) & 15) == 0 && ld % 4 == 0;
    logprob_rows_kernel<<<(unsigned)rows, LP_THREADS, 0, st>>>(lg, ld, V, tgt, tgt_stride, out, vec);
    return check_launch("logprob_rows_kernel");
}

// dst[(a*A2 + c)*G + g] = src[off + a*sa + c*sc + g*sg]: the targets of a token-major logits layout gathered from a code map
__global__ void gather_targets_kernel(const int64_t* __restrict__ src, int A2, int G, int64_t sa, int64_t sc, int64_t sg, int64_t off,
                                      int64_t n, int64_t* __restrict__ dst) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t g = i % G, ac = i / G, c = ac % A2, a = ac / A2;
        dst[i] = src[off + a * sa + c * sc + g * sg];
    }
}

int launch_gather_targets(const int64_t* src, int A1, int A2, int G, int64_t sa, int64_t sc, int64_t sg, int64_t off, int64_t* dst,
                          cudaStream_t st) {
    const int64_t n = (int64_t)A1 * A2 * G;
    if (n <= 0) return 0;
    gather_targets_kernel<<<(unsigned)std::min<int64_t>(ceil_div(n, 256), 4096), 256, 0, st>>>(src, A2, G, sa, sc, sg, off, n, dst);
    return check_launch("gather_targets_kernel");
}

}  // namespace rqb

extern "C" int rqb200_dbg_log_prob_rows(const float* logits, int64_t ld, int V, int64_t rows, const int64_t* targets, float* out,
                                        void* stream) {
    if (!logits || !targets || !out) return rqb::fail(RQB200_EINVAL, "dbg_log_prob_rows: null argument");
    if (rqb200_device_count() <= 0) return rqb::fail(RQB200_ENODEV, "dbg_log_prob_rows: no CUDA device");
    return rqb::launch_logprob_rows(logits, ld, V, rows, targets, 1, out, (cudaStream_t)stream);
}
