// P3 epilogue -- sample_from_logits as ONE kernel per token, no host sync.
//
// Replaces (reference, rqvae/utils/utils.py): top_k_logits :60-64 (torch.topk + threshold mask, ties >= k-th value
// kept), the NaN check :103-105 (a device->host sync per token in the reference), F.softmax :108, top_p_probs :67-79
// (torch.sort + cumsum + shifted `>=` mask + scatter + renormalise) and torch.multinomial :114, which for one draw is
// argmax(probs / q), q ~ Exp(1) (aten: multinomial_with_replacement is NOT taken for n_sample == 1) -- the caller
// passes the identical q tensor, so the draw is RNG-stream identical to the reference.
//
// One CTA (1024 threads) per row; the row (V <= 16384 fp32) is staged once in shared memory.
//   1. x = logit / T                                  (true division, like `logits / temperature`)
//   2. k-th largest by 4-pass 8-bit radix select on order-preserving uint keys (exact value, no sort) ; x < kth -> -inf
//   3. NaN -> -inf ; softmax: m = max, e = exp(x - m), s = sum e, p = e / s
//   4. top-p (only when p < 1; for p >= 1 the reference's branch removes nothing but a tail of total mass < 2^-24,
//      see DESIGN.md "sampler short-circuit"): compact the survivors, bitonic sort descending (ties: lower index
//      first), inclusive prefix sum accumulated in fp64 and rounded to fp32 per element (ATen's CPU cumsum uses a
//      double accumulator for float), cut after the first position whose cumulative mass >= p, renormalise by the
//      kept mass.
//   5. out = argmax_i p_i / q_i, first index on ties.
//
// Masked sampling (keep != NULL, same addressing as force): a CTA whose row keeps its token returns without writing; that takes
// precedence over teacher forcing.
//
// Classifier-free guidance (cfg_n > 0): the logits hold 2n rows, conditional rows [0, n) then unconditional rows [n, 2n).  CTA r < n
// reads rows r and r + n in step 1 and samples l = u + s (c - u), formed in fp32 as three rounded operations (no FMA contraction,
// so torch's `u + s * (c - u)` gives the same bits), with noise row r; it writes the code to rows r and r + n of the output.  CTAs
// r >= n (the fast tier's captured grid covers all 2n rows) leave at once.  Teacher forcing still copies every row's own code.
#include <cstdlib>

#include "kernels.h"
#include "tc_common.cuh"

namespace rqb {

constexpr int SMP_THREADS = 1024;
constexpr int SMP_MAXV = 16384;
constexpr int SMP_NB = 2048;       // buckets of the linear-map select
constexpr int SMP_MAXC = 1024;     // candidates of the threshold bucket that are ranked exactly; more -> radix select

__device__ __forceinline__ uint32_t f2key(float f) {   // monotone: larger float -> larger key
    uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key2f(uint32_t k) {
    uint32_t u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
    return __uint_as_float(u);
}

struct SortItem {
    float p;
    int idx;
};
__device__ __forceinline__ bool item_before(const SortItem& a, const SortItem& b) {   // descending p, then ascending idx
    return (a.p > b.p) || (a.p == b.p && a.idx < b.idx);
}

// CV (the fast tier's canvas graphs): the token's code lives at the canvas position of stt->idx (stt->cv, kernels.h)
template <bool CV>
__global__ void __launch_bounds__(SMP_THREADS, 1)
sample_kernel(const float* __restrict__ logits, const float* __restrict__ qnoise, int V, float temperature, int top_k,
              float top_p, int64_t* __restrict__ out_idx, const int64_t* __restrict__ force, int64_t out_stride,
              const StepState* __restrict__ stt, int dyn_d, int dyn_HW, int dyn_D, int algo, int cfg_n, float cfg_s,
              const uint8_t* __restrict__ keep) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* xs = reinterpret_cast<float*>(smem_raw);                       // [V]   scaled logits, later probabilities
    SortItem* items = reinterpret_cast<SortItem*>(xs + V);                // [Vpad] only touched when top_p < 1
    __shared__ unsigned int hist[256];
    __shared__ float red[33];
    __shared__ int redi[33];
    __shared__ unsigned int sel_prefix, sel_remaining, n_surv;
    __shared__ unsigned int bk_hist[SMP_NB];                // bucket select (algo 1)
    __shared__ float bk_cand[SMP_MAXC];
    __shared__ unsigned int bk_ncand, bk_bin, bk_rem, bk_fallback;
    __shared__ float bk_kth;
    __shared__ double scan_carry[33];
    __shared__ int cut_pos;
    __shared__ float kept_mass;
    __shared__ int guided_n;                                // cfg_n for step 5's write (kept out of registers through 2-4)

    const int row = blockIdx.x, t = threadIdx.x, lane = t & 31, wid = t >> 5;
    const float* lg = logits + (int64_t)row * V;
    tc::pdl_launch_dependents();
    // guided fast tier: an unconditional row's CTA has nothing to do.  (cfg_n and force are written by init_state_kernel before the
    // graph launch, not by a kernel of the chain, so they may be read before the dependency wait.)
    if (stt != nullptr && stt->cfg_n > 0 && row >= stt->cfg_n && stt->force == nullptr) return;
    tc::pdl_wait();
    if (stt != nullptr) {   // fast AR tier: per-token pointers and settings come from the device-resident StepState
        const int64_t off = (CV ? stt->cv.at(0, stt->idx) : (int64_t)stt->idx) * dyn_D + dyn_d;
        out_idx = stt->codes + off;
        force = stt->force ? stt->force + off : nullptr;
        out_stride = (int64_t)(CV ? stt->cv.chw : dyn_HW) * dyn_D;
        qnoise = stt->noise ? stt->noise + (int64_t)(stt->step + dyn_d) * stt->noise_stride : nullptr;
        temperature = stt->temperature;
        top_k = stt->top_k[dyn_d];
        top_p = stt->top_p[dyn_d];
        cfg_n = stt->cfg_n;
        cfg_s = stt->cfg_scale;
        keep = stt->keep ? stt->keep + off : nullptr;
    }
    // a kept token: `out` was initialised with its code (in both branch rows when guided).  The mask is constant during the call, but
    // the fast tier's position stt->idx is advanced by launches of the chain, so the fast tier reads it only after the dependency wait.
    if (keep != nullptr && keep[(int64_t)row * out_stride]) return;

    if (force != nullptr) {   // teacher forcing: emit the forced code, skip the work
        if (t == 0) out_idx[(int64_t)row * out_stride] = force[(int64_t)row * out_stride];
        return;
    }

    if (t == 0) guided_n = cfg_n;
    if (cfg_n > 0) {
        const float* lu = lg + (int64_t)cfg_n * V;
        for (int i = t; i < V; i += SMP_THREADS) {
            const float c = lg[i], u = lu[i];
            xs[i] = __fadd_rn(u, __fmul_rn(cfg_s, __fsub_rn(c, u))) / temperature;
        }
    } else {
        for (int i = t; i < V; i += SMP_THREADS) xs[i] = lg[i] / temperature;
    }
    __syncthreads();

    // ---- 2. top-k threshold: exact k-th largest by an 8-pass, 4-bit radix select.  No shared-memory atomics and no
    // MATCH: every thread keeps its <= 16 order-preserving keys in registers, counts the 16 digit values in packed
    // 16-bit lanes (8 words), the warp reduces them with shuffles, one word per thread sums the 32 warps.
    bool kth_done = false;
    if (algo == 1 && top_k > 0 && top_k < V) {
        // ---- 2'. bucket select: the k-th largest VALUE through one 2048-bucket histogram over the row's
        // [min, max] range (a monotone linear map, so bucket order == value order), a suffix scan to find the bucket that holds
        // it, and an exact ranking of that bucket's few members.  Rows with non-finite entries, a degenerate range or an
        // overfull threshold bucket take the radix select below.  Same threshold value => identical masking.
        float vals[16];
        float lo = INFINITY, hi = -INFINITY;
        bool bad = false;
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const int i = t + j * SMP_THREADS;
            vals[j] = 0.f;
            if (i < V) {
                const float v = xs[i];
                vals[j] = v;
                bad |= !(fabsf(v) <= 3.0e38f);               // NaN or +-inf
                lo = fminf(lo, v);
                hi = fmaxf(hi, v);
            }
        }
        for (int i = t; i < SMP_NB; i += SMP_THREADS) bk_hist[i] = 0u;
        if (t == 0) { bk_ncand = 0u; bk_fallback = 0u; bk_bin = 0u; bk_rem = 0u; }
        const float gmax = block_max(hi, red);
        const float gmin = -block_max(-lo, red);
        const int anybad = __syncthreads_or(bad ? 1 : 0);
        if (!anybad && gmax > gmin) {                          // block-uniform
            const float scale = (float)SMP_NB / (gmax - gmin);
            int bins[16];
#pragma unroll
            for (int j = 0; j < 16; j++) {
                const int i = t + j * SMP_THREADS;
                int b = (int)((vals[j] - gmin) * scale);
                b = b < 0 ? 0 : (b > SMP_NB - 1 ? SMP_NB - 1 : b);
                bins[j] = b;
                if (i < V) atomicAdd(&bk_hist[b], 1u);
            }
            __syncthreads();
            // suffix scan: thread t owns buckets 2t (low) and 2t+1 (high); `above` = members of all buckets above 2t+1
            const unsigned h0 = bk_hist[2 * t], h1 = bk_hist[2 * t + 1];
            unsigned incl = h0 + h1;                           // inclusive suffix sum over lanes >= lane
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned dn = __shfl_down_sync(0xffffffffu, incl, o);
                if (lane + o < 32) incl += dn;
            }
            unsigned* wtot = reinterpret_cast<unsigned*>(redi);
            if (lane == 0) wtot[wid] = incl;                   // this warp's total
            __syncthreads();
            unsigned wabove = 0u;                              // members held by warps above this one
            for (int w = wid + 1; w < SMP_THREADS / 32; w++) wabove += wtot[w];
            const unsigned above = wabove + incl - (h0 + h1);
            const unsigned k_u = (unsigned)top_k;
            if (above < k_u && k_u <= above + h1) { bk_bin = 2u * t + 1u; bk_rem = k_u - above; if (h1 > SMP_MAXC) bk_fallback = 1u; }
            else if (above + h1 < k_u && k_u <= above + h1 + h0) { bk_bin = 2u * t; bk_rem = k_u - above - h1; if (h0 > SMP_MAXC) bk_fallback = 1u; }
            __syncthreads();
            if (!bk_fallback) {                                // block-uniform (written before the barrier)
                const int bstar = (int)bk_bin;
#pragma unroll
                for (int j = 0; j < 16; j++) {
                    const int i = t + j * SMP_THREADS;
                    if (i < V && bins[j] == bstar) bk_cand[atomicAdd(&bk_ncand, 1u)] = vals[j];
                }
                __syncthreads();
                const int nc = (int)bk_ncand;
                const unsigned rem_u = bk_rem;
                if (t < nc) {
                    const float v = bk_cand[t];
                    unsigned gt = 0u, ge = 0u;
                    for (int i = 0; i < nc; i++) {
                        const float o2 = bk_cand[i];
                        gt += o2 > v ? 1u : 0u;
                        ge += o2 >= v ? 1u : 0u;
                    }
                    if (gt < rem_u && rem_u <= ge) bk_kth = v;   // every thread that qualifies holds the same value
                }
                __syncthreads();
                const float kth = bk_kth;
                for (int i = t; i < V; i += SMP_THREADS) {
                    float v = xs[i];
                    if (v < kth) xs[i] = -INFINITY;
                }
                __syncthreads();
                kth_done = true;
            }
        }
    }
    if (!kth_done && top_k > 0 && top_k < V) {
        uint32_t keys[16];
        uint32_t valid = 0;
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const int i = t + j * SMP_THREADS;
            keys[j] = 0u;
            if (i < V) { keys[j] = f2key(xs[i]); valid |= 1u << j; }
        }
        uint32_t* whist = reinterpret_cast<uint32_t*>(hist);           // [32 warps][8 packed words]
        uint32_t prefix = 0u, rem = (uint32_t)top_k;
#pragma unroll 1
        for (int pass = 7; pass >= 0; pass--) {
            const int shift = pass * 4;
            const uint32_t himask = (pass == 7) ? 0u : (0xffffffffu << (shift + 4));
            // 16 four-bit counters per 64-bit word; two words (keys 0-7 / 8-15) so that no counter can exceed 8
            unsigned long long acc0 = 0ull, acc1 = 0ull;
#pragma unroll
            for (int j = 0; j < 16; j++) {
                const bool hit = ((valid >> j) & 1u) && ((keys[j] & himask) == (prefix & himask));
                const unsigned long long inc = hit ? (1ull << (4u * ((keys[j] >> shift) & 15u))) : 0ull;
                if (j < 8) acc0 += inc; else acc1 += inc;
            }
            uint32_t cnt[8];
#pragma unroll
            for (int w = 0; w < 8; w++) {
                const uint32_t e = (uint32_t)((acc0 >> (8 * w)) & 0xffull), o2 = (uint32_t)((acc1 >> (8 * w)) & 0xffull);
                // byte w holds digits 2w (low nibble) and 2w+1 (high nibble)
                cnt[w] = ((e & 15u) + (o2 & 15u)) | (((e >> 4) + (o2 >> 4)) << 16);
            }
#pragma unroll
            for (int w = 0; w < 8; w++) {
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) cnt[w] += __shfl_xor_sync(0xffffffffu, cnt[w], o);   // <= 512 per half: no carry
            }
            if (lane == 0) {
#pragma unroll
                for (int w = 0; w < 8; w++) whist[wid * 8 + w] = cnt[w];
            }
            __syncthreads();
            if (wid == 0) {
                // lane l holds warp l's 8 packed words; butterfly-add across lanes (totals <= 16384 per 16-bit half: no carry)
                uint32_t tw[8];
#pragma unroll
                for (int w = 0; w < 8; w++) tw[w] = whist[lane * 8 + w];
#pragma unroll
                for (int w = 0; w < 8; w++) {
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) tw[w] += __shfl_xor_sync(0xffffffffu, tw[w], o);
                }
                // digit 2w -> low half of word w, digit 2w+1 -> high half; give lane l (< 8) word l as before
                uint32_t lo = 0u, hi = 0u;
#pragma unroll
                for (int w = 0; w < 8; w++)
                    if (lane == w) { lo = tw[w] & 0xffffu; hi = tw[w] >> 16; }
                // digit 2*lane -> lo, 2*lane+1 -> hi ; walk digits 15..0 accumulating from the top
                uint32_t acc = 0u, digit = 0u, newrem = rem;
                bool found = false;
#pragma unroll
                for (int dgt = 15; dgt >= 0; dgt--) {
                    const uint32_t c = __shfl_sync(0xffffffffu, (dgt & 1) ? hi : lo, dgt >> 1);
                    if (!found && acc + c >= rem) { digit = (uint32_t)dgt; newrem = rem - acc; found = true; }
                    if (!found) acc += c;
                }
                if (lane == 0) { sel_prefix = prefix | (digit << shift); sel_remaining = newrem; }
            }
            __syncthreads();
            prefix = sel_prefix;
            rem = sel_remaining;
        }
        const float kth = key2f(prefix);
        for (int i = t; i < V; i += SMP_THREADS) {
            float v = xs[i];
            if (v < kth) xs[i] = -INFINITY;            // out[out < v[:, [-1]]] = -inf  (utils.py:63)
        }
        __syncthreads();
    }

    // ---- 3. NaN -> -inf, softmax
    float m = -INFINITY;
    for (int i = t; i < V; i += SMP_THREADS) {
        float v = xs[i];
        if (v != v) { v = -INFINITY; xs[i] = v; }
        m = fmaxf(m, v);
    }
    m = block_max(m, red);
    float ssum = 0.f;
    for (int i = t; i < V; i += SMP_THREADS) {
        float e = expf(xs[i] - m);
        xs[i] = e;
        ssum += e;
    }
    ssum = block_sum(ssum, red);
    __syncthreads();
    for (int i = t; i < V; i += SMP_THREADS) xs[i] = xs[i] / ssum;
    __syncthreads();

    // ---- 4. top-p
    if (top_p < 1.0f) {
        if (t == 0) n_surv = 0u;
        __syncthreads();
        // compact survivors (p > 0); order is irrelevant, the sort fixes it
        for (int base = 0; base < V; base += SMP_THREADS) {
            int i = base + t;
            float p = (i < V) ? xs[i] : 0.f;
            bool alive = p > 0.f;
            unsigned bal = __ballot_sync(0xffffffffu, alive);
            unsigned wbase = 0;
            if (lane == 0 && bal) wbase = atomicAdd(&n_surv, (unsigned)__popc(bal));
            wbase = __shfl_sync(0xffffffffu, wbase, 0);
            if (alive) {
                int pos = wbase + __popc(bal & ((1u << lane) - 1u));
                items[pos].p = p;
                items[pos].idx = i;
            }
        }
        __syncthreads();
        const int ns = (int)n_surv;
        int npad = 1;
        while (npad < ns) npad <<= 1;
        for (int i = ns + t; i < npad; i += SMP_THREADS) { items[i].p = -1.f; items[i].idx = 0x7fffffff; }
        __syncthreads();
        for (int k = 2; k <= npad; k <<= 1) {
            for (int j = k >> 1; j > 0; j >>= 1) {
                for (int i = t; i < npad; i += SMP_THREADS) {
                    int ixj = i ^ j;
                    if (ixj > i) {
                        SortItem a = items[i], b = items[ixj];
                        bool up = ((i & k) == 0);               // "up" block: a must come before b
                        bool swap = up ? item_before(b, a) : item_before(a, b);
                        if (swap) { items[i] = b; items[ixj] = a; }
                    }
                }
                __syncthreads();
            }
        }
        // inclusive scan in fp64 (chunked: each thread owns a contiguous run), rounded to fp32 per element
        const int per = (ns + SMP_THREADS - 1) / SMP_THREADS;
        const int lo = min(t * per, ns), hi = min(lo + per, ns);
        double local = 0.0;
        for (int i = lo; i < hi; i++) local += (double)items[i].p;
        double incl = local;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            double up = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += up;
        }
        if (lane == 31) scan_carry[wid] = incl;
        __syncthreads();
        if (wid == 0) {
            double c = scan_carry[lane];
            double ci = c;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                double up = __shfl_up_sync(0xffffffffu, ci, o);
                if (lane >= o) ci += up;
            }
            scan_carry[lane] = ci - c;                           // exclusive warp offsets
        }
        if (t == 0) cut_pos = ns - 1;
        __syncthreads();
        double run = scan_carry[wid] + (incl - local);
        for (int i = lo; i < hi; i++) {
            run += (double)items[i].p;
            if ((float)run >= top_p) { atomicMin(&cut_pos, i); break; }   // first position with cum >= p is the last one kept
        }
        __syncthreads();
        const int cut = cut_pos;
        // kept mass: sum of the ORIGINAL-order probabilities that survive == torch.sum(probs) after masked_fill
        for (int i = cut + 1 + t; i < ns; i += SMP_THREADS) xs[items[i].idx] = 0.f;
        __syncthreads();
        float km = 0.f;
        for (int i = t; i < V; i += SMP_THREADS) km += xs[i];
        km = block_sum(km, red);
        if (t == 0) kept_mass = km;
        __syncthreads();
        const float kmv = kept_mass;
        for (int i = t; i < V; i += SMP_THREADS) xs[i] = xs[i] / kmv;
        __syncthreads();
    }

    // ---- 5. argmax p/q (first index on ties)
    float best = -INFINITY;
    int besti = 0x7fffffff;
    const float* qr = qnoise ? qnoise + (int64_t)row * V : nullptr;
    for (int i = t; i < V; i += SMP_THREADS) {
        float r = qr ? xs[i] / qr[i] : xs[i];
        if (r > best || (r == best && i < besti)) { best = r; besti = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        float ob = __shfl_xor_sync(0xffffffffu, best, o);
        int oi = __shfl_xor_sync(0xffffffffu, besti, o);
        if (ob > best || (ob == best && oi < besti)) { best = ob; besti = oi; }
    }
    if (lane == 0) { red[wid] = best; redi[wid] = besti; }
    __syncthreads();
    if (wid == 0) {
        best = red[lane];
        besti = redi[lane];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            float ob = __shfl_xor_sync(0xffffffffu, best, o);
            int oi = __shfl_xor_sync(0xffffffffu, besti, o);
            if (ob > best || (ob == best && oi < besti)) { best = ob; besti = oi; }
        }
        if (lane == 0) {
            const int code = (besti == 0x7fffffff) ? 0 : besti;
            out_idx[(int64_t)row * out_stride] = code;
            const int gn = guided_n;
            if (gn > 0) out_idx[(int64_t)(row + gn) * out_stride] = code;
        }
    }
}

// top-k threshold search: 0 = 8-pass radix select, 1 = bucket select (default: 24.7 vs 43.7 us per call at B = 64, V = 16384;
// identical indices -- tests/test_gpu_parity.py pins both to the reference's golden vectors)
constexpr int SAMPLER_ALGO_DEFAULT = 1;

// out_stride: distance (in int64 elements) between consecutive rows' outputs -- lets the AR loop write straight into
// codes[b, h, w, d] (stride H*W*D).  force (nullable) uses the same addressing.  cfg_n > 0: guided over B = 2 cfg_n rows, one CTA per
// image (one per row when teacher forcing).
int launch_sample(const float* logits, const float* q, int B, int V, float temperature, int top_k, float top_p,
                  int64_t* out_idx, const int64_t* force, int64_t out_stride, cudaStream_t st, int algo, int cfg_n, float cfg_s,
                  const uint8_t* keep) {
    if (B <= 0) return B == 0 ? 0 : fail(RQB200_EINVAL, "sample: B < 0");
    if (cfg_n < 0 || (cfg_n > 0 && B != 2 * cfg_n)) return fail(RQB200_EINVAL, "sample: a guided call takes B = 2 cfg_n rows");
    if (V <= 0 || V > SMP_MAXV) return fail(RQB200_EINVAL, "sample: V must be in [1,16384]");
    if (!(temperature > 0.f)) return fail(RQB200_EINVAL, "sample: temperature must be > 0");
    int vpad = 1;
    while (vpad < V) vpad <<= 1;
    size_t smem = (size_t)V * sizeof(float) + (top_p < 1.0f ? (size_t)vpad * sizeof(SortItem) : 0);
    RQB_ENSURE_SMEM(SMP_MAXV * 12, sample_kernel<false>);
    const int grid = (cfg_n > 0 && force == nullptr) ? cfg_n : B;
    sample_kernel<false><<<grid, SMP_THREADS, smem, st>>>(logits, q, V, temperature, top_k, top_p, out_idx, force, out_stride, nullptr, 0, 0,
                                                   0, algo, cfg_n, cfg_s, keep);
    return check_launch("sample_logits");
}

int launch_sample_dyn(const float* logits, const StepState* stt, int d, int B, int V, int HW, int D, cudaStream_t st, bool pdl,
                      bool canvas) {
    if (V <= 0 || V > SMP_MAXV) return fail(RQB200_EINVAL, "sample: V must be in [1,16384]");
    int vpad = 1;
    while (vpad < V) vpad <<= 1;
    size_t smem = (size_t)V * sizeof(float) + (size_t)vpad * sizeof(SortItem);   // top_p is only known on the device
    if (canvas) {
        RQB_ENSURE_SMEM(SMP_MAXV * 12, sample_kernel<true>);
        return launch_pdl(sample_kernel<true>, dim3(B), dim3(SMP_THREADS), smem, st, pdl, logits, (const float*)nullptr, V, 1.0f, 0, 1.0f,
                          (int64_t*)nullptr, (const int64_t*)nullptr, (int64_t)0, stt, d, HW, D, SAMPLER_ALGO_DEFAULT, 0, 0.0f,
                          (const uint8_t*)nullptr);
    }
    RQB_ENSURE_SMEM(SMP_MAXV * 12, sample_kernel<false>);
    return launch_pdl(sample_kernel<false>, dim3(B), dim3(SMP_THREADS), smem, st, pdl, logits, (const float*)nullptr, V, 1.0f, 0, 1.0f,
                      (int64_t*)nullptr, (const int64_t*)nullptr, (int64_t)0, stt, d, HW, D, SAMPLER_ALGO_DEFAULT, 0, 0.0f,
                      (const uint8_t*)nullptr);
}

}  // namespace rqb

extern "C" int rqb200_sample_logits(const float* logits, const float* q, int B, int V, float temperature, int top_k,
                                    float top_p, int64_t* out_idx, void* stream) {
    return rqb::launch_sample(logits, q, B, V, temperature, top_k, top_p, out_idx, nullptr, 1, (cudaStream_t)stream,
                              rqb::SAMPLER_ALGO_DEFAULT, 0, 0.f);
}
extern "C" int rqb200_dbg_sample_logits(int algo, const float* logits, const float* q, int B, int V, float temperature, int top_k,
                                        float top_p, int64_t* out_idx, void* stream) {
    return rqb::launch_sample(logits, q, B, V, temperature, top_k, top_p, out_idx, nullptr, 1, (cudaStream_t)stream, algo, 0, 0.f);
}
