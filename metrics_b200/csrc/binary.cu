// K2 — binary / multilabel stat scores and confusion matrices: one pass over [n_outer, num_labels, inner] scores or
// labels producing (tp, fp, tn, fn) per group (label, or sample x label when `samplewise`).
//
// Reference op chains replaced (src/torchmetrics/functional/classification/):
//   stat_scores.py:95-134   _binary_stat_scores_format/_update      (sigmoid-if-logits, > threshold, 4 masked sums)
//   stat_scores.py:681-714  _multilabel_stat_scores_format/_update
//   confusion_matrix.py:119-152, :477-516  binary / multilabel confusion matrices ([[tn, fp], [fn, tp]] = same 4 counts)
// The reference runs ~12 elementwise + reduction launches per update; here: a batch-global range-flag kernel (only for
// floating scores) and ONE counting kernel.  Counters are privatised per thread (runs of equal group), then per CTA in
// shared memory, then added to the int64 outputs with 64-bit REDs.
#include <algorithm>
#include <cmath>

#include "common.cuh"

namespace mb200 {

template <typename T>
__device__ __forceinline__ bool out_of_unit_range(T x) {
    if constexpr (sizeof(T) == 8) {
        return (x < 0.0) | (x > 1.0);
    } else {
        const float v = to_f32(x);
        return (v < 0.f) | (v > 1.f);
    }
}
// batch-global "are these logits?" vote: 16-byte streaming loads over the aligned body, scalar head / tail
template <typename T>
__global__ void __launch_bounds__(256) bin_range_flag_kernel(const T* __restrict__ x, long long n, unsigned* flag) {
    bool bad = false;
    constexpr int kVec = 16 / (int)sizeof(T);
    long long head = (long long)(((16 - (reinterpret_cast<uintptr_t>(x) & 15)) & 15) / sizeof(T));
    if (head > n) head = n;
    const long long nvec = (n - head) / kVec;
    const uint4* __restrict__ xv = reinterpret_cast<const uint4*>(x + head);
    const long long gtid = (long long)blockIdx.x * blockDim.x + threadIdx.x, stride = (long long)gridDim.x * blockDim.x;
    for (long long i = gtid; i < nvec; i += stride) {
        const uint4 q = ld_stream16(xv + i);
        const T* e = reinterpret_cast<const T*>(&q);
#pragma unroll
        for (int k = 0; k < kVec; ++k) bad |= out_of_unit_range<T>(e[k]);
    }
    const long long tail0 = head + nvec * kVec;
    for (long long i = gtid; i < head + (n - tail0); i += stride) bad |= out_of_unit_range<T>(x[i < head ? i : tail0 + (i - head)]);
    if (__any_sync(kFull, bad) && (threadIdx.x & 31) == 0) atomicOr(flag, 1u);
}

struct BinArgs {
    const void* preds;
    const void* target;
    int preds_dtype;
    int target_dtype;
    long long n_outer;
    long long num_labels;
    long long inner;
    float threshold;  // rounded to the score dtype, as ATen rounds the reference's scalar (threshold_in_dtype)
    double threshold_d;
    int has_ignore;
    long long ignore_index;
    int samplewise;
    long long* counts;       // [G][4] tp, fp, tn, fn
    const unsigned* logits;  // batch flag written by bin_range_flag_kernel (NULL for integer preds)
    unsigned* err;
    int smem_groups;  // > 0: groups privatised in shared memory
};

// prediction as the integer the reference compares with the target
template <typename T>
__device__ __forceinline__ long long pred_label(const BinArgs& a, long long i, bool logits) {
    const T* __restrict__ p = reinterpret_cast<const T*>(a.preds);
    float v = to_f32(p[i]);
    if (logits) v = round_to<T>(1.0f / (1.0f + expf(-v)));  // ATen's sigmoid: fp32 math, result stored in T
    return v > a.threshold ? 1 : 0;
}
template <>
__device__ __forceinline__ long long pred_label<double>(const BinArgs& a, long long i, bool logits) {
    double v = reinterpret_cast<const double*>(a.preds)[i];
    if (logits) v = 1.0 / (1.0 + exp(-v));
    return v > a.threshold_d ? 1 : 0;
}
struct IntPred {};
template <>
__device__ __forceinline__ long long pred_label<IntPred>(const BinArgs& a, long long i, bool) {
    const long long p = load_label(a.preds, a.preds_dtype, i);
    if ((unsigned long long)p > 1ull && a.err) atomicOr(a.err, MB200_FLAG_PREDS_RANGE);
    return p;
}

__device__ __forceinline__ void flush_group(const BinArgs& a, long long group, unsigned (&c)[4], unsigned* sh) {
    if (group < 0) return;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        if (c[k] == 0) continue;
        if (sh) atomicAdd(&sh[group * 4 + k], c[k]);
        else red_add_u64(a.counts + group * 4 + k, c[k]);
        c[k] = 0;
    }
}

template <typename T>
__global__ void __launch_bounds__(256) bin_count_kernel(BinArgs a) {
    extern __shared__ unsigned sh_counts[];
    unsigned* sh = a.smem_groups > 0 ? sh_counts : nullptr;
    if (sh) {
        for (int i = threadIdx.x; i < a.smem_groups * 4; i += blockDim.x) sh[i] = 0;
        __syncthreads();
    }
    const bool logits = a.logits != nullptr && (*a.logits) != 0u;
    const long long per_outer = a.num_labels * a.inner;
    const long long total = a.n_outer * per_outer;
    // contiguous chunk per thread so that runs of equal group stay in registers
    const long long nthreads = (long long)gridDim.x * blockDim.x;
    const long long chunk = (total + nthreads - 1) / nthreads;
    const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    // warp-interleaved assignment keeps loads coalesced: thread handles i = base + k*32 + lane inside its warp's span
    const long long warp_id = tid >> 5;
    const int lane = threadIdx.x & 31;
    const long long span = chunk * 32;
    const long long begin = warp_id * span;
    const long long end = min(begin + span, total);
    long long cur = -1;
    unsigned c[4] = {0, 0, 0, 0};
    const bool small = total < (1ll << 31);
    const unsigned per_outer_u = (unsigned)per_outer, inner_u = (unsigned)a.inner;
    for (long long i = begin + lane; i < end; i += 32) {
        const long long t = load_label(a.target, a.target_dtype, i);
        if (a.has_ignore && t == a.ignore_index) continue;
        if ((unsigned long long)t > 1ull) {
            if (a.err) atomicOr(a.err, MB200_FLAG_TARGET_RANGE);
            continue;  // the reference counts such elements in none of the four masks
        }
        const long long p = pred_label<T>(a, i, logits);
        long long n, l;
        if (small) {  // 32-bit index arithmetic: a 64-bit division is ~4x the instructions, and there are two per element
            const unsigned iu = (unsigned)i;
            const unsigned nu = iu / per_outer_u;
            const unsigned rem = iu - nu * per_outer_u;
            n = nu;
            l = inner_u == 1u ? rem : rem / inner_u;
        } else {
            n = i / per_outer;
            l = (i - n * per_outer) / a.inner;
        }
        const long long group = a.samplewise ? n * a.num_labels + l : l;
        if (group != cur) {
            flush_group(a, cur, c, sh);
            cur = group;
        }
        const bool eq = (p == t);
        c[0] += (eq && t == 1);   // tp
        c[1] += (!eq && t == 0);  // fp
        c[2] += (eq && t == 0);   // tn
        c[3] += (!eq && t == 1);  // fn
    }
    if (!a.samplewise && a.num_labels == 1) {
        // single group: reduce across the warp before touching memory
#pragma unroll
        for (int k = 0; k < 4; ++k) c[k] = __reduce_add_sync(kFull, c[k]);
        if (lane == 0) {
            cur = 0;
            flush_group(a, cur, c, sh);
        }
    } else {
        flush_group(a, cur, c, sh);
    }
    if (sh) {
        __syncthreads();
        for (int i = threadIdx.x; i < a.smem_groups * 4; i += blockDim.x) {
            const unsigned v = sh[i];
            if (v) red_add_u64(a.counts + i, v);
        }
    }
}

// prediction from a score VALUE (same arithmetic as pred_label)
template <typename T>
__device__ __forceinline__ int pred_from_value(const BinArgs& a, T x, bool logits) {
    if constexpr (sizeof(T) == 8) {
        double v = x;
        if (logits) v = 1.0 / (1.0 + exp(-v));
        return v > a.threshold_d ? 1 : 0;
    } else {
        float v = to_f32(x);
        if (logits) v = round_to<T>(1.0f / (1.0f + expf(-v)));
        return v > a.threshold ? 1 : 0;
    }
}

// Single-group fast path (binary task, global counts, int64 targets, 16-byte aligned inputs): no per-element group
// arithmetic (the generic kernel spends two 64-bit divisions per element on it), 16-byte streaming loads for scores and
// labels, counters in registers, one warp reduction and four REDs per warp at the end.
template <typename T>
__global__ void __launch_bounds__(256) bin_count_flat_kernel(BinArgs a) {
    const bool logits = a.logits != nullptr && (*a.logits) != 0u;
    const long long total = a.n_outer * a.num_labels * a.inner;
    constexpr int kVec = 16 / (int)sizeof(T);
    const long long nvec = total / kVec;
    const uint4* __restrict__ pv = reinterpret_cast<const uint4*>(a.preds);
    const uint4* __restrict__ tv = reinterpret_cast<const uint4*>(a.target);  // two int64 labels per vector
    const T* __restrict__ ps = reinterpret_cast<const T*>(a.preds);
    const long long* __restrict__ ts = reinterpret_cast<const long long*>(a.target);
    const long long gtid = (long long)blockIdx.x * blockDim.x + threadIdx.x, stride = (long long)gridDim.x * blockDim.x;
    unsigned c[4] = {0, 0, 0, 0};
    bool bad_target = false;
    auto count = [&](T x, long long t) {
        if (a.has_ignore && t == a.ignore_index) return;
        if ((unsigned long long)t > 1ull) {
            bad_target = true;
            return;  // the reference counts such elements in none of the four masks
        }
        const int p = pred_from_value<T>(a, x, logits);
        const bool eq = (p == (int)t);
        c[0] += (eq && t == 1);
        c[1] += (!eq && t == 0);
        c[2] += (eq && t == 0);
        c[3] += (!eq && t == 1);
    };
    for (long long v = gtid; v < nvec; v += stride) {
        const uint4 q = ld_stream16(pv + v);
        const T* e = reinterpret_cast<const T*>(&q);
        uint4 lab[kVec / 2];
#pragma unroll
        for (int k = 0; k < kVec / 2; ++k) lab[k] = ld_stream16(tv + v * (kVec / 2) + k);
        const long long* l = reinterpret_cast<const long long*>(lab);
#pragma unroll
        for (int k = 0; k < kVec; ++k) count(e[k], l[k]);
    }
    for (long long i = nvec * kVec + gtid; i < total; i += stride) count(ps[i], ts[i]);
    if (__any_sync(kFull, bad_target) && (threadIdx.x & 31) == 0 && a.err) atomicOr(a.err, MB200_FLAG_TARGET_RANGE);
#pragma unroll
    for (int k = 0; k < 4; ++k) c[k] = __reduce_add_sync(kFull, c[k]);
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int k = 0; k < 4; ++k)
            if (c[k]) red_add_u64(a.counts + k, c[k]);
    }
}

// Single-pass variant of the flat path (f32 / f16 / bf16 scores): the batch-global "are these logits?" vote needs the whole
// batch before the first threshold decision, which is why the kernels above read the scores twice (16 B / element of traffic
// for 12 algorithmic).  Here every element is counted under BOTH outcomes of the vote in one read — four counters assuming
// probabilities, four assuming logits — while the vote itself is taken on the way; a one-warp epilogue kernel adds the set the
// vote selected to the states.  Counting under "logits" does not evaluate a sigmoid per element: sigmoid(x) > thr is decided
// by comparing x with a bracket [x_lo, x_hi] around logit(thr) computed on the host in double precision, wide enough to cover
// the rounding of the float32 sigmoid and of its store in T; only scores INSIDE the bracket (one spacing of T above the
// threshold, plus a 2^-20 relative band) run the exact arithmetic of `pred_from_value`, so the result is bit-identical to the
// two-pass kernels.
struct BothArgs {
    float x_lo, x_hi;            // outside (x_lo, x_hi): sigmoid(x) > thr is decided by the side; NaN bracket = always exact
    unsigned long long* both;    // [8] zeroed scratch: tp fp tn fn under "probabilities", then under "logits"
    unsigned* vote;              // zeroed word, set when any score lies outside [0, 1]
};

template <typename T>
__global__ void __launch_bounds__(256) bin_count_flat_both_kernel(BinArgs a, BothArgs b) {
    const long long total = a.n_outer * a.num_labels * a.inner;
    constexpr int kVec = 16 / (int)sizeof(T);
    const long long nvec = total / kVec;
    const uint4* __restrict__ pv = reinterpret_cast<const uint4*>(a.preds);
    const uint4* __restrict__ tv = reinterpret_cast<const uint4*>(a.target);
    const T* __restrict__ ps = reinterpret_cast<const T*>(a.preds);
    const long long* __restrict__ ts = reinterpret_cast<const long long*>(a.target);
    const long long gtid = (long long)blockIdx.x * blockDim.x + threadIdx.x, stride = (long long)gridDim.x * blockDim.x;
    unsigned cp[4] = {0, 0, 0, 0}, cl[4] = {0, 0, 0, 0};
    bool bad_target = false, outside = false;
    const bool bracket = b.x_lo == b.x_lo;  // NaN bracket: no shortcut for this threshold
    auto count = [&](T x, long long t) {
        const float v = to_f32(x);
        outside |= (v < 0.f) | (v > 1.f);  // the vote runs over EVERY score, ignored targets included, like the reference's
                                           // `torch.all((preds >= 0) * (preds <= 1))` (stat_scores.py:118-121)
        if (a.has_ignore && t == a.ignore_index) return;
        if ((unsigned long long)t > 1ull) {
            bad_target = true;
            return;
        }
        const int pp = v > a.threshold ? 1 : 0;
        int pl;
        if (bracket && v > b.x_hi) pl = 1;
        else if (bracket && v < b.x_lo) pl = 0;
        else pl = pred_from_value<T>(a, x, true);
        const int ti = (int)t;
        cp[0] += (pp == 1 && ti == 1), cp[1] += (pp == 1 && ti == 0), cp[2] += (pp == 0 && ti == 0), cp[3] += (pp == 0 && ti == 1);
        cl[0] += (pl == 1 && ti == 1), cl[1] += (pl == 1 && ti == 0), cl[2] += (pl == 0 && ti == 0), cl[3] += (pl == 0 && ti == 1);
    };
    for (long long v = gtid; v < nvec; v += stride) {
        const uint4 q = ld_stream16(pv + v);
        const T* e = reinterpret_cast<const T*>(&q);
        uint4 lab[kVec / 2];
#pragma unroll
        for (int k = 0; k < kVec / 2; ++k) lab[k] = ld_stream16(tv + v * (kVec / 2) + k);
        const long long* l = reinterpret_cast<const long long*>(lab);
#pragma unroll
        for (int k = 0; k < kVec; ++k) count(e[k], l[k]);
    }
    for (long long i = nvec * kVec + gtid; i < total; i += stride) count(ps[i], ts[i]);
    if (__any_sync(kFull, bad_target) && (threadIdx.x & 31) == 0 && a.err) atomicOr(a.err, MB200_FLAG_TARGET_RANGE);
    if (__any_sync(kFull, outside) && (threadIdx.x & 31) == 0) atomicOr(b.vote, 1u);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        cp[k] = __reduce_add_sync(kFull, cp[k]);
        cl[k] = __reduce_add_sync(kFull, cl[k]);
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if (cp[k]) atomicAdd(b.both + k, (unsigned long long)cp[k]);
            if (cl[k]) atomicAdd(b.both + 4 + k, (unsigned long long)cl[k]);
        }
    }
}

__global__ void bin_select_kernel(const unsigned long long* __restrict__ both, const unsigned* __restrict__ vote,
                                  long long* __restrict__ counts) {
    if (threadIdx.x < 4) {
        const unsigned long long v = both[(*vote != 0u ? 4 : 0) + threadIdx.x];
        if (v) red_add_u64(counts + threadIdx.x, v);
    }
}

// Multilabel fast path (global counts, `[N, L]` layout with inner == 1, L <= 256): every thread OWNS one label column
// (column = threadIdx % L, rows strided over the grid), so its four counters live in registers for the whole kernel and
// consecutive threads still read consecutive addresses.  The generic kernel flushes its register counters to shared
// memory whenever the group changes — with inner == 1 that is every element.
template <typename T>
__global__ void __launch_bounds__(256) bin_count_cols_kernel(BinArgs a) {
    __shared__ unsigned sh[256 * 4];
    const int L = (int)a.num_labels;
    for (int i = threadIdx.x; i < L * 4; i += blockDim.x) sh[i] = 0;
    __syncthreads();
    const bool logits = a.logits != nullptr && (*a.logits) != 0u;
    const int rows_per_block = 256 / L;
    const int col = threadIdx.x % L;
    const int rloc = threadIdx.x / L;
    unsigned c[4] = {0, 0, 0, 0};
    bool bad_target = false;
    if (rloc < rows_per_block) {
        const T* __restrict__ ps = reinterpret_cast<const T*>(a.preds);
        const long long rstride = (long long)gridDim.x * rows_per_block;
        long long r = (long long)blockIdx.x * rows_per_block + rloc;
        auto count = [&](T x, long long t) {
            if (a.has_ignore && t == a.ignore_index) return;
            if ((unsigned long long)t > 1ull) {
                bad_target = true;
                return;
            }
            const int p = pred_from_value<T>(a, x, logits);
            const bool eq = (p == (int)t);
            c[0] += (eq && t == 1);
            c[1] += (!eq && t == 0);
            c[2] += (eq && t == 0);
            c[3] += (!eq && t == 1);
        };
        for (; r + rstride < a.n_outer; r += 2 * rstride) {  // two independent elements in flight
            const long long i0 = r * L + col, i1 = (r + rstride) * L + col;
            const T x0 = ps[i0], x1 = ps[i1];
            const long long t0 = load_label(a.target, a.target_dtype, i0), t1 = load_label(a.target, a.target_dtype, i1);
            count(x0, t0);
            count(x1, t1);
        }
        for (; r < a.n_outer; r += rstride) {
            const long long i0 = r * L + col;
            count(ps[i0], load_label(a.target, a.target_dtype, i0));
        }
#pragma unroll
        for (int k = 0; k < 4; ++k)
            if (c[k]) atomicAdd(&sh[col * 4 + k], c[k]);
    }
    if (__any_sync(kFull, bad_target) && (threadIdx.x & 31) == 0 && a.err) atomicOr(a.err, MB200_FLAG_TARGET_RANGE);
    __syncthreads();
    for (int i = threadIdx.x; i < L * 4; i += blockDim.x) {
        const unsigned v = sh[i];
        if (v) red_add_u64(a.counts + i, v);
    }
}

}  // namespace mb200

using namespace mb200;

// The threshold the reference's `preds > threshold` compares a score with: ATen casts the Python float to the score dtype
// first (double -> float -> half / bfloat16, each round-to-nearest-even), so a float16 score of 0.30004883 is NOT above 0.3.
static float threshold_in_dtype(double threshold, int dtype) {
    const float f = (float)threshold;
    if (dtype == MB200_F16) return __half2float(__float2half_rn(f));
    if (dtype == MB200_BF16) return __bfloat162float(__float2bfloat16_rn(f));
    return f;
}

// the next value above v (finite, >= 0) representable in the score dtype
static float next_in_dtype(float v, int dtype) {
    if (dtype == MB200_F16) {
        __half_raw r = __float2half_rn(v);
        ++r.x;
        return __half2float(__half(r));
    }
    if (dtype == MB200_BF16) {
        __nv_bfloat16_raw r = __float2bfloat16_rn(v);
        ++r.x;
        return __bfloat162float(__nv_bfloat16(r));
    }
    return std::nextafter(v, INFINITY);
}

static int binary_stat_counts_impl(const void* preds, int preds_dtype, const void* target, int target_dtype, int64_t n_outer,
                                   int64_t num_labels, int64_t inner, double threshold, int has_ignore_index,
                                   int64_t ignore_index, int samplewise, int64_t* counts, uint32_t* flag_scratch,
                                   int64_t flag_scratch_bytes, uint32_t* err_flag, void* stream) {
    MB200_REQUIRE(n_outer >= 0 && num_labels >= 1 && inner >= 1, "bad sizes");
    const long long total = n_outer * num_labels * inner;
    if (total == 0) return 0;
    MB200_REQUIRE(preds && target && counts, "NULL pointer");
    MB200_REQUIRE(is_label_tag(target_dtype), "target must be an integer tensor");
    const bool float_preds = is_float_tag(preds_dtype);
    MB200_REQUIRE(!float_preds || flag_scratch, "flag_scratch is required for floating scores");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const long long groups = samplewise ? n_outer * num_labels : num_labels;
    BinArgs a;
    a.preds = preds, a.target = target, a.preds_dtype = preds_dtype, a.target_dtype = target_dtype;
    a.n_outer = n_outer, a.num_labels = num_labels, a.inner = inner;
    a.threshold = threshold_in_dtype(threshold, preds_dtype), a.threshold_d = threshold;
    a.has_ignore = has_ignore_index, a.ignore_index = ignore_index, a.samplewise = samplewise;
    a.counts = reinterpret_cast<long long*>(counts);
    a.logits = float_preds ? flag_scratch : nullptr;
    a.err = err_flag;
    a.smem_groups = (groups <= 2048) ? (int)groups : 0;
    const size_t smem = (size_t)a.smem_groups * 4 * sizeof(unsigned);
    long long blocks = (total + 256 * 16 - 1) / (256 * 16);
    const long long cap = (long long)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    const int grid = (int)blocks;
    const bool flat = float_preds && !samplewise && num_labels == 1 && target_dtype == MB200_I64 &&
                      ((reinterpret_cast<uintptr_t>(preds) | reinterpret_cast<uintptr_t>(target)) & 15) == 0;
    // single pass (see bin_count_flat_both_kernel): flag_scratch then holds the vote word and, 8 bytes in, the 8 counters
    const bool single_pass = flat && preds_dtype != MB200_F64 && flag_scratch_bytes >= 72 &&
                             (reinterpret_cast<uintptr_t>(flag_scratch) & 7) == 0;
    if (single_pass) {
        MB200_CUDA_OK(cudaMemsetAsync(flag_scratch, 0, 72, st));
        BothArgs b;
        b.vote = flag_scratch;
        b.both = reinterpret_cast<unsigned long long*>(flag_scratch + 2);
        // bracket around logit(threshold).  The exact decision compares s = the float32 sigmoid (rounded to T) with the
        // T-valued a.threshold; it can only flip for s in (thr, up], up the next T value above thr: s <= thr rounds to at
        // most thr, s >= up to at least up.  The float32 sigmoid is within 2^-21 relative of sigmoid(x) (expf <= 2 ulp,
        // add and divide 0.5 ulp each) while s is a normal float32, so eps = 2^-20 around [thr, up] holds every score
        // whose side is in doubt.  up - thr is T's absolute spacing at thr, float16 subnormals included.  A threshold
        // that rounds to <= 1e-6 or whose band reaches 1 has no bracket: every score runs the exact arithmetic.
        const double eps = 0x1p-20, thr = a.threshold, up = next_in_dtype(a.threshold, preds_dtype);
        const double lo_p = thr * (1.0 - eps), hi_p = up * (1.0 + eps);
        if (thr > 1e-6 && hi_p < 1.0 - 1e-6) {
            const double xl = std::log(lo_p / (1.0 - lo_p)), xh = std::log(hi_p / (1.0 - hi_p));
            b.x_lo = (float)(xl - 1e-5 * (1.0 + std::fabs(xl)));
            b.x_hi = (float)(xh + 1e-5 * (1.0 + std::fabs(xh)));
        } else {
            b.x_lo = b.x_hi = std::nanf("");
        }
        with_float_type<kNoF64>(preds_dtype, [&](auto t) {
            bin_count_flat_both_kernel<typename decltype(t)::type><<<grid, 256, 0, st>>>(a, b);
            return 0;
        });
        bin_select_kernel<<<1, 32, 0, st>>>(b.both, b.vote, a.counts);
        count_launch();
        count_launch();
        return check_cuda(cudaGetLastError(), "binary stat counts launch");
    }
    if (float_preds) {
        MB200_CUDA_OK(cudaMemsetAsync(flag_scratch, 0, sizeof(uint32_t), st));
        const int fgrid = (int)std::min<long long>(cap, (total + 2047) / 2048);
        with_float_type(preds_dtype, [&](auto t) {
            using T = typename decltype(t)::type;
            bin_range_flag_kernel<T><<<fgrid, 256, 0, st>>>((const T*)preds, total, flag_scratch);
            return 0;
        });
        count_launch();
    }
    if (flat) {
        with_float_type(preds_dtype, [&](auto t) {
            bin_count_flat_kernel<typename decltype(t)::type><<<grid, 256, 0, st>>>(a);
            return 0;
        });
        count_launch();
        return check_cuda(cudaGetLastError(), "binary stat counts launch");
    }
    if (float_preds && !samplewise && inner == 1 && num_labels >= 2 && num_labels <= 256) {
        with_float_type(preds_dtype, [&](auto t) {
            bin_count_cols_kernel<typename decltype(t)::type><<<grid, 256, 0, st>>>(a);
            return 0;
        });
        count_launch();
        return check_cuda(cudaGetLastError(), "binary stat counts launch");
    }
    const int rc = with_float_type(preds_dtype, [&](auto t) {
        bin_count_kernel<typename decltype(t)::type><<<grid, 256, smem, st>>>(a);
        return 0;
    });
    if (rc == kNoType) bin_count_kernel<IntPred><<<grid, 256, smem, st>>>(a);
    count_launch();
    return check_cuda(cudaGetLastError(), "binary stat counts launch");
}

extern "C" int mb200_binary_stat_counts(const void* preds, int preds_dtype, const void* target, int target_dtype,
                                        int64_t n_outer, int64_t num_labels, int64_t inner, double threshold,
                                        int has_ignore_index, int64_t ignore_index, int samplewise, int64_t* counts,
                                        uint32_t* flag_scratch, uint32_t* err_flag, void* stream) {
    return binary_stat_counts_impl(preds, preds_dtype, target, target_dtype, n_outer, num_labels, inner, threshold,
                                   has_ignore_index, ignore_index, samplewise, counts, flag_scratch, 4, err_flag, stream);
}

// Same contract with a larger caller-owned scratch (>= MB200_BINARY_SCRATCH_BYTES, 8-byte aligned): lets the binary task count
// in ONE pass over the scores (both outcomes of the logits vote at once, see bin_count_flat_both_kernel).
extern "C" int mb200_binary_stat_counts_scratch(const void* preds, int preds_dtype, const void* target, int target_dtype,
                                                int64_t n_outer, int64_t num_labels, int64_t inner, double threshold,
                                                int has_ignore_index, int64_t ignore_index, int samplewise, int64_t* counts,
                                                uint32_t* scratch, int64_t scratch_bytes, uint32_t* err_flag, void* stream) {
    return binary_stat_counts_impl(preds, preds_dtype, target, target_dtype, n_outer, num_labels, inner, threshold,
                                   has_ignore_index, ignore_index, samplewise, counts, scratch, scratch_bytes, err_flag, stream);
}
