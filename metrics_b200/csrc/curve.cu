// K3 / K5 / K6 — exact ROC / PR-curve family on sm_90a: score formatting, key packing, segmented LSD radix sort,
// tie-collapsing TP/FP scan with fused AUROC / average-precision accumulation.
//
// Reference op chain replaced (src/torchmetrics/):
//   utilities/compute.py:190-229                      normalize_logits_if_needed (batch-global range test + sigmoid/softmax)
//   functional/classification/precision_recall_curve.py:30-82   _binary_clf_curve: argsort(desc) -> gathers -> distinct
//                                                     thresholds (where) -> cumsum -> fps = 1 + idx - tps
//   functional/classification/roc.py:40-80, auroc.py:83-107, average_precision.py:70-75, compute.py:101-109 (trapz)
//   functional/classification/{roc.py:162-204, precision_recall_curve.py:565-569}  per-class Python loop (one sort each)
//
// Data layout: a "segment" is one curve (binary: 1 segment; multiclass one-vs-rest: one segment per class, stored
// class-major so that a segment is contiguous).  Per element we keep a 4-byte key (order-preserving transform of the fp32
// score, inverted so that ascending key order == descending score order) and a 1-byte label (target == positive class).
// The 8-bit LSD radix sort moves 5 B/element/pass; with <= ~5 M elements both ping-pong buffers fit the 50 MB L2.
// The scan counts in integers: TP/FP are exact for any N < 2^32 per segment (the reference counts in fp32 and is exact
// only below 2^24), AUROC is accumulated as the exact integer  sum dFP * (TP_prev + TP)  (== 2 * Mann-Whitney U),
// AP in fp64 with a fixed reduction order (deterministic).
#include "common.cuh"
#include "radix_sort.cuh"

namespace mb200 {

// =====================================================================================================
// helpers
// =====================================================================================================
// Runs the reference splits.  It finds thresholds with where(preds[1:] - preds[:-1]): NaN - NaN and inf - inf are NaN, so
// every NaN, +inf or -inf score ends its own group.  Their desc keys sit at the two ends of the key range, next to the
// NaN payloads no score maps to: NaN 0, +inf 0x007fffff, -inf 0xff800000 (64-bit: 0, 0x000fffffffffffff,
// 0xfff0000000000000).  Inside such a run the order is fixed as negatives before positives, on every path: the bit-0 path
// gets it from the label in the low bit, the pair paths from label_key, which moves one label of each special value to the
// unused neighbour key (NaN 0/1, +inf 0x..fe/0x..ff, -inf 0x..00/0x..01 as (negative, positive)).
template <typename KeyT>
struct SpecialKeys {
    static constexpr KeyT kPosInf = sizeof(KeyT) == 4 ? (KeyT)0x007fffffu : (KeyT)0x000fffffffffffffull;
    static constexpr KeyT kNegInf = sizeof(KeyT) == 4 ? (KeyT)0xff800000u : (KeyT)0xfff0000000000000ull;
};
// true for the keys of NaN, +inf and -inf (and their label neighbours): k < kPosInf + 1 or k >= kNegInf, as one compare
template <typename KeyT>
__device__ __forceinline__ bool is_special_key(KeyT k) {
    return (KeyT)(k + (SpecialKeys<KeyT>::kPosInf + 1)) < (KeyT)(2 * (SpecialKeys<KeyT>::kPosInf + 1));
}
template <typename KeyT>
__device__ __forceinline__ KeyT label_key(KeyT k, bool positive) {
    if (positive) return (k == 0 || k == SpecialKeys<KeyT>::kNegInf) ? k + 1 : k;
    return k == SpecialKeys<KeyT>::kPosInf ? k - 1 : k;
}
// the canonical key of a label_key result
template <typename KeyT>
__device__ __forceinline__ KeyT canonical_key(KeyT k) {
    if (k == 1) return 0;
    if (k == SpecialKeys<KeyT>::kPosInf - 1) return SpecialKeys<KeyT>::kPosInf;
    if (k == SpecialKeys<KeyT>::kNegInf + 1) return SpecialKeys<KeyT>::kNegInf;
    return k;
}
__device__ __forceinline__ float score_of_key(unsigned k) {
    const unsigned ok = ~canonical_key(k);
    if (ok == 0xffffffffu) return __int_as_float(0x7fc00000);
    return f32_from_order_key(ok);
}
__device__ __forceinline__ double score_of_key(unsigned long long k) {
    const unsigned long long ok = ~canonical_key(k);
    if (ok == ~0ull) return __longlong_as_double(0x7ff8000000000000ll);
    const unsigned long long b = (ok & 0x8000000000000000ull) ? (ok & 0x7fffffffffffffffull) : ~ok;
    return __longlong_as_double((long long)b);
}
// Key type of a score type: float64 scores keep all 64 bits (the reference sorts them as doubles); everything else is
// compared as float32, like ATen compares half / bfloat16 values.
template <typename T>
struct KeyOf {
    using type = unsigned;
    static __device__ __forceinline__ unsigned make(T v) { return f32_desc_key(to_f32(v)); }
};
template <>
struct KeyOf<double> {
    using type = unsigned long long;
    static __device__ __forceinline__ unsigned long long make(double v) { return ~f64_order_key(v); }
};
template <typename KeyT>
struct ThrOf { using type = float; };
template <>
struct ThrOf<unsigned long long> { using type = double; };

// =====================================================================================================
// K6: batch-global "are these logits?" test and conditional sigmoid  (utilities/compute.py:223-229, device branch:
// cond = any(x < 0) | any(x > 1); out = where(cond, sigmoid(x), x) — decided per batch tensor, no host sync)
// =====================================================================================================
template <typename T>
__global__ void __launch_bounds__(256) range_flag_kernel(const T* __restrict__ x, long long n, unsigned* flag) {
    bool bad = false;
    constexpr int kVec = 16 / (int)sizeof(T);
    // 16-byte streaming loads over the aligned body, scalar head / tail
    const uintptr_t addr = reinterpret_cast<uintptr_t>(x);
    long long head = (long long)(((16 - (addr & 15)) & 15) / sizeof(T));
    if (head > n) head = n;
    const long long nvec = (n - head) / kVec;
    const uint4* __restrict__ xv = reinterpret_cast<const uint4*>(x + head);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
        const uint4 q = ld_stream16(xv + i);
        const T* e = reinterpret_cast<const T*>(&q);
#pragma unroll
        for (int k = 0; k < kVec; ++k) {
            const float v = to_f32(e[k]);
            bad |= (v < 0.f) | (v > 1.f);
        }
    }
    const long long tail0 = head + nvec * kVec;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < head + (n - tail0); i += (long long)gridDim.x * blockDim.x) {
        const long long j = i < head ? i : tail0 + (i - head);
        const float v = to_f32(x[j]);
        bad |= (v < 0.f) | (v > 1.f);
    }
    if (__any_sync(kFull, bad) && (threadIdx.x & 31) == 0) atomicOr(flag, 1u);
}
template <>
__global__ void __launch_bounds__(256) range_flag_kernel<double>(const double* __restrict__ x, long long n, unsigned* flag) {
    bool bad = false;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const double v = x[i];
        bad |= (v < 0.0) | (v > 1.0);
    }
    if (__any_sync(kFull, bad) && (threadIdx.x & 31) == 0) atomicOr(flag, 1u);
}

template <typename T>
__global__ void __launch_bounds__(256) sigmoid_if_kernel(const T* __restrict__ x, T* __restrict__ out, long long n,
                                                         const unsigned* __restrict__ flag) {
    const bool apply = (*flag) != 0u;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        if (apply) {
            const float v = to_f32(x[i]);
            out[i] = narrow<T>(sigmoid_f32(v));  // fp32 math, rounded to T like ATen's sigmoid
        } else {
            out[i] = x[i];
        }
    }
}
template <>
__global__ void __launch_bounds__(256) sigmoid_if_kernel<double>(const double* __restrict__ x, double* __restrict__ out,
                                                                 long long n, const unsigned* __restrict__ flag) {
    const bool apply = (*flag) != 0u;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        out[i] = apply ? 1.0 / (1.0 + exp(-x[i])) : x[i];
}

// Speculative single pass for large batches (f32 / f16 / bf16, 16-byte aligned): the vote is batch-global, but a TILE that
// itself holds a score outside [0, 1] already knows the outcome — it writes sigmoids; a tile with all scores inside [0, 1]
// writes them through and marks itself pending.  Real logits leave no pending tile (the chance that 4096 logits all fall in
// [0, 1] is nil), real probabilities leave every tile pending AND the vote at "not logits": in both cases the batch was read
// once and written once (8 B / element for f32 instead of 12) and the fix-up launch below finds nothing to do; only a batch
// of logits with in-range stretches makes it revisit the pending tiles.
constexpr int kSpecVecPerThread = 4;
constexpr int kSpecTileVecs = 256 * kSpecVecPerThread;  // 16 KB of scores per tile
template <typename T, bool kFix>
__global__ void __launch_bounds__(256) sigmoid_spec_kernel(const T* __restrict__ x, T* __restrict__ out, long long n,
                                                           unsigned* __restrict__ vote, unsigned char* __restrict__ pending,
                                                           long long ntiles) {
    constexpr int kVec = 16 / (int)sizeof(T);
    const long long nvec = n / kVec;
    const uint4* __restrict__ xv = reinterpret_cast<const uint4*>(x);
    uint4* __restrict__ ov = reinterpret_cast<uint4*>(out);
    if (kFix && *vote == 0u) return;
    bool cta_voted = false;
    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        if (kFix && pending[tile] == 0) continue;
        const long long v0 = tile * kSpecTileVecs + threadIdx.x;
        uint4 q[kSpecVecPerThread];
        bool outside = false;
#pragma unroll
        for (int k = 0; k < kSpecVecPerThread; ++k) {
            const long long v = v0 + (long long)k * 256;
            if (v < nvec) {
                q[k] = ld_stream16(xv + v);
                const T* e = reinterpret_cast<const T*>(&q[k]);
#pragma unroll
                for (int j = 0; j < kVec; ++j) {
                    const float f = to_f32(e[j]);
                    outside |= (f < 0.f) | (f > 1.f);
                }
            }
        }
        const bool last = tile == ntiles - 1;
        if (last)  // the (< one vector) scalar tail belongs to the last tile
            for (long long i = nvec * kVec + threadIdx.x; i < n; i += 256) {
                const float f = to_f32(x[i]);
                outside |= (f < 0.f) | (f > 1.f);
            }
        const bool apply = kFix ? true : (__syncthreads_or(outside) != 0);
        if (!kFix && threadIdx.x == 0) {
            if (apply) {
                if (!cta_voted) atomicOr(vote, 1u);
                cta_voted = true;
            } else {
                pending[tile] = 1;
            }
        }
#pragma unroll
        for (int k = 0; k < kSpecVecPerThread; ++k) {
            const long long v = v0 + (long long)k * 256;
            if (v < nvec) {
                if (apply) {
                    T* e = reinterpret_cast<T*>(&q[k]);
#pragma unroll
                    for (int j = 0; j < kVec; ++j) e[j] = narrow<T>(sigmoid_f32(to_f32(e[j])));
                }
                ov[v] = q[k];
            }
        }
        if (last)
            for (long long i = nvec * kVec + threadIdx.x; i < n; i += 256)
                out[i] = apply ? narrow<T>(sigmoid_f32(to_f32(x[i]))) : x[i];
    }
}

// Small batches (n <= 1024 * kSmallItems): ONE CTA holds the whole batch in registers, votes with __syncthreads_or and
// writes the result — one launch instead of memset + flag kernel + apply kernel (cfg3: 10 000 scores per update; the
// launch sequence, not the 40 KB of traffic, is what an update costs).
constexpr int kSmallItems = 32;
constexpr int kSmallItemsF64 = 12;
template <typename T, int kItems>
__global__ void __launch_bounds__(1024) sigmoid_if_small_kernel(const T* __restrict__ x, T* __restrict__ out, int n) {
    constexpr int kSmallItems = kItems;
    T v[kSmallItems];
    bool bad = false;
#pragma unroll
    for (int k = 0; k < kSmallItems; ++k) {
        const int i = k * 1024 + threadIdx.x;
        if (i < n) {
            v[k] = x[i];
            if constexpr (sizeof(T) == 8) {
                const double d = (double)v[k];
                bad |= (d < 0.0) | (d > 1.0);
            } else {
                const float f = to_f32(v[k]);
                bad |= (f < 0.f) | (f > 1.f);
            }
        }
    }
    const bool apply = __syncthreads_or(bad) != 0;
#pragma unroll
    for (int k = 0; k < kSmallItems; ++k) {
        const int i = k * 1024 + threadIdx.x;
        if (i < n) {
            if (!apply) {
                out[i] = v[k];
            } else if constexpr (sizeof(T) == 8) {
                out[i] = (T)(1.0 / (1.0 + exp(-(double)v[k])));
            } else {
                out[i] = narrow<T>(sigmoid_f32(to_f32(v[k])));
            }
        }
    }
}

// Row softmax over [N, C] when the batch flag is set (utilities/compute.py:226-229 with normalization="softmax").
// One warp per row, values staged in registers chunk-wise; fp32 math.
template <typename T>
__global__ void __launch_bounds__(256) softmax_if_kernel(const T* __restrict__ x, T* __restrict__ out, int n, int C,
                                                         const unsigned* __restrict__ flag) {
    const bool apply = (*flag) != 0u;
    const int lane = threadIdx.x & 31;
    const int wpb = blockDim.x >> 5;
    for (int r = blockIdx.x * wpb + (threadIdx.x >> 5); r < n; r += gridDim.x * wpb) {
        const T* __restrict__ row = x + (size_t)r * C;
        T* __restrict__ orow = out + (size_t)r * C;
        if (!apply) {
            for (int c = lane; c < C; c += 32) orow[c] = row[c];
            continue;
        }
        float m = -INFINITY;
        for (int c = lane; c < C; c += 32) m = fmaxf(m, to_f32(row[c]));
        m = warp_max(m);
        float s = 0.f;
        for (int c = lane; c < C; c += 32) s += expf(to_f32(row[c]) - m);
        s = warp_sum(s);
        for (int c = lane; c < C; c += 32) orow[c] = narrow<T>(expf(to_f32(row[c]) - m) / s);
    }
}

// Speculative single pass over [N, C <= 1024] rows (f32 / f16 / bf16): a warp keeps its row in registers, so the maximum, the
// sum and the quotient need ONE read and ONE `expf` per score (the kernel above reads the row three times and exponentiates
// twice), and the batch-global vote is handled like in `sigmoid_spec_kernel`: a row that itself holds a score outside [0, 1]
// knows the outcome and writes its softmax; an in-range row is written through and marked pending, to be revisited by the
// fix-up launch only if the batch turns out to be logits.  Same summation order as above (lane-strided partial sums,
// butterfly), hence the same bits as ATen's warp softmax.
template <typename T, int kIter, bool kFix>
__global__ void __launch_bounds__(256, 3) softmax_spec_kernel(const T* __restrict__ x, T* __restrict__ out, int n, int C,
                                                           unsigned* __restrict__ vote, unsigned char* __restrict__ pending) {
    if (kFix && *vote == 0u) return;
    const int lane = threadIdx.x & 31;
    const int wpb = blockDim.x >> 5;
    bool warp_voted = false;
    for (int r = blockIdx.x * wpb + (threadIdx.x >> 5); r < n; r += gridDim.x * wpb) {
        if (kFix && pending[r] == 0) continue;
        const T* __restrict__ row = x + (size_t)r * C;
        T* __restrict__ orow = out + (size_t)r * C;
        float v[kIter];
        bool outside = false;
        float m = -INFINITY;
#pragma unroll
        for (int it = 0; it < kIter; ++it) {
            const int c = lane + 32 * it;
            if (c < C) {
                v[it] = to_f32(row[c]);
                outside |= (v[it] < 0.f) | (v[it] > 1.f);
                m = fmaxf(m, v[it]);
            }
        }
        const bool apply = kFix ? true : (__any_sync(kFull, outside) != 0);
        if (!kFix && lane == 0) {
            if (apply) {
                if (!warp_voted) atomicOr(vote, 1u);
            } else {
                pending[r] = 1;
            }
        }
        warp_voted |= apply;
        if (!apply) {  // write-through from the registers: T -> float -> T is exact
#pragma unroll
            for (int it = 0; it < kIter; ++it) {
                const int c = lane + 32 * it;
                if (c < C) orow[c] = narrow<T>(v[it]);
            }
            continue;
        }
        m = warp_max(m);
        float s = 0.f;
#pragma unroll
        for (int it = 0; it < kIter; ++it) {
            const int c = lane + 32 * it;
            if (c < C) {
                v[it] = expf(v[it] - m);
                s += v[it];
            }
        }
        s = warp_sum(s);
#pragma unroll
        for (int it = 0; it < kIter; ++it) {
            const int c = lane + 32 * it;
            if (c < C) orow[c] = narrow<T>(v[it] / s);
        }
    }
}

// float64 rows: the same warp layout in double arithmetic (ATen's CUDA softmax accumulates doubles in double)
template <>
__global__ void __launch_bounds__(256) softmax_if_kernel<double>(const double* __restrict__ x, double* __restrict__ out, int n,
                                                                 int C, const unsigned* __restrict__ flag) {
    const bool apply = (*flag) != 0u;
    const int lane = threadIdx.x & 31;
    const int wpb = blockDim.x >> 5;
    for (int r = blockIdx.x * wpb + (threadIdx.x >> 5); r < n; r += gridDim.x * wpb) {
        const double* __restrict__ row = x + (size_t)r * C;
        double* __restrict__ orow = out + (size_t)r * C;
        if (!apply) {
            for (int c = lane; c < C; c += 32) orow[c] = row[c];
            continue;
        }
        double m = -INFINITY;
        for (int c = lane; c < C; c += 32) m = fmax(m, row[c]);
        m = warp_max(m);
        double s = 0.0;
        for (int c = lane; c < C; c += 32) s += exp(row[c] - m);
        s = warp_sum(s);
        for (int c = lane; c < C; c += 32) orow[c] = exp(row[c] - m) / s;
    }
}

// =====================================================================================================
// key packing
// =====================================================================================================
// binary: keys[i] = f32_desc_key(preds[i]), labels[i] = (target[i] == pos_label)
// kBit0 (scores promised to be non-negative or NaN — in particular everything normalize_logits_if_needed returns): their
// 32-bit keys use 31 bits (no sign; NaN -> 0), so the label rides in bit 0 of the key and the sort moves 4-byte keys only
// (radix_sort_passes_bit0); a negative score (other than -0) raises MB200_FLAG_PREDS_RANGE.
template <typename T, bool kBit0 = false, bool kI64 = false>
__global__ void __launch_bounds__(256) pack_binary_kernel(const T* __restrict__ preds, const void* __restrict__ target,
                                                          int tdtype, long long n, long long pos_label,
                                                          typename KeyOf<T>::type* __restrict__ keys,
                                                          unsigned char* __restrict__ labels, unsigned* __restrict__ err = nullptr,
                                                          unsigned* __restrict__ hist = nullptr) {
    // kBit0 also counts the four digit histograms of the sort (radix_sort.cuh, layout [pass][256]) while the key is in a
    // register; the sort's own histogram read of the keys goes away.  The shared-memory atomics (4 per key, ~4.6 lanes per
    // clock per SM measured) are the floor of this kernel, so the loads of kVec elements per thread are issued together
    // (coalesced, kI64: no dtype switch in between) and hide behind them.
    constexpr int kVec = 4;
    __shared__ unsigned sh_hist[kBit0 ? 4 * 256 : 1];
    if constexpr (kBit0) {
        for (int i = threadIdx.x; i < 4 * 256; i += blockDim.x) sh_hist[i] = 0;
        __syncthreads();
    }
    bool bad = false;
    const long long step = (long long)gridDim.x * (256 * kVec);
    for (long long base = (long long)blockIdx.x * (256 * kVec) + threadIdx.x; base < n; base += step) {
        T v[kVec];
        long long lab[kVec];
#pragma unroll
        for (int q = 0; q < kVec; ++q) {
            const long long i = base + q * 256;
            const bool ok = i < n;
            v[q] = ok ? preds[i] : T(0);
            lab[q] = !ok ? 0ll : kI64 ? reinterpret_cast<const long long*>(target)[i] : load_label(target, tdtype, i);
        }
#pragma unroll
        for (int q = 0; q < kVec; ++q) {
            const long long i = base + q * 256;
            if (i >= n) continue;
            const typename KeyOf<T>::type k = KeyOf<T>::make(v[q]);
            const unsigned one = (unsigned)(lab[q] == pos_label);
            if constexpr (kBit0) {
                bad |= (k >> 31) != 0;
                const unsigned ck = (unsigned)((k << 1) | one);
                keys[i] = ck;
#pragma unroll
                for (int p = 0; p < 4; ++p) atomicAdd(&sh_hist[p * 256 + ((ck >> (8 * p)) & 255u)], 1u);
            } else {
                keys[i] = label_key(k, one != 0u);
                labels[i] = (unsigned char)one;
            }
        }
    }
    if constexpr (kBit0) {
        if (bad && err) atomicOr(err, MB200_FLAG_PREDS_RANGE);
        __syncthreads();
        for (int i = threadIdx.x; i < 4 * 256; i += blockDim.x) {
            const unsigned v = sh_hist[i];
            if (v) atomicAdd(&hist[i], v);
        }
    }
}

// multiclass one-vs-rest: preds [N, C] row-major -> keys [C][N] (class-major), labels[c][n] = (target[n] == c).
// 32x32 shared-memory tile transpose so that both the read and the write are coalesced.
template <typename T, bool kBit0 = false>
__global__ void __launch_bounds__(256) pack_ovr_kernel(const T* __restrict__ preds, const void* __restrict__ target,
                                                       int tdtype, int n, int C,
                                                       typename KeyOf<T>::type* __restrict__ keys,
                                                       unsigned char* __restrict__ labels, unsigned* __restrict__ err = nullptr) {
    __shared__ typename KeyOf<T>::type tile[32][33];
    __shared__ long long tgt[32];  // compared in 64 bits: an int64 target of 2^32 + c is not class c
    const int n0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 8 rows of 32 threads
    if (threadIdx.x < 32) {
        const int nn = n0 + threadIdx.x;
        tgt[threadIdx.x] = nn < n ? load_label(target, tdtype, nn) : -1;
    }
    for (int j = ty; j < 32; j += 8) {
        const int nn = n0 + j, cc = c0 + tx;
        if (nn < n && cc < C) tile[j][tx] = KeyOf<T>::make(preds[(size_t)nn * C + cc]);
    }
    __syncthreads();
    for (int j = ty; j < 32; j += 8) {
        const int cc = c0 + j, nn = n0 + tx;
        if (nn < n && cc < C) {
            if constexpr (kBit0) {
                const typename KeyOf<T>::type k = tile[tx][j];
                if ((k >> 31) != 0 && err) atomicOr(err, MB200_FLAG_PREDS_RANGE);
                keys[(size_t)cc * n + nn] = (k << 1) | (typename KeyOf<T>::type)(tgt[tx] == cc);
                continue;
            }
            const bool one = tgt[tx] == cc;
            keys[(size_t)cc * n + nn] = label_key(tile[tx][j], one);
            labels[(size_t)cc * n + nn] = (unsigned char)one;
        }
    }
}

// multilabel: preds [N, L] and target [N, L] row-major -> keys / labels [L][N]; label = (target == 1).
// Entries whose target equals `ignore` get the largest key (they sort behind every real score) and are counted per
// label in seg_ignored[L]: the scan then works on the first n - seg_ignored[l] elements of segment l only — the
// reference filters them per label before its sort (functional/classification/precision_recall_curve.py:826-830).
template <typename T>
__global__ void __launch_bounds__(256) pack_multilabel_kernel(const T* __restrict__ preds, const void* __restrict__ target,
                                                              int tdtype, int n, int L, int has_ignore, long long ignore,
                                                              typename KeyOf<T>::type* __restrict__ keys,
                                                              unsigned char* __restrict__ labels,
                                                              int* __restrict__ seg_ignored) {
    using KeyT = typename KeyOf<T>::type;
    constexpr KeyT kIgnoredKey = ~(KeyT)0;
    __shared__ KeyT tile[32][33];
    __shared__ unsigned char ltile[32][33];
    const int n0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int j = ty; j < 32; j += 8) {
        const int nn = n0 + j, cc = c0 + tx;
        if (nn < n && cc < L) {
            const long long t = load_label(target, tdtype, (long long)nn * L + cc);
            const bool ign = has_ignore && t == ignore;
            const bool one = t == 1 && !ign;
            tile[j][tx] = ign ? kIgnoredKey : label_key(KeyOf<T>::make(preds[(size_t)nn * L + cc]), one);
            ltile[j][tx] = (unsigned char)one;
        }
    }
    __syncthreads();
    for (int j = ty; j < 32; j += 8) {
        const int cc = c0 + j, nn = n0 + tx;
        const bool ok = nn < n && cc < L;
        const KeyT k = ok ? tile[tx][j] : (KeyT)0;
        if (ok) {
            keys[(size_t)cc * n + nn] = k;
            labels[(size_t)cc * n + nn] = ltile[tx][j];
        }
        if (has_ignore) {  // warp-uniform; one warp = 32 samples of label cc
            const unsigned m = __ballot_sync(kFull, ok && k == kIgnoredKey);
            if (tx == 0 && m) atomicAdd(seg_ignored + cc, __popc(m));
        }
    }
}

// keys only, class-major, rows >= C (padding up to rows_out) left untouched: used by the class-sharded multi-GPU path
template <typename T>
__global__ void __launch_bounds__(256) pack_keys_kernel(const T* __restrict__ preds, int n, int C,
                                                        unsigned* __restrict__ keys) {
    __shared__ unsigned tile[32][33];
    load_desc_key_tile(preds, n, C, tile);
    __syncthreads();
    const int n0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int j = ty; j < 32; j += 8) {
        const int cc = c0 + j, nn = n0 + tx;
        if (nn < n && cc < C) keys[(size_t)cc * n + nn] = tile[tx][j];
    }
}

// labels[s][i] = (target[i] == first_class + s); the keys of NaN / +-inf scores move to their label's key (label_key)
__global__ void __launch_bounds__(256) labels_from_target_kernel(unsigned* __restrict__ keys, const void* __restrict__ target,
                                                                 int tdtype, int n, int segments, long long first_class,
                                                                 unsigned char* __restrict__ labels) {
    const long long total = (long long)n * segments;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int s = (int)(i / n);
        const int k = (int)(i - (long long)s * n);
        const bool one = load_label(target, tdtype, k) == first_class + s;
        labels[i] = (unsigned char)one;
        const unsigned key = keys[i];
        if (is_special_key(key)) keys[i] = label_key(key, one);
    }
}

// keys[s][i] = (keys[s][i] << 1) | (target[i] == first_class + s)   — packed keys of non-negative scores (31 bits), in place
__global__ void __launch_bounds__(256) fold_labels_into_keys_kernel(unsigned* __restrict__ keys, const void* __restrict__ target,
                                                                    int tdtype, int n, int segments, long long first_class,
                                                                    unsigned* __restrict__ err) {
    const long long total = (long long)n * segments;
    bool bad = false;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int s = (int)(i / n);
        const int k = (int)(i - (long long)s * n);
        const unsigned key = keys[i];
        bad |= (key >> 31) != 0;
        keys[i] = (key << 1) | (unsigned)(load_label(target, tdtype, k) == first_class + s);
    }
    if (bad && err) atomicOr(err, MB200_FLAG_PREDS_RANGE);
}

// =====================================================================================================
// tie-collapsing TP/FP scan over sorted (key, label): scan_chained_kernel below (tile states, look-back, apply) and the two
// finalize kernels that fold the per-tile AP partials in tile order.
// =====================================================================================================
// finalize: one warp per segment folds the per-tile AP partials in tile order and emits the scalars.
// out[seg] = {auroc, ap, n_pos, n_neg, n_thresholds} as fp32 (counts < 2^24 are exact; larger ones only inform weights)
__global__ void __launch_bounds__(256) scan_finalize_kernel(const unsigned long long* __restrict__ auroc_acc,
                                                            const double* __restrict__ ap_partial,
                                                            const unsigned* __restrict__ seg_totals, int tiles, int n_stride,
                                                            const int* __restrict__ seg_ignored,
                                                            int segments, float* __restrict__ out_auroc,
                                                            float* __restrict__ out_ap, long long* __restrict__ out_counts) {
    const int seg = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (seg >= segments) return;
    const int n = seg_ignored ? n_stride - seg_ignored[seg] : n_stride;
    double s = 0.0;
    // fixed order: lane-strided partial sums then a fixed shuffle tree
    for (int t = lane; t < tiles; t += 32) s += ap_partial[(size_t)seg * tiles + t];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(kFull, s, o);
    if (lane == 0) {
        const double P = (double)seg_totals[2 * seg + 0];
        const double Nn = (double)n - P;
        const double auc = (P > 0.0 && Nn > 0.0) ? (double)auroc_acc[seg] / (2.0 * P * Nn) : 0.0;
        // all-negative: the reference forces recall to 1 everywhere and gets -0.0 (precision_recall_curve.py:278-283)
        const double ap = P > 0.0 ? s / P : -0.0;
        out_auroc[seg] = (float)auc;
        out_ap[seg] = (float)ap;
        out_counts[3 * seg + 0] = (long long)seg_totals[2 * seg + 0];
        out_counts[3 * seg + 1] = (long long)n - (long long)seg_totals[2 * seg + 0];
        out_counts[3 * seg + 2] = (long long)seg_totals[2 * seg + 1];
    }
}

// Same as scan_finalize_kernel for segments with many tiles (binary curves over millions of samples: one segment, thousands
// of per-tile AP partials): a whole CTA folds one segment — thread-strided sums, then a fixed shuffle / shared-memory tree
// (deterministic; a single warp walking the partials is a chain of dependent L2 loads).
__global__ void __launch_bounds__(256) scan_finalize_wide_kernel(const unsigned long long* __restrict__ auroc_acc,
                                                                 const double* __restrict__ ap_partial,
                                                                 const unsigned* __restrict__ seg_totals, int tiles,
                                                                 int n_stride, const int* __restrict__ seg_ignored,
                                                                 float* __restrict__ out_auroc, float* __restrict__ out_ap,
                                                                 long long* __restrict__ out_counts) {
    __shared__ double part[8];
    const int seg = blockIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int n = seg_ignored ? n_stride - seg_ignored[seg] : n_stride;
    double s = 0.0;
    for (int t = threadIdx.x; t < tiles; t += 256) s += ap_partial[(size_t)seg * tiles + t];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(kFull, s, o);
    if (lane == 0) part[warp] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double tot = 0.0;
#pragma unroll
        for (int w = 0; w < 8; ++w) tot += part[w];
        const double P = (double)seg_totals[2 * seg + 0];
        const double Nn = (double)n - P;
        const double auc = (P > 0.0 && Nn > 0.0) ? (double)auroc_acc[seg] / (2.0 * P * Nn) : 0.0;
        const double ap = P > 0.0 ? tot / P : -0.0;
        out_auroc[seg] = (float)auc;
        out_ap[seg] = (float)ap;
        out_counts[3 * seg + 0] = (long long)seg_totals[2 * seg + 0];
        out_counts[3 * seg + 1] = (long long)n - (long long)seg_totals[2 * seg + 0];
        out_counts[3 * seg + 2] = (long long)seg_totals[2 * seg + 1];
    }
}

// =====================================================================================================
// The scan as ONE chained kernel: tiles of 4096 take a ticket, compute their aggregates, publish them, resolve their carries
// by decoupled look-back over the earlier tiles of the segment and go straight on to the apply phase, so the sorted records
// are read once.
//
// Tile state = two 64-bit words, each [flag:2 | hi:31 | lo:31]:
//     sums  [npos | nbound]                           aggregate: of the tile          prefix: inclusive, from the segment start
//     last  [pos1 | tp]   last group end so far       aggregate: tile-local pos1 =    prefix: segment-global pos1 and TP;
//                          (pos1 = index + 1, 0 =      index+1 in the tile, TP local           pos1 = 0: no group end yet
//                          none; FP = pos1 - TP)
// A reader accepts a tile when both words carry the SAME non-zero flag: each word is written at most twice (aggregate, then
// prefix), so equal flags mean the same generation.  Warp 0 looks back 32 tiles per round trip.  TP at the last group end before
// the tile comes either from a prefix word (global already) or from the nearest aggregate that has one: then
// TP = (positives before THAT tile) + its local TP = (positives before this tile) - (positives from that tile up to here) + ...
// The spin is bounded (MB200_FLAG_SPIN_TIMEOUT instead of a hang).
// =====================================================================================================
constexpr int kChainThreads = 256;
constexpr int kChainItems = 16;
constexpr int kChainTile = kChainThreads * kChainItems;  // 4096
constexpr unsigned long long kChainAgg = 1ull << 62;
constexpr unsigned long long kChainPrefix = 2ull << 62;
constexpr unsigned long long kChainField = 0x7fffffffull;

__device__ __forceinline__ unsigned long long chain_word(unsigned long long flag, unsigned hi, unsigned lo) {
    return flag | ((unsigned long long)hi << 31) | (unsigned long long)lo;
}

__device__ __forceinline__ unsigned long long block_excl_sum64(unsigned long long v, unsigned long long* sm8,
                                                               unsigned long long& total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long t = __shfl_up_sync(kFull, incl, o);
        if (lane >= o) incl += t;
    }
    __syncthreads();
    if (lane == 31) sm8[warp] = incl;
    __syncthreads();
    unsigned long long woff = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < kChainThreads / 32; ++w) {
        const unsigned long long x = sm8[w];
        if (w < warp) woff += x;
        tot += x;
    }
    total = tot;
    return woff + incl - v;
}
__device__ __forceinline__ unsigned long long block_excl_max64(unsigned long long v, unsigned long long* sm8,
                                                               unsigned long long& total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long t = __shfl_up_sync(kFull, incl, o);
        if (lane >= o) incl = max(incl, t);
    }
    __syncthreads();
    if (lane == 31) sm8[warp] = incl;
    __syncthreads();
    unsigned long long wmax = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < kChainThreads / 32; ++w) {
        const unsigned long long x = sm8[w];
        if (w < warp) wmax = max(wmax, x);
        tot = max(tot, x);
    }
    total = tot;
    unsigned long long excl = __shfl_up_sync(kFull, incl, 1);
    if (lane == 0) excl = 0;
    return max(wmax, excl);
}

// tp / (tp + fp) in fp64 without the ~40-instruction IEEE division (it was a third of the scan at one group end per element):
// hardware reciprocal seed (2^-23) + two Newton steps -> relative error < 2^-50, the same instruction sequence everywhere
// (bitwise reproducible); the results leave the kernel as float32.
__device__ __forceinline__ double precision_at(unsigned tp, unsigned total) {
    const double x = (double)total;
    double r;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
    r = fma(r, fma(-x, r, 1.0), r);
    r = fma(r, fma(-x, r, 1.0), r);
    return (double)tp * r;
}

template <bool kWriteCurve, typename KeyT>
__global__ void __launch_bounds__(kChainThreads, sizeof(KeyT) == 4 ? 4 : 2) scan_chained_kernel(
    const KeyT* __restrict__ keys, const unsigned char* __restrict__ labels, int n_stride, const int* __restrict__ seg_ignored,
    int tiles, unsigned long long* status /*[segments*tiles][2], zeroed*/, unsigned* ticket /*zeroed*/,
    unsigned long long* __restrict__ auroc_acc /*[seg], zeroed*/, double* __restrict__ ap_partial /*[seg][tiles]*/,
    unsigned* __restrict__ seg_totals /*[seg][2]: P, U*/, float* __restrict__ fps_out, float* __restrict__ tps_out,
    typename ThrOf<KeyT>::type* __restrict__ thr_out, long long curve_stride, unsigned* __restrict__ err) {
    __shared__ unsigned long long sm8[kChainThreads / 32];
    __shared__ double dsum[kChainThreads / 32];
    __shared__ unsigned long long usum[kChainThreads / 32];
    __shared__ unsigned s_ticket;
    __shared__ unsigned s_carry[4];  // positives before the tile, group ends before it, TP / FP at the last group end before it
    if (threadIdx.x == 0) s_ticket = atomicAdd(ticket, 1u);
    __syncthreads();
    const unsigned tg = s_ticket;
    const int seg = (int)(tg / (unsigned)tiles), tile = (int)(tg % (unsigned)tiles);
    const int n = seg_ignored ? n_stride - seg_ignored[seg] : n_stride;  // ignored entries sit behind the valid ones
    const KeyT* __restrict__ k = keys + (size_t)seg * n_stride;
    const unsigned char* __restrict__ l = labels + (size_t)seg * n_stride;

    // ---- load: thread t owns elements [16 t, 16 t + 16) of the tile ----
    const int base = tile * kChainTile + threadIdx.x * kChainItems;
    const int count = max(0, min(kChainItems, n - base));
    // Decided on n, not as count == kChainItems: nvcc 12.9 for sm_90a folds that test into the min/max of count and took the
    // 16-wide path for partial chunks, which then summed the stale workspace bytes behind the segment as labels.
    const bool full = base + kChainItems <= n;
    KeyT key[kChainItems];
    unsigned labw[4];
    const bool aligned = ((reinterpret_cast<uintptr_t>(k + base) & 15) == 0) && ((reinterpret_cast<uintptr_t>(l + base) & 15) == 0);
    if (full && aligned) {
        if constexpr (sizeof(KeyT) == 4) {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const uint4 a = *reinterpret_cast<const uint4*>(k + base + 4 * q);
                key[4 * q] = a.x, key[4 * q + 1] = a.y, key[4 * q + 2] = a.z, key[4 * q + 3] = a.w;
            }
        } else {
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const ulonglong2 a = *reinterpret_cast<const ulonglong2*>(k + base + 2 * q);
                key[2 * q] = a.x, key[2 * q + 1] = a.y;
            }
        }
        const uint4 lb = *reinterpret_cast<const uint4*>(l + base);
        labw[0] = lb.x, labw[1] = lb.y, labw[2] = lb.z, labw[3] = lb.w;
    } else {
        labw[0] = labw[1] = labw[2] = labw[3] = 0u;
#pragma unroll
        for (int i = 0; i < kChainItems; ++i) {
            key[i] = i < count ? k[base + i] : (KeyT)0;
            if (i < count) labw[i >> 2] |= (unsigned)l[base + i] << (8 * (i & 3));
        }
    }
    const KeyT key_next = (full && base + kChainItems < n) ? k[base + kChainItems] : (KeyT)0;

    // ---- thread-local: positives, group ends, the thread's last group end ----
    unsigned npos = 0, nb = 0, ends = 0, cum_at_last = 0;
    int last_i = -1;
#pragma unroll
    for (int i = 0; i < kChainItems; ++i) {
        npos += (labw[i >> 2] >> (8 * (i & 3))) & 0xffu;
        bool e = false;
        if (i < count) {
            const KeyT nk = (i + 1 < kChainItems) ? key[i + 1] : key_next;
            e = (base + i == n - 1) || key[i] != nk || is_special_key(key[i]);  // NaN / +-inf: one group each
        }
        if (e) {
            ends |= 1u << i;
            nb++;
            last_i = i;
            cum_at_last = npos;
        }
    }
    unsigned long long tile_sums, tile_last;
    const unsigned long long excl = block_excl_sum64(((unsigned long long)npos << 32) | nb, sm8, tile_sums);
    const unsigned pos_excl_l = (unsigned)(excl >> 32), nb_excl_l = (unsigned)excl;
    const unsigned long long my_last =
        last_i >= 0 ? (((unsigned long long)(threadIdx.x * kChainItems + last_i + 1) << 32) | (pos_excl_l + cum_at_last)) : 0ull;
    const unsigned long long prev_last_l = block_excl_max64(my_last, sm8, tile_last);  // ends with a __syncthreads-free read of sm8

    // ---- publish, look back, publish the prefix (warp 0) ----
    if (threadIdx.x < 32) {
        const int lane = threadIdx.x;
        const unsigned t_npos = (unsigned)(tile_sums >> 32), t_nb = (unsigned)tile_sums;
        const unsigned t_pos1 = (unsigned)(tile_last >> 32), t_tp = (unsigned)tile_last;
        volatile unsigned long long* st = status + 2 * (size_t)tg;
        unsigned sp = 0, sb = 0, f_tp = 0, f_pos1 = 0;
        if (tile > 0) {
            if (lane == 0) {
                st[0] = chain_word(kChainAgg, t_npos, t_nb);
                st[1] = chain_word(kChainAgg, t_pos1, t_tp);
            }
            bool found = false, pending = false;
            unsigned p_tp_l = 0, p_pos1_g = 0, p_acc = 0;
            const long long seg_first = (long long)tg - tile;
            long long j = (long long)tg - 1;
            unsigned spins = 0;
            while (true) {
                const long long jj = j - lane;
                unsigned long long a = kChainPrefix, b = kChainPrefix;  // in front of the segment: an empty prefix
                if (jj >= seg_first) {
                    a = *(volatile unsigned long long*)(status + 2 * (size_t)jj);
                    b = *(volatile unsigned long long*)(status + 2 * (size_t)jj + 1);
                }
                const unsigned fa = (unsigned)(a >> 62), fb = (unsigned)(b >> 62);
                const unsigned ready = __ballot_sync(kFull, fa != 0u && fa == fb);
                const int first_not = __ffs(~ready) - 1;  // -1: all 32 ready
                const unsigned usable = first_not < 0 ? kFull : ((1u << first_not) - 1u);
                const unsigned pm = __ballot_sync(kFull, fa == 2u) & ready & usable;
                const int stop = __ffs(pm) - 1;  // nearest tile that holds a prefix (-1: none in the window)
                const unsigned consumed = stop >= 0 ? (stop == 31 ? kFull : ((1u << (stop + 1)) - 1u)) : usable;
                const bool in_c = (consumed >> lane) & 1u;
                const unsigned my_np = in_c ? (unsigned)((a >> 31) & kChainField) : 0u;
                const unsigned my_nb = in_c ? (unsigned)(a & kChainField) : 0u;
                unsigned incl_np = my_np;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const unsigned t = __shfl_up_sync(kFull, incl_np, o);
                    if (lane >= o) incl_np += t;
                }
                const unsigned tot_np = __shfl_sync(kFull, incl_np, 31);
                const unsigned tot_nb = __reduce_add_sync(kFull, my_nb);
                if (!found && !pending) {
                    const unsigned pos1 = (unsigned)((b >> 31) & kChainField), tpw = (unsigned)(b & kChainField);
                    const unsigned hb = __ballot_sync(kFull, in_c && pos1 != 0u);
                    if (hb) {
                        const int ls = __ffs(hb) - 1;  // the nearest tile with a group end
                        const bool is_prefix = __shfl_sync(kFull, fa, ls) == 2u;
                        const unsigned tp_s = __shfl_sync(kFull, tpw, ls), pos_s = __shfl_sync(kFull, pos1, ls);
                        const unsigned acc_s = __shfl_sync(kFull, incl_np, ls);
                        if (is_prefix) {
                            found = true, f_tp = tp_s, f_pos1 = pos_s;
                        } else {
                            pending = true, p_tp_l = tp_s;
                            p_pos1_g = (unsigned)(j - ls - seg_first) * (unsigned)kChainTile + pos_s;
                            p_acc = sp + acc_s;  // positives from that tile (inclusive) up to this one (exclusive)
                        }
                    }
                }
                sp += tot_np;
                sb += tot_nb;
                if (stop >= 0) break;
                const int adv = __popc(consumed);
                j -= adv;
                if (adv < 32) {  // ran into a tile that has not published yet
                    if (++spins > (1u << 22)) {
                        if (lane == 0 && err) atomicOr(err, MB200_FLAG_SPIN_TIMEOUT);
                        break;
                    }
                    __nanosleep(20);
                }
            }
            if (pending) f_tp = sp - p_acc + p_tp_l, f_pos1 = p_pos1_g;
        }
        if (lane == 0) {
            const unsigned g_pos1 = t_pos1 ? (unsigned)tile * (unsigned)kChainTile + t_pos1 : f_pos1;
            const unsigned g_tp = t_pos1 ? sp + t_tp : f_tp;
            st[0] = chain_word(kChainPrefix, sp + t_npos, sb + t_nb);
            st[1] = chain_word(kChainPrefix, g_pos1, g_tp);
            s_carry[0] = sp, s_carry[1] = sb, s_carry[2] = f_tp, s_carry[3] = f_pos1 - f_tp;
            if (tile == tiles - 1) seg_totals[2 * seg + 0] = sp + t_npos, seg_totals[2 * seg + 1] = sb + t_nb;
        }
    }
    __syncthreads();

    // ---- apply ----
    const unsigned c_pos = s_carry[0], c_nb = s_carry[1];
    unsigned tp_prev = s_carry[2], fp_prev = s_carry[3];
    if (prev_last_l) {  // a group end earlier in this tile
        tp_prev = c_pos + (unsigned)prev_last_l;
        fp_prev = (unsigned)tile * (unsigned)kChainTile + (unsigned)(prev_last_l >> 32) - tp_prev;
    }
    unsigned long long s_auc = 0;
    double s_ap = 0.0;
    unsigned run = c_pos + pos_excl_l, bi = c_nb + nb_excl_l;
#pragma unroll
    for (int i = 0; i < kChainItems; ++i) {
        run += (labw[i >> 2] >> (8 * (i & 3))) & 0xffu;
        if ((ends >> i) & 1u) {
            const unsigned tp = run;
            const unsigned fp = (unsigned)(base + i) + 1u - tp;
            s_auc += (unsigned long long)(fp - fp_prev) * (unsigned long long)(tp_prev + tp);
            if (tp != tp_prev) s_ap += (double)(tp - tp_prev) * precision_at(tp, tp + fp);
            if (kWriteCurve) {
                const long long o = (long long)seg * curve_stride + bi;
                fps_out[o] = (float)fp;
                tps_out[o] = (float)tp;
                thr_out[o] = score_of_key(key[i]);
            }
            tp_prev = tp;
            fp_prev = fp;
            bi++;
        }
    }
    // block reductions in a fixed order (deterministic fp64 result)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s_auc += __shfl_down_sync(kFull, s_auc, o);
        s_ap += __shfl_down_sync(kFull, s_ap, o);
    }
    if (lane == 0) usum[warp] = s_auc, dsum[warp] = s_ap;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long a = 0;
        double p = 0.0;
#pragma unroll
        for (int w = 0; w < kChainThreads / 32; ++w) a += usum[w], p += dsum[w];
        if (a) atomicAdd(auroc_acc + seg, a);  // integer: order-independent, exact
        ap_partial[(size_t)seg * tiles + tile] = p;
    }
}

// =====================================================================================================
// weighted `_binary_clf_curve` (sample_weights; functional/classification/precision_recall_curve.py:64, 73-78):
// keys sorted with the sample INDEX as payload, then one CTA walks the sorted order in chunks and emits, at every
// distinct score, tps = cumsum(w * [t == pos]) and fps = cumsum(w * [t != pos]) accumulated in fp64 in a fixed order.
// A private-API path of the reference (no public functional passes weights): built for exactness, not for speed.
// =====================================================================================================
template <typename T>
__global__ void __launch_bounds__(256) pack_indexed_kernel(const T* __restrict__ preds, const void* __restrict__ target,
                                                           int tdtype, long long pos_label, long long n,
                                                           typename KeyOf<T>::type* __restrict__ keys,
                                                           unsigned* __restrict__ idx) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        keys[i] = label_key(KeyOf<T>::make(preds[i]), load_label(target, tdtype, i) == pos_label);
        idx[i] = (unsigned)i;
    }
}

constexpr int kWThreads = 1024;
template <typename KeyT>
__global__ void __launch_bounds__(kWThreads) weighted_curve_kernel(const KeyT* __restrict__ keys,
                                                                   const unsigned* __restrict__ idx,
                                                                   const void* __restrict__ target, int tdtype,
                                                                   const double* __restrict__ weights, long long pos_label,
                                                                   int n, double* __restrict__ fps_out,
                                                                   double* __restrict__ tps_out,
                                                                   typename ThrOf<KeyT>::type* __restrict__ thr_out,
                                                                   long long* __restrict__ count_out) {
    __shared__ double wsum[2][kWThreads / 32];
    __shared__ unsigned wcnt[kWThreads / 32];
    __shared__ double carry_p, carry_n;
    __shared__ unsigned carry_b;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) carry_p = 0.0, carry_n = 0.0, carry_b = 0u;
    __syncthreads();
    for (int base = 0; base < n; base += kWThreads) {
        const int i = base + threadIdx.x;
        double wp = 0.0, wn = 0.0;
        unsigned end = 0u;
        KeyT k = 0;
        if (i < n) {
            k = keys[i];
            const unsigned src = idx[i];
            const double w = weights[src];
            const bool pos = load_label(target, tdtype, src) == pos_label;
            wp = pos ? w : 0.0;
            wn = pos ? 0.0 : w;
            end = (i == n - 1 || keys[i + 1] != k || is_special_key(k)) ? 1u : 0u;
        }
        // inclusive block scans of (wp, wn, end) in a fixed order
        double ip = wp, in_ = wn;
        unsigned ib = end;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const double tp = __shfl_up_sync(kFull, ip, o), tn = __shfl_up_sync(kFull, in_, o);
            const unsigned tb = __shfl_up_sync(kFull, ib, o);
            if (lane >= o) ip += tp, in_ += tn, ib += tb;
        }
        if (lane == 31) wsum[0][warp] = ip, wsum[1][warp] = in_, wcnt[warp] = ib;
        __syncthreads();
        double op = carry_p, on = carry_n;
        unsigned ob = carry_b;
        for (int w = 0; w < warp; ++w) op += wsum[0][w], on += wsum[1][w], ob += wcnt[w];
        ip += op, in_ += on, ib += ob;
        if (end) {
            const unsigned o = ib - 1u;
            tps_out[o] = ip;
            fps_out[o] = in_;
            thr_out[o] = score_of_key(k);
        }
        __syncthreads();
        if (threadIdx.x == kWThreads - 1) carry_p = ip, carry_n = in_, carry_b = ib;
        __syncthreads();
    }
    if (threadIdx.x == 0) *count_out = (long long)carry_b;
}

static inline int blocks_for(long long n, int per_block, int cap) {
    long long b = (n + per_block - 1) / per_block;
    if (b < 1) b = 1;
    if (b > cap) b = cap;
    return (int)b;
}

}  // namespace mb200

using namespace mb200;

// =====================================================================================================
// C-ABI
// =====================================================================================================
extern "C" int mb200_curve_sigmoid_if_logits(const void* preds, int dtype, int64_t n, void* out, uint32_t* flag_scratch,
                                             void* stream) {
    MB200_REQUIRE(n >= 0, "negative n");
    if (n == 0) return 0;
    MB200_REQUIRE(preds && out && flag_scratch, "NULL pointer");
    MB200_REQUIRE(is_float_tag(dtype), "scores must be floating point (dtype tag %d)", dtype);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    return with_float_type(dtype, [&](auto t) {
        using T = typename decltype(t)::type;
        constexpr int kItems = std::is_same_v<T, double> ? kSmallItemsF64 : kSmallItems;
        if (n <= 1024 * kItems) {
            sigmoid_if_small_kernel<T, kItems><<<1, 1024, 0, st>>>((const T*)preds, (T*)out, (int)n);
            count_launch();
            return check_cuda(cudaGetLastError(), "curve format launch");
        }
        MB200_CUDA_OK(cudaMemsetAsync(flag_scratch, 0, sizeof(uint32_t), st));
        const int grid = blocks_for(n, 256 * 8, sm_count() * 8);
        range_flag_kernel<T><<<grid, 256, 0, st>>>(reinterpret_cast<const T*>(preds), n, flag_scratch);
        sigmoid_if_kernel<T><<<grid, 256, 0, st>>>(reinterpret_cast<const T*>(preds), reinterpret_cast<T*>(out), n, flag_scratch);
        count_launch();
        count_launch();
        return check_cuda(cudaGetLastError(), "curve format launch");
    });
}

extern "C" int mb200_curve_softmax_if_logits(const void* preds, int dtype, int64_t n, int64_t num_classes, void* out,
                                             uint32_t* flag_scratch, void* stream) {
    MB200_REQUIRE(n >= 0 && num_classes >= 1, "bad sizes");
    if (n == 0) return 0;
    MB200_REQUIRE(preds && out && flag_scratch, "NULL pointer");
    MB200_REQUIRE(n < (1ll << 31) && num_classes < (1ll << 31), "sizes exceed int32");
    MB200_REQUIRE(is_float_tag(dtype), "softmax scores must be f32/f16/bf16/f64 (dtype tag %d)", dtype);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    MB200_CUDA_OK(cudaMemsetAsync(flag_scratch, 0, sizeof(uint32_t), st));
    const long long total = n * num_classes;
    const int grid = blocks_for(total, 256 * 8, sm_count() * 8);
    const int grid_rows = blocks_for(n, 8, sm_count() * 8);
    with_float_type(dtype, [&](auto t) {
        using T = typename decltype(t)::type;
        range_flag_kernel<T><<<grid, 256, 0, st>>>(reinterpret_cast<const T*>(preds), total, flag_scratch);
        softmax_if_kernel<T><<<grid_rows, 256, 0, st>>>(reinterpret_cast<const T*>(preds), reinterpret_cast<T*>(out), (int)n,
                                                        (int)num_classes, flag_scratch);
        return 0;
    });
    count_launch();
    count_launch();
    return check_cuda(cudaGetLastError(), "curve softmax launch");
}

static int64_t curve_workspace_bytes(int64_t segments, int64_t n, int key_bytes) {
    if (segments < 1 || n < 0) return -1;
    const int64_t scan_tiles = (n + kChainTile - 1) / kChainTile;
    int64_t b = 0;
    b += segments * n * key_bytes + 256;            // keys ping
    b += segments * n * key_bytes + 256;            // keys pong
    b += segments * n * 1 + 16;                     // labels ping
    b += segments * n * 1 + 16;                     // labels pong
    b += (int64_t)radix_sort_scratch_words(n, segments, key_bytes) * 4 + 256;  // digit histograms, look-back status, tickets
    b += segments * (scan_tiles + 1) * 16 + 256;    // chained-scan tile states + ticket
    b += segments * 2 * 4;                          // seg_totals
    b += segments * 4 + 256;                        // seg_ignored (multilabel + ignore_index)
    b += segments * 8;                              // auroc_acc
    b += segments * (scan_tiles + 1) * 8;           // ap_partial
    return b + 16 * 256;                            // alignment slack
}
extern "C" int64_t mb200_curve_workspace_bytes(int64_t segments, int64_t n) { return curve_workspace_bytes(segments, n, 4); }
extern "C" int64_t mb200_curve_workspace_bytes_for(int64_t segments, int64_t n, int preds_dtype) {
    return curve_workspace_bytes(segments, n, preds_dtype == MB200_F64 ? 8 : 4);
}

namespace {
template <typename KeyT>
struct CurveWs {
    KeyT *keys_a, *keys_b;
    unsigned char *lab_a, *lab_b;
    unsigned *sort_scratch, *seg_totals;
    int* seg_ignored;
    unsigned long long* chain;  // chained-scan tile states [segments * tiles][2], then the ticket
    unsigned long long* auroc_acc;
    double* ap_partial;
};
inline unsigned char* bump(unsigned char*& p, int64_t bytes) {
    unsigned char* r = p;
    p += (bytes + 255) / 256 * 256;
    return r;
}
template <typename KeyT>
CurveWs<KeyT> carve(void* workspace, int64_t segments, int64_t n) {
    const int64_t scan_tiles = (n + kChainTile - 1) / kChainTile;
    unsigned char* p = reinterpret_cast<unsigned char*>(workspace);
    CurveWs<KeyT> w;
    w.keys_a = (KeyT*)bump(p, segments * n * (int64_t)sizeof(KeyT));
    w.keys_b = (KeyT*)bump(p, segments * n * (int64_t)sizeof(KeyT));
    w.lab_a = bump(p, segments * n + 16);
    w.lab_b = bump(p, segments * n + 16);
    w.sort_scratch = (unsigned*)bump(p, (int64_t)radix_sort_scratch_words(n, segments, (int)sizeof(KeyT)) * 4);
    w.chain = (unsigned long long*)bump(p, segments * (scan_tiles + 1) * 16 + 256);
    w.seg_totals = (unsigned*)bump(p, segments * 2 * 4);
    w.seg_ignored = (int*)bump(p, segments * 4);
    w.auroc_acc = (unsigned long long*)bump(p, segments * 8);
    w.ap_partial = (double*)bump(p, segments * (scan_tiles + 1) * 8);
    return w;
}

// sort (keys_a/lab_a are clobbered; the sorted result lands back in them) + tie-collapsing scan + finalize
template <typename KeyT>
int sort_and_scan(KeyT* keys_a, unsigned char* lab_a, const CurveWs<KeyT>& w, int ni, int64_t segments, int64_t n,
                  const int* seg_ignored, float* out_auroc, float* out_ap, int64_t* out_counts, float* fps_out, float* tps_out,
                  void* thr_out_v, uint32_t* err_flag, cudaStream_t st, bool bit0 = false, bool hist_done = false) {
    using ThrT = typename ThrOf<KeyT>::type;
    ThrT* thr_out = reinterpret_cast<ThrT*>(thr_out_v);
    // ---- one-sweep radix passes, one per key byte (ping-pong; an even number of passes leaves the result in *_a) ----
    // bit0: the keys carry the label in bit 0 — 4-byte records until the last pass, which splits them into (key, label)
    {
        const int where = bit0 ? radix_sort_passes_bit0<KeyT, unsigned char>(keys_a, lab_a, w.keys_b, w.lab_b, ni, (int)segments,
                                                                             (int)sizeof(KeyT), w.sort_scratch, err_flag, st, &count_launch,
                                                                             hist_done)
                               : radix_sort_passes<KeyT, unsigned char>(keys_a, lab_a, w.keys_b, w.lab_b, ni, (int)segments,
                                                                        (int)sizeof(KeyT), w.sort_scratch, err_flag, st, &count_launch);
        if (where < 0) return check_cuda(cudaGetLastError(), "radix sort");
    }
    KeyT* kin = keys_a;
    unsigned char* lin = lab_a;

    // ---- scan: one chained kernel (tile states + ticket live in the tile-info region), then the finalize ----
    const int chain_tiles = (ni + kChainTile - 1) / kChainTile;
    unsigned long long* status = w.chain;
    const size_t status_bytes = (size_t)segments * chain_tiles * 16;
    unsigned* ticket = reinterpret_cast<unsigned*>(reinterpret_cast<unsigned char*>(w.chain) + status_bytes);
    if (cudaMemsetAsync(w.chain, 0, status_bytes + 16, st) != cudaSuccess ||
        cudaMemsetAsync(w.auroc_acc, 0, (size_t)segments * 8, st) != cudaSuccess)
        return check_cuda(cudaGetLastError(), "curve scan memset");
    const unsigned sgrid = (unsigned)(segments * chain_tiles);
    if (fps_out)
        scan_chained_kernel<true, KeyT><<<sgrid, kChainThreads, 0, st>>>(kin, lin, ni, seg_ignored, chain_tiles, status, ticket,
                                                                         w.auroc_acc, w.ap_partial, w.seg_totals, fps_out, tps_out,
                                                                         thr_out, n, err_flag);
    else
        scan_chained_kernel<false, KeyT><<<sgrid, kChainThreads, 0, st>>>(kin, lin, ni, seg_ignored, chain_tiles, status, ticket,
                                                                          w.auroc_acc, w.ap_partial, w.seg_totals, nullptr, nullptr,
                                                                          nullptr, n, err_flag);
    if (chain_tiles > 256)
        scan_finalize_wide_kernel<<<(unsigned)segments, 256, 0, st>>>(w.auroc_acc, w.ap_partial, w.seg_totals, chain_tiles, ni,
                                                                      seg_ignored, out_auroc, out_ap,
                                                                      reinterpret_cast<long long*>(out_counts));
    else
        scan_finalize_kernel<<<(int)((segments + 7) / 8), 256, 0, st>>>(w.auroc_acc, w.ap_partial, w.seg_totals, chain_tiles,
                                                                        ni, seg_ignored, (int)segments, out_auroc, out_ap, reinterpret_cast<long long*>(out_counts));
    for (int i = 0; i < 2; ++i) count_launch();
    return check_cuda(cudaGetLastError(), "curve evaluate launch");
}

template <typename T>
int evaluate_typed(const void* preds, const void* target, int target_dtype, int64_t n, int64_t segments, int64_t pos_label,
                   void* workspace, float* out_auroc, float* out_ap, int64_t* out_counts, float* fps_out, float* tps_out,
                   void* thr_out, uint32_t* err_flag, cudaStream_t st, bool unit_range = false) {
    using KeyT = typename KeyOf<T>::type;
    CurveWs<KeyT> w = carve<KeyT>(workspace, segments, n);
    const int ni = (int)n;
    constexpr bool kCanBit0 = sizeof(KeyT) == 4;
    const bool bit0 = kCanBit0 && unit_range;
    bool hist_done = false;  // the pack kernel already counted the sort's digit histograms
    if (segments == 1) {
        const int grid = blocks_for(n, 256 * 4, sm_count() * 8);
        if constexpr (kCanBit0) {
            if (bit0) {
                if (radix_sort_zero_scratch(w.sort_scratch, ni, 1, 4, st)) return check_cuda(cudaGetLastError(), "sort scratch");
                if (target_dtype == MB200_I64)
                    pack_binary_kernel<T, true, true><<<grid, 256, 0, st>>>(reinterpret_cast<const T*>(preds), target, target_dtype,
                                                                            n, pos_label, w.keys_a, w.lab_a, err_flag, w.sort_scratch);
                else
                    pack_binary_kernel<T, true, false><<<grid, 256, 0, st>>>(reinterpret_cast<const T*>(preds), target, target_dtype,
                                                                             n, pos_label, w.keys_a, w.lab_a, err_flag, w.sort_scratch);
                hist_done = true;
            }
        }
        if (!bit0) {
            if (target_dtype == MB200_I64)
                pack_binary_kernel<T, false, true><<<grid, 256, 0, st>>>(reinterpret_cast<const T*>(preds), target, target_dtype, n,
                                                                         pos_label, w.keys_a, w.lab_a);
            else
                pack_binary_kernel<T><<<grid, 256, 0, st>>>(reinterpret_cast<const T*>(preds), target, target_dtype, n, pos_label,
                                                            w.keys_a, w.lab_a);
        }
    } else {
        const dim3 grid((unsigned)((ni + 31) / 32), (unsigned)((segments + 31) / 32));
        if constexpr (kCanBit0) {
            if (bit0)
                pack_ovr_kernel<T, true><<<grid, 256, 0, st>>>(reinterpret_cast<const T*>(preds), target, target_dtype, ni,
                                                               (int)segments, w.keys_a, w.lab_a, err_flag);
        }
        if (!bit0)
            pack_ovr_kernel<T><<<grid, 256, 0, st>>>(reinterpret_cast<const T*>(preds), target, target_dtype, ni, (int)segments,
                                                     w.keys_a, w.lab_a);
    }
    count_launch();
    return sort_and_scan<KeyT>(w.keys_a, w.lab_a, w, ni, segments, n, nullptr, out_auroc, out_ap, out_counts, fps_out, tps_out,
                               thr_out, err_flag, st, bit0, hist_done);
}

template <typename T>
int evaluate_multilabel_typed(const void* preds, const void* target, int target_dtype, int64_t n, int64_t num_labels,
                              int has_ignore, int64_t ignore_index, void* workspace, float* out_auroc, float* out_ap,
                              int64_t* out_counts, float* fps_out, float* tps_out, void* thr_out, uint32_t* err_flag,
                              cudaStream_t st) {
    using KeyT = typename KeyOf<T>::type;
    CurveWs<KeyT> w = carve<KeyT>(workspace, num_labels, n);
    const int ni = (int)n;
    if (has_ignore) MB200_CUDA_OK(cudaMemsetAsync(w.seg_ignored, 0, (size_t)num_labels * sizeof(int), st));
    const dim3 grid((unsigned)((ni + 31) / 32), (unsigned)((num_labels + 31) / 32));
    pack_multilabel_kernel<T><<<grid, 256, 0, st>>>(reinterpret_cast<const T*>(preds), target, target_dtype, ni, (int)num_labels,
                                                    has_ignore, label_ignore_index(ignore_index, target_dtype), w.keys_a,
                                                    w.lab_a, w.seg_ignored);
    count_launch();
    return sort_and_scan<KeyT>(w.keys_a, w.lab_a, w, ni, num_labels, n, has_ignore ? w.seg_ignored : nullptr, out_auroc, out_ap,
                               out_counts, fps_out, tps_out, thr_out, err_flag, st);
}
}  // namespace

// Exact-mode curve evaluation for `segments` one-vs-rest curves over `n` samples each.
//   preds  : binary (num_classes == 1): [n] scores.  multiclass: [n, num_classes] row-major scores.
//   target : [n] integer labels; positive for segment c is (target == c) (binary: target == pos_label).
//   out_auroc / out_ap : float32 [segments];  out_counts : int64 [segments][3] = {n_pos, n_neg, n_distinct_thresholds}
//   curve outputs (optional, all three or none): float32 [segments][n] each, valid prefix = n_distinct_thresholds.
static int curve_evaluate_impl(const void* preds, int preds_dtype, const void* target, int target_dtype,
                               int64_t n, int64_t num_classes, int64_t pos_label, void* workspace,
                               int64_t workspace_bytes, float* out_auroc, float* out_ap, int64_t* out_counts,
                               float* fps_out, float* tps_out, void* thr_out, uint32_t* err_flag, void* stream, bool unit_range) {
    MB200_REQUIRE(n >= 1, "curve evaluation needs at least one sample (got %lld)", (long long)n);
    MB200_REQUIRE(n < (1ll << 30), "more than 2^30-1 samples per curve are not supported");
    MB200_REQUIRE(num_classes >= 1, "bad num_classes");
    MB200_REQUIRE(preds && target && workspace && out_auroc && out_ap && out_counts, "NULL pointer");
    const int64_t segments = num_classes;
    MB200_REQUIRE(workspace_bytes >= mb200_curve_workspace_bytes_for(segments, n, preds_dtype), "workspace too small");
    MB200_REQUIRE((fps_out == nullptr) == (tps_out == nullptr) && (fps_out == nullptr) == (thr_out == nullptr),
                  "curve outputs must be given all together or not at all");
    MB200_REQUIRE(segments <= 65535, "at most 65535 curves per call");
    if (!is_float_tag(preds_dtype)) {
        set_error("scores must be f32/f16/bf16/f64 (dtype tag %d)", preds_dtype);
        return MB200_ERR_UNSUPPORTED;
    }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    return with_float_type(preds_dtype, [&](auto t) {
        return evaluate_typed<typename decltype(t)::type>(preds, target, target_dtype, n, segments, pos_label, workspace, out_auroc,
                                                          out_ap, out_counts, fps_out, tps_out, thr_out, err_flag, st, unit_range);
    });
}

extern "C" int mb200_curve_evaluate(const void* preds, int preds_dtype, const void* target, int target_dtype,
                                    int64_t n, int64_t num_classes, int64_t pos_label, void* workspace,
                                    int64_t workspace_bytes, float* out_auroc, float* out_ap, int64_t* out_counts,
                                    float* fps_out, float* tps_out, void* thr_out, uint32_t* err_flag, void* stream) {
    return curve_evaluate_impl(preds, preds_dtype, target, target_dtype, n, num_classes, pos_label, workspace, workspace_bytes,
                               out_auroc, out_ap, out_counts, fps_out, tps_out, thr_out, err_flag, stream, false);
}

// The same evaluation for scores PROMISED to be non-negative or NaN — in particular what normalize_logits_if_needed returns,
// i.e. every state of the curve metric classes.  Their sort keys need 31 bits, so the label rides in bit 0 and the radix
// passes move 4-byte keys only.  A negative score (-0 is fine) raises MB200_FLAG_PREDS_RANGE in err_flag (results invalid).
extern "C" int mb200_curve_evaluate_nonneg(const void* preds, int preds_dtype, const void* target, int target_dtype,
                                         int64_t n, int64_t num_classes, int64_t pos_label, void* workspace,
                                         int64_t workspace_bytes, float* out_auroc, float* out_ap, int64_t* out_counts,
                                         float* fps_out, float* tps_out, void* thr_out, uint32_t* err_flag, void* stream) {
    return curve_evaluate_impl(preds, preds_dtype, target, target_dtype, n, num_classes, pos_label, workspace, workspace_bytes,
                               out_auroc, out_ap, out_counts, fps_out, tps_out, thr_out, err_flag, stream, true);
}

// Exact-mode evaluation of `num_labels` independent binary curves (multilabel task).
//   preds / target : [n, num_labels] row-major; positives are target == 1; with has_ignore, entries whose target equals
//   ignore_index are dropped from THEIR label's curve only (reference: precision_recall_curve.py:822-834).
//   Outputs as in mb200_curve_evaluate; out_counts[l] = {n_pos, n_neg, n_distinct_thresholds} over the kept entries.
extern "C" int mb200_curve_evaluate_multilabel(const void* preds, int preds_dtype, const void* target, int target_dtype,
                                               int64_t n, int64_t num_labels, int has_ignore, int64_t ignore_index,
                                               void* workspace, int64_t workspace_bytes, float* out_auroc, float* out_ap,
                                               int64_t* out_counts, float* fps_out, float* tps_out, void* thr_out,
                                               uint32_t* err_flag, void* stream) {
    MB200_REQUIRE(n >= 1 && n < (1ll << 30), "curve evaluation needs 1 <= n < 2^30 samples (got %lld)", (long long)n);
    MB200_REQUIRE(num_labels >= 1 && num_labels <= 65535, "bad num_labels");
    MB200_REQUIRE(preds && target && workspace && out_auroc && out_ap && out_counts, "NULL pointer");
    MB200_REQUIRE(workspace_bytes >= mb200_curve_workspace_bytes_for(num_labels, n, preds_dtype), "workspace too small");
    MB200_REQUIRE((fps_out == nullptr) == (tps_out == nullptr) && (fps_out == nullptr) == (thr_out == nullptr),
                  "curve outputs must be given all together or not at all");
    if (!is_float_tag(preds_dtype)) {
        set_error("scores must be f32/f16/bf16/f64 (dtype tag %d)", preds_dtype);
        return MB200_ERR_UNSUPPORTED;
    }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    return with_float_type(preds_dtype, [&](auto t) {
        return evaluate_multilabel_typed<typename decltype(t)::type>(preds, target, target_dtype, n, num_labels, has_ignore,
                                                                     ignore_index, workspace, out_auroc, out_ap, out_counts,
                                                                     fps_out, tps_out, thr_out, err_flag, st);
    });
}

// Class-major keys of [n, num_classes] scores: keys_out [num_classes][n] (the packing step of mb200_curve_evaluate on
// its own; used by the class-sharded multi-GPU path, which exchanges key rows between ranks before sorting).
extern "C" int mb200_curve_pack_keys(const void* preds, int preds_dtype, int64_t n, int64_t num_classes,
                                     uint32_t* keys_out, void* stream) {
    MB200_REQUIRE(n >= 0 && num_classes >= 1 && n < (1ll << 30), "bad sizes");
    if (n == 0) return 0;
    MB200_REQUIRE(preds && keys_out, "NULL pointer");
    if (!is_float_tag<kNoF64>(preds_dtype)) {
        set_error("scores must be f32/f16/bf16 (dtype tag %d)", preds_dtype);
        return MB200_ERR_UNSUPPORTED;
    }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const dim3 grid((unsigned)((n + 31) / 32), (unsigned)((num_classes + 31) / 32));
    with_float_type<kNoF64>(preds_dtype, [&](auto t) {
        using T = typename decltype(t)::type;
        pack_keys_kernel<T><<<grid, 256, 0, st>>>((const T*)preds, (int)n, (int)num_classes, keys_out);
        return 0;
    });
    count_launch();
    return check_cuda(cudaGetLastError(), "curve pack keys launch");
}

// Sort + scan for `segments` curves whose keys are already packed: keys [segments][n] (clobbered: sorted in place),
// positives of curve s are the samples with target == first_class + s.  Outputs as in mb200_curve_evaluate.
extern "C" int mb200_curve_evaluate_keys(uint32_t* keys, const void* target, int target_dtype, int64_t n,
                                         int64_t segments, int64_t first_class, void* workspace, int64_t workspace_bytes,
                                         float* out_auroc, float* out_ap, int64_t* out_counts, uint32_t* err_flag,
                                         void* stream) {
    MB200_REQUIRE(n >= 1 && n < (1ll << 30) && segments >= 1 && segments <= 65535, "bad sizes");
    MB200_REQUIRE(keys && target && workspace && out_auroc && out_ap && out_counts, "NULL pointer");
    MB200_REQUIRE(workspace_bytes >= mb200_curve_workspace_bytes(segments, n), "workspace too small");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    CurveWs<unsigned> w = carve<unsigned>(workspace, segments, n);
    const long long total = n * segments;
    labels_from_target_kernel<<<blocks_for(total, 256 * 8, sm_count() * 8), 256, 0, st>>>(keys, target, target_dtype, (int)n,
                                                                                          (int)segments, first_class, w.lab_a);
    count_launch();
    return sort_and_scan<unsigned>(keys, w.lab_a, w, (int)n, segments, n, nullptr, out_auroc, out_ap, out_counts, nullptr, nullptr,
                                   nullptr, err_flag, st);
}

// mb200_curve_evaluate_keys for keys of non-negative (or NaN) scores — the class-sharded exchange of metric states: the label is
// folded into bit 0 of the key in place and the sort moves 4-byte records (see mb200_curve_evaluate_nonneg).
extern "C" int mb200_curve_evaluate_keys_nonneg(uint32_t* keys, const void* target, int target_dtype, int64_t n,
                                                int64_t segments, int64_t first_class, void* workspace, int64_t workspace_bytes,
                                                float* out_auroc, float* out_ap, int64_t* out_counts, uint32_t* err_flag,
                                                void* stream) {
    MB200_REQUIRE(n >= 1 && n < (1ll << 30) && segments >= 1 && segments <= 65535, "bad sizes");
    MB200_REQUIRE(keys && target && workspace && out_auroc && out_ap && out_counts, "NULL pointer");
    MB200_REQUIRE(workspace_bytes >= mb200_curve_workspace_bytes(segments, n), "workspace too small");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    CurveWs<unsigned> w = carve<unsigned>(workspace, segments, n);
    const long long total = n * segments;
    fold_labels_into_keys_kernel<<<blocks_for(total, 256 * 8, sm_count() * 8), 256, 0, st>>>(keys, target, target_dtype, (int)n,
                                                                                             (int)segments, first_class, err_flag);
    count_launch();
    return sort_and_scan<unsigned>(keys, w.lab_a, w, (int)n, segments, n, nullptr, out_auroc, out_ap, out_counts, nullptr, nullptr,
                                   nullptr, err_flag, st, true);
}

namespace {
template <typename T>
int weighted_typed(const void* preds, const void* target, int target_dtype, const double* weights, int64_t n,
                   int64_t pos_label, void* workspace, double* fps_out, double* tps_out, void* thr_out, int64_t* count_out,
                   uint32_t* err_flag, cudaStream_t st) {
    using KeyT = typename KeyOf<T>::type;
    unsigned char* p = reinterpret_cast<unsigned char*>(workspace);
    KeyT* keys_a = (KeyT*)bump(p, n * (int64_t)sizeof(KeyT));
    KeyT* keys_b = (KeyT*)bump(p, n * (int64_t)sizeof(KeyT));
    unsigned* idx_a = (unsigned*)bump(p, n * 4);
    unsigned* idx_b = (unsigned*)bump(p, n * 4);
    unsigned* scratch = (unsigned*)bump(p, (int64_t)radix_sort_scratch_words(n, 1, (int)sizeof(KeyT)) * 4);
    pack_indexed_kernel<T><<<blocks_for(n, 256 * 4, sm_count() * 8), 256, 0, st>>>(reinterpret_cast<const T*>(preds), target,
                                                                                  target_dtype, (long long)pos_label, n, keys_a,
                                                                                  idx_a);
    count_launch();
    const int where = radix_sort_passes<KeyT, unsigned>(keys_a, idx_a, keys_b, idx_b, (int)n, 1, (int)sizeof(KeyT), scratch,
                                                        err_flag, st, &count_launch);
    if (where < 0) return check_cuda(cudaGetLastError(), "radix sort");
    weighted_curve_kernel<KeyT><<<1, kWThreads, 0, st>>>(keys_a, idx_a, target, target_dtype, weights, (long long)pos_label,
                                                         (int)n, fps_out, tps_out,
                                                         reinterpret_cast<typename ThrOf<KeyT>::type*>(thr_out),
                                                         reinterpret_cast<long long*>(count_out));
    count_launch();
    return check_cuda(cudaGetLastError(), "weighted curve launch");
}
}  // namespace

extern "C" int64_t mb200_curve_weighted_workspace_bytes(int64_t n, int preds_dtype) {
    if (n < 0) return -1;
    const int kb = preds_dtype == MB200_F64 ? 8 : 4;
    return 2 * (n * kb + 256) + 2 * (n * 4 + 256) + (int64_t)radix_sort_scratch_words(n, 1, kb) * 4 + 8 * 256;
}

extern "C" int mb200_curve_weighted_clf_curve(const void* preds, int preds_dtype, const void* target, int target_dtype,
                                              const double* weights, int64_t n, int64_t pos_label, void* workspace,
                                              int64_t workspace_bytes, double* fps_out, double* tps_out, void* thr_out,
                                              int64_t* count_out, uint32_t* err_flag, void* stream) {
    MB200_REQUIRE(n >= 1 && n < (1ll << 30), "curve evaluation needs 1 <= n < 2^30 samples (got %lld)", (long long)n);
    MB200_REQUIRE(preds && target && weights && workspace && fps_out && tps_out && thr_out && count_out, "NULL pointer");
    MB200_REQUIRE(workspace_bytes >= mb200_curve_weighted_workspace_bytes(n, preds_dtype), "workspace too small");
    if (!is_float_tag(preds_dtype)) {
        set_error("scores must be f32/f16/bf16/f64 (dtype tag %d)", preds_dtype);
        return MB200_ERR_UNSUPPORTED;
    }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    return with_float_type(preds_dtype, [&](auto t) {
        return weighted_typed<typename decltype(t)::type>(preds, target, target_dtype, weights, n, pos_label, workspace, fps_out,
                                                          tps_out, thr_out, count_out, err_flag, st);
    });
}

extern "C" int64_t mb200_curve_normalize_scratch_bytes(int64_t n) {
    if (n < 0) return -1;
    return 8 + (n / 1024 + 2);  // vote word + one byte per 16 KB tile (tiles hold >= 1024 elements)
}

// The vote word of the original kernels inside a caller-owned scratch: its first 4-byte aligned word (the word is the
// target of atomicOr, which needs natural alignment), or NULL (an error) when the scratch holds no such word.
static uint32_t* vote_word(void* scratch, int64_t scratch_bytes) {
    const uintptr_t a = (reinterpret_cast<uintptr_t>(scratch) + 3) & ~uintptr_t(3);
    return (int64_t)(a - reinterpret_cast<uintptr_t>(scratch)) + 4 <= scratch_bytes ? reinterpret_cast<uint32_t*>(a) : nullptr;
}

// mb200_curve_sigmoid_if_logits with a caller-owned scratch of mb200_curve_normalize_scratch_bytes(n): large aligned
// f32 / f16 / bf16 batches then take the speculative single pass (one read + one write); everything else the original path.
extern "C" int mb200_curve_sigmoid_if_logits_scratch(const void* preds, int dtype, int64_t n, void* out, void* scratch,
                                                     int64_t scratch_bytes, void* stream) {
    MB200_REQUIRE(n >= 0, "negative n");
    if (n == 0) return 0;
    MB200_REQUIRE(preds && out && scratch, "NULL pointer");
    MB200_REQUIRE(scratch_bytes >= mb200_curve_normalize_scratch_bytes(n), "scratch too small");
    const bool spec = dtype != MB200_F64 && n > 1024 * kSmallItems &&
                      ((reinterpret_cast<uintptr_t>(preds) | reinterpret_cast<uintptr_t>(out)) & 15) == 0 &&
                      (reinterpret_cast<uintptr_t>(scratch) & 3) == 0;
    if (!spec) return mb200_curve_sigmoid_if_logits(preds, dtype, n, out, vote_word(scratch, scratch_bytes), stream);
    MB200_REQUIRE(is_float_tag<kNoF64>(dtype), "scores must be floating point (dtype tag %d)", dtype);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int esize = dtype == MB200_F32 ? 4 : 2;
    const long long kvec = 16 / esize;
    const long long nvec = n / kvec;
    const long long ntiles = (nvec + kSpecTileVecs - 1) / kSpecTileVecs + (nvec % kSpecTileVecs == 0 && n % kvec ? 1 : 0);
    MB200_CUDA_OK(cudaMemsetAsync(scratch, 0, (size_t)(8 + ntiles), st));
    unsigned* vote = reinterpret_cast<unsigned*>(scratch);
    unsigned char* pending = reinterpret_cast<unsigned char*>(scratch) + 8;
    long long grid = ntiles;
    const long long cap = (long long)sm_count() * 8;
    if (grid > cap) grid = cap;
    with_float_type<kNoF64>(dtype, [&](auto t) {
        using T = typename decltype(t)::type;
        sigmoid_spec_kernel<T, false><<<(unsigned)grid, 256, 0, st>>>(reinterpret_cast<const T*>(preds), reinterpret_cast<T*>(out),
                                                                     n, vote, pending, ntiles);
        sigmoid_spec_kernel<T, true><<<(unsigned)grid, 256, 0, st>>>(reinterpret_cast<const T*>(preds), reinterpret_cast<T*>(out),
                                                                    n, vote, pending, ntiles);
        return 0;
    });
    count_launch();
    count_launch();
    return check_cuda(cudaGetLastError(), "curve format launch");
}

// mb200_curve_softmax_if_logits with a caller-owned scratch of 8 + n bytes (vote word + one pending byte per row): rows of at
// most 1024 f32 / f16 / bf16 scores take the speculative single pass above; everything else the original kernels.
extern "C" int mb200_curve_softmax_if_logits_scratch(const void* preds, int dtype, int64_t n, int64_t num_classes, void* out,
                                                     void* scratch, int64_t scratch_bytes, void* stream) {
    MB200_REQUIRE(n >= 0 && num_classes >= 1, "bad sizes");
    if (n == 0) return 0;
    MB200_REQUIRE(preds && out && scratch, "NULL pointer");
    MB200_REQUIRE(n < (1ll << 31) && num_classes < (1ll << 31), "sizes exceed int32");
    const bool spec = dtype != MB200_F64 && num_classes <= 1024 && scratch_bytes >= 8 + n &&
                      (reinterpret_cast<uintptr_t>(scratch) & 3) == 0;
    if (!spec) return mb200_curve_softmax_if_logits(preds, dtype, n, num_classes, out, vote_word(scratch, scratch_bytes), stream);
    MB200_REQUIRE(is_float_tag<kNoF64>(dtype), "softmax scores must be f32/f16/bf16/f64 (dtype tag %d)", dtype);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    MB200_CUDA_OK(cudaMemsetAsync(scratch, 0, (size_t)(8 + n), st));
    unsigned* vote = reinterpret_cast<unsigned*>(scratch);
    unsigned char* pending = reinterpret_cast<unsigned char*>(scratch) + 8;
    const int grid = blocks_for(n, 8, sm_count() * 3);  // 3 resident CTAs per SM (<= 85 registers): one wave
    const int C = (int)num_classes;
    with_float_type<kNoF64>(dtype, [&](auto t) {
        using T = typename decltype(t)::type;
        const auto launch = [&](auto iter) {
            constexpr int kIter = decltype(iter)::value;
            softmax_spec_kernel<T, kIter, false><<<grid, 256, 0, st>>>(reinterpret_cast<const T*>(preds), reinterpret_cast<T*>(out),
                                                                       (int)n, C, vote, pending);
            softmax_spec_kernel<T, kIter, true><<<grid, 256, 0, st>>>(reinterpret_cast<const T*>(preds), reinterpret_cast<T*>(out),
                                                                      (int)n, C, vote, pending);
        };
        if (C <= 32) launch(std::integral_constant<int, 1>{});
        else if (C <= 64) launch(std::integral_constant<int, 2>{});
        else if (C <= 128) launch(std::integral_constant<int, 4>{});
        else if (C <= 256) launch(std::integral_constant<int, 8>{});
        else if (C <= 512) launch(std::integral_constant<int, 16>{});
        else launch(std::integral_constant<int, 32>{});
        return 0;
    });
    count_launch();
    count_launch();
    return check_cuda(cudaGetLastError(), "curve softmax launch");
}
