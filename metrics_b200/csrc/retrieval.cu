// K16 — retrieval metrics (MAP, MRR, Precision, Recall, HitRate, FallOut, R-Precision, NDCG, AUROC, precision-recall curve)
// on sm_90a.
//
// Reference replaced (src/torchmetrics/): retrieval/base.py:148-183 sorts by `indexes`, moves the group sizes to the host
// and runs a Python loop over the queries, each with its own topk / argsort, gathers and sums (functional/retrieval/*.py).
//
// Group sort (K16b): one u64 key per record, (index - min) << 32 | ~f32_order_key(score), the target as a float32 payload,
// sorted by the shared LSD radix sort (radix_sort.cuh) over 4 + bytes(max - min) passes.  LSD passes are stable, so ties in
// score keep their input order.  An index range of 2^32 or more sorts twice instead: by score key with the position as
// payload, then stably by the biased 64-bit index; the records are then gathered and the high word becomes the dense rank
// of the query.  Segment heads (high word differs from the predecessor) are counted per 4096-record tile, the tile counts
// scanned by one CTA, and every head writes its position to offsets[rank].
// Ideal order (K16c, NDCG only): a second sort of the same shape keyed by (segment key, descending target).
// Evaluation (K16d): a warp per query of up to kLongQuery records, a 512-thread CTA per longer one; the CTA queries are
// listed by the warp kernel and taken in a persistent loop.  Every group walks its query in chunks of one record per
// thread, with warp-shuffle scans, carries in registers and sums in float64 in a fixed order: deterministic.  NDCG's tie
// groups (equal score keys) may span chunks: a max-scan of head positions finds the run start, and the run's target sum and
// discount sum come from prefix differences.  AUROC (K16e) and the precision-recall curve (K16f) are further per-query
// bodies on the same scheduling; the curve's columns past each query's length are filled by a separate flat kernel.
#include <algorithm>

#include "common.cuh"
#include "radix_sort.cuh"
#include "../../include/metrics_b200_retrieval.h"

namespace mb200 {

extern void count_launch();

namespace {

constexpr int kThreads = 256;
constexpr int kTileItems = 16;
constexpr int kTile = kThreads * kTileItems;  // records per head-count tile
constexpr int kLongQuery = 1024;              // longer queries get a CTA
constexpr int kCtaThreads = 512;
constexpr int kScanThreads = 1024;

typedef unsigned long long u64;

__device__ __forceinline__ float load_target(const void* t, int dtype, long long i) {
    return dtype == MB200_F32 ? reinterpret_cast<const float*>(t)[i] : (float)reinterpret_cast<const long long*>(t)[i];
}
__device__ __forceinline__ unsigned score_key(float v) { return ~f32_order_key(v); }  // ascending sort = descending score

int bytes_of(u64 v) {
    int b = 0;
    while (v) ++b, v >>= 8;
    return b;
}

// ---- K16a: index range ------------------------------------------------------------------------------------------------
__global__ void range_init_kernel(long long* range) {
    range[0] = LLONG_MAX;
    range[1] = LLONG_MIN;
}

__global__ void __launch_bounds__(kThreads) range_kernel(const long long* __restrict__ idx, long long n, long long* range) {
    long long lo = LLONG_MAX, hi = LLONG_MIN;
    for (long long i = blockIdx.x * (long long)kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads) {
        const long long v = idx[i];
        lo = min(lo, v);
        hi = max(hi, v);
    }
    for (int o = 16; o; o >>= 1) {
        lo = min(lo, __shfl_xor_sync(kFull, lo, o));
        hi = max(hi, __shfl_xor_sync(kFull, hi, o));
    }
    if ((threadIdx.x & 31) == 0) {
        atomicMin(range, lo);
        atomicMax(range + 1, hi);
    }
}

// ---- K16b: packing -----------------------------------------------------------------------------------------------------
__global__ void pack_narrow_kernel(const long long* __restrict__ idx, const float* __restrict__ preds, const void* target,
                                   int tdtype, long long n, long long lo, u64* __restrict__ keys, unsigned* __restrict__ vals) {
    for (long long i = blockIdx.x * (long long)kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads) {
        keys[i] = ((u64)(idx[i] - lo) << 32) | score_key(preds[i]);
        vals[i] = __float_as_uint(load_target(target, tdtype, i));
    }
}

__global__ void pack_score_kernel(const float* __restrict__ preds, long long n, u64* __restrict__ keys, unsigned* __restrict__ vals) {
    for (long long i = blockIdx.x * (long long)kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads) {
        keys[i] = score_key(preds[i]);
        vals[i] = (unsigned)i;
    }
}

__global__ void pack_index_kernel(const long long* __restrict__ idx, const unsigned* __restrict__ perm, long long n, long long lo,
                                  u64* __restrict__ keys, unsigned* __restrict__ vals) {
    for (long long i = blockIdx.x * (long long)kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads) {
        const unsigned p = perm[i];
        keys[i] = (u64)idx[p] - (u64)lo;
        vals[i] = p;
    }
}

// ---- K16b: segment heads -> offsets --------------------------------------------------------------------------------------
__device__ __forceinline__ bool is_head(const u64* keys, long long i, int shift) {
    return i == 0 || (keys[i] >> shift) != (keys[i - 1] >> shift);
}

__global__ void __launch_bounds__(kThreads) head_count_kernel(const u64* __restrict__ keys, long long n, int shift,
                                                              unsigned* __restrict__ tile_count) {
    __shared__ unsigned warp_sum[kThreads / 32];
    const long long base = (long long)blockIdx.x * kTile;
    unsigned c = 0;
    for (int j = threadIdx.x; j < kTile; j += kThreads) {
        const long long i = base + j;
        if (i < n && is_head(keys, i, shift)) ++c;
    }
    for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(kFull, c, o);
    if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned s = 0;
        for (int w = 0; w < kThreads / 32; ++w) s += warp_sum[w];
        tile_count[blockIdx.x] = s;
    }
}

// one CTA: exclusive scan of the tile counts in place; info[0] = Q, offsets[Q] = n
__global__ void __launch_bounds__(kScanThreads) tile_scan_kernel(unsigned* __restrict__ tile_count, long long tiles, long long n,
                                                                 long long* __restrict__ offsets, long long* __restrict__ info) {
    __shared__ unsigned long long warp_sum[kScanThreads / 32];
    const long long per = (tiles + kScanThreads - 1) / kScanThreads;
    const long long b = threadIdx.x * per, e = min(tiles, b + per);
    unsigned long long s = 0;
    for (long long i = b; i < e; ++i) s += tile_count[i];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long incl = s;
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long t = __shfl_up_sync(kFull, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) warp_sum[warp] = incl;
    __syncthreads();
    unsigned long long run = incl - s;
    for (int w = 0; w < warp; ++w) run += warp_sum[w];
    for (long long i = b; i < e; ++i) {
        const unsigned c = tile_count[i];
        tile_count[i] = (unsigned)run;
        run += c;
    }
    if (threadIdx.x == kScanThreads - 1) {
        info[0] = (long long)run;
        offsets[run] = n;
    }
}

// Each thread owns kTileItems consecutive records of the tile; heads write their position to offsets[rank].  With `perm`
// (the two-sort path) the records are also gathered: keys_out = rank << 32 | score key, target as float32.
__global__ void __launch_bounds__(kThreads) head_write_kernel(const u64* __restrict__ keys, long long n, int shift,
                                                              const unsigned* __restrict__ tile_excl, long long* __restrict__ offsets,
                                                              const unsigned* __restrict__ perm, const float* __restrict__ preds,
                                                              const void* target, int tdtype, u64* __restrict__ keys_out,
                                                              float* __restrict__ tgt_out) {
    __shared__ unsigned warp_sum[kThreads / 32];
    const long long base = (long long)blockIdx.x * kTile + (long long)threadIdx.x * kTileItems;
    unsigned c = 0;
#pragma unroll
    for (int j = 0; j < kTileItems; ++j)
        if (base + j < n && is_head(keys, base + j, shift)) ++c;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned incl = c;
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned t = __shfl_up_sync(kFull, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) warp_sum[warp] = incl;
    __syncthreads();
    unsigned rank = tile_excl[blockIdx.x] + incl - c;
    for (int w = 0; w < warp; ++w) rank += warp_sum[w];
    // rank = number of heads before this thread's first record; the record's query is (heads up to and including it) - 1
#pragma unroll
    for (int j = 0; j < kTileItems; ++j) {
        const long long i = base + j;
        if (i >= n) break;
        if (is_head(keys, i, shift)) offsets[rank++] = i;
        if (perm) {
            const unsigned p = perm[i];
            keys_out[i] = ((u64)(rank - 1) << 32) | score_key(preds[p]);
            tgt_out[i] = load_target(target, tdtype, p);
        }
    }
}

// ---- K16c: ideal order ---------------------------------------------------------------------------------------------------
__global__ void pack_ideal_kernel(const u64* __restrict__ keys, const float* __restrict__ tgt, long long n, u64* __restrict__ out_keys,
                                  unsigned* __restrict__ out_vals) {
    for (long long i = blockIdx.x * (long long)kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads) {
        const float t = tgt[i];
        out_keys[i] = (keys[i] & 0xffffffff00000000ull) | score_key(t);
        out_vals[i] = __float_as_uint(t);
    }
}

// ---- K16d: evaluation --------------------------------------------------------------------------------------------------
template <int G>
struct GroupSmem {
    double s[G];  // exclusive target prefix at each rank of the chunk (NDCG)
    double d[G];  // exclusive discount prefix
    double wtmp[G / 32 > 0 ? G / 32 : 1];
    double slot;
};

// G threads working on one query: one warp (G = 32) or the whole CTA.  Scans and reductions combine in a fixed order.
template <int G>
struct Group {
    int r;  // rank in the group
    GroupSmem<G>* sm;
    __device__ __forceinline__ void bar() const {
        if (G == 32)
            __syncwarp();
        else
            __syncthreads();
    }
    template <typename T, typename Op>
    __device__ __forceinline__ T scan(T v, Op op) const {  // inclusive
        const int lane = r & 31, warp = r >> 5;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const T t = __shfl_up_sync(kFull, v, o);
            if (lane >= o) v = op(t, v);
        }
        if (G == 32) return v;
        T* tmp = reinterpret_cast<T*>(sm->wtmp);
        if (lane == 31) tmp[warp] = v;
        bar();
        if (warp > 0) {
            T pre = tmp[0];
            for (int w = 1; w < warp; ++w) pre = op(pre, tmp[w]);
            v = op(pre, v);
        }
        bar();
        return v;
    }
    template <typename T>
    __device__ __forceinline__ T last(T v) const {  // the value of rank G - 1, to every rank
        if (G == 32) return __shfl_sync(kFull, v, 31);
        T* slot = reinterpret_cast<T*>(&sm->slot);
        if (r == G - 1) *slot = v;
        bar();
        const T out = *slot;
        bar();
        return out;
    }
    template <typename T>
    __device__ __forceinline__ T sum(T v) const {
        return last(scan(v, [](T a, T b) { return a + b; }));
    }
    template <typename T>
    __device__ __forceinline__ T smax(T v) const {
        return scan(v, [](T a, T b) { return a > b ? a : b; });
    }
};

__device__ __forceinline__ double discount(long long rank, long long k) { return rank < k ? 1.0 / log2((double)rank + 2.0) : 0.0; }

struct EvalArgs {
    const u64* keys;
    const float* tgt;
    const float* ideal;
    const long long* offsets;
    int kind;
    long long top_k;
    int adaptive_k;
    float* value;
    unsigned char* empty;
};

template <int G>
__device__ void eval_query(const EvalArgs& a, long long q, const Group<G>& g) {
    const long long s = a.offsets[q], n = a.offsets[q + 1] - s;
    const u64* keys = a.keys + s;
    const float* tgt = a.tgt + s;
    // totals: target sum and the number of NaN scores (they sort first)
    double tsum = 0.0;
    long long nans = 0;
    for (long long i = g.r; i < n; i += G) {
        tsum += (double)tgt[i];
        nans += (unsigned)keys[i] == 0u;
    }
    tsum = g.sum(tsum);
    nans = g.sum(nans);
    const long long kk = a.top_k == 0 ? n : min(a.top_k, n);
    double v = 0.0;
    switch (a.kind) {
        case MB200_RET_PRECISION:
        case MB200_RET_RECALL:
        case MB200_RET_HIT_RATE:
        case MB200_RET_FALL_OUT:
        case MB200_RET_R_PRECISION: {
            long long len = kk;  // records counted: the top min(k, n)
            double kp = (double)kk;
            if (a.kind == MB200_RET_PRECISION) {
                const long long k2 = (a.top_k == 0 || (a.adaptive_k && a.top_k > n)) ? n : a.top_k;
                len = min(k2, n);
                kp = (double)k2;
            }
            if (a.kind == MB200_RET_R_PRECISION) len = min(n, (long long)tsum);
            double top = 0.0;
            for (long long i = g.r; i < len; i += G) top += (double)tgt[i];
            top = g.sum(top);
            const double negs = (double)n - tsum;
            if (a.kind == MB200_RET_PRECISION) v = tsum == 0.0 ? 0.0 : top / kp;
            else if (a.kind == MB200_RET_RECALL) v = tsum == 0.0 ? 0.0 : top / tsum;
            else if (a.kind == MB200_RET_HIT_RATE) v = top > 0.0 ? 1.0 : 0.0;
            else if (a.kind == MB200_RET_FALL_OUT) v = negs == 0.0 ? 0.0 : ((double)len - top) / negs;
            else v = len == 0 ? 0.0 : top / (double)len;
            break;
        }
        case MB200_RET_AP: {
            long long carry = 0;
            double num = 0.0, top = 0.0;
            for (long long base = 0; base < kk; base += G) {
                const long long i = base + g.r;
                const float t = i < kk ? tgt[i] : 0.0f;
                const long long pos = t > 0.0f;
                const long long c = carry + g.scan(pos, [](long long x, long long y) { return x + y; });
                if (pos) num += (double)c / (double)(i + 1);
                top += (double)t;
                carry = g.last(c);
            }
            num = g.sum(num);
            top = g.sum(top);
            v = (top == 0.0 || carry == 0) ? 0.0 : num / (double)carry;
            break;
        }
        case MB200_RET_RR: {
            long long first = LLONG_MAX;
            for (long long i = g.r; i < kk; i += G)
                if (tgt[i] != 0.0f) {
                    first = i;
                    break;
                }
            first = g.last(g.scan(first, [](long long x, long long y) { return x < y ? x : y; }));
            v = first == LLONG_MAX ? 0.0 : 1.0 / (double)(first + 1);
            break;
        }
        case MB200_RET_NDCG: {
            double idcg = 0.0, dcg = 0.0;
            for (long long i = g.r; i < kk; i += G) idcg += (double)a.ideal[s + i] * discount(i, kk);
            // NaN scores: each its own tie group after every number, in input order (torch.unique(-preds))
            for (long long i = g.r; i < nans; i += G) dcg += (double)tgt[i] * discount(n - nans + i, kk);
            // numbers: tie groups of equal score keys, ranks from 0
            double sc = 0.0, dc = 0.0, head_s = 0.0, head_d = 0.0;
            long long head_pos = nans;
            for (long long base = nans; base < n; base += G) {
                const long long i = base + g.r;
                const bool valid = i < n;
                const double t = valid ? (double)tgt[i] : 0.0;
                const unsigned key = valid ? (unsigned)keys[i] : 0u;
                const double d = valid ? discount(i - nans, kk) : 0.0;
                const bool head = valid && (i == nans || (unsigned)keys[i - 1] != key);
                const bool end = valid && (i == n - 1 || (unsigned)keys[i + 1] != key);
                const double si = g.scan(t, [](double x, double y) { return x + y; });
                const double di = g.scan(d, [](double x, double y) { return x + y; });
                const double sx = sc + si - t, dx = dc + di - d;
                g.sm->s[g.r] = sx;
                g.sm->d[g.r] = dx;
                const int hp = g.smax(head ? g.r : -1);
                g.bar();
                if (end) {
                    double hs = head_s, hd = head_d;
                    long long a0 = head_pos;
                    if (hp >= 0) {
                        hs = g.sm->s[hp];
                        hd = g.sm->d[hp];
                        a0 = base + hp;
                    }
                    dcg += (sx + t - hs) * (dx + d - hd) / (double)(i - a0 + 1);
                }
                const int hl = g.last(hp);
                if (hl >= 0) {
                    head_s = g.sm->s[hl];
                    head_d = g.sm->d[hl];
                    head_pos = base + hl;
                }
                sc += g.last(si);
                dc += g.last(di);
                g.bar();
            }
            idcg = g.sum(idcg);
            dcg = g.sum(dcg);
            v = idcg == 0.0 ? 0.0 : dcg / idcg;
            break;
        }
        default: break;
    }
    if (g.r == 0) {
        a.value[q] = (float)v;
        a.empty[q] = a.kind == MB200_RET_FALL_OUT ? ((double)n - tsum == 0.0) : (tsum == 0.0);
    }
}

// The per-query bodies: `body(q, g)` evaluates query q with the G threads of g; `body.offsets` are the query offsets.
struct MetricBody {
    EvalArgs a;
    const long long* offsets;
    template <int G>
    __device__ __forceinline__ void operator()(long long q, const Group<G>& g) const {
        eval_query<G>(a, q, g);
    }
};

template <class Body>
__global__ void __launch_bounds__(kThreads) eval_warp_kernel(Body body, const long long* __restrict__ num_queries,
                                                             unsigned* __restrict__ long_list, unsigned* __restrict__ long_count) {
    __shared__ GroupSmem<32> sm[kThreads / 32];
    const int warp = threadIdx.x >> 5;
    Group<32> g{(int)(threadIdx.x & 31), &sm[warp]};
    const long long nq = *num_queries;
    const long long stride = (long long)gridDim.x * (kThreads / 32);
    for (long long q = (long long)blockIdx.x * (kThreads / 32) + warp; q < nq; q += stride) {
        if (body.offsets[q + 1] - body.offsets[q] > kLongQuery) {
            if (g.r == 0) long_list[atomicAdd(long_count, 1u)] = (unsigned)q;
            continue;
        }
        body(q, g);
    }
}

template <class Body>
__global__ void __launch_bounds__(kCtaThreads) eval_cta_kernel(Body body, const unsigned* __restrict__ long_list,
                                                               const unsigned* __restrict__ long_count) {
    __shared__ GroupSmem<kCtaThreads> sm;
    Group<kCtaThreads> g{(int)threadIdx.x, &sm};
    const unsigned count = *long_count;
    for (unsigned j = blockIdx.x; j < count; j += gridDim.x) body((long long)long_list[j], g);
}

// ---- K16e: AUROC of each query's top min(top_k, n) records ---------------------------------------------------------------
// restates retrieval_auroc -> binary_auroc: a slice without a target equal to 0 or without one equal to 1 scores 0; a
// positive is a target equal to 1; when any (non-NaN) score of the slice lies outside [0, 1] every score is replaced by its
// fp32 sigmoid before the tie groups (runs of equal values, each NaN its own group) are formed.  The full area is the exact
// integer sum_g fp_g * (2 TP_before + tp_g) over 2 P N.  The partial area stops at the first ROC point whose fp32 FPR
// exceeds max_fpr (rounded to fp32), interpolates TPR linearly there and takes McClish's standardisation.
struct AurocBody {
    const u64* keys;
    const float* tgt;
    const long long* offsets;
    long long top_k;
    double max_fpr;  // < 0: the full area
    float* value;
    unsigned char* empty;

    template <int G>
    __device__ void operator()(long long q, const Group<G>& g) const {
        const long long s = offsets[q], n = offsets[q + 1] - s;
        const u64* k = keys + s;
        const float* t = tgt + s;
        const long long len = top_k == 0 ? n : min(top_k, n);
        double tsum = 0.0;
        long long has0 = 0, has1 = 0, logit = 0;
        for (long long i = g.r; i < n; i += G) {
            const float ti = t[i];
            tsum += (double)ti;
            if (i < len) {
                const float v = f32_from_order_key(~(unsigned)k[i]);
                has0 |= ti == 0.0f;
                has1 |= ti == 1.0f;
                logit |= v < 0.0f || v > 1.0f;
            }
        }
        tsum = g.sum(tsum);
        has0 = g.sum(has0);
        has1 = g.sum(has1);
        logit = g.sum(logit);
        double v = 0.0;
        if (has0 && has1) {
            const bool sig = logit != 0;
            auto score = [k, sig](long long i) {
                const float x = f32_from_order_key(~(unsigned)k[i]);
                return sig ? sigmoid_f32(x) : x;
            };
            long long npos = 0;
            for (long long i = g.r; i < len; i += G) npos += t[i] == 1.0f;
            const long long P = g.sum(npos), N = len - P;
            const bool partial = max_fpr >= 0.0;
            const float m32 = (float)max_fpr;
            const float nf = (float)N;
            // area: exact sum of fp_g (2 TP_before + tp_g) over the groups that end at or before the crossing point
            unsigned long long area = 0;
            long long cfp0 = 0, cfp1 = 0, ctp0 = 0, ctp1 = 0;  // the crossing segment, held by the one rank that ends it
            long long carry = 0, head_tp = 0, head_pos = 0;
            double* sx = g.sm->s;
            for (long long base = 0; base < len; base += G) {
                const long long i = base + g.r;
                const bool valid = i < len;
                const float w = valid ? score(i) : 0.0f;
                const long long pos = valid && t[i] == 1.0f;
                const bool head = valid && (i == 0 || !(score(i - 1) == w));
                const bool end = valid && (i == len - 1 || !(score(i + 1) == w));
                const long long tp = carry + g.scan(pos, [](long long x, long long y) { return x + y; });
                sx[g.r] = (double)(tp - pos);  // exclusive TP count at this rank
                const int hp = g.smax(head ? g.r : -1);
                g.bar();
                if (end) {
                    long long tp0 = head_tp, a0 = head_pos;
                    if (hp >= 0) {
                        tp0 = (long long)sx[hp];
                        a0 = base + hp;
                    }
                    const long long fp0 = a0 - tp0, fp1 = i + 1 - tp;
                    const unsigned long long contrib = (unsigned long long)(fp1 - fp0) * (unsigned long long)(tp0 + tp);
                    if (!partial || (float)fp1 / nf <= m32) {
                        area += contrib;
                    } else if ((float)fp0 / nf <= m32) {  // the first ROC point past max_fpr
                        cfp0 = fp0, cfp1 = fp1, ctp0 = tp0, ctp1 = tp;
                    }
                }
                const int hl = g.last(hp);
                if (hl >= 0) {
                    head_tp = (long long)sx[hl];
                    head_pos = base + hl;
                }
                carry = g.last(tp);
                g.bar();
            }
            area = g.sum(area);
            const double full = (double)area / (2.0 * (double)P * (double)N);
            if (!partial) {
                v = full;
            } else {
                const double x0 = (double)g.sum(cfp0) / (double)N, x1 = (double)g.sum(cfp1) / (double)N;
                const double y0 = (double)g.sum(ctp0) / (double)P, y1 = (double)g.sum(ctp1) / (double)P;
                const double m = (double)m32, min_area = 0.5 * m * m;
                const double y = y0 + (m - x0) / (x1 - x0) * (y1 - y0);  // TPR interpolated at max_fpr
                v = 0.5 * (1.0 + (full + (m - x0) * (y0 + y) * 0.5 - min_area) / (m - min_area));
            }
        }
        if (g.r == 0) {
            value[q] = (float)v;
            empty[q] = tsum == 0.0;
        }
    }
};

// ---- K16f: precision / recall at k = 1..max_k of each query ---------------------------------------------------------------
// The per-query body writes the columns k <= min(n, max_k) (a scan of the query's head) and keeps P; the columns past n,
// where the cumulative count stays P, are written by pr_tail_kernel over the whole matrix so that short queries with a long
// max_k spread over every SM.  cum(k) / d and cum(k) / P are fp32 divisions of exact counts, as in the reference.
struct PrCurveBody {
    const float* tgt;
    const long long* offsets;
    long long max_k;
    float* precision;
    float* recall;
    unsigned char* empty;
    float* positives;  // [Q] scratch: P as float32, for the tail

    template <int G>
    __device__ void operator()(long long q, const Group<G>& g) const {
        const long long s = offsets[q], n = offsets[q + 1] - s;
        const float* t = tgt + s;
        double tsum = 0.0;
        for (long long i = g.r; i < n; i += G) tsum += (double)t[i];
        tsum = g.sum(tsum);
        const float pf = (float)tsum;
        const bool none = tsum == 0.0;
        float* prow = precision + q * max_k;
        float* rrow = recall + q * max_k;
        const long long len = min(n, max_k);
        double carry = 0.0;
        for (long long base = 0; base < len; base += G) {
            const long long i = base + g.r;
            const double ti = i < len ? (double)t[i] : 0.0;
            const double cum = carry + g.scan(ti, [](double x, double y) { return x + y; });
            if (i < len) {
                const float c = (float)cum;
                prow[i] = none ? 0.0f : c / (float)(i + 1);
                rrow[i] = none ? 0.0f : c / pf;
            }
            carry = g.last(cum);
        }
        if (g.r == 0) {
            positives[q] = pf;
            empty[q] = none;
        }
    }
};

// columns c >= n of every row, in blocks of kThreads columns: cum = P, d = k (adaptive_k: n)
__global__ void __launch_bounds__(kThreads) pr_tail_kernel(const long long* __restrict__ offsets, const long long* __restrict__ num_queries,
                                                           long long max_k, int adaptive_k, const float* __restrict__ positives,
                                                           float* __restrict__ precision, float* __restrict__ recall) {
    const long long col_blocks = (max_k + kThreads - 1) / kThreads;
    const long long units = *num_queries * col_blocks;
    for (long long u = blockIdx.x; u < units; u += gridDim.x) {
        const long long q = u / col_blocks;
        const long long c = (u - q * col_blocks) * kThreads + threadIdx.x;
        const long long n = offsets[q + 1] - offsets[q];
        if (c >= max_k || c < n) continue;
        const float pf = positives[q];
        const bool none = pf == 0.0f;
        const long long d = adaptive_k ? n : c + 1;
        precision[q * max_k + c] = none ? 0.0f : pf / (float)d;
        recall[q * max_k + c] = none ? 0.0f : pf / pf;
    }
}

int grid_for(long long n) { return (int)std::max(1ll, std::min((n + kThreads - 1) / kThreads, (long long)sm_count() * 16)); }

// Warp per query of up to kLongQuery records, listed CTA per longer one: one memset and two launches on `st`.
// scratch: the long-query count (16 bytes) then the list, mb200_retrieval_evaluate_scratch_bytes(n) bytes in all.
template <class Body>
int launch_per_query(const Body& body, const long long* num_queries, long long n, void* scratch, cudaStream_t st) {
    unsigned* long_count = reinterpret_cast<unsigned*>(scratch);
    unsigned* long_list = reinterpret_cast<unsigned*>(reinterpret_cast<unsigned char*>(scratch) + 16);
    MB200_CUDA_OK(cudaMemsetAsync(long_count, 0, 4, st));
    const int wgrid = (int)std::max(1ll, std::min((long long)(n + kThreads / 32 - 1) / (kThreads / 32), (long long)sm_count() * 16));
    eval_warp_kernel<Body><<<wgrid, kThreads, 0, st>>>(body, num_queries, long_list, long_count);
    count_launch();
    const int cgrid = (int)std::max(1ll, std::min((long long)n / kLongQuery, (long long)sm_count() * 2));
    eval_cta_kernel<Body><<<cgrid, kCtaThreads, 0, st>>>(body, long_list, long_count);
    count_launch();
    return 0;
}

size_t align16(size_t b) { return (b + 15) & ~(size_t)15; }

// workspace of the group sort: radix scratch | keys_b | vals_b | (two-sort path) keys_a | vals_a | tile counts
struct SortWs {
    unsigned* radix;
    u64* keys_b;
    unsigned* vals_b;
    u64* keys_a;
    unsigned* vals_a;
    unsigned* tiles;
    size_t bytes;
};
SortWs sort_ws(long long n, int index_bytes, unsigned char* base) {
    const bool wide = index_bytes > 4;
    const int key_bytes = wide ? 8 : 4 + index_bytes;
    SortWs w{};
    size_t off = 0;
    auto take = [&](size_t b) {
        unsigned char* p = base ? base + off : nullptr;
        off += align16(b);
        return p;
    };
    w.radix = reinterpret_cast<unsigned*>(take(radix_sort_scratch_words(n, 1, key_bytes) * 4));
    w.keys_b = reinterpret_cast<u64*>(take((size_t)n * 8));
    w.vals_b = reinterpret_cast<unsigned*>(take((size_t)n * 4));
    if (wide) {
        w.keys_a = reinterpret_cast<u64*>(take((size_t)n * 8));
        w.vals_a = reinterpret_cast<unsigned*>(take((size_t)n * 4));
    }
    w.tiles = reinterpret_cast<unsigned*>(take((size_t)((n + kTile - 1) / kTile + 1) * 4));
    w.bytes = off;
    return w;
}

int heads_to_offsets(const u64* keys, long long n, int shift, unsigned* tiles, long long* offsets, long long* info,
                     const unsigned* perm, const float* preds, const void* target, int tdtype, u64* keys_out, float* tgt_out,
                     cudaStream_t st) {
    const long long ntiles = (n + kTile - 1) / kTile;
    head_count_kernel<<<(unsigned)ntiles, kThreads, 0, st>>>(keys, n, shift, tiles);
    count_launch();
    tile_scan_kernel<<<1, kScanThreads, 0, st>>>(tiles, ntiles, n, offsets, info);
    count_launch();
    head_write_kernel<<<(unsigned)ntiles, kThreads, 0, st>>>(keys, n, shift, tiles, offsets, perm, preds, target, tdtype, keys_out,
                                                              tgt_out);
    count_launch();
    return check_cuda(cudaGetLastError(), "retrieval heads");
}

}  // namespace
}  // namespace mb200

using namespace mb200;

// =====================================================================================================
// C-ABI
// =====================================================================================================
extern "C" int mb200_retrieval_index_range(const int64_t* indexes, int64_t n, int64_t* range, void* stream) {
    MB200_REQUIRE(n >= 1 && n <= MB200_RET_MAX_ELEMENTS, "bad size %lld", (long long)n);
    MB200_REQUIRE(indexes && range, "NULL pointer");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    range_init_kernel<<<1, 1, 0, st>>>(reinterpret_cast<long long*>(range));
    count_launch();
    range_kernel<<<grid_for(n), kThreads, 0, st>>>(reinterpret_cast<const long long*>(indexes), n, reinterpret_cast<long long*>(range));
    count_launch();
    return check_cuda(cudaGetLastError(), "retrieval_index_range");
}

extern "C" int64_t mb200_retrieval_sort_scratch_bytes(int64_t n, int index_bytes) {
    if (n < 1 || n > MB200_RET_MAX_ELEMENTS || index_bytes < 0 || index_bytes > 8) return -1;
    return (int64_t)sort_ws(n, index_bytes, nullptr).bytes;
}

extern "C" int mb200_retrieval_sort(const int64_t* indexes, const float* preds, const void* target, int target_dtype, int64_t n,
                                    int64_t index_min, int64_t index_max, uint64_t* keys, float* sorted_target, int64_t* offsets,
                                    int64_t* info, void* scratch, int64_t scratch_bytes, void* stream) {
    MB200_REQUIRE((is_label_tag(target_dtype) && target_dtype == MB200_I64) || (is_float_tag(target_dtype) && target_dtype == MB200_F32),
                  "target must be int64 or float32 (dtype tag %d)", target_dtype);
    MB200_REQUIRE(n >= 1 && n <= MB200_RET_MAX_ELEMENTS, "retrieval inputs hold %lld elements; at most 2^30 - 1 are supported",
                  (long long)n);
    MB200_REQUIRE(index_max >= index_min, "index_max < index_min");
    MB200_REQUIRE(indexes && preds && target && keys && sorted_target && offsets && info, "NULL pointer");
    const u64 span = (u64)index_max - (u64)index_min;
    const int index_bytes = bytes_of(span);
    SortWs w = sort_ws(n, index_bytes, reinterpret_cast<unsigned char*>(scratch));
    MB200_REQUIRE(scratch && scratch_bytes >= (int64_t)w.bytes, "scratch too small (%lld < %lld bytes)", (long long)scratch_bytes,
                  (long long)w.bytes);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const long long* idx = reinterpret_cast<const long long*>(indexes);
    u64* kout = reinterpret_cast<u64*>(keys);
    unsigned* err = reinterpret_cast<unsigned*>(info + 1);
    const int grid = grid_for(n);
    if (index_bytes <= 4) {
        const int key_bytes = 4 + index_bytes;
        unsigned* vout = reinterpret_cast<unsigned*>(sorted_target);
        pack_narrow_kernel<<<grid, kThreads, 0, st>>>(idx, preds, target, target_dtype, n, index_min, kout, vout);
        count_launch();
        const int where = radix_sort_passes<u64, unsigned>(kout, vout, w.keys_b, w.vals_b, (int)n, 1, key_bytes, w.radix, err, st,
                                                           &count_launch);
        if (where < 0) return where;
        if (where == 1) {
            MB200_CUDA_OK(cudaMemcpyAsync(kout, w.keys_b, (size_t)n * 8, cudaMemcpyDeviceToDevice, st));
            MB200_CUDA_OK(cudaMemcpyAsync(vout, w.vals_b, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
        }
        return heads_to_offsets(kout, n, 32, w.tiles, reinterpret_cast<long long*>(offsets), reinterpret_cast<long long*>(info),
                                nullptr, nullptr, nullptr, 0, nullptr, nullptr, st);
    }
    // two sorts: by score (position payload), then stably by the biased index
    pack_score_kernel<<<grid, kThreads, 0, st>>>(preds, n, w.keys_a, w.vals_a);
    count_launch();
    int where = radix_sort_passes<u64, unsigned>(w.keys_a, w.vals_a, w.keys_b, w.vals_b, (int)n, 1, 4, w.radix, err, st, &count_launch);
    if (where < 0) return where;
    u64 *rk = where ? w.keys_b : w.keys_a, *ok = where ? w.keys_a : w.keys_b;
    unsigned *rv = where ? w.vals_b : w.vals_a, *ov = where ? w.vals_a : w.vals_b;
    pack_index_kernel<<<grid, kThreads, 0, st>>>(idx, rv, n, index_min, ok, ov);
    count_launch();
    where = radix_sort_passes<u64, unsigned>(ok, ov, rk, rv, (int)n, 1, index_bytes, w.radix, err, st, &count_launch);
    if (where < 0) return where;
    const u64* sk = where ? rk : ok;
    const unsigned* sv = where ? rv : ov;
    return heads_to_offsets(sk, n, 0, w.tiles, reinterpret_cast<long long*>(offsets), reinterpret_cast<long long*>(info), sv, preds,
                            target, target_dtype, kout, sorted_target, st);
}

extern "C" int64_t mb200_retrieval_ideal_scratch_bytes(int64_t n, int segment_bytes) {
    if (n < 1 || n > MB200_RET_MAX_ELEMENTS || segment_bytes < 0 || segment_bytes > 4) return -1;
    return (int64_t)(align16(radix_sort_scratch_words(n, 1, 4 + segment_bytes) * 4) + align16((size_t)n * 8) * 2 +
                     align16((size_t)n * 4));
}

extern "C" int mb200_retrieval_sort_ideal(const uint64_t* keys, const float* sorted_target, int64_t n, int segment_bytes,
                                          float* ideal, void* scratch, int64_t scratch_bytes, uint32_t* err_flag, void* stream) {
    const int64_t need = mb200_retrieval_ideal_scratch_bytes(n, segment_bytes);
    MB200_REQUIRE(need > 0, "bad size %lld or segment_bytes %d", (long long)n, segment_bytes);
    MB200_REQUIRE(keys && sorted_target && ideal && scratch, "NULL pointer");
    MB200_REQUIRE(scratch_bytes >= need, "scratch too small (%lld < %lld bytes)", (long long)scratch_bytes, (long long)need);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    unsigned char* p = reinterpret_cast<unsigned char*>(scratch);
    unsigned* radix = reinterpret_cast<unsigned*>(p);
    p += align16(radix_sort_scratch_words(n, 1, 4 + segment_bytes) * 4);
    u64* ka = reinterpret_cast<u64*>(p);
    p += align16((size_t)n * 8);
    u64* kb = reinterpret_cast<u64*>(p);
    p += align16((size_t)n * 8);
    unsigned* vb = reinterpret_cast<unsigned*>(p);
    unsigned* va = reinterpret_cast<unsigned*>(ideal);
    pack_ideal_kernel<<<grid_for(n), kThreads, 0, st>>>(reinterpret_cast<const u64*>(keys), sorted_target, n, ka, va);
    count_launch();
    const int where = radix_sort_passes<u64, unsigned>(ka, va, kb, vb, (int)n, 1, 4 + segment_bytes, radix, err_flag, st, &count_launch);
    if (where < 0) return where;
    if (where == 1) MB200_CUDA_OK(cudaMemcpyAsync(va, vb, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
    return check_cuda(cudaGetLastError(), "retrieval_sort_ideal");
}

extern "C" int64_t mb200_retrieval_evaluate_scratch_bytes(int64_t n) {
    if (n < 1 || n > MB200_RET_MAX_ELEMENTS) return -1;
    return (int64_t)(16 + align16((size_t)n * 4));
}

extern "C" int mb200_retrieval_evaluate(const uint64_t* keys, const float* sorted_target, const float* ideal,
                                        const int64_t* offsets, const int64_t* num_queries, int64_t n, int kind, int64_t top_k,
                                        int adaptive_k, float* value, uint8_t* empty, void* scratch, int64_t scratch_bytes,
                                        void* stream) {
    MB200_REQUIRE(kind >= MB200_RET_AP && kind <= MB200_RET_NDCG, "unknown metric kind %d", kind);
    MB200_REQUIRE(top_k >= 0, "top_k must be >= 0 (0: the query length), got %lld", (long long)top_k);
    const int64_t need = mb200_retrieval_evaluate_scratch_bytes(n);
    MB200_REQUIRE(need > 0, "bad size %lld", (long long)n);
    MB200_REQUIRE(keys && sorted_target && offsets && num_queries && value && empty && scratch, "NULL pointer");
    MB200_REQUIRE(kind != MB200_RET_NDCG || ideal, "NDCG needs the ideal order");
    MB200_REQUIRE(scratch_bytes >= need, "scratch too small (%lld < %lld bytes)", (long long)scratch_bytes, (long long)need);
    const long long* off = reinterpret_cast<const long long*>(offsets);
    EvalArgs a{reinterpret_cast<const u64*>(keys), sorted_target, ideal, off, kind, (long long)top_k, adaptive_k, value, empty};
    const int rc = launch_per_query(MetricBody{a, off}, reinterpret_cast<const long long*>(num_queries), n, scratch,
                                    reinterpret_cast<cudaStream_t>(stream));
    return rc ? rc : check_cuda(cudaGetLastError(), "retrieval_evaluate");
}

extern "C" int mb200_retrieval_auroc(const uint64_t* keys, const float* sorted_target, const int64_t* offsets,
                                     const int64_t* num_queries, int64_t n, int64_t top_k, double max_fpr, float* value,
                                     uint8_t* empty, void* scratch, int64_t scratch_bytes, void* stream) {
    MB200_REQUIRE(top_k >= 0, "top_k must be >= 0 (0: the query length), got %lld", (long long)top_k);
    MB200_REQUIRE(max_fpr < 0.0 || max_fpr == 1.0 || (float)max_fpr < 1.0f,
                  "max_fpr must be negative (none), 1, or round to a float32 below 1; got %g", max_fpr);
    const int64_t need = mb200_retrieval_evaluate_scratch_bytes(n);
    MB200_REQUIRE(need > 0, "bad size %lld", (long long)n);
    MB200_REQUIRE(keys && sorted_target && offsets && num_queries && value && empty && scratch, "NULL pointer");
    MB200_REQUIRE(scratch_bytes >= need, "scratch too small (%lld < %lld bytes)", (long long)scratch_bytes, (long long)need);
    const long long* off = reinterpret_cast<const long long*>(offsets);
    const AurocBody body{reinterpret_cast<const u64*>(keys), sorted_target, off, (long long)top_k, max_fpr == 1.0 ? -1.0 : max_fpr,
                         value, empty};
    const int rc = launch_per_query(body, reinterpret_cast<const long long*>(num_queries), n, scratch,
                                    reinterpret_cast<cudaStream_t>(stream));
    return rc ? rc : check_cuda(cudaGetLastError(), "retrieval_auroc");
}

extern "C" int64_t mb200_retrieval_pr_curve_scratch_bytes(int64_t n) {
    const int64_t eval = mb200_retrieval_evaluate_scratch_bytes(n);
    return eval < 0 ? -1 : eval + (int64_t)align16((size_t)n * 4);
}

extern "C" int mb200_retrieval_pr_curve(const uint64_t* keys, const float* sorted_target, const int64_t* offsets, const int64_t* num_queries, int64_t n,
                                        int64_t max_k, int adaptive_k, float* precision, float* recall, uint8_t* empty,
                                        void* scratch, int64_t scratch_bytes, void* stream) {
    MB200_REQUIRE(max_k >= 1, "max_k must be >= 1, got %lld", (long long)max_k);
    const int64_t need = mb200_retrieval_pr_curve_scratch_bytes(n);
    MB200_REQUIRE(need > 0, "bad size %lld", (long long)n);
    MB200_REQUIRE(keys && sorted_target && offsets && num_queries && precision && recall && empty && scratch, "NULL pointer");
    MB200_REQUIRE(scratch_bytes >= need, "scratch too small (%lld < %lld bytes)", (long long)scratch_bytes, (long long)need);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const long long* off = reinterpret_cast<const long long*>(offsets);
    const long long* nq = reinterpret_cast<const long long*>(num_queries);
    float* positives = reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(scratch) + mb200_retrieval_evaluate_scratch_bytes(n));
    const PrCurveBody body{sorted_target, off, (long long)max_k, precision, recall, empty, positives};
    int rc = launch_per_query(body, nq, n, scratch, st);
    if (rc) return rc;
    // the tail: up to Q * max_k values whatever the query lengths; Q <= n
    const long long units = std::min((long long)n * ((max_k + kThreads - 1) / kThreads), (long long)sm_count() * 16);
    pr_tail_kernel<<<(int)std::max(1ll, units), kThreads, 0, st>>>(off, nq, (long long)max_k, adaptive_k, positives, precision, recall);
    count_launch();
    return check_cuda(cudaGetLastError(), "retrieval_pr_curve");
}
