// K4 — binned (fixed-threshold) curve state update: multi-threshold confusion matrix `[T, (C,) 2, 2]` in one pass.
//
// Reference op chains replaced (functional/classification/precision_recall_curve.py): binary :191-251
// (`_binary_precision_recall_curve_update_vectorized` = N*T int64 temporaries + bincount, or `_loop` = T passes over
// the data above 50 000 samples) and multiclass :464-533 (N*C*T temporaries, or T passes above 10^6 elements).
// Here every score does ONE binary search over the (ascending) thresholds — k = #{thr <= score} — and bumps a
// shared-memory counter (class, target == class, k); the suffix sums over k that turn bucket counts into
// "predicted positive at threshold i" counts cost O(C * T) at the end of the kernel that finishes last.
#include "common.cuh"

namespace mb200 {

// The comparand c of threshold t for `score >= t` evaluated in dtype cmp_dtype (DESIGN §2 K4): for every score p of the
// kernel's score type, `p >= c` in Cmp holds exactly when the reference's comparison does.
//  * f16 / bf16: ATen casts t to the score dtype (through float, as c10::Half / c10::BFloat16 do) and compares;
//  * f32: t rounded to float;
//  * f64 with float scores: the least float >= t (round up), since a float p is >= t exactly when it is >= that float;
//  * f64 with double scores (Cmp = double): t itself.
// Every case is a monotone function of t, so an ascending list stays ascending.
template <typename Cmp>
__device__ __forceinline__ Cmp binned_comparand(const void* thr, int thr_dtype, int cmp_dtype, long long i) {
    const double t = load_f64(thr, thr_dtype, i);
    if constexpr (std::is_same<Cmp, double>::value) {
        return t;
    } else {
        switch (cmp_dtype) {
            case MB200_F16: return round_to<__half>((float)t);
            case MB200_BF16: return round_to<__nv_bfloat16>((float)t);
            case MB200_F64: return __double2float_ru(t);
            default: return (float)t;
        }
    }
}

// The same, for threshold lists read from global memory inside the bucket search: kept out of line, so that the conversion
// does not inflate the search loop of the common case (comparands staged in shared memory).
template <typename Cmp>
__device__ __noinline__ Cmp binned_comparand_global(const void* thr, int thr_dtype, int cmp_dtype, long long i) {
    return binned_comparand<Cmp>(thr, thr_dtype, cmp_dtype, i);
}

// bucket counts: scratch[(c * 2 + y) * (T + 1) + k], zero on entry, self-cleaning (the folding CTA re-zeroes it)
template <typename T>
__global__ void __launch_bounds__(256) binned_bucket_kernel(const T* __restrict__ preds, const void* __restrict__ target,
                                                            int tdtype, long long n, int C, const void* __restrict__ thr,
                                                            int thr_dtype, int cmp_dtype, int nthr,
                                                            unsigned long long* __restrict__ scratch,
                                                            long long* __restrict__ confmat, int use_smem, int multilabel,
                                                            int thr_in_smem, int has_ignore, long long ignore) {
    // [C * 2 * (nthr + 1) when use_smem] counters, then nthr comparands (8-byte aligned: the counter count is even)
    extern __shared__ __align__(8) unsigned sh_cnt[];
    const int stride = nthr + 1;
    const int ncnt = C * 2 * stride;
    typedef compute_t<T> Cmp;
    Cmp* sh_stage = reinterpret_cast<Cmp*>(sh_cnt + (use_smem ? ncnt : 0));
    if (thr_in_smem)
        for (int i = threadIdx.x; i < nthr; i += blockDim.x) sh_stage[i] = binned_comparand<Cmp>(thr, thr_dtype, cmp_dtype, i);
    // very long threshold lists (or f64 ones next to large counters) stay in global memory and are converted per read
    auto sh_thr = [&](int k) -> Cmp {
        return thr_in_smem ? sh_stage[k] : binned_comparand_global<Cmp>(thr, thr_dtype, cmp_dtype, k);
    };
    if (use_smem)
        for (int i = threadIdx.x; i < ncnt; i += blockDim.x) sh_cnt[i] = 0;
    __syncthreads();
    // bucket hint for (near-)uniform grids: k ~ (p - thr[0]) * (nthr - 1) / (thr[last] - thr[0]); the exact bucket is then
    // found by stepping against the real thresholds, so the hint only affects speed, never the result
    const float t_first = (float)sh_thr(0), t_last = (float)sh_thr(nthr - 1);
    const float scale = (nthr > 1 && t_last > t_first) ? (float)(nthr - 1) / (t_last - t_first) : 0.f;
    const long long total = n * C;
    const bool flat = (C == 1) || multilabel;  // label index == element index
    // bucket of one score: k = number of thresholds <= p  (p >= thr[j]  <=>  j < k);  NaN compares false everywhere -> 0
    auto bucket_of = [&](Cmp p) -> int {
        int k = 0;
        if (p == p) {
            const float h = ((float)p - t_first) * scale;
            k = h <= 0.f ? 0 : (h >= (float)nthr ? nthr : (int)h);
            int steps = 0;
            while (k < nthr && sh_thr(k) <= p && steps < 4) ++k, ++steps;
            while (k > 0 && !(sh_thr(k - 1) <= p) && steps < 8) --k, ++steps;
            const bool settled = (k == nthr || !(sh_thr(k) <= p)) && (k == 0 || sh_thr(k - 1) <= p);
            if (!settled) {  // irregular thresholds: plain binary search
                int lo = 0, hi = nthr;
                while (lo < hi) {
                    const int mid = (lo + hi) >> 1;
                    if (sh_thr(mid) <= p) lo = mid + 1;
                    else hi = mid;
                }
                k = lo;
            }
        }
        return k;
    };
    auto commit = [&](int c, long long t, Cmp p) {
        // multilabel: target is [n, C] like preds, every label is its own binary problem
        const int y = (C == 1 || multilabel) ? (t == 1) : (t == c);
        if ((C == 1 || multilabel) && (unsigned long long)t > 1ull) return;  // binary: only {0,1} targets take part
        if (has_ignore && t == ignore) return;                               // multilabel ignore_index (0 or 1)
        const int slot = (c * 2 + y) * stride + bucket_of(p);
        if (use_smem) atomicAdd(&sh_cnt[slot], 1u);
        else atomicAdd(&scratch[slot], 1ull);
    };
    const long long gstride = (long long)gridDim.x * blockDim.x;
    const bool small = total < (1ll << 31);
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    constexpr int kUnroll = 4;  // independent elements in flight per thread: loads first, then the dependent bucket work
    for (; i + (kUnroll - 1) * gstride < total; i += kUnroll * gstride) {
        long long tt[kUnroll];
        Cmp pp[kUnroll];
        int cc[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
            const long long e = i + u * gstride;
            long long srow = e;
            cc[u] = 0;
            if (C > 1) {
                srow = small ? (long long)((unsigned)e / (unsigned)C) : e / C;  // 32-bit division when it fits
                cc[u] = (int)(e - srow * C);
            }
            tt[u] = load_label(target, tdtype, flat ? e : srow);
            pp[u] = widen(preds[e]);
        }
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) commit(cc[u], tt[u], pp[u]);
    }
    for (; i < total; i += gstride) {
        long long srow = i;
        int c = 0;
        if (C > 1) {
            srow = small ? (long long)((unsigned)i / (unsigned)C) : i / C;
            c = (int)(i - srow * C);
        }
        commit(c, load_label(target, tdtype, flat ? i : srow), widen(preds[i]));
    }
    if (use_smem) {
        __syncthreads();
        for (int i = threadIdx.x; i < ncnt; i += blockDim.x) {
            const unsigned v = sh_cnt[i];
            if (v) atomicAdd(&scratch[i], (unsigned long long)v);
        }
    }
    // ---- last CTA folds the bucket counts into the [T, C, 2, 2] state and cleans the scratch ----
    __shared__ int is_last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned long long ticket = atomicAdd(&scratch[ncnt], 1ull);
        is_last = ticket == (unsigned long long)gridDim.x - 1ull;
    }
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    // one thread per (class, y): serial suffix sum over k (T is small), confmat[i, c, y, pred] layout [T][C][2][2]
    for (int cy = threadIdx.x; cy < C * 2; cy += blockDim.x) {
        const int c = cy >> 1, y = cy & 1;
        unsigned long long* row = scratch + (size_t)cy * stride;
        unsigned long long tot = 0;
        for (int k = 0; k <= nthr; ++k) tot += __ldcg(row + k);
        unsigned long long ge = tot;  // samples with k > i, starting at i = -1
        for (int i = 0; i < nthr; ++i) {
            ge -= __ldcg(row + i);  // now: samples with k > i  <=>  score >= thr[i]
            // fire-and-forget REDs: a load-add-store here would chain one L2 round trip per threshold
            unsigned long long* cell = reinterpret_cast<unsigned long long*>(confmat + (((size_t)i * C + c) * 2 + y) * 2);
            if (ge) atomicAdd(cell + 1, ge);
            if (tot - ge) atomicAdd(cell + 0, tot - ge);
        }
        for (int k = 0; k <= nthr; ++k) row[k] = 0ull;
    }
    __syncthreads();
    if (threadIdx.x == 0) scratch[ncnt] = 0ull;
}

// ---- binary fast path ------------------------------------------------------------------------------------------------
// The generic kernel above is instruction-bound, not memory-bound: runtime label dtype switch, 64-bit indexing, class division, loop-shaped bucket search.  The binary
// task (C == 1, the shape of cfg3's binned variant) gets its own kernel: f32 scores, int64 / int32 / uint8-family labels
// resolved at compile time, 16-byte vector loads of four scores (+ their four labels), 32-bit indices, thresholds in shared
// memory, and a table-driven bucket search (one shared-memory lookup for most scores, see `bucket_of` below).
template <typename LabelT>
__device__ __forceinline__ void load4_labels(const LabelT* __restrict__ t, unsigned q, long long (&out)[4]) {
    if constexpr (sizeof(LabelT) == 8) {
        const longlong2 a = reinterpret_cast<const longlong2*>(t)[2 * (size_t)q];
        const longlong2 b = reinterpret_cast<const longlong2*>(t)[2 * (size_t)q + 1];
        out[0] = a.x, out[1] = a.y, out[2] = b.x, out[3] = b.y;
    } else if constexpr (sizeof(LabelT) == 4) {
        const int4 a = reinterpret_cast<const int4*>(t)[q];
        out[0] = a.x, out[1] = a.y, out[2] = a.z, out[3] = a.w;
    } else {
        const uchar4 a = reinterpret_cast<const uchar4*>(t)[q];
        out[0] = a.x, out[1] = a.y, out[2] = a.z, out[3] = a.w;
    }
}

constexpr int kBinCells = 4096;
template <typename LabelT>
__global__ void __launch_bounds__(256) binned_binary_fast_kernel(const float* __restrict__ preds, const LabelT* __restrict__ target,
                                                                 unsigned n, const void* __restrict__ thr, int thr_dtype,
                                                                 int cmp_dtype, int nthr,
                                                                 unsigned long long* __restrict__ scratch,
                                                                 long long* __restrict__ confmat) {
    extern __shared__ unsigned sh_fast[];  // [2 * (nthr + 1)] counters | nthr thresholds | kBinCells cell table
    const int stride = nthr + 1;
    const int ncnt = 2 * stride;
    float* sh_thr = reinterpret_cast<float*>(sh_fast + ncnt);
    unsigned* cell = sh_fast + ncnt + nthr;  // per cell: low 16 bits = #thresholds in lower cells, high 16 = #thresholds inside
    for (int i = threadIdx.x; i < nthr; i += blockDim.x) sh_thr[i] = binned_comparand<float>(thr, thr_dtype, cmp_dtype, i);
    for (int i = threadIdx.x; i < ncnt; i += blockDim.x) sh_fast[i] = 0;
    for (int i = threadIdx.x; i < kBinCells; i += blockDim.x) cell[i] = 0;
    __syncthreads();
    // Bucket of a score = k = #{thr_j <= p}.  A MONOTONE cell function f(p) = clamp(int((p - thr_0) * scale)) splits the score
    // axis into kBinCells cells; thresholds in lower cells are certainly <= p, thresholds in higher cells certainly > p
    // (monotonicity — whatever the rounding of f), so only the thresholds that fall into p's own cell are compared with p
    // itself: none for ~95 % of the cells of a 200-point grid.  Exact for any threshold list; NaN lands in cell 0, passes no
    // comparison and gets k = 0, like the reference's `preds >= thr`.
    const float t_first = sh_thr[0], t_last = sh_thr[nthr - 1];
    const float scale = (nthr > 1 && t_last > t_first) ? (float)(kBinCells - 2) / (t_last - t_first) : 0.f;
    auto cell_of = [&](float p) -> int {
        const float h = (p - t_first) * scale;
        return h >= (float)(kBinCells - 1) ? kBinCells - 1 : (h > 0.f ? (int)h : 0);
    };
    for (int j = threadIdx.x; j < nthr; j += blockDim.x) atomicAdd(&cell[cell_of(sh_thr[j])], 1u << 16);
    __syncthreads();
    {  // exclusive prefix of the per-cell counts -> low half (kBinCells / 256 consecutive cells per thread + block scan)
        constexpr int kPer = kBinCells / 256;
        __shared__ unsigned wsum[8];
        unsigned local = 0;
#pragma unroll
        for (int i = 0; i < kPer; ++i) local += cell[threadIdx.x * kPer + i] >> 16;
        unsigned incl = local;
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned v = __shfl_up_sync(kFull, incl, o);
            if (lane >= o) incl += v;
        }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        unsigned run = incl - local;
        for (int w = 0; w < warp; ++w) run += wsum[w];
#pragma unroll
        for (int i = 0; i < kPer; ++i) {
            const unsigned e = cell[threadIdx.x * kPer + i];
            cell[threadIdx.x * kPer + i] = e | run;
            run += e >> 16;
        }
    }
    __syncthreads();
    auto bucket_of = [&](float p) -> int {
        const unsigned e = cell[cell_of(p)];
        const int k_lo = (int)(e & 0xffffu);
        const unsigned inside = e >> 16;  // thresholds sharing p's cell: 0 for most cells, 1 for the rest of a regular grid
        int k = k_lo + (int)((inside != 0u) & (sh_thr[min(k_lo, nthr - 1)] <= p));  // branch-free for inside <= 1
        if (inside > 1u)
            for (unsigned j = 1; j < inside; ++j) k += (sh_thr[k_lo + j] <= p);
        return k;
    };
    auto commit = [&](long long t, float p) {
        if ((unsigned long long)t > 1ull) return;  // only {0, 1} targets take part
        atomicAdd(&sh_fast[(int)t * stride + bucket_of(p)], 1u);
    };
    const unsigned quads = n >> 2;
    const unsigned gstride = gridDim.x * blockDim.x;
    unsigned q = blockIdx.x * blockDim.x + threadIdx.x;
    for (; q + gstride < quads; q += 2 * gstride) {  // two independent quads in flight
        const float4 p0 = reinterpret_cast<const float4*>(preds)[q], p1 = reinterpret_cast<const float4*>(preds)[q + gstride];
        long long t0[4], t1[4];
        load4_labels<LabelT>(target, q, t0);
        load4_labels<LabelT>(target, q + gstride, t1);
        commit(t0[0], p0.x), commit(t0[1], p0.y), commit(t0[2], p0.z), commit(t0[3], p0.w);
        commit(t1[0], p1.x), commit(t1[1], p1.y), commit(t1[2], p1.z), commit(t1[3], p1.w);
    }
    for (; q < quads; q += gstride) {
        const float4 p0 = reinterpret_cast<const float4*>(preds)[q];
        long long t0[4];
        load4_labels<LabelT>(target, q, t0);
        commit(t0[0], p0.x), commit(t0[1], p0.y), commit(t0[2], p0.z), commit(t0[3], p0.w);
    }
    for (unsigned i = (quads << 2) + blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gstride)
        commit((long long)target[i], preds[i]);
    __syncthreads();
    for (int i = threadIdx.x; i < ncnt; i += blockDim.x) {
        const unsigned v = sh_fast[i];
        if (v) atomicAdd(&scratch[i], (unsigned long long)v);
    }
    // ---- last CTA folds the bucket counts into the [T, 2, 2] state and cleans the scratch (as in the generic kernel) ----
    __shared__ int is_last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned long long ticket = atomicAdd(&scratch[ncnt], 1ull);
        is_last = ticket == (unsigned long long)gridDim.x - 1ull;
    }
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    if (threadIdx.x < 2) {
        const int y = threadIdx.x;
        unsigned long long* row = scratch + (size_t)y * stride;
        unsigned long long tot = 0;
        for (int k = 0; k <= nthr; ++k) tot += __ldcg(row + k);
        unsigned long long ge = tot;
        for (int i = 0; i < nthr; ++i) {
            ge -= __ldcg(row + i);
            unsigned long long* cell = reinterpret_cast<unsigned long long*>(confmat + ((size_t)i * 2 + y) * 2);
            if (ge) atomicAdd(cell + 1, ge);
            if (tot - ge) atomicAdd(cell + 0, tot - ge);
        }
        for (int k = 0; k <= nthr; ++k) row[k] = 0ull;
    }
    __syncthreads();
    if (threadIdx.x == 0) scratch[ncnt] = 0ull;
}

}  // namespace mb200

using namespace mb200;

extern "C" int64_t mb200_binned_curve_scratch_words(int64_t num_classes, int64_t num_thresholds) {
    if (num_classes < 1 || num_thresholds < 1) return -1;
    return num_classes * 2 * (num_thresholds + 1) + 8;
}

// The dtype D in which the reference evaluates `score >= threshold` for one update (DESIGN §2 K4).  Binary (and micro)
// updates of more than 50 000 scores and multiclass updates with n * C * C > 10^6 take the reference's loop branch,
// `preds >= thresholds[i]` with a 0-dim threshold: D is the score dtype.  Smaller ones and every multilabel update take
// its vectorized branch, `preds.unsqueeze(-1) >= thresholds.unsqueeze(0)`: D is torch.promote_types(score, threshold).
extern "C" int mb200_binned_curve_compare_dtype(int preds_dtype, int thresholds_dtype, int64_t n, int64_t num_classes,
                                                int multilabel) {
    if (!is_float_tag(preds_dtype) || !(is_float_tag(thresholds_dtype) || with_label_type(thresholds_dtype, [](auto) { return 0; }) == 0))
        return -1;
    const bool loop = !multilabel && (num_classes == 1 ? n > 50000 : (double)n * (double)num_classes * (double)num_classes > 1e6);
    if (loop || !is_float_tag(thresholds_dtype) || thresholds_dtype == preds_dtype) return preds_dtype;
    if (preds_dtype == MB200_F64 || thresholds_dtype == MB200_F64) return MB200_F64;
    return MB200_F32;  // f32 with anything narrower, and f16 with bf16
}

static int binned_update_impl(int multilabel, const void* preds, int preds_dtype, const void* target, int target_dtype,
                              int64_t n, int64_t num_classes, const void* thresholds_sorted, int thr_dtype, int cmp_dtype,
                              int64_t num_thresholds, int has_ignore, int64_t ignore_index, int64_t* confmat, uint64_t* scratch,
                              void* stream) {
    MB200_REQUIRE(n >= 0 && num_classes >= 1 && num_thresholds >= 1, "bad sizes");
    MB200_REQUIRE(num_thresholds < (1 << 24) && num_classes < (1 << 24), "sizes too large");
    if (n == 0) return 0;
    MB200_REQUIRE(preds && target && thresholds_sorted && confmat && scratch, "NULL pointer");
    MB200_REQUIRE(is_float_tag(preds_dtype), "scores must be floating point (dtype tag %d)", preds_dtype);
    MB200_REQUIRE(is_float_tag(thr_dtype) || with_label_type(thr_dtype, [](auto) { return 0; }) == 0,
                  "thresholds must be floating point or integer (dtype tag %d)", thr_dtype);
    MB200_REQUIRE(cmp_dtype == MB200_F64 || (cmp_dtype == MB200_F32 && preds_dtype != MB200_F64) || cmp_dtype == preds_dtype,
                  "comparison dtype tag %d is not reachable from score dtype tag %d", cmp_dtype, preds_dtype);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const long long total = n * num_classes;
    const long long ignore = has_ignore ? label_ignore_index(ignore_index, target_dtype) : 0;
    const size_t smem_need = (size_t)num_classes * 2 * (num_thresholds + 1) * sizeof(unsigned);
    const int use_smem = smem_need <= 40 * 1024;
    long long blocks = (total + 256 * 8 - 1) / (256 * 8);
    const long long cap = (long long)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    unsigned long long* sc = reinterpret_cast<unsigned long long*>(scratch);
    long long* cm = reinterpret_cast<long long*>(confmat);
    // binary fast path: f32 scores, 16-byte aligned inputs, the usual label dtypes, counters + thresholds in shared memory
    const bool label_ok = target_dtype == MB200_I64 || target_dtype == MB200_I32 || target_dtype == MB200_U8 ||
                          target_dtype == MB200_BOOL || target_dtype == MB200_I8;
    if (!multilabel && num_classes == 1 && preds_dtype == MB200_F32 && label_ok && num_thresholds <= 2048 && n < (1ll << 31) &&
        n >= 4096 && ((reinterpret_cast<uintptr_t>(preds) | reinterpret_cast<uintptr_t>(target)) & 15) == 0) {
        const size_t smem_fast = (size_t)(2 * (num_thresholds + 1)) * sizeof(unsigned) + (size_t)num_thresholds * sizeof(float) +
                                 (size_t)kBinCells * sizeof(unsigned);
        long long fb = (n / 4 + 256 * 4 - 1) / (256 * 4);
        const long long fcap = (long long)sm_count() * 6;
        if (fb > fcap) fb = fcap;
        if (fb < 1) fb = 1;
        const float* pf = reinterpret_cast<const float*>(preds);
        const int nt = (int)num_thresholds;
        if (target_dtype == MB200_I64)
            binned_binary_fast_kernel<long long><<<(int)fb, 256, smem_fast, st>>>(pf, (const long long*)target, (unsigned)n,
                                                                                 thresholds_sorted, thr_dtype, cmp_dtype, nt, sc, cm);
        else if (target_dtype == MB200_I32)
            binned_binary_fast_kernel<int><<<(int)fb, 256, smem_fast, st>>>(pf, (const int*)target, (unsigned)n, thresholds_sorted,
                                                                           thr_dtype, cmp_dtype, nt, sc, cm);
        else if (target_dtype == MB200_I8)
            binned_binary_fast_kernel<signed char><<<(int)fb, 256, smem_fast, st>>>(pf, (const signed char*)target, (unsigned)n,
                                                                                   thresholds_sorted, thr_dtype, cmp_dtype, nt, sc, cm);
        else
            binned_binary_fast_kernel<unsigned char><<<(int)fb, 256, smem_fast, st>>>(pf, (const unsigned char*)target, (unsigned)n,
                                                                                     thresholds_sorted, thr_dtype, cmp_dtype, nt, sc, cm);
        count_launch();
        return check_cuda(cudaGetLastError(), "binned curve launch");
    }
    with_float_type(preds_dtype, [&](auto t) {
        using T = typename decltype(t)::type;
        using Cmp = compute_t<T>;
        // comparands in shared memory when they fit beside the counters under the 48 KB that needs no opt-in: always for
        // float comparands (40 KB + 2048 * 4 B), not for 2048 double ones next to more than 32 KB of counters
        const size_t thr_bytes = (size_t)num_thresholds * sizeof(Cmp);
        const size_t cnt_bytes = use_smem ? smem_need : 0;
        const int thr_in_smem = num_thresholds <= 2048 && cnt_bytes + thr_bytes <= 48 * 1024;
        binned_bucket_kernel<T><<<(int)blocks, 256, cnt_bytes + (thr_in_smem ? thr_bytes : 0), st>>>(
            reinterpret_cast<const T*>(preds), target, target_dtype, n, (int)num_classes, thresholds_sorted, thr_dtype, cmp_dtype,
            (int)num_thresholds, sc, cm, use_smem, multilabel, thr_in_smem, has_ignore ? 1 : 0, ignore);
        return 0;
    });
    count_launch();
    return check_cuda(cudaGetLastError(), "binned curve launch");
}

extern "C" int mb200_binned_curve_update(const void* preds, int preds_dtype, const void* target, int target_dtype,
                                         int64_t n, int64_t num_classes, const void* thresholds_sorted, int thresholds_dtype,
                                         int compare_dtype, int64_t num_thresholds, int64_t* confmat, uint64_t* scratch,
                                         void* stream) {
    return binned_update_impl(0, preds, preds_dtype, target, target_dtype, n, num_classes, thresholds_sorted, thresholds_dtype,
                              compare_dtype, num_thresholds, 0, 0, confmat, scratch, stream);
}

// multilabel: target is [n, num_labels] like preds; entries whose target is not 0 / 1, or equals ignore_index reduced to the
// target dtype's width, are skipped
extern "C" int mb200_binned_curve_update_multilabel(const void* preds, int preds_dtype, const void* target,
                                                    int target_dtype, int64_t n, int64_t num_labels,
                                                    const void* thresholds_sorted, int thresholds_dtype, int compare_dtype,
                                                    int64_t num_thresholds, int has_ignore_index, int64_t ignore_index,
                                                    int64_t* confmat, uint64_t* scratch, void* stream) {
    return binned_update_impl(1, preds, preds_dtype, target, target_dtype, n, num_labels, thresholds_sorted, thresholds_dtype,
                              compare_dtype, num_thresholds, has_ignore_index, ignore_index, confmat, scratch, stream);
}
