// K14 — calibration error on sm_90a: the fused top-label update (K14a) and the deterministic binning (K14b).
//
// Reference op chain replaced (src/torchmetrics/):
//   functional/classification/calibration_error.py:239-246   normalize_logits_if_needed(preds, "softmax") -> max(dim=1)
//                                                     -> eq(target) -> float()  (three passes over [N, C] + an [N, C]
//                                                     temporary; utilities/compute.py:190-229)
//   functional/classification/calibration_error.py:30-61     bucketize(right=True) - 1 -> three scatter_add_ into n_bins + 1
//                                                     slots in the state dtype
//
// K14a reads each logit once.  The "are these logits?" vote is batch-global over the rows that are not ignored; like K6's
// softmax_spec_kernel (curve.cu), a row that itself holds a score outside [0, 1] knows the outcome, and a row with all scores
// inside [0, 1] still has them in registers, so it produces BOTH candidates — the top label of the scores as they are and
// the top label of their softmax — and a one-byte "pending" mark; a second launch swaps in the softmax candidate when the
// vote says the batch was logits.  The maximum is taken over the softmax output ROUNDED TO THE INPUT DTYPE (two logits can
// round to the same bf16 probability; the first index then wins), with ATen's max semantics: NaN is maximal, the first NaN
// wins, -0 == +0.
//
// K14b counts exactly (integers) and sums in fp64 with a fixed order: per-warp partial bins in shared memory (lanes that
// share a slot are combined in lane order by their leader), warps combined in warp order, blocks in block order.  The grid
// depends on n only, so the bits do not depend on the GPU or on scheduling.
#include "common.cuh"
#include "../../include/metrics_b200_calibration.h"

namespace mb200 {

namespace {

__device__ __forceinline__ float exp_a(float x) { return expf(x); }
__device__ __forceinline__ double exp_a(double x) { return exp(x); }
__device__ __forceinline__ float max_a(float a, float b) { return fmaxf(a, b); }
__device__ __forceinline__ double max_a(double a, double b) { return fmax(a, b); }

// Does (bv, bi) beat (av, ai) under ATen's max(dim) order?  NaN is maximal and the first NaN wins; otherwise the larger
// value wins and equal values (-0 == +0 included) go to the smaller index.
template <typename A>
__device__ __forceinline__ bool beats(A bv, int bi, A av, int ai) {
    const bool an = av != av, bn = bv != bv;
    if (an | bn) return bn && (!an || bi < ai);
    return bv > av || (bv == av && bi < ai);
}
// every lane ends with the warp's winner
template <typename A>
__device__ __forceinline__ void warp_top(A& v, int& i) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const A ov = __shfl_xor_sync(kFull, v, o);
        const int oi = __shfl_xor_sync(kFull, i, o);
        if (beats(ov, oi, v, i)) {
            v = ov;
            i = oi;
        }
    }
}

__device__ __forceinline__ bool is_ignored(long long t, int has_ignore, long long ignore_index) {
    return has_ignore && t == ignore_index;
}

// ---- K14a, speculative single pass: rows of C <= 32 * kIter f32 / f16 / bf16 scores, one warp per row ----------------
// The softmax arithmetic (fmaxf maximum, lane-strided partial sums of expf(x - m), butterfly, quotient rounded to T) is the
// one of softmax_spec_kernel, hence the same bits as ATen's warp softmax.
template <typename T, int kIter>
__global__ void __launch_bounds__(256, kIter >= 32 ? 2 : 3) top_label_spec_kernel(const T* __restrict__ x, const void* __restrict__ target,
                                                                 int tdtype, int n, int C, int has_ignore,
                                                                 long long ignore_index, float* __restrict__ conf,
                                                                 float* __restrict__ acc, unsigned* __restrict__ vote,
                                                                 unsigned char* __restrict__ pending,
                                                                 float2* __restrict__ cand, unsigned* __restrict__ err) {
    const int lane = threadIdx.x & 31;
    const int wpb = blockDim.x >> 5;
    bool warp_voted = false;
    for (int r = blockIdx.x * wpb + (threadIdx.x >> 5); r < n; r += gridDim.x * wpb) {
        const long long t = load_label(target, tdtype, r);
        if (is_ignored(t, has_ignore, ignore_index)) {  // removed before the vote; the caller drops the row
            if (lane == 0) conf[r] = acc[r] = 0.f;
            continue;
        }
        if (err != nullptr && lane == 0 && (t < 0 || t >= C)) atomicOr(err, MB200_FLAG_TARGET_RANGE);
        const int label = (t >= 0 && t < C) ? (int)t : -1;  // an index never equals -1: a miss
        const T* __restrict__ row = x + (size_t)r * C;
        float v[kIter];
        bool outside = false;
        float m = -INFINITY;
#pragma unroll
        for (int it = 0; it < kIter; ++it) {
            const int c = lane + 32 * it;
            if (c < C) {
                v[it] = widen(row[c]);
                outside |= (v[it] < 0.f) | (v[it] > 1.f);
                m = fmaxf(m, v[it]);
            }
        }
        const bool apply = __any_sync(kFull, outside) != 0;
        if (lane == 0 && apply && !warp_voted) atomicOr(vote, 1u);
        warp_voted |= apply;
        if (!apply) {  // top label of the scores as they are, in case the batch holds probabilities; written right away
            float pv = -INFINITY;
            int pi = 0x7fffffff;
#pragma unroll
            for (int it = 0; it < kIter; ++it) {
                const int c = lane + 32 * it;
                if (c < C && beats(v[it], c, pv, pi)) {
                    pv = v[it];
                    pi = c;
                }
            }
            warp_top(pv, pi);
            if (lane == 0) {
                conf[r] = pv;
                acc[r] = pi == label ? 1.f : 0.f;
                pending[r] = 1;
            }
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
        // Top label of the softmax rounded to T (in case the batch holds logits).  Without a NaN in the row every e lies in
        // [0, 1] and s in [1, C <= 1024], so the largest probability round(1 / s) and half of it are normal numbers of T: a
        // quotient of e < 0.5 rounds to at most half the maximum and cannot win, and the division is skipped for it (the
        // other quotients are the softmax's bits).  A NaN anywhere makes s NaN and every quotient NaN: then all take part.
        const bool all = s != s;
        float sv = -INFINITY;
        int si = 0x7fffffff;
#pragma unroll
        for (int it = 0; it < kIter; ++it) {
            const int c = lane + 32 * it;
            if (c < C && (all || v[it] >= 0.5f)) {
                const float q = round_to<T>(v[it] / s);
                if (beats(q, c, sv, si)) {
                    sv = q;
                    si = c;
                }
            }
        }
        warp_top(sv, si);
        if (lane == 0) {
            if (apply) {
                conf[r] = sv;
                acc[r] = si == label ? 1.f : 0.f;
            } else {
                cand[r] = make_float2(sv, si == label ? 1.f : 0.f);
            }
        }
    }
}

// the batch turned out to be logits: in-range rows take their softmax candidate
__global__ void __launch_bounds__(256) top_label_fix_kernel(int n, const unsigned* __restrict__ vote,
                                                            const unsigned char* __restrict__ pending,
                                                            const float2* __restrict__ cand, float* __restrict__ conf,
                                                            float* __restrict__ acc) {
    if (*vote == 0u) return;
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x) {
        if (pending[r]) {
            const float2 c = cand[r];
            conf[r] = c.x;
            acc[r] = c.y;
        }
    }
}

// ---- K14a, general rows (C > 1024, or f64): a vote pass, then one warp per row with the arithmetic of softmax_if_kernel
template <typename T>
__global__ void __launch_bounds__(256) top_label_vote_kernel(const T* __restrict__ x, const void* __restrict__ target, int tdtype,
                                                             int n, int C, int has_ignore, long long ignore_index,
                                                             unsigned* __restrict__ vote, unsigned* __restrict__ err) {
    using A = compute_t<T>;
    const int lane = threadIdx.x & 31;
    const int wpb = blockDim.x >> 5;
    bool voted = false;
    for (int r = blockIdx.x * wpb + (threadIdx.x >> 5); r < n; r += gridDim.x * wpb) {
        const long long t = load_label(target, tdtype, r);
        if (is_ignored(t, has_ignore, ignore_index)) continue;
        if (err != nullptr && lane == 0 && (t < 0 || t >= C)) atomicOr(err, MB200_FLAG_TARGET_RANGE);
        if (voted) continue;  // this warp already told the batch; only the label check is left
        const T* __restrict__ row = x + (size_t)r * C;
        bool outside = false;
        for (int c = lane; c < C; c += 32) {
            const A a = widen(row[c]);
            outside |= (a < A(0)) | (a > A(1));
        }
        if (__any_sync(kFull, outside)) {
            if (lane == 0) atomicOr(vote, 1u);
            voted = true;
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(256) top_label_rows_kernel(const T* __restrict__ x, const void* __restrict__ target, int tdtype,
                                                             int n, int C, int has_ignore, long long ignore_index,
                                                             const unsigned* __restrict__ vote, float* __restrict__ conf,
                                                             float* __restrict__ acc) {
    using A = compute_t<T>;
    const bool apply = (*vote) != 0u;
    const int lane = threadIdx.x & 31;
    const int wpb = blockDim.x >> 5;
    for (int r = blockIdx.x * wpb + (threadIdx.x >> 5); r < n; r += gridDim.x * wpb) {
        const long long t = load_label(target, tdtype, r);
        if (is_ignored(t, has_ignore, ignore_index)) {
            if (lane == 0) conf[r] = acc[r] = 0.f;
            continue;
        }
        const T* __restrict__ row = x + (size_t)r * C;
        A bv = -INFINITY;
        int bi = 0x7fffffff;
        if (!apply) {
            for (int c = lane; c < C; c += 32) {
                const A a = widen(row[c]);
                if (beats(a, c, bv, bi)) {
                    bv = a;
                    bi = c;
                }
            }
        } else {
            A m = -INFINITY;
            for (int c = lane; c < C; c += 32) m = max_a(m, widen(row[c]));
            m = warp_max(m);
            A s = 0;
            for (int c = lane; c < C; c += 32) s += exp_a(widen(row[c]) - m);
            s = warp_sum(s);
            for (int c = lane; c < C; c += 32) {
                const A q = round_to<T>(exp_a(widen(row[c]) - m) / s);
                if (beats(q, c, bv, bi)) {
                    bv = q;
                    bi = c;
                }
            }
        }
        warp_top(bv, bi);
        if (lane == 0) {
            conf[r] = (float)bv;
            acc[r] = bi == t ? 1.f : 0.f;
        }
    }
}

// ---- K14b ------------------------------------------------------------------------------------------------------------
constexpr int kBinMaxBlocks = 1024;
constexpr long long kBinRowsPerBlock = 4096;
constexpr int kBinMaxSlots = 8192;  // n_bins + 1
constexpr int kBinSmemCap = 227 * 1024;

int bin_blocks(long long n) {
    long long g = (n + kBinRowsPerBlock - 1) / kBinRowsPerBlock;
    if (g < 1) g = 1;
    if (g > kBinMaxBlocks) g = kBinMaxBlocks;
    return (int)g;
}
template <typename A>
size_t bin_smem_bytes(int warps, int slots) {
    // per warp: fp64 confidence and accuracy sums, a 32-entry fp64 staging pair, u32 counts; once: the boundaries
    return (size_t)warps * ((size_t)slots * (8 + 8 + 4) + 32 * 16) + (size_t)slots * sizeof(A);
}
template <typename A>
int bin_warps(int slots) {
    for (int w = 8; w > 1; w >>= 1)
        if (bin_smem_bytes<A>(w, slots) <= 96 * 1024) return w;
    return 1;
}

// Block b bins rows [b * chunk, min(n, (b + 1) * chunk)); warp w of W takes 32 rows at a time, W * 32 apart.  Partials of
// block b go to part[(b * 3 + k) * slots + s]: k = 0 count (int64 bits), 1 confidence sum, 2 accuracy sum.
template <typename T>
__global__ void __launch_bounds__(256) bin_partials_kernel(const T* __restrict__ conf, const void* __restrict__ accp, int acc_dtype,
                                                           long long n, long long chunk, const T* __restrict__ bounds,
                                                           int slots, double* __restrict__ part) {
    using A = compute_t<T>;
    extern __shared__ __align__(16) unsigned char smem[];
    const int W = blockDim.x >> 5;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double* s_conf = reinterpret_cast<double*>(smem);           // [W][slots]
    double* s_acc = s_conf + (size_t)W * slots;                  // [W][slots]
    double* s_stage = s_acc + (size_t)W * slots;                 // [W][2][32]
    A* s_bounds = reinterpret_cast<A*>(s_stage + (size_t)W * 64);  // [slots]
    unsigned* s_cnt = reinterpret_cast<unsigned*>(s_bounds + slots);  // [W][slots]
    for (int i = threadIdx.x; i < W * slots; i += blockDim.x) {
        s_conf[i] = 0.0;
        s_acc[i] = 0.0;
        s_cnt[i] = 0u;
    }
    for (int i = threadIdx.x; i < slots; i += blockDim.x) s_bounds[i] = widen(bounds[i]);
    __syncthreads();

    double* my_conf = s_conf + (size_t)warp * slots;
    double* my_acc = s_acc + (size_t)warp * slots;
    unsigned* my_cnt = s_cnt + (size_t)warp * slots;
    double* stage = s_stage + warp * 64;
    const long long b0 = (long long)blockIdx.x * chunk;
    const long long b1 = b0 + chunk < n ? b0 + chunk : n;
    for (long long base = b0 + (long long)warp * 32; base < b1; base += (long long)W * 32) {
        const long long i = base + lane;
        int bin = -1;
        double cd = 0.0, ad = 0.0;
        if (i < b1) {
            const A xv = widen(conf[i]);
            // torch.bucketize(right=True): the first boundary with b > x; NaN compares false and runs to the end
            int lo = 0, hi = slots;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (!(s_bounds[mid] > xv)) lo = mid + 1;
                else hi = mid;
            }
            bin = lo - 1;  // -1 only for a negative confidence, which normalised scores never are: not counted
            cd = (double)xv;
            ad = (double)round_to<T>((A)load_f64(accp, acc_dtype, i));
        }
        const unsigned peers = __match_any_sync(kFull, bin);
        stage[lane] = cd;
        stage[32 + lane] = ad;
        __syncwarp();
        if (bin >= 0 && lane == __ffs(peers) - 1) {
            double sc = 0.0, sa = 0.0;
            for (unsigned m = peers; m; m &= m - 1) {
                const int j = __ffs(m) - 1;
                sc += stage[j];
                sa += stage[32 + j];
            }
            my_cnt[bin] += (unsigned)__popc(peers);
            my_conf[bin] += sc;
            my_acc[bin] += sa;
        }
        __syncwarp();
    }
    __syncthreads();
    for (int s = threadIdx.x; s < slots; s += blockDim.x) {
        long long cnt = 0;
        double sc = 0.0, sa = 0.0;
        for (int w = 0; w < W; ++w) {
            cnt += s_cnt[(size_t)w * slots + s];
            sc += s_conf[(size_t)w * slots + s];
            sa += s_acc[(size_t)w * slots + s];
        }
        double* out = part + (size_t)blockIdx.x * 3 * slots;
        out[s] = __longlong_as_double(cnt);
        out[slots + s] = sc;
        out[2 * slots + s] = sa;
    }
}

// one block per slot: thread t folds blocks t, t + 256, ... in order, then a fixed shared-memory tree
__global__ void __launch_bounds__(256) bin_final_kernel(const double* __restrict__ part, int blocks, int slots,
                                                        long long* __restrict__ count, double* __restrict__ sum_conf,
                                                        double* __restrict__ sum_acc) {
    __shared__ long long s_cnt[256];
    __shared__ double s_conf[256], s_acc[256];
    const int s = blockIdx.x;
    long long cnt = 0;
    double sc = 0.0, sa = 0.0;
    for (int g = threadIdx.x; g < blocks; g += 256) {
        const double* p = part + (size_t)g * 3 * slots;
        cnt += __double_as_longlong(p[s]);
        sc += p[slots + s];
        sa += p[2 * slots + s];
    }
    s_cnt[threadIdx.x] = cnt;
    s_conf[threadIdx.x] = sc;
    s_acc[threadIdx.x] = sa;
    __syncthreads();
    for (int h = 128; h > 0; h >>= 1) {
        if (threadIdx.x < h) {
            s_cnt[threadIdx.x] += s_cnt[threadIdx.x + h];
            s_conf[threadIdx.x] += s_conf[threadIdx.x + h];
            s_acc[threadIdx.x] += s_acc[threadIdx.x + h];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        count[s] = s_cnt[0];
        sum_conf[s] = s_conf[0];
        sum_acc[s] = s_acc[0];
    }
}

int64_t align16(int64_t b) { return (b + 15) & ~int64_t(15); }

int grid_for_rows(int64_t n, int rows_per_block, int cap) {
    int64_t b = (n + rows_per_block - 1) / rows_per_block;
    if (b < 1) b = 1;
    if (b > cap) b = cap;
    return (int)b;
}

template <typename T>
int launch_top_label(const void* preds, const void* target, int tdtype, int n, int C, int has_ignore, long long ignore_index,
                     float* conf, float* acc, unsigned char* scratch, unsigned* err, cudaStream_t st) {
    unsigned* vote = reinterpret_cast<unsigned*>(scratch);
    const T* x = reinterpret_cast<const T*>(preds);
    if constexpr (sizeof(T) != 8) {
        if (C <= 1024) {
            unsigned char* pending = scratch + 16;
            float2* cand = reinterpret_cast<float2*>(scratch + 16 + align16(n));
            MB200_CUDA_OK(cudaMemsetAsync(scratch, 0, (size_t)(16 + n), st));
            // one wave: 3 resident CTAs per SM (<= 85 registers), 2 for rows of more than 512 scores (32 in registers per lane)
            const int grid = grid_for_rows(n, 8, sm_count() * (C > 512 ? 2 : 3));
#define MB200_TOP(ITER)                                                                                                      \
    top_label_spec_kernel<T, ITER><<<grid, 256, 0, st>>>(x, target, tdtype, n, C, has_ignore, ignore_index, conf, acc, vote, \
                                                         pending, cand, err)
            if (C <= 32) MB200_TOP(1);
            else if (C <= 64) MB200_TOP(2);
            else if (C <= 128) MB200_TOP(4);
            else if (C <= 256) MB200_TOP(8);
            else if (C <= 512) MB200_TOP(16);
            else MB200_TOP(32);
#undef MB200_TOP
            top_label_fix_kernel<<<grid_for_rows(n, 256 * 8, sm_count() * 4), 256, 0, st>>>(n, vote, pending, cand, conf, acc);
            count_launch();
            count_launch();
            return check_cuda(cudaGetLastError(), "calibration top-label launch");
        }
    }
    MB200_CUDA_OK(cudaMemsetAsync(vote, 0, sizeof(unsigned), st));
    const int grid = grid_for_rows(n, 8, sm_count() * 8);
    top_label_vote_kernel<T><<<grid, 256, 0, st>>>(x, target, tdtype, n, C, has_ignore, ignore_index, vote, err);
    top_label_rows_kernel<T><<<grid, 256, 0, st>>>(x, target, tdtype, n, C, has_ignore, ignore_index, vote, conf, acc);
    count_launch();
    count_launch();
    return check_cuda(cudaGetLastError(), "calibration top-label launch");
}

template <typename T>
int launch_bin_sums(const void* confidences, const void* accuracies, int acc_dtype, int64_t n, const void* boundaries, int slots,
                    int64_t* count, double* sum_conf, double* sum_acc, double* part, cudaStream_t st) {
    using A = compute_t<T>;
    const int W = bin_warps<A>(slots);
    const size_t smem = bin_smem_bytes<A>(W, slots);
    MB200_REQUIRE(smem <= (size_t)kBinSmemCap, "n_bins = %d needs %zu bytes of shared memory per warp", slots - 1, smem);
    // the opt-in is made once per (kernel, device) with the largest size any n_bins can ask for: a smaller first value would
    // cap later launches
    MB200_CUDA_OK(ensure_dynamic_smem(bin_partials_kernel<T>, kBinSmemCap));
    const int G = bin_blocks(n);
    const long long chunk = (n + G - 1) / G;
    bin_partials_kernel<T><<<G, 32 * W, smem, st>>>(reinterpret_cast<const T*>(confidences), accuracies, acc_dtype, n, chunk,
                                                   reinterpret_cast<const T*>(boundaries), slots, part);
    bin_final_kernel<<<slots, 256, 0, st>>>(part, G, slots, reinterpret_cast<long long*>(count), sum_conf, sum_acc);
    count_launch();
    count_launch();
    return check_cuda(cudaGetLastError(), "calibration binning launch");
}

}  // namespace
}  // namespace mb200

using namespace mb200;

// =====================================================================================================
// C-ABI
// =====================================================================================================
extern "C" int64_t mb200_calibration_scratch_bytes(int64_t n) {
    if (n < 0) return -1;
    return 16 + align16(n) + 8 * n;  // vote word, one pending byte per row, one (confidence, accuracy) candidate per row
}

extern "C" int mb200_calibration_top_label(const void* preds, int preds_dtype, const void* target, int target_dtype, int64_t n,
                                           int64_t num_classes, int has_ignore, int64_t ignore_index, float* confidence,
                                           float* accuracy, void* scratch, int64_t scratch_bytes, uint32_t* err_flag,
                                           void* stream) {
    MB200_REQUIRE(n >= 0 && num_classes >= 1, "bad sizes");
    MB200_REQUIRE(n < (1ll << 31) && num_classes < (1ll << 31), "sizes exceed int32");
    MB200_REQUIRE(is_float_tag(preds_dtype), "preds must be f32/f16/bf16/f64 (dtype tag %d)", preds_dtype);
    MB200_REQUIRE(is_label_tag(target_dtype), "target must be an integer tensor (dtype tag %d)", target_dtype);
    if (n == 0) return 0;
    MB200_REQUIRE(preds && target && confidence && accuracy && scratch, "NULL pointer");
    MB200_REQUIRE(scratch_bytes >= mb200_calibration_scratch_bytes(n) && (reinterpret_cast<uintptr_t>(scratch) & 15) == 0,
                  "scratch must be 16-byte aligned and hold mb200_calibration_scratch_bytes(n) bytes");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    unsigned char* s = reinterpret_cast<unsigned char*>(scratch);
    const int N = (int)n, C = (int)num_classes;
    return with_float_type(preds_dtype, [&](auto t) {
        return launch_top_label<typename decltype(t)::type>(preds, target, target_dtype, N, C, has_ignore, ignore_index, confidence,
                                                            accuracy, s, err_flag, st);
    });
}

extern "C" int64_t mb200_calibration_bin_scratch_bytes(int64_t n, int64_t n_bins) {
    if (n < 0 || n_bins < 1) return -1;
    return (int64_t)bin_blocks(n) * 3 * (n_bins + 1) * 8;
}

extern "C" int mb200_calibration_bin_sums(const void* confidences, int conf_dtype, const void* accuracies, int acc_dtype,
                                          int64_t n, const void* boundaries, int64_t n_bins, int64_t* count, double* sum_conf,
                                          double* sum_acc, void* scratch, int64_t scratch_bytes, void* stream) {
    MB200_REQUIRE(n >= 0, "negative n");
    MB200_REQUIRE(n_bins >= 1 && n_bins + 1 <= kBinMaxSlots, "n_bins must lie in [1, %d], got %lld", kBinMaxSlots - 1,
                  (long long)n_bins);
    MB200_REQUIRE(is_float_tag(conf_dtype), "confidences must be f32/f16/bf16/f64 (dtype tag %d)", conf_dtype);
    MB200_REQUIRE(is_float_tag(acc_dtype) || is_label_tag(acc_dtype), "unsupported accuracies dtype tag %d", acc_dtype);
    MB200_REQUIRE(boundaries && count && sum_conf && sum_acc && scratch, "NULL pointer");
    MB200_REQUIRE(n == 0 || (confidences && accuracies), "NULL pointer");
    MB200_REQUIRE(scratch_bytes >= mb200_calibration_bin_scratch_bytes(n, n_bins) && (reinterpret_cast<uintptr_t>(scratch) & 15) == 0,
                  "scratch must be 16-byte aligned and hold mb200_calibration_bin_scratch_bytes(n, n_bins) bytes");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int slots = (int)(n_bins + 1);
    double* part = reinterpret_cast<double*>(scratch);
    return with_float_type(conf_dtype, [&](auto t) {
        return launch_bin_sums<typename decltype(t)::type>(confidences, accuracies, acc_dtype, n, boundaries, slots, count, sum_conf,
                                                           sum_acc, part, st);
    });
}
