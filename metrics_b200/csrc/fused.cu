// K11 — collection-level fusion: ONE pass over a shared (logits, target) batch for a stat-scores metric AND an exact-mode
// curve metric of the same MetricCollection (SURVEY.md §8(f)4-i; reference seam: collections.py:231-262 fans the batch out
// to every member, so MulticlassF1Score runs argmax -> bincount (functional/classification/stat_scores.py:328-448) and
// MulticlassAUROC runs the range vote + softmax (utilities/compute.py:190-229) and keeps the probabilities
// (classification/precision_recall_curve.py list states) — three reads and one write of the batch).
//
// Here a warp owns a row and keeps it in registers (C <= 1024):
//   * argmax with torch.argmax semantics (first index wins ties, NaN is maximal, -0 == +0)  -> tp/fp/fn deltas in the
//     self-cleaning workspace of the stat-scores kernels (sinks.cuh StatsSink, last CTA folds them and tn into the states);
//   * "is this batch logits?" vote (any x < 0 or x > 1)                                     -> device flag word;
//   * softmax in exactly the summation order of K6 / ATen's warp softmax (lane-strided sums, butterfly reduction), written
//     to the curve metric's next list-state tensor.
// One read + one write of the batch.  The vote is batch-global, so the probabilities are written speculatively; if the
// vote ends at "not logits" (the batch already held probabilities) a second, normally empty launch restores the raw scores.
#include "common.cuh"
#include "sinks.cuh"

namespace mb200 {

constexpr int kFusedThreads = 256;

template <typename T, int kIter, bool kI64>
__global__ void __launch_bounds__(kFusedThreads) stats_softmax_kernel(const T* __restrict__ preds, const void* __restrict__ target,
                                                                      int tdtype, int n, int C, StatsSink<false> sink,
                                                                      T* __restrict__ probs, unsigned* __restrict__ logits_flag,
                                                                      unsigned* __restrict__ err) {
    sink.block_init();
    StatsSink<false>::Local loc;
    sink.init(loc);
    const int lane = threadIdx.x & 31;
    const int wpb = blockDim.x >> 5;
    const int nwarps = gridDim.x * wpb;
    bool saw_logits = false;
    for (int r = blockIdx.x * wpb + (threadIdx.x >> 5); r < n; r += nwarps) {
        const T* __restrict__ row = preds + (size_t)r * C;
        const long long t = kI64 ? __ldg(reinterpret_cast<const long long*>(target) + r) : load_label(target, tdtype, r);
        float v[kIter];
#pragma unroll
        for (int it = 0; it < kIter; ++it) {
            const int c = lane + 32 * it;
            v[it] = c < C ? to_f32(row[c]) : -INFINITY;
        }
        // ---- argmax (order keys: NaN largest, -0 == +0; first index among equals) + range vote + row maximum ----
        unsigned best_key = 0u;
        int best_idx = 0x7fffffff;
        float m = -INFINITY;
#pragma unroll
        for (int it = 0; it < kIter; ++it) {
            const int c = lane + 32 * it;
            if (c < C) {
                const unsigned k = f32_order_key(v[it]);
                if (best_idx == 0x7fffffff || k > best_key) best_key = k, best_idx = c;
                saw_logits |= (v[it] < 0.f) | (v[it] > 1.f);
                m = fmaxf(m, v[it]);
            }
        }
        const unsigned kmax = __reduce_max_sync(kFull, best_idx == 0x7fffffff ? 0u : best_key);
        const int p = (int)__reduce_min_sync(kFull, (best_idx != 0x7fffffff && best_key == kmax) ? (unsigned)best_idx : 0x7fffffffu);
        m = warp_max(m);
        // ---- softmax, K6's order: lane-strided partial sums, butterfly ----
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
        T* __restrict__ orow = probs + (size_t)r * C;
#pragma unroll
        for (int it = 0; it < kIter; ++it) {
            const int c = lane + 32 * it;
            if (c < C) orow[c] = narrow<T>(v[it] / s);
        }
        // ---- stat scores ----
        if ((unsigned long long)t >= (unsigned long long)C) {
            if (lane == 0 && err) atomicOr(err, MB200_FLAG_TARGET_RANGE);
        } else if (lane == 0) {
            sink.row(loc, r, t, p);
        }
    }
    if (__any_sync(kFull, saw_logits) && lane == 0) atomicOr(logits_flag, 1u);
    sink.finish(loc);
}

// the batch held probabilities after all: put the raw scores back (no-op launch otherwise)
template <typename T>
__global__ void __launch_bounds__(256) restore_if_not_logits_kernel(const T* __restrict__ preds, T* __restrict__ probs,
                                                                    long long total, const unsigned* __restrict__ logits_flag) {
    if (*logits_flag != 0u) return;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
        probs[i] = preds[i];
}

template <typename T, bool kI64>
static int launch_fused(const void* preds, const void* target, int tdtype, int n, int C, StatsSink<false> sink, void* probs,
                        unsigned* flag, unsigned* err, cudaStream_t st) {
    int grid = (n + kFusedThreads / 32 - 1) / (kFusedThreads / 32);
    const int cap = sm_count() * 3;  // 80 registers x 256 threads: 3 resident CTAs per SM = one wave
    if (grid > cap) grid = cap;
    if (grid < 1) grid = 1;
#define MB200_FZ(ITER)                                                                                                  \
    stats_softmax_kernel<T, ITER, kI64><<<grid, kFusedThreads, 0, st>>>(reinterpret_cast<const T*>(preds), target, tdtype, n, C, \
                                                                        sink, reinterpret_cast<T*>(probs), flag, err)
    if (C <= 32) MB200_FZ(1);
    else if (C <= 64) MB200_FZ(2);
    else if (C <= 128) MB200_FZ(4);
    else if (C <= 256) MB200_FZ(8);
    else if (C <= 512) MB200_FZ(16);
    else MB200_FZ(32);
#undef MB200_FZ
    const long long total = (long long)n * C;
    long long rb = (total + 256 * 8 - 1) / (256 * 8);
    if (rb > 4ll * sm_count()) rb = 4ll * sm_count();
    restore_if_not_logits_kernel<T><<<(unsigned)(rb < 1 ? 1 : rb), 256, 0, st>>>(reinterpret_cast<const T*>(preds),
                                                                               reinterpret_cast<T*>(probs), total, flag);
    count_launch();
    count_launch();
    return check_cuda(cudaGetLastError(), "fused stats + softmax launch");
}

}  // namespace mb200

using namespace mb200;

extern "C" int mb200_multiclass_stats_softmax_update(const void* preds, int preds_dtype, const void* target, int target_dtype,
                                                     int64_t n, int64_t num_classes, int micro, int64_t* tp, int64_t* fp,
                                                     int64_t* tn, int64_t* fn, int64_t* workspace, void* probs_out,
                                                     uint32_t* logits_flag, uint32_t* err_flag, void* stream) {
    MB200_REQUIRE(n >= 0 && n < (1ll << 31), "bad n");
    MB200_REQUIRE(num_classes >= 1 && num_classes <= 1024, "the fused update keeps a row in registers: 1 <= num_classes <= 1024 (got %lld)",
                  (long long)num_classes);
    MB200_REQUIRE(tp && fp && tn && fn && workspace && logits_flag, "state / workspace / flag pointer is NULL");
    MB200_REQUIRE(is_label_tag(target_dtype), "target must have an integer dtype (got dtype tag %d)", target_dtype);
    if (n == 0) return 0;
    MB200_REQUIRE(preds && target && probs_out, "NULL pointer");
    MB200_REQUIRE(is_float_tag<kNoF64>(preds_dtype), "scores must be f32/f16/bf16 (dtype tag %d)", preds_dtype);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    MB200_CUDA_OK(cudaMemsetAsync(logits_flag, 0, sizeof(uint32_t), st));
    StatsSink<false> sink{(long long*)tp, (long long*)fp, (long long*)tn, (long long*)fn, (long long*)workspace,
                          (int)num_classes, micro};
    return with_float_type<kNoF64>(preds_dtype, [&](auto t) {
        using T = typename decltype(t)::type;
        return target_dtype == MB200_I64
                   ? launch_fused<T, true>(preds, target, target_dtype, (int)n, (int)num_classes, sink, probs_out, logits_flag, err_flag, st)
                   : launch_fused<T, false>(preds, target, target_dtype, (int)n, (int)num_classes, sink, probs_out, logits_flag, err_flag, st);
    });
}
