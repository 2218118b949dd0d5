// K1 / K1b — fused row-argmax + confusion-matrix / stat-scores accumulation for sm_90a.
//
// Reference op chain replaced (src/torchmetrics/):
//   functional/classification/confusion_matrix.py:297-328  (argmax -> flatten -> ignore drop -> t*C+p -> bincount)
//   functional/classification/stat_scores.py:328-344, 424-448 (same chain, then diag / row / col sums)
//   utilities/data.py:178-206 (_bincount)  and the `state += ...` of the modular classes.
//
// Design (DESIGN.md §K1): one warp owns one row of the [N, C] score matrix.  Each lane issues up to four
// independent 16-byte streaming loads (the whole 2000-byte bf16 row of the C=1000 config is one "chunk"),
// reduces its registers with NaN-propagating packed max (HMNMX2), the warp agrees on the row maximum with a
// single REDUX on an order-preserving integer key, and a second register-only pass finds the FIRST column
// holding that maximum (torch.argmax tie rule) — again one REDUX.  Lane 0 then commits one 64-bit RED to
// the L2-resident state.  No intermediate (argmax vector, t*C+p, C*C bins) ever touches HBM, so the
// algorithmic traffic is the logits read itself.
#include "argmax_core.cuh"
#include "common.cuh"
#include "sinks.cuh"

namespace mb200 {

// =====================================================================================================
// Kernels
// =====================================================================================================
struct RowArgs {
    const void* preds;
    const void* target;
    int target_dtype;
    long long n_outer;
    int C;
    long long inner;
    int has_ignore;
    long long ignore_index;
    unsigned* err;
};

template <bool kI64>
__device__ __forceinline__ long long fetch_label(const RowArgs& a, long long idx) {
    if (kI64) return __ldg(reinterpret_cast<const long long*>(a.target) + idx);
    return load_label(a.target, a.target_dtype, idx);
}

// Decide whether a row with label t takes part; flags out-of-range labels.
__device__ __forceinline__ bool admit_label(const RowArgs& a, long long t, bool report) {
    if (a.has_ignore && t == a.ignore_index) return false;
    if ((unsigned long long)t >= (unsigned long long)a.C) {  // also catches negatives
        if (report && a.err) atomicOr(a.err, MB200_FLAG_TARGET_RANGE);
        return false;
    }
    return true;
}

constexpr int kRowThreads = 256;

// (1) aligned path: warp per row, 16-byte streaming vector loads from global memory.  The label of the warp's NEXT
// row is requested before the current row is reduced, so label latency never sits in front of the row loads.
// With >= 4 resident CTAs/SM the reduction is meant to hide behind the HBM stream; tools/confmat_sweep.cu times this loop
// against a read-only streaming probe over the same 131 MB (DESIGN.md §K1 lists the alternatives that measured slower).
template <typename T, typename Sink, bool kI64>
__global__ void __launch_bounds__(kRowThreads) rows_vec_kernel(RowArgs a, Sink sink) {
    // Let the next update's grid (launched with programmatic stream serialization, see launch_overlapped) start filling
    // SMs as soon as this grid's CTAs retire, instead of after the whole grid has drained and a launch gap has passed.
    if constexpr (Sink::kOverlapSafe) {
        asm volatile("griddepcontrol.launch_dependents;");
        // Overlapped launch: this CTA may be resident while the previous grid of the stream is still draining; that
        // grid's memory (it may be the producer of our inputs, triggering its dependents early) is only guaranteed
        // visible after griddepcontrol.wait, so no input is touched before it.  (Prefetching the first rows into L2
        // ahead of the wait was measured and is slower.)
        asm volatile("griddepcontrol.wait;" ::: "memory");
    }
    sink.block_init();
    typename Sink::Local loc;
    sink.init(loc);
    const int lane = threadIdx.x & 31;
    const int wpb = blockDim.x >> 5;
    const int nwarps = gridDim.x * wpb;
    const int n = (int)a.n_outer;
    const int nvec = (int)(((long long)a.C * sizeof(T)) >> 4);
    const T* __restrict__ preds = reinterpret_cast<const T*>(a.preds);
    constexpr bool kLabels = Sink::kNeedsTarget;
    int r = blockIdx.x * wpb + (threadIdx.x >> 5);
    long long t_next = 0;
    if (kLabels && r < n) t_next = fetch_label<kI64>(a, r);
    for (; r < n; r += nwarps) {
        const long long t = t_next;
        if (kLabels && r + nwarps < n) t_next = fetch_label<kI64>(a, r + nwarps);
        if (kLabels && !admit_label(a, t, lane == 0)) continue;  // ignored rows are never read
        const GlobalVecLoader load{reinterpret_cast<const uint4*>(preds + (size_t)r * a.C)};
        const int p = warp_row_argmax_vec<T>(load, nvec, lane);
        if (lane == 0) sink.row(loc, r, t, p);
    }
    sink.finish(loc);
}

// (2) warp per row, scalar loads
template <typename T, typename Sink, bool kI64>
__global__ void __launch_bounds__(kRowThreads) rows_scalar_kernel(RowArgs a, Sink sink) {
    sink.block_init();
    typename Sink::Local loc;
    sink.init(loc);
    const int lane = threadIdx.x & 31;
    const long long wpb = blockDim.x >> 5;
    const long long nwarps = (long long)gridDim.x * wpb;
    const T* __restrict__ preds = reinterpret_cast<const T*>(a.preds);
    for (long long r = (long long)blockIdx.x * wpb + (threadIdx.x >> 5); r < a.n_outer; r += nwarps) {
        long long t = 0;
        if (Sink::kNeedsTarget) {
            t = fetch_label<kI64>(a, r);
            if (!admit_label(a, t, lane == 0)) continue;
        }
        const int p = warp_row_argmax_scalar<T>(preds + r * a.C, a.C, lane);
        if (lane == 0) sink.row(loc, r, t, p);
    }
    sink.finish(loc);
}

// (2b) top-k "refined" prediction (functional/classification/stat_scores.py:347-368 `_refine_preds_oh`): the effective
// label is the target when it is among the k best scores of the row, else the argmax.  Warp per row, scalar loads;
// "among the k best" = fewer than k columns beat the target's score (greater key, or equal key and lower index —
// the order a stable descending sort gives).
template <typename T, typename Sink, bool kI64>
__global__ void __launch_bounds__(kRowThreads) rows_topk_kernel(RowArgs a, Sink sink, int top_k) {
    sink.block_init();
    typename Sink::Local loc;
    sink.init(loc);
    const int lane = threadIdx.x & 31;
    const long long wpb = blockDim.x >> 5;
    const long long nwarps = (long long)gridDim.x * wpb;
    const T* __restrict__ preds = reinterpret_cast<const T*>(a.preds);
    for (long long r = (long long)blockIdx.x * wpb + (threadIdx.x >> 5); r < a.n_outer; r += nwarps) {
        const long long t = fetch_label<kI64>(a, r);
        if (!admit_label(a, t, lane == 0)) continue;
        const T* __restrict__ row = preds + r * a.C;
        const unsigned long long kt = order_key<T>(row[t]);
        int beats = 0;
        for (int c = lane; c < a.C; c += kWarp) {
            const unsigned long long k = order_key<T>(row[c]);
            beats += (k > kt) || (k == kt && c < (int)t);
        }
        beats = __reduce_add_sync(kFull, beats);
        int p = (int)t;
        if (beats >= top_k) p = warp_row_argmax_scalar<T>(row, a.C, lane);
        if (lane == 0) sink.row(loc, r, t, p);
    }
    sink.finish(loc);
}

// (3) thread per (outer, inner) position, class dim strided by `inner` (also the tiny-C path with inner == 1)
template <typename T, typename Sink, bool kI64>
__global__ void __launch_bounds__(kRowThreads) rows_strided_kernel(RowArgs a, Sink sink) {
    sink.block_init();
    typename Sink::Local loc;
    sink.init(loc);
    const long long total = a.n_outer * a.inner;
    const long long nthreads = (long long)gridDim.x * blockDim.x;
    const T* __restrict__ preds = reinterpret_cast<const T*>(a.preds);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += nthreads) {
        long long t = 0;
        if (Sink::kNeedsTarget) {
            t = fetch_label<kI64>(a, i);
            if (!admit_label(a, t, true)) continue;
        }
        const long long n = i / a.inner, x = i - n * a.inner;
        const int p = thread_argmax_strided<T>(preds + (n * a.C) * a.inner + x, a.C, a.inner);
        sink.row(loc, i, t, p);
    }
    sink.finish(loc);
}

// (4) integer label predictions: thread per sample
template <typename Sink, bool kI64>
__global__ void __launch_bounds__(kRowThreads) labels_kernel(RowArgs a, int preds_dtype, Sink sink) {
    sink.block_init();
    typename Sink::Local loc;
    sink.init(loc);
    const long long total = a.n_outer * a.inner;
    const long long nthreads = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += nthreads) {
        const long long t = fetch_label<kI64>(a, i);
        if (!admit_label(a, t, true)) continue;
        const long long p = load_label(a.preds, preds_dtype, i);
        if ((unsigned long long)p >= (unsigned long long)a.C) {
            if (a.err) atomicOr(a.err, MB200_FLAG_PREDS_RANGE);
            continue;
        }
        sink.row(loc, i, t, (int)p);
    }
    sink.finish(loc);
}

// =====================================================================================================
// Host dispatch
// =====================================================================================================
static inline int grid_for(long long work_items, int items_per_block, int max_blocks) {
    long long g = (work_items + items_per_block - 1) / items_per_block;
    if (g < 1) g = 1;
    if (g > max_blocks) g = max_blocks;
    return (int)g;
}

// Launch with cudaLaunchAttributeProgrammaticStreamSerialization: the grid may begin while the previous kernel of the
// stream is still draining (that kernel opts in with griddepcontrol.launch_dependents).  Only used for launches whose
// sole shared data are commutative atomics on the state.
template <typename Kernel, typename... Args>
static cudaError_t launch_overlapped(Kernel kern, int grid, int threads, size_t smem, cudaStream_t st, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3((unsigned)threads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kern, args...);
}

// One-wave grid size of a kernel: resident CTAs per SM x SMs.  The occupancy query takes a driver lock and costs 1-2 us —
// a tenth of a small update's host time — so its answer is kept per (kernel, block size, dynamic smem, device).
template <typename Kernel>
static int resident_blocks(Kernel k, int threads, size_t smem) {
    struct Entry { const void* fn; int threads; size_t smem; int dev; int blocks; };
    static thread_local Entry cache[8] = {};
    static thread_local int next = 0;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) dev = -1;
    const void* fn = reinterpret_cast<const void*>(k);
    for (const Entry& e : cache)
        if (e.fn == fn && e.threads == threads && e.smem == smem && e.dev == dev && e.blocks > 0) return e.blocks;
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, threads, smem) != cudaSuccess || per_sm < 1)
        per_sm = 1;
    const int blocks = per_sm * sm_count();
    if (dev >= 0) {
        cache[next] = Entry{fn, threads, smem, dev, blocks};
        next = (next + 1) & 7;
    }
    return blocks;
}

template <typename T, typename Sink, bool kI64>
static int launch_rows(const RowArgs& a, Sink sink, size_t smem, cudaStream_t st) {
    const size_t row_bytes = (size_t)a.C * sizeof(T);
    const bool vec_ok = sizeof(T) <= 4 && a.inner == 1 && a.C >= 32 && (row_bytes % 16 == 0) &&
                        ((reinterpret_cast<uintptr_t>(a.preds) & 15) == 0);
    if (vec_ok) {
        if constexpr (sizeof(T) <= 4) {
            auto kern = rows_vec_kernel<T, Sink, kI64>;
            const int grid = grid_for(a.n_outer, kRowThreads / 32, resident_blocks(kern, kRowThreads, smem));
            if constexpr (Sink::kOverlapSafe)
                MB200_CUDA_OK(launch_overlapped(kern, grid, kRowThreads, smem, st, a, sink));
            else
                kern<<<grid, kRowThreads, smem, st>>>(a, sink);
        }
    } else if (a.inner == 1 && a.C >= 32) {
        auto kern = rows_scalar_kernel<T, Sink, kI64>;
        const int grid = grid_for(a.n_outer, kRowThreads / 32, resident_blocks(kern, kRowThreads, smem));
        kern<<<grid, kRowThreads, smem, st>>>(a, sink);
    } else {
        auto kern = rows_strided_kernel<T, Sink, kI64>;
        const int grid = grid_for(a.n_outer * a.inner, kRowThreads, resident_blocks(kern, kRowThreads, smem));
        kern<<<grid, kRowThreads, smem, st>>>(a, sink);
    }
    count_launch();
    return check_cuda(cudaGetLastError(), "row kernel launch");
}

template <typename Sink, bool kI64>
static int dispatch_rows_t(int preds_dtype, int preds_has_class_dim, const RowArgs& a, Sink sink, size_t smem,
                           cudaStream_t st) {
    if (!preds_has_class_dim) {
        if constexpr (Sink::kNeedsTarget) {
            MB200_REQUIRE(is_label_tag(preds_dtype), "label-format preds must have an integer dtype (got dtype tag %d)",
                          preds_dtype);
            auto kern = labels_kernel<Sink, kI64>;
            const int grid = grid_for(a.n_outer * a.inner, kRowThreads, resident_blocks(kern, kRowThreads, smem));
            kern<<<grid, kRowThreads, smem, st>>>(a, preds_dtype, sink);
            count_launch();
            return check_cuda(cudaGetLastError(), "labels kernel launch");
        } else {
            set_error("argmax needs a class dimension");
            return MB200_ERR_INVALID;
        }
    }
    MB200_REQUIRE(is_float_tag(preds_dtype), "preds with a class dimension must be floating point (got dtype tag %d)",
                  preds_dtype);
    return with_float_type(preds_dtype,
                           [&](auto t) { return launch_rows<typename decltype(t)::type, Sink, kI64>(a, sink, smem, st); });
}

template <typename Sink>
static int dispatch_rows(int preds_dtype, int preds_has_class_dim, const RowArgs& a, Sink sink, size_t smem,
                         cudaStream_t st) {
    MB200_REQUIRE(a.n_outer * a.inner < (1ll << 31), "more than 2^31-1 rows per call are not supported (got %lld)",
                  (long long)(a.n_outer * a.inner));
    if (a.target_dtype == MB200_I64) return dispatch_rows_t<Sink, true>(preds_dtype, preds_has_class_dim, a, sink, smem, st);
    return dispatch_rows_t<Sink, false>(preds_dtype, preds_has_class_dim, a, sink, smem, st);
}

static int validate_common(const void* preds, const void* target, int target_dtype, int64_t n_outer,
                           int64_t num_classes, int64_t inner, bool need_target) {
    MB200_REQUIRE(n_outer >= 0 && inner >= 1, "negative sizes (n_outer=%lld inner=%lld)", (long long)n_outer,
                  (long long)inner);
    MB200_REQUIRE(num_classes >= 1 && num_classes <= (1ll << 24),
                  "num_classes must be in [1, 2^24] (got %lld)", (long long)num_classes);
    if (n_outer * inner > 0) {
        MB200_REQUIRE(preds != nullptr, "preds is NULL");
        if (need_target) MB200_REQUIRE(target != nullptr, "target is NULL");
    }
    if (need_target)
        MB200_REQUIRE(is_label_tag(target_dtype), "target must have an integer dtype (got dtype tag %d)", target_dtype);
    return 0;
}

}  // namespace mb200

using namespace mb200;

extern "C" int mb200_multiclass_confmat_update(const void* preds, int preds_dtype, int preds_has_class_dim,
                                               const void* target, int target_dtype, int64_t n_outer,
                                               int64_t num_classes, int64_t inner, int has_ignore_index,
                                               int64_t ignore_index, int64_t* confmat, uint32_t* err_flag,
                                               void* stream) {
    if (int rc = validate_common(preds, target, target_dtype, n_outer, num_classes, inner, true)) return rc;
    MB200_REQUIRE(confmat != nullptr, "confmat is NULL");
    MB200_REQUIRE(num_classes <= 46340, "num_classes^2 must fit in int32 indexing (got %lld)",
                  (long long)num_classes);
    if (n_outer * inner == 0) return 0;
    RowArgs a{preds, target, target_dtype, n_outer, (int)num_classes, inner, has_ignore_index,
              label_ignore_index(ignore_index, target_dtype), err_flag};
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const bool priv = num_classes * num_classes <= 4096 && n_outer * inner >= 4096;
    if (priv) {
        ConfmatSink<true> s{reinterpret_cast<long long*>(confmat), (int)num_classes};
        return dispatch_rows(preds_dtype, preds_has_class_dim, a, s,
                             (size_t)(num_classes * num_classes) * sizeof(unsigned), st);
    }
    ConfmatSink<false> s{reinterpret_cast<long long*>(confmat), (int)num_classes};
    return dispatch_rows(preds_dtype, preds_has_class_dim, a, s, 0, st);
}

extern "C" int mb200_multiclass_stat_scores_update(const void* preds, int preds_dtype, int preds_has_class_dim,
                                                   const void* target, int target_dtype, int64_t n_outer,
                                                   int64_t num_classes, int64_t inner, int has_ignore_index,
                                                   int64_t ignore_index, int micro, int64_t* tp, int64_t* fp,
                                                   int64_t* tn, int64_t* fn, int64_t* workspace,
                                                   uint32_t* err_flag, void* stream) {
    if (int rc = validate_common(preds, target, target_dtype, n_outer, num_classes, inner, true)) return rc;
    MB200_REQUIRE(tp && fp && tn && fn && workspace, "state / workspace pointer is NULL");
    if (n_outer * inner == 0) return 0;
    RowArgs a{preds, target, target_dtype, n_outer, (int)num_classes, inner, has_ignore_index,
              label_ignore_index(ignore_index, target_dtype), err_flag};
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    // Shared-memory privatisation pays when many rows hit few class bins (L2 atomics on a handful of addresses
    // serialise).  With hundreds of classes the ~2 REDs per row spread over 3C L2-resident words cost nothing, while
    // zero-filling and flushing 3C counters per CTA does (at the cfg2 shape the privatised variant is the slower one).
    const bool priv = !micro && num_classes <= 256 && n_outer * inner >= 4096 && n_outer * inner >= 16 * num_classes;
    if (priv) {
        StatsSink<true> s{(long long*)tp, (long long*)fp, (long long*)tn, (long long*)fn,
                          (long long*)workspace, (int)num_classes, micro};
        return dispatch_rows(preds_dtype, preds_has_class_dim, a, s, (size_t)(3 * num_classes) * sizeof(unsigned),
                             st);
    }
    // Large launches: rows only RED into the workspace, the fold follows as its own one-CTA kernel (see sinks.cuh kDeferFold);
    // small ones keep the single launch (an extra launch costs more host time than the fold tail costs device time).
    if (preds_has_class_dim && inner == 1 && n_outer * num_classes >= (1ll << 24)) {
        StatsSink<false, true> s{(long long*)tp, (long long*)fp, (long long*)tn, (long long*)fn, (long long*)workspace,
                                 (int)num_classes, micro};
        if (int rc = dispatch_rows(preds_dtype, preds_has_class_dim, a, s, 0, st)) return rc;
        MB200_CUDA_OK(launch_overlapped(stats_fold_kernel, 1, 1024, 0, st, (long long*)tp, (long long*)fp, (long long*)tn,
                                        (long long*)fn, (long long*)workspace, (int)num_classes, micro));
        count_launch();
        return check_cuda(cudaGetLastError(), "stat-scores fold launch");
    }
    StatsSink<false> s{(long long*)tp, (long long*)fp, (long long*)tn, (long long*)fn, (long long*)workspace,
                       (int)num_classes, micro};
    return dispatch_rows(preds_dtype, preds_has_class_dim, a, s, 0, st);
}

template <typename Sink, bool kI64>
static int launch_topk_t(int preds_dtype, const RowArgs& a, Sink sink, size_t smem, int top_k, cudaStream_t st) {
    MB200_REQUIRE(is_float_tag(preds_dtype), "top-k needs floating scores (dtype tag %d)", preds_dtype);
    with_float_type(preds_dtype, [&](auto t) {
        auto kern = rows_topk_kernel<typename decltype(t)::type, Sink, kI64>;
        const int grid = grid_for(a.n_outer, kRowThreads / 32, resident_blocks(kern, kRowThreads, smem));
        kern<<<grid, kRowThreads, smem, st>>>(a, sink, top_k);
        return 0;
    });
    count_launch();
    return check_cuda(cudaGetLastError(), "top-k kernel launch");
}

extern "C" int mb200_multiclass_stat_scores_topk_update(const void* preds, int preds_dtype, const void* target,
                                                        int target_dtype, int64_t n, int64_t num_classes, int64_t top_k,
                                                        int has_ignore_index, int64_t ignore_index, int64_t* tp,
                                                        int64_t* fp, int64_t* tn, int64_t* fn, int64_t* workspace,
                                                        uint32_t* err_flag, void* stream) {
    if (int rc = validate_common(preds, target, target_dtype, n, num_classes, 1, true)) return rc;
    MB200_REQUIRE(tp && fp && tn && fn && workspace, "state / workspace pointer is NULL");
    MB200_REQUIRE(top_k >= 1 && top_k <= num_classes, "top_k must be in [1, num_classes]");
    if (n == 0) return 0;
    RowArgs a{preds, target, target_dtype, n, (int)num_classes, 1, has_ignore_index,
              label_ignore_index(ignore_index, target_dtype), err_flag};
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    StatsSink<false> s{(long long*)tp, (long long*)fp, (long long*)tn, (long long*)fn, (long long*)workspace,
                       (int)num_classes, 0};
    if (target_dtype == MB200_I64) return launch_topk_t<StatsSink<false>, true>(preds_dtype, a, s, 0, (int)top_k, st);
    return launch_topk_t<StatsSink<false>, false>(preds_dtype, a, s, 0, (int)top_k, st);
}

extern "C" int mb200_multiclass_stat_scores_samplewise(const void* preds, int preds_dtype, int preds_has_class_dim,
                                                       const void* target, int target_dtype, int64_t n_outer,
                                                       int64_t num_classes, int64_t inner, int has_ignore_index,
                                                       int64_t ignore_index, int64_t* counts, int64_t* n_valid,
                                                       uint32_t* err_flag, void* stream) {
    if (int rc = validate_common(preds, target, target_dtype, n_outer, num_classes, inner, true)) return rc;
    MB200_REQUIRE(counts && n_valid, "NULL pointer");
    if (n_outer * inner == 0) return 0;
    RowArgs a{preds, target, target_dtype, n_outer, (int)num_classes, inner, has_ignore_index,
              label_ignore_index(ignore_index, target_dtype), err_flag};
    SamplewiseSink s{(long long*)counts, (long long*)n_valid, n_outer, inner, (int)num_classes};
    return dispatch_rows(preds_dtype, preds_has_class_dim, a, s, 0, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int mb200_argmax_rows(const void* preds, int preds_dtype, int64_t n_outer, int64_t num_classes,
                                 int64_t inner, int64_t* out, void* stream) {
    if (int rc = validate_common(preds, nullptr, MB200_I64, n_outer, num_classes, inner, false)) return rc;
    MB200_REQUIRE(out != nullptr || n_outer * inner == 0, "out is NULL");
    if (n_outer * inner == 0) return 0;
    RowArgs a{preds, nullptr, MB200_I64, n_outer, (int)num_classes, inner, 0, 0, nullptr};
    ArgmaxOutSink s{reinterpret_cast<long long*>(out)};
    return dispatch_rows(preds_dtype, 1, a, s, 0, reinterpret_cast<cudaStream_t>(stream));
}
