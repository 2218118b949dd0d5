// Sinks of the row kernels: what happens with one (target, prediction) pair.  See confmat.cu.
#pragma once
#include "common.cuh"

namespace mb200 {

// =====================================================================================================
// Sinks: what happens with one (target, prediction) pair.
// =====================================================================================================
struct ArgmaxOutSink {
    long long* out;
    struct Local {};
    __device__ __forceinline__ void block_init() {}
    __device__ __forceinline__ void init(Local&) {}
    __device__ __forceinline__ void row(Local&, long long idx, long long /*t*/, int p) { out[idx] = p; }
    __device__ __forceinline__ void finish(Local&) {}
    static constexpr bool kNeedsTarget = false;
    static constexpr bool kOverlapSafe = false;
    static constexpr bool kBlockTail = false;
};

// confmat[t, p] += 1 straight into the (L2-resident) state; optional shared-memory privatisation for tiny C.
template <bool kSmem>
struct ConfmatSink {
    long long* confmat;
    int C;
    struct Local {};
    static constexpr bool kNeedsTarget = true;
    // Two consecutive launches may overlap (programmatic dependent launch): all they share is the state, and they only
    // ever touch it with commutative 64-bit REDs.
    static constexpr bool kOverlapSafe = true;
    // Each CTA zeroes and flushes its C*C shared-memory bins (see kBlockTail in confmat.cu).
    static constexpr bool kBlockTail = kSmem;
    __device__ __forceinline__ void block_init() {
        if (kSmem) {
            extern __shared__ unsigned sh_bins[];
            for (int i = threadIdx.x; i < C * C; i += blockDim.x) sh_bins[i] = 0;
            __syncthreads();
        }
    }
    __device__ __forceinline__ void init(Local&) {}
    __device__ __forceinline__ void row(Local&, long long, long long t, int p) {
        if (kSmem) {
            extern __shared__ unsigned sh_bins[];
            atomicAdd(&sh_bins[(int)t * C + p], 1u);
        } else {
            red_add_u64(confmat + t * C + p, 1ull);
        }
    }
    __device__ __forceinline__ void finish(Local&) {
        if (kSmem) {
            extern __shared__ unsigned sh_bins[];
            __syncthreads();
            for (int i = threadIdx.x; i < C * C; i += blockDim.x) {
                const unsigned v = sh_bins[i];
                if (v) red_add_u64(confmat + i, v);
            }
        }
    }
};

// tp/fp/fn deltas go to a zeroed workspace; the last block to finish folds them (and tn) into the states and
// re-zeroes the workspace.  ws layout: [0,C) dtp | [C,2C) dfp | [2C,3C) dfn | [3C] n_valid | [3C+1] ticket.
// micro: ws[0] = #match, ws[1] = #mismatch.
// kDeferFold (large launches): the row kernel only REDs into the workspace and exits — no fence, no ticket — and the fold runs
// as its own one-CTA kernel behind it (stats_fold_kernel, launched with programmatic stream serialization, waiting for this
// grid with griddepcontrol.wait).  The fence + ticket round trip that every CTA pays otherwise, and the last CTA's fold while
// the rest of the GPU idles, are a fixed cost that a large update does not need to pay.
template <bool kSmem, bool kDeferFold = false>
struct StatsSink {
    long long *tp, *fp, *tn, *fn, *ws;
    int C;
    int micro;
    struct Local {
        unsigned n_valid, n_match;
    };
    static constexpr bool kNeedsTarget = true;
    // self-cleaning workspace + last-CTA ticket: launches must not overlap — unless the fold is deferred: then this grid only
    // issues commutative REDs, and its successor in the stream (the fold kernel) waits for it explicitly.  Its own
    // griddepcontrol.wait also orders its REDs after the previous update's fold, which re-zeroes this workspace.
    static constexpr bool kOverlapSafe = kDeferFold;
    // Every warp REDs its totals into ONE word, and (unless deferred) every CTA pays a fence + ticket.
    static constexpr bool kBlockTail = true;
    __device__ __forceinline__ void block_init() {
        if (kSmem) {
            extern __shared__ unsigned sh_bins[];
            for (int i = threadIdx.x; i < 3 * C; i += blockDim.x) sh_bins[i] = 0;
            __syncthreads();
        }
    }
    __device__ __forceinline__ void init(Local& l) { l.n_valid = 0, l.n_match = 0; }
    __device__ __forceinline__ void row(Local& l, long long, long long t, int p) {
        l.n_valid++;
        if (micro) {
            l.n_match += ((long long)p == t);
            return;
        }
        if (kSmem) {
            extern __shared__ unsigned sh_bins[];
            if ((long long)p == t) {
                atomicAdd(&sh_bins[p], 1u);
            } else {
                atomicAdd(&sh_bins[C + p], 1u);
                atomicAdd(&sh_bins[2 * C + (int)t], 1u);
            }
        } else {
            if ((long long)p == t) {
                red_add_u64(ws + p, 1ull);
            } else {
                red_add_u64(ws + C + p, 1ull);
                red_add_u64(ws + 2 * C + t, 1ull);
            }
        }
    }
    __device__ __forceinline__ void finish(Local& l) {
        // per-warp totals -> one atomic per warp
        const unsigned nv = __reduce_add_sync(kFull, l.n_valid);
        const unsigned nm = __reduce_add_sync(kFull, l.n_match);
        if ((threadIdx.x & 31) == 0) {
            if (nv) red_add_u64(ws + 3 * C, nv);
            if (micro) {
                if (nm) red_add_u64(ws + 0, nm);
                if (nv - nm) red_add_u64(ws + 1, nv - nm);
            }
        }
        if (kSmem && !micro) {
            extern __shared__ unsigned sh_bins[];
            __syncthreads();
            for (int i = threadIdx.x; i < 3 * C; i += blockDim.x) {
                const unsigned v = sh_bins[i];
                if (v) red_add_u64(ws + i, v);
            }
        }
        if (kDeferFold) return;  // stats_fold_kernel takes it from here
        // ---- last-block fold -------------------------------------------------------------------
        __shared__ int is_last;
        __threadfence();
        __syncthreads();
        if (threadIdx.x == 0) {
            const unsigned long long ticket =
                atomicAdd(reinterpret_cast<unsigned long long*>(ws + 3 * C + 1), 1ull);
            is_last = (ticket == (unsigned long long)gridDim.x - 1ull);
        }
        __syncthreads();
        if (!is_last) return;
        __threadfence();
        long long* vws = ws;
        const long long n_valid = __ldcg(ws + 3 * C);
        if (micro) {
            if (threadIdx.x == 0) {
                const long long m = __ldcg(ws + 0), mm = __ldcg(ws + 1);
                red_add_u64(tp, (unsigned long long)m);
                red_add_u64(fp, (unsigned long long)mm);
                red_add_u64(fn, (unsigned long long)mm);
                red_add_u64(tn, (unsigned long long)((long long)C * n_valid - (m + 2 * mm)));
                vws[0] = 0;
                vws[1] = 0;
            }
        } else {
            // One CTA runs this while the rest of the GPU idles, so keep it to ONE memory round trip: read the deltas,
            // then fire-and-forget 64-bit REDs into the states (a load-add-store per state would chain 3 more trips per
            // class and made this tail 2/3 of a small update's duration).
            for (int c = threadIdx.x; c < C; c += blockDim.x) {
                const long long a = __ldcg(ws + c), b = __ldcg(ws + C + c), d = __ldcg(ws + 2 * C + c);
                if (a) red_add_u64(tp + c, (unsigned long long)a), vws[c] = 0;
                if (b) red_add_u64(fp + c, (unsigned long long)b), vws[C + c] = 0;
                if (d) red_add_u64(fn + c, (unsigned long long)d), vws[2 * C + c] = 0;
                red_add_u64(tn + c, (unsigned long long)(n_valid - (a + b + d)));
            }
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            vws[3 * C] = 0;
            vws[3 * C + 1] = 0;
        }
    }
};


// The deferred fold of StatsSink<false, true>: ONE CTA, launched behind the row kernel with programmatic stream serialization.
static __global__ void __launch_bounds__(1024) stats_fold_kernel(long long* tp, long long* fp, long long* tn, long long* fn,
                                                                 long long* ws, int C, int micro) {
    asm volatile("griddepcontrol.launch_dependents;");  // the next update's row kernel may queue up; it waits for this grid
    asm volatile("griddepcontrol.wait;" ::: "memory");  // all REDs of the row kernel have landed
    const long long n_valid = __ldcg(ws + 3 * C);
    if (micro) {
        if (threadIdx.x == 0) {
            const long long m = __ldcg(ws + 0), mm = __ldcg(ws + 1);
            red_add_u64(tp, (unsigned long long)m);
            red_add_u64(fp, (unsigned long long)mm);
            red_add_u64(fn, (unsigned long long)mm);
            red_add_u64(tn, (unsigned long long)((long long)C * n_valid - (m + 2 * mm)));
            ws[0] = 0;
            ws[1] = 0;
        }
    } else {
        for (int c = threadIdx.x; c < C; c += blockDim.x) {
            const long long a = __ldcg(ws + c), b = __ldcg(ws + C + c), d = __ldcg(ws + 2 * C + c);
            if (a) red_add_u64(tp + c, (unsigned long long)a), ws[c] = 0;
            if (b) red_add_u64(fp + c, (unsigned long long)b), ws[C + c] = 0;
            if (d) red_add_u64(fn + c, (unsigned long long)d), ws[2 * C + c] = 0;
            red_add_u64(tn + c, (unsigned long long)(n_valid - (a + b + d)));
        }
    }
    __syncthreads();  // every thread has read n_valid
    if (threadIdx.x == 0) ws[3 * C] = 0;
}

// Samplewise stat scores: per (sample, class) tp / fp / fn deltas in a zeroed [3][n_samples][C] int64 scratch plus the
// number of admitted positions per sample; `idx / inner` is the sample.  tn is derived by the caller.
struct SamplewiseSink {
    long long* counts;   // [3][n_samples][C]
    long long* n_valid;  // [n_samples]
    long long n_samples;
    long long inner;
    int C;
    struct Local {};
    static constexpr bool kNeedsTarget = true;
    static constexpr bool kOverlapSafe = false;
    static constexpr bool kBlockTail = false;
    __device__ __forceinline__ void block_init() {}
    __device__ __forceinline__ void init(Local&) {}
    __device__ __forceinline__ void row(Local&, long long idx, long long t, int p) {
        const long long s = idx / inner;
        const long long plane = n_samples * C;
        red_add_u64(n_valid + s, 1ull);
        if ((long long)p == t) {
            red_add_u64(counts + s * C + p, 1ull);
        } else {
            red_add_u64(counts + plane + s * C + p, 1ull);
            red_add_u64(counts + 2 * plane + s * C + t, 1ull);
        }
    }
    __device__ __forceinline__ void finish(Local&) {}
};

}  // namespace mb200
