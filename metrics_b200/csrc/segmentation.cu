// K15 — per-sample, per-class overlap counts for semantic segmentation (MeanIoU, DiceScore, GeneralizedDiceScore) on sm_90a.
//
// Reference op chain replaced (src/torchmetrics/functional/segmentation/):
//   mean_iou.py:51-61, dice.py:53-66, generalized_dice.py:58-71
//       index input: one_hot(preds).movedim(-1, 1), one_hot(target).movedim(-1, 1)   (two int64 [N, C, ...] tensors)
//       -> [:, 1:] when the background is dropped -> sum(p & t) or sum(p * t), sum(t), sum(p) over the spatial axes
//
// Index format: one read of the two label maps.  A CTA owns one slice of one sample and keeps a 3 x C' histogram of 32-bit
// counters in shared memory (a slice holds at most 2^31 pixels, so no counter can overflow); every non-zero counter is
// flushed with one 64-bit RED.  Label maps are spatially coherent, so a warp often holds one class: each warp first checks
// whether all lanes agree (one shared atomic for 32 pixels) and otherwise groups equal lanes with __match_any_sync (one
// atomic per distinct class).  Above kSmemMaxClasses the same warp-aggregated adds go straight to the int64 output.
// Out-of-range labels are not counted; they set MB200_SEG_* bits, kept apart for preds / target and < 0 / >= C.
//
// One-hot format: a segmented reduction over the (n, c) planes, in the input dtype's arithmetic.  Planar inputs (inner
// stride 1) are read with 16-byte vectors when preds and target share their alignment; channels-last inputs (class stride
// 1) are read row by row, each thread owning one class column.  Integer sums are exact (int64, two's-complement wrap like
// torch.sum) and several CTAs per plane combine with 64-bit REDs.  Float sums are float64 of the values and of the
// products rounded to the input dtype.  They are split over as many CTAs as the integer sums; each CTA stores its float64
// partials in scratch, and the last CTA of a plane (planar) or sample (channels-last) to arrive folds them in slice order.
// The result does not depend on which CTA arrives last, so float sums are deterministic.
#include <algorithm>
#include <type_traits>

#include "common.cuh"
#include "../../include/metrics_b200_segmentation.h"

namespace mb200 {

namespace {

constexpr int kThreads = 256;
constexpr int kIdxUnroll = 4;
constexpr int kSmemMaxClasses = 4096;  // 3 x 4096 x 4 B = 48 KB: the histogram of the widest shared-memory launch
constexpr long long kMaxSlice = 1ll << 31;

// ---- index format ------------------------------------------------------------------------------------------------------
// Add this lane's key (class column, or -1 for nothing) to hist[key] (shared) or gout[key] (global): one atomic per distinct
// key of the warp.  Every lane of the warp calls it.
template <bool kShared>
__device__ __forceinline__ void tally(int key, unsigned* hist, unsigned long long* gout, int lane) {
    const int k0 = __shfl_sync(kFull, key, 0);
    unsigned peers;
    if (__all_sync(kFull, key == k0)) {
        peers = lane == 0 ? kFull : 0u;
    } else {
        peers = __match_any_sync(kFull, key);
        if (lane != __ffs(peers) - 1) peers = 0u;
    }
    if (peers != 0u && key >= 0) {
        if constexpr (kShared) atomicAdd(&hist[key], (unsigned)__popc(peers));
        else atomicAdd(&gout[key], (unsigned long long)__popc(peers));
    }
}

// grid: n * bps CTAs; CTA b counts pixels [part * chunk, min(S, (part + 1) * chunk)) of sample b / bps
template <bool kShared>
__global__ void __launch_bounds__(kThreads) index_counts_kernel(const long long* __restrict__ preds,
                                                                const long long* __restrict__ target, long long S, int C,
                                                                int off, int Cp, long long N, long long bps, long long chunk,
                                                                unsigned long long* __restrict__ out, unsigned* err) {
    extern __shared__ unsigned hist[];  // [3][Cp]: intersection, pred_sum, target_sum
    const long long n = blockIdx.x / bps, part = blockIdx.x % bps;
    const long long s0 = part * chunk, s1 = min(S, s0 + chunk);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if constexpr (kShared) {
        for (int j = threadIdx.x; j < 3 * Cp; j += kThreads) hist[j] = 0u;
        __syncthreads();
    }
    const long long plane = N * Cp;
    unsigned long long* g_int = out + n * Cp;
    unsigned long long* g_pred = g_int + plane;
    unsigned long long* g_tgt = g_pred + plane;
    const long long* P = preds + n * S;
    const long long* T = target + n * S;
    unsigned flags = 0u;
    constexpr long long kWarpSpan = 32 * kIdxUnroll;
    for (long long base = s0 + warp * kWarpSpan; base < s1; base += kWarpSpan * (kThreads / 32)) {
        long long pv[kIdxUnroll], tv[kIdxUnroll];
#pragma unroll
        for (int k = 0; k < kIdxUnroll; ++k) {
            const long long i = base + k * 32 + lane;
            pv[k] = i < s1 ? __ldg(P + i) : -1;
            tv[k] = i < s1 ? __ldg(T + i) : -1;
        }
#pragma unroll
        for (int k = 0; k < kIdxUnroll; ++k) {
            const bool in = base + k * 32 + lane < s1;
            const long long p = pv[k], t = tv[k];
            if (in) {
                flags |= p < 0 ? MB200_SEG_PREDS_NEGATIVE : (p >= C ? MB200_SEG_PREDS_TOO_LARGE : 0u);
                flags |= t < 0 ? MB200_SEG_TARGET_NEGATIVE : (t >= C ? MB200_SEG_TARGET_TOO_LARGE : 0u);
            }
            // class column, or -1: out of the slice, out of range, or the dropped background
            const int kp = (in && p >= off && p < C) ? (int)p - off : -1;
            const int kt = (in && t >= off && t < C) ? (int)t - off : -1;
            const int ki = p == t ? kp : -1;
            tally<kShared>(ki, hist, g_int, lane);
            tally<kShared>(kp, hist + Cp, g_pred, lane);
            tally<kShared>(kt, hist + 2 * Cp, g_tgt, lane);
        }
    }
    flags = __reduce_or_sync(kFull, flags);
    if (lane == 0 && flags != 0u && err != nullptr) atomicOr(err, flags);
    if constexpr (kShared) {
        __syncthreads();
        for (int j = threadIdx.x; j < 3 * Cp; j += kThreads) {
            const unsigned v = hist[j];
            if (v != 0u) {
                const int q = j / Cp, c = j - q * Cp;
                atomicAdd(out + q * plane + n * Cp + c, (unsigned long long)v);
            }
        }
    }
}

// ---- one-hot format: element arithmetic in the input dtype -------------------------------------------------------------
// Storage type, accumulator and the three terms of one element pair.  OP 0: p & t, OP 1: p * t, both rounded to T.
template <typename T>
struct OH {  // signed / unsigned integers: int64 sums with wrap, accumulated as unsigned
    using A = unsigned long long;
    __device__ static A val(T x) { return (A)(long long)x; }
    template <int OP>
    __device__ static A prod(T a, T b) {
        if constexpr (OP == MB200_SEG_AND) return val((T)(a & b));
        else return val((T)((unsigned long long)(long long)a * (unsigned long long)(long long)b));
    }
};
struct Bool {
    unsigned char v;
};
template <>
struct OH<Bool> {  // torch.bool: & and * are both the logical and
    using A = unsigned long long;
    __device__ static A val(Bool x) { return x.v != 0; }
    template <int OP>
    __device__ static A prod(Bool a, Bool b) { return (a.v != 0) & (b.v != 0); }
};
template <>
struct OH<float> {
    using A = double;
    __device__ static A val(float x) { return widen(x); }
    template <int OP>
    __device__ static A prod(float a, float b) { return __fmul_rn(a, b); }
};
template <>
struct OH<__half> {  // the float product of two halves is exact; one rounding gives the half product
    using A = double;
    __device__ static A val(__half x) { return widen(x); }
    template <int OP>
    __device__ static A prod(__half a, __half b) { return __half2float(__float2half_rn(__fmul_rn(__half2float(a), __half2float(b)))); }
};
template <>
struct OH<__nv_bfloat16> {
    using A = double;
    __device__ static A val(__nv_bfloat16 x) { return widen(x); }
    template <int OP>
    __device__ static A prod(__nv_bfloat16 a, __nv_bfloat16 b) {
        return __bfloat162float(__float2bfloat16_rn(__fmul_rn(__bfloat162float(a), __bfloat162float(b))));
    }
};

template <typename T, int OP>
__device__ __forceinline__ void add3(T a, T b, typename OH<T>::A& ai, typename OH<T>::A& ap, typename OH<T>::A& at) {
    ai += OH<T>::template prod<OP>(a, b);
    ap += OH<T>::val(a);
    at += OH<T>::val(b);
}

__device__ __forceinline__ void emit(unsigned long long* p, unsigned long long v) {
    if (v != 0ull) atomicAdd(p, v);
}
__device__ __forceinline__ void emit(double* p, double v) { *p = v; }  // float launches own their (n, c) outright

// Sum the three per-thread accumulators over the CTA in a fixed order and emit them to out[q * plane + idx].
template <typename A>
__device__ __forceinline__ void block_emit(A ai, A ap, A at, A* out, long long plane, long long idx) {
    __shared__ A red[3][kThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    ai = warp_sum(ai);
    ap = warp_sum(ap);
    at = warp_sum(at);
    if (lane == 0) {
        red[0][warp] = ai;
        red[1][warp] = ap;
        red[2][warp] = at;
    }
    __syncthreads();
    if (threadIdx.x < 3) {
        A s = 0;
        for (int w = 0; w < kThreads / 32; ++w) s += red[threadIdx.x][w];
        emit(out + threadIdx.x * plane + idx, s);
    }
}

// Float launches: every CTA has stored its 3 * width partials at unit_parts[part * 3 * width + e]; the last CTA of the unit
// to arrive sums them over the parts and writes out[k * plane + out_base + col] for e = k * width + col.  Lane l of warp w
// adds parts w, w + 8, ... of entry e0 + l in part order, then the eight warp sums are added in warp order: a fixed order,
// whichever CTA folds.
__device__ __forceinline__ void fold_if_last(const double* unit_parts, unsigned* arrival, long long bps, int width,
                                             double* out, long long plane, long long out_base) {
    __shared__ bool last;
    __shared__ double red[kThreads / 32][32];
    __threadfence();  // this CTA's partials are visible before its arrival is counted
    __syncthreads();
    if (threadIdx.x == 0) last = atomicAdd(arrival, 1u) == (unsigned)(bps - 1);
    __syncthreads();
    if (!last) return;
    __threadfence();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int E = 3 * width;
    for (int e0 = 0; e0 < E; e0 += 32) {
        const int e = e0 + lane;
        double s = 0.0;
        if (e < E) {
#pragma unroll 4
            for (long long p = warp; p < bps; p += kThreads / 32) s += __ldcg(unit_parts + p * E + e);
        }
        red[warp][lane] = s;
        __syncthreads();
        if (warp == 0 && e < E) {
            double t = 0.0;
            for (int w = 0; w < kThreads / 32; ++w) t += red[w][lane];
            const int k = e / width, col = e - k * width;
            out[k * plane + out_base + col] = t;
        }
        __syncthreads();
    }
}

// Planar: grid N * Cp * bps; CTA b reduces elements [part * chunk, ...) of plane (n, c).  16-byte vectors when both plane
// starts share their offset modulo 16 (chunk is a multiple of 1024 elements, so every slice then starts the same way).
template <typename T, int OP>
__global__ void __launch_bounds__(kThreads) onehot_planar_kernel(const T* __restrict__ preds, const T* __restrict__ target,
                                                                 long long p_sn, long long t_sn, long long S, int off, int Cp,
                                                                 long long N, long long bps, long long chunk,
                                                                 typename OH<T>::A* __restrict__ out, double* parts,
                                                                 unsigned* arrivals) {
    using A = typename OH<T>::A;
    constexpr int V = 16 / sizeof(T);
    const long long q = blockIdx.x / bps, part = blockIdx.x % bps;
    const long long n = q / Cp, c = q % Cp + off;
    const long long s0 = part * chunk, s1 = min(S, s0 + chunk);
    const T* P = preds + n * p_sn + c * S;
    const T* Tt = target + n * t_sn + c * S;
    A ai = 0, ap = 0, at = 0;
    long long head = s1;  // [s0, head) and [tail, s1) element by element, [head, tail) in vectors
    long long tail = s1;
    const uintptr_t pa = reinterpret_cast<uintptr_t>(P + s0) & 15, ta = reinterpret_cast<uintptr_t>(Tt + s0) & 15;
    if (pa == ta) {
        head = min(s1, s0 + (long long)(((16 - pa) & 15) / sizeof(T)));
        tail = head + (s1 - head) / V * V;
    }
    for (long long i = s0 + threadIdx.x; i < head; i += kThreads) add3<T, OP>(P[i], Tt[i], ai, ap, at);
    const long long nvec = (tail - head) / V;
    const uint4* Pv = reinterpret_cast<const uint4*>(P + head);
    const uint4* Tv = reinterpret_cast<const uint4*>(Tt + head);
    long long v = threadIdx.x;
    for (; v + kThreads < nvec; v += 2 * kThreads) {  // two vectors in flight per thread
        const uint4 a0 = ld_stream16(Pv + v), b0 = ld_stream16(Tv + v);
        const uint4 a1 = ld_stream16(Pv + v + kThreads), b1 = ld_stream16(Tv + v + kThreads);
        const T* x0 = reinterpret_cast<const T*>(&a0);
        const T* y0 = reinterpret_cast<const T*>(&b0);
        const T* x1 = reinterpret_cast<const T*>(&a1);
        const T* y1 = reinterpret_cast<const T*>(&b1);
#pragma unroll
        for (int k = 0; k < V; ++k) {
            add3<T, OP>(x0[k], y0[k], ai, ap, at);
            add3<T, OP>(x1[k], y1[k], ai, ap, at);
        }
    }
    if (v < nvec) {
        const uint4 a0 = ld_stream16(Pv + v), b0 = ld_stream16(Tv + v);
        const T* x0 = reinterpret_cast<const T*>(&a0);
        const T* y0 = reinterpret_cast<const T*>(&b0);
#pragma unroll
        for (int k = 0; k < V; ++k) add3<T, OP>(x0[k], y0[k], ai, ap, at);
    }
    for (long long i = tail + threadIdx.x; i < s1; i += kThreads) add3<T, OP>(P[i], Tt[i], ai, ap, at);
    if constexpr (std::is_same<A, double>::value) {
        block_emit<A>(ai, ap, at, parts + (q * bps + part) * 3, 1, 0);
        fold_if_last(parts + q * bps * 3, arrivals + q, bps, 1, out, N * Cp, n * Cp + (c - off));
    } else {
        block_emit<A>(ai, ap, at, out, N * Cp, n * Cp + (c - off));
    }
}

// Channels-last: sample n is a row-major [S, C] block.  Grid N * bps; CTA b reduces rows [part * chunk, ...) of sample
// b / bps.  Thread (g, w) = (tid / W, tid % W), W = min(C, 256), G = 256 / W: column j * W + w of rows g, g + G, ...; the
// G partials of a column are then summed in g order.
template <typename T, int OP>
__global__ void __launch_bounds__(kThreads) onehot_cl_kernel(const T* __restrict__ preds, const T* __restrict__ target,
                                                             long long p_sn, long long t_sn, long long S, int C, int off, int Cp,
                                                             long long N, long long bps, long long chunk,
                                                             typename OH<T>::A* __restrict__ out, double* parts,
                                                             unsigned* arrivals) {
    using A = typename OH<T>::A;
    constexpr bool kFloat = std::is_same<A, double>::value;
    __shared__ A part_sum[3][kThreads];
    const long long n = blockIdx.x / bps, part = blockIdx.x % bps;
    const long long r0 = part * chunk, r1 = min(S, r0 + chunk);
    const int W = C < kThreads ? C : kThreads, G = kThreads / W;
    const int g = threadIdx.x / W, w = threadIdx.x - g * W;
    const T* P = preds + n * p_sn;
    const T* Tt = target + n * t_sn;
    const long long plane = N * Cp;
    // integers add into the planes; floats store this CTA's [3][Cp] partials for the fold
    A* dst;
    long long dst_stride;
    if constexpr (kFloat) {
        dst = parts + (n * bps + part) * 3 * Cp;
        dst_stride = Cp;
    } else {
        dst = out + n * Cp;
        dst_stride = plane;
    }
    for (int j0 = 0; j0 < C; j0 += W) {
        const int c = j0 + w;
        A ai = 0, ap = 0, at = 0;
        if (g < G && c < C) {
            long long r = r0 + g;
            for (; r + 3 * G < r1; r += 4 * G) {
                T x[4], y[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    x[k] = P[(r + k * G) * C + c];
                    y[k] = Tt[(r + k * G) * C + c];
                }
#pragma unroll
                for (int k = 0; k < 4; ++k) add3<T, OP>(x[k], y[k], ai, ap, at);
            }
            for (; r < r1; r += G) add3<T, OP>(P[r * C + c], Tt[r * C + c], ai, ap, at);
        }
        part_sum[0][threadIdx.x] = ai;
        part_sum[1][threadIdx.x] = ap;
        part_sum[2][threadIdx.x] = at;
        __syncthreads();
        for (int e = threadIdx.x; e < 3 * W; e += kThreads) {  // 3 * W entries, up to 3 per thread
            const int k = e / W, col = e - k * W;
            const int cc = j0 + col;
            if (cc < C && cc >= off) {
                A s = 0;
                for (int gg = 0; gg < G; ++gg) s += part_sum[k][gg * W + col];
                emit(dst + k * dst_stride + (cc - off), s);
            }
        }
        __syncthreads();
    }
    if constexpr (kFloat) fold_if_last(parts + n * bps * 3 * Cp, arrivals + n, bps, Cp, out, plane, n * Cp);
}

// ---- launchers -----------------------------------------------------------------------------------------------------------
long long cdiv(long long a, long long b) { return (a + b - 1) / b; }

// slices per row of `len` elements for `rows` independent rows: about 8 CTAs per SM in all, at least `min_len` per slice,
// slice length a multiple of `align`
void split(long long rows, long long len, long long min_len, long long align, long long max_len, long long* bps, long long* chunk) {
    const long long want = cdiv((long long)sm_count() * 8, rows);
    long long b = std::min(want, std::max(1ll, len / min_len));
    long long ch = cdiv(cdiv(len, std::max(1ll, b)), align) * align;
    if (ch > max_len) ch = max_len;
    if (ch < 1) ch = 1;
    *chunk = ch;
    *bps = std::max(1ll, cdiv(len, ch));
}

int launch_index(const long long* p, const long long* t, long long N, int C, long long S, int off, int Cp,
                 unsigned long long* out, unsigned* err, cudaStream_t st) {
    long long bps, chunk;
    split(N, S, 8 * kThreads * kIdxUnroll, kThreads * kIdxUnroll, kMaxSlice, &bps, &chunk);
    MB200_REQUIRE(N * bps < (1ll << 31), "sample count %lld too large for one launch", (long long)N);
    const unsigned grid = (unsigned)(N * bps);
    if (Cp <= kSmemMaxClasses) {
        index_counts_kernel<true><<<grid, kThreads, (size_t)3 * Cp * sizeof(unsigned), st>>>(p, t, S, C, off, Cp, N, bps, chunk, out, err);
    } else {
        index_counts_kernel<false><<<grid, kThreads, 0, st>>>(p, t, S, C, off, Cp, N, bps, chunk, out, err);
    }
    count_launch();
    return check_cuda(cudaGetLastError(), "segmentation index-count launch");
}

// Slices of a one-hot launch: integer and float sums share the split; float launches keep at most kMaxFoldParts partials per
// unit and at most kMaxFoldLoads partial values per unit, so the last CTA's fold stays a few microseconds.
constexpr long long kMaxFoldParts = 256;
constexpr long long kMaxFoldLoads = 1 << 16;

void onehot_geometry(long long N, int Cp, long long S, int layout, bool is_float, long long* bps, long long* chunk) {
    const bool planar = layout == MB200_SEG_PLANAR;
    if (planar) split(N * Cp, S, 16 * kThreads * 4, 1024, kMaxSlice, bps, chunk);
    else split(N, S, 64, 1, kMaxSlice, bps, chunk);
    if (!is_float) return;
    const long long width = planar ? 1 : Cp;
    const long long cap = std::max(1ll, std::min(kMaxFoldParts, kMaxFoldLoads / (3 * width)));
    if (*bps > cap) {
        *chunk = cdiv(cdiv(S, cap), planar ? 1024 : 1) * (planar ? 1024 : 1);
        *bps = std::max(1ll, cdiv(S, *chunk));
    }
}

// float64 partials and per-unit arrival counters of a float launch (0 for integer launches)
long long onehot_scratch_bytes(long long N, int Cp, long long S, int layout, bool is_float) {
    if (!is_float || N == 0 || S == 0) return 0;
    long long bps, chunk;
    onehot_geometry(N, Cp, S, layout, true, &bps, &chunk);
    const long long units = layout == MB200_SEG_PLANAR ? N * Cp : N;
    const long long width = layout == MB200_SEG_PLANAR ? 1 : Cp;
    return cdiv(units * 4, 16) * 16 + units * bps * 3 * width * 8;
}

template <typename T, int OP>
int launch_onehot(const void* preds, const void* target, long long N, int C, long long S, int layout, long long p_sn,
                  long long t_sn, int off, int Cp, void* counts, void* scratch, long long scratch_bytes, cudaStream_t st) {
    using A = typename OH<T>::A;
    constexpr bool kFloat = std::is_same<A, double>::value;
    const T* p = reinterpret_cast<const T*>(preds);
    const T* t = reinterpret_cast<const T*>(target);
    A* out = reinterpret_cast<A*>(counts);
    long long bps, chunk;
    onehot_geometry(N, Cp, S, layout, kFloat, &bps, &chunk);
    const long long units = layout == MB200_SEG_PLANAR ? N * Cp : N;
    unsigned* arrivals = nullptr;
    double* parts = nullptr;
    if (kFloat) {
        MB200_REQUIRE(scratch != nullptr && scratch_bytes >= onehot_scratch_bytes(N, Cp, S, layout, true) &&
                          (reinterpret_cast<uintptr_t>(scratch) & 15) == 0,
                      "float inputs need 16-byte aligned scratch of mb200_segmentation_scratch_bytes(...) bytes");
        arrivals = reinterpret_cast<unsigned*>(scratch);
        parts = reinterpret_cast<double*>(reinterpret_cast<char*>(scratch) + cdiv(units * 4, 16) * 16);
        MB200_CUDA_OK(cudaMemsetAsync(arrivals, 0, (size_t)(units * 4), st));
    }
    MB200_REQUIRE(units * bps < (1ll << 31), "n * num_classes too large for one launch");
    if (layout == MB200_SEG_PLANAR) {
        onehot_planar_kernel<T, OP><<<(unsigned)(units * bps), kThreads, 0, st>>>(p, t, p_sn, t_sn, S, off, Cp, N, bps, chunk, out,
                                                                                 parts, arrivals);
    } else {
        onehot_cl_kernel<T, OP><<<(unsigned)(units * bps), kThreads, 0, st>>>(p, t, p_sn, t_sn, S, C, off, Cp, N, bps, chunk, out,
                                                                             parts, arrivals);
    }
    count_launch();
    return check_cuda(cudaGetLastError(), "segmentation one-hot launch");
}

template <typename T>
int launch_onehot_op(int op, const void* preds, const void* target, long long N, int C, long long S, int layout,
                     long long p_sn, long long t_sn, int off, int Cp, void* counts, cudaStream_t st) {
    if (op == MB200_SEG_AND)
        return launch_onehot<T, MB200_SEG_AND>(preds, target, N, C, S, layout, p_sn, t_sn, off, Cp, counts, nullptr, 0, st);
    return launch_onehot<T, MB200_SEG_MUL>(preds, target, N, C, S, layout, p_sn, t_sn, off, Cp, counts, nullptr, 0, st);
}

}  // namespace
}  // namespace mb200

using namespace mb200;

// =====================================================================================================
// C-ABI
// =====================================================================================================
extern "C" int mb200_segmentation_overlap_counts(const void* preds, int preds_dtype, const void* target, int target_dtype,
                                                 int64_t n, int64_t num_classes, int64_t inner, int input_format, int layout,
                                                 int64_t preds_batch_stride, int64_t target_batch_stride, int op,
                                                 int drop_background, void* counts, void* scratch, int64_t scratch_bytes,
                                                 uint32_t* err_flag, void* stream) {
    MB200_REQUIRE(n >= 0 && inner >= 0 && num_classes >= 1, "bad sizes");
    MB200_REQUIRE(num_classes < (1ll << 31), "num_classes exceeds int32");
    MB200_REQUIRE(input_format == MB200_SEG_INDEX || input_format == MB200_SEG_ONE_HOT, "unknown input_format %d", input_format);
    MB200_REQUIRE(op == MB200_SEG_AND || op == MB200_SEG_MUL, "unknown op %d", op);
    const bool is_float = is_float_tag<kNoF64>(preds_dtype);
    if (input_format == MB200_SEG_INDEX) {
        MB200_REQUIRE(preds_dtype == MB200_I64 && target_dtype == MB200_I64, "index labels must be int64 (dtype tags %d, %d)",
                      preds_dtype, target_dtype);
    } else {
        MB200_REQUIRE(preds_dtype == target_dtype, "preds and target must share a dtype (tags %d, %d)", preds_dtype, target_dtype);
        MB200_REQUIRE(is_float || is_label_tag(preds_dtype), "unsupported dtype tag %d", preds_dtype);
        MB200_REQUIRE(!is_float || op == MB200_SEG_MUL, "floating-point inputs support only the product");
        MB200_REQUIRE(layout == MB200_SEG_PLANAR || layout == MB200_SEG_CHANNELS_LAST, "unknown layout %d", layout);
    }
    MB200_REQUIRE(counts != nullptr, "NULL pointer");
    const int off = (drop_background && num_classes > 1) ? 1 : 0;
    const int C = (int)num_classes, Cp = C - off;
    if (n == 0) return 0;
    MB200_REQUIRE(inner == 0 || (preds && target), "NULL pointer");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    // integer launches add into the planes (several CTAs per plane); float launches store every entry
    if (!is_float || inner == 0) MB200_CUDA_OK(cudaMemsetAsync(counts, 0, (size_t)(3 * n * Cp * 8), st));
    if (inner == 0) return 0;
    if (input_format == MB200_SEG_INDEX)
        return launch_index(reinterpret_cast<const long long*>(preds), reinterpret_cast<const long long*>(target), n, C, inner, off,
                            Cp, reinterpret_cast<unsigned long long*>(counts), err_flag, st);
    const long long p_sn = preds_batch_stride, t_sn = target_batch_stride;
    switch (preds_dtype) {
        case MB200_BOOL: return launch_onehot_op<Bool>(op, preds, target, n, C, inner, layout, p_sn, t_sn, off, Cp, counts, st);
        case MB200_U8: return launch_onehot_op<unsigned char>(op, preds, target, n, C, inner, layout, p_sn, t_sn, off, Cp, counts, st);
        case MB200_I8: return launch_onehot_op<signed char>(op, preds, target, n, C, inner, layout, p_sn, t_sn, off, Cp, counts, st);
        case MB200_I16: return launch_onehot_op<short>(op, preds, target, n, C, inner, layout, p_sn, t_sn, off, Cp, counts, st);
        case MB200_I32: return launch_onehot_op<int>(op, preds, target, n, C, inner, layout, p_sn, t_sn, off, Cp, counts, st);
        case MB200_I64: return launch_onehot_op<long long>(op, preds, target, n, C, inner, layout, p_sn, t_sn, off, Cp, counts, st);
        default:  // f32 / f16 / bf16: the tag was checked above
            return with_float_type<kNoF64>(preds_dtype, [&](auto t) {
                return launch_onehot<typename decltype(t)::type, MB200_SEG_MUL>(preds, target, n, C, inner, layout, p_sn, t_sn, off,
                                                                                Cp, counts, scratch, scratch_bytes, st);
            });
    }
}

extern "C" int64_t mb200_segmentation_scratch_bytes(int64_t n, int64_t num_classes, int64_t inner, int input_format, int layout,
                                                   int dtype, int drop_background) {
    if (n < 0 || inner < 0 || num_classes < 1 || num_classes >= (1ll << 31)) return -1;
    if (input_format != MB200_SEG_ONE_HOT || !is_float_tag<kNoF64>(dtype)) return 0;
    const int Cp = (int)num_classes - ((drop_background && num_classes > 1) ? 1 : 0);
    return onehot_scratch_bytes(n, Cp, inner, layout, true);
}
