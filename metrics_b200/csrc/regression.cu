// K9 — regression running sums: one fused map-reduce pass producing every sum a metric's `update` needs.
//
// Reference op chains replaced (src/torchmetrics/functional/regression/): mse.py:22-40, mae.py:22-42, mape.py:22-45,
// symmetric_mape.py:22-46, wmape.py:22-38, log_mse.py:22-34, log_cosh.py:32-52, minkowski.py:21-38, r2.py:22-45 (also
// used by rse.py), explained_variance.py:25-40 — each 2-5 elementwise + reduction launches per call.
// Per-element terms are evaluated in fp32 with the reference's operation order (fp64 for fp64 inputs); the sums are
// accumulated in fp64 with a fixed reduction order (per-thread strided rows -> fixed shared-memory tree -> ordered sum of
// the per-CTA partials), so results are bitwise reproducible and at least as accurate as the reference's fp32 `torch.sum`.
#include "common.cuh"

#include "regression_terms.cuh"

namespace mb200 {

// grid.x CTAs of 256 threads laid out as rows x cols_per_block; grid.y tiles the columns.
template <typename T, bool kDouble, bool kTweedie = false>
__global__ void __launch_bounds__(256) reg_partial_kernel(const T* __restrict__ preds, const T* __restrict__ target,
                                                          long long n, int d, int op, double param, double eps,
                                                          int cols_per_block, double* __restrict__ partial) {
    __shared__ double sm[256];
    const int K = reg_num_sums(op);
    const int rows_per_block = 256 / cols_per_block;
    const int c_local = threadIdx.x % cols_per_block;
    const int r_local = threadIdx.x / cols_per_block;
    const int c = blockIdx.y * cols_per_block + c_local;
    double acc[kRegMaxK] = {0.0, 0.0, 0.0, 0.0};
    if (r_local < rows_per_block && c < d) {
        for (long long r = (long long)blockIdx.x * rows_per_block + r_local; r < n; r += (long long)gridDim.x * rows_per_block) {
            const long long i = r * d + c;
            if (kDouble) {
                double out[kRegMaxK];
                reg_terms<double, kTweedie>(op, (double)widen(preds[i]), (double)widen(target[i]), param, eps, out);
                for (int k = 0; k < K; ++k) acc[k] += out[k];
            } else {
                float out[kRegMaxK];
                reg_terms<float, kTweedie>(op, to_f32(preds[i]), to_f32(target[i]), (float)param, (float)eps, out);
                for (int k = 0; k < K; ++k) acc[k] += (double)out[k];
            }
        }
    }
    // fixed-order reduction over the rows of the CTA, one sum at a time
    for (int k = 0; k < K; ++k) {
        __syncthreads();
        sm[threadIdx.x] = acc[k];
        __syncthreads();
        if (r_local == 0 && c < d) {
            double s = 0.0;
            for (int r = 0; r < rows_per_block; ++r) s += sm[r * cols_per_block + c_local];
            partial[((size_t)blockIdx.x * K + k) * d + c] = s;
        }
    }
}

// d == 1 (one output: the common case): flat, vectorised map-reduce.  Every thread streams 16-byte vectors of both inputs
// (two independent vector pairs in flight), accumulates its terms in fp64, then a fixed shuffle / shared-memory tree folds
// the CTA (deterministic order).  The generic kernel above walks one element per thread per iteration with 16 warps per SM
// and is latency-bound; this one is bound by HBM.
constexpr int kRegFlatThreads = 512;
// kOp >= 0 fixes the op at compile time (the switch over ops and the loops over the op's sums fold away: MSE / MAE, the
// hottest ops, get their own instantiations); kOp < 0 reads it from the argument.
template <typename T, bool kDouble, bool kTweedie = false, int kOp = -1>
__global__ void __launch_bounds__(kRegFlatThreads) reg_flat_kernel(const T* __restrict__ preds, const T* __restrict__ target,
                                                                   long long n, int op_arg, double param, double eps,
                                                                   double* __restrict__ partial) {
    __shared__ double sm[kRegFlatThreads / 32];
    const int op = kOp >= 0 ? kOp : op_arg;
    const int K = kOp >= 0 ? reg_num_sums(kOp) : reg_num_sums(op);
    constexpr int kVec = 16 / (int)sizeof(T);
    double acc[kRegMaxK] = {0.0, 0.0, 0.0, 0.0};
    const long long gtid = (long long)blockIdx.x * kRegFlatThreads + threadIdx.x;
    const long long stride = (long long)gridDim.x * kRegFlatThreads;
    const bool aligned = ((reinterpret_cast<uintptr_t>(preds) | reinterpret_cast<uintptr_t>(target)) & 15) == 0;
    const long long nvec = aligned ? n / kVec : 0;
    auto consume = [&](const T& pv, const T& tv) {
        if (kDouble) {
            double out[kRegMaxK];
            reg_terms<double, kTweedie>(op, (double)pv, (double)tv, param, eps, out);
            for (int k = 0; k < K; ++k) acc[k] += out[k];
        } else {
            float out[kRegMaxK];
            reg_terms<float, kTweedie>(op, to_f32(pv), to_f32(tv), (float)param, (float)eps, out);
            for (int k = 0; k < K; ++k) acc[k] += (double)out[k];
        }
    };
    const uint4* __restrict__ pv4 = reinterpret_cast<const uint4*>(preds);
    const uint4* __restrict__ tv4 = reinterpret_cast<const uint4*>(target);
    long long v = gtid;
    for (; v + stride < nvec; v += 2 * stride) {  // two vector pairs in flight
        const uint4 p0 = ld_stream16(pv4 + v), t0 = ld_stream16(tv4 + v);
        const uint4 p1 = ld_stream16(pv4 + v + stride), t1 = ld_stream16(tv4 + v + stride);
        const T* a0 = reinterpret_cast<const T*>(&p0);
        const T* b0 = reinterpret_cast<const T*>(&t0);
        const T* a1 = reinterpret_cast<const T*>(&p1);
        const T* b1 = reinterpret_cast<const T*>(&t1);
#pragma unroll
        for (int e = 0; e < kVec; ++e) consume(a0[e], b0[e]);
#pragma unroll
        for (int e = 0; e < kVec; ++e) consume(a1[e], b1[e]);
    }
    for (; v < nvec; v += stride) {
        const uint4 p0 = ld_stream16(pv4 + v), t0 = ld_stream16(tv4 + v);
        const T* a0 = reinterpret_cast<const T*>(&p0);
        const T* b0 = reinterpret_cast<const T*>(&t0);
#pragma unroll
        for (int e = 0; e < kVec; ++e) consume(a0[e], b0[e]);
    }
    for (long long i = nvec * kVec + gtid; i < n; i += stride) consume(preds[i], target[i]);  // tail / unaligned
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int k = 0; k < K; ++k) {
        double s = acc[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(kFull, s, o);
        __syncthreads();
        if (lane == 0) sm[warp] = s;
        __syncthreads();
        if (threadIdx.x == 0) {
            double tot = 0.0;
#pragma unroll
            for (int w = 0; w < kRegFlatThreads / 32; ++w) tot += sm[w];
            partial[(size_t)blockIdx.x * K + k] = tot;
        }
    }
}

// out[k][c] = sum over CTAs (in order) of partial[cta][k][c]
__global__ void reg_final_kernel(const double* __restrict__ partial, int n_cta, int K, int d, double* __restrict__ out) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= K * d) return;
    double s = 0.0;
    for (int b = 0; b < n_cta; ++b) s += partial[(size_t)b * K * d + idx];
    out[idx] = s;
}

}  // namespace mb200

using namespace mb200;

extern "C" int mb200_regression_num_sums(int op) { return (op >= 0 && op <= REG_LAST) ? reg_num_sums(op) : -1; }

extern "C" int64_t mb200_regression_scratch_doubles(int64_t n, int64_t d, int op) {
    if (n < 0 || d < 1 || op < 0 || op > REG_LAST) return -1;
    return (int64_t)296 * reg_num_sums(op) * d + 8;
}

extern "C" int mb200_regression_sums(const void* preds, const void* target, int dtype, int64_t n, int64_t d, int op,
                                     double param, double epsilon, double* out_sums, double* scratch, void* stream) {
    MB200_REQUIRE(n >= 0 && d >= 1 && d < (1 << 30), "bad sizes");
    MB200_REQUIRE(op >= 0 && op <= REG_LAST, "unknown regression op %d", op);
    MB200_REQUIRE(out_sums && scratch, "NULL pointer");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int K = reg_num_sums(op);
    const int cols_per_block = d >= 256 ? 256 : (int)d;
    const int rows_per_block = 256 / cols_per_block;
    long long want = (n + (long long)rows_per_block * 8 - 1) / ((long long)rows_per_block * 8);
    const int col_tiles = (int)((d + cols_per_block - 1) / cols_per_block);
    long long cap = 296 / col_tiles;
    if (cap < 1) cap = 1;
    int gx = (int)(want < 1 ? 1 : (want > cap ? cap : want));
    if ((int64_t)gx * K * d + 8 > mb200_regression_scratch_doubles(n, d, op)) gx = 1;
    if (n > 0) MB200_REQUIRE(preds && target, "NULL pointer");
    MB200_REQUIRE(is_float_tag(dtype), "regression inputs must be floating point (dtype tag %d)", dtype);
    if (d == 1 && n > 0) {  // flat vectorised path
        constexpr int per_cta = kRegFlatThreads * 8;
        long long fg = (n + per_cta - 1) / per_cta;
        if (fg > 296) fg = 296;  // scratch holds 296 partial rows
        const int g1 = (int)(fg < 1 ? 1 : fg);
        with_float_type(dtype, [&](auto t) {
            using T = typename decltype(t)::type;
            constexpr bool DBL = std::is_same_v<T, double>;
            const T *p = (const T*)preds, *q = (const T*)target;
            if (op == REG_TWEEDIE)
                reg_flat_kernel<T, DBL, true><<<g1, kRegFlatThreads, 0, st>>>(p, q, n, op, param, epsilon, scratch);
            else if (op == REG_MSE)
                reg_flat_kernel<T, DBL, false, REG_MSE><<<g1, kRegFlatThreads, 0, st>>>(p, q, n, op, param, epsilon, scratch);
            else if (op == REG_MAE)
                reg_flat_kernel<T, DBL, false, REG_MAE><<<g1, kRegFlatThreads, 0, st>>>(p, q, n, op, param, epsilon, scratch);
            else
                reg_flat_kernel<T, DBL, false><<<g1, kRegFlatThreads, 0, st>>>(p, q, n, op, param, epsilon, scratch);
            return 0;
        });
        reg_final_kernel<<<1, 256, 0, st>>>(scratch, g1, K, 1, out_sums);
        count_launch();
        count_launch();
        return check_cuda(cudaGetLastError(), "regression sums launch");
    }
    const dim3 grid((unsigned)gx, (unsigned)col_tiles);
    with_float_type(dtype, [&](auto t) {
        using T = typename decltype(t)::type;
        constexpr bool DBL = std::is_same_v<T, double>;
        const T *p = (const T*)preds, *q = (const T*)target;
        if (op == REG_TWEEDIE)
            reg_partial_kernel<T, DBL, true><<<grid, 256, 0, st>>>(p, q, n, (int)d, op, param, epsilon, cols_per_block, scratch);
        else
            reg_partial_kernel<T, DBL, false><<<grid, 256, 0, st>>>(p, q, n, (int)d, op, param, epsilon, cols_per_block, scratch);
        return 0;
    });
    reg_final_kernel<<<(int)((K * d + 255) / 256), 256, 0, st>>>(scratch, gx, K, (int)d, out_sums);
    count_launch();
    count_launch();
    return check_cuda(cudaGetLastError(), "regression sums launch");
}
