// K13 — per-row KL divergence (reference seam: functional/regression/kl_divergence.py:25-46 `_kld_update`).
//
// The reference chain for probabilities is eight ATen passes with [N, d] temporaries (two row sums, two broadcast divisions,
// p / q, log, multiply, masked fill, row sum); for log-probabilities four (exp, subtract, multiply, row sum).  Here a warp owns
// a row: one pass over p and q for the two normalising sums, a second pass over the SAME row (it is in L1 / L2: the HBM
// traffic stays one read of p and q) for  sum_j xlogy(p_j / sum p,  (p_j / sum p) / (q_j / sum q))  with  xlogy(0, .) = 0
// (utilities/compute.py:32-44), the elementwise arithmetic in the input precision class (float for f32 / f16 / bf16, double
// for f64) like ATen's, row sums accumulated in double.  Output: measures [N] in the input dtype.
#include "common.cuh"

namespace mb200 {

// f32 / f16 / bf16: elementwise in float
template <typename T>
__global__ void __launch_bounds__(256) kl_rows_kernel(const T* __restrict__ p, const T* __restrict__ q, long long n, int d,
                                                      int log_prob, T* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const long long wstep = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long r = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < n; r += wstep) {
        const T* __restrict__ pr = p + r * d;
        const T* __restrict__ qr = q + r * d;
        double acc = 0.0;
        if constexpr (sizeof(T) == 4) {
            // float rows of a multiple of 4 columns: 16-byte loads, lane l owns columns [4 l, 4 l + 4) of every 128-column
            // stripe (four times fewer load instructions and four times the bytes in flight: the scalar loop below stalls on
            // the long scoreboard)
            if ((d & 3) == 0 && ((reinterpret_cast<uintptr_t>(pr) | reinterpret_cast<uintptr_t>(qr)) & 15) == 0) {
                const float4* __restrict__ p4 = reinterpret_cast<const float4*>(pr);
                const float4* __restrict__ q4 = reinterpret_cast<const float4*>(qr);
                const int d4 = d >> 2;
                if (log_prob) {
#pragma unroll 2
                    for (int j = lane; j < d4; j += 32) {
                        const float4 a = p4[j], b = q4[j];
                        acc += (double)(expf(a.x) * (a.x - b.x)) + (double)(expf(a.y) * (a.y - b.y)) +
                               ((double)(expf(a.z) * (a.z - b.z)) + (double)(expf(a.w) * (a.w - b.w)));
                    }
                } else {
                    double sp = 0.0, sq = 0.0;
#pragma unroll 4
                    for (int j = lane; j < d4; j += 32) {
                        const float4 a = p4[j], b = q4[j];
                        sp += ((double)a.x + (double)a.y) + ((double)a.z + (double)a.w);
                        sq += ((double)b.x + (double)b.y) + ((double)b.z + (double)b.w);
                    }
                    const float fp = (float)warp_sum(sp), fq = (float)warp_sum(sq);
#pragma unroll 2
                    for (int j = lane; j < d4; j += 32) {
                        const float4 a = p4[j], b = q4[j];
                        const float pa[4] = {a.x / fp, a.y / fp, a.z / fp, a.w / fp};
                        const float qb[4] = {b.x / fq, b.y / fq, b.z / fq, b.w / fq};
#pragma unroll
                        for (int k = 0; k < 4; ++k)
                            if (pa[k] != 0.f) acc += (double)(pa[k] * logf(pa[k] / qb[k]));
                    }
                }
                acc = warp_sum(acc);
                if (lane == 0) out[r] = narrow<T>((float)acc);
                continue;
            }
        }
        if (log_prob) {
#pragma unroll 4
            for (int j = lane; j < d; j += 32) {
                const float a = widen(pr[j]), b = widen(qr[j]);
                acc += (double)(expf(a) * (a - b));
            }
        } else {
            double sp = 0.0, sq = 0.0;
#pragma unroll 8
            for (int j = lane; j < d; j += 32) sp += (double)widen(pr[j]), sq += (double)widen(qr[j]);
            const float fp = (float)warp_sum(sp), fq = (float)warp_sum(sq);
#pragma unroll 4
            for (int j = lane; j < d; j += 32) {
                const float a = widen(pr[j]) / fp, b = widen(qr[j]) / fq;
                if (a != 0.f) acc += (double)(a * logf(a / b));  // a NaN `a` takes this branch too, like `res[x == 0] = 0`
            }
        }
        acc = warp_sum(acc);
        if (lane == 0) out[r] = narrow<T>((float)acc);
    }
}

__global__ void __launch_bounds__(256) kl_rows_kernel_f64(const double* __restrict__ p, const double* __restrict__ q,
                                                          long long n, int d, int log_prob, double* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const long long wstep = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long r = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < n; r += wstep) {
        const double* __restrict__ pr = p + r * d;
        const double* __restrict__ qr = q + r * d;
        double acc = 0.0;
        if (log_prob) {
            for (int j = lane; j < d; j += 32) acc += exp(pr[j]) * (pr[j] - qr[j]);
        } else {
            double sp = 0.0, sq = 0.0;
            for (int j = lane; j < d; j += 32) sp += pr[j], sq += qr[j];
            sp = warp_sum(sp), sq = warp_sum(sq);
            for (int j = lane; j < d; j += 32) {
                const double a = pr[j] / sp, b = qr[j] / sq;
                if (a != 0.0) acc += a * log(a / b);
            }
        }
        acc = warp_sum(acc);
        if (lane == 0) out[r] = acc;
    }
}

}  // namespace mb200

using namespace mb200;

extern "C" int mb200_kl_divergence_rows(const void* p, const void* q, int dtype, int64_t n, int64_t d, int log_prob,
                                        void* measures_out, void* stream) {
    MB200_REQUIRE(n >= 0 && d >= 0 && d < (1ll << 31), "bad sizes");
    if (n == 0) return 0;
    MB200_REQUIRE(measures_out && (d == 0 || (p && q)), "NULL pointer");
    MB200_REQUIRE(is_float_tag(dtype), "distributions must be f32/f16/bf16/f64 (dtype tag %d)", dtype);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    long long grid = (n + 7) / 8;
    const long long cap = (long long)sm_count() * 8;
    if (grid > cap) grid = cap;
    with_float_type(dtype, [&](auto t) {
        using T = typename decltype(t)::type;
        const T *pt = reinterpret_cast<const T*>(p), *qt = reinterpret_cast<const T*>(q);
        if constexpr (std::is_same_v<T, double>)
            kl_rows_kernel_f64<<<(unsigned)grid, 256, 0, st>>>(pt, qt, n, (int)d, log_prob, reinterpret_cast<T*>(measures_out));
        else
            kl_rows_kernel<T><<<(unsigned)grid, 256, 0, st>>>(pt, qt, n, (int)d, log_prob, reinterpret_cast<T*>(measures_out));
        return 0;
    });
    count_launch();
    return check_cuda(cudaGetLastError(), "kl divergence launch");
}
