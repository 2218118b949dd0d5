// Shared device/host helpers for the metrics_b200 sm_90a kernels.
// Everything here is header-only; the C-ABI entry points live in the individual .cu files and are
// declared in include/metrics_b200.h.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <limits.h>
#include <stdint.h>
#include <stdio.h>

#include <type_traits>
#include <unordered_map>
#include <utility>

#include "../../include/metrics_b200.h"

namespace mb200 {

constexpr int kWarp = 32;
constexpr unsigned kFull = 0xffffffffu;

// ---- host-side error plumbing -------------------------------------------------------------------
void set_error(const char* fmt, ...);
int check_cuda(cudaError_t e, const char* what);
int sm_count();  // cached multiprocessor count of the current device
void count_launch();  // adds one to mb200_launch_count(): called once per kernel launch

#define MB200_CUDA_OK(expr)                                      \
    do {                                                         \
        int _rc = ::mb200::check_cuda((expr), #expr);            \
        if (_rc != 0) return _rc;                                \
    } while (0)

#define MB200_REQUIRE(cond, ...)                                 \
    do {                                                         \
        if (!(cond)) {                                           \
            ::mb200::set_error(__VA_ARGS__);                     \
            return MB200_ERR_INVALID;                            \
        }                                                        \
    } while (0)

// ---- dtype tags (enum mb200_dtype) -----------------------------------------------------------------
// An entry point checks its score tag with is_float_tag before its first CUDA call, under its own error code and message,
// then picks the kernel instantiation with with_float_type.  kNoF64 selects the score types of kernels without an f64
// instantiation: f32 / f16 / bf16.
constexpr bool kNoF64 = false;

template <bool kF64 = true>
constexpr bool is_float_tag(int d) {
    return d == MB200_F32 || d == MB200_F16 || d == MB200_BF16 || (kF64 && d == MB200_F64);
}
constexpr bool is_label_tag(int d) { return d >= MB200_I64 && d <= MB200_BOOL; }

template <typename T>
struct As {
    using type = T;
};
constexpr int kNoType = INT_MIN;

// Returns f(As<T>{}) for the score type T of `dtype`: float, __half, __nv_bfloat16, and double unless kF64 is false.
// Any tag for which is_float_tag<kF64> is false returns kNoType without calling f.
template <bool kF64 = true, typename F>
int with_float_type(int dtype, F&& f) {
    switch (dtype) {
        case MB200_F32: return f(As<float>{});
        case MB200_F16: return f(As<__half>{});
        case MB200_BF16: return f(As<__nv_bfloat16>{});
        case MB200_F64:
            if constexpr (kF64) return f(As<double>{});
            return kNoType;
        default: return kNoType;
    }
}

// Returns f(As<T>{}) for the integer type T of `dtype`: long long, int, short, signed char, unsigned char.  MB200_BOOL and
// every non-integer tag return kNoType without calling f.
template <typename F>
int with_label_type(int dtype, F&& f) {
    switch (dtype) {
        case MB200_I64: return f(As<long long>{});
        case MB200_I32: return f(As<int>{});
        case MB200_I16: return f(As<short>{});
        case MB200_I8: return f(As<signed char>{});
        case MB200_U8: return f(As<unsigned char>{});
        default: return kNoType;
    }
}

// ---- device helpers -------------------------------------------------------------------------------
// Streaming 16-byte load: data is consumed exactly once, keep it out of L1.
__device__ __forceinline__ uint4 ld_stream16(const void* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}

// Integer label load with a runtime dtype tag (labels are one load per row/sample: the switch is free).
__device__ __forceinline__ long long load_label(const void* p, int dtype, long long i) {
    switch (dtype) {
        case MB200_I64: return reinterpret_cast<const long long*>(p)[i];
        case MB200_I32: return reinterpret_cast<const int*>(p)[i];
        case MB200_I16: return reinterpret_cast<const short*>(p)[i];
        case MB200_I8: return reinterpret_cast<const signed char*>(p)[i];
        case MB200_U8: return reinterpret_cast<const unsigned char*>(p)[i];
        case MB200_BOOL: return reinterpret_cast<const unsigned char*>(p)[i] != 0;
        default: return 0;
    }
}

// `ignore_index` as the reference compares it with labels of this dtype: `target != ignore_index` casts the Python int to
// the target's dtype first (two's complement wrap), so with uint8 targets 257 is 1 and -1 is 255, with int8 255 is -1.
// int64 keeps the value; a bool target promotes the comparison to int64, so it is not wrapped either.
inline long long label_ignore_index(long long v, int dtype) {
    switch (dtype) {
        case MB200_I32: return (int32_t)(uint32_t)v;
        case MB200_I16: return (int16_t)(uint16_t)v;
        case MB200_I8: return (int8_t)(uint8_t)v;
        case MB200_U8: return (uint8_t)v;
        default: return v;
    }
}

__device__ __forceinline__ void red_add_u64(long long* addr, unsigned long long v) {
    atomicAdd(reinterpret_cast<unsigned long long*>(addr), v);
}

// Order-preserving u32 key of an f32: a > b (IEEE, non-NaN) <=> key(a) > key(b); -0 and +0 share a key;
// NaN maps to the largest key (torch.argmax treats NaN as maximal).
__device__ __forceinline__ unsigned f32_order_key(float v) {
    unsigned b = __float_as_uint(v);
    if ((b & 0x7fffffffu) > 0x7f800000u) return 0xffffffffu;
    if (b == 0x80000000u) b = 0u;
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float f32_from_order_key(unsigned k) {
    unsigned b = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
    return __uint_as_float(b);
}

// The logistic function in fp32 math, as ATen's CUDA sigmoid computes it (the logits-to-probabilities step of
// normalize_logits_if_needed); NaN stays NaN.
__device__ __forceinline__ float sigmoid_f32(float v) { return 1.0f / (1.0f + expf(-v)); }

__device__ __forceinline__ unsigned long long f64_order_key(double v) {
    unsigned long long b = (unsigned long long)__double_as_longlong(v);
    if ((b & 0x7fffffffffffffffull) > 0x7ff0000000000000ull) return ~0ull;
    if (b == 0x8000000000000000ull) b = 0ull;
    return (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);
}

// ---- score types ----------------------------------------------------------------------------------------------------
// What a kernel does with one value of a score type T (float, __half, __nv_bfloat16, double) once with_float_type has
// picked T.  half and bfloat16 widen exactly to float and compute in float; double computes in double.  Keys and score
// comparisons see every type as float32 (to_f32), as ATen compares half and bfloat16; float64 is rounded to float there.
__device__ __forceinline__ float widen(float v) { return v; }
__device__ __forceinline__ float widen(__half v) { return __half2float(v); }
__device__ __forceinline__ float widen(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ double widen(double v) { return v; }
template <typename T>
using compute_t = decltype(widen(std::declval<T>()));

template <typename T>
__device__ __forceinline__ float to_f32(T v) { return (float)widen(v); }

// a computed value stored in T, rounded to nearest
template <typename T>
__device__ __forceinline__ T narrow(compute_t<T> x) {
    if constexpr (std::is_same_v<T, __half>) return __float2half_rn(x);
    else if constexpr (std::is_same_v<T, __nv_bfloat16>) return __float2bfloat16_rn(x);
    else return x;
}
// the value a tensor of dtype T would hold
template <typename T>
__device__ __forceinline__ compute_t<T> round_to(compute_t<T> x) { return widen(narrow<T>(x)); }

// element i of a tensor of any float or integer tag, exactly (integers up to 2^53)
__device__ __forceinline__ double load_f64(const void* p, int dtype, long long i) {
    switch (dtype) {
        case MB200_F32: return reinterpret_cast<const float*>(p)[i];
        case MB200_F16: return widen(reinterpret_cast<const __half*>(p)[i]);
        case MB200_BF16: return widen(reinterpret_cast<const __nv_bfloat16*>(p)[i]);
        case MB200_F64: return reinterpret_cast<const double*>(p)[i];
        default: return (double)load_label(p, dtype, i);
    }
}

// ascending sort of this key == descending sort of the score; NaN first (torch.argsort(descending=True) puts NaN first)
__device__ __forceinline__ unsigned f32_desc_key(float v) { return ~f32_order_key(v); }

// butterfly over the 32 lanes (offsets 16, 8, 4, 2, 1): every lane ends with the same sum / maximum
template <typename V>
__device__ __forceinline__ V warp_sum(V v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(kFull, v, o));
    return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(kFull, v, o));
    return v;
}

// ---- key tiles ------------------------------------------------------------------------------------------------------
// This CTA's 32 x 32 tile of [n, C] row-major scores (samples from blockIdx.x * 32, classes from blockIdx.y * 32) as
// tile[sample][class] = f32_desc_key(to_f32(score)), read along the class dimension by 256 threads.  Both key-packing
// transposes, the exact curves' (curve.cu) and the class-sharded peer exchange's (peer.cu), load through it: the sharded
// curves rely on the two producing the same keys.  Entries outside [n, C] are not written.
template <typename T>
__device__ __forceinline__ void load_desc_key_tile(const T* __restrict__ preds, int n, int C, unsigned (&tile)[32][33]) {
    const int n0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int j = ty; j < 32; j += 8) {
        const int nn = n0 + j, cc = c0 + tx;
        if (nn < n && cc < C) tile[j][tx] = f32_desc_key(to_f32(preds[(size_t)nn * C + cc]));
    }
}

// Opt a kernel into more than 48 KB of dynamic shared memory.  The attribute is per (function, device): remember which
// devices were configured per function address, so a process that drives several GPUs configures each of them.
template <typename Kernel>
inline cudaError_t ensure_dynamic_smem(Kernel kern, int bytes) {
    static thread_local std::unordered_map<const void*, unsigned long long> done;
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    unsigned long long& mask = done[reinterpret_cast<const void*>(kern)];
    if (dev < 64 && ((mask >> dev) & 1ull)) return cudaSuccess;
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess && dev < 64) mask |= 1ull << dev;
    return e;
}

}  // namespace mb200
