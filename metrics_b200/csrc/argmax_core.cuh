// Warp-level row argmax with torch.argmax semantics (first maximal index, NaN maximal, -0 == +0).
//
// One "vector" is 16 bytes; one "chunk" is kVPL vectors per lane (2 KiB of a row).  Per chunk:
//   phase 1  each lane reduces its 4 vectors to per-vector pair-maxima with NaN-propagating packed max
//            (HMNMX2 / 3-input VHMNMX for 16-bit types, max.NaN.f32 for fp32), the warp agrees on the chunk maximum
//            with ONE REDUX.MAX over an order-preserving u32 key;
//   phase 2  4 packed compares per lane tell which of its vectors contain the maximum, ONE REDUX.MIN over
//            (vector slot * 32 + lane) elects the first such vector in column order, and only that vector is searched
//            element-wise (warp-uniform branch), the winning lane broadcasting the element index.
#pragma once
#include "common.cuh"

namespace mb200 {

constexpr int kVPL = 4;  // vectors per lane per chunk

template <typename T>
struct RowTraits;

__device__ __forceinline__ float fmax_nan(float a, float b) {
    float r;
    asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}

// ---- 16-bit element types share everything but the intrinsic names -------------------------------------------------
#define MB200_DEFINE_HALF_TRAITS(ELEM, PAIR, F2PAIR, ELEM2FLOAT, LOW, HIGH)                                         \
    template <>                                                                                                      \
    struct RowTraits<ELEM> {                                                                                         \
        static constexpr int EPV = 8;                                                                                \
        using Acc = PAIR;                                                                                            \
        static __device__ __forceinline__ Acc as2(unsigned u) { return *reinterpret_cast<Acc*>(&u); }               \
        static __device__ __forceinline__ Acc vmax(const uint4& v) {                                                 \
            return __hmax2_nan(__hmax2_nan(as2(v.x), as2(v.y)), __hmax2_nan(as2(v.z), as2(v.w)));                    \
        }                                                                                                            \
        static __device__ __forceinline__ Acc amax(Acc a, Acc b) { return __hmax2_nan(a, b); }                       \
        static __device__ __forceinline__ unsigned lane_key(Acc a) {                                                 \
            return f32_order_key(ELEM2FLOAT(__hmax_nan(LOW(a), HIGH(a))));                                           \
        }                                                                                                            \
        /* does the pair-maximum `pm` of a vector contain the row maximum? */                                        \
        template <bool kNaN>                                                                                         \
        static __device__ __forceinline__ bool holds(Acc pm, unsigned rowkey) {                                      \
            if (kNaN) return ~__heq2_mask(pm, pm) != 0u;                                                             \
            return __heq2_mask(pm, F2PAIR(f32_from_order_key(rowkey))) != 0u;                                        \
        }                                                                                                            \
        /* index (0..7) of the first element of `v` equal to the row maximum (or first NaN); 8 if none */            \
        template <bool kNaN>                                                                                         \
        static __device__ __forceinline__ int first_in(const uint4& v, unsigned rowkey) {                            \
            unsigned e0, e1, e2, e3;                                                                                 \
            if (kNaN) {                                                                                              \
                e0 = ~__heq2_mask(as2(v.x), as2(v.x));                                                               \
                e1 = ~__heq2_mask(as2(v.y), as2(v.y));                                                               \
                e2 = ~__heq2_mask(as2(v.z), as2(v.z));                                                               \
                e3 = ~__heq2_mask(as2(v.w), as2(v.w));                                                               \
            } else {                                                                                                 \
                const Acc m = F2PAIR(f32_from_order_key(rowkey));                                                    \
                e0 = __heq2_mask(as2(v.x), m);                                                                       \
                e1 = __heq2_mask(as2(v.y), m);                                                                       \
                e2 = __heq2_mask(as2(v.z), m);                                                                       \
                e3 = __heq2_mask(as2(v.w), m);                                                                       \
            }                                                                                                        \
            const unsigned w0 = __byte_perm(e0, e1, 0x6420); /* bytes = elements 0..3 */                             \
            const unsigned w1 = __byte_perm(e2, e3, 0x6420); /* bytes = elements 4..7 */                             \
            if (w0) return (__ffs(w0) - 1) >> 3;                                                                     \
            if (w1) return 4 + ((__ffs(w1) - 1) >> 3);                                                               \
            return 8;                                                                                                \
        }                                                                                                            \
        static __device__ __forceinline__ float to_f32(ELEM x) { return ELEM2FLOAT(x); }                             \
    };

MB200_DEFINE_HALF_TRAITS(__nv_bfloat16, __nv_bfloat162, __float2bfloat162_rn, __bfloat162float, __low2bfloat16,
                         __high2bfloat16)
MB200_DEFINE_HALF_TRAITS(__half, __half2, __float2half2_rn, __half2float, __low2half, __high2half)
#undef MB200_DEFINE_HALF_TRAITS

template <>
struct RowTraits<float> {
    static constexpr int EPV = 4;
    using Acc = float;
    static __device__ __forceinline__ Acc vmax(const uint4& v) {
        return fmax_nan(fmax_nan(__uint_as_float(v.x), __uint_as_float(v.y)),
                        fmax_nan(__uint_as_float(v.z), __uint_as_float(v.w)));
    }
    static __device__ __forceinline__ Acc amax(Acc a, Acc b) { return fmax_nan(a, b); }
    static __device__ __forceinline__ unsigned lane_key(Acc a) { return f32_order_key(a); }
    template <bool kNaN>
    static __device__ __forceinline__ bool holds(Acc pm, unsigned rowkey) {
        if (kNaN) return pm != pm;
        return pm == f32_from_order_key(rowkey);
    }
    template <bool kNaN>
    static __device__ __forceinline__ int first_in(const uint4& v, unsigned rowkey) {
        const float x0 = __uint_as_float(v.x), x1 = __uint_as_float(v.y), x2 = __uint_as_float(v.z),
                    x3 = __uint_as_float(v.w);
        if (kNaN) return (x0 != x0) ? 0 : (x1 != x1) ? 1 : (x2 != x2) ? 2 : (x3 != x3) ? 3 : 4;
        const float m = f32_from_order_key(rowkey);
        return (x0 == m) ? 0 : (x1 == m) ? 1 : (x2 == m) ? 2 : (x3 == m) ? 3 : 4;
    }
    static __device__ __forceinline__ float to_f32(float x) { return x; }
};

// Generic order key used by the scalar paths (any float dtype, incl. f64).
template <typename T>
__device__ __forceinline__ unsigned long long order_key(T x) {
    return (unsigned long long)f32_order_key(RowTraits<T>::to_f32(x));
}
template <>
__device__ __forceinline__ unsigned long long order_key<double>(double x) {
    return f64_order_key(x);
}

// A chunk of one row held in registers.
struct Chunk {
    uint4 v[kVPL];
};

struct GlobalVecLoader {  // streaming 16-byte loads straight from HBM (consumed once: no L1 allocation)
    const uint4* __restrict__ base;
    __device__ __forceinline__ uint4 operator()(int vi) const { return ld_stream16(base + vi); }
};

// Vector slots past the end of the row re-read the row's LAST vector (index clamp) instead of being predicated off:
// duplicates cannot change the maximum, and a duplicate sits in a later slot than the original, so the REDUX.MIN over
// slots still elects the true first column.
template <typename Loader>
__device__ __forceinline__ void load_chunk(Chunk& c, const Loader& load, int cv, int nvec, int lane) {
#pragma unroll
    for (int j = 0; j < kVPL; ++j) c.v[j] = load(min(cv + j * kWarp + lane, nvec - 1));
}

template <typename T, bool kNaN>
__device__ __forceinline__ unsigned chunk_first_col(const Chunk& c, const typename RowTraits<T>::Acc (&pm)[kVPL],
                                                    unsigned ckey, int cv, int lane) {
    using TR = RowTraits<T>;
    unsigned slot = 0x7fffffffu;
#pragma unroll
    for (int j = kVPL - 1; j >= 0; --j)
        if (TR::template holds<kNaN>(pm[j], ckey)) slot = (unsigned)(j * kWarp + lane);
    slot = __reduce_min_sync(kFull, slot);  // always valid: some lane holds the maximum
    const int js = (int)(slot >> 5), ls = (int)(slot & 31);
    int e;
    if (js == 0) e = TR::template first_in<kNaN>(c.v[0], ckey);
    else if (js == 1) e = TR::template first_in<kNaN>(c.v[1], ckey);
    else if (js == 2) e = TR::template first_in<kNaN>(c.v[2], ckey);
    else e = TR::template first_in<kNaN>(c.v[3], ckey);
    e = __shfl_sync(kFull, e, ls);
    return (unsigned)((cv + (int)slot) * TR::EPV + e);
}

// (key, first column) of the maximum of one chunk; identical in all lanes.
template <typename T>
__device__ __forceinline__ void chunk_argmax(const Chunk& c, int cv, int lane, unsigned& ckey, unsigned& ccol) {
    using TR = RowTraits<T>;
    typename TR::Acc pm[kVPL];
#pragma unroll
    for (int j = 0; j < kVPL; ++j) pm[j] = TR::vmax(c.v[j]);
    const typename TR::Acc lane_max = TR::amax(TR::amax(pm[0], pm[1]), TR::amax(pm[2], pm[3]));
    ckey = __reduce_max_sync(kFull, TR::lane_key(lane_max));
    ccol = (ckey == 0xffffffffu) ? chunk_first_col<T, true>(c, pm, ckey, cv, lane)
                                 : chunk_first_col<T, false>(c, pm, ckey, cv, lane);
}

// Whole-row argmax through a loader (used by the shared-memory staged path and by multi-chunk rows).
template <typename T, typename Loader>
__device__ __forceinline__ int warp_row_argmax_vec(const Loader& load, int nvec, int lane) {
    unsigned best_key = 0;
    int best_col = 0;
    for (int cv = 0; cv < nvec; cv += kVPL * kWarp) {
        Chunk c;
        load_chunk(c, load, cv, nvec, lane);
        unsigned ckey, ccol;
        chunk_argmax<T>(c, cv, lane, ckey, ccol);
        // strictly-greater keeps the earliest chunk on ties (and the first NaN chunk: all NaN keys are equal)
        if (cv == 0 || ckey > best_key) {
            best_key = ckey;
            best_col = (int)ccol;
        }
    }
    return best_col;
}

// Warp-per-row argmax, scalar loads (any alignment / any C).  All lanes return the same column.
template <typename T>
__device__ __forceinline__ int warp_row_argmax_scalar(const T* __restrict__ row, int C, int lane) {
    unsigned long long bk = 0;
    int bc = 0x7fffffff;
    for (int c = lane; c < C; c += kWarp) {
        const unsigned long long k = order_key<T>(row[c]);
        if (bc == 0x7fffffff || k > bk) {
            bk = k;
            bc = c;
        }
    }
    // lanes without any element (C < 32) carry key 0 / col INT_MAX and can never win against a real element
    unsigned long long mk = bk;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long other = __shfl_xor_sync(kFull, mk, o);
        mk = other > mk ? other : mk;
    }
    const unsigned col = (bk == mk && bc != 0x7fffffff) ? (unsigned)bc : 0x7fffffffu;
    return (int)__reduce_min_sync(kFull, col);
}

// Thread-per-(outer, inner) argmax over a strided class dimension: element c at base[c * stride].
template <typename T>
__device__ __forceinline__ int thread_argmax_strided(const T* __restrict__ base, int C, long long stride) {
    unsigned long long bk = order_key<T>(base[0]);
    int bc = 0;
    for (int c = 1; c < C; ++c) {
        const unsigned long long k = order_key<T>(base[(long long)c * stride]);
        if (k > bk) {
            bk = k;
            bc = c;
        }
    }
    return bc;
}

}  // namespace mb200
