// K17 — rank correlations (SpearmanCorrCoef, KendallRankCorrCoef) on sm_90a.
//
// Reference replaced (src/torchmetrics/): functional/regression/spearman.py ranks every column with an argsort in the input
// dtype and averages ties with one Python iteration per repeated value; functional/regression/kendall.py compares every row
// with all later rows in a Python loop (O(n^2) work, n iterations).
//
// Rank phase (both metrics, once per variable): an order key per element (-0 -> +0, NaN after +inf), the column-segmented
// LSD radix sort of radix_sort.cuh with the row as payload, then one tie-group pass over the sorted keys.  A tie group may
// span any number of tiles: the start of the group holding a tile's first key (and the end of the one holding its last key)
// comes from a binary search over the sorted column, every other boundary from block scans of the head flags.  Each NaN is
// a group of its own.  The pass scatters one value per row back to its original position — Spearman the doubled average
// rank start + end + 1, Kendall the dense rank — and sums the tie statistics per element: with k = position - group start,
// sum k = sum t(t-1)/2, sum 3k(k-1) = sum t(t-1)(t-2) and sum 3k(k+1) = sum (t^3 - t), exact in u64 / u128.
// Spearman finish: the y pass multiplies its doubled rank with x's (gathered by row) into an exact u128 sum; the moments
// then follow from closed forms on exact integers, the last few operations in float64.
// Kendall concordance: the y pass emits, in y order, key = dense x rank (all ones when either value is NaN) and payload =
// dense y rank; a stable sort by that key gives (x, y) order with the NaN rows last.  Discordant pairs D are the inversions
// of the dense-y sequence in that order, counted level by level from the most significant bit (a wavelet-tree pass): per
// level one column scan counts the 1-bits before each 0-bit of its prefix group, then every group is stably partitioned.
// The group bounds come from the y histogram's prefix sums.  C = n0 - n1 - n2 + n3 - D (Knight) over the non-NaN rows.
#include <algorithm>
#include <type_traits>

#include "common.cuh"
#include "radix_sort.cuh"
#include "../../include/metrics_b200_rankcorr.h"

namespace mb200 {

namespace {

typedef unsigned long long u64;
typedef unsigned __int128 u128;
typedef __int128 i128;

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kItems = 8;
constexpr int kTile = kThreads * kItems;  // elements per tie / scan tile
constexpr unsigned kNoRank = 0xffffffffu;  // dense x rank of a NaN row

enum { kSpearmanX, kSpearmanY, kKendallX, kKendallY };

// per column and variable; word-addressed so that u128 sums can be added with two u64 atomics
struct ColStats {
    u64 distinct, pairs, p1[2], cube[2], pad[2];
};
struct KendallCol {
    u64 m, n1, n2, n3, disc, pad[3];
};

size_t align16(size_t v) { return (v + 15) & ~(size_t)15; }
int grid_for(long long n) {
    long long g = (n + kThreads - 1) / kThreads;
    const long long cap = (long long)sm_count() * 16;
    return (int)std::max(1LL, std::min(g, cap));
}
int bits_of(u64 v) {
    int b = 0;
    while (v) ++b, v >>= 1;
    return b;
}

// Returns f(As<T>{}) for the rankable types: the float tags, int32 and int64.
template <typename F>
int with_rank_type(int dtype, F&& f) {
    if (dtype == MB200_I32) return f(As<int>{});
    if (dtype == MB200_I64) return f(As<long long>{});
    return with_float_type(dtype, f);
}

// ---- order keys: ascending key = ascending value, -0 == +0, NaN = all ones (2-byte keys for the half types) ----------------
__device__ __forceinline__ unsigned order_key(float v) { return f32_order_key(v); }
__device__ __forceinline__ u64 order_key(double v) { return f64_order_key(v); }
__device__ __forceinline__ unsigned order_key(__half v) {
    unsigned h = __half_as_ushort(v);
    if ((h & 0x7fffu) > 0x7c00u) return 0xffffu;
    if (h == 0x8000u) h = 0u;
    return (h & 0x8000u) ? (~h & 0xffffu) : (h | 0x8000u);
}
__device__ __forceinline__ unsigned order_key(__nv_bfloat16 v) { return f32_order_key(__bfloat162float(v)) >> 16; }
__device__ __forceinline__ unsigned order_key(int v) { return (unsigned)v ^ 0x80000000u; }
__device__ __forceinline__ u64 order_key(long long v) { return (u64)v ^ 0x8000000000000000ull; }

template <typename T, typename KeyT>
__global__ void __launch_bounds__(kThreads) pack_kernel(const T* __restrict__ in, int n, int d, KeyT* __restrict__ keys,
                                                        unsigned* __restrict__ rows) {
    const long long total = (long long)n * d;
    for (long long o = blockIdx.x * (long long)kThreads + threadIdx.x; o < total; o += (long long)gridDim.x * kThreads) {
        const int col = (int)(o / n), i = (int)(o - (long long)col * n);
        keys[o] = (KeyT)order_key(in[(long long)i * d + col]);
        rows[o] = (unsigned)i;
    }
}

// ---- block-wide helpers ------------------------------------------------------------------------------------------------
// Exclusive scan of one value per thread in thread order (kReverse: from the last thread down).  op is associative and
// commutative; id its identity.  wsum: kWarps words of shared memory.
template <bool kReverse, typename T, typename Op>
__device__ __forceinline__ T block_exclusive(T v, Op op, T id, T* wsum) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    T incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const T t = kReverse ? __shfl_down_sync(kFull, incl, o) : __shfl_up_sync(kFull, incl, o);
        if (kReverse ? lane + o < 32 : lane >= o) incl = op(incl, t);
    }
    T ex = kReverse ? __shfl_down_sync(kFull, incl, 1) : __shfl_up_sync(kFull, incl, 1);
    if (kReverse ? lane == 31 : lane == 0) ex = id;
    if (kReverse ? lane == 0 : lane == 31) wsum[warp] = incl;
    __syncthreads();
    T pre = id;
    if (kReverse) {
        for (int w = kWarps - 1; w > warp; --w) pre = op(pre, wsum[w]);
    } else {
        for (int w = 0; w < warp; ++w) pre = op(pre, wsum[w]);
    }
    __syncthreads();
    return op(pre, ex);
}

// Sum over the block, valid in thread 0.  wsum: 2 * kWarps u64 words.
__device__ __forceinline__ u128 block_sum_u128(u128 v, u64* wsum) {
    u64 lo = (u64)v, hi = (u64)(v >> 64);
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const u64 l2 = __shfl_down_sync(kFull, lo, o), h2 = __shfl_down_sync(kFull, hi, o);
        const u64 s = lo + l2;
        hi += h2 + (s < lo ? 1ull : 0ull);
        lo = s;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) wsum[2 * warp] = lo, wsum[2 * warp + 1] = hi;
    __syncthreads();
    u128 s = 0;
    if (threadIdx.x == 0)
        for (int w = 0; w < kWarps; ++w) s += ((u128)wsum[2 * w + 1] << 64) | wsum[2 * w];
    __syncthreads();
    return s;
}
__device__ __forceinline__ u64 block_sum_u64(u64 v, u64* wsum) { return (u64)block_sum_u128(v, wsum); }

// Exact u128 accumulation with two u64 atomics: the carry of the low word goes to the high word exactly once.
__device__ __forceinline__ void atomic_add_u128(u64* w, u128 v) {
    const u64 lo = (u64)v, hi = (u64)(v >> 64);
    const u64 old = atomicAdd(w, lo);
    const u64 carry = old + lo < old ? 1ull : 0ull;
    if (hi + carry) atomicAdd(w + 1, hi + carry);
}

__device__ __forceinline__ double u128_to_double(u128 v) {
    return (double)(u64)(v >> 64) * 18446744073709551616.0 + (double)(u64)v;
}
__device__ __forceinline__ double i128_to_double(i128 v) { return v < 0 ? -u128_to_double((u128)(-v)) : u128_to_double((u128)v); }
__device__ __forceinline__ u128 load_u128(const u64* w) { return ((u128)w[1] << 64) | w[0]; }

// ---- tie-group pass ------------------------------------------------------------------------------------------------------
template <typename KeyT>
struct TieArgs {
    const KeyT* keys;          // [d][n] sorted per column
    const unsigned* rows;      // [d][n] payload: the row of each sorted key
    int n, tiles;
    bool nan_keys;             // float input: the all-ones key is NaN
    KeyT nan_key;
    const unsigned* head_excl; // [d][tiles + 1] heads before each tile (Kendall)
    ColStats* stats;           // [d]
    unsigned* rank_out;        // x pass: [d][n] by row
    const unsigned* rank_x;    // y pass: the x pass's values by row
    u64* spear_sum;            // Spearman y: [d][2] u128 sum of 2r_x * 2r_y
    unsigned* k2;              // Kendall y: [d][n] composite key, in y order
    unsigned* v2;              // Kendall y: [d][n] dense y rank, in y order
    unsigned* cnt;             // Kendall y: [d][n + 1] histogram of the dense y rank over the non-NaN rows
    unsigned k2_invalid;
};

template <typename KeyT, int kMode>
__global__ void __launch_bounds__(kThreads) ties_kernel(TieArgs<KeyT> a) {
    constexpr bool kSpearman = kMode == kSpearmanX || kMode == kSpearmanY;
    __shared__ KeyT sk[kTile + 2];  // sk[0] = key before the tile, sk[1 + j] = tile key j, sk[cnt + 1] = key after the tile
    __shared__ u64 wsum[2 * kWarps];
    __shared__ int edge[2];
    __shared__ unsigned vex[kMode == kKendallY ? kTile : 1];
    const int col = blockIdx.x / a.tiles, tile = blockIdx.x % a.tiles, n = a.n;
    const int base = tile * kTile, cnt = min(kTile, n - base);
    const size_t off = (size_t)col * n;
    const KeyT* __restrict__ k = a.keys + off;
    for (int j = threadIdx.x; j < cnt; j += kThreads) sk[1 + j] = k[base + j];
    if (threadIdx.x == 0) sk[0] = base > 0 ? k[base - 1] : (KeyT)0;
    if (threadIdx.x == 1) sk[cnt + 1] = base + cnt < n ? k[base + cnt] : (KeyT)0;
    auto is_nan = [&](KeyT v) { return a.nan_keys && v == a.nan_key; };
    if (threadIdx.x == 32) {  // start of the group that holds the tile's first key
        const KeyT v = k[base];
        int s = base;
        if (base > 0 && !is_nan(v) && k[base - 1] == v) {
            int lo = 0, hi = base - 1;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (k[mid] < v) lo = mid + 1; else hi = mid;
            }
            s = lo;
        }
        edge[0] = s;
    }
    if (kSpearman && threadIdx.x == 64) {  // end of the group that holds the tile's last key
        const int last = base + cnt - 1;
        const KeyT v = k[last];
        int e = last + 1;
        if (e < n && !is_nan(v) && k[e] == v) {
            int lo = e + 1, hi = n;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (k[mid] == v) lo = mid + 1; else hi = mid;
            }
            e = lo;
        }
        edge[1] = e;
    }
    __syncthreads();

    const int j0 = threadIdx.x * kItems;
    bool head[kItems], nhead[kItems];
    int last_head = -1, first_next = INT_MAX;
    unsigned heads = 0;
#pragma unroll
    for (int i = 0; i < kItems; ++i) {
        const int j = j0 + i, p = base + j;
        head[i] = nhead[i] = false;
        if (j < cnt) {
            const KeyT v = sk[1 + j];
            head[i] = p == 0 || is_nan(v) || v != sk[j];
            nhead[i] = p + 1 == n || is_nan(sk[2 + j]) || sk[2 + j] != v;
            if (head[i]) last_head = p, ++heads;
            if (nhead[i] && first_next == INT_MAX) first_next = p + 1;
        }
    }
    const int s_pre = block_exclusive<false>(last_head, [](int x, int y) { return max(x, y); }, -1, reinterpret_cast<int*>(wsum));
    int e_suf = INT_MAX;
    if (kSpearman) e_suf = block_exclusive<true>(first_next, [](int x, int y) { return min(x, y); }, INT_MAX, reinterpret_cast<int*>(wsum));
    unsigned dense = 0;
    if (!kSpearman)
        dense = a.head_excl[(size_t)col * (a.tiles + 1) + tile] +
                block_exclusive<false>(heads, [](unsigned x, unsigned y) { return x + y; }, 0u, reinterpret_cast<unsigned*>(wsum));

    int s[kItems], e[kItems];
    {
        int cur = s_pre;
#pragma unroll
        for (int i = 0; i < kItems; ++i) {
            if (head[i]) cur = base + j0 + i;
            s[i] = cur >= 0 ? cur : edge[0];
        }
    }
    if (kSpearman) {
        int cur = e_suf;
#pragma unroll
        for (int i = kItems - 1; i >= 0; --i) {
            if (nhead[i]) cur = base + j0 + i + 1;
            e[i] = cur != INT_MAX ? cur : edge[1];
        }
    }

    u64 pairs = 0;
    u128 p1 = 0, cube = 0, prod = 0;
    bool valid[kItems];
    unsigned dr[kItems];
    unsigned nvalid = 0;
#pragma unroll
    for (int i = 0; i < kItems; ++i) {
        const int j = j0 + i, p = base + j;
        valid[i] = false;
        dr[i] = 0;
        if (j >= cnt) continue;
        const u64 kk = (u64)(p - s[i]);
        pairs += kk;
        p1 += (u128)(3 * kk * (kk ? kk - 1 : 0));
        cube += (u128)(3 * kk * (kk + 1));
        const unsigned row = a.rows[off + p];
        if (!kSpearman) {
            if (head[i]) ++dense;
            dr[i] = dense - 1;
        }
        if (kMode == kSpearmanX) a.rank_out[off + row] = (unsigned)(s[i] + e[i] + 1);
        if (kMode == kSpearmanY) prod += (u128)((u64)a.rank_x[off + row] * (u64)(unsigned)(s[i] + e[i] + 1));
        if (kMode == kKendallX) a.rank_out[off + row] = is_nan(sk[1 + j]) ? kNoRank : dr[i];
        if (kMode == kKendallY) {
            const unsigned rx = a.rank_x[off + row];
            valid[i] = !is_nan(sk[1 + j]) && rx != kNoRank;
            a.k2[off + p] = valid[i] ? rx : a.k2_invalid;
            a.v2[off + p] = dr[i];
            nvalid += valid[i];
        }
    }
    if (kMode == kKendallY) {
        // histogram of the dense y rank over the non-NaN rows: one atomic per (tie group, tile)
        unsigned run = block_exclusive<false>(nvalid, [](unsigned x, unsigned y) { return x + y; }, 0u, reinterpret_cast<unsigned*>(wsum));
#pragma unroll
        for (int i = 0; i < kItems; ++i) {
            if (j0 + i < cnt) vex[j0 + i] = run;
            run += valid[i];
        }
        __syncthreads();
#pragma unroll
        for (int i = 0; i < kItems; ++i) {
            const int j = j0 + i;
            if (j >= cnt || !(nhead[i] || j == cnt - 1)) continue;
            const int first = max(s[i], base) - base;
            const unsigned c = vex[j] + valid[i] - vex[first];
            if (c) atomicAdd(&a.cnt[(size_t)col * (n + 1) + dr[i]], c);
        }
    }
    const u64 distinct = block_sum_u64(heads, wsum);
    const u64 pair_sum = block_sum_u64(pairs, wsum);
    const u128 p1_sum = block_sum_u128(p1, wsum);
    const u128 cube_sum = block_sum_u128(cube, wsum);
    u128 prod_sum = 0;
    if (kMode == kSpearmanY) prod_sum = block_sum_u128(prod, wsum);
    if (threadIdx.x == 0) {
        ColStats& st = a.stats[col];
        atomicAdd(&st.distinct, distinct);
        atomicAdd(&st.pairs, pair_sum);
        if (!kSpearman) atomic_add_u128(st.p1, p1_sum);
        atomic_add_u128(st.cube, cube_sum);
        if (kMode == kSpearmanY) atomic_add_u128(a.spear_sum + 2 * col, prod_sum);
    }
}

// ---- column scans: tile sums, a scan of the tile sums per column, then the exclusive prefix of every element ----------------
template <typename KeyT>
struct HeadSrc {  // 1 at the first key of every tie group (each NaN its own)
    const KeyT* keys;
    int n;
    bool nan_keys;
    KeyT nan_key;
    __device__ bool active(int) const { return true; }
    __device__ unsigned operator()(int col, int i) const {
        const KeyT* k = keys + (size_t)col * n;
        const KeyT v = k[i];
        return i == 0 || (nan_keys && v == nan_key) || v != k[i - 1];
    }
};
struct CountSrc {  // the dense-y histogram
    const unsigned* cnt;
    int n;
    __device__ bool active(int) const { return true; }
    __device__ unsigned operator()(int col, int i) const { return cnt[(size_t)col * (n + 1) + i]; }
};
// Bit b of the dense-y sequence of the inversion level b.  Column c runs levels levels(c) - 1 .. 0 (values < 2^levels);
// its sequence ping-pongs between buf0 (level levels - 1 reads it) and buf1.
struct BitSrc {
    const unsigned* buf0;
    const unsigned* buf1;
    const ColStats* ystats;
    const KendallCol* kc;
    int n, b;
    __device__ int levels(int col) const {
        const u64 dd = ystats[col].distinct;
        return dd > 1 ? 64 - __clzll((long long)(dd - 1)) : 0;
    }
    __device__ bool active(int col) const { return b < levels(col); }
    __device__ const unsigned* in(int col) const { return ((levels(col) - 1 - b) & 1) ? buf1 : buf0; }
    __device__ unsigned operator()(int col, int i) const {
        return (u64)i < kc[col].m ? (in(col)[(size_t)col * n + i] >> b) & 1u : 0u;
    }
};

template <typename Src, bool kPairs>
__global__ void __launch_bounds__(kThreads) tile_reduce_kernel(Src src, int n, int tiles, unsigned* __restrict__ tsum,
                                                               KendallCol* kc) {
    __shared__ u64 wsum[2 * kWarps];
    const int col = blockIdx.x / tiles, tile = blockIdx.x % tiles;
    if (!src.active(col)) return;
    const int base = tile * kTile, cnt = min(kTile, n - base);
    u64 s = 0, pr = 0;
    for (int j = threadIdx.x; j < cnt; j += kThreads) {
        const u64 v = src(col, base + j);
        s += v;
        if (kPairs) pr += v * (v ? v - 1 : 0) / 2;
    }
    s = block_sum_u64(s, wsum);
    if (kPairs) pr = block_sum_u64(pr, wsum);
    if (threadIdx.x == 0) {
        tsum[(size_t)col * (tiles + 1) + tile] = (unsigned)s;
        if (kPairs && pr) atomicAdd(&kc[col].n2, pr);
    }
}

// one CTA per column: exclusive scan of the tile sums in place, the total at index `tiles`
__global__ void __launch_bounds__(1024) tile_scan_kernel(unsigned* __restrict__ tsum, int tiles) {
    __shared__ unsigned ws[32];
    unsigned* t = tsum + (size_t)blockIdx.x * (tiles + 1);
    const int per = (tiles + 1023) / 1024;
    const int b = threadIdx.x * per, e = min(tiles, b + per);
    unsigned s = 0;
    for (int i = b; i < e; ++i) s += t[i];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned incl = s;
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned v = __shfl_up_sync(kFull, incl, o);
        if (lane >= o) incl += v;
    }
    if (lane == 31) ws[warp] = incl;
    __syncthreads();
    unsigned run = incl - s;
    for (int w = 0; w < warp; ++w) run += ws[w];
    for (int i = b; i < e; ++i) {
        const unsigned c = t[i];
        t[i] = run;
        run += c;
    }
    if (threadIdx.x == 1023) t[tiles] = run;
}

// out[col][i] = exclusive prefix of src over the column, out[col][n] = the column total.  May run in place over CountSrc.
template <typename Src>
__global__ void __launch_bounds__(kThreads) tile_apply_kernel(Src src, int n, int tiles, const unsigned* __restrict__ tsum,
                                                              unsigned* out) {
    __shared__ unsigned wsum[kWarps];
    const int col = blockIdx.x / tiles, tile = blockIdx.x % tiles;
    if (!src.active(col)) return;
    const int base = tile * kTile, cnt = min(kTile, n - base);
    const int j0 = threadIdx.x * kItems;
    unsigned v[kItems], tot = 0;
#pragma unroll
    for (int i = 0; i < kItems; ++i) {
        v[i] = j0 + i < cnt ? src(col, base + j0 + i) : 0u;
        tot += v[i];
    }
    unsigned run = tsum[(size_t)col * (tiles + 1) + tile] +
                   block_exclusive<false>(tot, [](unsigned x, unsigned y) { return x + y; }, 0u, wsum);
    unsigned* o = out + (size_t)col * (n + 1);
#pragma unroll
    for (int i = 0; i < kItems; ++i) {
        if (j0 + i < cnt) o[base + j0 + i] = run;
        run += v[i];
    }
    if (tile == tiles - 1 && threadIdx.x == 0) o[n] = tsum[(size_t)col * (tiles + 1) + tiles];
}

// ---- Kendall: runs of the (x, y)-sorted non-NaN rows -> n1, n3 and the row count m -------------------------------------
__global__ void __launch_bounds__(kThreads) runs_kernel(const unsigned* __restrict__ k2, const unsigned* __restrict__ v2, int n,
                                                        int tiles, unsigned invalid, KendallCol* kc) {
    __shared__ unsigned sk[kTile + 1], sv[kTile + 1];
    __shared__ u64 wsum[2 * kWarps];
    __shared__ int edge[2];
    const int col = blockIdx.x / tiles, tile = blockIdx.x % tiles;
    const int base = tile * kTile, cnt = min(kTile, n - base);
    const size_t off = (size_t)col * n;
    const unsigned* k = k2 + off;
    const unsigned* v = v2 + off;
    for (int j = threadIdx.x; j < cnt; j += kThreads) sk[1 + j] = k[base + j], sv[1 + j] = v[base + j];
    if (threadIdx.x == 0) {
        sk[0] = base > 0 ? k[base - 1] : 0u;
        sv[0] = base > 0 ? v[base - 1] : 0u;
    }
    if (threadIdx.x == 32) {  // start of the x run holding the tile's first row
        const unsigned kv = k[base];
        int lo = 0, hi = base;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (k[mid] < kv) lo = mid + 1; else hi = mid;
        }
        edge[0] = lo;
    }
    if (threadIdx.x == 64) {  // start of the (x, y) run holding it
        const unsigned kv = k[base], vv = v[base];
        int lo = 0, hi = base;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (k[mid] < kv || (k[mid] == kv && v[mid] < vv)) lo = mid + 1; else hi = mid;
        }
        edge[1] = lo;
    }
    __syncthreads();
    const int j0 = threadIdx.x * kItems;
    bool hx[kItems], hxy[kItems];
    int lx = -1, lxy = -1;
#pragma unroll
    for (int i = 0; i < kItems; ++i) {
        const int j = j0 + i, p = base + j;
        hx[i] = hxy[i] = false;
        if (j < cnt) {
            hx[i] = p == 0 || sk[1 + j] != sk[j];
            hxy[i] = hx[i] || sv[1 + j] != sv[j];
            if (hx[i]) lx = p;
            if (hxy[i]) lxy = p;
        }
    }
    auto mx = [](int x, int y) { return max(x, y); };
    int cx = block_exclusive<false>(lx, mx, -1, reinterpret_cast<int*>(wsum));
    int cxy = block_exclusive<false>(lxy, mx, -1, reinterpret_cast<int*>(wsum));
    u64 n1 = 0, n3 = 0, m = 0;
#pragma unroll
    for (int i = 0; i < kItems; ++i) {
        const int j = j0 + i, p = base + j;
        if (j >= cnt) continue;
        if (hx[i]) cx = p;
        if (hxy[i]) cxy = p;
        if (sk[1 + j] == invalid) continue;
        n1 += (u64)(p - (cx >= 0 ? cx : edge[0]));
        n3 += (u64)(p - (cxy >= 0 ? cxy : edge[1]));
        ++m;
    }
    n1 = block_sum_u64(n1, wsum);
    n3 = block_sum_u64(n3, wsum);
    m = block_sum_u64(m, wsum);
    if (threadIdx.x == 0) {
        if (n1) atomicAdd(&kc[col].n1, n1);
        if (n3) atomicAdd(&kc[col].n3, n3);
        if (m) atomicAdd(&kc[col].m, m);
    }
}

// ---- Kendall: one inversion level.  Counts, for every 0-bit, the 1-bits before it in its prefix group (the discordant pairs
// whose highest differing bit is b), then stably partitions every group by bit b. ---------------------------------------
__global__ void __launch_bounds__(kThreads) level_scatter_kernel(BitSrc src, unsigned* buf0, unsigned* buf1,
                                                                 const unsigned* __restrict__ cum, const unsigned* __restrict__ ones,
                                                                 KendallCol* kc, int n, int tiles) {
    __shared__ u64 wsum[2 * kWarps];
    const int col = blockIdx.x / tiles, tile = blockIdx.x % tiles;
    if (!src.active(col)) return;
    const int base = tile * kTile, cnt = min(kTile, n - base);
    const u64 m = kc[col].m;
    const unsigned* in = src.in(col);
    unsigned* out = in == buf0 ? buf1 : buf0;
    const size_t off = (size_t)col * n;
    const unsigned* C = cum + (size_t)col * (n + 1);
    const unsigned* O = ones + (size_t)col * (n + 1);
    const int b = src.b;
    u64 inv = 0;
    for (int j = threadIdx.x; j < cnt; j += kThreads) {
        const unsigned p = (unsigned)(base + j);
        if (p >= m) break;
        const unsigned s = in[off + p];
        const unsigned bit = (s >> b) & 1u;
        const unsigned lo = (s >> (b + 1)) << (b + 1), mid = lo + (1u << b);
        const unsigned g = C[min(lo, (unsigned)n)];
        const unsigned z = C[min(mid, (unsigned)n)] - g;  // 0-bits of the group
        const unsigned before = O[p] - O[g];              // 1-bits of the group before p
        if (!bit) inv += before;
        out[off + (bit ? g + z + before : p - before)] = s;
    }
    inv = block_sum_u64(inv, wsum);
    if (threadIdx.x == 0 && inv) atomicAdd(&kc[col].disc, inv);
}

// ---- epilogues (float64) ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ double clamp1(double v) { return v < -1.0 ? -1.0 : (v > 1.0 ? 1.0 : v); }

// out[c] = v rounded once to the float dtype of the tag
__device__ __forceinline__ void store_as(void* out, int dtype, int c, double v) {
    switch (dtype) {
        case MB200_F64: reinterpret_cast<double*>(out)[c] = v; break;
        case MB200_F16: reinterpret_cast<__half*>(out)[c] = __double2half(v); break;
        case MB200_BF16: reinterpret_cast<__nv_bfloat16*>(out)[c] = __double2bfloat16(v); break;
        default: reinterpret_cast<float*>(out)[c] = (float)v;
    }
}

__global__ void spearman_finish_kernel(const ColStats* sx, const ColStats* sy, const u64* prod, long long n, int d, double eps, int out_dtype,
                                       void* out) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= d) return;
    double r = __longlong_as_double(0x7ff8000000000000ll);
    if (n > 0) {
        const u128 nn = (u128)n, base = nn * (nn * nn - 1);
        const double vx = u128_to_double(base - load_u128(sx[c].cube)) / (12.0 * (double)n);
        const double vy = u128_to_double(base - load_u128(sy[c].cube)) / (12.0 * (double)n);
        const double cov = i128_to_double((i128)load_u128(prod + 2 * c) - (i128)(nn * (nn + 1) * (nn + 1))) / (4.0 * (double)n);
        r = clamp1(cov / (sqrt(vx) * sqrt(vy) + eps));
    }
    store_as(out, out_dtype, c, r);
}

__global__ void kendall_finish_kernel(const ColStats* sx, const ColStats* sy, const KendallCol* kc, long long n, int d, int variant,
                                      int alternative, void* tau_out, int tau_dtype, float* p_out) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= d) return;
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    double tau = nan, t = nan;
    if (n > 0) {
        const ColStats &X = sx[c], &Y = sy[c];
        const KendallCol& K = kc[c];
        const i128 n0 = (i128)K.m * (i128)(K.m ? K.m - 1 : 0) / 2;
        const i128 conc = n0 - (i128)K.n1 - (i128)K.n2 + (i128)K.n3 - (i128)K.disc;
        const double cmd = i128_to_double(conc - (i128)K.disc);
        const double nd = (double)n;
        const u128 un = (u128)n, total = un * (un - 1) / 2;
        if (variant == MB200_KENDALL_A) {
            tau = cmd / i128_to_double(conc + (i128)K.disc);
        } else if (variant == MB200_KENDALL_B) {
            tau = cmd / sqrt(u128_to_double((total - X.pairs) * (total - Y.pairs)));
        } else {
            const double mc = (double)min(X.distinct, Y.distinct);
            tau = 2.0 * cmd / ((mc - 1.0) / mc * nd * nd);
        }
        tau = clamp1(tau);
        const u128 base = un * (un - 1) * (2 * un + 5);
        if (variant == MB200_KENDALL_A) {
            t = 3.0 * cmd / sqrt(u128_to_double(base) / 2.0);
        } else {
            const u128 p2x = 2 * load_u128(X.cube) + 6 * (u128)X.pairs, p2y = 2 * load_u128(Y.cube) + 6 * (u128)Y.pairs;
            const double mm = nd * (nd - 1.0);
            // a column with every pair tied has Var(S) = 0 exactly; the float64 sum of its terms would leave rounding noise
            const bool constant = (u128)X.pairs == total || (u128)Y.pairs == total;
            const double den = constant ? 0.0 : i128_to_double((i128)base - (i128)p2x - (i128)p2y) / 18.0 +
                               2.0 * (double)X.pairs * (double)Y.pairs / mm +
                               u128_to_double(load_u128(X.p1)) * u128_to_double(load_u128(Y.p1)) / (9.0 * mm * (nd - 2.0));
            t = cmd / sqrt(den);
        }
    }
    store_as(tau_out, tau_dtype, c, tau);
    if (alternative == MB200_KENDALL_ALT_NONE || !p_out) return;
    if (alternative == MB200_KENDALL_ALT_TWO_SIDED) t = -fabs(t);
    if (alternative == MB200_KENDALL_ALT_GREATER) t = -t;
    double p = 0.5 * erfc(-t * 0.70710678118654752440);
    if (alternative == MB200_KENDALL_ALT_TWO_SIDED) p *= 2.0;
    p_out[c] = (float)p;
}

// ---- host driver -------------------------------------------------------------------------------------------------------------
struct Ws {
    u64 *ka, *kb;
    unsigned *va, *vb, *rx, *radix, *tsum, *cnt, *ones;
    ColStats *sx, *sy;
    KendallCol* kc;
    u64* prod;
    size_t zero_bytes;  // ColStats / KendallCol / prod region, from sx
    size_t bytes;
    int tiles;
};

Ws make_ws(long long n, long long d, bool kendall, unsigned char* p) {
    Ws w{};
    const size_t N = (size_t)n * (size_t)d;
    w.tiles = (int)std::max(1LL, (n + kTile - 1) / kTile);
    size_t o = 0;
    auto take = [&](size_t bytes) {
        unsigned char* q = p ? p + o : nullptr;
        o += align16(bytes);
        return q;
    };
    w.sx = reinterpret_cast<ColStats*>(take(sizeof(ColStats) * d));
    w.sy = reinterpret_cast<ColStats*>(take(sizeof(ColStats) * d));
    w.kc = reinterpret_cast<KendallCol*>(take(sizeof(KendallCol) * d));
    w.prod = reinterpret_cast<u64*>(take(16 * (size_t)d));
    w.zero_bytes = o;
    if (n > 0) {
        w.ka = reinterpret_cast<u64*>(take(8 * N));
        w.kb = reinterpret_cast<u64*>(take(8 * N));
        w.va = reinterpret_cast<unsigned*>(take(4 * N));
        w.vb = reinterpret_cast<unsigned*>(take(4 * N));
        w.rx = reinterpret_cast<unsigned*>(take(4 * N));
        w.radix = reinterpret_cast<unsigned*>(take(4 * radix_sort_scratch_words(n, d, 8)));
        w.tsum = reinterpret_cast<unsigned*>(take(4 * (size_t)d * (w.tiles + 1)));
        if (kendall) {
            w.cnt = reinterpret_cast<unsigned*>(take(4 * (size_t)d * (n + 1)));
            w.ones = reinterpret_cast<unsigned*>(take(4 * (size_t)d * (n + 1)));
        }
    }
    w.bytes = o;
    return w;
}

// Exclusive prefix of src per column into w.tsum (per tile) and, unless out is NULL, into out (per element).
template <typename Src, bool kPairs = false>
void column_scan(Src src, int n, int d, Ws& w, unsigned* out, cudaStream_t st) {
    const unsigned grid = (unsigned)(d * w.tiles);
    tile_reduce_kernel<Src, kPairs><<<grid, kThreads, 0, st>>>(src, n, w.tiles, w.tsum, w.kc);
    tile_scan_kernel<<<(unsigned)d, 1024, 0, st>>>(w.tsum, w.tiles);
    count_launch(), count_launch();
    if (!out) return;
    tile_apply_kernel<Src><<<grid, kThreads, 0, st>>>(src, n, w.tiles, w.tsum, out);
    count_launch();
}

// composite key of a row with a NaN value: all ones over the bytes(n) bytes the concordance sort orders by
unsigned nan_row_key(long long n) {
    const int kb = (bits_of((u64)n) + 7) / 8;
    return kb >= 4 ? 0xffffffffu : (1u << (8 * kb)) - 1u;
}

// Sorts one variable per column and runs its tie pass in mode kMode.  Returns the radix sort's result buffer (0: ka/va,
// 1: kb/vb) or a negative MB200_ERR_* code.
template <int kMode>
int rank_phase(const void* in, int dtype, int n, int d, Ws& w, unsigned* err, cudaStream_t st) {
    return with_rank_type(dtype, [&](auto tag) -> int {
        using T = typename decltype(tag)::type;
        using KeyT = std::conditional_t<sizeof(T) == 8, u64, unsigned>;
        KeyT* ka = reinterpret_cast<KeyT*>(w.ka);
        KeyT* kb = reinterpret_cast<KeyT*>(w.kb);
        pack_kernel<T, KeyT><<<grid_for((long long)n * d), kThreads, 0, st>>>(reinterpret_cast<const T*>(in), n, d, ka, w.va);
        count_launch();
        const int where = radix_sort_passes<KeyT, unsigned>(ka, w.va, kb, w.vb, n, d, (int)sizeof(T), w.radix, err, st, &count_launch);
        if (where < 0) return where;
        TieArgs<KeyT> a{};
        a.keys = where ? kb : ka;
        a.rows = where ? w.vb : w.va;
        a.n = n;
        a.tiles = w.tiles;
        a.nan_keys = is_float_tag(dtype);
        a.nan_key = sizeof(T) == 2 ? (KeyT)0xffffu : ~(KeyT)0;
        a.stats = (kMode == kSpearmanX || kMode == kKendallX) ? w.sx : w.sy;
        a.rank_out = w.rx;
        a.rank_x = w.rx;
        a.spear_sum = w.prod;
        a.k2 = reinterpret_cast<unsigned*>(where ? w.ka : w.kb);
        a.v2 = where ? w.va : w.vb;
        a.cnt = w.cnt;
        a.k2_invalid = nan_row_key(n);
        if (kMode == kKendallX || kMode == kKendallY) {
            column_scan(HeadSrc<KeyT>{a.keys, n, a.nan_keys, a.nan_key}, n, d, w, nullptr, st);
            a.head_excl = w.tsum;
        }
        ties_kernel<KeyT, kMode><<<(unsigned)(d * w.tiles), kThreads, 0, st>>>(a);
        count_launch();
        return where;
    });
}

}  // namespace
}  // namespace mb200

using namespace mb200;

// =====================================================================================================
// C-ABI
// =====================================================================================================
extern "C" int64_t mb200_rankcorr_scratch_bytes(int64_t n, int64_t d, int kendall) {
    if (n < 0 || n > MB200_RANKCORR_MAX_ROWS || d < 1 || d > (1 << 20)) return -1;
    if (d * ((n + kTile - 1) / kTile) > INT_MAX) return -1;  // one CTA per (column, tile)
    return (int64_t)make_ws(n, d, kendall != 0, nullptr).bytes;
}

static int rankcorr_check(const void* preds, const void* target, int64_t n, int64_t d, bool kendall, void* scratch,
                          int64_t scratch_bytes, Ws* w) {
    const int64_t need = mb200_rankcorr_scratch_bytes(n, d, kendall);
    MB200_REQUIRE(need >= 0, "rank correlation inputs of %lld rows x %lld columns; rows must be below 2^30 and columns in [1, 2^20]",
                  (long long)n, (long long)d);
    MB200_REQUIRE(preds && target && scratch, "NULL pointer");
    MB200_REQUIRE(scratch_bytes >= need, "scratch too small (%lld < %lld bytes)", (long long)scratch_bytes, (long long)need);
    *w = make_ws(n, d, kendall, reinterpret_cast<unsigned char*>(scratch));
    return 0;
}

extern "C" int mb200_spearman_corrcoef(const void* preds, int preds_dtype, const void* target, int target_dtype, int64_t n,
                                       int64_t d, void* out, int out_dtype, double eps, void* scratch, int64_t scratch_bytes,
                                       uint32_t* err_flag, void* stream) {
    MB200_REQUIRE(is_float_tag(preds_dtype) && is_float_tag(target_dtype) && is_float_tag(out_dtype),
                  "spearman inputs and output must be floating point (dtype tags %d, %d, %d)", preds_dtype, target_dtype, out_dtype);
    MB200_REQUIRE(out, "NULL pointer");
    Ws w;
    const int rc = rankcorr_check(preds, target, n, d, false, scratch, scratch_bytes, &w);
    if (rc) return rc;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    MB200_CUDA_OK(cudaMemsetAsync(w.sx, 0, w.zero_bytes, st));
    if (n > 0) {
        int r = rank_phase<kSpearmanX>(preds, preds_dtype, (int)n, (int)d, w, err_flag, st);
        if (r < 0) return r;
        r = rank_phase<kSpearmanY>(target, target_dtype, (int)n, (int)d, w, err_flag, st);
        if (r < 0) return r;
    }
    spearman_finish_kernel<<<(unsigned)((d + 127) / 128), 128, 0, st>>>(w.sx, w.sy, w.prod, n, (int)d, eps, out_dtype, out);
    count_launch();
    return check_cuda(cudaGetLastError(), "spearman_corrcoef");
}

extern "C" int mb200_kendall_rank_corrcoef(const void* preds, int preds_dtype, const void* target, int target_dtype, int64_t n,
                                           int64_t d, int variant, int alternative, void* tau, int tau_dtype, float* p_value,
                                           void* scratch, int64_t scratch_bytes, uint32_t* err_flag, void* stream) {
    auto rankable = [](int t) { return is_float_tag(t) || t == MB200_I32 || t == MB200_I64; };
    MB200_REQUIRE(rankable(preds_dtype) && rankable(target_dtype),
                  "kendall inputs must be floating point, int32 or int64 (dtype tags %d, %d)", preds_dtype, target_dtype);
    MB200_REQUIRE(variant >= MB200_KENDALL_A && variant <= MB200_KENDALL_C, "bad variant %d", variant);
    MB200_REQUIRE(alternative >= MB200_KENDALL_ALT_NONE && alternative <= MB200_KENDALL_ALT_GREATER, "bad alternative %d", alternative);
    MB200_REQUIRE(is_float_tag(tau_dtype), "tau must be floating point (dtype tag %d)", tau_dtype);
    MB200_REQUIRE(tau && (p_value || alternative == MB200_KENDALL_ALT_NONE), "NULL pointer");
    Ws w;
    const int rc = rankcorr_check(preds, target, n, d, true, scratch, scratch_bytes, &w);
    if (rc) return rc;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    MB200_CUDA_OK(cudaMemsetAsync(w.sx, 0, w.zero_bytes, st));
    if (n > 0) {
        const int ni = (int)n, di = (int)d;
        MB200_CUDA_OK(cudaMemsetAsync(w.cnt, 0, 4 * (size_t)d * (n + 1), st));
        int r = rank_phase<kKendallX>(preds, preds_dtype, ni, di, w, err_flag, st);
        if (r < 0) return r;
        const int wy = rank_phase<kKendallY>(target, target_dtype, ni, di, w, err_flag, st);
        if (wy < 0) return wy;
        // the y pass wrote (dense x, dense y) into the buffers its sort did not end in; sort them by dense x, stably
        unsigned* k2a = reinterpret_cast<unsigned*>(wy ? w.ka : w.kb);
        unsigned* v2a = wy ? w.va : w.vb;
        unsigned* k2b = reinterpret_cast<unsigned*>(wy ? w.kb : w.ka);
        unsigned* v2b = wy ? w.vb : w.va;
        const int kb2 = (bits_of((u64)n) + 7) / 8;
        const unsigned invalid = nan_row_key(n);
        const int w2 = radix_sort_passes<unsigned, unsigned>(k2a, v2a, k2b, v2b, ni, di, kb2, w.radix, err_flag, st, &count_launch);
        if (w2 < 0) return w2;
        const unsigned* ks = w2 ? k2b : k2a;
        unsigned* vs = w2 ? v2b : v2a;
        unsigned* vo = w2 ? v2a : v2b;
        runs_kernel<<<(unsigned)(d * w.tiles), kThreads, 0, st>>>(ks, vs, ni, w.tiles, invalid, w.kc);
        count_launch();
        column_scan<CountSrc, true>(CountSrc{w.cnt, ni}, ni, di, w, w.cnt, st);  // histogram -> group starts, n2
        for (int b = bits_of((u64)(n - 1)) - 1; b >= 0; --b) {
            const BitSrc src{vs, vo, w.sy, w.kc, ni, b};
            column_scan(src, ni, di, w, w.ones, st);
            level_scatter_kernel<<<(unsigned)(d * w.tiles), kThreads, 0, st>>>(src, vs, vo, w.cnt, w.ones, w.kc, ni, w.tiles);
            count_launch();
        }
    }
    kendall_finish_kernel<<<(unsigned)((d + 127) / 128), 128, 0, st>>>(w.sx, w.sy, w.kc, n, (int)d, variant, alternative, tau,
                                                                       tau_dtype, p_value);
    count_launch();
    return check_cuda(cudaGetLastError(), "kendall_rank_corrcoef");
}
