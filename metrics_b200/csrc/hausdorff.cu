// K19 — Hausdorff distance of 2-D segmentation masks (HausdorffDistance, hausdorff_distance) on sm_90a: an exact
// distance transform restricted to edge pixels, in two passes over every (sample, class) pair.
//
// Reference op chain replaced (src/torchmetrics/functional/segmentation/):
//   hausdorff_distance.py:94-113  one_hot of index labels, background dropped, then a Python loop over every pair
//   utils.py:284-322              mask_edges: pad, binary erosion with the connectivity-1 cross through unfold, xor
//   utils.py:342-389, 250-271     surface_distance: torch.any / torch.where, then dense [pixels, edge pixels] distances
//                                 in int64 and float32 and their row minimum, once per direction
//
// Column pass (column_kernel): one thread per (pair, column) walks the column down, deriving both edge masks on the fly
// from the four axis neighbours, and stores per pixel an edge byte (bit 0 preds, bit 1 target) and the row distance to
// the nearest target (and, undirected, pred) edge above; walking back up it lowers that to the nearest edge below.  A
// column without such edges keeps the sentinel (the largest value of G, the narrowest unsigned type that holds height).
// The same pass records which masks of the pair have edges, non-binary values and out-of-range labels.
//
// Row scan (scan_kernel): one warp per (pair, row) takes every pred edge pixel (i, j) of the row in turn and computes
// min over columns j' of f(g_T(i, j'), |j - j'|), 16 columns on each side per step, until f(0, |j - j'|) >= best; then
// the same for target edges against g_P when undirected.  The warp's maximum goes to out[pair] with one atomicMax on the
// float bits, exact for non-negative floats and independent of the order.
//
// Exactness: f is the reference's float32 expression, with int spacing entries in int64 and float ones in float32 as
// torch promotes them (explicit __fmul_rn / __fadd_rn / __fsqrt_rn, no contraction).  Each step of f is monotone in each
// argument, so within a column the nearest edge row gives the smallest f, the minimum over columns is the reference's
// minimum over all edge pixels, and f(0, dc) bounds every column at distance dc or more from below.
#include <algorithm>

#include "common.cuh"
#include "../../include/metrics_b200_hausdorff.h"

namespace mb200 {

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kHalfSpan = 16;  // columns per side per step of the row scan

__host__ __device__ long long cdiv(long long a, long long b) { return (a + b - 1) / b; }
__host__ __device__ long long align16(long long v) { return cdiv(v, 16) * 16; }

int g_bytes(long long height) { return height <= 255 ? 1 : (height <= 65535 ? 2 : 4); }

// bytes of one pair's scratch: edge bytes, then g_T and (undirected) g_P
long long pair_bytes(long long H, long long W, int directed) {
    return align16(H * W) + (directed ? 1 : 2) * align16(H * W * g_bytes(H));
}

struct Src {
    const void* p;
    int dtype;
    long long sn, sc, sh, sw;
};

struct Geo {
    int index;  // MB200_SEG_INDEX
    long long H, W;
    long long C;  // num_classes
    int off, Cp;
    long long q0, m;  // first global pair of the launch, pairs in the launch
    int directed;
};

struct Spacing {
    int metric;
    int int_mask;
    long long i0, i1;
    float f0, f1;
};

// One term of f: axis spacing times a distance, kept in int64 (int spacing) or rounded to float32.
struct Term {
    bool is_int;
    long long i;
    float f;
};
__device__ __forceinline__ Term term(bool is_int, long long si, float sf, long long d) {
    Term t;
    t.is_int = is_int;
    if (is_int) t.i = si * d;
    else t.f = __fmul_rn(sf, __ll2float_rn(d));
    return t;
}
__device__ __forceinline__ float as_f32(const Term& t) { return t.is_int ? __ll2float_rn(t.i) : t.f; }

// f(dr, dc) as the reference's float32 expression evaluates it (utils.py:260-265)
__device__ __forceinline__ float distance(const Spacing& s, long long dr, long long dc) {
    const Term a = term(s.int_mask & 1, s.i0, s.f0, dr);
    const Term b = term(s.int_mask & 2, s.i1, s.f1, dc);
    const bool both_int = a.is_int && b.is_int;
    if (s.metric == MB200_HD_EUCLIDEAN) {
        if (both_int) return __fsqrt_rn(__ll2float_rn(a.i * a.i + b.i * b.i));
        const float x = a.is_int ? __ll2float_rn(a.i * a.i) : __fmul_rn(a.f, a.f);
        const float y = b.is_int ? __ll2float_rn(b.i * b.i) : __fmul_rn(b.f, b.f);
        return __fsqrt_rn(__fadd_rn(x, y));
    }
    if (s.metric == MB200_HD_CHESSBOARD) {
        if (both_int) return __ll2float_rn(a.i > b.i ? a.i : b.i);
        return fmaxf(as_f32(a), as_f32(b));
    }
    if (both_int) return __ll2float_rn(a.i + b.i);
    return __fadd_rn(as_f32(a), as_f32(b));
}

// ---- column pass ---------------------------------------------------------------------------------------------------------
struct Masks {
    bool p, t;
};

// The two masks at (i, j) of pair (b, cls); false outside the image.
__device__ __forceinline__ Masks masks_at(const Src& P, const Src& T, const Geo& g, long long b, long long cls, long long i,
                                          long long j) {
    if (i < 0 || i >= g.H || j < 0 || j >= g.W) return {false, false};
    const long long vp = load_label(P.p, P.dtype, b * P.sn + cls * P.sc + i * P.sh + j * P.sw);
    const long long vt = load_label(T.p, T.dtype, b * T.sn + cls * T.sc + i * T.sh + j * T.sw);
    if (g.index) return {vp == cls, vt == cls};
    return {vp != 0, vt != 0};
}

// grid: cdiv(m * W, kThreads) CTAs; thread (q, j) for local pair q = t / W, column j = t % W
template <typename G>
__global__ void __launch_bounds__(kThreads) column_kernel(Src P, Src T, Geo g, unsigned char* __restrict__ scratch,
                                                          long long pbytes, unsigned* __restrict__ has_edges,
                                                          unsigned long long* __restrict__ err) {
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (t >= g.m * g.W) return;
    const long long ql = t / g.W, j = t - ql * g.W;
    const long long q = g.q0 + ql;
    const long long b = q / g.Cp, cls = q % g.Cp + g.off;
    const long long H = g.H, W = g.W;
    unsigned char* E = scratch + ql * pbytes;
    G* gT = reinterpret_cast<G*>(E + align16(H * W));
    G* gP = reinterpret_cast<G*>(reinterpret_cast<unsigned char*>(gT) + align16(H * W * (long long)sizeof(G)));
    constexpr G kSent = (G)~(G)0;
    // one-hot: non-binary preds (bit 0) / target (bit 1); index: MB200_SEG_* bits of the labels
    unsigned bad = 0u, labels = 0u, has = 0u;
    const long long sP = b * P.sn + (g.index ? 0 : cls * P.sc) + j * P.sw;
    const long long sT = b * T.sn + (g.index ? 0 : cls * T.sc) + j * T.sw;
    Src Pc = P, Tc = T;
    if (g.index) Pc.sc = Tc.sc = 0;
    long long lastT = -1, lastP = -1;
    Masks up = {false, false};
    Masks cur;
    // row 0 centre, checked below with every later centre
    long long vp = load_label(P.p, P.dtype, sP), vt = load_label(T.p, T.dtype, sT);
    for (long long i = 0; i < H; ++i) {
        if (g.index) {
            labels |= vp < 0 ? MB200_SEG_PREDS_NEGATIVE : (vp >= g.C ? MB200_SEG_PREDS_TOO_LARGE : 0u);
            labels |= vt < 0 ? MB200_SEG_TARGET_NEGATIVE : (vt >= g.C ? MB200_SEG_TARGET_TOO_LARGE : 0u);
            cur = {vp == cls, vt == cls};
        } else {
            bad |= (vp != 0 && vp != 1) ? 1u : 0u;
            bad |= (vt != 0 && vt != 1) ? 2u : 0u;
            cur = {vp != 0, vt != 0};
        }
        Masks down = {false, false};
        if (i + 1 < H) {
            vp = load_label(P.p, P.dtype, sP + (i + 1) * P.sh);
            vt = load_label(T.p, T.dtype, sT + (i + 1) * T.sh);
            down = g.index ? Masks{vp == cls, vt == cls} : Masks{vp != 0, vt != 0};
        }
        const Masks left = masks_at(Pc, Tc, g, b, cls, i, j - 1);
        const Masks right = masks_at(Pc, Tc, g, b, cls, i, j + 1);
        const bool ep = cur.p && !(up.p && down.p && left.p && right.p);
        const bool et = cur.t && !(up.t && down.t && left.t && right.t);
        const long long k = i * W + j;
        E[k] = (unsigned char)((ep ? 1 : 0) | (et ? 2 : 0));
        has |= (ep ? 1u : 0u) | (et ? 2u : 0u);
        if (et) lastT = i;
        gT[k] = lastT < 0 ? kSent : (G)(i - lastT);
        if (!g.directed) {
            if (ep) lastP = i;
            gP[k] = lastP < 0 ? kSent : (G)(i - lastP);
        }
        up = cur;
    }
    long long nextT = -1, nextP = -1;
    for (long long i = H - 1; i >= 0; --i) {
        const long long k = i * W + j;
        const unsigned e = E[k];
        if (e & 2u) nextT = i;
        if (nextT >= 0 && (G)(nextT - i) < gT[k]) gT[k] = (G)(nextT - i);
        if (!g.directed) {
            if (e & 1u) nextP = i;
            if (nextP >= 0 && (G)(nextP - i) < gP[k]) gP[k] = (G)(nextP - i);
        }
    }
    if (has != 0u && (__ldcg(has_edges + ql) & has) != has) atomicOr(has_edges + ql, has);
    if (bad != 0u) atomicMin(err, (unsigned long long)q * 4ull + ((bad & 1u) ? MB200_HD_PREDS_NOT_BINARY : MB200_HD_TARGET_NOT_BINARY));
    if (labels != 0u) atomicOr(reinterpret_cast<unsigned*>(err + 1), labels);
}

// ---- row scan ------------------------------------------------------------------------------------------------------------
// min over the columns of row `g_row` of f(g_row[j'], |jq - j'|): warp-uniform, every lane calls it
template <typename G>
__device__ __forceinline__ float nearest(const G* __restrict__ g_row, long long jq, long long W, Spacing s, int lane) {
    constexpr G kSent = (G)~(G)0;
    const long long reach = max(jq + 1, W - jq);  // every column is at a distance below reach
    unsigned best = __float_as_uint(INFINITY);
    for (long long k0 = 0; k0 < reach; k0 += kHalfSpan) {
        if (__float_as_uint(distance(s, 0, k0)) >= best) break;  // no column at distance k0 or more can be nearer
        const long long dc = k0 + (lane >> 1);
        const long long col = (lane & 1) ? jq + dc : jq - dc;
        unsigned v = __float_as_uint(INFINITY);
        if (col >= 0 && col < W) {
            const G d = g_row[col];
            if (d != kSent) v = __float_as_uint(distance(s, (long long)d, dc));
        }
        best = min(best, __reduce_min_sync(kFull, v));
    }
    return __uint_as_float(best);
}

// grid: cdiv(m * H, kWarps) CTAs; warp (q, i) for local pair q = w / H, row i = w % H
template <typename G>
__global__ void __launch_bounds__(kThreads, 2) scan_kernel(Geo g, Spacing s, const unsigned char* __restrict__ scratch,
                                                        long long pbytes, const unsigned* __restrict__ has_edges,
                                                        float* __restrict__ out, unsigned long long* __restrict__ err) {
    const long long w = (long long)blockIdx.x * kWarps + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (w >= g.m * g.H) return;
    const long long ql = w / g.H, i = w - ql * g.H;
    const long long q = g.q0 + ql;
    const long long H = g.H, W = g.W;
    const unsigned has = has_edges[ql];
    if (has != 3u) {
        if (i == 0 && lane == 0) {
            if (has == 0u) atomicMin(err, (unsigned long long)q * 4ull + MB200_HD_NO_EDGES);
            else out[q] = INFINITY;
        }
        return;
    }
    const unsigned char* E = scratch + ql * pbytes;
    const G* gT = reinterpret_cast<const G*>(E + align16(H * W));
    const G* gP = reinterpret_cast<const G*>(reinterpret_cast<const unsigned char*>(gT) + align16(H * W * (long long)sizeof(G)));
    const unsigned char* Erow = E + i * W;
    unsigned row_max = 0u;  // bits of +0.0f
    for (long long seg = 0; seg < W; seg += 32) {
        const long long j = seg + lane;
        const unsigned e = j < W ? Erow[j] : 0u;
        for (unsigned qp = __ballot_sync(kFull, e & 1u); qp != 0u; qp &= qp - 1u) {
            const float d = nearest(gT + i * W, seg + __ffs(qp) - 1, W, s, lane);
            row_max = max(row_max, __float_as_uint(d));
        }
        if (!g.directed) {
            for (unsigned qt = __ballot_sync(kFull, e & 2u); qt != 0u; qt &= qt - 1u) {
                const float d = nearest(gP + i * W, seg + __ffs(qt) - 1, W, s, lane);
                row_max = max(row_max, __float_as_uint(d));
            }
        }
    }
    if (lane == 0 && row_max != 0u) atomicMax(reinterpret_cast<unsigned*>(out + q), row_max);
}

template <typename G>
int launch(const Src& P, const Src& T, Geo g, const Spacing& s, long long pairs, long long mpl, float* out,
           unsigned char* scratch, unsigned long long* err, cudaStream_t st) {
    const long long pbytes = pair_bytes(g.H, g.W, g.directed);
    unsigned* has_edges = reinterpret_cast<unsigned*>(scratch);
    unsigned char* pair_scratch = scratch + align16(mpl * 4);
    for (long long q0 = 0; q0 < pairs; q0 += mpl) {
        g.q0 = q0;
        g.m = std::min(mpl, pairs - q0);
        MB200_CUDA_OK(cudaMemsetAsync(has_edges, 0, (size_t)(g.m * 4), st));
        const long long cols = cdiv(g.m * g.W, kThreads), rows = cdiv(g.m * g.H, kWarps);
        MB200_REQUIRE(cols < (1ll << 31) && rows < (1ll << 31), "too many pairs for one launch");
        column_kernel<G><<<(unsigned)cols, kThreads, 0, st>>>(P, T, g, pair_scratch, pbytes, has_edges, err);
        count_launch();
        scan_kernel<G><<<(unsigned)rows, kThreads, 0, st>>>(g, s, pair_scratch, pbytes, has_edges, out, err);
        count_launch();
        MB200_CUDA_OK(cudaGetLastError());
    }
    return 0;
}

}  // namespace
}  // namespace mb200

using namespace mb200;

// =====================================================================================================
// C-ABI
// =====================================================================================================
extern "C" int64_t mb200_hausdorff_scratch_bytes(int64_t height, int64_t width, int directed, int64_t pairs_per_launch) {
    if (height < 1 || width < 1 || pairs_per_launch < 1 || height > (1ll << 31) || width > (1ll << 31)) return -1;
    const long long pb = pair_bytes(height, width, directed ? 1 : 0);
    if (pb > (1ll << 56) / pairs_per_launch) return -1;
    return align16(pairs_per_launch * 4) + pairs_per_launch * pb;
}

extern "C" int mb200_hausdorff_distance(const void* preds, int preds_dtype, const void* target, int target_dtype,
                                        int input_format, int64_t n, int64_t num_classes, int64_t height, int64_t width,
                                        int64_t preds_s_n, int64_t preds_s_c, int64_t preds_s_h, int64_t preds_s_w,
                                        int64_t target_s_n, int64_t target_s_c, int64_t target_s_h, int64_t target_s_w,
                                        int drop_background, int metric, int spacing_int_mask, double spacing_0,
                                        double spacing_1, int directed, int64_t pairs_per_launch, float* out, void* scratch,
                                        int64_t scratch_bytes, uint64_t* err, void* stream) {
    MB200_REQUIRE(n >= 0 && num_classes >= 1 && num_classes < (1ll << 31), "bad sizes");
    MB200_REQUIRE(input_format == MB200_SEG_INDEX || input_format == MB200_SEG_ONE_HOT, "unknown input_format %d", input_format);
    if (input_format == MB200_SEG_INDEX) {
        MB200_REQUIRE(preds_dtype == MB200_I64 && target_dtype == MB200_I64, "index labels must be int64 (dtype tags %d, %d)",
                      preds_dtype, target_dtype);
    } else {
        MB200_REQUIRE(is_label_tag(preds_dtype) && is_label_tag(target_dtype), "unsupported dtype tags %d, %d", preds_dtype,
                      target_dtype);
    }
    MB200_REQUIRE(metric == MB200_HD_EUCLIDEAN || metric == MB200_HD_CHESSBOARD || metric == MB200_HD_TAXICAB,
                  "unknown metric %d", metric);
    MB200_REQUIRE(spacing_int_mask >= 0 && spacing_int_mask <= 3, "bad spacing_int_mask %d", spacing_int_mask);
    MB200_REQUIRE(out && err, "NULL pointer");
    const int off = (drop_background && num_classes > 1) ? 1 : 0;
    const long long Cp = num_classes - off, pairs = n * Cp;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    MB200_CUDA_OK(cudaMemsetAsync(err, 0xff, sizeof(uint64_t), st));
    MB200_CUDA_OK(cudaMemsetAsync(err + 1, 0, sizeof(uint64_t), st));
    if (pairs == 0) return 0;
    const int64_t need = mb200_hausdorff_scratch_bytes(height, width, directed, pairs_per_launch);
    MB200_REQUIRE(need >= 0, "bad image size %lld x %lld or pairs_per_launch %lld", (long long)height, (long long)width,
                  (long long)pairs_per_launch);
    MB200_REQUIRE(preds && target && scratch, "NULL pointer");
    MB200_REQUIRE(scratch_bytes >= need && (reinterpret_cast<uintptr_t>(scratch) & 15) == 0,
                  "scratch must be 16-byte aligned and mb200_hausdorff_scratch_bytes(...) bytes");
    MB200_CUDA_OK(cudaMemsetAsync(out, 0, (size_t)(pairs * sizeof(float)), st));
    const Src P{preds, preds_dtype, preds_s_n, preds_s_c, preds_s_h, preds_s_w};
    const Src T{target, target_dtype, target_s_n, target_s_c, target_s_h, target_s_w};
    Geo g{input_format == MB200_SEG_INDEX, height, width, num_classes, off, (int)Cp, 0, 0, directed ? 1 : 0};
    Spacing s;
    s.metric = metric;
    s.int_mask = spacing_int_mask;
    s.i0 = (long long)spacing_0;
    s.i1 = (long long)spacing_1;
    s.f0 = (float)spacing_0;
    s.f1 = (float)spacing_1;
    const long long mpl = std::min((long long)pairs_per_launch, pairs);
    unsigned char* sc = reinterpret_cast<unsigned char*>(scratch);
    unsigned long long* e = reinterpret_cast<unsigned long long*>(err);
    switch (g_bytes(height)) {
        case 1: return launch<unsigned char>(P, T, g, s, pairs, mpl, out, sc, e, st);
        case 2: return launch<unsigned short>(P, T, g, s, pairs, mpl, out, sc, e, st);
        default: return launch<unsigned>(P, T, g, s, pairs, mpl, out, sc, e, st);
    }
}
