// K18 — panoptic quality (PanopticQuality, ModifiedPanopticQuality) on sm_90a: per-image segment areas and segment-pair
// intersections in one read of the two label maps, then the matching step on the counted pairs.
//
// Reference op chain replaced (src/torchmetrics/functional/detection/_panoptic_quality_common.py):
//   :175-211  clone, isin against things / stuffs, stuff instance ids -> 0, unknown categories -> the void color
//   :312-394  per image: three torch.unique(dim=0) sorts (pred colors, target colors, [P, 2, 2] color pairs), .tolist(),
//             a Python loop over every pair (IoU, match at > 0.5) and over every unmatched color (false positive / negative)
//   :431-442  per-image results summed in image order
//
// Pixel pass (pixel_kernel): a CTA reads one tile of one image; every warp owns a contiguous run of the tile, one pixel per
// lane per step, each (category, instance) pair in one vector load.  The category becomes its continuous id by binary search
// over the sorted ids (in shared memory up to kSmemCats categories).  Lanes holding the same (pred color, target color) are
// grouped by AND-ing three __match_any_sync masks (one compare when the whole warp agrees); the group leader resolves both
// colors to their slots in the image's pred / target color tables and adds the group size to a run count it keeps in
// registers for the last pair it saw.  Label maps are spatially coherent, so a run spans many steps and is added to the
// image's pair table once.  Every lane caches the slots of the last pred and target color of its group, so a leader looks
// a color up only where the map changes.
//
// Hash tables (global scratch, open addressing, linear probing, never moved or deleted): a color key is 16 bytes {int64
// instance, int32 continuous id, int32 tag = 1} claimed with one 16-byte atomicCAS, whose return value is also the atomic
// read of an occupied slot.  A pair key is the two color slot indices + 1 packed into 64 bits (0 = empty).  Slot indices
// are therefore stable segment ids.  A table more than half full sets MB200_FLAG_CAPACITY; the caller then repeats the
// update with tables of at least 2 * pixels slots, which cannot fill.
//
// Evaluation: areas_kernel adds every pair's count to the areas of its two colors and records the pairs with a void side;
// match_kernel applies the IoU rule to every same-category pair with a non-void target (IoU = float32(inter) /
// float32(union), IEEE round to nearest, as torch divides two int64 tensors); unmatched_kernel counts false positives /
// negatives and, for ModifiedPanopticQuality, the stuff target segments.  They write per-image [n][K] partials with atomics:
// integer sums are exact, and so are the float64 IoU sums, because every term above 0.5 is a float32 multiple of 2^-24 and
// a stuff category has at most one pair per image.  fold_kernel adds the partials in image order, as the reference does,
// and does nothing when the error word is set, so a failed update leaves the states as they were.
#include <algorithm>

#include "common.cuh"
#include "../../include/metrics_b200_panoptic.h"

namespace mb200 {

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kUnroll = 4;
constexpr int kSmemCats = 2048;          // 2 x 2048 x 8 B = 32 KB of categories in shared memory
constexpr long long kMinTile = 4096;     // pixels per CTA at least
constexpr long long kMinCapacity = 64;
constexpr long long kMaxCapacity = 1ll << 31;

struct alignas(16) Color {
    long long inst;
    int cid;
    int tag;  // 1 once claimed
};

template <typename T>
struct alignas(2 * sizeof(T)) Seg {
    T cat, inst;
};

// The hash tables of one launch of `m` images, image b at offset b * ccap (colors) or b * pcap (pairs).
struct Tables {
    Color* pcol;
    Color* tcol;
    unsigned long long* parea;  // pixels of each pred color
    unsigned long long* tarea;
    unsigned long long* pvoid;  // inter(pred color, void target)
    unsigned long long* tvoid;  // inter(void pred, target color)
    unsigned char* pmatch;
    unsigned char* tmatch;
    unsigned long long* pkey;
    unsigned long long* pcnt;
    unsigned* used;  // [m][3]: claimed pred colors, target colors, pairs
    long long ccap, pcap;
};

// Partials of all n images: [n][K] each.
struct Partials {
    double* iou;
    int* tp;
    int* fp;
    int* fn;
};

__device__ __forceinline__ unsigned long long mix64(unsigned long long x) {
    x ^= x >> 33;
    x *= 0xff51afd7ed558ccdull;
    x ^= x >> 33;
    x *= 0xc4ceb9fe1a85ec53ull;
    x ^= x >> 33;
    return x;
}

__device__ __forceinline__ void claimed(unsigned* used, long long cap, unsigned* err) {
    if ((long long)atomicAdd(used, 1u) + 1 > cap / 2) atomicOr(err, MB200_FLAG_CAPACITY);
}

// Once a table has overflowed the update is repeated, so the remaining inserts of this pass stop early instead of probing a
// full table.  A table of the repeat never holds more than half its slots, so there the probe always ends at its key.
__device__ __forceinline__ bool overflowed(const unsigned* used, long long cap) {
    return (long long)*(const volatile unsigned*)used > cap / 2;
}

// Slot of color (inst, cid) in `tab`, claiming an empty slot for a new color; -1 when the table is full.
__device__ __forceinline__ long long color_slot(Color* tab, long long cap, long long inst, int cid, unsigned* used, unsigned* err) {
    const Color key{inst, cid, 1};
    long long h = (long long)(mix64((unsigned long long)inst ^ ((unsigned long long)(unsigned)cid << 40)) & (unsigned long long)(cap - 1));
    for (long long probe = 0; probe < cap; ++probe) {
        if ((probe & 15) == 15 && overflowed(used, cap)) return -1;
        const Color cur = atomicCAS(tab + h, Color{0, 0, 0}, key);
        if (cur.tag == 0) {
            claimed(used, cap, err);
            return h;
        }
        if (cur.inst == inst && cur.cid == cid) return h;
        h = (h + 1) & (cap - 1);
    }
    atomicOr(err, MB200_FLAG_CAPACITY);
    return -1;
}

// count += c for pair `key` (non-zero) of one image's pair table
__device__ __forceinline__ void pair_add(unsigned long long* keys, unsigned long long* cnts, long long cap, unsigned long long key,
                         unsigned long long c, unsigned* used, unsigned* err) {
    long long h = (long long)(mix64(key) & (unsigned long long)(cap - 1));
    for (long long probe = 0; probe < cap; ++probe) {
        if ((probe & 15) == 15 && overflowed(used, cap)) return;
        unsigned long long cur = keys[h];
        if (cur == 0ull) {
            cur = atomicCAS(keys + h, 0ull, key);
            if (cur == 0ull) {
                claimed(used, cap, err);
                cur = key;
            }
        }
        if (cur == key) {
            atomicAdd(cnts + h, c);
            return;
        }
        h = (h + 1) & (cap - 1);
    }
    atomicOr(err, MB200_FLAG_CAPACITY);
}

// continuous id of `cat` (K: unknown, the void color) and the instance id it keeps
__device__ __forceinline__ int classify(long long cat, long long inst, const long long* ids, const long long* cids, int K,
                                        int n_things, long long* inst_out) {
    int lo = 0, hi = K;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (ids[mid] < cat) lo = mid + 1;
        else hi = mid;
    }
    const int cid = (lo < K && ids[lo] == cat) ? (int)cids[lo] : K;
    *inst_out = cid < n_things ? inst : 0;
    return cid;
}

// grid: m * tiles CTAs; CTA b counts pixels [part * tile, min(P, (part + 1) * tile)) of image b / tiles of this launch
template <typename TP, typename TT>
__global__ void __launch_bounds__(kThreads, 2) pixel_kernel(const Seg<TP>* __restrict__ preds, const Seg<TT>* __restrict__ target,
                                                         long long P, long long tiles, long long tile,
                                                         const long long* __restrict__ cats, int K, int n_things,
                                                         int check_preds, Tables tb, unsigned* err) {
    extern __shared__ long long s_cats[];  // [K] ids, [K] continuous ids
    const long long* ids = cats;
    if (K <= kSmemCats) {
        for (int j = threadIdx.x; j < 2 * K; j += kThreads) s_cats[j] = cats[j];
        __syncthreads();
        ids = s_cats;
    }
    const long long* cids = ids + K;
    const long long b = blockIdx.x / tiles, part = blockIdx.x % tiles;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long span = tile / kWarps;  // a multiple of 32
    const long long w0 = min(P, part * tile + warp * span), w1 = min(P, w0 + span);
    const Seg<TP>* Pp = preds + b * P;
    const Seg<TT>* Tp = target + b * P;
    Color* pcol = tb.pcol + b * tb.ccap;
    Color* tcol = tb.tcol + b * tb.ccap;
    unsigned* used = tb.used + b * 3;
    // leader state: the last pred / target color resolved, and the pair run being counted
    long long lp_inst = 0, lt_inst = 0, lp_slot = -1, lt_slot = -1;
    int lp_cid = -1, lt_cid = -1;
    unsigned long long run_key = 0ull, run_cnt = 0ull;
    unsigned flags = 0u;
    for (long long base = w0; base < w1; base += 32 * kUnroll) {
        long long pcat[kUnroll], pins[kUnroll], tcat[kUnroll], tins[kUnroll];
#pragma unroll
        for (int k = 0; k < kUnroll; ++k) {
            const long long i = base + k * 32 + lane;
            const Seg<TP> a = i < w1 ? Pp[i] : Seg<TP>{0, 0};
            const Seg<TT> c = i < w1 ? Tp[i] : Seg<TT>{0, 0};
            pcat[k] = (long long)a.cat;
            pins[k] = (long long)a.inst;
            tcat[k] = (long long)c.cat;
            tins[k] = (long long)c.inst;
        }
#pragma unroll
        for (int k = 0; k < kUnroll; ++k) {
            const bool valid = base + k * 32 + lane < w1;
            long long pi, ti;
            const int pc = classify(pcat[k], pins[k], ids, cids, K, n_things, &pi);
            const int tc = classify(tcat[k], tins[k], ids, cids, K, n_things, &ti);
            if (valid && pc == K && check_preds) flags |= MB200_PQ_UNKNOWN_PREDS;
            const long long k3 = valid ? (long long)(((unsigned long long)(unsigned)pc << 32) | (unsigned)tc) : -1ll;
            const long long a0 = __shfl_sync(kFull, pi, 0), b0 = __shfl_sync(kFull, ti, 0), c0 = __shfl_sync(kFull, k3, 0);
            unsigned peers;
            if (__all_sync(kFull, pi == a0 && ti == b0 && k3 == c0)) {
                peers = kFull;
            } else {
                peers = __match_any_sync(kFull, pi) & __match_any_sync(kFull, ti) & __match_any_sync(kFull, k3);
            }
            // the group leader resolves the colors its lane has not cached; every lane of the group then caches them
            const int leader = __ffs(peers) - 1;
            const bool lead = valid && lane == leader;
            if (lead && (pc != lp_cid || pi != lp_inst || tc != lt_cid || ti != lt_inst)) {
                if (*(const volatile unsigned*)err & MB200_FLAG_CAPACITY) {
                    lp_slot = lt_slot = -1;  // this pass is repeated with larger tables
                } else {
                    if (pc != lp_cid || pi != lp_inst) lp_slot = color_slot(pcol, tb.ccap, pi, pc, used, err);
                    if (tc != lt_cid || ti != lt_inst) lt_slot = color_slot(tcol, tb.ccap, ti, tc, used + 1, err);
                }
            }
            const long long ps = __shfl_sync(kFull, lp_slot, leader), ts = __shfl_sync(kFull, lt_slot, leader);
            if (valid) {
                lp_cid = ps < 0 ? -1 : pc;
                lp_inst = pi;
                lp_slot = ps;
                lt_cid = ts < 0 ? -1 : tc;
                lt_inst = ti;
                lt_slot = ts;
            }
            if (lead && ps >= 0 && ts >= 0) {  // else a table is full and the update is repeated
                const unsigned long long key = ((unsigned long long)(ps + 1) << 32) | (unsigned long long)(ts + 1);
                if (key != run_key) {
                    if (run_key != 0ull)
                        pair_add(tb.pkey + b * tb.pcap, tb.pcnt + b * tb.pcap, tb.pcap, run_key, run_cnt, used + 2, err);
                    run_key = key;
                    run_cnt = 0ull;
                }
                run_cnt += (unsigned)__popc(peers);
            }
        }
    }
    if (run_key != 0ull) pair_add(tb.pkey + b * tb.pcap, tb.pcnt + b * tb.pcap, tb.pcap, run_key, run_cnt, used + 2, err);
    flags = __reduce_or_sync(kFull, flags);
    if (lane == 0 && flags != 0u) atomicOr(err, flags);
}

__device__ __forceinline__ long long pair_pred(unsigned long long key) { return (long long)(key >> 32) - 1; }
__device__ __forceinline__ long long pair_target(unsigned long long key) { return (long long)(key & 0xffffffffull) - 1; }

// every pair's count into the areas of its two colors; the counts of pairs with a void side
__global__ void __launch_bounds__(kThreads) areas_kernel(Tables tb, long long m, int K) {
    const long long total = m * tb.pcap;
    for (long long j = blockIdx.x * (long long)kThreads + threadIdx.x; j < total; j += (long long)gridDim.x * kThreads) {
        const unsigned long long key = tb.pkey[j];
        if (key == 0ull) continue;
        const unsigned long long cnt = tb.pcnt[j];
        const long long base = j / tb.pcap * tb.ccap;
        const long long ps = base + pair_pred(key), ts = base + pair_target(key);
        atomicAdd(tb.parea + ps, cnt);
        atomicAdd(tb.tarea + ts, cnt);
        if (tb.tcol[ts].cid == K) tb.pvoid[ps] = cnt;  // each color has one pair with the void color at most
        if (tb.pcol[ps].cid == K) tb.tvoid[ts] = cnt;
    }
}

__device__ __forceinline__ float f32_ratio(long long a, long long b) { return __fdiv_rn(__ll2float_rn(a), __ll2float_rn(b)); }

// IoU of every same-category pair whose target is not void: matches (> 0.5) and ModifiedPQ stuff IoU sums (> 0)
__global__ void __launch_bounds__(kThreads) match_kernel(Tables tb, long long m, long long img0, int K, int n_things,
                                                         int modified, Partials out) {
    const long long total = m * tb.pcap;
    for (long long j = blockIdx.x * (long long)kThreads + threadIdx.x; j < total; j += (long long)gridDim.x * kThreads) {
        const unsigned long long key = tb.pkey[j];
        if (key == 0ull) continue;
        const long long b = j / tb.pcap, base = b * tb.ccap;
        const long long ps = base + pair_pred(key), ts = base + pair_target(key);
        const int c = tb.tcol[ts].cid;
        if (c == K || tb.pcol[ps].cid != c) continue;
        const long long inter = (long long)tb.pcnt[j];
        const long long uni = (long long)(tb.parea[ps] - tb.pvoid[ps] + tb.tarea[ts] - tb.tvoid[ts]) - inter;
        const float iou = f32_ratio(inter, uni);
        const long long row = (img0 + b) * K + c;
        if (modified && c >= n_things) {
            if (iou > 0.0f) atomicAdd(out.iou + row, (double)iou);
        } else if (iou > 0.5f) {
            tb.pmatch[ps] = 1;
            tb.tmatch[ts] = 1;
            atomicAdd(out.iou + row, (double)iou);
            atomicAdd(out.tp + row, 1);
        }
    }
}

// unmatched non-void colors that are at most half void: false positives (pred table) and false negatives (target table);
// ModifiedPQ counts every stuff target segment as a true positive instead
__global__ void __launch_bounds__(kThreads) unmatched_kernel(Tables tb, long long m, long long img0, int K, int n_things,
                                                             int modified, Partials out) {
    const long long half = m * tb.ccap;
    for (long long j2 = blockIdx.x * (long long)kThreads + threadIdx.x; j2 < 2 * half; j2 += (long long)gridDim.x * kThreads) {
        const bool tgt = j2 >= half;
        const long long j = tgt ? j2 - half : j2;
        const Color col = tgt ? tb.tcol[j] : tb.pcol[j];
        if (col.tag == 0 || col.cid == K) continue;
        const long long row = (img0 + j / tb.ccap) * K + col.cid;
        if (modified && col.cid >= n_things) {
            if (tgt) atomicAdd(out.tp + row, 1);
            continue;
        }
        if (tgt ? tb.tmatch[j] : tb.pmatch[j]) continue;
        const long long vd = (long long)(tgt ? tb.tvoid[j] : tb.pvoid[j]);
        const long long area = (long long)(tgt ? tb.tarea[j] : tb.parea[j]);
        if (f32_ratio(vd, area) <= 0.5f) atomicAdd((tgt ? out.fn : out.fp) + row, 1);
    }
}

// states += sum of the per-image partials in image order; nothing when the update failed
__global__ void __launch_bounds__(kThreads) fold_kernel(Partials part, long long n, int K, double* iou_sum, int* tp, int* fp,
                                                        int* fn, const unsigned* err) {
    if (*(const volatile unsigned*)err != 0u) return;
    for (int c = blockIdx.x * kThreads + threadIdx.x; c < K; c += gridDim.x * kThreads) {
        double s = 0.0;
        unsigned t = 0u, f = 0u, g = 0u;
        for (long long b = 0; b < n; ++b) {
            s += part.iou[b * K + c];
            t += (unsigned)part.tp[b * K + c];
            f += (unsigned)part.fp[b * K + c];
            g += (unsigned)part.fn[b * K + c];
        }
        iou_sum[c] += s;
        tp[c] = (int)((unsigned)tp[c] + t);
        fp[c] = (int)((unsigned)fp[c] + f);
        fn[c] = (int)((unsigned)fn[c] + g);
    }
}

// ---- launchers -----------------------------------------------------------------------------------------------------------
long long cdiv(long long a, long long b) { return (a + b - 1) / b; }
long long align16(long long v) { return cdiv(v, 16) * 16; }

long long partial_bytes(long long n, long long K) { return align16(n * K * 8) + 3 * align16(n * K * 4); }

// hash tables of `m` images
long long table_bytes(long long m, long long ccap, long long pcap) {
    return 2 * align16(m * ccap * 16) + 4 * align16(m * ccap * 8) + 2 * align16(m * ccap) + 2 * align16(m * pcap * 8) +
           align16(m * 3 * 4);
}

Tables carve_tables(char* p, long long m, long long ccap, long long pcap) {
    Tables tb;
    auto take = [&p](long long bytes) {
        char* q = p;
        p += align16(bytes);
        return q;
    };
    tb.pcol = reinterpret_cast<Color*>(take(m * ccap * 16));
    tb.tcol = reinterpret_cast<Color*>(take(m * ccap * 16));
    tb.parea = reinterpret_cast<unsigned long long*>(take(m * ccap * 8));
    tb.tarea = reinterpret_cast<unsigned long long*>(take(m * ccap * 8));
    tb.pvoid = reinterpret_cast<unsigned long long*>(take(m * ccap * 8));
    tb.tvoid = reinterpret_cast<unsigned long long*>(take(m * ccap * 8));
    tb.pmatch = reinterpret_cast<unsigned char*>(take(m * ccap));
    tb.tmatch = reinterpret_cast<unsigned char*>(take(m * ccap));
    tb.pkey = reinterpret_cast<unsigned long long*>(take(m * pcap * 8));
    tb.pcnt = reinterpret_cast<unsigned long long*>(take(m * pcap * 8));
    tb.used = reinterpret_cast<unsigned*>(take(m * 3 * 4));
    tb.ccap = ccap;
    tb.pcap = pcap;
    return tb;
}

bool pow2_capacity(long long c) { return c >= kMinCapacity && c <= kMaxCapacity && (c & (c - 1)) == 0; }

int eval_grid(long long work) { return (int)std::max(1ll, std::min(cdiv(work, kThreads), (long long)sm_count() * 4)); }

template <typename TP, typename TT>
int launch_update(const void* preds, const void* target, long long n, long long P, const long long* cats, int K, int n_things,
                  int modified, int check_preds, long long mpl, long long ccap, long long pcap, double* iou_sum, int* tp,
                  int* fp, int* fn, char* scratch, unsigned* err, cudaStream_t st) {
    const long long pb = partial_bytes(n, K);
    Partials part;
    part.iou = reinterpret_cast<double*>(scratch);
    part.tp = reinterpret_cast<int*>(scratch + align16(n * K * 8));
    part.fp = part.tp + align16(n * K * 4) / 4;
    part.fn = part.fp + align16(n * K * 4) / 4;
    MB200_CUDA_OK(cudaMemsetAsync(scratch, 0, (size_t)pb, st));
    const size_t smem = K <= kSmemCats ? (size_t)2 * K * sizeof(long long) : 0;
    const Seg<TP>* p = reinterpret_cast<const Seg<TP>*>(preds);
    const Seg<TT>* t = reinterpret_cast<const Seg<TT>*>(target);
    for (long long img0 = 0; img0 < n; img0 += mpl) {
        const long long m = std::min(mpl, n - img0);
        Tables tb = carve_tables(scratch + pb, m, ccap, pcap);
        MB200_CUDA_OK(cudaMemsetAsync(scratch + pb, 0, (size_t)table_bytes(m, ccap, pcap), st));
        // about 8 CTAs per SM over the launch, at least kMinTile pixels each; tiles split evenly over the 8 warps
        long long tiles = std::max(1ll, std::min(cdiv((long long)sm_count() * 8, m), cdiv(P, kMinTile)));
        const long long tile = cdiv(cdiv(P, tiles), 32 * kWarps) * 32 * kWarps;
        tiles = cdiv(P, tile);
        MB200_REQUIRE(m * tiles < (1ll << 31), "too many images for one launch");
        pixel_kernel<TP, TT><<<(unsigned)(m * tiles), kThreads, smem, st>>>(p + img0 * P, t + img0 * P, P, tiles, tile, cats, K,
                                                                             n_things, check_preds, tb, err);
        count_launch();
        MB200_CUDA_OK(cudaGetLastError());
        areas_kernel<<<eval_grid(m * pcap), kThreads, 0, st>>>(tb, m, K);
        count_launch();
        match_kernel<<<eval_grid(m * pcap), kThreads, 0, st>>>(tb, m, img0, K, n_things, modified, part);
        count_launch();
        unmatched_kernel<<<eval_grid(2 * m * ccap), kThreads, 0, st>>>(tb, m, img0, K, n_things, modified, part);
        count_launch();
        MB200_CUDA_OK(cudaGetLastError());
    }
    fold_kernel<<<(unsigned)cdiv(K, kThreads), kThreads, 0, st>>>(part, n, K, iou_sum, tp, fp, fn, err);
    count_launch();
    return check_cuda(cudaGetLastError(), "panoptic update launch");
}

}  // namespace
}  // namespace mb200

using namespace mb200;

// =====================================================================================================
// C-ABI
// =====================================================================================================
extern "C" int64_t mb200_panoptic_scratch_bytes(int64_t n, int64_t pixels, int64_t num_categories, int64_t images_per_launch,
                                               int64_t color_capacity, int64_t pair_capacity, int preds_dtype, int target_dtype) {
    if (n < 0 || pixels < 0 || pixels > (1ll << 30) || num_categories < 1 || num_categories >= (1ll << 30) ||
        images_per_launch < 1 || !pow2_capacity(color_capacity) || !pow2_capacity(pair_capacity) ||
        !is_label_tag(preds_dtype) || preds_dtype == MB200_BOOL || !is_label_tag(target_dtype) || target_dtype == MB200_BOOL)
        return -1;
    const long long m = std::max(1ll, std::min((long long)images_per_launch, (long long)n));
    return partial_bytes(n, num_categories) + table_bytes(m, color_capacity, pair_capacity);
}

extern "C" int mb200_panoptic_update(const void* preds, int preds_dtype, const void* target, int target_dtype, int64_t n,
                                     int64_t pixels, const int64_t* categories, int64_t num_categories, int64_t num_things,
                                     int modified, int allow_unknown_preds, int64_t images_per_launch, int64_t color_capacity,
                                     int64_t pair_capacity, double* iou_sum, int32_t* true_positives, int32_t* false_positives,
                                     int32_t* false_negatives, void* scratch, int64_t scratch_bytes, uint32_t* err_flag,
                                     void* stream) {
    const int64_t need = mb200_panoptic_scratch_bytes(n, pixels, num_categories, images_per_launch, color_capacity, pair_capacity,
                                                      preds_dtype, target_dtype);
    MB200_REQUIRE(need >= 0, "bad sizes, capacities or dtype tags (%d, %d)", preds_dtype, target_dtype);
    MB200_REQUIRE(num_things >= 0 && num_things <= num_categories, "num_things %lld out of range", (long long)num_things);
    MB200_REQUIRE(categories && iou_sum && true_positives && false_positives && false_negatives && err_flag && scratch,
                  "NULL pointer");
    MB200_REQUIRE(scratch_bytes >= need && (reinterpret_cast<uintptr_t>(scratch) & 15) == 0,
                  "scratch must be 16-byte aligned and mb200_panoptic_scratch_bytes(...) bytes");
    MB200_REQUIRE(n * pixels == 0 || (preds && target), "NULL pointer");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    MB200_CUDA_OK(cudaMemsetAsync(err_flag, 0, sizeof(uint32_t), st));
    if (n == 0 || pixels == 0) return 0;
    const long long mpl = std::min((long long)images_per_launch, (long long)n);
    const long long* cats = reinterpret_cast<const long long*>(categories);
    unsigned* err = reinterpret_cast<unsigned*>(err_flag);
    return with_label_type(preds_dtype, [&](auto a) {
        return with_label_type(target_dtype, [&](auto b) -> int {
            using TP = typename decltype(a)::type;
            using TT = typename decltype(b)::type;
            MB200_REQUIRE((reinterpret_cast<uintptr_t>(preds) % (2 * sizeof(TP))) == 0 &&
                              (reinterpret_cast<uintptr_t>(target) % (2 * sizeof(TT))) == 0,
                          "preds and target must be aligned to one (category, instance) pair");
            return launch_update<TP, TT>(preds, target, n, pixels, cats, (int)num_categories, (int)num_things, modified,
                                         allow_unknown_preds ? 0 : 1, mpl, color_capacity, pair_capacity, iou_sum,
                                         reinterpret_cast<int*>(true_positives), reinterpret_cast<int*>(false_positives),
                                         reinterpret_cast<int*>(false_negatives), reinterpret_cast<char*>(scratch), err, st);
        });
    });
}
