// K8 — COCO-style mean average precision / recall for bounding boxes, evaluated on the device.
//
// Reference path replaced: detection/mean_ap.py:521-598 (`MeanAveragePrecision.compute`), which marshals every box to
// host Python objects (:867-958, one `.cpu().tolist()` per element) and hands all arithmetic to the third-party
// `pycocotools.cocoeval.COCOeval` (`evaluate` / `accumulate`; `summarize` stays in Python here too) and `maskApi.c:bbIou`.
// The algorithm restated (and cited step by step) in oracle/coco_map.py is what these kernels implement:
//
//   evaluate   one CTA per image: class index lookup, per-(image, class) score ranks (stable, = mergesort on -score,
//              NaN last), greedy matching for every (class, area range, IoU threshold) with fp64 IoUs computed on the
//              fly from the fp32 xywh boxes, crowd / area-range ignore rules, per-detection match+ignore bit words (area*T + thr),
//              non-ignored ground-truth counts per (class, area).
//   sort       stable LSD radix sort of all detections by (class, score desc, NaN last) — 64-bit key, 32-bit payload
//              (radix_sort.cuh); the natural order (image, original index) is exactly COCOeval's concatenation order.
//   accumulate one CTA per (class, area, maxDet): compaction to rank < maxDet, integer TP/FP prefix sums per IoU
//              threshold, fp64 precision with `np.spacing(1)`, right-to-left running maximum, 101-point
//              `searchsorted(side="left")` sampling, recall.
//
// Everything is integer or fp64 and order-deterministic: results are bitwise reproducible.
#include <algorithm>

#include "common.cuh"
#include "radix_sort.cuh"

namespace mb200 {

constexpr int kMapAreas = 4;
constexpr int kMapMaxThr = 16;  // T <= 16 so that area*T + thr fits a 64-bit word
constexpr int kGtmWords = 4;    // "matched" bit mask kept in registers: <= 256 ground truths of one class in one image;
                                // busier images switch to a per-thread mask in shared memory (kSmemMask)

struct MapEvalArgs {
    const float4* det_box;  // xywh
    const float* det_score;
    const long long* det_label;
    const int* det_off;  // [n_img + 1]
    const float4* gt_box;
    const long long* gt_label;
    const unsigned char* gt_crowd;
    const double* gt_area_given;  // <= 0: use w*h (unless gt_area_exact)
    const int* gt_off;
    // instance masks (K12, maskiou.cu) instead of boxes: per image a [D][G] table of intersection pixel counts + mask areas
    const double* pair_inter;     // NULL: box IoU
    const long long* pair_off;    // [n_img] offset of the image's table
    const double* det_mask_area;  // [n_det]
    const double* gt_mask_area;   // [n_gt]   (union of the IoU; the area-range test uses gt_area_given)
    int gt_area_exact;            // gt_area_given is final (the caller resolved "given or computed")
    const long long* classes;  // sorted unique labels, [K]
    int K;
    int micro;
    int T;
    int max_det_last;
    double iou_thr[kMapMaxThr];
    // outputs
    int* det_cat;
    int* det_rank;
    unsigned long long* det_match;
    unsigned long long* det_ignore;
    int* npig;  // [K][4]
    unsigned* err;
};

__device__ __forceinline__ int class_index(const long long* __restrict__ classes, int K, long long label) {
    int lo = 0, hi = K;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (classes[mid] < label) lo = mid + 1;
        else hi = mid;
    }
    return lo;  // labels come from the same set the class list was built from
}

__device__ __forceinline__ bool area_outside(double area, int a) {
    // COCOeval.params.areaRng: all [0, 1e10], small [0, 32^2], medium [32^2, 96^2], large [96^2, 1e10]
    const double lo = (a == 2) ? 1024.0 : (a == 3) ? 9216.0 : 0.0;
    const double hi = (a == 1) ? 1024.0 : (a == 2) ? 9216.0 : 1e10;
    return area < lo || area > hi;
}

// maskApi.c:bbIou in double; `crowd`: union = detection area
__device__ __forceinline__ double bb_iou(const float4 d, const float4 g, bool crowd) {
    const double dx = d.x, dy = d.y, dw = d.z, dh = d.w, gx = g.x, gy = g.y, gw = g.z, gh = g.w;
    const double w = fmin(dx + dw, gx + gw) - fmax(dx, gx);
    if (w <= 0) return 0.0;
    const double h = fmin(dy + dh, gy + gh) - fmax(dy, gy);
    if (h <= 0) return 0.0;
    const double inter = w * h;
    const double da = dw * dh, ga = gw * gh;
    const double uni = crowd ? da : da + ga - inter;
    return inter / uni;
}

// maskApi.c:rleIou: intersection / union from pixel counts; no intersection -> 0 (also for empty masks)
__device__ __forceinline__ double mask_iou(double inter, double det_area, double gt_area, bool crowd) {
    if (inter <= 0.0) return 0.0;
    return inter / (crowd ? det_area : det_area + gt_area - inter);
}

// COCOeval's detection order (`np.argsort(-score, kind="mergesort")`, per image in evaluateImg and across images in
// accumulate) as an ascending u32 key: descending score, -0 and +0 equal, NaN after everything (-inf included); equal keys keep
// the input order.  The per-image rank and the accumulate sort key both use it.  (f32_order_key puts NaN on top, as
// torch.argmax does; negated, that would sort NaN first.)
__device__ __forceinline__ unsigned coco_det_order_key(float s) {
    return s != s ? 0xffffffffu : ~f32_order_key(s);
}

__host__ __device__ inline size_t map_eval_smem_bytes(int max_d, int max_g) {
    size_t b = 0;
    b += (size_t)(max_d + max_g) * 8;       // mask areas (mask mode; boxes leave them unused)
    b += (size_t)max_d * (16 + 8 + 8);      // box, match word, ignore word
    b += (size_t)max_g * (16 + 8);          // box, area
    b += (size_t)max_d * (4 + 4 + 4 + 4);   // score key, cat, rank, by_pos
    b += (size_t)max_g * (4 + 4);           // cat, crowd(int)
    b += (size_t)(max_d + max_g) * 4 * 3;   // cats list, cat_start, cat_cnt
    return b + 64;
}

template <bool kSmemMask>
__global__ void __launch_bounds__(256) map_evaluate_kernel(MapEvalArgs p, int max_d, int max_g) {
    extern __shared__ __align__(16) unsigned char sm_raw[];
    __shared__ int ncats;
    const int img = blockIdx.x;
    const int d0 = p.det_off[img], D = p.det_off[img + 1] - d0;
    const int g0 = p.gt_off[img], G = p.gt_off[img + 1] - g0;
    // carve (8/16-byte members first)
    unsigned char* ptr = sm_raw;
    float4* dbox = reinterpret_cast<float4*>(ptr); ptr += (size_t)max_d * 16;
    float4* gbox = reinterpret_cast<float4*>(ptr); ptr += (size_t)max_g * 16;
    unsigned long long* dmatch = reinterpret_cast<unsigned long long*>(ptr); ptr += (size_t)max_d * 8;
    unsigned long long* dign = reinterpret_cast<unsigned long long*>(ptr); ptr += (size_t)max_d * 8;
    double* garea = reinterpret_cast<double*>(ptr); ptr += (size_t)max_g * 8;
    double* dmarea = reinterpret_cast<double*>(ptr); ptr += (size_t)max_d * 8;  // mask mode: detection mask areas
    double* gmarea = reinterpret_cast<double*>(ptr); ptr += (size_t)max_g * 8;  //            ground-truth mask areas
    const bool masks = p.pair_inter != nullptr;
    const double* __restrict__ inter_tab = masks ? p.pair_inter + p.pair_off[img] : nullptr;
    unsigned* dkey = reinterpret_cast<unsigned*>(ptr); ptr += (size_t)max_d * 4;  // coco_det_order_key of the score
    int* dcat = reinterpret_cast<int*>(ptr); ptr += (size_t)max_d * 4;
    int* drank = reinterpret_cast<int*>(ptr); ptr += (size_t)max_d * 4;
    int* by_pos = reinterpret_cast<int*>(ptr); ptr += (size_t)max_d * 4;
    int* gcat = reinterpret_cast<int*>(ptr); ptr += (size_t)max_g * 4;
    int* gcrowd = reinterpret_cast<int*>(ptr); ptr += (size_t)max_g * 4;
    int* cats = reinterpret_cast<int*>(ptr); ptr += (size_t)(max_d + max_g) * 4;
    int* cat_start = reinterpret_cast<int*>(ptr); ptr += (size_t)(max_d + max_g) * 4;
    int* cat_cnt = reinterpret_cast<int*>(ptr); ptr += (size_t)(max_d + max_g) * 4;
    // kSmemMask: one "ground truth already matched" bit per ground truth of the image, per thread
    const int mask_words = kSmemMask ? (max_g + 63) / 64 : kGtmWords;
    unsigned long long* smem_mask = reinterpret_cast<unsigned long long*>(sm_raw + (((size_t)(ptr - sm_raw) + 7) & ~(size_t)7));

    const int tid = threadIdx.x, nth = blockDim.x;
    if (tid == 0) ncats = 0;
    for (int i = tid; i < D; i += nth) {
        dbox[i] = p.det_box[d0 + i];
        dkey[i] = coco_det_order_key(p.det_score[d0 + i]);
        dcat[i] = p.micro ? 0 : class_index(p.classes, p.K, p.det_label[d0 + i]);
        dmatch[i] = 0ull;
        dign[i] = 0ull;
        if (masks) dmarea[i] = p.det_mask_area[d0 + i];
    }
    for (int i = tid; i < G; i += nth) {
        const float4 b = p.gt_box[g0 + i];
        gbox[i] = b;
        gcat[i] = p.micro ? 0 : class_index(p.classes, p.K, p.gt_label[g0 + i]);
        gcrowd[i] = p.gt_crowd[g0 + i] != 0;
        const double given = p.gt_area_given[g0 + i];
        garea[i] = (p.gt_area_exact || given > 0.0) ? given : (double)b.z * (double)b.w;  // detection/mean_ap.py:920-925
        if (masks) gmarea[i] = p.gt_mask_area[g0 + i];
    }
    __syncthreads();

    // ---- per-(image, class) rank in COCOeval's order (coco_det_order_key, ties by original index) ----
    for (int i = tid; i < D; i += nth) {
        const int c = dcat[i];
        const unsigned key = dkey[i];
        int r = 0;
        for (int j = 0; j < D; ++j)
            if (dcat[j] == c && (dkey[j] < key || (dkey[j] == key && j < i))) r++;
        drank[i] = r;
    }
    // ---- distinct classes of this image (detections and ground truths) ----
    for (int e = tid; e < D + G; e += nth) {
        const int c = e < D ? dcat[e] : gcat[e - D];
        bool first = true;
        for (int j = 0; j < e && first; ++j) first = (j < D ? dcat[j] : gcat[j - D]) != c;
        if (first) cats[atomicAdd(&ncats, 1)] = c;
    }
    __syncthreads();
    const int nc = ncats;
    for (int ci = tid; ci < nc; ci += nth) {
        int cnt = 0;
        for (int j = 0; j < D; ++j) cnt += dcat[j] == cats[ci];
        cat_cnt[ci] = cnt;
    }
    __syncthreads();
    if (tid == 0) {
        int run = 0;
        for (int ci = 0; ci < nc; ++ci) {
            cat_start[ci] = run;
            run += cat_cnt[ci];
        }
    }
    __syncthreads();
    for (int i = tid; i < D; i += nth) {
        int ci = 0;
        while (cats[ci] != dcat[i]) ++ci;
        by_pos[cat_start[ci] + drank[i]] = i;
    }
    __syncthreads();

    // ---- greedy matching: one thread per (class, area range, IoU threshold) ----
    const int T = p.T;
    const int work = nc * kMapAreas * T;
    for (int w = tid; w < work; w += nth) {
        const int ci = w / (kMapAreas * T);
        const int a = (w / T) % kMapAreas;
        const int t = w % T;
        const int c = cats[ci];
        const int bit = a * T + t;
        const int nd = min(cat_cnt[ci], p.max_det_last);
        const double thr0 = fmin(p.iou_thr[t], 1.0 - 1e-10);
        unsigned long long gtm_regs[kGtmWords];
        unsigned long long* gtm = kSmemMask ? smem_mask + (size_t)tid * mask_words : gtm_regs;
        if (kSmemMask) {
            for (int q = 0; q < mask_words; ++q) gtm[q] = 0ull;
        } else {
#pragma unroll
            for (int q = 0; q < kGtmWords; ++q) gtm_regs[q] = 0ull;
        }
        const int mask_bits = 64 * mask_words;

        if (t == 0) {  // one thread per (class, area) counts the non-ignored ground truths
            int n_valid = 0, n_c = 0;
            for (int g = 0; g < G; ++g) {
                if (gcat[g] != c) continue;
                n_c++;
                n_valid += !(gcrowd[g] || area_outside(garea[g], a));
            }
            if (n_valid) atomicAdd(&p.npig[c * kMapAreas + a], n_valid);
            if (n_c > mask_bits && p.err) atomicOr(p.err, MB200_FLAG_CAPACITY);
        }
        for (int r = 0; r < nd; ++r) {
            const int d = by_pos[cat_start[ci] + r];
            const float4 db = dbox[d];
            double best = thr0;
            int m = -1;
            bool m_ig = false;
            for (int phase = 0; phase < 2; ++phase) {
                if (phase == 1 && m > -1 && !m_ig) break;  // a non-ignored match is never traded for an ignored gt
                int ord = -1;
                for (int g = 0; g < G; ++g) {
                    if (gcat[g] != c) continue;
                    ++ord;
                    const bool crowd = gcrowd[g] != 0;
                    const bool ig = crowd || area_outside(garea[g], a);
                    if ((int)ig != phase) continue;
                    if (ord < mask_bits && ((gtm[ord >> 6] >> (ord & 63)) & 1ull) && !crowd) continue;
                    const double iou = masks ? mask_iou(inter_tab[(long long)d * G + g], dmarea[d], gmarea[g], crowd)
                                             : bb_iou(db, gbox[g], crowd);
                    if (iou < best) continue;
                    best = iou;
                    m = ord;
                    m_ig = ig;
                }
            }
            if (m == -1) {
                if (area_outside(masks ? dmarea[d] : (double)db.z * (double)db.w, a)) atomicOr(&dign[d], 1ull << bit);
            } else {
                atomicOr(&dmatch[d], 1ull << bit);
                if (m_ig) atomicOr(&dign[d], 1ull << bit);
                if (m < mask_bits) gtm[m >> 6] |= 1ull << (m & 63);
            }
        }
    }
    __syncthreads();
    for (int i = tid; i < D; i += nth) {
        p.det_cat[d0 + i] = dcat[i];
        p.det_rank[d0 + i] = drank[i];
        p.det_match[d0 + i] = dmatch[i];
        p.det_ignore[d0 + i] = dign[i];
    }
}

// sort key: (class << 32) | COCOeval order key of the score; payload: detection index
__global__ void __launch_bounds__(256) map_pack_keys_kernel(const int* __restrict__ det_cat,
                                                            const float* __restrict__ det_score, int n,
                                                            unsigned long long* __restrict__ keys,
                                                            unsigned* __restrict__ vals) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        keys[i] = ((unsigned long long)(unsigned)det_cat[i] << 32) | (unsigned long long)coco_det_order_key(det_score[i]);
        vals[i] = (unsigned)i;
    }
}

// range_start[k] = first sorted position whose class is >= k   (k = 0..K)
__global__ void map_class_ranges_kernel(const unsigned long long* __restrict__ sorted_keys, int n, int K,
                                        int* __restrict__ range_start) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k > K) return;
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if ((int)(sorted_keys[mid] >> 32) < k) lo = mid + 1;
        else hi = mid;
    }
    range_start[k] = lo;
}

struct MapAccArgs {
    const unsigned* sorted_idx;  // detection index in (class, score desc) order
    const int* range_start;      // [K + 1]
    const int* det_rank;
    const unsigned long long* det_match;
    const unsigned long long* det_ignore;
    const float* det_score;
    const int* npig;
    const double* rec_thr;  // [R]
    int K, T, R, M;
    int class_lo;  // blockIdx.x counts from here (class-sharded accumulation)
    int max_dets[8];
    int n_det;
    // scratch planes [A*M][n_det]
    unsigned* tp_cum;
    double* prec;
    unsigned* cidx;
    // outputs (pre-filled with -1)
    double* precision;  // [T, R, K, A, M]
    double* recall;     // [T, K, A, M]
    double* scores;     // [T, R, K, A, M]
};

__device__ __forceinline__ unsigned block_scan_excl_u32(unsigned v, unsigned* sm8, unsigned& total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned t = __shfl_up_sync(kFull, incl, o);
        if (lane >= o) incl += t;
    }
    __syncthreads();
    if (lane == 31) sm8[warp] = incl;
    __syncthreads();
    unsigned woff = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < 8; ++w) {
        const unsigned s = sm8[w];
        if (w < warp) woff += s;
        tot += s;
    }
    total = tot;
    return woff + incl - v;
}

__global__ void __launch_bounds__(256) map_accumulate_kernel(MapAccArgs p) {
    __shared__ unsigned sm8[8];
    __shared__ double smd[8];
    const int k = blockIdx.x + p.class_lo;
    const int a = blockIdx.y / p.M, m = blockIdx.y % p.M;
    const int np_ig = p.npig[k * kMapAreas + a];
    if (np_ig == 0) return;  // COCOeval.accumulate: `if npig == 0: continue` -> stays -1
    const int base = p.range_start[k];
    const int n = p.range_start[k + 1] - base;
    const int max_det = p.max_dets[m];
    const size_t plane = (size_t)blockIdx.y * p.n_det + base;
    unsigned* __restrict__ tp_cum = p.tp_cum + plane;
    double* __restrict__ prec = p.prec + plane;
    unsigned* __restrict__ cidx = p.cidx + plane;
    const int tid = threadIdx.x;

    // ---- compaction: detections of this class with rank < maxDet, in sorted order ----
    unsigned nd = 0;
    for (int t0 = 0; t0 < n; t0 += 256) {
        const int j = t0 + tid;
        unsigned o = 0, keep = 0;
        if (j < n) {
            o = p.sorted_idx[base + j];
            keep = p.det_rank[o] < max_det;
        }
        unsigned tot;
        const unsigned pos = nd + block_scan_excl_u32(keep, sm8, tot);
        if (keep) cidx[pos] = o;
        nd += tot;
    }
    __syncthreads();
    const double dnp = (double)np_ig;
    const double eps = 2.220446049250313e-16;  // np.spacing(1)
    const size_t sK = (size_t)kMapAreas * p.M, sR = (size_t)p.K * sK, sT = (size_t)p.R * sR;
    const size_t out_off = (size_t)k * sK + (size_t)a * p.M + m;

    for (int t = 0; t < p.T; ++t) {
        const int bit = a * p.T + t;
        if (nd == 0) {  // no detections: recall 0, precision/scores 0 at every recall threshold
            for (int r = tid; r < p.R; r += 256) {
                p.precision[(size_t)t * sT + (size_t)r * sR + out_off] = 0.0;
                p.scores[(size_t)t * sT + (size_t)r * sR + out_off] = 0.0;
            }
            if (tid == 0) p.recall[(size_t)t * sR + out_off] = 0.0;
            continue;
        }
        // ---- pass 1: TP / FP prefix sums, precision ----
        unsigned c_tp = 0, c_fp = 0;
        for (unsigned t0 = 0; t0 < nd; t0 += 256) {
            const unsigned j = t0 + tid;
            unsigned tp = 0, fp = 0;
            if (j < nd) {
                const unsigned o = cidx[j];
                const bool matched = (p.det_match[o] >> bit) & 1ull;
                const bool ign = (p.det_ignore[o] >> bit) & 1ull;
                tp = matched && !ign;
                fp = !matched && !ign;
            }
            unsigned tot_tp, tot_fp;
            const unsigned etp = c_tp + block_scan_excl_u32(tp, sm8, tot_tp);
            const unsigned efp = c_fp + block_scan_excl_u32(fp, sm8, tot_fp);
            if (j < nd) {
                const unsigned itp = etp + tp, ifp = efp + fp;
                tp_cum[j] = itp;
                prec[j] = (double)itp / ((double)ifp + (double)itp + eps);
            }
            c_tp += tot_tp;
            c_fp += tot_fp;
        }
        __syncthreads();
        // ---- pass 2: right-to-left running maximum of the precision ----
        double carry = 0.0;
        for (int t0 = (int)((nd - 1) / 256) * 256; t0 >= 0; t0 -= 256) {
            const unsigned j = (unsigned)t0 + tid;
            double v = j < nd ? prec[j] : 0.0;
            const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const double other = __shfl_down_sync(kFull, v, o);
                if (lane + o < 32) v = fmax(v, other);
            }
            __syncthreads();
            if (lane == 0) smd[warp] = v;
            __syncthreads();
            double later = carry;
#pragma unroll
            for (int w2 = 0; w2 < 8; ++w2)
                if (w2 > warp) later = fmax(later, smd[w2]);
            v = fmax(v, later);
            if (j < nd) prec[j] = v;
            double tile_max = carry;
#pragma unroll
            for (int w2 = 0; w2 < 8; ++w2) tile_max = fmax(tile_max, smd[w2]);
            carry = tile_max;
            __syncthreads();
        }
        // ---- pass 3: sample at the recall thresholds (np.searchsorted(rc, recThrs, side="left")) ----
        for (int r = tid; r < p.R; r += 256) {
            const double thr = p.rec_thr[r];
            unsigned lo = 0, hi = nd;
            while (lo < hi) {
                const unsigned mid = (lo + hi) >> 1;
                if ((double)tp_cum[mid] / dnp < thr) lo = mid + 1;
                else hi = mid;
            }
            double q = 0.0, s = 0.0;
            if (lo < nd) {
                q = prec[lo];
                s = (double)p.det_score[cidx[lo]];
            }
            p.precision[(size_t)t * sT + (size_t)r * sR + out_off] = q;
            p.scores[(size_t)t * sT + (size_t)r * sR + out_off] = s;
        }
        if (tid == 0) p.recall[(size_t)t * sR + out_off] = (double)tp_cum[nd - 1] / dnp;
        __syncthreads();
    }
}

__global__ void fill_double_kernel(double* p, long long n, double v) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        p[i] = v;
}
__global__ void zero_int_kernel(int* p, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = 0;
}

namespace {
struct MapWs {
    int *det_cat, *det_rank, *npig, *range_start;
    unsigned long long *det_match, *det_ignore, *keys_a, *keys_b;
    unsigned *vals_a, *vals_b, *sort_scratch, *tp_cum, *cidx;
    double* prec;
};
inline unsigned char* bump(unsigned char*& p, int64_t bytes) {
    unsigned char* r = p;
    p += (bytes + 255) / 256 * 256;
    return r;
}
MapWs carve(void* ws, int64_t nd, int64_t K, int64_t M, int64_t* total) {
    unsigned char* p = reinterpret_cast<unsigned char*>(ws);
    unsigned char* p0 = p;
    const int64_t n1 = nd > 0 ? nd : 1;
    const int64_t tiles = (n1 + kSortTile - 1) / kSortTile;
    MapWs w;
    w.det_match = (unsigned long long*)bump(p, n1 * 8);
    w.det_ignore = (unsigned long long*)bump(p, n1 * 8);
    w.keys_a = (unsigned long long*)bump(p, n1 * 8);
    w.keys_b = (unsigned long long*)bump(p, n1 * 8);
    w.prec = (double*)bump(p, kMapAreas * M * n1 * 8);
    w.det_cat = (int*)bump(p, n1 * 4);
    w.det_rank = (int*)bump(p, n1 * 4);
    w.vals_a = (unsigned*)bump(p, n1 * 4);
    w.vals_b = (unsigned*)bump(p, n1 * 4);
    w.tp_cum = (unsigned*)bump(p, kMapAreas * M * n1 * 4);
    w.cidx = (unsigned*)bump(p, kMapAreas * M * n1 * 4);
    w.npig = (int*)bump(p, (K + 1) * kMapAreas * 4);
    w.range_start = (int*)bump(p, (K + 2) * 4);
    w.sort_scratch = (unsigned*)bump(p, (int64_t)radix_sort_scratch_words(n1, 1, 8) * 4);
    (void)tiles;
    if (total) *total = (int64_t)(p - p0) + 256;
    return w;
}
}  // namespace

}  // namespace mb200

using namespace mb200;

extern "C" int64_t mb200_coco_map_workspace_bytes(int64_t n_det, int64_t num_classes, int64_t num_max_dets) {
    if (n_det < 0 || num_classes < 0 || num_max_dets < 1) return -1;
    int64_t total = 0;
    (void)carve(nullptr, n_det, num_classes, num_max_dets, &total);
    return total;
}

namespace {

// Phase 1 — per-image greedy matching (COCOeval.evaluateImg): one CTA per image of THIS call.  Outputs per detection (image
// order): class index, rank inside its (image, class), match / ignore bit words; `npig` [K][4] is ADDED to (caller zeroes it).
int map_match_impl(const float* det_box_xywh, const float* det_score, const int64_t* det_label, const int32_t* det_off,
                   const float* gt_box_xywh, const int64_t* gt_label, const uint8_t* gt_crowd, const double* gt_area,
                   const int32_t* gt_off, int64_t n_img, int64_t max_det_per_img, int64_t max_gt_per_img,
                   const int64_t* classes, int64_t num_classes, int micro, const double* iou_thr_host, int T, int max_det_last,
                   int* det_cat, int* det_rank, unsigned long long* det_match, unsigned long long* det_ignore, int* npig,
                   uint32_t* err_flag, cudaStream_t st, const double* pair_inter = nullptr, const int64_t* pair_off = nullptr,
                   const double* det_mask_area = nullptr, const double* gt_mask_area = nullptr, int gt_area_exact = 0) {
    if (n_img == 0) return 0;
    // More than 256 ground truths in one image MAY put more than 256 of one class there: then the per-thread "matched" masks
    // move from registers to shared memory, one bit per ground truth of the image per thread.
    const bool smem_mask = max_gt_per_img > 64 * kGtmWords;
    const size_t smem = map_eval_smem_bytes((int)max_det_per_img, (int)max_gt_per_img) +
                        (smem_mask ? (size_t)256 * ((max_gt_per_img + 63) / 64) * 8 + 8 : 0);
    if (smem > 200 * 1024) {
        set_error("an image holds %lld detections / %lld ground truths: more than the evaluate kernel can stage in "
                  "shared memory", (long long)max_det_per_img, (long long)max_gt_per_img);
        return MB200_ERR_UNSUPPORTED;
    }
    MapEvalArgs ea;
    ea.det_box = reinterpret_cast<const float4*>(det_box_xywh);
    ea.det_score = det_score;
    ea.det_label = reinterpret_cast<const long long*>(det_label);
    ea.det_off = det_off;
    ea.gt_box = reinterpret_cast<const float4*>(gt_box_xywh);
    ea.gt_label = reinterpret_cast<const long long*>(gt_label);
    ea.gt_crowd = gt_crowd;
    ea.gt_area_given = gt_area;
    ea.gt_off = gt_off;
    ea.pair_inter = pair_inter;
    ea.pair_off = reinterpret_cast<const long long*>(pair_off);
    ea.det_mask_area = det_mask_area;
    ea.gt_mask_area = gt_mask_area;
    ea.gt_area_exact = gt_area_exact;
    ea.classes = reinterpret_cast<const long long*>(classes);
    ea.K = (int)num_classes;
    ea.micro = micro;
    ea.T = T;
    ea.max_det_last = max_det_last;
    for (int t = 0; t < T; ++t) ea.iou_thr[t] = iou_thr_host[t];
    ea.det_cat = det_cat;
    ea.det_rank = det_rank;
    ea.det_match = det_match;
    ea.det_ignore = det_ignore;
    ea.npig = npig;
    ea.err = err_flag;
    if (smem_mask) {
        MB200_CUDA_OK(ensure_dynamic_smem(map_evaluate_kernel<true>, 200 * 1024));
        map_evaluate_kernel<true><<<(unsigned)n_img, 256, smem, st>>>(ea, (int)max_det_per_img, (int)max_gt_per_img);
    } else {
        MB200_CUDA_OK(ensure_dynamic_smem(map_evaluate_kernel<false>, 200 * 1024));
        map_evaluate_kernel<false><<<(unsigned)n_img, 256, smem, st>>>(ea, (int)max_det_per_img, (int)max_gt_per_img);
    }
    count_launch();
    return check_cuda(cudaGetLastError(), "coco map match launch");
}

// Phase 2 — COCOeval.accumulate for classes [class_lo, class_hi): stable sort of the records by (class, score desc) — ties keep
// the order the records are GIVEN in —, integer TP / FP prefix sums, fp64 precision envelope, recall-threshold sampling.
// precision / recall / scores are full-size [.., K, ..] arrays, pre-filled with -1 here; only the owned classes are written.
int map_accumulate_impl(const int* det_cat, const float* det_score, const int* det_rank, const unsigned long long* det_match,
                        const unsigned long long* det_ignore, int nd, const int* npig, int K, int class_lo, int class_hi, int T,
                        const double* rec_thr_dev, int R, const int64_t* max_dets_host, int M, const MapWs& w, double* precision,
                        double* recall, double* scores, uint32_t* err_flag, cudaStream_t st) {
    const long long n_prec = (long long)T * R * K * kMapAreas * M;
    const long long n_rec = (long long)T * K * kMapAreas * M;
    fill_double_kernel<<<256, 256, 0, st>>>(precision, n_prec, -1.0);
    fill_double_kernel<<<256, 256, 0, st>>>(scores, n_prec, -1.0);
    fill_double_kernel<<<64, 256, 0, st>>>(recall, n_rec, -1.0);
    for (int i = 0; i < 3; ++i) count_launch();
    const unsigned long long* skeys = w.keys_a;
    const unsigned* sidx = w.vals_a;
    if (nd > 0) {
        map_pack_keys_kernel<<<(nd + 255) / 256, 256, 0, st>>>(det_cat, det_score, nd, w.keys_a, w.vals_a);
        count_launch();
        int key_bytes = 4;  // score
        for (long long kk = K - 1; kk > 0; kk >>= 8) key_bytes++;
        const int where = radix_sort_passes<unsigned long long, unsigned>(w.keys_a, w.vals_a, w.keys_b, w.vals_b, nd,
                                                                           1, key_bytes, w.sort_scratch, err_flag, st,
                                                                           &count_launch);
        if (where < 0) return check_cuda(cudaGetLastError(), "radix sort");
        skeys = where ? w.keys_b : w.keys_a;
        sidx = where ? w.vals_b : w.vals_a;
    }
    map_class_ranges_kernel<<<(K + 1 + 255) / 256, 256, 0, st>>>(skeys, nd, K, w.range_start);
    count_launch();
    if (class_hi <= class_lo) return check_cuda(cudaGetLastError(), "coco map launch");

    MapAccArgs aa;
    aa.sorted_idx = sidx;
    aa.range_start = w.range_start;
    aa.det_rank = det_rank;
    aa.det_match = det_match;
    aa.det_ignore = det_ignore;
    aa.det_score = det_score;
    aa.npig = npig;
    aa.rec_thr = rec_thr_dev;
    aa.K = K, aa.T = T, aa.R = R, aa.M = M;
    aa.class_lo = class_lo;
    for (int i = 0; i < M; ++i) aa.max_dets[i] = (int)max_dets_host[i];
    aa.n_det = nd;
    aa.tp_cum = w.tp_cum;
    aa.prec = w.prec;
    aa.cidx = w.cidx;
    aa.precision = precision;
    aa.recall = recall;
    aa.scores = scores;
    map_accumulate_kernel<<<dim3((unsigned)(class_hi - class_lo), (unsigned)(kMapAreas * M)), 256, 0, st>>>(aa);
    count_launch();
    return check_cuda(cudaGetLastError(), "coco map launch");
}

int check_map_sizes(int64_t n_iou_thr, int64_t n_max_dets, int64_t n_rec_thr) {
    MB200_REQUIRE(n_iou_thr >= 1 && n_iou_thr <= kMapMaxThr, "between 1 and %d IoU thresholds are supported (got %lld)",
                  kMapMaxThr, (long long)n_iou_thr);
    MB200_REQUIRE(n_max_dets >= 1 && n_max_dets <= 8, "between 1 and 8 max-detection thresholds are supported");
    MB200_REQUIRE(n_rec_thr >= 1, "need recall thresholds");
    return 0;
}

}  // namespace

extern "C" int mb200_coco_map_evaluate(
    const float* det_box_xywh, const float* det_score, const int64_t* det_label, const int32_t* det_off,
    const float* gt_box_xywh, const int64_t* gt_label, const uint8_t* gt_crowd, const double* gt_area,
    const int32_t* gt_off, int64_t n_img, int64_t n_det, int64_t n_gt, int64_t max_det_per_img, int64_t max_gt_per_img,
    const int64_t* classes, int64_t num_classes, int micro, const double* iou_thr_host, int64_t n_iou_thr,
    const double* rec_thr_dev, int64_t n_rec_thr, const int64_t* max_dets_host, int64_t n_max_dets, void* workspace,
    int64_t workspace_bytes, double* precision, double* recall, double* scores, uint32_t* err_flag, void* stream) {
    MB200_REQUIRE(n_img >= 1 && n_det >= 0 && n_gt >= 0, "bad sizes");
    MB200_REQUIRE(num_classes >= 1, "need at least one class");
    if (int rc = check_map_sizes(n_iou_thr, n_max_dets, n_rec_thr)) return rc;
    MB200_REQUIRE(n_det < (1ll << 31) && n_gt < (1ll << 31), "too many boxes");
    MB200_REQUIRE(workspace && precision && recall && scores && det_off && gt_off && classes && rec_thr_dev,
                  "NULL pointer");
    MB200_REQUIRE(workspace_bytes >= mb200_coco_map_workspace_bytes(n_det, num_classes, n_max_dets),
                  "workspace too small");
    const int K = micro ? 1 : (int)num_classes;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    MapWs w = carve(workspace, n_det, num_classes, n_max_dets, nullptr);
    const int M = (int)n_max_dets, T = (int)n_iou_thr, R = (int)n_rec_thr;
    zero_int_kernel<<<(K * kMapAreas + 255) / 256, 256, 0, st>>>(w.npig, K * kMapAreas);
    count_launch();
    if (int rc = map_match_impl(det_box_xywh, det_score, det_label, det_off, gt_box_xywh, gt_label, gt_crowd, gt_area, gt_off,
                                n_img, max_det_per_img, max_gt_per_img, classes, num_classes, micro, iou_thr_host, T,
                                (int)max_dets_host[n_max_dets - 1], w.det_cat, w.det_rank, w.det_match, w.det_ignore, w.npig,
                                err_flag, st))
        return rc;
    return map_accumulate_impl(w.det_cat, det_score, w.det_rank, w.det_match, w.det_ignore, (int)n_det, w.npig, K, 0, K, T,
                               rec_thr_dev, R, max_dets_host, M, w, precision, recall, scores, err_flag, st);
}

// The two phases on their own, for evaluation sharded over ranks (detection/mean_ap.py `_compute_distributed`): every rank
// MATCHES its own images, the per-detection records are exchanged, and every rank ACCUMULATES its own classes.
extern "C" int mb200_coco_map_match(
    const float* det_box_xywh, const float* det_score, const int64_t* det_label, const int32_t* det_off,
    const float* gt_box_xywh, const int64_t* gt_label, const uint8_t* gt_crowd, const double* gt_area,
    const int32_t* gt_off, int64_t n_img, int64_t max_det_per_img, int64_t max_gt_per_img, const int64_t* classes,
    int64_t num_classes, const double* iou_thr_host, int64_t n_iou_thr, int64_t max_det_last, int32_t* det_cat,
    int32_t* det_rank, uint64_t* det_match, uint64_t* det_ignore, int32_t* npig, uint32_t* err_flag, void* stream) {
    MB200_REQUIRE(n_img >= 0 && num_classes >= 1, "bad sizes");
    MB200_REQUIRE(n_iou_thr >= 1 && n_iou_thr <= kMapMaxThr, "between 1 and %d IoU thresholds are supported (got %lld)",
                  kMapMaxThr, (long long)n_iou_thr);
    MB200_REQUIRE(npig && classes && (n_img == 0 || (det_off && gt_off)), "NULL pointer");
    return map_match_impl(det_box_xywh, det_score, det_label, det_off, gt_box_xywh, gt_label, gt_crowd, gt_area, gt_off, n_img,
                          max_det_per_img, max_gt_per_img, classes, num_classes, 0, iou_thr_host, (int)n_iou_thr,
                          (int)max_det_last, det_cat, det_rank, reinterpret_cast<unsigned long long*>(det_match),
                          reinterpret_cast<unsigned long long*>(det_ignore), npig, err_flag,
                          reinterpret_cast<cudaStream_t>(stream));
}

// mb200_coco_map_match with the two extensions `iou_type="segm"` needs (reference detection/mean_ap.py:527-547, 917-944):
//  * instance masks: `pair_inter` (NULL = boxes) holds per image the [detections x ground truths] intersection pixel counts
//    (mb200_mask_pair_intersections), `pair_off` the table offsets, `det_mask_area` / `gt_mask_area` the pixel counts of the
//    masks; IoU and the detections' area ranges come from them (maskApi.c:rleIou), the boxes are ignored;
//  * `gt_area_exact`: `gt_area` already is the annotation's final "area" (the reference resolves "given, else mask area, else
//    w*h" on the host — with both IoU types it uses the MASK area for the box evaluation too), no w*h fallback here;
//  * `micro`: every label is class 0.
extern "C" int mb200_coco_map_match_ex(
    const float* det_box_xywh, const float* det_score, const int64_t* det_label, const int32_t* det_off,
    const float* gt_box_xywh, const int64_t* gt_label, const uint8_t* gt_crowd, const double* gt_area,
    const int32_t* gt_off, int64_t n_img, int64_t max_det_per_img, int64_t max_gt_per_img, const int64_t* classes,
    int64_t num_classes, int micro, const double* iou_thr_host, int64_t n_iou_thr, int64_t max_det_last,
    const double* pair_inter, const int64_t* pair_off, const double* det_mask_area, const double* gt_mask_area,
    int gt_area_exact, int32_t* det_cat, int32_t* det_rank, uint64_t* det_match, uint64_t* det_ignore, int32_t* npig,
    uint32_t* err_flag, void* stream) {
    MB200_REQUIRE(n_img >= 0 && num_classes >= 1, "bad sizes");
    MB200_REQUIRE(n_iou_thr >= 1 && n_iou_thr <= kMapMaxThr, "between 1 and %d IoU thresholds are supported (got %lld)",
                  kMapMaxThr, (long long)n_iou_thr);
    MB200_REQUIRE(npig && classes && (n_img == 0 || (det_off && gt_off)), "NULL pointer");
    MB200_REQUIRE(!pair_inter || (pair_off && det_mask_area && gt_mask_area), "mask mode needs table offsets and both areas");
    return map_match_impl(det_box_xywh, det_score, det_label, det_off, gt_box_xywh, gt_label, gt_crowd, gt_area, gt_off, n_img,
                          max_det_per_img, max_gt_per_img, classes, num_classes, micro, iou_thr_host, (int)n_iou_thr,
                          (int)max_det_last, det_cat, det_rank, reinterpret_cast<unsigned long long*>(det_match),
                          reinterpret_cast<unsigned long long*>(det_ignore), npig, err_flag,
                          reinterpret_cast<cudaStream_t>(stream), pair_inter, pair_off, det_mask_area, gt_mask_area, gt_area_exact);
}

extern "C" int mb200_coco_map_accumulate(
    const int32_t* det_cat, const float* det_score, const int32_t* det_rank, const uint64_t* det_match,
    const uint64_t* det_ignore, int64_t n_det, const int32_t* npig, int64_t num_classes, int64_t class_lo, int64_t class_hi,
    int64_t n_iou_thr, const double* rec_thr_dev, int64_t n_rec_thr, const int64_t* max_dets_host, int64_t n_max_dets,
    void* workspace, int64_t workspace_bytes, double* precision, double* recall, double* scores, uint32_t* err_flag,
    void* stream) {
    MB200_REQUIRE(n_det >= 0 && n_det < (1ll << 31) && num_classes >= 1, "bad sizes");
    MB200_REQUIRE(class_lo >= 0 && class_lo <= class_hi && class_hi <= num_classes, "bad class range [%lld, %lld)",
                  (long long)class_lo, (long long)class_hi);
    if (int rc = check_map_sizes(n_iou_thr, n_max_dets, n_rec_thr)) return rc;
    MB200_REQUIRE(workspace && precision && recall && scores && npig && rec_thr_dev, "NULL pointer");
    MB200_REQUIRE(workspace_bytes >= mb200_coco_map_workspace_bytes(n_det, num_classes, n_max_dets), "workspace too small");
    MapWs w = carve(workspace, n_det, num_classes, n_max_dets, nullptr);
    return map_accumulate_impl(det_cat, det_score, det_rank, reinterpret_cast<const unsigned long long*>(det_match),
                               reinterpret_cast<const unsigned long long*>(det_ignore), (int)n_det, npig, (int)num_classes,
                               (int)class_lo, (int)class_hi, (int)n_iou_thr, rec_thr_dev, (int)n_rec_thr, max_dets_host,
                               (int)n_max_dets, w, precision, recall, scores, err_flag,
                               reinterpret_cast<cudaStream_t>(stream));
}
