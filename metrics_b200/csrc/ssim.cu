// K20 — structural similarity (StructuralSimilarityIndexMeasure, MultiScaleStructuralSimilarityIndexMeasure and their
// functionals) on sm_90a: one read of preds and target per scale, the five windowed moments of a separable filter in
// shared memory, the reference's epilogue, and per-image float64 means in a fixed order.
//
// K21 — VisualInformationFidelity and UniversalImageQualityIndex on the same moment kernel with their own epilogues
// (functional/image/vif.py:45-83, functional/image/uqi.py:87-116), and the decimation between VIF scales.
//
// Reference op chain replaced (src/torchmetrics/functional/image/ssim.py):
//   :113-121   data range (Python max of two tensor ranges, a host synchronisation), tuple clamp, c1 / c2
//   :135-150   reflect padding of both inputs, gaussian / uniform kernel
//   :152-156   cat of preds, target, preds², target², preds·target into a 5·B batch and one grouped conv over it
//   :158-186   the element-wise epilogue, the contrast crop and the per-image means
//   :408-413   the average pool to the next MS-SSIM scale
//
// ssim_kernel: one CTA per output tile of TH x 32 positions of one (image, channel, output depth).  For every depth tap it
// stages the reflect-padded input tile of both tensors in shared memory (target rounded to the preds dtype, the tuple clamp
// applied, a per-tile shift subtracted), filters along w into five moment rows, then along h into registers, and adds
// the depth tap's weight times the result.  Variance and covariance do not change under a shift, so taking the moments
// about a value of the tile keeps float32 accurate where E[x²] − E[x]² about zero cancels.  The epilogue is the
// reference's (clamped variances, upper, lower, the map); each CTA writes its float64 sums of the map and of upper / lower
// over the crop to its own slot, and finalize_kernel adds an image's slots in slot order.
#include <algorithm>

#include "common.cuh"
#include "../../include/metrics_b200_image.h"

namespace mb200 {

extern void count_launch();

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kTW = 32;                  // output columns of a tile: one per lane
constexpr int kRangeBlocks = 1024;       // CTAs of the data-range pass: its partials have a fixed size
constexpr int kMaxSmem = 226 * 1024;     // dynamic shared memory of one CTA: sm_90's 227 KB less the static arrays

template <typename T>
struct Cvt;
template <>
struct Cvt<float> {
    using A = float;
    static constexpr bool kHalf = false;
    __device__ static float to_a(float v) { return v; }
    __device__ static float from_f(float v) { return v; }
    __device__ static float from_d(double v) { return (float)v; }
    __device__ static float from_a(float v) { return v; }
};
template <>
struct Cvt<double> {
    using A = double;
    static constexpr bool kHalf = false;
    __device__ static double to_a(double v) { return v; }
    __device__ static double from_f(float v) { return v; }
    __device__ static double from_d(double v) { return v; }
    __device__ static double from_a(double v) { return v; }
};
template <>
struct Cvt<__half> {
    using A = float;
    static constexpr bool kHalf = true;
    __device__ static float to_a(__half v) { return __half2float(v); }
    __device__ static __half from_f(float v) { return __float2half_rn(v); }
    __device__ static __half from_d(double v) { return __float2half_rn((float)v); }  // as torch: through float
    __device__ static __half from_a(float v) { return __float2half_rn(v); }
};
template <>
struct Cvt<__nv_bfloat16> {
    using A = float;
    static constexpr bool kHalf = true;
    __device__ static float to_a(__nv_bfloat16 v) { return __bfloat162float(v); }
    __device__ static __nv_bfloat16 from_f(float v) { return __float2bfloat16_rn(v); }
    __device__ static __nv_bfloat16 from_d(double v) { return __float2bfloat16_rn((float)v); }
    __device__ static __nv_bfloat16 from_a(float v) { return __float2bfloat16_rn(v); }
};

// element i of a float tensor with tag `dtype`, converted to T as `tensor.to(T)` converts it
template <typename T>
__device__ __forceinline__ T load_as(const void* p, int dtype, long long i) {
    switch (dtype) {
        case MB200_F32: return Cvt<T>::from_f(reinterpret_cast<const float*>(p)[i]);
        case MB200_F64: return Cvt<T>::from_d(reinterpret_cast<const double*>(p)[i]);
        case MB200_F16: return Cvt<T>::from_f(__half2float(reinterpret_cast<const __half*>(p)[i]));
        default: return Cvt<T>::from_f(__bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p)[i]));
    }
}

struct Vol {
    const void* p;
    int dtype;
    long long sn, sc, sd, sh, sw;
};

struct Geo {
    long long b, c, d, h, w;
    int kd, kh, kw, pd, ph, pw;
    long long od, oh, ow;
    int crop_depth;
    long long tiles_h, tiles_w;
};

struct Clamp {
    int on;
    double lo, hi;
};

__host__ __device__ long long cdiv(long long a, long long b) { return (a + b - 1) / b; }

// reflect-pad index (pad < n); positions past the output of a partial tile are clamped into the image, their values unused
__device__ __forceinline__ long long reflect(long long i, long long n) {
    if (i < 0) i = -i;
    if (i >= n) i = 2 * (n - 1) - i;
    return i < 0 ? 0 : (i >= n ? n - 1 : i);
}

// one input value as the reference sees it after _ssim_check_inputs and the tuple clamp: in T, then in A
template <typename T>
__device__ __forceinline__ typename Cvt<T>::A load_px(const Vol& v, long long off, const Clamp& cl) {
    using A = typename Cvt<T>::A;
    A a = Cvt<T>::to_a(load_as<T>(v.p, v.dtype, off));
    if (cl.on && !isnan(a)) {
        a = a < (A)cl.lo ? (A)cl.lo : a;  // torch.clamp: min(max(v, lo), hi) in the op math type, NaN kept
        a = a > (A)cl.hi ? (A)cl.hi : a;
        if (Cvt<T>::kHalf) a = Cvt<T>::to_a(Cvt<T>::from_a(a));
    }
    return a;
}

template <typename A>
__host__ __device__ constexpr int weights_slots(int taps) {
    return (taps + 1) & ~1;  // keeps the tiles after the weights 16-byte aligned for double
}

template <typename T, int TH>
__host__ __device__ long long tile_smem(int kd, int kh, int kw) {
    using A = typename Cvt<T>::A;
    const long long ih = TH + kh - 1, iw = kTW + kw - 1;
    return (long long)sizeof(A) * (weights_slots<A>(kd + kh + kw) + 2 * ih * iw + 5 * ih * kTW);
}

template <typename T>
struct Tile {
    static constexpr int kH = sizeof(typename Cvt<T>::A) == 8 ? 16 : 32;  // output rows of a tile
};

__device__ __forceinline__ double warp_sum(double v) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
    return v;
}

// ---- epilogues: what ssim_kernel makes of the moments of one output position ---------------------------------------
// begin() runs once per CTA on its own copy; operator() takes the means, the clamped variances and the covariance of
// one position and returns the map value and two float64 addends for the CTA's sums.
template <typename A>
struct EpiOut {
    A map;
    double s0, s1;
};

// SSIM: the map into s0; upper / lower inside the crop [pad : o − pad] of every axis (and depth when crop_depth) into s1
template <typename A>
struct SsimEpilogue {
    const double* consts;  // device [MB200_SSIM_CONSTS] of the data-range pass, or NULL for c1_arg / c2_arg
    double c1_arg, c2_arg;
    A c1, c2;
    bool depth_in_crop;

    __device__ __forceinline__ void begin(const Geo& g, long long od) {
        if (consts) {
            c1 = (A)consts[MB200_SSIM_C1];
            c2 = (A)consts[MB200_SSIM_C2];
        } else {
            c1 = (A)c1_arg;
            c2 = (A)c2_arg;
        }
        depth_in_crop = !g.crop_depth || (g.pd > 0 && od >= g.pd && od < g.od - g.pd);
    }
    __device__ __forceinline__ EpiOut<A> operator()(A mux, A muy, A vx, A vy, A cxy, const Geo& g, long long oh,
                                                    long long ow) const {
        const A upper = (A)2 * cxy + c2;
        const A lower = (vx + vy) + c2;
        const A s = (((A)2 * (mux * muy) + c1) * upper) / ((mux * mux + muy * muy + c1) * lower);
        const bool in_crop =
            depth_in_crop && g.ph > 0 && g.pw > 0 && oh >= g.ph && oh < g.oh - g.ph && ow >= g.pw && ow < g.ow - g.pw;
        return {s, (double)s, in_crop ? (double)(upper / lower) : 0.0};
    }
};

// UQI (functional/image/uqi.py:101-114): SSIM with c1 = c2 = 0 and the dtype's eps in the denominator; the map inside
// the crop [crop_h : o_h − crop_h] x [crop_w : o_w − crop_w] into s0 (a zero margin is an empty crop, as x[0:-0])
template <typename A>
struct UqiEpilogue {
    double eps;
    int crop_h, crop_w;

    __device__ __forceinline__ void begin(const Geo&, long long) {}
    __device__ __forceinline__ EpiOut<A> operator()(A mux, A muy, A vx, A vy, A cxy, const Geo& g, long long oh,
                                                    long long ow) const {
        const A s = (((A)2 * (mux * muy)) * ((A)2 * cxy)) / ((mux * mux + muy * muy) * (vx + vy) + (A)eps);
        const bool in_crop = crop_h > 0 && crop_w > 0 && oh >= crop_h && oh < g.oh - crop_h && ow >= crop_w &&
                             ow < g.ow - crop_w;
        return {s, in_crop ? (double)s : 0.0, 0.0};
    }
};

// VIF-P, one scale (functional/image/vif.py:63-82): x is preds, y is target.  The reference's masks in its order, then
// log10(1 + g²σt / (σv + σn²)) into s0 and log10(1 + σt / σn²) into s1.  No map.
template <typename A>
struct VifEpilogue {
    double eps, sigma_n_sq;  // rounded to the input dtype by the caller, as torch.tensor(..., dtype=dtype) rounds them

    __device__ __forceinline__ void begin(const Geo&, long long) {}
    __device__ __forceinline__ EpiOut<A> operator()(A, A, A vx, A vy, A cxy, const Geo&, long long, long long) const {
        const A e = (A)eps, sn = (A)sigma_n_sq;
        A st = vy;
        A gain = cxy / (st + e);
        A sv = vx - gain * cxy;
        if (st < e) {
            gain = 0;
            sv = vx;
            st = 0;
        }
        if (vx < e) {
            gain = 0;
            sv = 0;
        }
        if (gain < (A)0) {
            sv = vx;
            gain = 0;
        }
        sv = sv < e ? e : sv;  // torch.clamp(min=eps): NaN stays NaN
        return {(A)0, (double)log10((A)1 + gain * gain * st / (sv + sn)), (double)log10((A)1 + st / sn)};
    }
};

// grid: one CTA per (image, channel, output depth, tile row, tile column), in that order, slowest first.  A CTA's slot
// holds its two epilogue sums, so the slots of one image, and of one (image, channel), are consecutive.
// Two CTAs per SM, as K20 has always run: without the bound, ptxas holds some epilogue instantiations to 80 registers
// and spills.
template <typename T, int TH, class Epi>
__global__ void __launch_bounds__(kThreads, 2) ssim_kernel(Vol P, Vol Q, Geo g, const T* __restrict__ weights, Clamp cl,
                                                        Epi epi, T* __restrict__ map, double2* __restrict__ partials) {
    using A = typename Cvt<T>::A;
    constexpr int RPT = TH / kWarps;  // output rows per thread
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ A shift[2];
    __shared__ double red[2][kWarps];
    const int kd = g.kd, kh = g.kh, kw = g.kw;
    const int IH = TH + kh - 1, IW = kTW + kw - 1;
    A* wD = reinterpret_cast<A*>(smem_raw);
    A* wH = wD + kd;
    A* wW = wH + kh;
    A* inx = wD + weights_slots<A>(kd + kh + kw);
    A* iny = inx + IH * IW;
    A* hb = iny + IH * IW;  // five moment planes of IH x kTW

    long long t = blockIdx.x;
    const long long tw = t % g.tiles_w;
    t /= g.tiles_w;
    const long long th = t % g.tiles_h;
    t /= g.tiles_h;
    const long long od = t % g.od;
    t /= g.od;
    const long long ch = t % g.c, bi = t / g.c;
    const long long oh0 = th * TH, ow0 = tw * kTW;
    const int tid = threadIdx.x, lane = tid & 31, rg = tid >> 5;
    const long long baseP = bi * P.sn + ch * P.sc, baseQ = bi * Q.sn + ch * Q.sc;

    for (int i = tid; i < kd + kh + kw; i += kThreads) wD[i] = Cvt<T>::to_a(weights[i]);
    __syncthreads();
    if (tid < 3) {
        // each axis's taps divided by their float64 sum: moments about a shift equal the reference's only for a filter
        // of weight 1, and a float16 / bfloat16 gaussian sums to 1 within about 1e-3 only
        A* w = tid == 0 ? wD : (tid == 1 ? wH : wW);
        const int k = tid == 0 ? kd : (tid == 1 ? kh : kw);
        double sum = 0.0;
        for (int i = 0; i < k; ++i) sum += (double)w[i];
        for (int i = 0; i < k; ++i) w[i] = (A)((double)w[i] / sum);
    }
    // the shift: each input's value at the tile's centre.  A non-finite shift would spread to every window of the tile,
    // so when the centre is not finite the shift is the first finite value of the tile's input rows in that depth plane
    // (lowest index, so the choice does not depend on thread timing), and 0 only when the plane has none.
    __shared__ int need, first[2];
    const long long dc = min(od, g.d - 1);
    if (tid == 0) {
        const long long hc = min(oh0 + TH / 2, g.h - 1), wc = min(ow0 + kTW / 2, g.w - 1);
        const A sx = load_px<T>(P, baseP + dc * P.sd + hc * P.sh + wc * P.sw, cl);
        const A sy = load_px<T>(Q, baseQ + dc * Q.sd + hc * Q.sh + wc * Q.sw, cl);
        shift[0] = isfinite(sx) ? sx : (A)0;
        shift[1] = isfinite(sy) ? sy : (A)0;
        need = (isfinite(sx) ? 0 : 1) | (isfinite(sy) ? 0 : 2);
        first[0] = first[1] = INT_MAX;
    }
    __syncthreads();
    if (need) {
        for (int i = tid; i < IH * IW; i += kThreads) {
            const int r = i / IW, c = i - r * IW;
            const long long o = reflect(oh0 + r - g.ph, g.h), q = reflect(ow0 + c - g.pw, g.w);
            if ((need & 1) && isfinite(load_px<T>(P, baseP + dc * P.sd + o * P.sh + q * P.sw, cl))) atomicMin(&first[0], i);
            if ((need & 2) && isfinite(load_px<T>(Q, baseQ + dc * Q.sd + o * Q.sh + q * Q.sw, cl))) atomicMin(&first[1], i);
        }
        __syncthreads();
        if (tid == 0) {
            for (int k = 0; k < 2; ++k) {
                if (!((need >> k) & 1) || first[k] == INT_MAX) continue;
                const Vol& v = k == 0 ? P : Q;
                const int r = first[k] / IW, c = first[k] - r * IW;
                const long long o = reflect(oh0 + r - g.ph, g.h), q = reflect(ow0 + c - g.pw, g.w);
                shift[k] = load_px<T>(v, (k == 0 ? baseP : baseQ) + dc * v.sd + o * v.sh + q * v.sw, cl);
            }
        }
    }
    A acc[5][RPT];
#pragma unroll
    for (int m = 0; m < 5; ++m)
#pragma unroll
        for (int j = 0; j < RPT; ++j) acc[m][j] = 0;

    for (int td = 0; td < kd; ++td) {
        const long long di = reflect(od + td - g.pd, g.d);
        __syncthreads();  // weights and shift written; the previous depth tap is done with the tiles
        const A sx = shift[0], sy = shift[1];
        const long long offP = baseP + di * P.sd, offQ = baseQ + di * Q.sd;
        for (int i = tid; i < IH * IW; i += kThreads) {
            const int r = i / IW, c = i - r * IW;
            const long long hi = reflect(oh0 + r - g.ph, g.h), wi = reflect(ow0 + c - g.pw, g.w);
            inx[i] = load_px<T>(P, offP + hi * P.sh + wi * P.sw, cl) - sx;
            iny[i] = load_px<T>(Q, offQ + hi * Q.sh + wi * Q.sw, cl) - sy;
        }
        __syncthreads();
        // along w: row r, column lane of the tile -> the five moments of the kw taps
        for (int i = tid; i < IH * kTW; i += kThreads) {
            const int r = i / kTW, c = i - r * kTW;
            const A* xr = inx + r * IW + c;
            const A* yr = iny + r * IW + c;
            A s0 = 0, s1 = 0, s2 = 0, s3 = 0, s4 = 0;
            for (int k = 0; k < kw; ++k) {
                const A wk = wW[k], x = xr[k], y = yr[k];
                const A wx = wk * x, wy = wk * y;
                s0 += wx;
                s1 += wy;
                s2 += wx * x;
                s3 += wy * y;
                s4 += wx * y;
            }
            const int plane = IH * kTW;
            hb[i] = s0;
            hb[plane + i] = s1;
            hb[2 * plane + i] = s2;
            hb[3 * plane + i] = s3;
            hb[4 * plane + i] = s4;
        }
        __syncthreads();
        // along h: RPT consecutive output rows of column lane share every moment row they read
        A v[5][RPT];
#pragma unroll
        for (int m = 0; m < 5; ++m)
#pragma unroll
            for (int j = 0; j < RPT; ++j) v[m][j] = 0;
        const int plane = IH * kTW;
        for (int i = 0; i < kh + RPT - 1; ++i) {
            const int idx = (rg * RPT + i) * kTW + lane;
            A mv[5];
#pragma unroll
            for (int m = 0; m < 5; ++m) mv[m] = hb[m * plane + idx];
#pragma unroll
            for (int j = 0; j < RPT; ++j) {
                const int k = i - j;
                if (k >= 0 && k < kh) {
                    const A wk = wH[k];
#pragma unroll
                    for (int m = 0; m < 5; ++m) v[m][j] += wk * mv[m];
                }
            }
        }
        const A wd = wD[td];
#pragma unroll
        for (int m = 0; m < 5; ++m)
#pragma unroll
            for (int j = 0; j < RPT; ++j) acc[m][j] += wd * v[m][j];
    }

    Epi e = epi;
    e.begin(g, od);
    const A sx = shift[0], sy = shift[1];
    double ssum = 0.0, csum = 0.0;
    const long long ow = ow0 + lane;
#pragma unroll
    for (int j = 0; j < RPT; ++j) {
        const long long oh = oh0 + rg * RPT + j;
        if (oh < g.oh && ow < g.ow) {
            const A mx = acc[0][j], my = acc[1][j];
            A vx = acc[2][j] - mx * mx;
            A vy = acc[3][j] - my * my;
            vx = vx < (A)0 ? (A)0 : vx;  // torch.clamp(min=0): NaN stays NaN
            vy = vy < (A)0 ? (A)0 : vy;
            const EpiOut<A> r = e(mx + sx, my + sy, vx, vy, acc[4][j] - mx * my, g, oh, ow);
            ssum += r.s0;
            csum += r.s1;
            if (map) map[(((bi * g.c + ch) * g.od + od) * g.oh + oh) * g.ow + ow] = Cvt<T>::from_a(r.map);
        }
    }
    ssum = warp_sum(ssum);
    csum = warp_sum(csum);
    if (lane == 0) {
        red[0][rg] = ssum;
        red[1][rg] = csum;
    }
    __syncthreads();
    if (tid == 0) {
        double a = 0.0, b = 0.0;
        for (int k = 0; k < kWarps; ++k) {
            a += red[0][k];
            b += red[1][k];
        }
        partials[blockIdx.x] = make_double2(a, b);
    }
}

// one CTA per image: its slots in slot order, then the two means
__global__ void __launch_bounds__(kThreads) finalize_kernel(const double2* __restrict__ partials, long long per_image,
                                                            double count, double crop_count, double* __restrict__ sim,
                                                            double* __restrict__ cs) {
    __shared__ double red[2][kWarps];
    const double2* p = partials + blockIdx.x * per_image;
    double a = 0.0, b = 0.0;
    for (long long i = threadIdx.x; i < per_image; i += kThreads) {
        a += p[i].x;
        b += p[i].y;
    }
    a = warp_sum(a);
    b = warp_sum(b);
    if ((threadIdx.x & 31) == 0) {
        red[0][threadIdx.x >> 5] = a;
        red[1][threadIdx.x >> 5] = b;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        a = b = 0.0;
        for (int k = 0; k < kWarps; ++k) {
            a += red[0][k];
            b += red[1][k];
        }
        sim[blockIdx.x] = a / count;
        if (cs) cs[blockIdx.x] = b / crop_count;  // an empty crop is 0 / 0: NaN, as the mean of an empty tensor
    }
}

// ---- data range -------------------------------------------------------------------------------------------------------
template <typename A>
__device__ __forceinline__ A nan_max(A a, A b) { return isnan(a) ? a : (isnan(b) ? b : (b > a ? b : a)); }
template <typename A>
__device__ __forceinline__ A nan_min(A a, A b) { return isnan(a) ? a : (isnan(b) ? b : (b < a ? b : a)); }

template <typename A>
__device__ void block_minmax(A (&v)[4], A (*red)[kWarps]) {
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const A u = __shfl_xor_sync(kFull, v[k], o);
            v[k] = (k & 1) ? nan_max(v[k], u) : nan_min(v[k], u);
        }
    }
    if ((threadIdx.x & 31) == 0)
        for (int k = 0; k < 4; ++k) red[k][threadIdx.x >> 5] = v[k];
    __syncthreads();
    if (threadIdx.x == 0)
        for (int w = 1; w < kWarps; ++w)
            for (int k = 0; k < 4; ++k) v[k] = (k & 1) ? nan_max(v[k], red[k][w]) : nan_min(v[k], red[k][w]);
}

// partial[blk] = (pmin, pmax, tmin, tmax) over rows blk, blk + grid, ...; a row is one (n, c, d, h) line along w
template <typename T>
__global__ void __launch_bounds__(kThreads) range_kernel(Vol P, Vol Q, Geo g, typename Cvt<T>::A* __restrict__ partial) {
    using A = typename Cvt<T>::A;
    __shared__ A red[4][kWarps];
    A v[4] = {INFINITY, -INFINITY, INFINITY, -INFINITY};
    const Clamp none{0, 0.0, 0.0};
    const long long rows = g.b * g.c * g.d * g.h;
    for (long long r = blockIdx.x; r < rows; r += gridDim.x) {
        long long q = r;
        const long long hi = q % g.h;
        q /= g.h;
        const long long di = q % g.d;
        q /= g.d;
        const long long ci = q % g.c, bi = q / g.c;
        const long long oP = bi * P.sn + ci * P.sc + di * P.sd + hi * P.sh;
        const long long oQ = bi * Q.sn + ci * Q.sc + di * Q.sd + hi * Q.sh;
        for (long long wi = threadIdx.x; wi < g.w; wi += kThreads) {
            const A x = load_px<T>(P, oP + wi * P.sw, none), y = load_px<T>(Q, oQ + wi * Q.sw, none);
            v[0] = nan_min(v[0], x);
            v[1] = nan_max(v[1], x);
            v[2] = nan_min(v[2], y);
            v[3] = nan_max(v[3], y);
        }
    }
    block_minmax<A>(v, red);
    if (threadIdx.x == 0)
        for (int k = 0; k < 4; ++k) partial[blockIdx.x * 4 + k] = v[k];
}

template <typename T>
__global__ void __launch_bounds__(kThreads) range_final_kernel(const typename Cvt<T>::A* __restrict__ partial, int blocks,
                                                               double k1, double k2, double* __restrict__ consts) {
    using A = typename Cvt<T>::A;
    __shared__ A red[4][kWarps];
    A v[4] = {INFINITY, -INFINITY, INFINITY, -INFINITY};
    for (int i = threadIdx.x; i < blocks; i += kThreads)
        for (int k = 0; k < 4; ++k) v[k] = (k & 1) ? nan_max(v[k], partial[i * 4 + k]) : nan_min(v[k], partial[i * 4 + k]);
    block_minmax<A>(v, red);
    if (threadIdx.x == 0) {
        // preds.max() - preds.min() in the preds dtype; Python's max(a, b) keeps a unless b > a
        const A pr = Cvt<T>::to_a(Cvt<T>::from_a(v[1] - v[0]));
        const A tr = Cvt<T>::to_a(Cvt<T>::from_a(v[3] - v[2]));
        const A r = tr > pr ? tr : pr;
        const A a = (A)k1 * r, b = (A)k2 * r;
        consts[MB200_SSIM_RANGE] = (double)r;
        consts[MB200_SSIM_C1] = (double)(a * a);
        consts[MB200_SSIM_C2] = (double)(b * b);
    }
}

// ---- average pool to the next scale -----------------------------------------------------------------------------------
// as ATen's avg_pool2d / avg_pool3d: the window summed along d, h, w in the accumulation type, divided by its size
template <typename T>
__global__ void __launch_bounds__(kThreads) pool_kernel(Vol P, Vol Q, Geo g, int pool_depth, T* __restrict__ po,
                                                        T* __restrict__ qo) {
    using A = typename Cvt<T>::A;
    const long long od = pool_depth ? g.d / 2 : g.d, oh = g.h / 2, ow = g.w / 2;
    const long long n = g.b * g.c * od * oh * ow;
    const Clamp none{0, 0.0, 0.0};
    const int fd = pool_depth ? 2 : 1;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads) {
        long long q = i;
        const long long x = q % ow;
        q /= ow;
        const long long y = q % oh;
        q /= oh;
        const long long z = q % od;
        q /= od;
        const long long ci = q % g.c, bi = q / g.c;
        A sp = 0, sq = 0;
        for (int a = 0; a < fd; ++a)
            for (int b = 0; b < 2; ++b)
                for (int c = 0; c < 2; ++c) {
                    const long long dz = z * fd + a, hy = 2 * y + b, wx = 2 * x + c;
                    sp += load_px<T>(P, bi * P.sn + ci * P.sc + dz * P.sd + hy * P.sh + wx * P.sw, none);
                    sq += load_px<T>(Q, bi * Q.sn + ci * Q.sc + dz * Q.sd + hy * Q.sh + wx * Q.sw, none);
                }
        po[i] = Cvt<T>::from_a(sp / (A)(4 * fd));
        qo[i] = Cvt<T>::from_a(sq / (A)(4 * fd));
    }
}

// ---- VIF decimation between scales --------------------------------------------------------------------------------------
// conv2d(x, k)[..., ::2, ::2] of both inputs (functional/image/vif.py:49-51): the valid separable filter evaluated at even
// output positions only, per depth plane, in the accumulation type, rounded to the preds dtype.  No shift: filtering is
// linear, so nothing cancels.  Each axis's taps are divided by their float64 sum, as in ssim_kernel.
template <typename T>
__global__ void __launch_bounds__(kThreads) decimate_kernel(Vol P, Vol Q, Geo g, const T* __restrict__ weights,
                                                            T* __restrict__ po, T* __restrict__ qo) {
    using A = typename Cvt<T>::A;
    __shared__ A wt[2 * MB200_SSIM_MAX_TAPS];
    const int kh = g.kh, kw = g.kw;
    A* wH = wt;
    A* wW = wt + kh;
    for (int i = threadIdx.x; i < kh + kw; i += kThreads) wt[i] = Cvt<T>::to_a(weights[i]);
    __syncthreads();
    if (threadIdx.x < 2) {
        A* w = threadIdx.x == 0 ? wH : wW;
        const int k = threadIdx.x == 0 ? kh : kw;
        double sum = 0.0;
        for (int i = 0; i < k; ++i) sum += (double)w[i];
        for (int i = 0; i < k; ++i) w[i] = (A)((double)w[i] / sum);
    }
    __syncthreads();
    const Clamp none{0, 0.0, 0.0};
    const long long n = g.b * g.c * g.d * g.oh * g.ow;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads) {
        long long q = i;
        const long long x = q % g.ow;
        q /= g.ow;
        const long long y = q % g.oh;
        q /= g.oh;
        const long long z = q % g.d;
        q /= g.d;
        const long long ci = q % g.c, bi = q / g.c;
        const long long oP = bi * P.sn + ci * P.sc + z * P.sd + 2 * y * P.sh + 2 * x * P.sw;
        const long long oQ = bi * Q.sn + ci * Q.sc + z * Q.sd + 2 * y * Q.sh + 2 * x * Q.sw;
        A sp = 0, sq = 0;
        for (int a = 0; a < kh; ++a) {
            A rp = 0, rq = 0;
            for (int c = 0; c < kw; ++c) {
                rp += wW[c] * load_px<T>(P, oP + a * P.sh + c * P.sw, none);
                rq += wW[c] * load_px<T>(Q, oQ + a * Q.sh + c * Q.sw, none);
            }
            sp += wH[a] * rp;
            sq += wH[a] * rq;
        }
        po[i] = Cvt<T>::from_a(sp);
        qo[i] = Cvt<T>::from_a(sq);
    }
}

// ---- host side ----------------------------------------------------------------------------------------------------------
struct Layout {
    long long od, oh, ow, tiles_h, tiles_w, tiles, smem;
};

// -1 in smem when the geometry is invalid or the tile does not fit in shared memory
template <typename T>
Layout layout(long long b, long long c, long long d, long long h, long long w, int kd, int kh, int kw, int pd, int ph,
              int pw) {
    constexpr int TH = Tile<T>::kH;
    Layout L{0, 0, 0, 0, 0, 0, -1};
    if (b < 0 || c < 1 || d < 1 || h < 1 || w < 1) return L;
    if (kd < 1 || kh < 1 || kw < 1 || kd > MB200_SSIM_MAX_TAPS || kh > MB200_SSIM_MAX_TAPS || kw > MB200_SSIM_MAX_TAPS) return L;
    if (pd < 0 || ph < 0 || pw < 0 || pd >= d || ph >= h || pw >= w) return L;
    L.od = d + 2ll * pd - kd + 1;
    L.oh = h + 2ll * ph - kh + 1;
    L.ow = w + 2ll * pw - kw + 1;
    if (L.od < 1 || L.oh < 1 || L.ow < 1) return L;
    L.tiles_h = cdiv(L.oh, TH);
    L.tiles_w = cdiv(L.ow, kTW);
    L.tiles = b * c * L.od * L.tiles_h * L.tiles_w;
    const long long smem = tile_smem<T, TH>(kd, kh, kw);
    if (smem > kMaxSmem || L.tiles >= (1ll << 31)) return L;
    L.smem = smem;
    return L;
}

long long align16(long long v) { return (v + 15) / 16 * 16; }

Geo geo(const Layout& L, long long b, long long c, long long d, long long h, long long w, int kd, int kh, int kw, int pd,
        int ph, int pw, int crop_depth) {
    return Geo{b, c, d, h, w, kd, kh, kw, pd, ph, pw, L.od, L.oh, L.ow, crop_depth ? 1 : 0, L.tiles_h, L.tiles_w};
}

// the moment pass with epilogue `epi`, then one finalize CTA per group of consecutive slots (an image, or an (image,
// channel)): s0[group] = its first sums / count, s1[group] = its second sums / count1 (s1 NULL: not written)
template <typename T, class Epi>
int moments(const Vol& P, const Vol& Q, const Layout& L, const Geo& g, const void* weights, const Clamp& cl, const Epi& epi,
            void* map, void* scratch, long long groups, double count, double count1, double* s0, double* s1,
            cudaStream_t st) {
    constexpr int TH = Tile<T>::kH;
    double2* partials = reinterpret_cast<double2*>(scratch);
    MB200_CUDA_OK(ensure_dynamic_smem(ssim_kernel<T, TH, Epi>, kMaxSmem));
    ssim_kernel<T, TH, Epi><<<(unsigned)L.tiles, kThreads, (size_t)L.smem, st>>>(
        P, Q, g, reinterpret_cast<const T*>(weights), cl, epi, reinterpret_cast<T*>(map), partials);
    count_launch();
    finalize_kernel<<<(unsigned)groups, kThreads, 0, st>>>(partials, L.tiles / groups, count, count1, s0, s1);
    count_launch();
    MB200_CUDA_OK(cudaGetLastError());
    return 0;
}

long long scratch_for(const Layout& L) { return align16(L.tiles * (long long)sizeof(double2)) + kRangeBlocks * 4 * 8; }

int range_blocks(long long rows) { return (int)std::min<long long>(rows, kRangeBlocks); }

}  // namespace
}  // namespace mb200

using namespace mb200;

// =====================================================================================================
// C-ABI
// =====================================================================================================
extern "C" int64_t mb200_ssim_scratch_bytes(int preds_dtype, int64_t b, int64_t c, int64_t d, int64_t h, int64_t w,
                                            int taps_d, int taps_h, int taps_w, int pad_d, int pad_h, int pad_w) {
    // not through with_float_type, which returns int: the size passes 2^31 bytes from 2^27 tiles on
    Layout L{};
    L.smem = -1;
    switch (preds_dtype) {
        case MB200_F32: L = layout<float>(b, c, d, h, w, taps_d, taps_h, taps_w, pad_d, pad_h, pad_w); break;
        case MB200_F16: L = layout<__half>(b, c, d, h, w, taps_d, taps_h, taps_w, pad_d, pad_h, pad_w); break;
        case MB200_BF16: L = layout<__nv_bfloat16>(b, c, d, h, w, taps_d, taps_h, taps_w, pad_d, pad_h, pad_w); break;
        case MB200_F64: L = layout<double>(b, c, d, h, w, taps_d, taps_h, taps_w, pad_d, pad_h, pad_w); break;
        default: break;
    }
    return L.smem < 0 ? -1 : scratch_for(L);
}

#define MB200_SSIM_CHECK_TAGS()                                                                                      \
    MB200_REQUIRE(is_float_tag(preds_dtype), "preds must be a floating-point tensor (dtype tag %d)", preds_dtype);  \
    MB200_REQUIRE(is_float_tag(target_dtype), "target must be a floating-point tensor (dtype tag %d)", target_dtype)

extern "C" int mb200_ssim_data_range(const void* preds, int preds_dtype, const void* target, int target_dtype, int64_t b,
                                     int64_t c, int64_t d, int64_t h, int64_t w, int64_t preds_s_n, int64_t preds_s_c,
                                     int64_t preds_s_d, int64_t preds_s_h, int64_t preds_s_w, int64_t target_s_n,
                                     int64_t target_s_c, int64_t target_s_d, int64_t target_s_h, int64_t target_s_w,
                                     double k1, double k2, double* consts, void* scratch, int64_t scratch_bytes,
                                     void* stream) {
    MB200_SSIM_CHECK_TAGS();
    MB200_REQUIRE(b >= 1 && c >= 1 && d >= 1 && h >= 1 && w >= 1, "the data range of an empty tensor is undefined");
    MB200_REQUIRE(preds && target && consts && scratch, "NULL pointer");
    MB200_REQUIRE(scratch_bytes >= (int64_t)kRangeBlocks * 4 * 8 && (reinterpret_cast<uintptr_t>(scratch) & 15) == 0,
                  "scratch must be 16-byte aligned and hold %d bytes", kRangeBlocks * 4 * 8);
    const Vol P{preds, preds_dtype, preds_s_n, preds_s_c, preds_s_d, preds_s_h, preds_s_w};
    const Vol Q{target, target_dtype, target_s_n, target_s_c, target_s_d, target_s_h, target_s_w};
    Geo g{};
    g.b = b, g.c = c, g.d = d, g.h = h, g.w = w;
    const int blocks = range_blocks(b * c * d * h);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    return with_float_type(preds_dtype, [&](auto tag) -> int {
        using T = typename decltype(tag)::type;
        using A = typename Cvt<T>::A;
        A* part = reinterpret_cast<A*>(scratch);
        range_kernel<T><<<blocks, kThreads, 0, st>>>(P, Q, g, part);
        count_launch();
        range_final_kernel<T><<<1, kThreads, 0, st>>>(part, blocks, k1, k2, consts);
        count_launch();
        MB200_CUDA_OK(cudaGetLastError());
        return 0;
    });
}

extern "C" int mb200_ssim_update(const void* preds, int preds_dtype, const void* target, int target_dtype, int64_t b,
                                 int64_t c, int64_t d, int64_t h, int64_t w, int64_t preds_s_n, int64_t preds_s_c,
                                 int64_t preds_s_d, int64_t preds_s_h, int64_t preds_s_w, int64_t target_s_n,
                                 int64_t target_s_c, int64_t target_s_d, int64_t target_s_h, int64_t target_s_w, int taps_d,
                                 int taps_h, int taps_w, int pad_d, int pad_h, int pad_w, int crop_depth,
                                 const void* weights, int clamp, double clamp_lo, double clamp_hi, const double* consts,
                                 double c1, double c2, double* sim, double* cs, void* map, void* scratch,
                                 int64_t scratch_bytes, void* stream) {
    MB200_SSIM_CHECK_TAGS();
    MB200_REQUIRE(b >= 0 && c >= 1 && d >= 1 && h >= 1 && w >= 1, "bad sizes");
    MB200_REQUIRE(taps_d >= 1 && taps_h >= 1 && taps_w >= 1 && taps_d <= MB200_SSIM_MAX_TAPS && taps_h <= MB200_SSIM_MAX_TAPS &&
                      taps_w <= MB200_SSIM_MAX_TAPS,
                  "tap counts must lie in [1, %d], got %d, %d, %d", MB200_SSIM_MAX_TAPS, taps_d, taps_h, taps_w);
    MB200_REQUIRE(pad_d >= 0 && pad_h >= 0 && pad_w >= 0 && pad_d < d && pad_h < h && pad_w < w,
                  "reflect pads (%d, %d, %d) must be non-negative and below the sizes", pad_d, pad_h, pad_w);
    const int64_t need = mb200_ssim_scratch_bytes(preds_dtype, b, c, d, h, w, taps_d, taps_h, taps_w, pad_d, pad_h, pad_w);
    MB200_REQUIRE(need >= 0,
                  "the filter (%d, %d, %d taps) gives an empty output or does not fit in shared memory, or the batch has "
                  "2^31 tiles or more", taps_d, taps_h, taps_w);
    MB200_REQUIRE(preds && target && weights && sim && scratch, "NULL pointer");
    MB200_REQUIRE(scratch_bytes >= need && (reinterpret_cast<uintptr_t>(scratch) & 15) == 0,
                  "scratch must be 16-byte aligned and mb200_ssim_scratch_bytes(...) bytes");
    if (b == 0) return 0;
    const Vol P{preds, preds_dtype, preds_s_n, preds_s_c, preds_s_d, preds_s_h, preds_s_w};
    const Vol Q{target, target_dtype, target_s_n, target_s_c, target_s_d, target_s_h, target_s_w};
    const Clamp cl{clamp ? 1 : 0, clamp_lo, clamp_hi};
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    return with_float_type(preds_dtype, [&](auto tag) -> int {
        using T = typename decltype(tag)::type;
        using A = typename Cvt<T>::A;
        const Layout L = layout<T>(b, c, d, h, w, taps_d, taps_h, taps_w, pad_d, pad_h, pad_w);
        auto crop = [](long long o, int p) -> long long { return p > 0 ? std::max(0ll, o - 2ll * p) : 0ll; };
        const double crop_count = (double)c * (crop_depth ? crop(L.od, pad_d) : L.od) * crop(L.oh, pad_h) * crop(L.ow, pad_w);
        const SsimEpilogue<A> epi{consts, c1, c2, (A)0, (A)0, false};
        return moments<T>(P, Q, L, geo(L, b, c, d, h, w, taps_d, taps_h, taps_w, pad_d, pad_h, pad_w, crop_depth), weights,
                          cl, epi, map, scratch, b, (double)(c * L.od * L.oh * L.ow), crop_count, sim, cs, st);
    });
}

extern "C" int mb200_ssim_avg_pool(const void* preds, int preds_dtype, const void* target, int target_dtype, int64_t b,
                                   int64_t c, int64_t d, int64_t h, int64_t w, int64_t preds_s_n, int64_t preds_s_c,
                                   int64_t preds_s_d, int64_t preds_s_h, int64_t preds_s_w, int64_t target_s_n,
                                   int64_t target_s_c, int64_t target_s_d, int64_t target_s_h, int64_t target_s_w,
                                   int pool_depth, void* preds_out, void* target_out, void* stream) {
    MB200_SSIM_CHECK_TAGS();
    MB200_REQUIRE(b >= 0 && c >= 1 && h >= 2 && w >= 2 && d >= (pool_depth ? 2 : 1), "pool output would be empty");
    MB200_REQUIRE(preds && target && preds_out && target_out, "NULL pointer");
    const long long n = b * c * (pool_depth ? d / 2 : d) * (h / 2) * (w / 2);
    if (n == 0) return 0;
    const Vol P{preds, preds_dtype, preds_s_n, preds_s_c, preds_s_d, preds_s_h, preds_s_w};
    const Vol Q{target, target_dtype, target_s_n, target_s_c, target_s_d, target_s_h, target_s_w};
    Geo g{};
    g.b = b, g.c = c, g.d = d, g.h = h, g.w = w;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const unsigned blocks = (unsigned)std::min<long long>(cdiv(n, kThreads), 65536ll * 4);
    return with_float_type(preds_dtype, [&](auto tag) -> int {
        using T = typename decltype(tag)::type;
        pool_kernel<T><<<blocks, kThreads, 0, st>>>(P, Q, g, pool_depth ? 1 : 0, reinterpret_cast<T*>(preds_out),
                                                   reinterpret_cast<T*>(target_out));
        count_launch();
        MB200_CUDA_OK(cudaGetLastError());
        return 0;
    });
}

#define MB200_MOMENT_CHECK_FILTER()                                                                                    \
    MB200_REQUIRE(b >= 0 && c >= 1 && d >= 1 && h >= 1 && w >= 1, "bad sizes");                                      \
    MB200_REQUIRE(taps_d >= 1 && taps_h >= 1 && taps_w >= 1 && taps_d <= MB200_SSIM_MAX_TAPS &&                      \
                      taps_h <= MB200_SSIM_MAX_TAPS && taps_w <= MB200_SSIM_MAX_TAPS,                                \
                  "tap counts must lie in [1, %d], got %d, %d, %d", MB200_SSIM_MAX_TAPS, taps_d, taps_h, taps_w)

extern "C" int mb200_vif_scale_update(const void* preds, int preds_dtype, const void* target, int target_dtype,
                                      int64_t b, int64_t c, int64_t d, int64_t h, int64_t w, int64_t preds_s_n,
                                      int64_t preds_s_c, int64_t preds_s_d, int64_t preds_s_h, int64_t preds_s_w,
                                      int64_t target_s_n, int64_t target_s_c, int64_t target_s_d, int64_t target_s_h,
                                      int64_t target_s_w, int taps_d, int taps_h, int taps_w, const void* weights,
                                      double eps, double sigma_n_sq, double* preds_sum, double* target_sum,
                                      void* scratch, int64_t scratch_bytes, void* stream) {
    MB200_SSIM_CHECK_TAGS();
    MB200_MOMENT_CHECK_FILTER();
    const int64_t need = mb200_ssim_scratch_bytes(preds_dtype, b, c, d, h, w, taps_d, taps_h, taps_w, 0, 0, 0);
    MB200_REQUIRE(need >= 0,
                  "the filter (%d, %d, %d taps) gives an empty output or does not fit in shared memory, or the batch has "
                  "2^31 tiles or more", taps_d, taps_h, taps_w);
    MB200_REQUIRE(preds && target && weights && preds_sum && target_sum && scratch, "NULL pointer");
    MB200_REQUIRE(scratch_bytes >= need && (reinterpret_cast<uintptr_t>(scratch) & 15) == 0,
                  "scratch must be 16-byte aligned and mb200_ssim_scratch_bytes(...) bytes");
    if (b == 0) return 0;
    const Vol P{preds, preds_dtype, preds_s_n, preds_s_c, preds_s_d, preds_s_h, preds_s_w};
    const Vol Q{target, target_dtype, target_s_n, target_s_c, target_s_d, target_s_h, target_s_w};
    const Clamp none{0, 0.0, 0.0};
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    return with_float_type(preds_dtype, [&](auto tag) -> int {
        using T = typename decltype(tag)::type;
        using A = typename Cvt<T>::A;
        const Layout L = layout<T>(b, c, d, h, w, taps_d, taps_h, taps_w, 0, 0, 0);
        const VifEpilogue<A> epi{eps, sigma_n_sq};
        return moments<T>(P, Q, L, geo(L, b, c, d, h, w, taps_d, taps_h, taps_w, 0, 0, 0, 0), weights, none, epi, nullptr,
                          scratch, b * c, 1.0, 1.0, preds_sum, target_sum, st);
    });
}

extern "C" int mb200_vif_decimate(const void* preds, int preds_dtype, const void* target, int target_dtype, int64_t b,
                                  int64_t c, int64_t d, int64_t h, int64_t w, int64_t preds_s_n, int64_t preds_s_c,
                                  int64_t preds_s_d, int64_t preds_s_h, int64_t preds_s_w, int64_t target_s_n,
                                  int64_t target_s_c, int64_t target_s_d, int64_t target_s_h, int64_t target_s_w,
                                  int taps_h, int taps_w, const void* weights, void* preds_out, void* target_out,
                                  void* stream) {
    MB200_SSIM_CHECK_TAGS();
    MB200_REQUIRE(b >= 0 && c >= 1 && d >= 1 && h >= 1 && w >= 1, "bad sizes");
    MB200_REQUIRE(taps_h >= 1 && taps_w >= 1 && taps_h <= MB200_SSIM_MAX_TAPS && taps_w <= MB200_SSIM_MAX_TAPS,
                  "tap counts must lie in [1, %d], got %d, %d", MB200_SSIM_MAX_TAPS, taps_h, taps_w);
    MB200_REQUIRE(taps_h <= h && taps_w <= w, "the filter (%d, %d taps) gives an empty output on %lld x %lld", taps_h,
                  taps_w, (long long)h, (long long)w);
    MB200_REQUIRE(preds && target && weights && preds_out && target_out, "NULL pointer");
    Geo g{};
    g.b = b, g.c = c, g.d = d, g.h = h, g.w = w, g.kh = taps_h, g.kw = taps_w;
    g.oh = (h - taps_h + 2) / 2;  // ceil((h - taps_h + 1) / 2): the even positions of the valid output
    g.ow = (w - taps_w + 2) / 2;
    const long long n = b * c * d * g.oh * g.ow;
    if (n == 0) return 0;
    const Vol P{preds, preds_dtype, preds_s_n, preds_s_c, preds_s_d, preds_s_h, preds_s_w};
    const Vol Q{target, target_dtype, target_s_n, target_s_c, target_s_d, target_s_h, target_s_w};
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const unsigned blocks = (unsigned)std::min<long long>(cdiv(n, kThreads), 65536ll * 4);
    return with_float_type(preds_dtype, [&](auto tag) -> int {
        using T = typename decltype(tag)::type;
        decimate_kernel<T><<<blocks, kThreads, 0, st>>>(P, Q, g, reinterpret_cast<const T*>(weights),
                                                        reinterpret_cast<T*>(preds_out), reinterpret_cast<T*>(target_out));
        count_launch();
        MB200_CUDA_OK(cudaGetLastError());
        return 0;
    });
}

extern "C" int mb200_uqi_update(const void* preds, int preds_dtype, const void* target, int target_dtype, int64_t b,
                                int64_t c, int64_t d, int64_t h, int64_t w, int64_t preds_s_n, int64_t preds_s_c,
                                int64_t preds_s_d, int64_t preds_s_h, int64_t preds_s_w, int64_t target_s_n,
                                int64_t target_s_c, int64_t target_s_d, int64_t target_s_h, int64_t target_s_w, int taps_d,
                                int taps_h, int taps_w, int pad_d, int pad_h, int pad_w, int crop_h, int crop_w,
                                const void* weights, double eps, double* sums, void* map, void* scratch,
                                int64_t scratch_bytes, void* stream) {
    MB200_SSIM_CHECK_TAGS();
    MB200_MOMENT_CHECK_FILTER();
    MB200_REQUIRE(pad_d >= 0 && pad_h >= 0 && pad_w >= 0 && pad_d < d && pad_h < h && pad_w < w,
                  "reflect pads (%d, %d, %d) must be non-negative and below the sizes", pad_d, pad_h, pad_w);
    MB200_REQUIRE(crop_h >= 0 && crop_w >= 0, "crop margins (%d, %d) must be non-negative", crop_h, crop_w);
    const int64_t need = mb200_ssim_scratch_bytes(preds_dtype, b, c, d, h, w, taps_d, taps_h, taps_w, pad_d, pad_h, pad_w);
    MB200_REQUIRE(need >= 0,
                  "the filter (%d, %d, %d taps) gives an empty output or does not fit in shared memory, or the batch has "
                  "2^31 tiles or more", taps_d, taps_h, taps_w);
    MB200_REQUIRE(preds && target && weights && sums && scratch, "NULL pointer");
    MB200_REQUIRE(scratch_bytes >= need && (reinterpret_cast<uintptr_t>(scratch) & 15) == 0,
                  "scratch must be 16-byte aligned and mb200_ssim_scratch_bytes(...) bytes");
    if (b == 0) return 0;
    const Vol P{preds, preds_dtype, preds_s_n, preds_s_c, preds_s_d, preds_s_h, preds_s_w};
    const Vol Q{target, target_dtype, target_s_n, target_s_c, target_s_d, target_s_h, target_s_w};
    const Clamp none{0, 0.0, 0.0};
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    return with_float_type(preds_dtype, [&](auto tag) -> int {
        using T = typename decltype(tag)::type;
        using A = typename Cvt<T>::A;
        const Layout L = layout<T>(b, c, d, h, w, taps_d, taps_h, taps_w, pad_d, pad_h, pad_w);
        const UqiEpilogue<A> epi{eps, crop_h, crop_w};
        return moments<T>(P, Q, L, geo(L, b, c, d, h, w, taps_d, taps_h, taps_w, pad_d, pad_h, pad_w, 0), weights, none,
                          epi, map, scratch, b, 1.0, 1.0, sums, nullptr, st);
    });
}
