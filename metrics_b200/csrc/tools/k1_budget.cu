// Prices where a cfg2 confusion-matrix update (K1, [65536, 1000] bf16, C = 1000) spends its time above the HBM read stream.
// Driven by benchmarks/k1_budget.py, which builds it, adds the card's name, power limit and clocks and writes the JSON.
// Build: nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a --expt-relaxed-constexpr -o k1_budget k1_budget.cu ../core.cu
//
// Every timing streams 16 distinct 131 MB batches (2.1 GB, far beyond the 50 MB L2), as bench.py does:
//   probe xN      one read-only launch (xor of every 16-byte vector) over N consecutive batches, N = 1, 2, 4, 8; the slope
//                 over N is the steady-state read time of one batch, the intercept the fixed cost of one launch;
//   k1            K1 back to back with programmatic dependent launch, exactly as update() launches it;
//   k1_one_wave   the same launch on one resident wave of CTAs (a grid-stride loop of about 12 rows per warp);
//   k1_state8k    k1_one_wave with every state RED aimed into 8 KB ((t*C+p) & 1023): the difference from k1_one_wave
//                 prices the [C, C] state's HBM round trips (its counts are thrown away);
//   k1_rpwN       the same launch on ceil(N_rows / (8 warps * N)) CTAs, N rows per warp: the hardware block scheduler hands
//                 out rows, so the difference from k1_one_wave prices the SM skew of the one-wave grid-stride loop;
//   rows_C{C}_N{N}_{wave,rpw1}
//                 the row-size sweep behind vec_grid's threshold: [N, C] bf16 confusion-matrix updates (labels in [0, 128))
//                 on one resident wave and on one row per warp, for rows of 256 B to 2000 B.
// Variants alternate; each is repeated `reps` times (argv[1], default 7).  The last line is one JSON document.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "../confmat.cu"

using namespace mb200;

namespace {

constexpr int kN = 65536, kC = 1000, kBatches = 16;
constexpr size_t kBatchElems = (size_t)kN * kC;
constexpr size_t kBatchBytes = kBatchElems * sizeof(__nv_bfloat16);

// ConfmatSink<false> with every RED folded into 1024 counters (8 KB): the state never leaves L2.
struct State8kSink {
    long long* confmat;
    int C;
    struct Local {};
    static constexpr bool kNeedsTarget = true;
    static constexpr bool kOverlapSafe = true;
    __device__ __forceinline__ void block_init() {}
    __device__ __forceinline__ void init(Local&) {}
    __device__ __forceinline__ void row(Local&, long long, long long t, int p) {
        red_add_u64(confmat + ((t * C + p) & 1023), 1ull);
    }
    __device__ __forceinline__ void finish(Local&) {}
};

__global__ void fill_kernel(unsigned short* logits, long long* target, size_t n_logits, size_t n_target, int C) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_logits; i += stride) {
        unsigned s = (unsigned)(i * 2654435761u) ^ (unsigned)(i >> 32) * 40503u;
        s ^= s >> 15, s *= 2246822519u, s ^= s >> 13, s *= 3266489917u, s ^= s >> 16;
        logits[i] = (unsigned short)((s & 0x8000u) | (0x3e00u + ((s >> 4) & 0x3ffu)));  // bf16 in about (-4, 4)
        if (i < n_target) target[i] = (long long)((s >> 11) % (unsigned)C);
    }
}

__global__ void __launch_bounds__(256) probe_kernel(const uint4* __restrict__ p, size_t nvec, unsigned* out) {
    constexpr int kUnroll = 8;
    unsigned acc = 0;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (; i + (kUnroll - 1) * stride < nvec; i += kUnroll * stride) {
        uint4 v[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) v[u] = ld_stream16(p + i + u * stride);
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) acc ^= v[u].x ^ v[u].y ^ v[u].z ^ v[u].w;
    }
    for (; i < nvec; i += stride) {
        const uint4 v = ld_stream16(p + i);
        acc ^= v.x ^ v.y ^ v.z ^ v.w;
    }
    if (acc == 0x12345678u) out[0] = acc;
}

#define CK(expr)                                                                                      \
    do {                                                                                              \
        cudaError_t _e = (expr);                                                                      \
        if (_e != cudaSuccess) {                                                                      \
            fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #expr, cudaGetErrorString(_e));     \
            exit(1);                                                                                  \
        }                                                                                             \
    } while (0)

__nv_bfloat16* g_logits;
long long* g_target;
long long* g_confmat;
long long* g_state8k;
unsigned* g_sink;
cudaStream_t g_st;
cudaEvent_t g_e0, g_e1;

long long* g_labels128;  // kBatches x kSweepMaxN labels in [0, 128) for the row-size sweep
constexpr int kSweepMaxN = 262144;

RowArgs args_of(int b) {
    return RowArgs{g_logits + (size_t)b * kBatchElems, g_target + (size_t)b * kN, MB200_I64, kN, kC, 1, 0, 0, nullptr};
}

// batch b of the sweep's [n, C] bf16 logits (16 x n x C fits in the 16 cfg2 batches)
RowArgs sweep_args_of(int b, int n, int C) {
    return RowArgs{g_logits + (size_t)b * n * C, g_labels128 + (size_t)b * kSweepMaxN, MB200_I64, n, C, 1, 0, 0, nullptr};
}

__global__ void fill_labels_kernel(long long* target, size_t n) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        unsigned s = (unsigned)(i * 2246822519u) ^ 0x9e3779b9u;
        s ^= s >> 15, s *= 2654435761u, s ^= s >> 13;
        target[i] = (long long)(s & 127u);
    }
}

// us per step of `steps` back-to-back updates (no host synchronisation between them), after a warm-up
template <typename F>
double per_step_us(F&& launch, int steps) {
    for (int i = 0; i < 32; ++i) launch(i % kBatches);
    CK(cudaStreamSynchronize(g_st));
    CK(cudaEventRecord(g_e0, g_st));
    for (int i = 0; i < steps; ++i) launch(i % kBatches);
    CK(cudaEventRecord(g_e1, g_st));
    CK(cudaEventSynchronize(g_e1));
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, g_e0, g_e1));
    CK(cudaGetLastError());
    return ms * 1000.0 / steps;
}

// us of ONE probe launch over `mult` consecutive batches starting at batch `first`
double probe_us(int first, int mult) {
    const int grid = sm_count() * 8;
    const size_t nvec = kBatchBytes * mult / 16;
    const uint4* p = reinterpret_cast<const uint4*>(g_logits + (size_t)first * kBatchElems);
    CK(cudaStreamSynchronize(g_st));
    CK(cudaEventRecord(g_e0, g_st));
    probe_kernel<<<grid, 256, 0, g_st>>>(p, nvec, g_sink);
    CK(cudaEventRecord(g_e1, g_st));
    CK(cudaEventSynchronize(g_e1));
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, g_e0, g_e1));
    CK(cudaGetLastError());
    return ms * 1000.0;
}

template <typename Sink>
void launch_k1(const RowArgs& a, Sink sink, int grid) {
    auto kern = rows_vec_kernel<__nv_bfloat16, Sink, true>;
    CK(launch_overlapped(kern, grid, kRowThreads, 0, g_st, a, sink));
}

struct Series {
    std::string name;
    std::vector<double> us;
};

}  // namespace

int main(int argc, char** argv) {
    const int reps = argc > 1 ? std::max(1, atoi(argv[1])) : 7;
    const int steps = argc > 2 ? std::max(16, atoi(argv[2])) : 1000;
    CK(cudaSetDevice(0));
    CK(cudaStreamCreateWithFlags(&g_st, cudaStreamNonBlocking));
    CK(cudaEventCreate(&g_e0));
    CK(cudaEventCreate(&g_e1));
    CK(cudaMalloc(&g_logits, kBatchBytes * kBatches));
    CK(cudaMalloc(&g_target, sizeof(long long) * kN * kBatches));
    CK(cudaMalloc(&g_confmat, sizeof(long long) * kC * kC));
    CK(cudaMalloc(&g_state8k, sizeof(long long) * 1024));
    CK(cudaMalloc(&g_sink, sizeof(unsigned)));
    CK(cudaMalloc(&g_labels128, sizeof(long long) * kSweepMaxN * kBatches));
    fill_labels_kernel<<<sm_count() * 16, 256, 0, g_st>>>(g_labels128, (size_t)kSweepMaxN * kBatches);
    CK(cudaMemsetAsync(g_confmat, 0, sizeof(long long) * kC * kC, g_st));
    fill_kernel<<<sm_count() * 16, 256, 0, g_st>>>(reinterpret_cast<unsigned short*>(g_logits), g_target,
                                                     kBatchElems * kBatches, (size_t)kN * kBatches, kC);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(g_st));

    const int wave = resident_blocks(rows_vec_kernel<__nv_bfloat16, ConfmatSink<false>, true>, kRowThreads, 0);
    const int wpb = kRowThreads / 32;
    const int rpw[] = {1, 2, 4, 8};
    const int mults[] = {1, 2, 4, 8};

    std::vector<Series> series;
    auto at = [&](const std::string& name) -> Series& {
        for (Series& s : series)
            if (s.name == name) return s;
        series.push_back(Series{name, {}});
        return series.back();
    };
    for (int rep = 0; rep < reps; ++rep) {
        for (int m : mults) {
            // four single launches per sample, each over batches not read by the launch before it
            std::vector<double> v;
            for (int j = 0; j < 4; ++j) v.push_back(probe_us(((rep * 4 + j) * m) % kBatches, m));
            std::sort(v.begin(), v.end());
            at("probe_x" + std::to_string(m)).us.push_back(0.5 * (v[1] + v[2]));
        }
        at("k1").us.push_back(per_step_us(
            [&](int b) {
                const RowArgs a = args_of(b);
                if (mb200_multiclass_confmat_update(a.preds, MB200_BF16, 1, a.target, MB200_I64, kN, kC, 1, 0, 0,
                                                    reinterpret_cast<int64_t*>(g_confmat), nullptr, g_st) != 0) {
                    fprintf(stderr, "update failed: %s\n", mb200_last_error());
                    exit(1);
                }
            },
            steps));
        at("k1_one_wave").us.push_back(
            per_step_us([&](int b) { launch_k1(args_of(b), ConfmatSink<false>{g_confmat, kC}, wave); }, steps));
        at("k1_state8k").us.push_back(
            per_step_us([&](int b) { launch_k1(args_of(b), State8kSink{g_state8k, kC}, wave); }, steps));
        for (int r : rpw) {
            const int grid = (kN + wpb * r - 1) / (wpb * r);
            at("k1_rpw" + std::to_string(r)).us.push_back(
                per_step_us([&](int b) { launch_k1(args_of(b), ConfmatSink<false>{g_confmat, kC}, grid); }, steps));
        }
        for (int C : {128, 256, 512, 768, 1000}) {
            for (int n : {16384, 65536, kSweepMaxN}) {
                if ((size_t)n * C > kBatchElems) continue;
                const std::string name = "rows_C" + std::to_string(C) + "_N" + std::to_string(n);
                const int one_wave = std::min(wave, (n + wpb - 1) / wpb), per_row = (n + wpb - 1) / wpb;
                at(name + "_wave").us.push_back(per_step_us(
                    [&](int b) { launch_k1(sweep_args_of(b, n, C), ConfmatSink<false>{g_confmat, C}, one_wave); },
                    steps / 4));
                at(name + "_rpw1").us.push_back(per_step_us(
                    [&](int b) { launch_k1(sweep_args_of(b, n, C), ConfmatSink<false>{g_confmat, C}, per_row); },
                    steps / 4));
            }
        }
        fprintf(stderr, "rep %d/%d done\n", rep + 1, reps);
    }

    std::string js = "{\"N\": " + std::to_string(kN) + ", \"C\": " + std::to_string(kC) +
                     ", \"batch_bytes\": " + std::to_string(kBatchBytes) + ", \"batches\": " + std::to_string(kBatches) +
                     ", \"sms\": " + std::to_string(sm_count()) + ", \"one_wave_ctas\": " + std::to_string(wave) +
                     ", \"steps_per_sample\": " + std::to_string(steps) + ", \"series\": {";
    for (size_t i = 0; i < series.size(); ++i) {
        js += (i ? ", \"" : "\"") + series[i].name + "\": [";
        for (size_t j = 0; j < series[i].us.size(); ++j) {
            char buf[32];
            snprintf(buf, sizeof buf, "%s%.4f", j ? ", " : "", series[i].us[j]);
            js += buf;
        }
        js += "]";
    }
    js += "}}";
    printf("%s\n", js.c_str());
    CK(cudaFree(g_logits));
    CK(cudaFree(g_target));
    CK(cudaFree(g_confmat));
    CK(cudaFree(g_state8k));
    CK(cudaFree(g_sink));
    CK(cudaFree(g_labels128));
    return 0;
}
