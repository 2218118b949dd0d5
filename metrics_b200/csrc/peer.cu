// K10 — state exchange over NVLink peer memory (one process per GPU, symmetric allocations).
//
// Replaces, for the states that shard naturally (SURVEY.md §8(e)), the reference's per-state
// `barrier + all_gather(shape) + all_gather(data)` (utilities/distributed.py:100-153, called from metric.py:501-540):
//
//   * mb200_peer_pack_keys_put   the class-sharded exchange of one-vs-rest curve scores FUSED with the key packing: the
//                                transpose kernel that turns [n, C] scores into class-major sort keys stores every key row
//                                straight into the memory of the rank that owns the class, at its final position
//                                [class - first_class][column offset of this rank + sample] — no staging buffer, no
//                                all-to-all, no reorder pass.  (W-1)/W of the stores travel over NVLink, overlapped with the
//                                local 1/W and with the loads of the next tile.
//   * mb200_peer_put_all         all-gather by peer stores: every rank writes its chunk at its offset into every rank
//                                (targets, per-class results; a few bytes per sample / class).
//   * mb200_peer_reduce_put_i64  all-reduce of integer states in two peer phases inside one launch per rank: rank r reduces
//                                slice r of every rank's input region (peer loads) and stores the reduced slice into every
//                                rank's output region (peer stores).  Bit-exact: integer add / max / min are associative.
//
// `peer_bases` is a DEVICE array of `world` base pointers of the same symmetric allocation on every rank (entry r = rank r's
// base; torch.distributed._symmetric_memory's `buffer_ptrs_dev`).  Cross-rank ordering (everybody's stores are visible
// before anybody reads) is the caller's: a signal-pad barrier on the same stream before and after (metrics_b200/peer.py).
#include "common.cuh"

namespace mb200 {

// [n, C] row-major scores -> keys of class c at peer (c / cpr): base + keys_off + ((c % cpr) * n_total + col_off + i) * 4.
// 32 x 32 shared-memory tile transpose: coalesced 128-byte reads along the class dimension, coalesced 128-byte stores along
// the sample dimension (one store instruction of a warp = one class row segment = one NVLink write of 128 B).
template <typename T>
__global__ void __launch_bounds__(256) pack_keys_put_kernel(const T* __restrict__ preds, int n, int C, int cpr,
                                                            long long n_total, long long col_off,
                                                            void* const* __restrict__ peer_bases, long long keys_off) {
    __shared__ unsigned tile[32][33];
    load_desc_key_tile(preds, n, C, tile);
    __syncthreads();
    const int n0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int j = ty; j < 32; j += 8) {
        const int cc = c0 + j, nn = n0 + tx;
        if (nn < n && cc < C) {
            const int owner = cc / cpr;
            unsigned* dst = reinterpret_cast<unsigned*>(static_cast<char*>(peer_bases[owner]) + keys_off);
            dst[(size_t)(cc - owner * cpr) * (size_t)n_total + (size_t)(col_off + nn)] = tile[tx][j];
        }
    }
}

// every rank's chunk -> all ranks: grid.y = destination rank
__global__ void __launch_bounds__(256) put_all_kernel(const unsigned char* __restrict__ src, long long nbytes,
                                                      void* const* __restrict__ peer_bases, long long dst_off) {
    unsigned char* dst = static_cast<unsigned char*>(peer_bases[blockIdx.y]) + dst_off;
    const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, nthr = (long long)gridDim.x * blockDim.x;
    const bool vec = ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0;
    long long done = 0;
    if (vec) {
        const long long n16 = nbytes >> 4;
        for (long long i = tid; i < n16; i += nthr)
            reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<const uint4*>(src)[i];
        done = n16 << 4;
    }
    for (long long i = done + tid; i < nbytes; i += nthr) dst[i] = src[i];
}

template <int kOp>
__device__ __forceinline__ long long combine(long long a, long long b) {
    if (kOp == 0) return a + b;
    if (kOp == 1) return a > b ? a : b;
    return a < b ? a : b;
}

// rank `rank` owns elements [lo, hi) of the n-element state (lo even): out[p][i] = op over q of in[q][i] for every peer p
template <int kOp, int kMaxWorld>
__global__ void __launch_bounds__(256) reduce_put_kernel(void* const* __restrict__ peer_bases, long long in_off,
                                                         long long out_off, long long lo, long long hi, int world) {
    const long long* in[kMaxWorld];
    long long* out[kMaxWorld];
#pragma unroll
    for (int p = 0; p < kMaxWorld; ++p) {
        const int q = p < world ? p : 0;
        in[p] = reinterpret_cast<const long long*>(static_cast<char*>(peer_bases[q]) + in_off);
        out[p] = reinterpret_cast<long long*>(static_cast<char*>(peer_bases[q]) + out_off);
    }
    const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, nthr = (long long)gridDim.x * blockDim.x;
    const long long pairs = (hi - lo) >> 1;
    for (long long k = tid; k < pairs; k += nthr) {  // 16 bytes per peer per iteration
        const long long i = lo + 2 * k;
        longlong2 acc = *reinterpret_cast<const longlong2*>(in[0] + i);
#pragma unroll
        for (int p = 1; p < kMaxWorld; ++p) {
            if (p < world) {
                const longlong2 v = *reinterpret_cast<const longlong2*>(in[p] + i);
                acc.x = combine<kOp>(acc.x, v.x);
                acc.y = combine<kOp>(acc.y, v.y);
            }
        }
#pragma unroll
        for (int p = 0; p < kMaxWorld; ++p)
            if (p < world) *reinterpret_cast<longlong2*>(out[p] + i) = acc;
    }
    if (((hi - lo) & 1) && tid == 0) {
        const long long i = hi - 1;
        long long acc = in[0][i];
#pragma unroll
        for (int p = 1; p < kMaxWorld; ++p)
            if (p < world) acc = combine<kOp>(acc, in[p][i]);
#pragma unroll
        for (int p = 0; p < kMaxWorld; ++p)
            if (p < world) out[p][i] = acc;
    }
}

}  // namespace mb200

using namespace mb200;

extern "C" int mb200_peer_pack_keys_put(const void* preds, int preds_dtype, int64_t n_local, int64_t num_classes,
                                        int64_t classes_per_rank, int world, int64_t n_total, int64_t col_offset,
                                        void* const* peer_bases, int64_t keys_offset_bytes, void* stream) {
    MB200_REQUIRE(n_local >= 0 && num_classes >= 1 && classes_per_rank >= 1 && world >= 1, "bad sizes");
    MB200_REQUIRE(classes_per_rank * world >= num_classes, "classes_per_rank * world must cover num_classes");
    MB200_REQUIRE(col_offset >= 0 && col_offset + n_local <= n_total, "column range [%lld, %lld) outside n_total=%lld",
                  (long long)col_offset, (long long)(col_offset + n_local), (long long)n_total);
    MB200_REQUIRE(n_local < (1ll << 31) && num_classes < (1ll << 24), "sizes out of range");
    MB200_REQUIRE(peer_bases != nullptr && (keys_offset_bytes & 3) == 0, "peer table is NULL or the key region is misaligned");
    if (n_local == 0) return 0;
    MB200_REQUIRE(preds != nullptr, "preds is NULL");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const dim3 grid((unsigned)((n_local + 31) / 32), (unsigned)((num_classes + 31) / 32));  // y <= 65535: C < 2^21
    MB200_REQUIRE(grid.y <= 65535u, "more than 2,097,120 classes are not supported (got %lld)", (long long)num_classes);
    MB200_REQUIRE(is_float_tag<kNoF64>(preds_dtype), "scores must be f32/f16/bf16 (dtype tag %d)", preds_dtype);
    with_float_type<kNoF64>(preds_dtype, [&](auto t) {
        using T = typename decltype(t)::type;
        pack_keys_put_kernel<T><<<grid, 256, 0, st>>>(reinterpret_cast<const T*>(preds), (int)n_local, (int)num_classes,
                                                     (int)classes_per_rank, (long long)n_total, (long long)col_offset, peer_bases,
                                                     (long long)keys_offset_bytes);
        return 0;
    });
    count_launch();
    return check_cuda(cudaGetLastError(), "peer pack+put launch");
}

extern "C" int mb200_peer_put_all(const void* src, int64_t nbytes, void* const* peer_bases, int64_t dst_offset_bytes,
                                  int world, void* stream) {
    MB200_REQUIRE(nbytes >= 0 && world >= 1 && dst_offset_bytes >= 0, "bad sizes");
    if (nbytes == 0) return 0;
    MB200_REQUIRE(src != nullptr && peer_bases != nullptr, "NULL pointer");
    long long blocks = (nbytes / 16 + 255) / 256;
    if (blocks < 1) blocks = 1;
    const long long cap = (long long)sm_count() * 4 / world + 1;
    if (blocks > cap) blocks = cap;
    put_all_kernel<<<dim3((unsigned)blocks, (unsigned)world), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        static_cast<const unsigned char*>(src), (long long)nbytes, peer_bases, (long long)dst_offset_bytes);
    count_launch();
    return check_cuda(cudaGetLastError(), "peer put launch");
}

extern "C" int mb200_peer_reduce_put_i64(void* const* peer_bases, int64_t in_offset_bytes, int64_t out_offset_bytes,
                                         int64_t n, int rank, int world, int op, void* stream) {
    MB200_REQUIRE(peer_bases != nullptr && n >= 0 && world >= 1 && world <= 16 && rank >= 0 && rank < world, "bad arguments");
    MB200_REQUIRE(op >= 0 && op <= 2, "op must be 0 (sum), 1 (max) or 2 (min)");
    MB200_REQUIRE(((in_offset_bytes | out_offset_bytes) & 15) == 0, "regions must be 16-byte aligned");
    if (n == 0) return 0;
    const long long per = ((n + world - 1) / world + 1) & ~1ll;  // even: every slice starts 16-byte aligned
    const long long lo = per * rank < n ? per * rank : n, hi = lo + per < n ? lo + per : n;
    if (hi <= lo) return 0;
    long long blocks = ((hi - lo) / 2 + 255) / 256;
    if (blocks < 1) blocks = 1;
    if (blocks > 2ll * sm_count()) blocks = 2ll * sm_count();
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
#define MB200_RP(OP)                                                                                        \
    reduce_put_kernel<OP, 16><<<(unsigned)blocks, 256, 0, st>>>(peer_bases, (long long)in_offset_bytes,     \
                                                                 (long long)out_offset_bytes, lo, hi, world)
    if (op == 0) MB200_RP(0);
    else if (op == 1) MB200_RP(1);
    else MB200_RP(2);
#undef MB200_RP
    count_launch();
    return check_cuda(cudaGetLastError(), "peer reduce+put launch");
}
