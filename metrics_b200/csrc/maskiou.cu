// K12 — instance-mask IoU for `MeanAveragePrecision(iou_type="segm")` (reference seam: detection/mean_ap.py:848-853 turns every
// mask into a run-length code on the HOST with pycocotools' `mask_utils.encode`, `COCOeval.computeIoU` then walks pairs of
// run-length codes on the host again, maskApi.c:rleIou).
//
// Here masks never leave the device: `mb200_mask_pack_bits` turns a batch of boolean masks into one bit per pixel (32 pixels
// per word) and counts their areas; `mb200_mask_pair_intersections` produces, for every image, the [detections x ground
// truths] table of intersection pixel counts = popcount(a & b) over the words of the two masks — integer exact; the bit rows
// come from HBM once and are re-read from L2 by the pair tiles.  The matching kernel
// (cocomap.cu, `mb200_coco_map_match_ex`) derives the IoU from the table and the areas exactly like maskApi.c:rleIou does
// (intersection 0 -> 0; crowd ground truth -> union = detection area).
#include "common.cuh"

namespace mb200 {

// 16 mask bytes (any non-zero value = set) -> 16 bits, pixel order
__device__ __forceinline__ unsigned nibble_of(unsigned x) {
    unsigned t = x | (x >> 4);
    t |= t >> 2;
    t |= t >> 1;
    t &= 0x01010101u;                       // one bit per byte, at bit 0 of the byte
    return (t * 0x01020408u) >> 24 & 0xfu;  // byte i's bit -> bit i (the partial products land on distinct bits: no carries)
}

// A warp turns 2048 pixels (bytes) of one mask into 64 words per step, as four pieces of 512: lane l owns pixels [16 l, 16 l +
// 16) of each piece — one 16-byte load when the address is 16-byte aligned, the four loads issued together —, neighbouring
// lanes join their halves, even lanes store.  (The first version read one byte per lane and balloted: 32 bytes per warp
// instruction; one 512-pixel piece per step is latency-bound.)
constexpr int kPackPieces = 4;
template <typename AreaT>  // long long: area array of mb200_mask_pack_bits; int: the area slots of a state entry
__global__ void __launch_bounds__(256) mask_pack_bits_kernel(const unsigned char* __restrict__ masks, long long n_masks,
                                                             long long hw, long long words, unsigned* __restrict__ out,
                                                             long long out_stride, AreaT* __restrict__ area, int* __restrict__ header,
                                                             int h0, int h1, int h2) {
    const int lane = threadIdx.x & 31;
    if (header && blockIdx.x == 0 && threadIdx.x == 0) header[0] = h0, header[1] = h1, header[2] = h2;
    const long long chunks = (hw + 512 * kPackPieces - 1) / (512 * kPackPieces);  // per mask
    const long long total = n_masks * chunks;
    const long long wstep = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long task = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); task < total; task += wstep) {
        const long long m = task / chunks, c = task % chunks;
        const unsigned char* __restrict__ row = masks + m * hw;
        unsigned bits[kPackPieces];
        uint4 v[kPackPieces];
        bool vec[kPackPieces];
#pragma unroll
        for (int q = 0; q < kPackPieces; ++q) {
            const long long p0 = (c * kPackPieces + q) * 512 + 16 * lane;  // first pixel of this lane in piece q
            vec[q] = p0 + 16 <= hw && ((reinterpret_cast<uintptr_t>(row + p0) & 15) == 0);
            if (vec[q]) v[q] = *reinterpret_cast<const uint4*>(row + p0);
        }
        unsigned cnt = 0;
#pragma unroll
        for (int q = 0; q < kPackPieces; ++q) {
            const long long p0 = (c * kPackPieces + q) * 512 + 16 * lane;
            if (vec[q]) {
                bits[q] = nibble_of(v[q].x) | (nibble_of(v[q].y) << 4) | (nibble_of(v[q].z) << 8) | (nibble_of(v[q].w) << 12);
            } else {
                bits[q] = 0;
#pragma unroll
                for (int k = 0; k < 16; ++k)
                    if (p0 + k < hw && row[p0 + k] != 0) bits[q] |= 1u << k;
            }
            const unsigned hi = __shfl_down_sync(kFull, bits[q], 1);
            const long long w = (c * kPackPieces + q) * 16 + (lane >> 1);
            if ((lane & 1) == 0 && w < words) out[m * out_stride + w] = bits[q] | (hi << 16);
            cnt += (unsigned)__popc(bits[q]);
        }
        cnt = __reduce_add_sync(kFull, cnt);
        if (lane == 0 && cnt) {
            if constexpr (sizeof(AreaT) == 8) atomicAdd(reinterpret_cast<unsigned long long*>(area + m), (unsigned long long)cnt);
            else atomicAdd(reinterpret_cast<unsigned*>(area + m), cnt);
        }
    }
}

// grid = (images, splits): the warps of the CTAs of one image share its detection x ground-truth pairs in tiles of 2 x 4: per
// word step a lane loads 2 detection words and 4 ground-truth words for 8 and+popc (one warp per PAIR loaded 2 words per
// popc and was bound by L2 reads: 9.8 GB for the 0.3 GB of bit rows of the 64-image benchmark).  A pair of different classes
// (unless micro) is never looked at by the matcher and is written as 0.
constexpr int kPairTd = 2, kPairTg = 4;
__global__ void __launch_bounds__(256) mask_pair_inter_kernel(const unsigned* __restrict__ det_words,
                                                              const long long* __restrict__ det_word_off,
                                                              const unsigned* __restrict__ gt_words,
                                                              const long long* __restrict__ gt_word_off,
                                                              const int* __restrict__ det_off, const int* __restrict__ gt_off,
                                                              const int* __restrict__ img_words,
                                                              const long long* __restrict__ det_label,
                                                              const long long* __restrict__ gt_label, int micro,
                                                              const long long* __restrict__ pair_off,
                                                              double* __restrict__ inter) {
    const int img = blockIdx.x;
    const int d0 = det_off[img], D = det_off[img + 1] - d0;
    const int g0 = gt_off[img], G = gt_off[img + 1] - g0;
    if (D == 0 || G == 0) return;
    const int words = img_words[img];
    const int tiles_g = (G + kPairTg - 1) / kPairTg;
    const long long tiles = (long long)((D + kPairTd - 1) / kPairTd) * tiles_g;
    const int lane = threadIdx.x & 31;
    const long long wstep = (long long)gridDim.y * (blockDim.x >> 5);
    double* __restrict__ table = inter + pair_off[img];
    for (long long tile = (long long)blockIdx.y * (blockDim.x >> 5) + (threadIdx.x >> 5); tile < tiles; tile += wstep) {
        const int db = (int)(tile / tiles_g) * kPairTd, gb = (int)(tile % tiles_g) * kPairTg;
        const unsigned* a[kPairTd];
        const unsigned* b[kPairTg];
        long long la[kPairTd], lb[kPairTg];
        bool any = micro != 0;
#pragma unroll
        for (int i = 0; i < kPairTd; ++i) {
            const int d = min(db + i, D - 1);  // clamped: a duplicate row whose results are not written
            a[i] = det_words + det_word_off[d0 + d];
            la[i] = det_label[d0 + d];
        }
#pragma unroll
        for (int j = 0; j < kPairTg; ++j) {
            const int g = min(gb + j, G - 1);
            b[j] = gt_words + gt_word_off[g0 + g];
            lb[j] = gt_label[g0 + g];
        }
#pragma unroll
        for (int i = 0; i < kPairTd; ++i)
#pragma unroll
            for (int j = 0; j < kPairTg; ++j) any |= la[i] == lb[j];
        unsigned cnt[kPairTd][kPairTg] = {};
        if (any) {
            for (int w = lane; w < words; w += 32) {
                unsigned av[kPairTd], bv[kPairTg];
#pragma unroll
                for (int i = 0; i < kPairTd; ++i) av[i] = a[i][w];
#pragma unroll
                for (int j = 0; j < kPairTg; ++j) bv[j] = b[j][w];
#pragma unroll
                for (int i = 0; i < kPairTd; ++i)
#pragma unroll
                    for (int j = 0; j < kPairTg; ++j) cnt[i][j] += (unsigned)__popc(av[i] & bv[j]);
            }
        }
#pragma unroll
        for (int i = 0; i < kPairTd; ++i)
#pragma unroll
            for (int j = 0; j < kPairTg; ++j) {
                const unsigned c = __reduce_add_sync(kFull, cnt[i][j]);
                if (lane == 0 && db + i < D && gb + j < G)
                    table[(long long)(db + i) * G + gb + j] = (micro || la[i] == lb[j]) ? (double)c : 0.0;
            }
    }
}

}  // namespace mb200

using namespace mb200;

extern "C" int mb200_mask_pack_bits(const uint8_t* masks, int64_t n_masks, int64_t pixels_per_mask, uint32_t* words_out,
                                    int64_t out_stride_words, int64_t* area_out, void* stream) {
    MB200_REQUIRE(n_masks >= 0 && pixels_per_mask >= 0, "bad sizes");
    const int64_t words = (pixels_per_mask + 31) / 32;
    MB200_REQUIRE(out_stride_words >= words, "output row stride %lld is smaller than the %lld words of a mask",
                  (long long)out_stride_words, (long long)words);
    if (n_masks == 0) return 0;
    MB200_REQUIRE(area_out, "NULL pointer");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    MB200_CUDA_OK(cudaMemsetAsync(area_out, 0, (size_t)n_masks * 8, st));
    if (words == 0) return 0;
    MB200_REQUIRE(masks && words_out, "NULL pointer");
    long long grid = (n_masks * ((pixels_per_mask + 512 * kPackPieces - 1) / (512 * kPackPieces)) + 7) / 8;
    const long long cap = (long long)sm_count() * 8;
    if (grid > cap) grid = cap;
    mask_pack_bits_kernel<long long><<<(unsigned)grid, 256, 0, st>>>(masks, n_masks, pixels_per_mask, words, words_out,
                                                                    out_stride_words, reinterpret_cast<long long*>(area_out),
                                                                    nullptr, 0, 0, 0);
    count_launch();
    return check_cuda(cudaGetLastError(), "mask pack launch");
}

// The per-image state entry of MeanAveragePrecision (detection/mean_ap.py `_mask_state`) in one call:
// entry_out int32 [3 + n + n * ceil(H*W/32)] = [n, H, W, area_0 .. area_{n-1}, bit rows].
extern "C" int mb200_mask_pack_entry(const uint8_t* masks, int64_t n_masks, int64_t height, int64_t width, int32_t* entry_out,
                                     void* stream) {
    MB200_REQUIRE(n_masks >= 0 && n_masks < (1ll << 31) && height >= 0 && width >= 0 && height < (1ll << 31) && width < (1ll << 31) &&
                      height * width < (1ll << 31),
                  "bad sizes");
    MB200_REQUIRE(entry_out && (n_masks == 0 || height * width == 0 || masks), "NULL pointer");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int64_t hw = height * width, words = (hw + 31) / 32;
    MB200_CUDA_OK(cudaMemsetAsync(entry_out, 0, (size_t)(3 + n_masks) * 4, st));  // areas are accumulated with atomics
    long long grid = (n_masks * ((hw + 512 * kPackPieces - 1) / (512 * kPackPieces)) + 7) / 8;
    const long long cap = (long long)sm_count() * 8;
    if (grid > cap) grid = cap;
    if (grid < 1) grid = 1;  // the header is written even for an image without masks
    mask_pack_bits_kernel<int><<<(unsigned)grid, 256, 0, st>>>(masks, n_masks, hw, words,
                                                              reinterpret_cast<unsigned*>(entry_out + 3 + n_masks), words,
                                                              entry_out + 3, entry_out, (int)n_masks, (int)height, (int)width);
    count_launch();
    return check_cuda(cudaGetLastError(), "mask entry launch");
}

extern "C" int mb200_mask_pair_intersections(const uint32_t* det_words, const int64_t* det_word_off, const uint32_t* gt_words,
                                             const int64_t* gt_word_off, const int32_t* det_off, const int32_t* gt_off,
                                             const int32_t* img_words, const int64_t* det_label, const int64_t* gt_label,
                                             int micro, const int64_t* pair_off, int64_t n_img, int64_t max_pairs_per_img,
                                             double* inter_out, void* stream) {
    MB200_REQUIRE(n_img >= 0 && max_pairs_per_img >= 0, "bad sizes");
    if (n_img == 0 || max_pairs_per_img == 0) return 0;
    MB200_REQUIRE(det_word_off && gt_word_off && det_off && gt_off && img_words && det_label && gt_label && pair_off && inter_out,
                  "NULL pointer");
    // enough CTAs per image that the busiest image's pairs are spread, without flooding the grid for thousands of images
    long long splits = (max_pairs_per_img / (kPairTd * kPairTg) + 1 + 7) / 8;  // 8 warps per CTA, one 2 x 4 tile per warp step
    const long long want = ((long long)sm_count() * 8 + n_img - 1) / n_img;
    if (splits > want) splits = want;
    if (splits < 1) splits = 1;
    if (splits > 65535) splits = 65535;
    mask_pair_inter_kernel<<<dim3((unsigned)n_img, (unsigned)splits), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        det_words, reinterpret_cast<const long long*>(det_word_off), gt_words, reinterpret_cast<const long long*>(gt_word_off),
        det_off, gt_off, img_words, reinterpret_cast<const long long*>(det_label), reinterpret_cast<const long long*>(gt_label),
        micro, reinterpret_cast<const long long*>(pair_off), inter_out);
    count_launch();
    return check_cuda(cudaGetLastError(), "mask pair launch");
}
