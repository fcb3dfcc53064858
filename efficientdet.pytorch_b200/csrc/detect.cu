// Inference post-processing on the device: box decode + clip + per-anchor class max + score
// threshold + sort + greedy NMS, for a batch of B images.  Every stage covers the whole batch in
// one set of launches, and the per-image counts stay in device memory, so the launches can be
// captured in a CUDA graph.
// Reference: models/module.py:24-49 (BBoxTransform), :57-67 (ClipBoxes),
//            models/efficientdet.py:70-86 (threshold, nms, gather), torchvision.ops.nms.
// Bit-exactness rules (the keep-set must equal torchvision's): fp32 IoU from separately rounded
// ops (no FMA contraction), suppress iff IoU > thr compared in double, candidates ordered by
// score descending with ties broken by lower anchor index (== stable sort of the masked list).
#include "bitonic.cuh"

namespace effdet {

__device__ __forceinline__ uint32_t float_order(float f) {  // monotone float -> uint32
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// one warp per anchor (coalesced over classes), blockIdx.y = image; anchors >= A emit sentinel keys
__global__ void __launch_bounds__(256) detect_candidates_kernel(const float* __restrict__ cls, const float* __restrict__ reg,
                                                                const float* __restrict__ anchors, float* __restrict__ boxes,
                                                                float* __restrict__ scores, int32_t* __restrict__ classes,
                                                                uint64_t* __restrict__ keys, int32_t* __restrict__ count,
                                                                int A, int K, int npad, float img_w, float img_h,
                                                                float threshold) {
    const int lane = threadIdx.x & 31;
    const int a = blockIdx.x * 8 + (threadIdx.x >> 5);
    const long long b = blockIdx.y;
    if (a >= npad) return;
    keys += b * npad;
    if (a >= A) {
        if (lane == 0) keys[a] = ~0ull;
        return;
    }
    cls += b * A * K;
    float best = -INFINITY;
    int arg = 0x7fffffff;
    for (int k = lane; k < K; k += 32) {
        const float v = __ldg(cls + (long long)a * K + k);
        if (v > best) { best = v; arg = k; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
        if (ov > best || (ov == best && oa < arg)) { best = ov; arg = oa; }
    }
    if (lane != 0) return;
    const float4 an = ldg4(anchors + (long long)a * 4);
    const float4 d = ldg4(reg + (b * A + a) * 4);
    const float w = __fsub_rn(an.z, an.x), h = __fsub_rn(an.w, an.y);
    const float cx = __fadd_rn(an.x, __fmul_rn(0.5f, w)), cy = __fadd_rn(an.y, __fmul_rn(0.5f, h));
    const float dx = __fadd_rn(__fmul_rn(d.x, 0.1f), 0.f), dy = __fadd_rn(__fmul_rn(d.y, 0.1f), 0.f);
    const float dw = __fadd_rn(__fmul_rn(d.z, 0.2f), 0.f), dh = __fadd_rn(__fmul_rn(d.w, 0.2f), 0.f);
    const float pcx = __fadd_rn(cx, __fmul_rn(dx, w)), pcy = __fadd_rn(cy, __fmul_rn(dy, h));
    const float pw = __fmul_rn(expf(dw), w), ph = __fmul_rn(expf(dh), h);
    float x1 = __fsub_rn(pcx, __fmul_rn(0.5f, pw)), y1 = __fsub_rn(pcy, __fmul_rn(0.5f, ph));
    float x2 = __fadd_rn(pcx, __fmul_rn(0.5f, pw)), y2 = __fadd_rn(pcy, __fmul_rn(0.5f, ph));
    x1 = fmaxf(x1, 0.f); y1 = fmaxf(y1, 0.f);
    x2 = fminf(x2, img_w); y2 = fminf(y2, img_h);
    st4(boxes + (b * A + a) * 4, make_float4(x1, y1, x2, y2));
    scores[b * A + a] = best;
    classes[b * A + a] = arg;
    if (best > threshold) {
        keys[a] = ((uint64_t)(~float_order(best)) << 32) | (uint32_t)a;
        atomicAdd(count + b, 1);
    } else {
        keys[a] = ~0ull;
    }
}

// ---- bitonic sort of 64-bit keys (ascending) in independent segments of `seg` keys (a power of two) ----
// The keys of all segments form one array; every compare-exchange stays inside its segment because j < k <= seg.
// The direction of stage k comes from the index inside the segment: at k == seg the global index would alternate it
// from one segment to the next.
constexpr int kChunk = 2048;

__device__ __forceinline__ void cmpswap(uint64_t& a, uint64_t& b, bool asc) {
    if ((a > b) == asc) { const uint64_t t = a; a = b; b = t; }
}

__device__ __forceinline__ bool bitonic_asc(int i, int seg, int k) { return ((i & (seg - 1)) & k) == 0; }

// sorts every aligned chunk (stages k = 2 .. chunk); chunk <= seg
__global__ void __launch_bounds__(1024) bitonic_chunk_sort_kernel(uint64_t* __restrict__ keys, int chunk, int seg) {
    extern __shared__ uint64_t sk[];
    const int base = blockIdx.x * chunk;
    for (int i = threadIdx.x; i < chunk; i += blockDim.x) sk[i] = keys[base + i];
    __syncthreads();
    for (int k = 2; k <= chunk; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int t = threadIdx.x; t < chunk / 2; t += blockDim.x) {
                const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
                cmpswap(sk[i], sk[i | j], bitonic_asc(base + i, seg, k));
            }
            __syncthreads();
        }
    }
    for (int i = threadIdx.x; i < chunk; i += blockDim.x) keys[base + i] = sk[i];
}

__global__ void __launch_bounds__(256) bitonic_global_step_kernel(uint64_t* __restrict__ keys, int n, int seg, int k, int j) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n / 2) return;
    const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
    const bool asc = bitonic_asc(i, seg, k);
    uint64_t a = keys[i], b = keys[i | j];
    if ((a > b) == asc) { keys[i] = b; keys[i | j] = a; }
}

// finishes stage k inside each chunk: j = chunk/2 .. 1
__global__ void __launch_bounds__(1024) bitonic_chunk_merge_kernel(uint64_t* __restrict__ keys, int chunk, int seg, int k) {
    extern __shared__ uint64_t sk[];
    const int base = blockIdx.x * chunk;
    for (int i = threadIdx.x; i < chunk; i += blockDim.x) sk[i] = keys[base + i];
    __syncthreads();
    for (int j = chunk >> 1; j > 0; j >>= 1) {
        for (int t = threadIdx.x; t < chunk / 2; t += blockDim.x) {
            const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
            cmpswap(sk[i], sk[i | j], bitonic_asc(base + i, seg, k));
        }
        __syncthreads();
    }
    for (int i = threadIdx.x; i < chunk; i += blockDim.x) keys[base + i] = sk[i];
}

__device__ __forceinline__ bool iou_gt(const float4 a, const float4 b, double thr) {
    const float left = fmaxf(a.x, b.x), right = fminf(a.z, b.z);
    const float top = fmaxf(a.y, b.y), bottom = fminf(a.w, b.w);
    const float width = fmaxf(__fsub_rn(right, left), 0.f), height = fmaxf(__fsub_rn(bottom, top), 0.f);
    // disjoint boxes (the overwhelming majority of pairs): inter == 0 -> IoU is 0 (or 0/0 = NaN): never > thr for thr >= 0,
    // so the exact division below is skipped; the result is unchanged
    if ((width <= 0.f || height <= 0.f) && thr >= 0.0) return false;
    const float inter = __fmul_rn(width, height);
    const float sa = __fmul_rn(__fsub_rn(a.z, a.x), __fsub_rn(a.w, a.y));
    const float sb = __fmul_rn(__fsub_rn(b.z, b.x), __fsub_rn(b.w, b.y));
    const float ovr = __fdiv_rn(inter, __fsub_rn(__fadd_rn(sa, sb), inter));
    return (double)ovr > thr;
}

// Candidates NMS works on in image b: count[b], or 0 when count[b] > cap (overflow).
__device__ __forceinline__ int nms_candidates(const int32_t* count, int b, int cap) {
    const int n = count[b];
    return n > cap ? 0 : n;
}

// Persistent over the upper-triangle 64x64 tiles of all B images, numbered image by image and row by row inside an
// image (row rb holds tiles cb = rb .. cw_b-1, cw_b = ceil(n_b/64)).  The grid depends on B and cap only.  Each CTA
// walks that numbering forward as its tile index grows, so the walk costs O(B + rows) per CTA in total.
// mask[b][i][cb] bit j set  <=>  sorted box (64*cb + j) of image b is suppressed by its sorted box i; row stride ceil(cap/64).
__global__ void __launch_bounds__(64) nms_mask_kernel(const float* __restrict__ boxes, const uint64_t* __restrict__ keys,
                                                      const int32_t* __restrict__ count, int B, int A, int npad, int cap,
                                                      double thr, uint64_t* __restrict__ mask) {
    __shared__ float4 cbx[64];
    const int cw_cap = (cap + 63) / 64;
    int b = 0, n = nms_candidates(count, 0, cap), cw = (n + 63) / 64;
    long long img_base = 0, img_tiles = (long long)cw * (cw + 1) / 2;   // first tile of image b, tiles of image b
    int rb = 0;
    long long row_base = 0;                                            // first tile of row rb, relative to img_base
    for (long long t = blockIdx.x;; t += gridDim.x) {
        while (t >= img_base + img_tiles) {
            img_base += img_tiles;
            if (++b >= B) return;
            n = nms_candidates(count, b, cap);
            cw = (n + 63) / 64;
            img_tiles = (long long)cw * (cw + 1) / 2;
            rb = 0;
            row_base = 0;
        }
        const long long local = t - img_base;
        while (local >= row_base + (cw - rb)) {
            row_base += cw - rb;
            ++rb;
        }
        const int cb = rb + (int)(local - row_base);
        const uint64_t* kb = keys + (long long)b * npad;
        const float* bx = boxes + (long long)b * A * 4;
        const int cj = cb * 64 + threadIdx.x;
        if (cj < n) cbx[threadIdx.x] = ldg4(bx + (long long)(uint32_t)kb[cj] * 4);
        __syncthreads();
        const int i = rb * 64 + threadIdx.x;
        if (i < n) {
            const float4 me = ldg4(bx + (long long)(uint32_t)kb[i] * 4);
            const int csize = min(64, n - cb * 64);
            uint64_t bits = 0;
            if (rb != cb && csize == 64) {             // almost every tile: fixed trip count, constant bit positions
#pragma unroll 8
                for (int j = 0; j < 64; ++j)
                    if (iou_gt(me, cbx[j], thr)) bits |= 1ull << j;
            } else {
                for (int j = (rb == cb ? threadIdx.x + 1 : 0); j < csize; ++j)
                    if (iou_gt(me, cbx[j], thr)) bits |= 1ull << j;
            }
            mask[((long long)b * cap + i) * cw_cap + cb] = bits;
        }
        __syncthreads();
    }
}

// Greedy scan over the sorted candidates, one CTA per image; the `removed` bitmap lives in shared memory.  Candidates are
// consumed 64 at a time: warp 0 resolves the block's internal dependencies from the 64 diagonal mask words (a
// sequential walk over 64 bits, registers + shuffles only), then every thread ORs the rows of the block's survivors
// into its slice of `removed`.  Two CTA barriers per 64 candidates instead of two per kept box: the scan used to be
// 255 ms for the 55 k survivors of a random-weight D7 image.  Result identical to the one-at-a-time scan.
// nkeep[b] = kept boxes, or -1 when count[b] > cap (nothing else is written for that image).
__global__ void __launch_bounds__(1024) nms_scan_kernel(const uint64_t* __restrict__ mask, const uint64_t* __restrict__ keys,
                                                        const int32_t* __restrict__ count, int npad, int cap,
                                                        int32_t* __restrict__ keep_idx, int32_t* __restrict__ nkeep) {
    extern __shared__ uint64_t removed[];
    __shared__ uint64_t keep_bits;
    const int b = blockIdx.x;
    const int n = count[b];
    if (n > cap) {
        if (threadIdx.x == 0) nkeep[b] = -1;
        return;
    }
    const int cw_cap = (cap + 63) / 64;
    mask += (long long)b * cap * cw_cap;
    keys += (long long)b * npad;
    keep_idx += (long long)b * cap;
    const int col_blocks = (n + 63) / 64;
    const int lane = threadIdx.x & 31;
    for (int j = threadIdx.x; j < col_blocks; j += blockDim.x) removed[j] = 0;
    __syncthreads();
    int kept = 0;
    for (int nb = 0; nb < col_blocks; ++nb) {
        if (threadIdx.x < 32) {
            const int i0 = nb * 64 + lane, i1 = i0 + 32;
            const uint64_t d0 = i0 < n ? mask[(long long)i0 * cw_cap + nb] : 0ull;     // bits j > i inside the block
            const uint64_t d1 = i1 < n ? mask[(long long)i1 * cw_cap + nb] : 0ull;
            uint64_t rem = removed[nb], kb = 0;
            const int valid = min(64, n - nb * 64);
#pragma unroll 1
            for (int bit = 0; bit < valid; ++bit) {
                const uint64_t row = __shfl_sync(0xffffffffu, bit < 32 ? d0 : d1, bit & 31);
                if (!((rem >> bit) & 1ull)) {
                    kb |= 1ull << bit;
                    rem |= row;
                }
            }
            if (lane == 0) keep_bits = kb;
        }
        __syncthreads();
        const uint64_t kb = keep_bits;
        if (threadIdx.x < 64 && ((kb >> threadIdx.x) & 1ull))
            keep_idx[kept + __popcll(kb & ((1ull << threadIdx.x) - 1ull))] = (int32_t)(uint32_t)keys[nb * 64 + threadIdx.x];
        for (int j = nb + 1 + threadIdx.x; j < col_blocks; j += blockDim.x) {
            uint64_t acc = 0, bits = kb;
            while (bits) {
                const int bit = __ffsll((long long)bits) - 1;
                bits &= bits - 1;
                acc |= mask[(long long)(nb * 64 + bit) * cw_cap + j];
            }
            removed[j] |= acc;
        }
        kept += __popcll(kb);
        __syncthreads();
    }
    if (threadIdx.x == 0) nkeep[b] = kept;
}

// row i of image b (blockIdx.y): the i-th kept detection, zero from nkeep[b] on
__global__ void gather_detections_kernel(const float* __restrict__ boxes, const float* __restrict__ scores,
                                         const int32_t* __restrict__ classes, const int32_t* __restrict__ keep_idx,
                                         const int32_t* __restrict__ nkeep, int A, int cap, float* __restrict__ out_scores,
                                         long long* __restrict__ out_classes, float* __restrict__ out_boxes) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const long long b = blockIdx.y;
    if (i >= cap) return;
    const long long o = b * cap + i;
    if (i < nkeep[b]) {
        const long long a = b * A + keep_idx[o];
        out_scores[o] = scores[a];
        out_classes[o] = (long long)classes[a];
        st4(out_boxes + o * 4, ldg4(boxes + a * 4));
    } else {
        out_scores[o] = 0.f;
        out_classes[o] = 0;
        st4(out_boxes + o * 4, f4zero());
    }
}

constexpr size_t kScanSmemLimit = 200 * 1024;

static int candidates_launch(const float* cls, const float* reg, const float* anchors, float* boxes, float* scores,
                             int32_t* classes, uint64_t* keys, int32_t* count, int B, int A, int K, int npad, float img_w,
                             float img_h, float threshold, cudaStream_t st) {
    cudaError_t e = cudaMemsetAsync(count, 0, (size_t)B * sizeof(int32_t), st);
    if (e != cudaSuccess) return fail(EFFDET_ERR_LAUNCH, "detect_candidates: memset: %s", cudaGetErrorString(e));
    detect_candidates_kernel<<<dim3(cdiv(npad, 8), B), 256, 0, st>>>(cls, reg, anchors, boxes, scores, classes, keys, count, A,
                                                                    K, npad, img_w, img_h, threshold);
    int s = launch_status("detect_candidates_kernel");
    if (s) return s;
    // sort every image's segment ascending: best candidates first, sentinels last
    return bitonic_sort_launch(keys, B * npad, npad, st);
}

int bitonic_sort_launch(uint64_t* keys, int n, int seg, cudaStream_t st) {
    int s;
    const int chunk = seg < kChunk ? seg : kChunk;
    if (chunk >= 2) {
        bitonic_chunk_sort_kernel<<<n / chunk, 1024, chunk * sizeof(uint64_t), st>>>(keys, chunk, seg);
        if ((s = launch_status("bitonic_chunk_sort_kernel"))) return s;
    }
    for (int k = chunk * 2; k <= seg; k <<= 1) {
        for (int j = k >> 1; j >= chunk; j >>= 1) {
            bitonic_global_step_kernel<<<cdiv(n / 2, 256), 256, 0, st>>>(keys, n, seg, k, j);
            if ((s = launch_status("bitonic_global_step_kernel"))) return s;
        }
        bitonic_chunk_merge_kernel<<<n / chunk, 1024, chunk * sizeof(uint64_t), st>>>(keys, chunk, seg, k);
        if ((s = launch_status("bitonic_chunk_merge_kernel"))) return s;
    }
    return EFFDET_OK;
}

static int nms_launch(const float* boxes, const uint64_t* keys, const int32_t* count, int B, int A, int npad, int cap,
                      double iou_threshold, uint64_t* mask_ws, int32_t* keep_idx, int32_t* nkeep, cudaStream_t st) {
    const long long cw = cdiv(cap, 64);
    const long long tiles = (long long)B * (cw * (cw + 1) / 2);        // upper bound: every image at `cap` candidates
    const int grid = (int)(tiles < (long long)num_sms() * 32 ? tiles : (long long)num_sms() * 32);
    nms_mask_kernel<<<grid, 64, 0, st>>>(boxes, keys, count, B, A, npad, cap, iou_threshold, mask_ws);
    int s = launch_status("nms_mask_kernel");
    if (s) return s;
    const size_t smem = (size_t)cw * sizeof(uint64_t);
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(nms_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return fail(EFFDET_ERR_LAUNCH, "nms: smem opt-in: %s", cudaGetErrorString(e));
    }
    nms_scan_kernel<<<B, 1024, smem, st>>>(mask_ws, keys, count, npad, cap, keep_idx, nkeep);
    return launch_status("nms_scan_kernel");
}

static int gather_launch(const float* boxes, const float* scores, const int32_t* classes, const int32_t* keep_idx,
                         const int32_t* nkeep, int B, int A, int cap, float* out_scores, int64_t* out_classes,
                         float* out_boxes, cudaStream_t st) {
    gather_detections_kernel<<<dim3(cdiv(cap, 256), B), 256, 0, st>>>(boxes, scores, classes, keep_idx, nkeep, A, cap,
                                                                      out_scores, (long long*)out_classes, out_boxes);
    return launch_status("gather_detections_kernel");
}

}  // namespace effdet

using namespace effdet;

extern "C" int effdet_detect_candidates_batch(const float* cls, const float* reg, const float* anchors, float* boxes,
                                              float* scores, int32_t* classes, uint64_t* keys, int32_t* count, int B, int A,
                                              int K, int npad, float img_w, float img_h, float threshold, int device,
                                              effdet_stream_t stream) {
    EFFDET_REQUIRE(cls && reg && anchors && boxes && scores && classes && keys && count, "detect_candidates_batch: null tensor");
    EFFDET_REQUIRE(B >= 1 && B <= 65535, "detect_candidates_batch: B=%d must be in [1, 65535]", B);
    EFFDET_REQUIRE(A > 0 && K > 0 && npad >= A && (npad & (npad - 1)) == 0,
                   "detect_candidates_batch: npad=%d must be a power of two >= A=%d (K=%d > 0)", npad, A, K);
    EFFDET_REQUIRE((long long)B * npad <= (1ll << 30), "detect_candidates_batch: B*npad = %lld keys is too many",
                   (long long)B * npad);
    EFFDET_REQUIRE(aligned16(reg) && aligned16(anchors) && aligned16(boxes), "detect_candidates_batch: alignment");
    EFFDET_DEVICE(device);
    return candidates_launch(cls, reg, anchors, boxes, scores, classes, keys, count, B, A, K, npad, img_w, img_h, threshold,
                             (cudaStream_t)stream);
}

extern "C" int effdet_nms_batch(const float* boxes, const uint64_t* keys, const int32_t* count, int B, int A, int npad,
                                int cap, double iou_threshold, uint64_t* mask_ws, int32_t* keep_idx, int32_t* nkeep,
                                int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(boxes && keys && count && mask_ws && keep_idx && nkeep, "nms_batch: null tensor");
    EFFDET_REQUIRE(B >= 1, "nms_batch: B=%d must be >= 1", B);
    EFFDET_REQUIRE(A > 0 && npad >= A && (npad & (npad - 1)) == 0, "nms_batch: npad=%d must be a power of two >= A=%d", npad, A);
    EFFDET_REQUIRE(cap >= 1 && cap <= A, "nms_batch: cap=%d must be in [1, A=%d]", cap, A);
    EFFDET_REQUIRE((size_t)cdiv(cap, 64) * sizeof(uint64_t) <= kScanSmemLimit,
                   "nms_batch: cap=%d is too large for the scan bitmap (%zu bytes of shared memory at most)", cap, kScanSmemLimit);
    EFFDET_REQUIRE(aligned16(boxes), "nms_batch: alignment");
    EFFDET_DEVICE(device);
    return nms_launch(boxes, keys, count, B, A, npad, cap, iou_threshold, mask_ws, keep_idx, nkeep, (cudaStream_t)stream);
}

extern "C" int effdet_gather_detections_batch(const float* boxes, const float* scores, const int32_t* classes,
                                              const int32_t* keep_idx, const int32_t* nkeep, int B, int A, int cap,
                                              float* out_scores, int64_t* out_classes, float* out_boxes, int device,
                                              effdet_stream_t stream) {
    EFFDET_REQUIRE(boxes && scores && classes && keep_idx && nkeep && out_scores && out_classes && out_boxes,
                   "gather_detections_batch: null tensor");
    EFFDET_REQUIRE(B >= 1 && B <= 65535, "gather_detections_batch: B=%d must be in [1, 65535]", B);
    EFFDET_REQUIRE(A > 0 && cap >= 1 && cap <= A, "gather_detections_batch: cap=%d must be in [1, A=%d]", cap, A);
    EFFDET_REQUIRE(aligned16(boxes) && aligned16(out_boxes), "gather_detections_batch: alignment");
    EFFDET_DEVICE(device);
    return gather_launch(boxes, scores, classes, keep_idx, nkeep, B, A, cap, out_scores, out_classes, out_boxes,
                         (cudaStream_t)stream);
}
