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

// BBoxTransform + ClipBoxes of one anchor: separately rounded fp32 ops, the reference's order of operations
__device__ __forceinline__ float4 decode_box(const float4 an, const float4 d, float img_w, float img_h) {
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
    return make_float4(x1, y1, x2, y2);
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
    st4(boxes + (b * A + a) * 4, decode_box(an, d, img_w, img_h));
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

// Greedy NMS in column chunks of `chunk` sorted candidates.  Chunk c of image b covers its sorted candidates
// [base, base + chunk) with base = c * chunk.  Candidate j is kept iff no kept i < j has IoU > thr: the cross step decides
// that against the boxes kept by earlier chunks, the mask + scan inside the chunk.  Every kernel calls
// iou_gt(earlier box, later box), so the keep set and its order do not depend on `chunk`.  With chunk = cap there is one
// chunk and no cross step: the mask + scan over all candidates.
//
// Candidates of image b inside the chunk at `base`: 0 when count[b] > cap (overflow) or when the image ends before it.
__device__ __forceinline__ int nms_candidates(const int32_t* count, int b, int cap, int base, int chunk) {
    const int n = count[b];
    return n > cap || n <= base ? 0 : min(n - base, chunk);
}

constexpr int kCrossThreads = 256;

// Cross step of the chunk at `base` > 0.  CTA (x, y, b) tests the 64 candidates of tile y against every gridDim.x-th
// tile of kCrossThreads boxes among the nkeep[b] that image b kept in earlier chunks (read through keep_idx, one kept box
// per thread) and ORs the candidates they suppress into removed[b][y].  A candidate already removed is not tested again,
// and a CTA stops once its whole tile is removed.  removed[b] is zero on entry: the scan of the previous chunk cleared it.
// kClasses: a kept box suppresses only candidates of its own class (classes [B,A], per-class NMS); otherwise classes is
// unused.
template <bool kClasses>
__global__ void __launch_bounds__(kCrossThreads) nms_cross_kernel(const float* __restrict__ boxes,
                                                                  const uint64_t* __restrict__ keys,
                                                                  const int32_t* __restrict__ count, int A, int npad,
                                                                  int cap, int base, int chunk, double thr,
                                                                  const int32_t* __restrict__ keep_idx,
                                                                  const int32_t* __restrict__ nkeep, uint64_t* removed,
                                                                  const int32_t* __restrict__ classes) {
    __shared__ float4 cbx[64];
    __shared__ int32_t ccl[kClasses ? 64 : 1];
    __shared__ uint64_t done;
    const int b = blockIdx.z;
    const int valid = min(64, nms_candidates(count, b, cap, base, chunk) - (int)blockIdx.y * 64);
    if (valid <= 0) return;
    const uint64_t valid_bits = valid == 64 ? ~0ull : (1ull << valid) - 1ull;
    const float* bx = boxes + (long long)b * A * 4;
    if (threadIdx.x < valid) {
        const uint32_t a = (uint32_t)keys[(long long)b * npad + base + blockIdx.y * 64 + threadIdx.x];
        cbx[threadIdx.x] = ldg4(bx + (long long)a * 4);
        if constexpr (kClasses) ccl[threadIdx.x] = classes[(long long)b * A + a];
    }
    uint64_t* word = removed + (long long)b * ((chunk + 63) / 64) + blockIdx.y;
    const int nk = nkeep[b];
    keep_idx += (long long)b * cap;
    for (int k0 = blockIdx.x * kCrossThreads; k0 < nk; k0 += gridDim.x * kCrossThreads) {
        __syncthreads();                       // cbx is stored, and every thread has read the previous `done`
        if (threadIdx.x == 0) done = *(volatile uint64_t*)word;
        __syncthreads();
        const uint64_t live = ~done & valid_bits;
        if (!live) break;
        uint64_t bits = 0;
        const int k = k0 + threadIdx.x;
        if (k < nk) {
            const float4 me = ldg4(bx + (long long)keep_idx[k] * 4);
            if constexpr (kClasses) {
                const int32_t mc = classes[(long long)b * A + keep_idx[k]];
                for (uint64_t m = live; m; m &= m - 1) {
                    const int j = __ffsll((long long)m) - 1;
                    if (ccl[j] == mc && iou_gt(me, cbx[j], thr)) bits |= 1ull << j;
                }
            } else {
                for (uint64_t m = live; m; m &= m - 1) {      // CTA-uniform: no divergence from the removed bits
                    const int j = __ffsll((long long)m) - 1;
                    if (iou_gt(me, cbx[j], thr)) bits |= 1ull << j;
                }
            }
        }
        const uint32_t lo = __reduce_or_sync(0xffffffffu, (uint32_t)bits);
        const uint32_t hi = __reduce_or_sync(0xffffffffu, (uint32_t)(bits >> 32));
        if ((threadIdx.x & 31) == 0 && (lo | hi))
            atomicOr((unsigned long long*)word, ((unsigned long long)hi << 32) | lo);
    }
}

// Persistent over the upper-triangle 64x64 tiles of the chunk at `base` in all B images, numbered image by image and row
// by row inside an image (row rb holds tiles cb = rb .. cw_b-1, cw_b = ceil(n_b/64), n_b the image's candidates in the
// chunk).  The grid depends on B and chunk only.  Each CTA walks that numbering forward as its tile index grows, so the
// walk costs O(B + rows) per CTA in total.
// mask[b][i][cb] bit j set  <=>  sorted box base + 64*cb + j of image b is suppressed by its sorted box base + i; row
// stride ceil(chunk/64).  removed (null for the first chunk): the cross step's bitmap.  A row whose candidate it removed
// is written as zero without testing, because the scan never uses that row.
// kClasses: a box suppresses only boxes of its own class (classes [B,A]); otherwise classes is unused.
template <bool kClasses>
__global__ void __launch_bounds__(64) nms_mask_kernel(const float* __restrict__ boxes, const uint64_t* __restrict__ keys,
                                                      const int32_t* __restrict__ count, int B, int A, int npad, int cap,
                                                      int base, int chunk, double thr, const uint64_t* __restrict__ removed,
                                                      uint64_t* __restrict__ mask, const int32_t* __restrict__ classes) {
    __shared__ float4 cbx[64];
    __shared__ int32_t ccl[kClasses ? 64 : 1];
    const int cw_chunk = (chunk + 63) / 64;
    int b = 0, n = nms_candidates(count, 0, cap, base, chunk), cw = (n + 63) / 64;
    long long img_base = 0, img_tiles = (long long)cw * (cw + 1) / 2;   // first tile of image b, tiles of image b
    int rb = 0;
    long long row_base = 0;                                            // first tile of row rb, relative to img_base
    for (long long t = blockIdx.x;; t += gridDim.x) {
        while (t >= img_base + img_tiles) {
            img_base += img_tiles;
            if (++b >= B) return;
            n = nms_candidates(count, b, cap, base, chunk);
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
        const uint64_t* kb = keys + (long long)b * npad + base;
        const float* bx = boxes + (long long)b * A * 4;
        const int cj = cb * 64 + threadIdx.x;
        if (cj < n) {
            cbx[threadIdx.x] = ldg4(bx + (long long)(uint32_t)kb[cj] * 4);
            if constexpr (kClasses) ccl[threadIdx.x] = classes[(long long)b * A + (uint32_t)kb[cj]];
        }
        __syncthreads();
        const int i = rb * 64 + threadIdx.x;
        if (i < n) {
            const float4 me = ldg4(bx + (long long)(uint32_t)kb[i] * 4);
            const int csize = min(64, n - cb * 64);
            uint64_t bits = 0;
            if (removed && ((removed[(long long)b * cw_chunk + rb] >> threadIdx.x) & 1ull)) {
                // suppressed by a box of an earlier chunk
            } else if constexpr (kClasses) {
                const int32_t mc = classes[(long long)b * A + (uint32_t)kb[i]];
                for (int j = (rb == cb ? threadIdx.x + 1 : 0); j < csize; ++j)
                    if (ccl[j] == mc && iou_gt(me, cbx[j], thr)) bits |= 1ull << j;
            } else if (rb != cb && csize == 64) {      // almost every tile: fixed trip count, constant bit positions
#pragma unroll 8
                for (int j = 0; j < 64; ++j)
                    if (iou_gt(me, cbx[j], thr)) bits |= 1ull << j;
            } else {
                for (int j = (rb == cb ? threadIdx.x + 1 : 0); j < csize; ++j)
                    if (iou_gt(me, cbx[j], thr)) bits |= 1ull << j;
            }
            mask[((long long)b * chunk + i) * cw_chunk + cb] = bits;
        }
        __syncthreads();
    }
}

// Greedy scan over the sorted candidates of the chunk at `base`, one CTA per image; the `removed` bitmap lives in shared
// memory.  Candidates are consumed 64 at a time: warp 0 resolves the block's internal dependencies from the 64 diagonal
// mask words (a sequential walk over 64 bits, registers + shuffles only), then every thread ORs the rows of the block's
// survivors into its slice of `removed`.  Two CTA barriers per 64 candidates instead of two per kept box: the scan used
// to be 255 ms for the 55 k survivors of a random-weight D7 image.  Result identical to the one-at-a-time scan.
// The first chunk starts from an empty bitmap and keep list; a later one starts from the cross step's bitmap
// removed_g[b] and appends at keep_idx[b][nkeep[b]].  The scan clears removed_g[b] for the next chunk's cross step;
// removed_g is null when there is one chunk.
// nkeep[b] = kept boxes, or -1 when count[b] > cap (nothing else is written for that image).
__global__ void __launch_bounds__(1024) nms_scan_kernel(const uint64_t* __restrict__ mask, const uint64_t* __restrict__ keys,
                                                        const int32_t* __restrict__ count, int npad, int cap, int base,
                                                        int chunk, uint64_t* __restrict__ removed_g,
                                                        int32_t* __restrict__ keep_idx, int32_t* __restrict__ nkeep) {
    extern __shared__ uint64_t removed[];
    __shared__ uint64_t keep_bits;
    const int b = blockIdx.x;
    const int total = count[b];
    if (total > cap) {
        if (threadIdx.x == 0 && base == 0) nkeep[b] = -1;
        return;
    }
    if (base > 0 && total <= base) return;                          // the image ended in an earlier chunk
    const int n = min(total - base, chunk);
    const int cw_chunk = (chunk + 63) / 64;
    mask += (long long)b * chunk * cw_chunk;
    keys += (long long)b * npad + base;
    keep_idx += (long long)b * cap;
    const int col_blocks = (n + 63) / 64;
    const int lane = threadIdx.x & 31;
    int kept = base > 0 ? nkeep[b] : 0;
    for (int j = threadIdx.x; j < col_blocks; j += blockDim.x) {
        uint64_t r = 0;
        if (removed_g) {
            uint64_t* w = removed_g + (long long)b * cw_chunk + j;
            if (base > 0) r = *w;
            *w = 0;
        }
        removed[j] = r;
    }
    __syncthreads();
    for (int nb = 0; nb < col_blocks; ++nb) {
        if (threadIdx.x < 32) {
            const int i0 = nb * 64 + lane, i1 = i0 + 32;
            const uint64_t d0 = i0 < n ? mask[(long long)i0 * cw_chunk + nb] : 0ull;   // bits j > i inside the block
            const uint64_t d1 = i1 < n ? mask[(long long)i1 * cw_chunk + nb] : 0ull;
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
                acc |= mask[(long long)(nb * 64 + bit) * cw_chunk + j];
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

// Workspace of the chunked NMS: the chunk's mask [B][chunk][ceil(chunk/64)], then (more than one chunk) the cross step's
// bitmaps [B][ceil(chunk/64)].  With one chunk this is effdet_nms_batch's mask [B][cap][ceil(cap/64)].
static long long nms_workspace_words(int B, int cap, int chunk) {
    const long long cw = cdiv(chunk, 64);
    return (long long)B * (chunk * cw + (cdiv(cap, chunk) > 1 ? cw : 0));
}

// ceil(cap/chunk) chunks, each a fixed set of launches (cross step from the second chunk on, mask, scan): the sequence
// depends on B, cap and chunk only, so it can be captured.  Launches for a chunk past an image's count exit at once.
// classes [B,A] non-null: per-class NMS (a pair of candidates counts only when their classes are equal).  Every class's
// candidates, taken in the global (score, anchor) order, are that class's own sorted list, so the greedy pass over the
// global order keeps exactly the per-class keep sets, already merged in output order.
static int nms_launch(const float* boxes, const uint64_t* keys, const int32_t* count, int B, int A, int npad, int cap,
                      int chunk, double iou_threshold, uint64_t* ws, int32_t* keep_idx, int32_t* nkeep, cudaStream_t st,
                      const int32_t* classes = nullptr) {
    const long long cw = cdiv(chunk, 64);
    const int chunks = cdiv(cap, chunk);
    uint64_t* mask = ws;
    uint64_t* removed = chunks > 1 ? ws + (long long)B * chunk * cw : nullptr;
    const long long tiles = (long long)B * (cw * (cw + 1) / 2);        // upper bound: every image at `chunk` candidates
    const int mask_grid = (int)(tiles < (long long)num_sms() * 32 ? tiles : (long long)num_sms() * 32);
    const size_t smem = (size_t)cw * sizeof(uint64_t);
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(nms_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return fail(EFFDET_ERR_LAUNCH, "nms: smem opt-in: %s", cudaGetErrorString(e));
    }
    int s;
    for (int c = 0; c < chunks; ++c) {
        const int base = c * chunk;
        if (c > 0) {
            // kept boxes before this chunk: at most `base`.  Enough CTAs along the kept list to fill the SMs about once
            // with the (candidate tile, image) pairs; each strides over the kept tiles.
            const int kept_tiles = cdiv(base, kCrossThreads);
            const int fill = cdiv((long long)num_sms() * (2048 / kCrossThreads), cw * B);
            const int gx = kept_tiles < fill ? kept_tiles : fill;
            if (classes)
                nms_cross_kernel<true><<<dim3(gx, (unsigned)cw, B), kCrossThreads, 0, st>>>(
                    boxes, keys, count, A, npad, cap, base, chunk, iou_threshold, keep_idx, nkeep, removed, classes);
            else
                nms_cross_kernel<false><<<dim3(gx, (unsigned)cw, B), kCrossThreads, 0, st>>>(
                    boxes, keys, count, A, npad, cap, base, chunk, iou_threshold, keep_idx, nkeep, removed, nullptr);
            if ((s = launch_status("nms_cross_kernel"))) return s;
        }
        if (classes)
            nms_mask_kernel<true><<<mask_grid, 64, 0, st>>>(boxes, keys, count, B, A, npad, cap, base, chunk,
                                                            iou_threshold, c > 0 ? removed : nullptr, mask, classes);
        else
            nms_mask_kernel<false><<<mask_grid, 64, 0, st>>>(boxes, keys, count, B, A, npad, cap, base, chunk,
                                                             iou_threshold, c > 0 ? removed : nullptr, mask, nullptr);
        if ((s = launch_status("nms_mask_kernel"))) return s;
        nms_scan_kernel<<<B, 1024, smem, st>>>(mask, keys, count, npad, cap, base, chunk, removed, keep_idx, nkeep);
        if ((s = launch_status("nms_scan_kernel"))) return s;
    }
    return EFFDET_OK;
}

static int gather_launch(const float* boxes, const float* scores, const int32_t* classes, const int32_t* keep_idx,
                         const int32_t* nkeep, int B, int A, int cap, float* out_scores, int64_t* out_classes,
                         float* out_boxes, cudaStream_t st) {
    gather_detections_kernel<<<dim3(cdiv(cap, 256), B), 256, 0, st>>>(boxes, scores, classes, keep_idx, nkeep, A, cap,
                                                                      out_scores, (long long*)out_classes, out_boxes);
    return launch_status("gather_detections_kernel");
}


// ---- multi-label candidates: the top_k best (anchor a, class k) pairs p = a*K + k of each image -------------------------
// Every pair with cls > threshold has the unique key (~float_order(score) << 32) | p; the k' = min(top_k, A*K) smallest
// keys are the pairs in (score descending, p ascending) order.  The k'-th smallest key is found by a radix select over
// its 64 bits in six digits, most significant first: each pass histograms one digit of the keys whose higher digits
// equal the ones resolved so far (per image, in the workspace), then one CTA per image picks the digit that holds the
// k'-th key.  An image is decided as soon as the bin it picks is taken whole (at the latest after the sixth digit, when
// the bin is one key); its later passes exit at once, and an image with at most k' pairs above the threshold is decided
// by the first pass.  The compaction then takes every key whose resolved digits are at most the picked ones (exactly
// count[b] keys), the segmented bitonic sort orders them, and the gather writes slot i's decoded box, score and class
// and rewrites its key as (score bits << 32) | i: effdet_detect_candidates_batch's format with the slots as anchors.
// cls is read once per histogram pass an undecided image takes part in (1 to 6) and once by the compaction; all
// counts are integer, so the result does not depend on the order of the atomics.
constexpr int kTopkDigits = 6;
constexpr int kTopkWidth[kTopkDigits] = {11, 11, 10, 11, 11, 10};
constexpr int kTopkBins = 2048;
constexpr int kTopkThreads = 256;

struct TopkState {                 // per image, after the histograms; zero at the start
    unsigned long long prefix;     // the resolved high bits of the k'-th key
    int resolved;                  // bits resolved: 0 (with done: take every pair above the threshold) .. 64
    uint32_t need;                 // keys still to take among those whose resolved bits equal prefix
    int done;                      // the keys to take are those whose resolved bits are <= prefix
    uint32_t taken;                // the compaction's slot counter
    uint32_t pad[2];
};
static_assert(sizeof(TopkState) == 32, "TopkState layout");

__device__ __forceinline__ uint64_t pair_key(float v, uint32_t p) {
    return ((uint64_t)(~float_order(v)) << 32) | p;
}

// histogram of digit (resolved, width) over the keys of image blockIdx.y whose resolved bits equal the prefix
__global__ void __launch_bounds__(kTopkThreads) topk_hist_kernel(const float* __restrict__ cls, long long N,
                                                                 float threshold, int resolved, int width,
                                                                 uint32_t* __restrict__ hist,
                                                                 const TopkState* __restrict__ state) {
    __shared__ uint32_t h[kTopkBins];
    const int b = blockIdx.y;
    if (state[b].done) return;
    const unsigned long long prefix = state[b].prefix;
    for (int i = threadIdx.x; i < kTopkBins; i += kTopkThreads) h[i] = 0;
    __syncthreads();
    const float* c = cls + (long long)b * N;
    const int shift = 64 - resolved - width;
    const uint32_t digit = (1u << width) - 1u;
    for (long long p = (long long)blockIdx.x * kTopkThreads + threadIdx.x; p < N; p += (long long)gridDim.x * kTopkThreads) {
        const float v = __ldg(c + p);
        if (!(v > threshold)) continue;
        const uint64_t key = pair_key(v, (uint32_t)p);
        if (resolved && (key >> (64 - resolved)) != prefix) continue;
        atomicAdd(&h[(uint32_t)(key >> shift) & digit], 1u);
    }
    __syncthreads();
    uint32_t* g = hist + (long long)b * kTopkBins;
    for (int i = threadIdx.x; i < kTopkBins; i += kTopkThreads)
        if (h[i]) atomicAdd(g + i, h[i]);
}

// one CTA of 1024 threads per image, two bins a thread: picks the bin of the k'-th key and clears the histogram.  The
// first pass also sets count[b] and writes the sentinel keys [count[b], kpad).
__global__ void __launch_bounds__(1024) topk_select_kernel(uint32_t* __restrict__ hist, TopkState* __restrict__ state,
                                                           int resolved, int width, int top_k,
                                                           int32_t* __restrict__ count, uint64_t* __restrict__ keys,
                                                           int kpad) {
    __shared__ uint32_t wsum[32];
    const int b = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
    TopkState* st = state + b;
    if (st->done) return;
    uint32_t* h = hist + (long long)b * kTopkBins;
    const uint32_t h0 = h[2 * t], h1 = h[2 * t + 1];
    const uint32_t need = resolved ? st->need : (uint32_t)top_k;
    uint32_t incl = h0 + h1;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    uint32_t before = 0, total = 0;
    for (int w = 0; w < 32; ++w) {
        const uint32_t v = wsum[w];
        before += w < warp ? v : 0;
        total += v;
    }
    const uint32_t excl = before + incl - (h0 + h1);
    h[2 * t] = 0;
    h[2 * t + 1] = 0;
    if (!resolved) {
        const uint32_t n = total < (uint32_t)top_k ? total : (uint32_t)top_k;
        if (t == 0) count[b] = (int32_t)n;
        for (long long i = (long long)n + t; i < kpad; i += 1024) keys[(long long)b * kpad + i] = ~0ull;
        if (total <= (uint32_t)top_k) {
            if (t == 0) st->done = 1;                      // every pair above the threshold is a candidate
            return;
        }
    }
    for (int j = 0; j < 2; ++j) {
        const uint32_t c = j ? h1 : h0, lo = j ? excl + h0 : excl;
        if (lo < need && need <= lo + c) {                 // exactly one bin of the image
            st->prefix = (resolved ? st->prefix << width : 0ull) | (unsigned long long)(2 * t + j);
            st->resolved = resolved + width;
            st->need = need - lo;
            st->done = c == need - lo;
        }
    }
}

// keys whose resolved bits are <= the prefix, into keys[b][0, count[b]) in any order (sorted next)
__global__ void __launch_bounds__(kTopkThreads) topk_compact_kernel(const float* __restrict__ cls, long long N,
                                                                    float threshold, TopkState* __restrict__ state,
                                                                    uint64_t* __restrict__ keys, int kpad) {
    const int b = blockIdx.y, lane = threadIdx.x & 31;
    const unsigned long long prefix = state[b].prefix;
    const int resolved = state[b].resolved;
    const float* c = cls + (long long)b * N;
    uint64_t* kb = keys + (long long)b * kpad;
    for (long long p0 = (long long)blockIdx.x * kTopkThreads; p0 < N; p0 += (long long)gridDim.x * kTopkThreads) {
        const long long p = p0 + threadIdx.x;                    // warp-uniform trip count: the ballot below is safe
        bool take = false;
        uint64_t key = 0;
        if (p < N) {
            const float v = __ldg(c + p);
            key = pair_key(v, (uint32_t)p);
            take = v > threshold && (!resolved || (key >> (64 - resolved)) <= prefix);
        }
        const uint32_t m = __ballot_sync(0xffffffffu, take);
        if (!m) continue;
        uint32_t base = 0;
        if (lane == 0) base = atomicAdd(&state[b].taken, (uint32_t)__popc(m));
        base = __shfl_sync(0xffffffffu, base, 0);
        if (take) kb[base + __popc(m & ((1u << lane) - 1u))] = key;
    }
}

// slot i < count[b]: decode the pair's box and write box, score, class and the slot's key; later slots are zero
__global__ void __launch_bounds__(256) topk_gather_kernel(const float* __restrict__ cls, const float* __restrict__ reg,
                                                          const float* __restrict__ anchors, int A, int K, int kprime,
                                                          int kpad, float img_w, float img_h,
                                                          const int32_t* __restrict__ count, uint64_t* __restrict__ keys,
                                                          float* __restrict__ boxes, float* __restrict__ scores,
                                                          int32_t* __restrict__ classes) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const long long b = blockIdx.y;
    if (i >= kprime) return;
    const long long o = b * kprime + i;
    if (i < count[b]) {
        const uint64_t key = keys[b * kpad + i];
        const uint32_t p = (uint32_t)key;
        const uint32_t a = p / (uint32_t)K;
        st4(boxes + o * 4, decode_box(ldg4(anchors + (long long)a * 4), ldg4(reg + (b * A + a) * 4), img_w, img_h));
        scores[o] = cls[b * A * K + p];
        classes[o] = (int32_t)(p - a * (uint32_t)K);
        keys[b * kpad + i] = (key & 0xffffffff00000000ull) | (uint32_t)i;
    } else {
        st4(boxes + o * 4, f4zero());
        scores[o] = 0.f;
        classes[o] = 0;
    }
}

static long long topk_workspace_bytes(int B) {
    return (long long)B * (kTopkBins * (long long)sizeof(uint32_t) + (long long)sizeof(TopkState));
}

static int topk_launch(const float* cls, const float* reg, const float* anchors, int B, int A, int K, float img_w,
                       float img_h, float threshold, int top_k, int kprime, int kpad, void* ws, float* boxes,
                       float* scores, int32_t* classes, uint64_t* keys, int32_t* count, cudaStream_t st) {
    const long long N = (long long)A * K;
    uint32_t* hist = (uint32_t*)ws;
    TopkState* state = (TopkState*)(hist + (long long)B * kTopkBins);
    cudaError_t e = cudaMemsetAsync(ws, 0, (size_t)topk_workspace_bytes(B), st);
    if (e != cudaSuccess) return fail(EFFDET_ERR_LAUNCH, "detect_topk: memset: %s", cudaGetErrorString(e));
    // about 8 CTAs per SM over the batch, each striding over its image's pairs
    const long long fill = cdiv((long long)num_sms() * 8, B);
    const long long want = cdiv(N, (long long)kTopkThreads * 16);
    const dim3 grid((unsigned)(want < fill ? want : fill), B);
    int s;
    int resolved = 0;
    for (int d = 0; d < kTopkDigits; ++d) {
        topk_hist_kernel<<<grid, kTopkThreads, 0, st>>>(cls, N, threshold, resolved, kTopkWidth[d], hist, state);
        if ((s = launch_status("topk_hist_kernel"))) return s;
        topk_select_kernel<<<B, 1024, 0, st>>>(hist, state, resolved, kTopkWidth[d], top_k, count, keys, kpad);
        if ((s = launch_status("topk_select_kernel"))) return s;
        resolved += kTopkWidth[d];
    }
    topk_compact_kernel<<<grid, kTopkThreads, 0, st>>>(cls, N, threshold, state, keys, kpad);
    if ((s = launch_status("topk_compact_kernel"))) return s;
    if ((s = bitonic_sort_launch(keys, B * kpad, kpad, st))) return s;
    topk_gather_kernel<<<dim3(cdiv(kprime, 256), B), 256, 0, st>>>(cls, reg, anchors, A, K, kprime, kpad, img_w, img_h,
                                                                   count, keys, boxes, scores, classes);
    return launch_status("topk_gather_kernel");
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
    return nms_launch(boxes, keys, count, B, A, npad, cap, cap, iou_threshold, mask_ws, keep_idx, nkeep,
                      (cudaStream_t)stream);
}

#define NMS_CHUNK_LIMITS(fn, B, cap, chunk)                                                                             \
    EFFDET_REQUIRE((B) >= 1 && (B) <= 65535, fn ": B=%d must be in [1, 65535]", (B));                                   \
    EFFDET_REQUIRE((cap) >= 1, fn ": cap=%d must be >= 1", (cap));                                                      \
    EFFDET_REQUIRE((chunk) >= 1 && (chunk) <= (cap) && ((chunk) % 64 == 0 || (chunk) == (cap)),                         \
                   fn ": chunk=%d must be a multiple of 64 in [64, cap=%d], or cap itself", (chunk), (cap));            \
    EFFDET_REQUIRE((size_t)cdiv((chunk), 64) * sizeof(uint64_t) <= kScanSmemLimit,                                      \
                   fn ": chunk=%d is too large for the scan bitmap (%zu bytes of shared memory at most)", (chunk),      \
                   kScanSmemLimit)

extern "C" int64_t effdet_nms_chunked_workspace(int B, int cap, int chunk) {
    NMS_CHUNK_LIMITS("nms_chunked_workspace", B, cap, chunk);
    return nms_workspace_words(B, cap, chunk) * (int64_t)sizeof(uint64_t);
}

extern "C" int effdet_nms_batch_chunked(const float* boxes, const uint64_t* keys, const int32_t* count, int B, int A,
                                        int npad, int cap, int chunk, double iou_threshold, void* workspace,
                                        int64_t workspace_bytes, int32_t* keep_idx, int32_t* nkeep, int device,
                                        effdet_stream_t stream) {
    EFFDET_REQUIRE(boxes && keys && count && workspace && keep_idx && nkeep, "nms_batch_chunked: null tensor");
    NMS_CHUNK_LIMITS("nms_batch_chunked", B, cap, chunk);
    EFFDET_REQUIRE(A > 0 && npad >= A && (npad & (npad - 1)) == 0,
                   "nms_batch_chunked: npad=%d must be a power of two >= A=%d", npad, A);
    EFFDET_REQUIRE(cap <= A, "nms_batch_chunked: cap=%d must be in [1, A=%d]", cap, A);
    const long long need = nms_workspace_words(B, cap, chunk) * (long long)sizeof(uint64_t);
    EFFDET_REQUIRE(workspace_bytes >= need, "nms_batch_chunked: workspace of %lld bytes, %lld needed",
                   (long long)workspace_bytes, need);
    EFFDET_REQUIRE(aligned16(boxes) && aligned16(workspace), "nms_batch_chunked: boxes and workspace must be 16-byte aligned");
    EFFDET_DEVICE(device);
    return nms_launch(boxes, keys, count, B, A, npad, cap, chunk, iou_threshold, (uint64_t*)workspace, keep_idx, nkeep,
                      (cudaStream_t)stream);
}

extern "C" int effdet_nms_batch_chunked_classes(const float* boxes, const uint64_t* keys, const int32_t* count,
                                                const int32_t* classes, int B, int A, int npad, int cap, int chunk,
                                                double iou_threshold, void* workspace, int64_t workspace_bytes,
                                                int32_t* keep_idx, int32_t* nkeep, int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(boxes && keys && count && classes && workspace && keep_idx && nkeep,
                   "nms_batch_chunked_classes: null tensor");
    NMS_CHUNK_LIMITS("nms_batch_chunked_classes", B, cap, chunk);
    EFFDET_REQUIRE(A > 0 && npad >= A && (npad & (npad - 1)) == 0,
                   "nms_batch_chunked_classes: npad=%d must be a power of two >= A=%d", npad, A);
    EFFDET_REQUIRE(cap <= A, "nms_batch_chunked_classes: cap=%d must be in [1, A=%d]", cap, A);
    const long long need = nms_workspace_words(B, cap, chunk) * (long long)sizeof(uint64_t);
    EFFDET_REQUIRE(workspace_bytes >= need, "nms_batch_chunked_classes: workspace of %lld bytes, %lld needed",
                   (long long)workspace_bytes, need);
    EFFDET_REQUIRE(aligned16(boxes) && aligned16(workspace),
                   "nms_batch_chunked_classes: boxes and workspace must be 16-byte aligned");
    EFFDET_DEVICE(device);
    return nms_launch(boxes, keys, count, B, A, npad, cap, chunk, iou_threshold, (uint64_t*)workspace, keep_idx, nkeep,
                      (cudaStream_t)stream, classes);
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

#define TOPK_LIMITS(fn, B, A, K, top_k)                                                                                 \
    EFFDET_REQUIRE((B) >= 1 && (B) <= 65535, fn ": B=%d must be in [1, 65535]", (B));                                   \
    EFFDET_REQUIRE((A) >= 1 && (K) >= 1, fn ": A=%d and K=%d must be >= 1", (A), (K));                                  \
    EFFDET_REQUIRE((long long)(A) * (K) < (1ll << 32), fn ": A*K = %lld pairs must be below 2^32", (long long)(A) * (K)); \
    EFFDET_REQUIRE((top_k) >= 1, fn ": top_k=%d must be >= 1", (top_k))

extern "C" int64_t effdet_detect_topk_workspace(int B, int A, int K, int top_k) {
    TOPK_LIMITS("detect_topk_workspace", B, A, K, top_k);
    return topk_workspace_bytes(B);
}

extern "C" int effdet_detect_topk_batch(const float* cls, const float* reg, const float* anchors, int B, int A, int K,
                                        float img_w, float img_h, float threshold, int top_k, int kpad, void* workspace,
                                        int64_t workspace_bytes, float* boxes, float* scores, int32_t* classes,
                                        uint64_t* keys, int32_t* count, int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(cls && reg && anchors && workspace && boxes && scores && classes && keys && count,
                   "detect_topk_batch: null tensor");
    TOPK_LIMITS("detect_topk_batch", B, A, K, top_k);
    const long long pairs = (long long)A * K;
    const int kprime = (int)(top_k < pairs ? top_k : pairs);
    EFFDET_REQUIRE(kpad >= kprime && (kpad & (kpad - 1)) == 0,
                   "detect_topk_batch: kpad=%d must be a power of two >= min(top_k, A*K) = %d", kpad, kprime);
    EFFDET_REQUIRE((long long)B * kpad <= (1ll << 30), "detect_topk_batch: B*kpad = %lld keys is too many",
                   (long long)B * kpad);
    const long long need = topk_workspace_bytes(B);
    EFFDET_REQUIRE(workspace_bytes >= need, "detect_topk_batch: workspace of %lld bytes, %lld needed",
                   (long long)workspace_bytes, need);
    EFFDET_REQUIRE(aligned16(reg) && aligned16(anchors) && aligned16(boxes) && aligned16(workspace),
                   "detect_topk_batch: reg, anchors, boxes and workspace must be 16-byte aligned");
    EFFDET_DEVICE(device);
    return topk_launch(cls, reg, anchors, B, A, K, img_w, img_h, threshold, top_k, kprime, kpad, workspace, boxes,
                       scores, classes, keys, count, (cudaStream_t)stream);
}
