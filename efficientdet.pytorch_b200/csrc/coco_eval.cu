// COCO box mAP on the device: eval.py::evaluate_coco (eval.py:260-338) with pycocotools' COCOeval (iouType 'bbox',
// default Params) as three steps, none of which reads anything back to the host.
//   selection    : eval.py:270-312  boxes /= scale, x,y,w,h, rows in NMS order up to the first score < threshold
//   matching     : COCOeval.computeIoU + evaluateImg per (image, category), 4 area ranges x 10 IoU thresholds
//   accumulation : COCOeval.accumulate per (category, area range, maxDets, IoU threshold)
// Bit-exactness rules (the results must equal pycocotools' float64 values):
//   - IoU of maskApi.c bbIou from separately rounded fp64 operations (no FMA contraction), as voc_eval.cu does;
//   - detections of one (image, category) ranked by score descending, ties in NMS order (COCOeval's mergesort);
//   - records of one category in the order a stable sort of the per-image lists, concatenated in sorted image id
//     order, gives: score descending, then image rank, then rank inside (image, category).
#include <float.h>

#include "bitonic.cuh"
#include "block_scan.cuh"

namespace effdet {

constexpr int kCocoMaxDet = 100;                                      // Params.maxDets[-1]
constexpr int kCocoIouThrs = 10;                                      // Params.iouThrs
constexpr int kCocoRecThrs = 101;                                     // Params.recThrs
constexpr int kCocoAreas = 4;                                         // all, small, medium, large
constexpr int kCocoMaxDets = 3;                                       // 1, 10, 100
constexpr int kCocoMaxCategories = 255;                               // category 255 would collide with the ~0 sentinel
constexpr int kCocoMaxImages = 1 << 18;
constexpr int kCocoPosBits = 25;
constexpr long long kCocoMaxRecords = 1ll << kCocoPosBits;
constexpr uint64_t kCocoPosMask = (1ull << kCocoPosBits) - 1;
constexpr int kCocoMaxGt = 256;                                       // ground truths of one (image, category)
constexpr int kCocoIgnoredShift = 16;                                 // flags: matched bits 0..9, ignored bits 16..25

// Params.areaRng, inclusive at both ends: [0, 1e5^2], [0, 32^2], [32^2, 96^2], [96^2, 1e5^2]
__device__ __forceinline__ bool coco_out_of_range(double area, int a) {
    const double lo = a == 0 ? 0.0 : a == 1 ? 0.0 : a == 2 ? 1024.0 : 9216.0;
    const double hi = a == 0 ? 1e10 : a == 1 ? 1024.0 : a == 2 ? 9216.0 : 1e10;
    return area < lo || area > hi;
}

// ---- selection ------------------------------------------------------------------------------------------------------
// kept[b] = the rows eval.py:290-311 records for image b: those before the first score < threshold (compared as
// Python compares float(score) < threshold, in fp64); -1 when the image overflowed NMS
__global__ void __launch_bounds__(256) coco_count_kernel(const float* __restrict__ scores, const int32_t* __restrict__ count,
                                                         int C, double thr, int32_t* __restrict__ kept) {
    __shared__ int first;
    const long long b = blockIdx.x;
    const int n = count[b];
    if (n < 0) {
        if (threadIdx.x == 0) kept[b] = -1;
        return;
    }
    const int m = min(n, C);
    if (threadIdx.x == 0) first = m;
    __syncthreads();
    for (int i = threadIdx.x; i < m; i += blockDim.x)
        if ((double)scores[b * C + i] < thr) atomicMin(&first, i);
    __syncthreads();
    if (threadIdx.x == 0) kept[b] = first;
}

// One CTA: the batch's record ranges at the cursor, in dataset order.  The cursor counts every record asked for, so
// after an overflow it says what capacity would have been enough; an image that does not fit records nothing.
__global__ void __launch_bounds__(1024) coco_place_kernel(const int32_t* __restrict__ image_rank, int B, int capacity,
                                                          unsigned long long* __restrict__ cursor,
                                                          int32_t* __restrict__ image_offset,
                                                          int32_t* __restrict__ image_count, int32_t* __restrict__ status,
                                                          int32_t* __restrict__ batch_offset,
                                                          int32_t* __restrict__ batch_count) {
    __shared__ int wi[32];
    const unsigned long long base = *cursor;
    int carry = 0;
    for (int b0 = 0; b0 < B; b0 += blockDim.x) {
        const int b = b0 + threadIdx.x;
        const int k = b < B ? batch_count[b] : 0;                       // kept rows (coco_count_kernel), -1 = overflow
        int tot;
        const int incl = carry + block_scan(max(k, 0), wi, IntAdd(), tot);
        if (b < B) {
            const unsigned long long off = base + (unsigned long long)(incl - max(k, 0));
            const bool fits = off + (unsigned long long)max(k, 0) <= (unsigned long long)capacity;
            const int cnt = (k > 0 && fits) ? k : 0;
            const int q = image_rank[b];
            status[b] = k < 0 ? 1 : (fits ? 0 : 2);
            batch_offset[b] = fits ? (int)off : capacity;
            batch_count[b] = cnt;
            image_offset[q] = fits ? (int)off : capacity;
            image_count[q] = cnt;
        }
        carry += tot;
    }
    __syncthreads();
    if (threadIdx.x == 0) *cursor = base + (unsigned long long)carry;
}

__device__ __forceinline__ int coco_category(const int64_t* labels, int i, const int32_t* label_category, int num_labels) {
    const int64_t l = labels[i];
    return (l >= 0 && l < num_labels) ? label_category[l] : -1;
}

// One CTA per image: record i of the image = row i in NMS order.  rank = position inside (image, category) after a
// stable sort by score descending (COCOeval.computeIoU / evaluateImg: np.argsort(-score, kind='mergesort')).
constexpr int kSelTile = 1024;
__global__ void __launch_bounds__(256, 1) coco_write_kernel(const float* __restrict__ scores, const int64_t* __restrict__ labels,
                                                         const float* __restrict__ boxes, const float* __restrict__ scale,
                                                         const int32_t* __restrict__ image_rank,
                                                         const int32_t* __restrict__ label_category, int num_labels, int C,
                                                         const int32_t* __restrict__ batch_offset,
                                                         const int32_t* __restrict__ batch_count, float4* __restrict__ rec_box,
                                                         float* __restrict__ rec_score, int4* __restrict__ rec_meta) {
    __shared__ float ts[kSelTile];
    __shared__ int tc[kSelTile];
    const long long b = blockIdx.x;
    const int m = batch_count[b];
    if (m <= 0) return;
    scores += b * C;
    labels += b * C;
    const float4* bx = reinterpret_cast<const float4*>(boxes) + b * C;
    const long long off = batch_offset[b];
    const float s_b = scale[b];
    const int q = image_rank[b];
    for (int i0 = 0; i0 < m; i0 += blockDim.x) {
        const int i = i0 + threadIdx.x;
        const bool mine = i < m;
        const float s = mine ? scores[i] : 0.f;
        const int c = mine ? coco_category(labels, i, label_category, num_labels) : -1;
        int rank = 0;
        for (int j0 = 0; j0 < m; j0 += kSelTile) {
            const int nj = min(kSelTile, m - j0);
            __syncthreads();
            for (int j = threadIdx.x; j < nj; j += blockDim.x) {
                ts[j] = scores[j0 + j];
                tc[j] = coco_category(labels, j0 + j, label_category, num_labels);
            }
            __syncthreads();
            if (mine && c >= 0)
                for (int j = 0; j < nj; ++j) rank += tc[j] == c && (ts[j] > s || (ts[j] == s && j0 + j < i));
        }
        if (!mine) continue;
        const float4 v = bx[i];
        const float x1 = __fdiv_rn(v.x, s_b), y1 = __fdiv_rn(v.y, s_b);      // boxes /= scale (float32)
        const float x2 = __fdiv_rn(v.z, s_b), y2 = __fdiv_rn(v.w, s_b);
        rec_box[off + i] = make_float4(x1, y1, __fsub_rn(x2, x1), __fsub_rn(y2, y1));
        rec_score[off + i] = s;
        rec_meta[off + i] = make_int4((int)labels[i], c, q, c >= 0 ? rank : 0x7fffffff);
    }
}

// ---- matching -------------------------------------------------------------------------------------------------------
// maskApi.c bbIou of detection (dx,dy,dw,dh) against ground truth g = (x,y,w,h), in its operation order
__device__ __forceinline__ double coco_iou(double dx, double dy, double dw, double dh, double da, const double* g,
                                           bool crowd) {
    const double w = __dsub_rn(fmin(__dadd_rn(dw, dx), __dadd_rn(g[2], g[0])), fmax(dx, g[0]));
    if (w <= 0.0) return 0.0;
    const double h = __dsub_rn(fmin(__dadd_rn(dh, dy), __dadd_rn(g[3], g[1])), fmax(dy, g[1]));
    if (h <= 0.0) return 0.0;
    const double i = __dmul_rn(w, h);
    const double ga = __dmul_rn(g[2], g[3]);
    const double u = crowd ? da : __dsub_rn(__dadd_rn(da, ga), i);
    return __ddiv_rn(i, u);
}

// One CTA per (category blockIdx.x, image blockIdx.y of the batch).  gt rows are (x, y, w, h, area, iscrowd) fp64,
// grouped by (image rank, category) in JSON order.  The IoU matrix [D][G] is computed once into dynamic shared memory
// (kCocoMaxDet * max_gt doubles); then thread a*10+t runs evaluateImg's greedy pass for area range a, threshold t.
__global__ void __launch_bounds__(128) coco_match_kernel(const float4* __restrict__ rec_box, const int4* __restrict__ rec_meta,
                                                         const int32_t* __restrict__ batch_offset,
                                                         const int32_t* __restrict__ batch_count,
                                                         const int32_t* __restrict__ image_rank, const double* __restrict__ gt,
                                                         const int32_t* __restrict__ gt_offsets, int K,
                                                         const double* __restrict__ iou_thrs, uint32_t* __restrict__ flags,
                                                         unsigned long long* __restrict__ npig) {
    extern __shared__ double iou[];                                   // [D][G]
    __shared__ uint16_t order[kCocoAreas][kCocoMaxGt];                // sorted gt j -> JSON index | ignored << 15
    __shared__ uint32_t taken[kCocoAreas * kCocoIouThrs][kCocoMaxGt / 32];
    __shared__ uint32_t fl[kCocoMaxDet][kCocoAreas];
    __shared__ int dt[kCocoMaxDet];
    __shared__ double dbox[kCocoMaxDet][5];                           // x, y, w, h, area
    __shared__ int nd;
    const int c = blockIdx.x;
    const long long b = blockIdx.y;
    const int q = image_rank[b];
    const long long g0 = gt_offsets[(long long)q * K + c];
    const int G = gt_offsets[(long long)q * K + c + 1] - (int)g0;
    gt += g0 * 6;
    // ground truth sorted by _ignore (stable) per area range, and the non-ignored count per area range
    if (threadIdx.x < kCocoAreas) {
        const int a = threadIdx.x;
        int j = 0;
        for (int pass = 0; pass < 2; ++pass)
            for (int g = 0; g < G; ++g) {
                const bool ig = gt[g * 6 + 5] != 0.0 || coco_out_of_range(gt[g * 6 + 4], a);
                if (ig == (pass == 1)) order[a][j++] = (uint16_t)(g | (ig << 15));
            }
        int n = 0;
        for (int g = 0; g < G; ++g) n += !(order[a][g] >> 15);
        if (n) atomicAdd(npig + c * kCocoAreas + a, (unsigned long long)n);
    }
    // the (image, category)'s detections by rank, truncated to maxDets[-1]
    for (int i = threadIdx.x; i < kCocoMaxDet; i += blockDim.x) dt[i] = -1;
    if (threadIdx.x == 0) nd = 0;
    __syncthreads();
    const int off = batch_offset[b], m = batch_count[b];
    for (int i = threadIdx.x; i < m; i += blockDim.x) {
        const int4 mt = rec_meta[off + i];
        if (mt.y == c && mt.w < kCocoMaxDet) {
            dt[mt.w] = off + i;
            atomicAdd(&nd, 1);
        }
    }
    __syncthreads();
    const int D = nd;
    if (D == 0) return;
    for (int d = threadIdx.x; d < D; d += blockDim.x) {
        const float4 v = rec_box[dt[d]];
        dbox[d][0] = v.x;
        dbox[d][1] = v.y;
        dbox[d][2] = v.z;
        dbox[d][3] = v.w;
        dbox[d][4] = __dmul_rn((double)v.z, (double)v.w);             // loadRes: area = w * h
        for (int a = 0; a < kCocoAreas; ++a) fl[d][a] = 0;
    }
    for (int i = threadIdx.x; i < kCocoAreas * kCocoIouThrs * (kCocoMaxGt / 32); i += blockDim.x) (&taken[0][0])[i] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < D * G; i += blockDim.x) {
        const int d = i / G, g = i - d * G;
        iou[i] = coco_iou(dbox[d][0], dbox[d][1], dbox[d][2], dbox[d][3], dbox[d][4], gt + g * 6, gt[g * 6 + 5] != 0.0);
    }
    __syncthreads();
    if (threadIdx.x < kCocoAreas * kCocoIouThrs) {
        const int p = threadIdx.x, a = p / kCocoIouThrs, t = p - a * kCocoIouThrs;
        const double thr = fmin(iou_thrs[t], 1.0 - 1e-10);
        uint32_t* tk = taken[p];
        for (int d = 0; d < D; ++d) {
            double best = thr;
            int mj = -1;
            bool mig = false;
            for (int j = 0; j < G; ++j) {
                const int e = order[a][j], g = e & 0x7fff;
                const bool ig = e >> 15;
                if (((tk[j >> 5] >> (j & 31)) & 1) && gt[g * 6 + 5] == 0.0) continue;   // taken, not crowd
                if (mj > -1 && !mig && ig) break;                                       // regular match, then ignored gt
                const double v = iou[d * G + g];
                if (v < best) continue;
                best = v;
                mj = j;
                mig = ig;
            }
            uint32_t bits = 0;
            if (mj >= 0) {
                tk[mj >> 5] |= 1u << (mj & 31);
                bits = (1u << t) | ((uint32_t)mig << (kCocoIgnoredShift + t));
            } else if (coco_out_of_range(dbox[d][4], a)) {
                bits = 1u << (kCocoIgnoredShift + t);
            }
            if (bits) atomicOr(&fl[d][a], bits);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < D * kCocoAreas; i += blockDim.x) flags[(long long)dt[i >> 2] * kCocoAreas + (i & 3)] = fl[i >> 2][i & 3];
}

// ---- accumulation ---------------------------------------------------------------------------------------------------
// position of a record = its index in the records laid out by image rank (each image's records in NMS order).  Inside
// one category, position order is (image rank, rank inside (image, category)) order.
__global__ void __launch_bounds__(1024) coco_base_kernel(const int32_t* __restrict__ image_count, int n,
                                                         int32_t* __restrict__ base) {
    __shared__ int wi[32];
    int carry = 0;
    for (int q0 = 0; q0 < n; q0 += blockDim.x) {
        const int q = q0 + threadIdx.x;
        const int k = q < n ? image_count[q] : 0;
        int tot;
        const int incl = carry + block_scan(k, wi, IntAdd(), tot);
        if (q < n) base[q] = incl - k;
        carry += tot;
    }
    if (threadIdx.x == 0) base[n] = carry;
}

// key = category (8 bits) | inverted score bits (31; scores are >= threshold >= 0) | position (25).  Records without a
// category, of rank >= maxDets[-1], and the padding up to a power of two are ~0 and sort last.
__global__ void __launch_bounds__(256) coco_keys_kernel(const float* __restrict__ rec_score, const int4* __restrict__ rec_meta,
                                                        const unsigned long long* __restrict__ cursor, int capacity,
                                                        const int32_t* __restrict__ image_offset,
                                                        const int32_t* __restrict__ base, int n_img, int npad,
                                                        uint64_t* __restrict__ keys, int32_t* __restrict__ perm) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int total = base[n_img];
    if (i >= total && i < npad) keys[i] = ~0ull;
    if ((unsigned long long)i >= min(*cursor, (unsigned long long)capacity)) return;
    const int4 mt = rec_meta[i];
    if (mt.z < 0) return;                                             // a slot no image wrote
    const int pos = base[mt.z] + i - image_offset[mt.z];
    uint64_t k = ~0ull;
    if (mt.y >= 0 && mt.w < kCocoMaxDet) {
        const uint32_t sb = __float_as_uint(rec_score[i]) & 0x7fffffffu;
        k = ((uint64_t)mt.y << 56) | ((uint64_t)(0x7fffffffu - sb) << kCocoPosBits) | (uint64_t)pos;
    }
    keys[pos] = k;
    perm[pos] = i;
}

// start[c] = first sorted position of category c, start[K] = end of the last category (c <= K, i in [0, npad])
__global__ void __launch_bounds__(256) coco_start_kernel(const uint64_t* __restrict__ keys, int npad, int K,
                                                         int32_t* __restrict__ start) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > npad) return;
    const int cur = i < npad ? (int)min((uint64_t)K, keys[i] >> 56) : K;
    const int prev = i > 0 ? (int)min((uint64_t)K, keys[i - 1] >> 56) : -1;
    for (int c = prev + 1; c <= cur; ++c) start[c] = i;
}

// COCOeval.accumulate for category blockIdx.x, area range blockIdx.y / 3, maxDets blockIdx.y % 3, IoU threshold
// blockIdx.z.  A position is a record of rank < maxDet; ignored positions stay in the arrays and add nothing.  The
// walk runs from the right, so the precision envelope is a running suffix maximum; the cumulative counts at a
// position are the totals minus what lies to its right.  q[r] = envelope at the first position with rc >= recThrs[r]:
// the position where rc crosses the threshold (or the first position, for thresholds <= its rc).
constexpr int kAccThreads = 256;
__global__ void __launch_bounds__(kAccThreads) coco_accumulate_kernel(const uint64_t* __restrict__ keys,
                                                                      const int32_t* __restrict__ perm,
                                                                      const int32_t* __restrict__ start,
                                                                      const int4* __restrict__ rec_meta,
                                                                      const uint32_t* __restrict__ flags,
                                                                      const unsigned long long* __restrict__ npig_all,
                                                                      const double* __restrict__ rec_thrs, int K,
                                                                      int md0, int md1, int md2,
                                                                      double* __restrict__ precision,
                                                                      double* __restrict__ recall) {
    __shared__ int wi[32];
    __shared__ double wd[32];
    __shared__ double rthr[kCocoRecThrs];
    const int c = blockIdx.x, a = blockIdx.y / kCocoMaxDets, mi = blockIdx.y % kCocoMaxDets, t = blockIdx.z;
    const int max_det = mi == 0 ? md0 : mi == 1 ? md1 : md2;
    // precision [T][R][K][A][M], recall [T][K][A][M]
    const long long pstride = (long long)K * kCocoAreas * kCocoMaxDets;
    double* prec = precision + (long long)t * kCocoRecThrs * pstride + ((long long)c * kCocoAreas + a) * kCocoMaxDets + mi;
    double* rec = recall + (long long)t * pstride + ((long long)c * kCocoAreas + a) * kCocoMaxDets + mi;
    const unsigned long long np = npig_all[c * kCocoAreas + a];
    for (int r = threadIdx.x; r < kCocoRecThrs; r += blockDim.x) {
        prec[r * pstride] = np == 0 ? -1.0 : 0.0;
        rthr[r] = rec_thrs[r];
    }
    if (np == 0) {
        if (threadIdx.x == 0) *rec = -1.0;
        return;
    }
    const double npd = (double)np;
    const int s = start[c], n = start[c + 1] - s;
    const uint32_t mbit = 1u << t, ibit = 1u << (kCocoIgnoredShift + t);
    auto classify = [&](int i, int& tp, int& fp, int& pos) {
        tp = fp = pos = 0;
        if (i < 0 || i >= n) return;
        const int r = perm[keys[s + i] & kCocoPosMask];
        if (rec_meta[r].w >= max_det) return;
        const uint32_t f = flags[(long long)r * kCocoAreas + a];
        pos = 1;
        if (!(f & ibit)) {
            tp = (f & mbit) != 0;
            fp = !tp;
        }
    };
    // totals
    int ttp = 0, tfp = 0, tpos = 0;
    for (int i0 = 0; i0 < n; i0 += blockDim.x) {
        int tp, fp, pos, tot;
        classify(i0 + threadIdx.x, tp, fp, pos);
        block_scan(tp, wi, IntAdd(), tot);
        ttp += tot;
        block_scan(fp, wi, IntAdd(), tot);
        tfp += tot;
        block_scan(pos, wi, IntAdd(), tot);
        tpos += tot;
    }
    // from the right: thread k of a chunk holds element top-1-k, so a scan in thread order is a suffix scan
    int rtp = 0, rfp = 0, rpos = 0;
    double env = 0.0;
    for (int top = n; top > 0; top -= blockDim.x) {
        const int i = top - 1 - (int)threadIdx.x;
        int tp, fp, pos, tot_tp, tot_fp, tot_pos;
        classify(i, tp, fp, pos);
        const int stp = rtp + block_scan(tp, wi, IntAdd(), tot_tp);    // to the right of i, i included
        const int sfp = rfp + block_scan(fp, wi, IntAdd(), tot_fp);
        const int spos = rpos + block_scan(pos, wi, IntAdd(), tot_pos);
        const int ctp = ttp - stp + tp, cfp = tfp - sfp + fp;            // cumulative at i, i included
        double pr = 0.0, rc = 0.0;
        if (pos) {
            rc = __ddiv_rn((double)ctp, npd);
            pr = __ddiv_rn((double)ctp, __dadd_rn(__dadd_rn((double)cfp, (double)ctp), DBL_EPSILON));
        }
        double tot_env;
        const double e = fmax(block_scan(pr, wd, DblMax(), tot_env), env);
        if (pos) {
            const bool first = spos == tpos;                                // no position to the left of i
            if (first || tp) {
                const double rc_prev = first ? -1.0 : __ddiv_rn((double)(ctp - tp), npd);
                for (int r = 0; r < kCocoRecThrs; ++r)
                    if (rc_prev < rthr[r] && rthr[r] <= rc) prec[r * pstride] = e;
            }
        }
        rtp += tot_tp;
        rfp += tot_fp;
        rpos += tot_pos;
        env = fmax(env, tot_env);
    }
    if (threadIdx.x == 0) *rec = tpos ? __ddiv_rn((double)ttp, npd) : 0.0;
}

struct AccLayout {
    long long npad;
    size_t keys, perm, base, start, total;
};

static size_t align256c(size_t x) { return (x + 255) & ~(size_t)255; }

static AccLayout acc_layout(int capacity, int n_img, int K) {
    AccLayout L;
    L.npad = 1;
    while (L.npad < capacity) L.npad <<= 1;
    L.keys = 0;
    L.perm = align256c(L.keys + (size_t)L.npad * 8);
    L.base = align256c(L.perm + (size_t)capacity * 4);
    L.start = align256c(L.base + ((size_t)n_img + 1) * 4);
    L.total = align256c(L.start + ((size_t)K + 1) * 4);
    return L;
}

}  // namespace effdet

using namespace effdet;

#define COCO_LIMITS(fn, cap, n_img, K)                                                                                  \
    EFFDET_REQUIRE((K) >= 1 && (K) <= kCocoMaxCategories, fn ": num_categories=%d must be in [1, %d]", (K),             \
                   kCocoMaxCategories);                                                                                 \
    EFFDET_REQUIRE((n_img) >= 1 && (n_img) <= kCocoMaxImages, fn ": num_images=%d must be in [1, %d]", (n_img),         \
                   kCocoMaxImages);                                                                                     \
    EFFDET_REQUIRE((cap) >= 1 && (long long)(cap) <= kCocoMaxRecords, fn ": capacity=%lld records must be in [1, %lld]", \
                   (long long)(cap), kCocoMaxRecords)

extern "C" int effdet_coco_select_batch(const float* scores, const int64_t* labels, const float* boxes,
                                        const int32_t* count, const float* scale, const int32_t* image_rank, int B, int C,
                                        double score_threshold, const int32_t* label_category, int num_labels,
                                        int num_categories, int num_images, int capacity, float* rec_box,
                                        float* rec_score, int32_t* rec_meta, int64_t* cursor, int32_t* image_offset,
                                        int32_t* image_count, int32_t* status, int32_t* batch_offset,
                                        int32_t* batch_count, int device, effdet_stream_t stream) {
    COCO_LIMITS("coco_select_batch", capacity, num_images, num_categories);
    EFFDET_REQUIRE(B >= 1 && B <= num_images && C >= 0, "coco_select_batch: B=%d must be in [1, num_images] and C=%d >= 0",
                   B, C);
    EFFDET_REQUIRE(num_labels >= 1, "coco_select_batch: num_labels=%d must be >= 1", num_labels);
    EFFDET_REQUIRE(score_threshold >= 0.0, "coco_select_batch: score_threshold=%g must be >= 0", score_threshold);
    EFFDET_REQUIRE(count && scale && image_rank && label_category && rec_box && rec_score && rec_meta && cursor &&
                       image_offset && image_count && status && batch_offset && batch_count &&
                       (C == 0 || (scores && labels && boxes)),
                   "coco_select_batch: null tensor");
    EFFDET_REQUIRE(aligned16(boxes) && aligned16(rec_box) && aligned16(rec_meta),
                   "coco_select_batch: boxes, rec_box and rec_meta must be 16-byte aligned");
    EFFDET_REQUIRE(((uintptr_t)cursor & 7) == 0, "coco_select_batch: cursor must be 8-byte aligned");
    EFFDET_DEVICE(device);
    cudaStream_t st = (cudaStream_t)stream;
    coco_count_kernel<<<B, 256, 0, st>>>(scores, count, C, score_threshold, batch_count);
    int s = launch_status("coco_count_kernel");
    if (s) return s;
    coco_place_kernel<<<1, 1024, 0, st>>>(image_rank, B, capacity, (unsigned long long*)cursor, image_offset, image_count,
                                          status, batch_offset, batch_count);
    if ((s = launch_status("coco_place_kernel"))) return s;
    coco_write_kernel<<<B, 256, 0, st>>>(scores, labels, boxes, scale, image_rank, label_category, num_labels, C,
                                         batch_offset, batch_count, (float4*)rec_box, rec_score, (int4*)rec_meta);
    return launch_status("coco_write_kernel");
}

extern "C" int effdet_coco_match(const float* rec_box, const int32_t* rec_meta, const int32_t* batch_offset,
                                 const int32_t* batch_count, const int32_t* image_rank, int B, const double* gt,
                                 const int32_t* gt_offsets, int num_images, int num_categories, int max_gt,
                                 const double* iou_thrs, int num_iou_thrs, int iou_type, uint32_t* flags, int64_t* npig,
                                 int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(iou_type == EFFDET_COCO_BBOX, "coco_match: iou_type=%d: only bbox (%d) is supported", iou_type,
                   EFFDET_COCO_BBOX);
    EFFDET_REQUIRE(num_iou_thrs == kCocoIouThrs, "coco_match: num_iou_thrs=%d: only the default %d thresholds",
                   num_iou_thrs, kCocoIouThrs);
    COCO_LIMITS("coco_match", 1, num_images, num_categories);
    EFFDET_REQUIRE(B >= 1 && B <= num_images, "coco_match: B=%d must be in [1, num_images]", B);
    EFFDET_REQUIRE(max_gt >= 0 && max_gt <= kCocoMaxGt, "coco_match: max_gt=%d must be in [0, %d]", max_gt, kCocoMaxGt);
    EFFDET_REQUIRE(rec_box && rec_meta && batch_offset && batch_count && image_rank && gt_offsets && iou_thrs && flags &&
                       npig && (max_gt == 0 || gt),
                   "coco_match: null tensor");
    EFFDET_REQUIRE(aligned16(rec_box) && aligned16(rec_meta), "coco_match: rec_box and rec_meta must be 16-byte aligned");
    EFFDET_DEVICE(device);
    const size_t smem = (size_t)kCocoMaxDet * (size_t)(max_gt > 0 ? max_gt : 1) * 8;
    cudaFuncSetAttribute(coco_match_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    coco_match_kernel<<<dim3(num_categories, B), 128, smem, (cudaStream_t)stream>>>(
        (const float4*)rec_box, (const int4*)rec_meta, batch_offset, batch_count, image_rank, gt, gt_offsets,
        num_categories, iou_thrs, flags, (unsigned long long*)npig);
    return launch_status("coco_match_kernel");
}

extern "C" int64_t effdet_coco_accumulate_workspace(int capacity, int num_images, int num_categories) {
    COCO_LIMITS("coco_accumulate_workspace", capacity, num_images, num_categories);
    return (int64_t)acc_layout(capacity, num_images, num_categories).total;
}

extern "C" int effdet_coco_accumulate(const float* rec_score, const int32_t* rec_meta, const uint32_t* flags,
                                      const int64_t* cursor, const int32_t* image_offset, const int32_t* image_count,
                                      const int64_t* npig, const double* rec_thrs, int num_rec_thrs, int max_det0,
                                      int max_det1, int max_det2, int capacity, int num_images, int num_categories,
                                      double* precision, double* recall, void* workspace, int64_t workspace_bytes,
                                      int device, effdet_stream_t stream) {
    COCO_LIMITS("coco_accumulate", capacity, num_images, num_categories);
    EFFDET_REQUIRE(num_rec_thrs == kCocoRecThrs, "coco_accumulate: num_rec_thrs=%d: only the default %d thresholds",
                   num_rec_thrs, kCocoRecThrs);
    EFFDET_REQUIRE(max_det0 == 1 && max_det1 == 10 && max_det2 == kCocoMaxDet,
                   "coco_accumulate: max_dets=(%d, %d, %d): only the default (1, 10, 100)", max_det0, max_det1, max_det2);
    EFFDET_REQUIRE(rec_score && rec_meta && flags && cursor && image_offset && image_count && npig && rec_thrs &&
                       precision && recall && workspace,
                   "coco_accumulate: null tensor");
    const AccLayout L = acc_layout(capacity, num_images, num_categories);
    EFFDET_REQUIRE(workspace_bytes >= (int64_t)L.total, "coco_accumulate: workspace of %lld bytes, %lld needed",
                   (long long)workspace_bytes, (long long)L.total);
    EFFDET_REQUIRE(aligned16(workspace) && aligned16(rec_meta),
                   "coco_accumulate: workspace and rec_meta must be 16-byte aligned");
    EFFDET_DEVICE(device);
    cudaStream_t st = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    uint64_t* keys = (uint64_t*)(ws + L.keys);
    int32_t* perm = (int32_t*)(ws + L.perm);
    int32_t* base = (int32_t*)(ws + L.base);
    int32_t* start = (int32_t*)(ws + L.start);
    const int npad = (int)L.npad;
    coco_base_kernel<<<1, 1024, 0, st>>>(image_count, num_images, base);
    int s = launch_status("coco_base_kernel");
    if (s) return s;
    coco_keys_kernel<<<cdiv(npad > capacity ? npad : capacity, 256), 256, 0, st>>>(
        rec_score, (const int4*)rec_meta, (const unsigned long long*)cursor, capacity, image_offset, base, num_images,
        npad, keys, perm);
    if ((s = launch_status("coco_keys_kernel"))) return s;
    if ((s = bitonic_sort_launch(keys, npad, npad, st))) return s;
    coco_start_kernel<<<cdiv(npad + 1, 256), 256, 0, st>>>(keys, npad, num_categories, start);
    if ((s = launch_status("coco_start_kernel"))) return s;
    coco_accumulate_kernel<<<dim3(num_categories, kCocoAreas * kCocoMaxDets, kCocoIouThrs), kAccThreads, 0, st>>>(
        keys, perm, start, (const int4*)rec_meta, flags, (const unsigned long long*)npig, rec_thrs, num_categories,
        max_det0, max_det1, max_det2, precision, recall);
    return launch_status("coco_accumulate_kernel");
}
