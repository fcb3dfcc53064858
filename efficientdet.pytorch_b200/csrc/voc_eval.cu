// VOC mean average precision on the device (SURVEY.md 8(f) rank 3): eval.py::evaluate (eval.py:165-257) as three steps
// over a batch of images, none of which reads anything back to the host.
//   selection : eval.py:107-128  boxes /= scale, score > threshold, top max_det by score, per-label split
//   matching  : eval.py:199-224  greedy TP / FP per (image, class), IoU of compute_overlap in fp64
//   AP        : eval.py:226-248  sort per class by score, cumulative TP / FP, precision envelope, np.sum of the areas
// Bit-exactness rules (the results must equal NumPy's):
//   - fp64 IoU and AP arithmetic from separately rounded operations (__dmul_rn / __dadd_rn / __dsub_rn / __ddiv_rn):
//     nvcc would otherwise contract a*b+c into an FMA, which differs from NumPy in the last bit and, at an IoU of exactly
//     the threshold, flips a TP;
//   - records of one class sort by score descending, ties by record index (image, then rank inside the image): the
//     order a STABLE sort of the reference's append order gives (np.argsort's default introsort leaves ties unspecified);
//   - the AP sum follows numpy's pairwise_sum over the whole float64 array (blocks of 8 partial sums up to 128
//     elements, split at n/2 rounded down to a multiple of 8 above that).
#include <float.h>

#include "bitonic.cuh"
#include "block_scan.cuh"

namespace effdet {

// ---- selection ------------------------------------------------------------------------------------------------------
// eval.py:108-128 for one image, run by one CTA.  Input rows are the model's detections (any order); a row is selected
// when score > thr and its rank by descending score (ties: lower input index first) is < max_det; selected rows are
// grouped by label (ascending), in score order inside a label -- exactly the per-label arrays eval.py builds.
// Dynamic shared memory: (max_det + num_classes + 1) int32.
__device__ __forceinline__ void eval_select_image(const float* __restrict__ scores, const int64_t* __restrict__ labels,
                                                  const float* __restrict__ boxes, int n, float scale, float thr, int max_det,
                                                  int num_classes, float* __restrict__ out_dets,
                                                  int32_t* __restrict__ out_labels, int32_t* __restrict__ class_off,
                                                  int32_t* __restrict__ count) {
    extern __shared__ int32_t sm[];
    int32_t* sel = sm;                    // [max_det] input index of the detection with rank r
    int32_t* cls_cnt = sm + max_det;      // [num_classes + 1]
    __shared__ int nsel;
    for (int i = threadIdx.x; i < max_det; i += blockDim.x) sel[i] = -1;
    for (int i = threadIdx.x; i <= num_classes; i += blockDim.x) cls_cnt[i] = 0;
    if (threadIdx.x == 0) nsel = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const float s = scores[i];
        if (!(s > thr)) continue;
        int rank = 0;
        for (int j = 0; j < n; ++j) {
            const float t = scores[j];
            rank += (t > thr) && (t > s || (t == s && j < i));
        }
        if (rank < max_det) {
            sel[rank] = i;
            atomicAdd(&nsel, 1);
        }
    }
    __syncthreads();
    const int m = nsel;
    for (int r = threadIdx.x; r < m; r += blockDim.x) {
        const int lab = (int)labels[sel[r]];
        if (lab >= 0 && lab < num_classes) atomicAdd(&cls_cnt[lab + 1], 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int c = 0; c < num_classes; ++c) cls_cnt[c + 1] += cls_cnt[c];
        count[0] = m;
    }
    __syncthreads();
    for (int c = threadIdx.x; c <= num_classes; c += blockDim.x) class_off[c] = cls_cnt[c];
    // stable placement: position of rank r inside its label group = number of lower ranks with the same label
    for (int r = threadIdx.x; r < m; r += blockDim.x) {
        const int i = sel[r];
        const int lab = (int)labels[i];
        if (lab < 0 || lab >= num_classes) continue;
        int pos = 0;
        for (int q = 0; q < r; ++q) pos += ((int)labels[sel[q]] == lab);
        const int dst = cls_cnt[lab] + pos;
        const float4 bx = *reinterpret_cast<const float4*>(boxes + (long long)i * 4);
        float* o = out_dets + (long long)dst * 5;
        o[0] = __fdiv_rn(bx.x, scale);                                // boxes /= scale   (float32 array / float32 scalar)
        o[1] = __fdiv_rn(bx.y, scale);
        o[2] = __fdiv_rn(bx.z, scale);
        o[3] = __fdiv_rn(bx.w, scale);
        o[4] = scores[i];
        out_labels[dst] = lab;
    }
}

__global__ void __launch_bounds__(256) eval_select_kernel(const float* __restrict__ scores, const int64_t* __restrict__ labels,
                                                          const float* __restrict__ boxes, int n, float scale, float thr,
                                                          int max_det, int num_classes, float* __restrict__ out_dets,
                                                          int32_t* __restrict__ out_labels, int32_t* __restrict__ class_off,
                                                          int32_t* __restrict__ count) {
    eval_select_image(scores, labels, boxes, n, scale, thr, max_det, num_classes, out_dets, out_labels, class_off, count);
}

// One CTA per image b of the padded detections [B,C]: the rows of image b go to slots b*max_det .. (b+1)*max_det-1.
// Slots without a detection get label -1.  count[b] == -1 (NMS overflow): overflow[b] = 1, every label -1.
__global__ void __launch_bounds__(256) eval_select_batch_kernel(const float* __restrict__ scores,
                                                                const int64_t* __restrict__ labels,
                                                                const float* __restrict__ boxes,
                                                                const int32_t* __restrict__ count,
                                                                const float* __restrict__ scale, int C, float thr, int max_det,
                                                                int num_classes, float* __restrict__ out_dets,
                                                                int32_t* __restrict__ out_labels,
                                                                int32_t* __restrict__ class_off,
                                                                int32_t* __restrict__ overflow) {
    __shared__ int32_t selected;
    const long long b = blockIdx.x;
    const int n = count[b];
    out_labels += b * max_det;
    class_off += b * (num_classes + 1);
    for (int i = threadIdx.x; i < max_det; i += blockDim.x) out_labels[i] = -1;
    if (threadIdx.x == 0) overflow[b] = n < 0;
    if (n < 0) {
        for (int c = threadIdx.x; c <= num_classes; c += blockDim.x) class_off[c] = 0;
        return;
    }
    eval_select_image(scores + b * C, labels + b * C, boxes + b * C * 4, min(n, C), scale[b], thr, max_det, num_classes,
                      out_dets + b * max_det * 5, out_labels, class_off, &selected);
}

// ---- matching -------------------------------------------------------------------------------------------------------
// compute_overlap (eval.py:19-46) of one detection against one ground-truth row, in its operation order
__device__ __forceinline__ double voc_overlap(double a0, double a1, double a2, double a3, const double* __restrict__ g) {
    const double area = __dmul_rn(__dsub_rn(g[2], g[0]), __dsub_rn(g[3], g[1]));
    double iw = __dsub_rn(fmin(a2, g[2]), fmax(a0, g[0]));
    double ih = __dsub_rn(fmin(a3, g[3]), fmax(a1, g[1]));
    iw = fmax(iw, 0.0);
    ih = fmax(ih, 0.0);
    const double inter = __dmul_rn(iw, ih);
    double ua = __dsub_rn(__dadd_rn(__dmul_rn(__dsub_rn(a2, a0), __dsub_rn(a3, a1)), area), inter);
    ua = fmax(ua, DBL_EPSILON);
    return __ddiv_rn(inter, ua);
}

// One CTA per image, one thread per class (strided): the class's detections in slot order (score descending), each
// matched greedily against the image's ground truth of that class (eval.py:205-224).  matched[s] = ground-truth row the
// slot took, -1 if none (dynamic shared memory, max_det int32).
__global__ void __launch_bounds__(128) voc_match_kernel(const float* __restrict__ dets, const int32_t* __restrict__ class_off,
                                                        const double* __restrict__ gt, const int32_t* __restrict__ gt_off,
                                                        int max_det, int K, double thr, uint8_t* __restrict__ tp,
                                                        unsigned long long* __restrict__ gt_count) {
    extern __shared__ int32_t matched[];
    const long long b = blockIdx.x;
    dets += b * max_det * 5;
    class_off += b * (K + 1);
    tp += b * max_det;
    const double* g = gt + (long long)gt_off[b] * 5;
    const int ng = gt_off[b + 1] - gt_off[b];
    for (int c = threadIdx.x; c < K; c += blockDim.x) {
        const double lab = (double)c;                                 // annotations[:, 4] == label
        int n_c = 0;
        for (int j = 0; j < ng; ++j) n_c += g[j * 5 + 4] == lab;
        if (n_c) atomicAdd(gt_count + c, (unsigned long long)n_c);
        const int s0 = class_off[c], s1 = class_off[c + 1];
        for (int s = s0; s < s1; ++s) {
            const float* d = dets + (long long)s * 5;
            const double a0 = d[0], a1 = d[1], a2 = d[2], a3 = d[3];  // float32 widened, as np.concatenate does
            int arg = -1;
            double best = 0.0;
            for (int j = 0; j < ng; ++j) {
                if (g[j * 5 + 4] != lab) continue;
                const double ov = voc_overlap(a0, a1, a2, a3, g + j * 5);
                if (arg < 0 || ov > best) {                           // np.argmax: the first maximum
                    best = ov;
                    arg = j;
                }
            }
            bool hit = arg >= 0 && best >= thr;
            for (int q = s0; hit && q < s; ++q) hit = matched[q] != arg;
            matched[s] = hit ? arg : -1;
            tp[s] = hit;
        }
    }
}

// ---- average precision ----------------------------------------------------------------------------------------------
// key = class (8 bits) | inverted score bits (31 bits; scores are > threshold >= 0, so the sign bit is free) | record
// index (25 bits).  Ascending order = class ascending, score descending, record index ascending.  Records without a
// label and the padding up to a power of two are ~0 and sort last.
constexpr int kVocIndexBits = 25;
constexpr int kVocMaxClasses = 255;                                   // class 255 would collide with the ~0 sentinel
constexpr long long kVocMaxRecords = 1ll << kVocIndexBits;
constexpr uint64_t kVocIndexMask = (1ull << kVocIndexBits) - 1;
constexpr int kApLog = 10;
constexpr int kApThreads = 1 << kApLog;
constexpr int kPwBlock = 128;                                         // numpy's PW_BLOCKSIZE

__global__ void __launch_bounds__(256) voc_keys_kernel(const float* __restrict__ dets, const int32_t* __restrict__ labels,
                                                       int R, int npad, int K, uint64_t* __restrict__ keys) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npad) return;
    uint64_t k = ~0ull;
    if (i < R) {
        const int c = labels[i];
        if (c >= 0 && c < K) {
            const uint32_t sb = __float_as_uint(dets[(long long)i * 5 + 4]) & 0x7fffffffu;
            k = ((uint64_t)c << 56) | ((uint64_t)(0x7fffffffu - sb) << kVocIndexBits) | (uint64_t)i;
        }
    }
    keys[i] = k;
}

// start[c] = first sorted position of class c, start[K] = end of the last class (c <= K, i in [0, npad])
__global__ void __launch_bounds__(256) voc_class_start_kernel(const uint64_t* __restrict__ keys, int npad, int K,
                                                              int32_t* __restrict__ start) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > npad) return;
    const int cur = i < npad ? (int)min((uint64_t)K, keys[i] >> 56) : K;
    const int prev = i > 0 ? (int)min((uint64_t)K, keys[i - 1] >> 56) : -1;
    for (int c = prev + 1; c <= cur; ++c) start[c] = i;
}

// numpy's pairwise_sum leaf (n <= 128)
__device__ double pw_leaf(const double* a, long long n) {
    if (n < 8) {
        double r = -0.0;
        for (long long i = 0; i < n; ++i) r = __dadd_rn(r, a[i]);
        return r;
    }
    double r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = a[j];
    long long i = 8;
    for (; i < n - (n % 8); i += 8) {
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = __dadd_rn(r[j], a[i + j]);
    }
    double res = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])),
                           __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
    for (; i < n; ++i) res = __dadd_rn(res, a[i]);
    return res;
}

__device__ __forceinline__ long long pw_split(long long n) {
    const long long h = n / 2;
    return h - h % 8;
}

// numpy's pairwise_sum of a[0..n) by one thread: the recursion as an explicit stack (depth <= log2(n / 64) + 1)
__device__ double pw_sum(const double* a, long long n) {
    constexpr int kDepth = 24;
    long long off[kDepth], len[kDepth];
    double left[kDepth];
    bool right[kDepth];
    int sp = 0;
    off[0] = 0;
    len[0] = n;
    for (;;) {
        if (len[sp] > kPwBlock) {                                     // descend into the left half
            right[sp] = false;
            off[sp + 1] = off[sp];
            len[sp + 1] = pw_split(len[sp]);
            ++sp;
            continue;
        }
        double v = pw_leaf(a + off[sp], len[sp]);
        for (;;) {                                                    // return v to the parents
            if (sp == 0) return v;
            --sp;
            if (!right[sp]) {                                         // left half done: descend into the right half
                left[sp] = v;
                right[sp] = true;
                const long long h = pw_split(len[sp]);
                off[sp + 1] = off[sp] + h;
                len[sp + 1] = len[sp] - h;
                ++sp;
                break;
            }
            v = __dadd_rn(left[sp], v);
        }
    }
}

// numpy's pairwise_sum of a[0..n) by the whole CTA (kApThreads threads): the top kApLog levels of the recursion tree
// give one subtree per thread (a leaf reached higher up goes to the thread whose remaining path bits are 0); the
// subtree sums are then combined level by level, left + right, exactly as the recursion does.
__device__ double pw_sum_block(const double* a, long long n, double* part) {
    const int p = threadIdx.x;
    long long off = 0, len = n;
    bool mine = true;
    for (int d = 0; d < kApLog; ++d) {
        if (len <= kPwBlock) {
            mine = (p & ((1 << (kApLog - d)) - 1)) == 0;
            break;
        }
        const long long h = pw_split(len);
        if ((p >> (kApLog - 1 - d)) & 1) {
            off += h;
            len -= h;
        } else {
            len = h;
        }
    }
    part[p] = mine ? pw_sum(a + off, len) : 0.0;
    __syncthreads();
    for (int d = kApLog - 1; d >= 0; --d) {
        if (p < (1 << d)) {
            long long l = n;
            bool exists = true;
            for (int q = 0; q < d; ++q) {
                if (l <= kPwBlock) {
                    exists = false;
                    break;
                }
                const long long h = pw_split(l);
                l = ((p >> (d - 1 - q)) & 1) ? l - h : h;
            }
            if (exists && l > kPwBlock) {
                const int idx = p << (kApLog - d);
                part[idx] = __dadd_rn(part[idx], part[idx + (1 << (kApLog - d - 1))]);
            }
        }
        __syncthreads();
    }
    return part[0];
}

// eval.py:226-248 for class blockIdx.x over its sorted records.  mrec / mpre hold n + 2 values at s + 2c, terms n + 1
// at s + c (s = the class's first sorted position), so the classes never overlap.
__global__ void __launch_bounds__(kApThreads) voc_ap_kernel(const uint64_t* __restrict__ keys,
                                                            const int32_t* __restrict__ start,
                                                            const uint8_t* __restrict__ tp,
                                                            const unsigned long long* __restrict__ gt_count,
                                                            double* __restrict__ mrec_ws, double* __restrict__ mpre_ws,
                                                            double* __restrict__ terms_ws, double* __restrict__ ap,
                                                            double* __restrict__ num_ann) {
    __shared__ int wi[32];
    __shared__ double wd[32];
    __shared__ double part[kApThreads];
    const int c = blockIdx.x;
    const int s = start[c], n = start[c + 1] - s;
    const unsigned long long na = gt_count[c];
    if (na == 0) {                                                    // eval.py:227-229
        if (threadIdx.x == 0) ap[c] = num_ann[c] = 0.0;
        return;
    }
    const double nad = (double)na;
    double* mrec = mrec_ws + s + 2 * c;
    double* mpre = mpre_ws + s + 2 * c;
    double* terms = terms_ws + s + c;
    // cumulative TP / FP (exact integers), recall and precision, behind the 0 sentinel
    int carry = 0;
    for (int base = 0; base < n; base += blockDim.x) {
        const int i = base + threadIdx.x;
        const int f = i < n ? tp[keys[s + i] & kVocIndexMask] : 0;
        int tot;
        const int t = carry + block_scan(f, wi, IntAdd(), tot);
        if (i < n) {
            const double tpd = (double)t, fpd = (double)(i + 1 - t);
            mrec[i + 1] = __ddiv_rn(tpd, nad);
            mpre[i + 1] = __ddiv_rn(tpd, fmax(__dadd_rn(tpd, fpd), DBL_EPSILON));
        }
        carry += tot;
    }
    if (threadIdx.x == 0) {
        mrec[0] = 0.0;
        mpre[0] = 0.0;
        mrec[n + 1] = 1.0;
        mpre[n + 1] = 0.0;
    }
    __syncthreads();
    // precision envelope: suffix maximum over the n + 2 values, walked from the end
    double run = 0.0;
    for (int top = n + 2; top > 0; top -= blockDim.x) {
        const int i = top - 1 - (int)threadIdx.x;
        double tot;
        const double v = fmax(block_scan(i >= 0 ? mpre[i] : 0.0, wd, DblMax(), tot), run);
        if (i >= 0) mpre[i] = v;
        run = fmax(run, tot);
    }
    __syncthreads();
    // (mrec[i+1] - mrec[i]) * mpre[i+1] where recall changes, in order
    int m = 0;
    for (int base = 0; base <= n; base += blockDim.x) {
        const int i = base + threadIdx.x;
        const bool f = i <= n && mrec[i + 1] != mrec[i];
        int tot;
        const int pos = m + block_scan((int)f, wi, IntAdd(), tot) - 1;
        if (f) terms[pos] = __dmul_rn(__dsub_rn(mrec[i + 1], mrec[i]), mpre[i + 1]);
        m += tot;
    }
    __syncthreads();
    const double sum = pw_sum_block(terms, m, part);
    if (threadIdx.x == 0) {
        ap[c] = sum;
        num_ann[c] = nad;
    }
}

struct ApLayout {
    long long npad;
    size_t keys, start, mrec, mpre, terms, total;
};

static size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

static ApLayout ap_layout(int R, int K) {
    ApLayout L;
    L.npad = 1;
    while (L.npad < R) L.npad <<= 1;
    L.keys = 0;
    L.start = align256(L.keys + (size_t)L.npad * 8);
    L.mrec = align256(L.start + (size_t)(K + 1) * 4);
    L.mpre = align256(L.mrec + ((size_t)R + 2 * (size_t)K) * 8);
    L.terms = align256(L.mpre + ((size_t)R + 2 * (size_t)K) * 8);
    L.total = align256(L.terms + ((size_t)R + (size_t)K) * 8);
    return L;
}

}  // namespace effdet

using namespace effdet;

#define VOC_LIMITS(fn, R, K)                                                                                              \
    EFFDET_REQUIRE((K) >= 1 && (K) <= kVocMaxClasses, fn ": num_classes=%d must be in [1, %d]", (K), kVocMaxClasses); \
    EFFDET_REQUIRE((R) >= 1 && (long long)(R) <= kVocMaxRecords, fn ": %lld records must be in [1, %lld]",            \
                   (long long)(R), kVocMaxRecords)

extern "C" int effdet_eval_select(const float* scores, const int64_t* labels, const float* boxes, int n, float scale,
                                  float score_threshold, int max_det, int num_classes, float* out_dets, int32_t* out_labels,
                                  int32_t* class_offsets, int32_t* count, int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(out_dets && out_labels && class_offsets && count && n >= 0 && max_det > 0 && num_classes > 0 &&
                       (n == 0 || (scores && labels && boxes)),
                   "eval_select: bad arguments");
    EFFDET_REQUIRE((size_t)(max_det + num_classes + 1) * 4 <= 48 * 1024, "eval_select: max_det + num_classes too large");
    EFFDET_REQUIRE(aligned16(boxes), "eval_select: boxes must be 16-byte aligned");
    EFFDET_REQUIRE(scale > 0.f, "eval_select: scale must be positive");
    EFFDET_DEVICE(device);
    eval_select_kernel<<<1, 256, (size_t)(max_det + num_classes + 1) * 4, (cudaStream_t)stream>>>(
        scores, labels, boxes, n, scale, score_threshold, max_det, num_classes, out_dets, out_labels, class_offsets, count);
    return launch_status("eval_select_kernel");
}

extern "C" int effdet_eval_select_batch(const float* scores, const int64_t* labels, const float* boxes,
                                        const int32_t* count, const float* scale, int B, int C, float score_threshold,
                                        int max_det, int num_classes, float* out_dets, int32_t* out_labels,
                                        int32_t* class_offsets, int32_t* overflow, int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(max_det >= 1, "eval_select_batch: max_det=%d must be >= 1", max_det);
    EFFDET_REQUIRE(num_classes >= 1, "eval_select_batch: num_classes=%d must be >= 1", num_classes);
    EFFDET_REQUIRE((size_t)(max_det + num_classes + 1) * 4 <= 48 * 1024,
                   "eval_select_batch: max_det=%d + num_classes=%d too large for shared memory", max_det, num_classes);
    EFFDET_REQUIRE(B >= 1 && C >= 0, "eval_select_batch: B=%d must be >= 1 and C=%d >= 0", B, C);
    EFFDET_REQUIRE(count && scale && out_dets && out_labels && class_offsets && overflow && (C == 0 || (scores && labels && boxes)),
                   "eval_select_batch: null tensor");
    EFFDET_REQUIRE(aligned16(boxes), "eval_select_batch: boxes must be 16-byte aligned");
    EFFDET_REQUIRE(score_threshold >= 0.f, "eval_select_batch: score_threshold=%g must be >= 0", score_threshold);
    EFFDET_DEVICE(device);
    eval_select_batch_kernel<<<B, 256, (size_t)(max_det + num_classes + 1) * 4, (cudaStream_t)stream>>>(
        scores, labels, boxes, count, scale, C, score_threshold, max_det, num_classes, out_dets, out_labels, class_offsets,
        overflow);
    return launch_status("eval_select_batch_kernel");
}

extern "C" int effdet_voc_match(const float* dets, const int32_t* class_offsets, const double* gt, const int32_t* gt_offsets,
                                int num_gt, int B, int max_det, int num_classes, double iou_threshold, uint8_t* tp,
                                int64_t* gt_count, int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(max_det >= 1 && (size_t)max_det * 4 <= 48 * 1024, "voc_match: max_det=%d must be in [1, %d]", max_det,
                   48 * 1024 / 4);
    EFFDET_REQUIRE(num_classes >= 1 && num_classes <= kVocMaxClasses, "voc_match: num_classes=%d must be in [1, %d]",
                   num_classes, kVocMaxClasses);
    EFFDET_REQUIRE(B >= 1 && num_gt >= 0, "voc_match: B=%d must be >= 1 and num_gt=%d >= 0", B, num_gt);
    EFFDET_REQUIRE(dets && class_offsets && gt_offsets && tp && gt_count && (num_gt == 0 || gt), "voc_match: null tensor");
    EFFDET_DEVICE(device);
    voc_match_kernel<<<B, 128, (size_t)max_det * 4, (cudaStream_t)stream>>>(
        dets, class_offsets, gt, gt_offsets, max_det, num_classes, iou_threshold, tp, (unsigned long long*)gt_count);
    return launch_status("voc_match_kernel");
}

extern "C" int64_t effdet_voc_ap_workspace(int num_records, int num_classes) {
    VOC_LIMITS("voc_ap_workspace", num_records, num_classes);
    return (int64_t)ap_layout(num_records, num_classes).total;
}

extern "C" int effdet_voc_ap(const float* dets, const int32_t* labels, const uint8_t* tp, const int64_t* gt_count,
                             int num_records, int num_classes, double* ap, double* num_annotations, void* workspace,
                             int64_t workspace_bytes, int device, effdet_stream_t stream) {
    VOC_LIMITS("voc_ap", num_records, num_classes);
    EFFDET_REQUIRE(dets && labels && tp && gt_count && ap && num_annotations && workspace, "voc_ap: null tensor");
    const ApLayout L = ap_layout(num_records, num_classes);
    EFFDET_REQUIRE(workspace_bytes >= (int64_t)L.total, "voc_ap: workspace of %lld bytes, %lld needed",
                   (long long)workspace_bytes, (long long)L.total);
    EFFDET_REQUIRE(aligned16(workspace), "voc_ap: workspace must be 16-byte aligned");
    EFFDET_DEVICE(device);
    cudaStream_t st = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    uint64_t* keys = (uint64_t*)(ws + L.keys);
    int32_t* start = (int32_t*)(ws + L.start);
    const int npad = (int)L.npad;
    voc_keys_kernel<<<cdiv(npad, 256), 256, 0, st>>>(dets, labels, num_records, npad, num_classes, keys);
    int s = launch_status("voc_keys_kernel");
    if (s) return s;
    if ((s = bitonic_sort_launch(keys, npad, npad, st))) return s;
    voc_class_start_kernel<<<cdiv(npad + 1, 256), 256, 0, st>>>(keys, npad, num_classes, start);
    if ((s = launch_status("voc_class_start_kernel"))) return s;
    voc_ap_kernel<<<num_classes, kApThreads, 0, st>>>(keys, start, tp, (const unsigned long long*)gt_count,
                                                       (double*)(ws + L.mrec), (double*)(ws + L.mpre),
                                                       (double*)(ws + L.terms), ap, num_annotations);
    return launch_status("voc_ap_kernel");
}
