// Soft-NMS (Bodla et al., ICCV 2017, Algorithm 1) for a batch of B images, after effdet_detect_candidates_batch's
// candidate and sort launches.  Each pick emits the live candidate with the highest current score (ties: lower anchor
// index, i.e. the smallest 64-bit key of detect.cu's format) and rescales the scores of the others by a weight of
// their IoU with it; a candidate whose score falls to the threshold or below leaves the live set.
//   linear  : w = (double)ov > iou_threshold ? 1 - ov : 1
//   gaussian: w = (float)exp(-((double)ov * ov) / sigma)       fp64, rounded once to fp32
//   s = s * w (fp32); live iff s > threshold (the candidate filter's comparison)
// IoU is detect.cu's iou_gt arithmetic (separately rounded fp32 ops, no FMA), and 0 without a division when the
// intersection is 0.  Output rows: the decayed score at the moment of the pick, the candidate's class and box, in pick
// order, so scores are non-increasing.  Rows past the pick count are zero; count[b] > cap gives out_count = -1 and zero
// rows, as effdet_nms_batch does.
//
// Design: one thread-block cluster of `cs` CTAs (kSoftThreads threads each) per image.  The live candidates (box, current
// score, anchor index) are split into contiguous slices, one per CTA.  Per pick every CTA:
//   1. takes its best key from the scores its threads just wrote (warp shuffles, then one block barrier),
//   2. publishes key and box in its slot[pick & 1] and passes one cluster barrier,
//   3. reads every CTA's slot through distributed shared memory: all CTAs agree on the winner, CTA 0 emits it,
//   4. decays its own slice against the winner's box and notes its next best key on the way.
// The slots are double-buffered: a slot is rewritten two picks later, after a barrier that every reader has passed.
// Dead candidates stay in the slice until fewer than half of it is live; then the CTA compacts the slice in place.
//
// Capacity boundaries (each is straddled by tests/test_soft_nms.py):
//   * cluster size, from cap on the host: cs = 1 for cap <= kSlice, 2 up to 2*kSlice, 4 up to 4*kSlice, 8 above.
//   * single CTA, from the runtime count n: n <= kSlice runs on CTA 0 alone with block barriers only; the other CTAs
//     of the cluster only zero their share of the rows and exit, and nobody touches their shared memory.
//   * residency, from n: slices of ceil(n/cs) <= kSlice candidates live in shared memory; larger ones (only possible
//     when cap > kMaxCluster*kSlice, where the workspace is non-empty) live in the global workspace [B][cap] of
//     (float4 box, float score, int32 anchor), which stays in L2 for realistic sizes.
//
// Per-class Soft-NMS (kClasses): picks still go in the global (score, anchor) order, but a pick decays only the live
// candidates of its own class (classes [B,A]); the others stay live and unchanged.  Restricted to one class, the picks
// are Soft-NMS run on that class alone.  A shared-memory slot then also holds the candidate's class (28 bytes a slot);
// a slice in the global workspace reads it from classes, so the workspace is the agnostic kernel's.
#include <cooperative_groups.h>

#include "common.cuh"

namespace cg = cooperative_groups;

namespace effdet {

constexpr int kSoftThreads = 1024;
constexpr int kSlice = 4096;                  // candidates of one CTA slice held in shared memory (96 KiB)
constexpr int kMaxCluster = 8;                // portable cluster size limit
constexpr int kSoftWarps = kSoftThreads / 32;

struct SoftSlot {
    uint64_t key;
    float4 box;
};

__device__ __forceinline__ uint32_t soft_order(float f) {  // detect.cu's float_order: monotone float -> uint32
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float soft_unorder(uint32_t o) {
    return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o);
}

__device__ __forceinline__ uint64_t soft_key(float s, int anchor) {
    return ((uint64_t)(~soft_order(s)) << 32) | (uint32_t)anchor;
}

// iou_gt's arithmetic, returning the IoU itself
__device__ __forceinline__ float soft_iou(const float4 a, const float4 b) {
    const float left = fmaxf(a.x, b.x), right = fminf(a.z, b.z);
    const float top = fmaxf(a.y, b.y), bottom = fminf(a.w, b.w);
    const float width = fmaxf(__fsub_rn(right, left), 0.f), height = fmaxf(__fsub_rn(bottom, top), 0.f);
    const float inter = __fmul_rn(width, height);
    if (inter == 0.f) return 0.f;
    const float sa = __fmul_rn(__fsub_rn(a.z, a.x), __fsub_rn(a.w, a.y));
    const float sb = __fmul_rn(__fsub_rn(b.z, b.x), __fsub_rn(b.w, b.y));
    return __fdiv_rn(inter, __fsub_rn(__fadd_rn(sa, sb), inter));
}

__device__ __forceinline__ float soft_weight(float ov, int method, double iou_threshold, double sigma) {
    if (method == EFFDET_SOFT_NMS_LINEAR) return (double)ov > iou_threshold ? __fsub_rn(1.f, ov) : 1.f;
    return (float)exp(__ddiv_rn(-__dmul_rn((double)ov, (double)ov), sigma));
}

__device__ __forceinline__ uint64_t shfl_min_u64(uint64_t v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const uint64_t w = __shfl_xor_sync(0xffffffffu, v, o);
        v = w < v ? w : v;
    }
    return v;
}

template <bool kClasses>
__global__ void __launch_bounds__(kSoftThreads, 1) soft_nms_kernel(
    const float* __restrict__ boxes, const float* __restrict__ scores, const int32_t* __restrict__ classes,
    const uint64_t* __restrict__ keys, const int32_t* __restrict__ count, int A, int npad, int cap, int method,
    double iou_threshold, double sigma, float threshold, float4* ws_box, float* ws_score, int32_t* ws_anchor,
    float* __restrict__ out_scores, long long* __restrict__ out_classes, float* __restrict__ out_boxes,
    int32_t* __restrict__ out_count) {
    extern __shared__ __align__(16) unsigned char soft_smem[];
    float4* s_box = reinterpret_cast<float4*>(soft_smem);
    float* s_score = reinterpret_cast<float*>(s_box + kSlice);
    int32_t* s_anchor = reinterpret_cast<int32_t*>(s_score + kSlice);
    int32_t* s_class = s_anchor + kSlice;          // kClasses only
    __shared__ SoftSlot slot[2];
    __shared__ uint64_t w_key[kSoftWarps];
    __shared__ float4 w_box[kSoftWarps];
    __shared__ int w_live[kSoftWarps];
    __shared__ int w_cnt[kSoftWarps];

    cg::cluster_group cluster = cg::this_cluster();
    const int cs = (int)cluster.num_blocks();
    const int rank = (int)cluster.block_rank();
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const long long b = blockIdx.y;
    const int n = count[b];
    const long long orow = b * cap;
    const bool overflow = n > cap;
    const int filled = overflow ? 0 : n;           // rows [filled, cap) are zero whatever the picks
    for (int i = filled + rank * kSoftThreads + tid; i < cap; i += cs * kSoftThreads) {
        out_scores[orow + i] = 0.f;
        out_classes[orow + i] = 0;
        st4(out_boxes + (orow + i) * 4, f4zero());
    }
    if (overflow || n == 0) {
        if (rank == 0 && tid == 0) out_count[b] = overflow ? -1 : 0;
        return;
    }
    const bool single = n <= kSlice || cs == 1;
    if (single && rank > 0) return;
    const int parts = single ? 1 : cs;
    const int per = (n + parts - 1) / parts;
    const int lo = rank * per;
    int len = max(0, min(n, lo + per) - lo);
    float4* box = s_box;
    float* score = s_score;
    int32_t* anchor = s_anchor;
    int32_t* klass = s_class;                      // kClasses: the slice's classes, null when read from `classes`
    if (per > kSlice) {                            // global residency: the host guarantees the workspace
        box = ws_box + b * cap + lo;
        score = ws_score + b * cap + lo;
        anchor = ws_anchor + b * cap + lo;
        klass = nullptr;
    }
    const int32_t* cb = classes + b * A;
    const float* bx = boxes + b * A * 4;
    const float* sc = scores + b * A;
    const uint64_t* kb = keys + b * npad;

    // load the slice; note each thread's best key and box and its live count
    uint64_t best = ~0ull;
    float4 bbox = f4zero();
    int live = 0;
    for (int i = tid; i < len; i += kSoftThreads) {
        const int a = (int)(uint32_t)kb[lo + i];
        const float4 v = ldg4(bx + (long long)a * 4);
        const float s = sc[a];
        box[i] = v;
        score[i] = s;
        anchor[i] = a;
        if constexpr (kClasses) {
            if (klass) klass[i] = cb[a];
        }
        const bool ok = s > threshold;             // false only through the C ABI, with a higher threshold
        const uint64_t k = ok ? soft_key(s, a) : ~0ull;
        if (k < best) { best = k; bbox = v; }
        live += ok;
    }
    int picks = 0;
    for (int p = 0;; p ^= 1) {
        // 1. the CTA's best key and its box
        const uint64_t wb = shfl_min_u64(best);
        const int wl = __reduce_add_sync(0xffffffffu, live);
        if (best == wb && wb != ~0ull) w_box[warp] = bbox;   // keys are unique: one lane
        if (lane == 0) { w_key[warp] = wb; w_live[warp] = wl; }
        __syncthreads();
        if (warp == 0) {
            const uint64_t k = w_key[lane];
            const uint64_t m = shfl_min_u64(k);
            if (lane == 0 && m == ~0ull) slot[p].key = m;
            if (k == m && m != ~0ull) slot[p] = SoftSlot{m, w_box[lane]};
        }
        int total = 0;
        for (int w = 0; w < kSoftWarps; ++w) total += w_live[w];
        // 2. publish; 3. every warp reads all slots and agrees on the winner
        if (single) __syncthreads(); else cluster.sync();
        uint64_t key = ~0ull;
        float4 wbox = f4zero();
        if (lane < parts) {
            const SoftSlot* sl = single ? &slot[p] : cluster.map_shared_rank(&slot[p], lane);
            key = sl->key;
            wbox = sl->box;
        }
        const uint64_t win = shfl_min_u64(key);
        const int src = __ffs(__ballot_sync(0xffffffffu, key == win)) - 1;
        wbox.x = __shfl_sync(0xffffffffu, wbox.x, src);
        wbox.y = __shfl_sync(0xffffffffu, wbox.y, src);
        wbox.z = __shfl_sync(0xffffffffu, wbox.z, src);
        wbox.w = __shfl_sync(0xffffffffu, wbox.w, src);
        if (win == ~0ull || picks == cap) break;
        const int wa = (int)(uint32_t)win;
        if (rank == 0 && tid == 0) {
            const long long o = orow + picks;
            out_scores[o] = soft_unorder(~(uint32_t)(win >> 32));
            out_classes[o] = (long long)classes[b * A + wa];
            st4(out_boxes + o * 4, wbox);
        }
        ++picks;
        // compaction: when fewer than half of the slice is live, move the live entries to its front, in order
        if (2 * total < len && len > kSoftThreads) {
            int out = 0;
            for (int base = 0; base < len; base += kSoftThreads) {
                const int i = base + tid;
                float4 v;
                float s = 0.f;
                int a = 0, c = 0;
                const bool keep = i < len && score[i] > threshold;
                if (keep) { v = box[i]; s = score[i]; a = anchor[i]; }
                if constexpr (kClasses) {
                    if (keep && klass) c = klass[i];
                }
                const uint32_t bal = __ballot_sync(0xffffffffu, keep);
                if (lane == 0) w_cnt[warp] = __popc(bal);
                __syncthreads();
                int off = 0, sum = 0;
                for (int w = 0; w < kSoftWarps; ++w) {
                    const int c = w_cnt[w];
                    off += w < warp ? c : 0;
                    sum += c;
                }
                if (keep) {
                    const int j = out + off + __popc(bal & ((1u << lane) - 1u));
                    box[j] = v;
                    score[j] = s;
                    anchor[j] = a;
                    if constexpr (kClasses) {
                        if (klass) klass[j] = c;
                    }
                }
                out += sum;
                __syncthreads();
            }
            len = out;
        }
        // 4. decay the slice against the winner; the winner itself leaves it
        best = ~0ull;
        live = 0;
        int32_t wc = 0;
        if constexpr (kClasses) wc = cb[wa];
        for (int i = tid; i < len; i += kSoftThreads) {
            float s = score[i];
            if (!(s > threshold)) continue;
            const int a = anchor[i];
            const float4 v = box[i];
            if (a == wa) {
                score[i] = __int_as_float(0x7fc00000);      // NaN: never > threshold
                continue;
            }
            bool same = true;
            if constexpr (kClasses) same = (klass ? klass[i] : cb[a]) == wc;
            const float ov = same ? soft_iou(wbox, v) : 0.f;
            if (ov != 0.f) {
                s = __fmul_rn(s, soft_weight(ov, method, iou_threshold, sigma));
                score[i] = s;
                if (!(s > threshold)) continue;
            }
            const uint64_t k = soft_key(s, a);
            if (k < best) { best = k; bbox = v; }
            ++live;
        }
    }
    if (rank == 0 && tid == 0) out_count[b] = picks;
    for (int i = picks + rank * kSoftThreads + tid; i < filled; i += parts * kSoftThreads) {   // candidates never picked
        out_scores[orow + i] = 0.f;
        out_classes[orow + i] = 0;
        st4(out_boxes + (orow + i) * 4, f4zero());
    }
    if (!single) cluster.sync();                   // no CTA leaves while another may still read its slots
}

static int soft_cluster_size(int cap) {
    int cs = 1;
    while (cs < kMaxCluster && (long long)cs * kSlice < cap) cs <<= 1;
    return cs;
}

static size_t soft_smem_bytes(bool with_classes) {
    return (size_t)kSlice * (sizeof(float4) + sizeof(float) + sizeof(int32_t) + (with_classes ? sizeof(int32_t) : 0));
}

// the global slices: [B][cap] boxes, then scores, then anchors, rounded up to 16 bytes; empty unless some image can
// need them
static long long soft_workspace_bytes(int B, int cap) {
    if ((long long)soft_cluster_size(cap) * kSlice >= cap) return 0;
    const long long bytes = (long long)B * cap * (long long)(sizeof(float4) + sizeof(float) + sizeof(int32_t));
    return (bytes + 15) / 16 * 16;
}

static int soft_nms_launch(const float* boxes, const float* scores, const int32_t* classes, const uint64_t* keys,
                           const int32_t* count, int B, int A, int npad, int cap, int method, double iou_threshold,
                           double sigma, float threshold, void* ws, float* out_scores, int64_t* out_classes,
                           float* out_boxes, int32_t* out_count, cudaStream_t st, bool with_classes = false) {
    const int cs = soft_cluster_size(cap);
    const size_t smem = soft_smem_bytes(with_classes);
    auto kernel = with_classes ? soft_nms_kernel<true> : soft_nms_kernel<false>;
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return fail(EFFDET_ERR_LAUNCH, "soft_nms: smem opt-in: %s", cudaGetErrorString(e));
    float4* ws_box = nullptr;
    float* ws_score = nullptr;
    int32_t* ws_anchor = nullptr;
    if (soft_workspace_bytes(B, cap) > 0) {
        ws_box = (float4*)ws;
        ws_score = (float*)(ws_box + (long long)B * cap);
        ws_anchor = (int32_t*)(ws_score + (long long)B * cap);
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(cs, B);
    cfg.blockDim = dim3(kSoftThreads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = cs;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    e = cudaLaunchKernelEx(&cfg, kernel, boxes, scores, classes, keys, count, A, npad, cap, method,
                           iou_threshold, sigma, threshold, ws_box, ws_score, ws_anchor, out_scores,
                           (long long*)out_classes, out_boxes, out_count);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(EFFDET_ERR_LAUNCH, "soft_nms_kernel: %s", cudaGetErrorString(e));
    }
    return launch_status("soft_nms_kernel");
}

}  // namespace effdet

using namespace effdet;

#define SOFT_NMS_LIMITS(fn, B, cap)                                                                                    \
    EFFDET_REQUIRE((B) >= 1 && (B) <= 65535, fn ": B=%d must be in [1, 65535]", (B));                                   \
    EFFDET_REQUIRE((cap) >= 1, fn ": cap=%d must be >= 1", (cap))

extern "C" int64_t effdet_soft_nms_workspace(int B, int cap) {
    SOFT_NMS_LIMITS("soft_nms_workspace", B, cap);
    return soft_workspace_bytes(B, cap);
}

// the refusals of effdet_soft_nms_batch and effdet_soft_nms_batch_classes, named after the entry `fn`
#define SOFT_NMS_CHECKS(fn)                                                                                            \
    EFFDET_REQUIRE(boxes && scores && classes && keys && count && out_scores && out_classes && out_boxes && out_count,  \
                   fn ": null tensor");                                                                                \
    SOFT_NMS_LIMITS(fn, B, cap);                                                                                       \
    EFFDET_REQUIRE(A > 0 && npad >= A && (npad & (npad - 1)) == 0,                                                     \
                   fn ": npad=%d must be a power of two >= A=%d", npad, A);                                            \
    EFFDET_REQUIRE(cap <= A, fn ": cap=%d must be in [1, A=%d]", cap, A);                                              \
    EFFDET_REQUIRE(method == EFFDET_SOFT_NMS_LINEAR || method == EFFDET_SOFT_NMS_GAUSSIAN,                             \
                   fn ": method=%d must be EFFDET_SOFT_NMS_LINEAR (1) or EFFDET_SOFT_NMS_GAUSSIAN (2)", method);       \
    EFFDET_REQUIRE(method != EFFDET_SOFT_NMS_LINEAR || (iou_threshold >= 0.0 && iou_threshold <= 1.0),                 \
                   fn ": iou_threshold=%g must be in [0, 1] for the linear method", iou_threshold);                    \
    EFFDET_REQUIRE(sigma > 0.0 && sigma <= 1.7976931348623157e308, fn ": sigma=%g must be finite and > 0", sigma);     \
    const long long need = soft_workspace_bytes(B, cap);                                                               \
    EFFDET_REQUIRE(workspace_bytes >= need, fn ": workspace of %lld bytes, %lld needed", (long long)workspace_bytes,    \
                   need);                                                                                              \
    EFFDET_REQUIRE(need == 0 || workspace, fn ": null workspace, %lld bytes needed", need);                            \
    EFFDET_REQUIRE(aligned16(boxes) && aligned16(out_boxes) && aligned16(workspace),                                   \
                   fn ": boxes, out_boxes and workspace must be 16-byte aligned");                                     \
    EFFDET_DEVICE(device)

extern "C" int effdet_soft_nms_batch(const float* boxes, const float* scores, const int32_t* classes,
                                     const uint64_t* keys, const int32_t* count, int B, int A, int npad, int cap,
                                     int method, double iou_threshold, double sigma, float threshold, void* workspace,
                                     int64_t workspace_bytes, float* out_scores, int64_t* out_classes, float* out_boxes,
                                     int32_t* out_count, int device, effdet_stream_t stream) {
    SOFT_NMS_CHECKS("soft_nms_batch");
    return soft_nms_launch(boxes, scores, classes, keys, count, B, A, npad, cap, method, iou_threshold, sigma, threshold,
                           workspace, out_scores, out_classes, out_boxes, out_count, (cudaStream_t)stream);
}

extern "C" int effdet_soft_nms_batch_classes(const float* boxes, const float* scores, const int32_t* classes,
                                             const uint64_t* keys, const int32_t* count, int B, int A, int npad,
                                             int cap, int method, double iou_threshold, double sigma, float threshold,
                                             void* workspace, int64_t workspace_bytes, float* out_scores,
                                             int64_t* out_classes, float* out_boxes, int32_t* out_count, int device,
                                             effdet_stream_t stream) {
    SOFT_NMS_CHECKS("soft_nms_batch_classes");
    return soft_nms_launch(boxes, scores, classes, keys, count, B, A, npad, cap, method, iou_threshold, sigma, threshold,
                           workspace, out_scores, out_classes, out_boxes, out_count, (cudaStream_t)stream, true);
}
