// FocalLoss (focal BCE + smooth-L1 with IoU anchor assignment), forward and backward, replacing
// the per-image Python loop of ~25 full-size element-wise kernels and 2 host syncs per image.
// Reference: models/losses.py:6-26 (calc_iou), :32-152 (FocalLoss.forward).
// Bandwidth-bound on cls [B,A,K]: forward reads it once; backward reads it once and writes dcls.
#include <climits>

#include "block_scan.cuh"

namespace effdet {

constexpr int kMaxG = 256;  // annotations per image staged in shared memory

// IoU exactly as the reference's separate fp32 tensor ops (no FMA contraction).
__device__ __forceinline__ float iou_ref(float a0, float a1, float a2, float a3, float b0, float b1, float b2, float b3) {
    const float area_b = __fmul_rn(__fsub_rn(b2, b0), __fsub_rn(b3, b1));
    float iw = __fsub_rn(fminf(a2, b2), fmaxf(a0, b0));
    float ih = __fsub_rn(fminf(a3, b3), fmaxf(a1, b1));
    iw = fmaxf(iw, 0.f);
    ih = fmaxf(ih, 0.f);
    const float inter = __fmul_rn(iw, ih);
    float ua = __fsub_rn(__fadd_rn(__fmul_rn(__fsub_rn(a2, a0), __fsub_rn(a3, a1)), area_b), inter);
    ua = fmaxf(ua, 1e-8f);
    return __fdiv_rn(inter, ua);
}

// assign_ws[b,a]: >=0 annotation row of the matched box, -1 background (IoU<0.4),
// -2 ignored (0.4<=IoU<0.5), -3 image has no annotation.  stats[b,0] += #positives.
// COUNTED: counts = [n_img, rows of image 0, ...] in device memory (see counted_rows); images b >= n_img read nothing
// and write -3.  The table is staged in chunks of kMaxG rows, so any G works; without counts G <= kMaxG (one chunk).
__device__ __forceinline__ int counted_images(const int32_t* counts, int B) { return min(max(__ldg(counts), 1), B); }
__device__ __forceinline__ int counted_rows(const int32_t* counts, int b, int G) {
    return min(max(__ldg(counts + 1 + b), 0), G);
}

template <bool COUNTED>
__global__ void __launch_bounds__(256) loss_assign_kernel(const float* __restrict__ anchors, const float* __restrict__ annots,
                                                          const int32_t* __restrict__ counts, int32_t* __restrict__ assign,
                                                          float* __restrict__ stats, int B, int A, int G) {
    __shared__ float gt[kMaxG * 5];
    __shared__ int cnt_sh;
    const int b = blockIdx.y;
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (COUNTED && b >= counted_images(counts, B)) {                   // padding image (CTA-uniform exit)
        if (a < A) assign[(long long)b * A + a] = -3;
        return;
    }
    const int rows = COUNTED ? counted_rows(counts, b, G) : G;
    const float* img = annots + (long long)b * G * 5;
    if (threadIdx.x == 0) cnt_sh = 0;
    float4 an = f4zero();
    if (a < A) an = ldg4(anchors + (long long)a * 4);
    float best = 0.f;
    int arg = -1;
    for (int g0 = 0; g0 < rows; g0 += kMaxG) {
        const int n = min(kMaxG, rows - g0);
        __syncthreads();                                                 // the previous chunk is no longer read
        for (int i = threadIdx.x; i < n * 5; i += blockDim.x) gt[i] = __ldg(img + (long long)g0 * 5 + i);
        __syncthreads();
        if (a < A) {
            for (int g = 0; g < n; ++g) {
                if (gt[g * 5 + 4] == -1.f) continue;                       // losses.py:52
                const float v = iou_ref(an.x, an.y, an.z, an.w, gt[g * 5], gt[g * 5 + 1], gt[g * 5 + 2], gt[g * 5 + 3]);
                if (arg < 0 || v > best) { best = v; arg = g0 + g; }       // first maximum, like torch.max
            }
        }
    }
    __syncthreads();                                                     // cnt_sh = 0 before any warp adds to it
    int state = -3;
    if (a < A) {
        if (arg >= 0) state = best < 0.4f ? -1 : (best >= 0.5f ? arg : -2);   // :74-76
        assign[(long long)b * A + a] = state;
    }
    const unsigned pos = __ballot_sync(0xffffffffu, state >= 0);
    if ((threadIdx.x & 31) == 0 && pos) atomicAdd(&cnt_sh, __popc(pos));
    __syncthreads();
    if (threadIdx.x == 0 && cnt_sh) atomicAdd(stats + b * 4, (float)cnt_sh);
}

__device__ __forceinline__ float powg(float x, float gamma) { return gamma == 2.f ? x * x : powf(x, gamma); }

// one focal-BCE term and (optionally) its derivative w.r.t. the unclamped probability
template <bool GRAD>
__device__ __forceinline__ float focal_term(float p, bool is_target, float alpha, float gamma, float& grad) {
    const float pc = fminf(fmaxf(p, 1e-4f), 1.0f - 1e-4f);            // :60
    float l;
    if (is_target) {
        const float q = 1.f - pc, lg = logf(pc);
        const float fw = powg(q, gamma);
        l = alpha * fw * (-lg);
        if (GRAD) grad = alpha * (gamma * (gamma == 2.f ? q : powf(q, gamma - 1.f)) * lg - fw / pc);
    } else {
        const float lg = logf(1.f - pc);
        const float fw = powg(pc, gamma);
        l = (1.f - alpha) * fw * (-lg);
        if (GRAD) grad = (1.f - alpha) * (-gamma * (gamma == 2.f ? pc : powf(pc, gamma - 1.f)) * lg + fw / (1.f - pc));
    }
    if (GRAD && !(p >= 1e-4f && p <= 1.0f - 1e-4f)) grad = 0.f;      // clamp backward
    return l;
}

// VEC elements per thread (4 when K % 4 == 0, else 1); grid.y = image.  COUNTED: the mean runs over n_img images and
// a padding image b >= n_img reads nothing of cls and gets dcls = 0.
template <int VEC, bool GRAD, bool COUNTED>
__global__ void __launch_bounds__(256) loss_cls_kernel(const float* __restrict__ cls, const float* __restrict__ annots,
                                                       const int32_t* __restrict__ counts, const int32_t* __restrict__ assign,
                                                       float* __restrict__ stats_rw, const float* __restrict__ gout,
                                                       float* __restrict__ dcls, int B, int A, int K, int G, float alpha,
                                                       float gamma) {
    __shared__ float red[8];
    const int b = blockIdx.y;
    const int n_img = COUNTED ? counted_images(counts, B) : B;
    const long long per_img = (long long)A * K;
    const long long e = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * VEC;
    float lsum = 0.f;
    if (COUNTED && b >= n_img) {                                         // padding image (CTA-uniform)
        if (!GRAD) return;
        if (e < per_img) {
            const long long off = (long long)b * per_img + e;
            if (VEC == 4) st4(dcls + off, f4zero());
            else dcls[off] = 0.f;
        }
        return;
    }
    if (e < per_img) {
        const int a = (int)(e / K);
        const int k0 = (int)(e - (long long)a * K);
        const int state = __ldg(assign + (long long)b * A + a);
        const long long off = (long long)b * per_img + e;
        float v[VEC], g[VEC];
        if (VEC == 4) {
            const float4 q = ldg4(cls + off);
            v[0] = q.x; v[VEC > 1 ? 1 : 0] = q.y; v[VEC > 2 ? 2 : 0] = q.z; v[VEC > 3 ? 3 : 0] = q.w;
        } else {
            v[0] = __ldg(cls + off);
        }
        int label = -1;
        if (state >= 0) label = (int)__ldg(annots + ((long long)b * G + state) * 5 + 4);
        float gs = 0.f;
        if (GRAD) {
            const float npos = stats_rw[b * 4];
            gs = __ldg(gout) / (fmaxf(npos, 1.f) * (float)n_img);
        }
#pragma unroll
        for (int i = 0; i < VEC; ++i) {
            g[i] = 0.f;
            if (state >= -1) {                                           // -2 ignored, -3 no boxes: zero
                float gr = 0.f;
                const float l = focal_term<GRAD>(v[i], (k0 + i) == label, alpha, gamma, gr);
                lsum += l;
                g[i] = gr * gs;
            }
        }
        if (GRAD) {
            if (VEC == 4) st4(dcls + off, make_float4(g[0], g[VEC > 1 ? 1 : 0], g[VEC > 2 ? 2 : 0], g[VEC > 3 ? 3 : 0]));
            else dcls[off] = g[0];
        }
    }
    if (!GRAD) {
        lsum = warp_sum(lsum);
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = lsum;
        __syncthreads();
        if (threadIdx.x == 0) {
            float s = 0.f;
            for (int i = 0; i < 8; ++i) s += red[i];
            if (s != 0.f) atomicAdd(stats_rw + b * 4 + 1, s);
        }
    }
}

// COUNTED: the mean runs over n_img images; padding images have state -3 everywhere, so they read nothing of reg and
// get dreg = 0 from the same code.
template <bool GRAD, bool COUNTED>
__global__ void __launch_bounds__(256) loss_reg_kernel(const float* __restrict__ reg, const float* __restrict__ anchors,
                                                       const float* __restrict__ annots, const int32_t* __restrict__ counts,
                                                       const int32_t* __restrict__ assign, float* __restrict__ stats_rw,
                                                       const float* __restrict__ gout, float* __restrict__ dreg, int B, int A,
                                                       int G) {
    __shared__ float red[8];
    const int b = blockIdx.y;
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    float lsum = 0.f;
    if (a < A) {
        const int state = __ldg(assign + (long long)b * A + a);
        float4 gr = f4zero();
        if (state >= 0) {
            const float4 an = ldg4(anchors + (long long)a * 4);
            const float* gp = annots + ((long long)b * G + state) * 5;
            const float g0 = __ldg(gp), g1 = __ldg(gp + 1), g2 = __ldg(gp + 2), g3 = __ldg(gp + 3);
            const float aw = an.z - an.x, ah = an.w - an.y;
            const float acx = an.x + 0.5f * aw, acy = an.y + 0.5f * ah;
            float gw = g2 - g0, gh = g3 - g1;
            const float gcx = g0 + 0.5f * gw, gcy = g1 + 0.5f * gh;
            gw = fmaxf(gw, 1.f);                                          // :127-128
            gh = fmaxf(gh, 1.f);
            const float t[4] = {((gcx - acx) / aw) / 0.1f, ((gcy - acy) / ah) / 0.1f, logf(gw / aw) / 0.2f,
                                logf(gh / ah) / 0.2f};
            const float4 rv = ldg4(reg + ((long long)b * A + a) * 4);
            const float r[4] = {rv.x, rv.y, rv.z, rv.w};
            float gg[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float diff = r[i] - t[i];
                const float d = fabsf(diff);
                if (d <= 1.0f / 9.0f) { lsum += 0.5f * 9.0f * d * d; gg[i] = 9.0f * diff; }     // :140-146
                else { lsum += d - 0.5f / 9.0f; gg[i] = diff > 0.f ? 1.f : -1.f; }
            }
            if (GRAD) {
                const float npos = stats_rw[b * 4];
                const float gs = __ldg(gout + 1) / (4.f * npos * (float)(COUNTED ? counted_images(counts, B) : B));
                gr = make_float4(gg[0] * gs, gg[1] * gs, gg[2] * gs, gg[3] * gs);
            }
        }
        if (GRAD) st4(dreg + ((long long)b * A + a) * 4, gr);
    }
    if (!GRAD) {
        lsum = warp_sum(lsum);
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = lsum;
        __syncthreads();
        if (threadIdx.x == 0) {
            float s = 0.f;
            for (int i = 0; i < 8; ++i) s += red[i];
            if (s != 0.f) atomicAdd(stats_rw + b * 4 + 2, s);
        }
    }
}

// counts NULL: the mean over B images; otherwise over n_img = counts[0]
__global__ void loss_finalize_kernel(const float* __restrict__ stats, const int32_t* __restrict__ counts,
                                     float* __restrict__ losses, int B) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    if (counts) B = counted_images(counts, B);
    float c = 0.f, r = 0.f;
    for (int b = 0; b < B; ++b) {
        const float npos = stats[b * 4];
        c += stats[b * 4 + 1] / fmaxf(npos, 1.f);                        // :103-104
        if (npos > 0.f) r += stats[b * 4 + 2] / (4.f * npos);            // :147
    }
    losses[0] = c / (float)B;                                            // :152
    losses[1] = r / (float)B;
}

__global__ void __launch_bounds__(256) sigmoid_bwd_kernel(const float* __restrict__ g, const float* __restrict__ p,
                                                          float* __restrict__ y, long long n4) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const float4 gv = ldg4(g + i * 4), pv = ldg4(p + i * 4);
        st4(y + i * 4, make_float4(gv.x * pv.x * (1.f - pv.x), gv.y * pv.y * (1.f - pv.y), gv.z * pv.z * (1.f - pv.z),
                                   gv.w * pv.w * (1.f - pv.w)));
    }
}

// Stable compaction of one image's rows whose label is not -1 into the front of its [Gcap,5] slot, -1 rows after them;
// counts[1+b] = rows kept (0 for b >= B), counts[0] = B.  One CTA per slot b < Bcap.
__global__ void __launch_bounds__(256) pack_annots_kernel(const float* __restrict__ annots, int B, int G,
                                                          float* __restrict__ out, int32_t* __restrict__ counts, int Gcap) {
    __shared__ int warp_tot[32];
    const int b = blockIdx.x;
    float* dst = out + (long long)b * Gcap * 5;
    int kept = 0;
    if (b < B) {
        const float* src = annots + (long long)b * G * 5;
        for (int r0 = 0; r0 < G; r0 += blockDim.x) {                    // CTA-uniform trip count
            const int r = r0 + threadIdx.x;
            const bool keep = r < G && __ldg(src + (long long)r * 5 + 4) != -1.f;
            int total;
            const int incl = block_scan(keep ? 1 : 0, warp_tot, IntAdd(), total);
            if (keep) {
                const int at = kept + incl - 1;
#pragma unroll
                for (int c = 0; c < 5; ++c) dst[(long long)at * 5 + c] = __ldg(src + (long long)r * 5 + c);
            }
            kept += total;
        }
    }
    for (long long i = (long long)kept * 5 + threadIdx.x; i < (long long)Gcap * 5; i += blockDim.x) dst[i] = -1.f;
    if (threadIdx.x == 0) {
        counts[1 + b] = kept;
        if (b == 0) counts[0] = B;
    }
}

}  // namespace effdet

using namespace effdet;

static int loss_check(const char* who, int B, int A, int K, int G) {
    EFFDET_REQUIRE(B > 0 && B <= 65535 && A > 0 && K > 0, "%s: bad shape", who);
    EFFDET_REQUIRE(G > 0 && G <= kMaxG, "%s: G=%d annotations per image unsupported (1..%d)", who, G, kMaxG);
    return EFFDET_OK;
}

// the counted pair stages the table in chunks: G is bounded only by the int row offsets (G * 5 within int)
static int counted_check(const char* who, int B, int A, int K, int G) {
    EFFDET_REQUIRE(B > 0 && B <= 65535, "%s: B=%d images unsupported (1..65535)", who, B);
    EFFDET_REQUIRE(A > 0 && K > 0, "%s: bad shape (A=%d, K=%d)", who, A, K);
    EFFDET_REQUIRE(G > 0 && G <= INT_MAX / 5, "%s: G=%d annotation rows unsupported (1..%d)", who, G, INT_MAX / 5);
    return EFFDET_OK;
}

// the launches of the forward and backward; counts is NULL for the uncounted pair (COUNTED = false)
template <bool COUNTED>
static int focal_fwd_launch(const float* cls, const float* reg, const float* anchors, const float* annots,
                            const int32_t* counts, float* losses, int32_t* assign_ws, float* stats_ws, int B, int A, int K,
                            int G, float alpha, float gamma, cudaStream_t st) {
    int s;
    cudaError_t e = cudaMemsetAsync(stats_ws, 0, sizeof(float) * 4 * B, st);
    if (e != cudaSuccess) return fail(EFFDET_ERR_LAUNCH, "focal_loss_fwd: memset: %s", cudaGetErrorString(e));
    loss_assign_kernel<COUNTED><<<dim3(cdiv(A, 256), B), 256, 0, st>>>(anchors, annots, counts, assign_ws, stats_ws, B, A, G);
    if ((s = launch_status("loss_assign_kernel"))) return s;
    const long long per_img = (long long)A * K;
    if (K % 4 == 0)
        loss_cls_kernel<4, false, COUNTED><<<dim3(cdiv(per_img / 4, 256), B), 256, 0, st>>>(
            cls, annots, counts, assign_ws, stats_ws, nullptr, nullptr, B, A, K, G, alpha, gamma);
    else
        loss_cls_kernel<1, false, COUNTED><<<dim3(cdiv(per_img, 256), B), 256, 0, st>>>(
            cls, annots, counts, assign_ws, stats_ws, nullptr, nullptr, B, A, K, G, alpha, gamma);
    if ((s = launch_status("loss_cls_kernel"))) return s;
    loss_reg_kernel<false, COUNTED><<<dim3(cdiv(A, 256), B), 256, 0, st>>>(reg, anchors, annots, counts, assign_ws, stats_ws,
                                                                          nullptr, nullptr, B, A, G);
    if ((s = launch_status("loss_reg_kernel"))) return s;
    loss_finalize_kernel<<<1, 32, 0, st>>>(stats_ws, counts, losses, B);
    return launch_status("loss_finalize_kernel");
}

template <bool COUNTED>
static int focal_bwd_launch(const float* cls, const float* reg, const float* anchors, const float* annots,
                            const int32_t* counts, const float* gout, const int32_t* assign_ws, const float* stats_ws,
                            float* dcls, float* dreg, int B, int A, int K, int G, float alpha, float gamma, cudaStream_t st) {
    int s;
    float* stats = const_cast<float*>(stats_ws);
    const long long per_img = (long long)A * K;
    if (K % 4 == 0)
        loss_cls_kernel<4, true, COUNTED><<<dim3(cdiv(per_img / 4, 256), B), 256, 0, st>>>(
            cls, annots, counts, assign_ws, stats, gout, dcls, B, A, K, G, alpha, gamma);
    else
        loss_cls_kernel<1, true, COUNTED><<<dim3(cdiv(per_img, 256), B), 256, 0, st>>>(
            cls, annots, counts, assign_ws, stats, gout, dcls, B, A, K, G, alpha, gamma);
    if ((s = launch_status("loss_cls_kernel<grad>"))) return s;
    loss_reg_kernel<true, COUNTED><<<dim3(cdiv(A, 256), B), 256, 0, st>>>(reg, anchors, annots, counts, assign_ws, stats, gout,
                                                                         dreg, B, A, G);
    return launch_status("loss_reg_kernel<grad>");
}

extern "C" int effdet_focal_loss_fwd(const float* cls, const float* reg, const float* anchors, const float* annots,
                                     float* losses, int32_t* assign_ws, float* stats_ws, int B, int A, int K, int G,
                                     float alpha, float gamma, int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(cls && reg && anchors && annots && losses && assign_ws && stats_ws, "focal_loss_fwd: null tensor");
    EFFDET_REQUIRE(aligned16(cls) && aligned16(reg) && aligned16(anchors), "focal_loss_fwd: alignment");
    int s = loss_check("focal_loss_fwd", B, A, K, G);
    if (s) return s;
    EFFDET_DEVICE(device);
    return focal_fwd_launch<false>(cls, reg, anchors, annots, nullptr, losses, assign_ws, stats_ws, B, A, K, G, alpha, gamma,
                                   (cudaStream_t)stream);
}

extern "C" int effdet_focal_loss_bwd(const float* cls, const float* reg, const float* anchors, const float* annots,
                                     const float* gout, const int32_t* assign_ws, const float* stats_ws, float* dcls,
                                     float* dreg, int B, int A, int K, int G, float alpha, float gamma, int device,
                                     effdet_stream_t stream) {
    EFFDET_REQUIRE(cls && reg && anchors && annots && gout && assign_ws && stats_ws && dcls && dreg,
                   "focal_loss_bwd: null tensor");
    EFFDET_REQUIRE(aligned16(cls) && aligned16(reg) && aligned16(anchors) && aligned16(dcls) && aligned16(dreg),
                   "focal_loss_bwd: alignment");
    int s = loss_check("focal_loss_bwd", B, A, K, G);
    if (s) return s;
    EFFDET_DEVICE(device);
    return focal_bwd_launch<false>(cls, reg, anchors, annots, nullptr, gout, assign_ws, stats_ws, dcls, dreg, B, A, K, G,
                                   alpha, gamma, (cudaStream_t)stream);
}

extern "C" int effdet_focal_loss_counted_fwd(const float* cls, const float* reg, const float* anchors, const float* annots,
                                             const int32_t* counts, float* losses, int32_t* assign_ws, float* stats_ws,
                                             int B, int A, int K, int G, float alpha, float gamma, int device,
                                             effdet_stream_t stream) {
    EFFDET_REQUIRE(cls && reg && anchors && annots && counts && losses && assign_ws && stats_ws,
                   "focal_loss_counted_fwd: null tensor");
    EFFDET_REQUIRE(aligned16(cls) && aligned16(reg) && aligned16(anchors), "focal_loss_counted_fwd: alignment");
    int s = counted_check("focal_loss_counted_fwd", B, A, K, G);
    if (s) return s;
    EFFDET_DEVICE(device);
    return focal_fwd_launch<true>(cls, reg, anchors, annots, counts, losses, assign_ws, stats_ws, B, A, K, G, alpha, gamma,
                                  (cudaStream_t)stream);
}

extern "C" int effdet_focal_loss_counted_bwd(const float* cls, const float* reg, const float* anchors, const float* annots,
                                             const int32_t* counts, const float* gout, const int32_t* assign_ws,
                                             const float* stats_ws, float* dcls, float* dreg, int B, int A, int K, int G,
                                             float alpha, float gamma, int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(cls && reg && anchors && annots && counts && gout && assign_ws && stats_ws && dcls && dreg,
                   "focal_loss_counted_bwd: null tensor");
    EFFDET_REQUIRE(aligned16(cls) && aligned16(reg) && aligned16(anchors) && aligned16(dcls) && aligned16(dreg),
                   "focal_loss_counted_bwd: alignment");
    int s = counted_check("focal_loss_counted_bwd", B, A, K, G);
    if (s) return s;
    EFFDET_DEVICE(device);
    return focal_bwd_launch<true>(cls, reg, anchors, annots, counts, gout, assign_ws, stats_ws, dcls, dreg, B, A, K, G, alpha,
                                  gamma, (cudaStream_t)stream);
}

extern "C" int effdet_pack_annots(const float* annots, int B, int G, float* out, int32_t* counts, int Bcap, int Gcap,
                                  int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(annots && out && counts, "pack_annots: null tensor");
    EFFDET_REQUIRE(Bcap > 0 && Bcap <= 65535 && Gcap > 0 && Gcap <= INT_MAX / 5,
                   "pack_annots: capacity Bcap=%d, Gcap=%d unsupported (1..65535, 1..%d)", Bcap, Gcap, INT_MAX / 5);
    EFFDET_REQUIRE(B > 0 && B <= Bcap, "pack_annots: B=%d images do not fit the capacity of %d", B, Bcap);
    EFFDET_REQUIRE(G > 0 && G <= Gcap,
                   "pack_annots: G=%d annotation rows do not fit max_annotations=%d (max_annotations=%d would be enough)", G,
                   Gcap, G);
    EFFDET_DEVICE(device);
    pack_annots_kernel<<<Bcap, 256, 0, (cudaStream_t)stream>>>(annots, B, G, out, counts, Gcap);
    return launch_status("pack_annots_kernel");
}

extern "C" int effdet_sigmoid_bwd(const float* g, const float* p, float* y, int64_t n, int device,
                                  effdet_stream_t stream) {
    EFFDET_REQUIRE(g && p && y && n > 0 && n % 4 == 0, "sigmoid_bwd: bad arguments (n must be a multiple of 4)");
    EFFDET_REQUIRE(aligned16(g) && aligned16(p) && aligned16(y), "sigmoid_bwd: alignment");
    EFFDET_DEVICE(device);
    int blocks = cdiv(n / 4, 256);
    if (blocks > num_sms() * 16) blocks = num_sms() * 16;
    sigmoid_bwd_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(g, p, y, n / 4);
    return launch_status("sigmoid_bwd_kernel");
}
