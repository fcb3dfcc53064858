// The step before the hot path, on the device (SURVEY.md 8(f) rank 2):
//   input side  : Normalizer + Augmenter (horizontal flip) + zero-pad to the common size + collater + `.cuda().float()`
//                 datasets/augmentation.py:69-91,111-150, train.py:105-106.  normalize_pad_kernel takes images at their
//                 final resolution; resize_normalize_pad_kernel also runs Resizer's cv2.resize, so everything after the
//                 decode is done here.
// (the output side, eval.py's selection, is in voc_eval.cu)
// Arithmetic follows the reference's dtypes exactly so the results are bit-identical to NumPy:
//   Normalizer computes (img.astype(float32) - mean[float64]) / std[float64] in float64 and train.py casts to float32 on
//   the device; collater writes float64 annotations into a float32 tensor.
#include <cfloat>
#include <climits>

#include "block_scan.cuh"
#include "common.cuh"

namespace effdet {

// one thread per output pixel (x fastest): reads 3 interleaved bytes, writes the three channel planes
__global__ void __launch_bounds__(256) normalize_pad_kernel(const uint8_t* __restrict__ pix, const int64_t* __restrict__ offs,
                                                            const int32_t* __restrict__ hw, const uint8_t* __restrict__ flip,
                                                            float* __restrict__ out, int S, double m0, double m1, double m2,
                                                            double s0, double s1, double s2) {
    const int b = blockIdx.z;
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    if (x >= S) return;
    const int h = hw[2 * b], w = hw[2 * b + 1];
    float v0 = 0.f, v1 = 0.f, v2 = 0.f;                              // np.zeros((S, S, 3)) padding
    if (y < h && x < w) {
        const int sx = (flip && flip[b]) ? (w - 1 - x) : x;          // image[:, ::-1, :]
        const uint8_t* p = pix + offs[b] + ((long long)y * w + sx) * 3;
        // (float32(u8) - mean) / std in float64 (exact subtraction, IEEE division), then the .float() of train.py:105
        v0 = (float)__ddiv_rn(__dsub_rn((double)(float)p[0], m0), s0);
        v1 = (float)__ddiv_rn(__dsub_rn((double)(float)p[1], m1), s1);
        v2 = (float)__ddiv_rn(__dsub_rn((double)(float)p[2], m2), s2);
    }
    const long long plane = (long long)S * S;
    float* o = out + (long long)b * 3 * plane + (long long)y * S + x;
    o[0] = v0;
    o[plane] = v1;
    o[2 * plane] = v2;
}

// Normalizer -> Augmenter flip -> Resizer (cv2.resize INTER_LINEAR on the float64 image, then the zero pad) -> .float(),
// datasets/augmentation.py:94-115,118-150.  The resize is OpenCV's generic (non-SIMD, non-IPP) algorithm for CV_64FC3:
//   same size            : copy
//   src/dst == 2 on both : INTER_AREA's 2x2 box, (((S00 + S01) + S10) + S11) * 0.25
//   otherwise            : per axis f = float((d + 0.5) * (1 / (dst / src)) - 0.5), s = floor(f), f -= s (float32),
//                          taps (1 - f, f) in float32.  Columns clamp s < 0 to (0, 0) and are single-tap from s + 1 >= w
//                          on (s >= w - 1 -> s = w - 1); rows keep f and clamp both row indices into [0, h - 1].
//                          D = H(r0) * b0 + H(r1) * b1 with H(r) = S[r][s] * a0 + S[r][s + 1] * a1, every float64
//                          product and sum rounded on its own (no FMA contraction).
// The input of the Normalizer is float32(u8) (COCO) or float32(u8) / 255.f (VOC, datasets/voc0712.py:109); since it
// only depends on the byte, each block first tabulates the 3 x 256 normalized float64 values in shared memory.
// One thread per output pixel (x fastest); each reads at most 4 source pixels, whose bytes stay in L1/L2.
// kCrop (scale jitter): output pixel (y, x) is pixel (y + y0, x + x0) of the resized image, (y0, x0) = crops[b], and 0
// where that lies outside it (the window past the resized image, or a negative offset).  Without kCrop, y0 = x0 = 0.
template <bool kCrop>
__device__ __forceinline__ void resize_normalize_pad_body(const uint8_t* __restrict__ pix, const int64_t* __restrict__ offs,
                                                          const int32_t* __restrict__ hw, const int32_t* __restrict__ rhw,
                                                          const int32_t* __restrict__ crops, const uint8_t* __restrict__ flip,
                                                          float* __restrict__ out, int S, int div255, double m0, double m1,
                                                          double m2, double s0, double s1, double s2) {
    __shared__ double lut[3][256];
    const int b = blockIdx.z;
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    const int h = hw[2 * b], w = hw[2 * b + 1], rh = rhw[2 * b], rw = rhw[2 * b + 1];
    const long long plane = (long long)S * S;
    float* o = out + (long long)b * 3 * plane + (long long)y * S + x;
    const int y0 = kCrop ? crops[2 * b] : 0, x0 = kCrop ? crops[2 * b + 1] : 0;
    const int Y = y + y0;                                               // the row of the resized image
    if (Y >= rh || h <= 0 || w <= 0 || (kCrop && (y0 < 0 || x0 < 0))) { // block-uniform: a padding row
        if (x < S) o[0] = o[plane] = o[2 * plane] = 0.f;
        return;
    }
    for (int i = threadIdx.x; i < 3 * 256; i += blockDim.x) {
        const int c = i >> 8;
        float v = (float)(i & 255);
        if (div255) v = __fdiv_rn(v, 255.f);                             // img.astype(np.float32) / 255.
        const double m = c == 0 ? m0 : (c == 1 ? m1 : m2), s = c == 0 ? s0 : (c == 1 ? s1 : s2);
        lut[c][i & 255] = __ddiv_rn(__dsub_rn((double)v, m), s);
    }
    __syncthreads();
    if (x >= S) return;
    const int X = x + x0;                                               // the column of the resized image
    double v[3] = {0.0, 0.0, 0.0};                                      // np.zeros((S, S, 3)) padding
    if (X < rw) {
        const uint8_t* img = pix + offs[b];
        const bool fl = flip && flip[b];
        // source pixel (r, c) of the flipped image: image[:, ::-1, :]
        auto px = [&](int r, int c) { return img + ((long long)r * w + (fl ? w - 1 - c : c)) * 3; };
        const double scale_x = __ddiv_rn(1.0, __ddiv_rn((double)rw, (double)w));
        const double scale_y = __ddiv_rn(1.0, __ddiv_rn((double)rh, (double)h));
        if (rh == h && rw == w) {
            const uint8_t* p = px(Y, X);
            for (int c = 0; c < 3; ++c) v[c] = lut[c][p[c]];
        } else if (fabs(__dsub_rn(scale_x, 2.0)) < DBL_EPSILON && fabs(__dsub_rn(scale_y, 2.0)) < DBL_EPSILON) {
            const uint8_t *p00 = px(2 * Y, 2 * X), *p01 = px(2 * Y, 2 * X + 1);
            const uint8_t *p10 = px(2 * Y + 1, 2 * X), *p11 = px(2 * Y + 1, 2 * X + 1);
            for (int c = 0; c < 3; ++c)
                v[c] = __dmul_rn(__dadd_rn(__dadd_rn(__dadd_rn(lut[c][p00[c]], lut[c][p01[c]]), lut[c][p10[c]]), lut[c][p11[c]]),
                                 0.25);
        } else {
            float fx = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn((double)X, 0.5), scale_x), 0.5));
            int sx = (int)floorf(fx);
            fx = __fsub_rn(fx, (float)sx);
            if (sx < 0) fx = 0.f, sx = 0;
            const bool single = sx + 1 >= w;
            if (sx >= w - 1) fx = 0.f, sx = w - 1;
            float fy = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn((double)Y, 0.5), scale_y), 0.5));
            const int sy = (int)floorf(fy);
            fy = __fsub_rn(fy, (float)sy);
            const int r0 = min(max(sy, 0), h - 1), r1 = min(max(sy + 1, 0), h - 1);
            const double a0 = (double)__fsub_rn(1.f, fx), a1 = (double)fx;
            const double b0 = (double)__fsub_rn(1.f, fy), b1 = (double)fy;
            const uint8_t *q0 = px(r0, sx), *q1 = px(r1, sx);
            const uint8_t *q0n = single ? q0 : px(r0, sx + 1), *q1n = single ? q1 : px(r1, sx + 1);
            for (int c = 0; c < 3; ++c) {
                const double h0 = single ? lut[c][q0[c]] : __dadd_rn(__dmul_rn(lut[c][q0[c]], a0), __dmul_rn(lut[c][q0n[c]], a1));
                const double h1 = single ? lut[c][q1[c]] : __dadd_rn(__dmul_rn(lut[c][q1[c]], a0), __dmul_rn(lut[c][q1n[c]], a1));
                v[c] = __dadd_rn(__dmul_rn(h0, b0), __dmul_rn(h1, b1));
            }
        }
    }
    o[0] = (float)v[0];                                                 // the .float() of train.py:105
    o[plane] = (float)v[1];
    o[2 * plane] = (float)v[2];
}

__global__ void __launch_bounds__(256) resize_normalize_pad_kernel(const uint8_t* __restrict__ pix, const int64_t* __restrict__ offs,
                                                                   const int32_t* __restrict__ hw, const int32_t* __restrict__ rhw,
                                                                   const uint8_t* __restrict__ flip, float* __restrict__ out, int S,
                                                                   int div255, double m0, double m1, double m2, double s0,
                                                                   double s1, double s2) {
    resize_normalize_pad_body<false>(pix, offs, hw, rhw, nullptr, flip, out, S, div255, m0, m1, m2, s0, s1, s2);
}

// Scale jitter: the S x S window at crops[b] = (y0, x0) of the image resized to resized_hw[b] (Resizer at the drawn
// common size L), zero where the window runs past it.
__global__ void __launch_bounds__(256) resize_crop_normalize_pad_kernel(const uint8_t* __restrict__ pix,
                                                                        const int64_t* __restrict__ offs,
                                                                        const int32_t* __restrict__ hw,
                                                                        const int32_t* __restrict__ rhw,
                                                                        const int32_t* __restrict__ crops,
                                                                        const uint8_t* __restrict__ flip,
                                                                        float* __restrict__ out, int S, int div255, double m0,
                                                                        double m1, double m2, double s0, double s1, double s2) {
    resize_normalize_pad_body<true>(pix, offs, hw, rhw, crops, flip, out, S, div255, m0, m1, m2, s0, s1, s2);
}

// demo.py's test transform, get_augumentation(phase='test') (datasets/augmentation.py:38-48, albumentations 0.5.2):
// Resize(H, W) = cv2.resize(frame, (W, H), INTER_LINEAR) on the uint8 BGR frame, then Normalize and ToTensor in float32.
// Unlike Resizer's float64 resize above, OpenCV resizes CV_8U in fixed point (tools/frame_oracle.py states the rules):
//   same size            : copy
//   src/dst == 2 on both : INTER_AREA's 2x2 box, (S00 + S01 + S10 + S11 + 2) >> 2
//   otherwise            : per axis f = float((d + 0.5) * (1 / (dst / src)) - 0.5), s = floor(f), f -= s (float32);
//                          columns clamp s < 0 to (0, 0) and s >= w - 1 to (w - 1, 0), second tap clamped to w - 1;
//                          rows keep f and clamp both row indices into [0, h - 1].  Taps a = rint((1 - f) * 2048),
//                          rint(f * 2048); H(r) = S[r][s] * a0 + S[r][s + 1] * a1 (int32, scale 2^11);
//                          out = ((((H(r0) >> 4) * b0) >> 16) + (((H(r1) >> 4) * b1) >> 16) + 2) >> 2, OpenCV's vector
//                          rounding (the scalar (H0 * b0 + H1 * b1 + 2^21) >> 22 differs in about a third of the pixels).
// Normalize: mean * 255 and std * 255 in float32, den = 1 / (std * 255) rounded once, then (float(u8) - mean) * den, each
// step rounded on its own (no FMA).  The channels keep the frame's byte order (BGR from cv2.imread).
// One thread per output pixel (x fastest), at most 4 source pixels each; a frame with h == 0 is padding and writes zeros.
__global__ void __launch_bounds__(256) frame_transform_kernel(const uint8_t* __restrict__ pix, const int64_t* __restrict__ offs,
                                                              const int32_t* __restrict__ hw, float* __restrict__ out, int H,
                                                              int W, float m0, float m1, float m2, float s0, float s1,
                                                              float s2) {
    const int b = blockIdx.z;
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    if (x >= W) return;
    const int h = hw[2 * b], w = hw[2 * b + 1];
    const long long plane = (long long)H * W;
    float* o = out + (long long)b * 3 * plane + (long long)y * W + x;
    if (h <= 0 || w <= 0) {
        o[0] = o[plane] = o[2 * plane] = 0.f;
        return;
    }
    const uint8_t* img = pix + offs[b];
    auto px = [&](int r, int c) { return img + ((long long)r * w + c) * 3; };
    int v[3];
    const double scale_x = __ddiv_rn(1.0, __ddiv_rn((double)W, (double)w));
    const double scale_y = __ddiv_rn(1.0, __ddiv_rn((double)H, (double)h));
    if (h == H && w == W) {
        const uint8_t* p = px(y, x);
        for (int c = 0; c < 3; ++c) v[c] = p[c];
    } else if (fabs(__dsub_rn(scale_x, 2.0)) < DBL_EPSILON && fabs(__dsub_rn(scale_y, 2.0)) < DBL_EPSILON) {
        const uint8_t *p00 = px(2 * y, 2 * x), *p01 = px(2 * y, 2 * x + 1);
        const uint8_t *p10 = px(2 * y + 1, 2 * x), *p11 = px(2 * y + 1, 2 * x + 1);
        for (int c = 0; c < 3; ++c) v[c] = (p00[c] + p01[c] + p10[c] + p11[c] + 2) >> 2;
    } else {
        float fx = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn((double)x, 0.5), scale_x), 0.5));
        int sx = (int)floorf(fx);
        fx = __fsub_rn(fx, (float)sx);
        if (sx < 0) fx = 0.f, sx = 0;
        if (sx >= w - 1) fx = 0.f, sx = w - 1;
        const int sx1 = min(sx + 1, w - 1);
        float fy = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn((double)y, 0.5), scale_y), 0.5));
        const int sy = (int)floorf(fy);
        fy = __fsub_rn(fy, (float)sy);
        const int r0 = min(max(sy, 0), h - 1), r1 = min(max(sy + 1, 0), h - 1);
        const int a0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, fx), 2048.f)), a1 = __float2int_rn(__fmul_rn(fx, 2048.f));
        const int b0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, fy), 2048.f)), b1 = __float2int_rn(__fmul_rn(fy, 2048.f));
        const uint8_t *q00 = px(r0, sx), *q01 = px(r0, sx1), *q10 = px(r1, sx), *q11 = px(r1, sx1);
        for (int c = 0; c < 3; ++c) {
            const int h0 = q00[c] * a0 + q01[c] * a1, h1 = q10[c] * a0 + q11[c] * a1;
            v[c] = min(max((((h0 >> 4) * b0 >> 16) + ((h1 >> 4) * b1 >> 16) + 2) >> 2, 0), 255);
        }
    }
    const float mean[3] = {__fmul_rn(m0, 255.f), __fmul_rn(m1, 255.f), __fmul_rn(m2, 255.f)};
    const float den[3] = {__frcp_rn(__fmul_rn(s0, 255.f)), __frcp_rn(__fmul_rn(s1, 255.f)), __frcp_rn(__fmul_rn(s2, 255.f))};
    for (int c = 0; c < 3; ++c) o[c * plane] = __fmul_rn(__fsub_rn((float)v[c], mean[c]), den[c]);
}

// demo.py:86-104 on the padded detections of a batch of frames: per kept row of frame b (h x w), in network-input
// pixels of an H x W input,
//   x = int(bbox[0] * w / W) (and y1, x2, y2 likewise), float32 product and quotient (NumPy >= 2, NEP 50), truncated;
//   score = int(np.around(s, 2) * 100) = trunc(rint(s * 100) / 100 * 100) in float32, rint half to even;
//   label = the row's class.
// rows [B, C, 6] int32 (x1, y1, x2, y2, label, score): rows past out_count[b] are not written.  out_count[b] = count[b],
// 0 for a padding frame (h == 0), -1 when the frame overflowed the candidate cap.  Grid (C / 256, B).
__global__ void __launch_bounds__(256) frame_boxes_kernel(const float* __restrict__ scores, const int64_t* __restrict__ classes,
                                                          const float4* __restrict__ boxes, const int32_t* __restrict__ count,
                                                          const int32_t* __restrict__ hw, int32_t* __restrict__ rows,
                                                          int32_t* __restrict__ out_count, int C, float H, float W) {
    const int b = blockIdx.y;
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    const int h = hw[2 * b], w = hw[2 * b + 1];
    const int n = h > 0 ? count[b] : 0;
    if (k == 0) out_count[b] = n;
    if (k >= n || k >= C) return;
    const long long i = (long long)b * C + k;
    const float4 bx = boxes[i];
    const float fw = (float)w, fh = (float)h;
    int32_t* r = rows + i * 6;
    r[0] = (int)__fdiv_rn(__fmul_rn(bx.x, fw), W);
    r[1] = (int)__fdiv_rn(__fmul_rn(bx.y, fh), H);
    r[2] = (int)__fdiv_rn(__fmul_rn(bx.z, fw), W);
    r[3] = (int)__fdiv_rn(__fmul_rn(bx.w, fh), H);
    r[4] = (int)classes[i];
    r[5] = (int)__fmul_rn(__fdiv_rn(rintf(__fmul_rn(scores[i], 100.f)), 100.f), 100.f);
}

// annotations: rows [n_b, 5] float64 (x1, y1, x2, y2, label) concatenated over the batch -> float32 [B, G, 5], -1 padded.
// Resizer scales the box by `scale` (float64), Augmenter mirrors x about the image width BEFORE the resize.
__global__ void collate_annots_kernel(const double* __restrict__ rows, const int32_t* __restrict__ row_off,
                                      const double* __restrict__ scale, const uint8_t* __restrict__ flip,
                                      const int32_t* __restrict__ width, float* __restrict__ out, int B, int G) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * G) return;
    const int b = i / G, g = i - b * G;
    const int n = row_off[b + 1] - row_off[b];
    float* o = out + (long long)i * 5;
    if (g >= n) {
        o[0] = o[1] = o[2] = o[3] = o[4] = -1.f;
        return;
    }
    const double* r = rows + (long long)(row_off[b] + g) * 5;
    double x1 = r[0], y1 = r[1], x2 = r[2], y2 = r[3];
    if (flip && flip[b]) {                                            // annots[:, 0] = cols - x2 ; annots[:, 2] = cols - x1
        const double cols = (double)width[b];
        const double nx1 = __dsub_rn(cols, x2), nx2 = __dsub_rn(cols, x1);
        x1 = nx1;
        x2 = nx2;
    }
    const double sc = scale ? scale[b] : 1.0;                         // annots[:, :4] *= scale
    o[0] = (float)__dmul_rn(x1, sc);
    o[1] = (float)__dmul_rn(y1, sc);
    o[2] = (float)__dmul_rn(x2, sc);
    o[3] = (float)__dmul_rn(y2, sc);
    o[4] = (float)r[4];
}

// collate_annots_kernel followed by pack_annots_kernel (loss.cu) in one pass, for the annotation sections of a raw batch
// (models/pipeline.py RawBatch): B = header[0] images; image b owns rows row_off[b] .. row_off[b+1].  Each row is
// flipped (fp64, before the scale), scaled by __dmul_rn and cast to float32 exactly as collate_annots_kernel does, then
// kept unless its float32 label is -1, in order, into the front of slot b of out [Bcap,Gcap,5], -1 rows after them.
// counts[1+b] = rows kept (0 for b >= B), counts[0] = B.  One CTA per slot b < Bcap; every image has <= Gcap rows (the
// host checks it).
// kCrop (scale jitter): after the scale, x1/x2 -= x0 and y1/y2 -= y0 ((y0, x0) = crops[b]), each coordinate clamped to
// [0, S] (S = header[4]), all in float64, then the one cast to float32; a row is kept only if, in float32, its label is
// not -1, x2 > x1 and y2 > y1.  A NaN coordinate stays NaN through the clamp, so its row is dropped.
template <bool kCrop>
__device__ __forceinline__ void collate_pack_annots_body(const int64_t* __restrict__ header, const double* __restrict__ rows,
                                                         const int32_t* __restrict__ row_off, const double* __restrict__ scale,
                                                         const uint8_t* __restrict__ flip, const int32_t* __restrict__ hw,
                                                         const int32_t* __restrict__ crops, float* __restrict__ out,
                                                         int32_t* __restrict__ counts, int Gcap) {
    __shared__ int warp_tot[32];
    const int b = blockIdx.x;
    const int B = (int)header[0];
    float* dst = out + (long long)b * Gcap * 5;
    int kept = 0;
    if (b < B) {
        const int r_begin = row_off[b], n = row_off[b + 1] - r_begin;
        const bool fl = flip[b] != 0;
        const double cols = (double)hw[2 * b + 1], sc = scale[b];
        const double y0 = kCrop ? (double)crops[2 * b] : 0.0, x0 = kCrop ? (double)crops[2 * b + 1] : 0.0;
        const double S = kCrop ? (double)header[4] : 0.0;
        auto crop = [&](double v, double o) {                           // v - o, clamped to [0, S] (NaN passes)
            const double c = __dsub_rn(v, o);
            return c < 0.0 ? 0.0 : (c > S ? S : c);
        };
        for (int g0 = 0; g0 < n; g0 += blockDim.x) {                    // CTA-uniform trip count
            const int g = g0 + threadIdx.x;
            float v[5];
            bool keep = false;
            if (g < n) {
                const double* r = rows + (long long)(r_begin + g) * 5;
                double x1 = r[0], x2 = r[2];
                if (fl) {                                               // annots[:, 0] = cols - x2 ; annots[:, 2] = cols - x1
                    const double nx1 = __dsub_rn(cols, x2), nx2 = __dsub_rn(cols, x1);
                    x1 = nx1;
                    x2 = nx2;
                }
                if (kCrop) {
                    v[0] = (float)crop(__dmul_rn(x1, sc), x0);
                    v[1] = (float)crop(__dmul_rn(r[1], sc), y0);
                    v[2] = (float)crop(__dmul_rn(x2, sc), x0);
                    v[3] = (float)crop(__dmul_rn(r[3], sc), y0);
                } else {
                    v[0] = (float)__dmul_rn(x1, sc);                    // annots[:, :4] *= scale, then the float32 table
                    v[1] = (float)__dmul_rn(r[1], sc);
                    v[2] = (float)__dmul_rn(x2, sc);
                    v[3] = (float)__dmul_rn(r[3], sc);
                }
                v[4] = (float)r[4];
                keep = v[4] != -1.f && (!kCrop || (v[2] > v[0] && v[3] > v[1]));
            }
            int total;
            const int incl = block_scan(keep ? 1 : 0, warp_tot, IntAdd(), total);
            if (keep) {
                float* o = dst + (long long)(kept + incl - 1) * 5;
#pragma unroll
                for (int c = 0; c < 5; ++c) o[c] = v[c];
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

__global__ void __launch_bounds__(256) collate_pack_annots_kernel(const int64_t* __restrict__ header,
                                                                  const double* __restrict__ rows,
                                                                  const int32_t* __restrict__ row_off,
                                                                  const double* __restrict__ scale,
                                                                  const uint8_t* __restrict__ flip,
                                                                  const int32_t* __restrict__ hw, float* __restrict__ out,
                                                                  int32_t* __restrict__ counts, int Gcap) {
    collate_pack_annots_body<false>(header, rows, row_off, scale, flip, hw, nullptr, out, counts, Gcap);
}

__global__ void __launch_bounds__(256) collate_pack_annots_crop_kernel(const int64_t* __restrict__ header,
                                                                       const double* __restrict__ rows,
                                                                       const int32_t* __restrict__ row_off,
                                                                       const double* __restrict__ scale,
                                                                       const uint8_t* __restrict__ flip,
                                                                       const int32_t* __restrict__ hw,
                                                                       const int32_t* __restrict__ crops,
                                                                       float* __restrict__ out, int32_t* __restrict__ counts,
                                                                       int Gcap) {
    collate_pack_annots_body<true>(header, rows, row_off, scale, flip, hw, crops, out, counts, Gcap);
}

}  // namespace effdet

using namespace effdet;

extern "C" int effdet_normalize_pad(const uint8_t* pixels, const int64_t* offsets, const int32_t* hw, const uint8_t* flip,
                                    float* out_nchw, int B, int S, const double* mean3, const double* std3, int device,
                                    effdet_stream_t stream) {
    EFFDET_REQUIRE(pixels && offsets && hw && out_nchw && mean3 && std3 && B > 0 && B <= 65535 && S > 0 && S <= 65535,
                   "normalize_pad: bad arguments");
    EFFDET_DEVICE(device);
    dim3 grid(cdiv(S, 256), S, B);
    normalize_pad_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(pixels, offsets, hw, flip, out_nchw, S, mean3[0], mean3[1], mean3[2],
                                                                std3[0], std3[1], std3[2]);
    return launch_status("normalize_pad_kernel");
}

extern "C" int effdet_resize_normalize_pad(const uint8_t* pixels, const int64_t* offsets, const int32_t* hw,
                                           const int32_t* resized_hw, const uint8_t* flip, float* out_nchw, int B, int S,
                                           int pixel_scale, const double* mean3, const double* std3, int device,
                                           effdet_stream_t stream) {
    EFFDET_REQUIRE(pixels && offsets && hw && resized_hw && out_nchw && mean3 && std3 && B > 0 && B <= 65535 && S > 0 &&
                       S <= 65535,
                   "resize_normalize_pad: bad arguments");
    EFFDET_REQUIRE(pixel_scale == 1 || pixel_scale == 255, "resize_normalize_pad: pixel_scale %d not in {1,255}", pixel_scale);
    EFFDET_DEVICE(device);
    dim3 grid(cdiv(S, 256), S, B);
    resize_normalize_pad_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(pixels, offsets, hw, resized_hw, flip, out_nchw, S,
                                                                       pixel_scale == 255, mean3[0], mean3[1], mean3[2],
                                                                       std3[0], std3[1], std3[2]);
    return launch_status("resize_normalize_pad_kernel");
}

extern "C" int effdet_resize_crop_normalize_pad(const uint8_t* pixels, const int64_t* offsets, const int32_t* hw,
                                                const int32_t* resized_hw, const int32_t* crops, const uint8_t* flip,
                                                float* out_nchw, int B, int S, int pixel_scale, const double* mean3,
                                                const double* std3, int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(pixels && offsets && hw && resized_hw && crops && out_nchw && mean3 && std3 && B > 0 && B <= 65535 &&
                       S > 0 && S <= 65535,
                   "resize_crop_normalize_pad: bad arguments");
    EFFDET_REQUIRE(pixel_scale == 1 || pixel_scale == 255, "resize_crop_normalize_pad: pixel_scale %d not in {1,255}",
                   pixel_scale);
    EFFDET_DEVICE(device);
    dim3 grid(cdiv(S, 256), S, B);
    resize_crop_normalize_pad_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(pixels, offsets, hw, resized_hw, crops, flip,
                                                                            out_nchw, S, pixel_scale == 255, mean3[0],
                                                                            mean3[1], mean3[2], std3[0], std3[1], std3[2]);
    return launch_status("resize_crop_normalize_pad_kernel");
}

extern "C" int effdet_frame_transform(const uint8_t* pixels, const int64_t* offsets, const int32_t* hw, float* out_nchw, int B,
                                      int H, int W, const float* mean3, const float* std3, int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(pixels && offsets && hw && out_nchw && mean3 && std3, "frame_transform: null argument");
    EFFDET_REQUIRE(B >= 1 && B <= 65535, "frame_transform: B=%d must be in [1, 65535]", B);
    EFFDET_REQUIRE(H >= 1 && H <= 65535 && W >= 1 && W <= 65535, "frame_transform: H=%d, W=%d must be in [1, 65535]", H, W);
    EFFDET_DEVICE(device);
    dim3 grid(cdiv(W, 256), H, B);
    frame_transform_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(pixels, offsets, hw, out_nchw, H, W, mean3[0], mean3[1],
                                                                  mean3[2], std3[0], std3[1], std3[2]);
    return launch_status("frame_transform_kernel");
}

extern "C" int effdet_frame_boxes(const float* scores, const int64_t* classes, const float* boxes, const int32_t* count,
                                  const int32_t* hw, int B, int C, int H, int W, int32_t* rows, int32_t* out_count, int device,
                                  effdet_stream_t stream) {
    EFFDET_REQUIRE(scores && classes && boxes && count && hw && rows && out_count, "frame_boxes: null argument");
    EFFDET_REQUIRE(B >= 1 && B <= 65535, "frame_boxes: B=%d must be in [1, 65535]", B);
    EFFDET_REQUIRE(C >= 1, "frame_boxes: C=%d must be >= 1", C);
    EFFDET_REQUIRE(H >= 1 && W >= 1, "frame_boxes: H=%d, W=%d must be >= 1", H, W);
    EFFDET_REQUIRE(aligned16(boxes), "frame_boxes: boxes must be 16-byte aligned");
    EFFDET_DEVICE(device);
    dim3 grid(cdiv(C, 256), B);
    frame_boxes_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(scores, classes, reinterpret_cast<const float4*>(boxes), count,
                                                              hw, rows, out_count, C, (float)H, (float)W);
    return launch_status("frame_boxes_kernel");
}

extern "C" int effdet_collate_annots(const double* rows, const int32_t* row_off, const double* scale, const uint8_t* flip,
                                     const int32_t* width, float* out, int B, int G, int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(row_off && out && B > 0 && G > 0 && (!flip || width), "collate_annots: bad arguments");
    EFFDET_DEVICE(device);
    collate_annots_kernel<<<cdiv((long long)B * G, 128), 128, 0, (cudaStream_t)stream>>>(rows, row_off, scale, flip, width, out, B, G);
    return launch_status("collate_annots_kernel");
}

extern "C" int effdet_collate_pack_annots(const int64_t* header, const double* rows, const int32_t* row_off,
                                          const double* scale, const uint8_t* flip, const int32_t* hw, float* out,
                                          int32_t* counts, int Bcap, int Gcap, int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(header && rows && row_off && scale && flip && hw && out && counts, "collate_pack_annots: null argument");
    EFFDET_REQUIRE(Bcap > 0 && Bcap <= 65535 && Gcap > 0 && Gcap <= INT_MAX / 5,
                   "collate_pack_annots: capacity Bcap=%d, Gcap=%d unsupported (1..65535, 1..%d)", Bcap, Gcap, INT_MAX / 5);
    EFFDET_DEVICE(device);
    collate_pack_annots_kernel<<<Bcap, 256, 0, (cudaStream_t)stream>>>(header, rows, row_off, scale, flip, hw, out, counts,
                                                                      Gcap);
    return launch_status("collate_pack_annots_kernel");
}

extern "C" int effdet_collate_pack_annots_crop(const int64_t* header, const double* rows, const int32_t* row_off,
                                               const double* scale, const uint8_t* flip, const int32_t* hw,
                                               const int32_t* crops, float* out, int32_t* counts, int Bcap, int Gcap,
                                               int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(header && rows && row_off && scale && flip && hw && crops && out && counts,
                   "collate_pack_annots_crop: null argument");
    EFFDET_REQUIRE(Bcap > 0 && Bcap <= 65535 && Gcap > 0 && Gcap <= INT_MAX / 5,
                   "collate_pack_annots_crop: capacity Bcap=%d, Gcap=%d unsupported (1..65535, 1..%d)", Bcap, Gcap,
                   INT_MAX / 5);
    EFFDET_DEVICE(device);
    collate_pack_annots_crop_kernel<<<Bcap, 256, 0, (cudaStream_t)stream>>>(header, rows, row_off, scale, flip, hw, crops,
                                                                           out, counts, Gcap);
    return launch_status("collate_pack_annots_crop_kernel");
}
