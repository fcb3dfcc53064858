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
__global__ void __launch_bounds__(256) resize_normalize_pad_kernel(const uint8_t* __restrict__ pix, const int64_t* __restrict__ offs,
                                                                   const int32_t* __restrict__ hw, const int32_t* __restrict__ rhw,
                                                                   const uint8_t* __restrict__ flip, float* __restrict__ out, int S,
                                                                   int div255, double m0, double m1, double m2, double s0,
                                                                   double s1, double s2) {
    __shared__ double lut[3][256];
    const int b = blockIdx.z;
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    const int h = hw[2 * b], w = hw[2 * b + 1], rh = rhw[2 * b], rw = rhw[2 * b + 1];
    const long long plane = (long long)S * S;
    float* o = out + (long long)b * 3 * plane + (long long)y * S + x;
    if (y >= rh || h <= 0 || w <= 0) {                                  // block-uniform: a padding row
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
    double v[3] = {0.0, 0.0, 0.0};                                      // np.zeros((S, S, 3)) padding
    if (x < rw) {
        const uint8_t* img = pix + offs[b];
        const bool fl = flip && flip[b];
        // source pixel (r, c) of the flipped image: image[:, ::-1, :]
        auto px = [&](int r, int c) { return img + ((long long)r * w + (fl ? w - 1 - c : c)) * 3; };
        const double scale_x = __ddiv_rn(1.0, __ddiv_rn((double)rw, (double)w));
        const double scale_y = __ddiv_rn(1.0, __ddiv_rn((double)rh, (double)h));
        if (rh == h && rw == w) {
            const uint8_t* p = px(y, x);
            for (int c = 0; c < 3; ++c) v[c] = lut[c][p[c]];
        } else if (fabs(__dsub_rn(scale_x, 2.0)) < DBL_EPSILON && fabs(__dsub_rn(scale_y, 2.0)) < DBL_EPSILON) {
            const uint8_t *p00 = px(2 * y, 2 * x), *p01 = px(2 * y, 2 * x + 1);
            const uint8_t *p10 = px(2 * y + 1, 2 * x), *p11 = px(2 * y + 1, 2 * x + 1);
            for (int c = 0; c < 3; ++c)
                v[c] = __dmul_rn(__dadd_rn(__dadd_rn(__dadd_rn(lut[c][p00[c]], lut[c][p01[c]]), lut[c][p10[c]]), lut[c][p11[c]]),
                                 0.25);
        } else {
            float fx = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn((double)x, 0.5), scale_x), 0.5));
            int sx = (int)floorf(fx);
            fx = __fsub_rn(fx, (float)sx);
            if (sx < 0) fx = 0.f, sx = 0;
            const bool single = sx + 1 >= w;
            if (sx >= w - 1) fx = 0.f, sx = w - 1;
            float fy = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn((double)y, 0.5), scale_y), 0.5));
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

extern "C" int effdet_collate_annots(const double* rows, const int32_t* row_off, const double* scale, const uint8_t* flip,
                                     const int32_t* width, float* out, int B, int G, int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(row_off && out && B > 0 && G > 0 && (!flip || width), "collate_annots: bad arguments");
    EFFDET_DEVICE(device);
    collate_annots_kernel<<<cdiv((long long)B * G, 128), 128, 0, (cudaStream_t)stream>>>(rows, row_off, scale, flip, width, out, B, G);
    return launch_status("collate_annots_kernel");
}
