// The step before the hot path, on the device (SURVEY.md 8(f) rank 2):
//   input side  : Normalizer + Augmenter (horizontal flip) + zero-pad to the common size + collater + `.cuda().float()`
//                 datasets/augmentation.py:69-91,111-150, train.py:105-106  (cv2.resize is NOT reproduced: images enter at
//                 their final resolution; everything after the decode is otherwise done here)
// (the output side, eval.py's selection, is in voc_eval.cu)
// Arithmetic follows the reference's dtypes exactly so the results are bit-identical to NumPy:
//   Normalizer computes (img.astype(float32) - mean[float64]) / std[float64] in float64 and train.py casts to float32 on
//   the device; collater writes float64 annotations into a float32 tensor.
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

extern "C" int effdet_collate_annots(const double* rows, const int32_t* row_off, const double* scale, const uint8_t* flip,
                                     const int32_t* width, float* out, int B, int G, int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(row_off && out && B > 0 && G > 0 && (!flip || width), "collate_annots: bad arguments");
    EFFDET_DEVICE(device);
    collate_annots_kernel<<<cdiv((long long)B * G, 128), 128, 0, (cudaStream_t)stream>>>(rows, row_off, scale, flip, width, out, B, G);
    return launch_status("collate_annots_kernel");
}
