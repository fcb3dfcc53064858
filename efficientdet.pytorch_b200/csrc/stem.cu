// EfficientNet stem: 3x3 stride-2 conv (3 -> C0) straight from the NCHW image, static TF-"SAME"
// pad (left,right,top,bottom) = (0,1,0,1), fused eval-BN affine + swish, NHWC output.
// Reference: models/efficientnet.py:140-143,193 ; pad rule models/utils.py:126-149.
// HBM-bound (AI ~ 10 FLOP/B): one pass over the image, one write of z (kept for backward) and y.
#include "common.cuh"

namespace effdet {

__global__ void __launch_bounds__(256) stem_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                       const float* __restrict__ scale, const float* __restrict__ shift,
                                                       float* __restrict__ z, float* __restrict__ y, int B, int H, int W,
                                                       int C0, int Ho, int Wo) {
    extern __shared__ __align__(16) float ws[];  // [27][C0], tap-major
    for (int i = threadIdx.x; i < 27 * C0; i += blockDim.x) {
        const int co = i % C0, tap = i / C0;  // tap = ci*9 + ky*3 + kx
        ws[i] = __ldg(w + co * 27 + tap);
    }
    __syncthreads();
    const int cvecs = C0 / 4;
    const long long total = (long long)B * Ho * Wo * cvecs;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int cv = (int)(idx % cvecs);
    long long pix = idx / cvecs;
    const int ox = (int)(pix % Wo);
    pix /= Wo;
    const int oy = (int)(pix % Ho);
    const int b = (int)(pix / Ho);
    float4 acc = f4zero();
    const float* xb = x + (long long)b * 3 * H * W;
#pragma unroll
    for (int ci = 0; ci < 3; ++ci) {
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
            const int iy = 2 * oy + ky;
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                const int ix = 2 * ox + kx;
                float v = 0.f;
                if (iy < H && ix < W) v = __ldg(xb + ((long long)ci * H + iy) * W + ix);
                const float4 wv = *reinterpret_cast<const float4*>(&ws[(ci * 9 + ky * 3 + kx) * C0 + cv * 4]);
                acc = f4fma(make_float4(v, v, v, v), wv, acc);
            }
        }
    }
    const long long o = (((long long)b * Ho + oy) * Wo + ox) * C0 + cv * 4;
    st4(z + o, acc);
    if (y == nullptr) return;
    float4 u = f4fma(acc, ldg4(scale + cv * 4), ldg4(shift + cv * 4));
    st4(y + o, make_float4(swishf_(u.x), swishf_(u.y), swishf_(u.z), swishf_(u.w)));
}

// One thread per output pixel, all C0 = 4*NV channels in registers: the 27 input taps are fetched once per pixel
// (not once per 4-channel group) and the weights are warp-broadcast 128-bit shared loads.
template <int NV>
__global__ void __launch_bounds__(128) stem_fwd_px_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                          const float* __restrict__ scale, const float* __restrict__ shift,
                                                          float* __restrict__ z, float* __restrict__ y, int B, int H, int W,
                                                          int Ho, int Wo) {
    constexpr int C0 = NV * 4;
    __shared__ __align__(16) float ws[27 * C0];
    __shared__ __align__(16) float sc_s[C0];
    __shared__ __align__(16) float sh_s[C0];
    for (int i = threadIdx.x; i < 27 * C0; i += blockDim.x) {
        const int co = i % C0, tap = i / C0;
        ws[i] = __ldg(w + co * 27 + tap);
    }
    for (int i = threadIdx.x; i < C0; i += blockDim.x) { sc_s[i] = __ldg(scale + i); sh_s[i] = __ldg(shift + i); }
    __syncthreads();
    const long long npix = (long long)B * Ho * Wo;
    const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= npix) return;
    const int ox = (int)(pix % Wo);
    const long long r = pix / Wo;
    const int oy = (int)(r % Ho);
    const int b = (int)(r / Ho);
    float v[27];
    const float* xb = x + (long long)b * 3 * H * W;
#pragma unroll
    for (int ci = 0; ci < 3; ++ci)
#pragma unroll
        for (int ky = 0; ky < 3; ++ky)
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                const int iy = 2 * oy + ky, ix = 2 * ox + kx;
                v[ci * 9 + ky * 3 + kx] = (iy < H && ix < W) ? __ldg(xb + ((long long)ci * H + iy) * W + ix) : 0.f;
            }
    float4 acc[NV];
#pragma unroll
    for (int j = 0; j < NV; ++j) acc[j] = f4zero();
#pragma unroll
    for (int tap = 0; tap < 27; ++tap) {
        const float4 xv = make_float4(v[tap], v[tap], v[tap], v[tap]);
#pragma unroll
        for (int j = 0; j < NV; ++j) acc[j] = f4fma(xv, *reinterpret_cast<const float4*>(&ws[tap * C0 + j * 4]), acc[j]);
    }
    float* zo = z + pix * C0;
    float* yo = y + pix * C0;
#pragma unroll
    for (int j = 0; j < NV; ++j) {
        st4(zo + j * 4, acc[j]);
        if (y == nullptr) continue;
        const float4 u = f4fma(acc[j], *reinterpret_cast<const float4*>(&sc_s[j * 4]), *reinterpret_cast<const float4*>(&sh_s[j * 4]));
        st4(yo + j * 4, make_float4(swishf_(u.x), swishf_(u.y), swishf_(u.z), swishf_(u.w)));
    }
}

constexpr int kStemP = 64;     // output pixels (one row segment) per work unit

// dw[co][tap] += sum_pixels x[pixel + tap] * dz[pixel][co]  -- a 27 x C0 GEMM over ~2 M pixels.  A work unit is a
// 64-pixel segment of one output row: the 3 x 3 input row segments it touches (129 floats each, read coalesced from
// the NCHW image) and the 64 x C0 slice of dz are staged in shared memory; a warp owns 8 of the pixels, a lane owns 4
// output channels x TPG taps (C0 = 32: 8 channel vectors x 4 tap groups of 7), i.e. per pixel one 128-bit load of dz
// and TPG broadcast loads of x feed 4*TPG FMAs -- FMA-bound instead of shared-memory-bound (the previous mapping
// issued 2 shared loads per 4 FMAs and sat at 0.09 of the HBM roofline).
template <int TPG>
__global__ void __launch_bounds__(256) stem_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ dz,
                                                         float* __restrict__ dw, int B, int H, int W, int C0, int Ho,
                                                         int Wo, int segs, long long units) {
    extern __shared__ __align__(16) float sm[];
    float* xr = sm;                    // [9][132]: (ci, ky) row segments, columns 2*ox0 .. 2*ox0 + 128
    float* ds = sm + 9 * 132;          // [kStemP][C0]; reused for the cross-warp reduction
    const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
    const int cvs = C0 / 4, tgs = 32 / cvs;
    const int cv = lane % cvs, tg = lane / cvs;
    const bool worker = tg < tgs;
    int off[TPG];                      // shared-memory offset of this lane's taps (pixel 0); -1 = no tap
#pragma unroll
    for (int j = 0; j < TPG; ++j) {
        const int tap = tg * TPG + j;
        off[j] = (worker && tap < 27) ? (tap / 3) * 132 + tap % 3 : -1;
    }
    float4 acc[TPG];
#pragma unroll
    for (int j = 0; j < TPG; ++j) acc[j] = f4zero();
    for (long long u = blockIdx.x; u < units; u += gridDim.x) {
        const int seg = (int)(u % segs);
        const long long r = u / segs;
        const int oy = (int)(r % Ho), b = (int)(r / Ho);
        const int ox0 = seg * kStemP;
        const int npx = min(kStemP, Wo - ox0);
        __syncthreads();                                   // the previous unit has been consumed
        for (int i = t; i < 9 * 132; i += 256) {
            const int row = i / 132, c = i - row * 132;
            const int ci = row / 3, ky = row - ci * 3;
            const int iy = 2 * oy + ky, ix = 2 * ox0 + c;
            xr[i] = (c <= 2 * kStemP && iy < H && ix < W) ? __ldg(x + (((long long)b * 3 + ci) * H + iy) * W + ix) : 0.f;
        }
        const float* dzr = dz + (((long long)b * Ho + oy) * Wo + ox0) * C0;
        for (int i = t; i < kStemP * cvs; i += 256) {
            const int pp = i / cvs;
            *reinterpret_cast<float4*>(&ds[i * 4]) = pp < npx ? ldg4(dzr + (long long)i * 4) : f4zero();
        }
        __syncthreads();
        if (worker) {
#pragma unroll
            for (int q = 0; q < kStemP / 8; ++q) {
                const int pp = warp + q * 8;
                const float4 g = *reinterpret_cast<const float4*>(&ds[pp * C0 + cv * 4]);
#pragma unroll
                for (int j = 0; j < TPG; ++j) {
                    if (off[j] < 0) continue;
                    const float v = xr[off[j] + 2 * pp];
                    acc[j] = f4fma(make_float4(v, v, v, v), g, acc[j]);
                }
            }
        }
    }
    // cross-warp sum through shared memory, then one atomic per (channel, tap) and CTA
    __syncthreads();
    float4* red = reinterpret_cast<float4*>(ds);           // [8 warps][32 lanes], one tap slot at a time
    for (int j = 0; j < TPG; ++j) {
        __syncthreads();
        red[warp * 32 + lane] = acc[j];
        __syncthreads();
        if (warp == 0 && worker) {
            float4 s = red[lane];
#pragma unroll
            for (int w = 1; w < 8; ++w) s = f4add(s, red[w * 32 + lane]);
            const int tap = tg * TPG + j;
            if (tap < 27) {
                float* o = dw + (cv * 4) * 27 + tap;
                atomicAdd(o, s.x); atomicAdd(o + 27, s.y); atomicAdd(o + 54, s.z); atomicAdd(o + 81, s.w);
            }
        }
    }
}

}  // namespace effdet

using namespace effdet;

extern "C" int effdet_stem_fwd(const float* x_nchw, const float* w_oihw, const float* scale, const float* shift,
                               float* z, float* y, int B, int H, int W, int C0, int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(x_nchw && w_oihw && scale && shift && z, "stem_fwd: null tensor");
    EFFDET_REQUIRE(C0 % 4 == 0 && C0 > 0 && C0 <= 256, "stem_fwd: C0=%d unsupported", C0);
    EFFDET_REQUIRE(B > 0 && H >= 2 && W >= 2, "stem_fwd: bad shape");
    EFFDET_REQUIRE(aligned16(z) && aligned16(y) && aligned16(scale) && aligned16(shift), "stem_fwd: alignment");
    EFFDET_DEVICE(device);
    const int Ho = (H + 1 - 3) / 2 + 1, Wo = (W + 1 - 3) / 2 + 1;
    const long long npix = (long long)B * Ho * Wo;
    cudaStream_t st = (cudaStream_t)stream;
    switch (C0) {      // stem widths of EfficientNet-B0..B7: 32, 32, 32, 40, 48, 48, 56, 64
        case 32: stem_fwd_px_kernel<8><<<cdiv(npix, 128), 128, 0, st>>>(x_nchw, w_oihw, scale, shift, z, y, B, H, W, Ho, Wo); break;
        case 40: stem_fwd_px_kernel<10><<<cdiv(npix, 128), 128, 0, st>>>(x_nchw, w_oihw, scale, shift, z, y, B, H, W, Ho, Wo); break;
        case 48: stem_fwd_px_kernel<12><<<cdiv(npix, 128), 128, 0, st>>>(x_nchw, w_oihw, scale, shift, z, y, B, H, W, Ho, Wo); break;
        case 56: stem_fwd_px_kernel<14><<<cdiv(npix, 128), 128, 0, st>>>(x_nchw, w_oihw, scale, shift, z, y, B, H, W, Ho, Wo); break;
        case 64: stem_fwd_px_kernel<16><<<cdiv(npix, 128), 128, 0, st>>>(x_nchw, w_oihw, scale, shift, z, y, B, H, W, Ho, Wo); break;
        default: {
            const long long total = npix * (C0 / 4);
            stem_fwd_kernel<<<cdiv(total, 256), 256, 27 * C0 * sizeof(float), st>>>(x_nchw, w_oihw, scale, shift, z, y, B, H, W, C0,
                                                                                     Ho, Wo);
        }
    }
    return launch_status("stem_fwd_kernel");
}

extern "C" int effdet_stem_wgrad(const float* x_nchw, const float* dz, float* dw_oihw, int B, int H, int W, int C0,
                                 int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(x_nchw && dz && dw_oihw, "stem_wgrad: null tensor");
    EFFDET_REQUIRE(C0 % 4 == 0 && C0 >= 8 && C0 <= 64, "stem_wgrad: C0=%d unsupported (8..64)", C0);
    EFFDET_REQUIRE(aligned16(dz), "stem_wgrad: alignment");
    EFFDET_DEVICE(device);
    const int Ho = (H + 1 - 3) / 2 + 1, Wo = (W + 1 - 3) / 2 + 1;
    // grid and TPG: tests/test_benchmark_plans.py (_stem_plan) mirrors this arithmetic
    const int segs = cdiv(Wo, kStemP);
    const long long units = (long long)B * Ho * segs;
    int blocks = (int)(units < num_sms() * 8 ? units : num_sms() * 8);
    size_t smem = (size_t)(9 * 132 + kStemP * C0) * sizeof(float);
    const size_t need = (size_t)(9 * 132) * sizeof(float) + 256 * sizeof(float4);     // cross-warp reduction scratch
    if (smem < need) smem = need;
    const int cvs = C0 / 4, tgs = 32 / cvs, tpg = cdiv(27, tgs);
    cudaStream_t st = (cudaStream_t)stream;
    if (tpg <= 7) stem_wgrad_kernel<7><<<blocks, 256, smem, st>>>(x_nchw, dz, dw_oihw, B, H, W, C0, Ho, Wo, segs, units);
    else if (tpg <= 9) stem_wgrad_kernel<9><<<blocks, 256, smem, st>>>(x_nchw, dz, dw_oihw, B, H, W, C0, Ho, Wo, segs, units);
    else stem_wgrad_kernel<14><<<blocks, 256, smem, st>>>(x_nchw, dz, dw_oihw, B, H, W, C0, Ho, Wo, segs, units);
    return launch_status("stem_wgrad_kernel");
}
