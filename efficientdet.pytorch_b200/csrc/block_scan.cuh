// CTA-wide inclusive scan, shared by the VOC AP kernel (voc_eval.cu) and the COCO accumulation (coco_eval.cu).
#pragma once
#include "common.cuh"

namespace effdet {

struct IntAdd {
    __device__ int operator()(int a, int b) const { return a + b; }
};
struct DblMax {
    __device__ double operator()(double a, double b) const { return fmax(a, b); }
};

// inclusive scan over the CTA in thread order; `total` = the last thread's result.  warp_tot: 32 shared elements.
template <typename T, typename Op>
__device__ __forceinline__ T block_scan(T v, T* warp_tot, Op op, T& total) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const T u = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v = op(u, v);
    }
    if (lane == 31) warp_tot[w] = v;
    __syncthreads();
    if (threadIdx.x == 0)
        for (int i = 1; i < nw; ++i) warp_tot[i] = op(warp_tot[i - 1], warp_tot[i]);
    __syncthreads();
    if (w > 0) v = op(warp_tot[w - 1], v);
    total = warp_tot[nw - 1];
    __syncthreads();
    return v;
}

}  // namespace effdet
