// Element-wise / reduction pieces of the MBConv block that are not convolutions:
//   * backward of swish(BN_eval(z)) with trainable affine (dgamma, dbeta reductions fused)
//   * squeeze-excite: spatial mean / gate-gradient reductions (the two tiny FC layers live in se_ops.cu)
// Reference: models/efficientnet.py:75-105 (block), :90-94 (SE), models/utils.py:31-47 (swish),
//            frozen BN models/efficientdet.py:88-92.  All HBM-bound; NHWC float4 row-packed.
#include "common.cuh"

namespace effdet {

__global__ void __launch_bounds__(256) bnact_bwd_kernel(const effdet_bnact_bwd_args p, const int rows_per_block) {
    __shared__ float4 red_g[256];
    __shared__ float4 red_b[256];
    const int cvecs = p.C / 4;
    const RowPack rp = rowpack(cvecs, blockIdx.y);
    const int b = blockIdx.z;
    float4 sg = f4zero(), sb = f4zero();
    if (rp.active) {
        const int c = rp.cv * 4;
        const float4 sc = ldg4(p.scale + c), sh = ldg4(p.shift + c), mu = ldg4(p.mean + c), rs = ldg4(p.rstd + c);
        float4 gt = make_float4(1.f, 1.f, 1.f, 1.f), dm = f4zero();
        if (p.gate) gt = ldg4(p.gate + (long long)b * p.C + c);
        if (p.dmean) dm = f4scale(ldg4(p.dmean + (long long)b * p.C + c), p.inv_hw);
        const float rowsc = p.row_scale ? __ldg(p.row_scale + b) : 1.f;
        const int r_begin = blockIdx.x * rows_per_block;
        const int r_end = min(p.HW, r_begin + rows_per_block);
        // 4 rows per trip: 8 independent 128-bit loads in flight per thread before any arithmetic
        constexpr int U = 4;
        for (int r0 = r_begin + rp.tr; r0 < r_end; r0 += U * rp.rows) {
            float4 gv[U], zv[U];
            long long offs[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int r = r0 + u * rp.rows;
                offs[u] = ((long long)b * p.HW + (r < r_end ? r : r0)) * p.C + c;
                gv[u] = ldg4(p.dy + offs[u]);
                zv[u] = ldg4(p.z + offs[u]);
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if (r0 + u * rp.rows >= r_end) break;
                float4 g = gv[u];
                const float4 zz = zv[u];
                if (p.gate) g = f4fma(g, gt, dm);
                g = f4scale(g, rowsc);
                float4 du = g;
                if (p.act == EFFDET_ACT_SWISH) {
                    const float4 u4 = f4fma(zz, sc, sh);
                    du = make_float4(g.x * swish_gradf_(u4.x), g.y * swish_gradf_(u4.y), g.z * swish_gradf_(u4.z),
                                     g.w * swish_gradf_(u4.w));
                }
                const float4 xh = make_float4((zz.x - mu.x) * rs.x, (zz.y - mu.y) * rs.y, (zz.z - mu.z) * rs.z,
                                              (zz.w - mu.w) * rs.w);
                sg = f4fma(du, xh, sg);
                sb = f4add(sb, du);
                st4(p.dz + offs[u], f4mul(du, sc));
            }
        }
    }
    red_g[threadIdx.x] = sg;
    red_b[threadIdx.x] = sb;
    __syncthreads();
    if (rp.tr == 0 && rp.cv < cvecs) {
        float4 ag = f4zero(), ab = f4zero();
        for (int r = 0; r < rp.rows; ++r) {
            ag = f4add(ag, red_g[r * rp.cvb + rp.tc]);
            ab = f4add(ab, red_b[r * rp.cvb + rp.tc]);
        }
        float* og = p.dgamma + rp.cv * 4;
        float* ob = p.dbeta + rp.cv * 4;
        atomicAdd(og + 0, ag.x); atomicAdd(og + 1, ag.y); atomicAdd(og + 2, ag.z); atomicAdd(og + 3, ag.w);
        atomicAdd(ob + 0, ab.x); atomicAdd(ob + 1, ab.y); atomicAdd(ob + 2, ab.z); atomicAdd(ob + 3, ab.w);
    }
}

// out[b,c] += alpha * sum_r a[b,r,c] * swish(z[b,r,c]*scale[c]+shift[c]): z is the raw conv output, and the activated
// tensor is recomputed instead of stored
__global__ void __launch_bounds__(256) spatial_reduce_kernel(const float* __restrict__ a, const float* __restrict__ z,
                                                             float* __restrict__ out, float alpha, int HW, int C,
                                                             int rows_per_block, const float* __restrict__ scale,
                                                             const float* __restrict__ shift) {
    __shared__ float4 red[256];
    const int cvecs = C / 4;
    const RowPack rp = rowpack(cvecs, blockIdx.y);
    const int b = blockIdx.z;
    float4 s = f4zero();
    if (rp.active) {
        const int r_begin = blockIdx.x * rows_per_block;
        const int r_end = min(HW, r_begin + rows_per_block);
        const float4 sc = ldg4(scale + rp.cv * 4), sh = ldg4(shift + rp.cv * 4);
        constexpr int U = 4;                            // 8 independent 128-bit loads in flight per thread
        for (int r0 = r_begin + rp.tr; r0 < r_end; r0 += U * rp.rows) {
            float4 av[U], zv[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int r = r0 + u * rp.rows;
                const long long off = ((long long)b * HW + (r < r_end ? r : r0)) * C + rp.cv * 4;
                av[u] = ldg4(a + off);
                zv[u] = ldg4(z + off);
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if (r0 + u * rp.rows >= r_end) break;
                const float4 q = f4fma(zv[u], sc, sh);
                s = f4fma(av[u], make_float4(swishf_(q.x), swishf_(q.y), swishf_(q.z), swishf_(q.w)), s);
            }
        }
    }
    red[threadIdx.x] = s;
    __syncthreads();
    if (rp.tr == 0 && rp.cv < cvecs) {
        float4 acc = f4zero();
        for (int r = 0; r < rp.rows; ++r) acc = f4add(acc, red[r * rp.cvb + rp.tc]);
        float* o = out + (long long)b * C + rp.cv * 4;
        atomicAdd(o + 0, alpha * acc.x); atomicAdd(o + 1, alpha * acc.y);
        atomicAdd(o + 2, alpha * acc.z); atomicAdd(o + 3, alpha * acc.w);
    }
}

// scale = gamma*rstd ; shift = beta - mean*scale ; rstd = 1/sqrt(var+eps)   (frozen BN -> affine)
__global__ void bn_fold_kernel(const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ mean,
                               const float* __restrict__ var, float eps, float* __restrict__ scale, float* __restrict__ shift,
                               float* __restrict__ rstd, int C) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    const float r = 1.0f / sqrtf(__ldg(var + c) + eps);
    const float s = __ldg(gamma + c) * r;
    rstd[c] = r;
    scale[c] = s;
    shift[c] = __ldg(beta + c) - __ldg(mean + c) * s;
}

// out = a + b
__global__ void __launch_bounds__(256) add_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ o,
                                                  long long n4) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x)
        st4(o + i * 4, f4add(ldg4(a + i * 4), ldg4(b + i * 4)));
}

// dz = y > 0 ? dy : 0
__global__ void __launch_bounds__(256) relu_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y,
                                                       float* __restrict__ dz, long long n4) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const float4 g = ldg4(dy + i * 4), v = ldg4(y + i * 4);
        st4(dz + i * 4, make_float4(v.x > 0.f ? g.x : 0.f, v.y > 0.f ? g.y : 0.f, v.z > 0.f ? g.z : 0.f, v.w > 0.f ? g.w : 0.f));
    }
}

}  // namespace effdet

using namespace effdet;

extern "C" int effdet_bn_fold(const float* gamma, const float* beta, const float* mean, const float* var, float eps,
                              float* scale, float* shift, float* rstd, int C, int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(gamma && beta && mean && var && scale && shift && rstd && C > 0, "bn_fold: bad arguments");
    EFFDET_DEVICE(device);
    bn_fold_kernel<<<cdiv(C, 128), 128, 0, (cudaStream_t)stream>>>(gamma, beta, mean, var, eps, scale, shift, rstd, C);
    return launch_status("bn_fold_kernel");
}

extern "C" int effdet_add(const float* a, const float* b, float* out, int64_t n, int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(a && b && out && n > 0 && n % 4 == 0, "add: bad arguments (n must be a multiple of 4)");
    EFFDET_REQUIRE(aligned16(a) && aligned16(b) && aligned16(out), "add: alignment");
    EFFDET_DEVICE(device);
    int blocks = cdiv(n / 4, 256);
    if (blocks > num_sms() * 16) blocks = num_sms() * 16;
    add_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(a, b, out, n / 4);
    return launch_status("add_kernel");
}

extern "C" int effdet_relu_bwd(const float* dy, const float* y, float* dz, int64_t n, int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(dy && y && dz && n > 0 && n % 4 == 0, "relu_bwd: bad arguments (n must be a multiple of 4)");
    EFFDET_REQUIRE(aligned16(dy) && aligned16(y) && aligned16(dz), "relu_bwd: alignment");
    EFFDET_DEVICE(device);
    int blocks = cdiv(n / 4, 256);
    if (blocks > num_sms() * 16) blocks = num_sms() * 16;
    relu_bwd_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(dy, y, dz, n / 4);
    return launch_status("relu_bwd_kernel");
}

static void row_grid(int HW, int cvecs, int B, dim3* grid, int* rpb_out) {
    const int rows = rowpack_rows(cvecs);
    const int chunks = rowpack_chunks(cvecs);
    // ~4 waves of CTAs, at least 8 row-iterations each (measured: more, smaller CTAs are slower -- the per-CTA
    // shared-memory reduction + atomics dominate)
    long long want_blocks = (num_sms() * 4 + (long long)B * chunks - 1) / ((long long)B * chunks);
    if (want_blocks < 1) want_blocks = 1;
    long long rpb = (HW + want_blocks - 1) / want_blocks;
    if (rpb < (long long)rows * 8) rpb = (long long)rows * 8;
    *rpb_out = (int)rpb;
    *grid = dim3(cdiv(HW, rpb), chunks, B);
}

extern "C" int effdet_bnact_bwd(const effdet_bnact_bwd_args* a, int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(a && a->dy && a->z && a->dz && a->scale && a->shift && a->mean && a->rstd && a->dgamma && a->dbeta,
                   "bnact_bwd: null tensor");
    EFFDET_REQUIRE(a->C % 4 == 0 && a->C > 0 && a->B > 0 && a->HW > 0 && a->B <= 65535, "bnact_bwd: bad shape");
    EFFDET_REQUIRE(a->act == EFFDET_ACT_NONE || a->act == EFFDET_ACT_SWISH, "bnact_bwd: act %d unsupported", a->act);
    EFFDET_REQUIRE(aligned16(a->dy) && aligned16(a->z) && aligned16(a->dz) && aligned16(a->scale) && aligned16(a->shift) &&
                       aligned16(a->mean) && aligned16(a->rstd) && aligned16(a->gate) && aligned16(a->dmean),
                   "bnact_bwd: alignment");
    EFFDET_DEVICE(device);
    dim3 grid;
    int rpb;
    row_grid(a->HW, a->C / 4, a->B, &grid, &rpb);
    bnact_bwd_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(*a, rpb);
    return launch_status("bnact_bwd_kernel");
}

extern "C" int effdet_spatial_reduce_act(const float* a, const float* z, const float* scale, const float* shift, float* out,
                                         float alpha, int B, int HW, int C, int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(a && z && scale && shift && out && B > 0 && B <= 65535 && HW > 0 && C > 0 && C % 4 == 0,
                   "spatial_reduce_act: bad arguments");
    EFFDET_REQUIRE(aligned16(a) && aligned16(z) && aligned16(scale) && aligned16(shift), "spatial_reduce_act: alignment");
    EFFDET_DEVICE(device);
    dim3 grid;
    int rpb;
    row_grid(HW, C / 4, B, &grid, &rpb);
    spatial_reduce_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(a, z, out, alpha, HW, C, rpb, scale, shift);
    return launch_status("spatial_reduce_kernel");
}
