// Depthwise convolution of the MBConv block, "pre-activation only" edition.
//
// The reference's MemoryEfficientSwish keeps only the pre-activation of every swish
// (models/utils.py:31-42); round 1 of this build wrote BOTH the raw conv output z and the activated
// tensor a for each of the three convs of a block, i.e. the 6x-expanded tensor crossed HBM seven times
// in forward and ~20 times in backward.  Here only the raw tensors exist:
//
//   forward  (effdet_dwconv_fwd_fused):   z1 = dw( swish(bn0(z0)) )          one read of z0, one write of z1,
//            the squeeze-excite spatial sums  sum_px swish(bn1(z1))  fall out of the epilogue (no second read)
//   backward (effdet_dwconv_bwd_fused):   from (dq, z1, gate, dmean) and z0 in ONE pass
//            dz1 = (dq*gate + dmean/HW) * swish'(bn1(z1)) * scale1        (never written to HBM)
//            da0 = dw^T(dz1),  dWd += a0 (*) dz1,  dz0 = da0 * swish'(bn0(z0)) * scale0  -> the only write
//            plus dgamma/dbeta of both BatchNorms.  Replaces bnact_bwd(BN1) + dw_bwd_weight + dw_bwd_data +
//            bnact_bwd(BN0): 2 reads of the small-side tensors + 1 read / 1 write of the expanded tensor.
//
// Reference: models/efficientnet.py:85-94 (expand BN swish, depthwise BN swish, SE), models/utils.py:31-47,126-155.
// Both kernels are HBM-bound: a CTA stages a spatial tile of 16 channels (64 B per pixel) in shared memory with
// 128-bit loads, applies BN+swish ONCE per staged element, and then works out of shared memory in 4-wide strips.
// Stride-2 data gradients are evaluated polyphase (per input parity class the transposed conv is a stride-1
// correlation with the taps of matching parity), so no thread ever tests divisibility at run time.
#include "common.cuh"

#include <cuda_bf16.h>

namespace effdet {

constexpr int kCVc = 4;         // float4 channel vectors per CTA (16 channels)
constexpr int kPS = 5;          // float4 slots per staged pixel (4 used + 1 pad: 80-byte pitch kills the 2-way conflict)

// The reference pads statically for image_size 224 (models/utils.py:126-149): as (top/left) k3s1 1, k5s1 2, k3s2 0, k5s2 1.
template <int K, int S, bool SMALL = false>
struct DwGeo {
    static constexpr int PT = (S == 1) ? (K - 1) / 2 : (K == 3 ? 0 : 1);
    // threads per CTA: the 5x5 kernels carry 25 float4 weight-gradient accumulators per thread (~250 registers), so one
    // CTA per SM is all that fits -- give it 8 warps instead of 4
    static constexpr int NT = (K == 5 && !SMALL) ? 256 : 128;
    // forward: output tile and the input region it needs (SMALL: late stages whose whole map is 8x8 or less)
    static constexpr int TOY = SMALL ? (S == 1 ? 8 : 4) : (S == 1 ? 16 : 8), TOX = SMALL ? 8 : 16;
    static constexpr int FIH = (TOY - 1) * S + K, FIW = (TOX - 1) * S + K;
    // backward: tile of "cells" (a cell = S x S input pixels = one output coordinate) and the output region whose dz1
    // the transposed convolution of those cells touches: rows a + d, d in [DMIN, DMAX]
    static constexpr int TCY = SMALL ? (S == 1 ? 8 : 4) : (S == 1 ? 16 : 8), TCX = SMALL ? 8 : 16;
    static constexpr int DMIN = (S == 1) ? -((K - 1) / 2) : -1;
    static constexpr int DMAX = (S == 1) ? (K - 1) / 2 : (K == 3 ? 0 : 1);
    static constexpr int GH = TCY + DMAX - DMIN, GW = TCX + DMAX - DMIN;
    static constexpr int BIH = TCY * S, BIW = TCX * S;
};

__device__ __forceinline__ float4 f4swish(const float4 u) { return make_float4(fswish(u.x), fswish(u.y), fswish(u.z), fswish(u.w)); }
__device__ __forceinline__ float4 f4swish_grad(const float4 u) {
    return make_float4(fswish_grad(u.x), fswish_grad(u.y), fswish_grad(u.z), fswish_grad(u.w));
}
// 16-byte asynchronous global->shared copy; src_bytes = 0 zero-fills the destination (halo / tail).  Every copy of a
// tile is issued before anything waits, so a CTA has its whole tile (tens of KB) in flight at once.
__device__ __forceinline__ void dw_cp_async16(void* smem_dst, const void* gsrc, int src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)),
                 "l"(gsrc), "r"(src_bytes)
                 : "memory");
}
__device__ __forceinline__ void dw_cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
__device__ __forceinline__ float4 f4sub(const float4 a, const float4 b) {
    return make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w);
}
// sum over the 8 lanes of a warp that share (lane & 3), result valid in lanes 0..3
__device__ __forceinline__ float4 cv_group_sum(float4 v) {
#pragma unroll
    for (int o = 4; o < 32; o <<= 1) {
        v.x += __shfl_xor_sync(0xffffffffu, v.x, o);
        v.y += __shfl_xor_sync(0xffffffffu, v.y, o);
        v.z += __shfl_xor_sync(0xffffffffu, v.z, o);
        v.w += __shfl_xor_sync(0xffffffffu, v.w, o);
    }
    return v;
}

// ------------------------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------------------------
template <int K, int S, bool PRE, bool SMALL>
__global__ void __launch_bounds__((DwGeo<K, S, SMALL>::NT)) dw_fwd_fused_kernel(const effdet_dw_fwd_args p, const int tiles_x,
                                                                                const int ntiles, const int tiles_per_cta) {
    using G = DwGeo<K, S, SMALL>;
    constexpr int kDwT = G::NT;
    extern __shared__ __align__(16) float4 dwsm[];
    float4* xs = dwsm;                                   // [FIH*FIW][kPS]
    float4* ws = xs + G::FIH * G::FIW * kPS;             // [K*K][kCVc]
    float4* red = ws + K * K * kCVc;                     // [4 warps][kCVc]
    const int t = threadIdx.x;
    const int cvl = t & 3;
    const int cvecs = p.C / 4;
    const int cv = blockIdx.x * kCVc + cvl;
    const bool cv_ok = cv < cvecs;
    const int b = blockIdx.z;
    const int cq = cv_ok ? cv * 4 : 0;
    float4 isc = f4zero(), ish = f4zero();
    if (PRE) { isc = ldg4(p.in_scale + cq); ish = ldg4(p.in_shift + cq); }
    const float4 sc1 = ldg4(p.scale + cq), sh1 = ldg4(p.shift + cq);
    for (int i = t; i < K * K * kCVc; i += kDwT)         // i & 3 == cvl
        ws[i] = cv_ok ? ldg4(p.w_kkc + (long long)(i >> 2) * p.C + cq) : f4zero();
    const float* xb = p.x + (long long)b * p.H * p.W * p.C + cq;
    float* zb = p.z + (long long)b * p.Ho * p.Wo * p.C + cq;
    float4 se = f4zero();
    const int tile_end = min(ntiles, (int)(blockIdx.y + 1) * tiles_per_cta);
    for (int tile = blockIdx.y * tiles_per_cta; tile < tile_end; ++tile) {
        const int ty = tile / tiles_x, tx = tile - ty * tiles_x;
        const int oy0 = ty * G::TOY, ox0 = tx * G::TOX;
        const int iy0 = oy0 * S - p.pad_t, ix0 = ox0 * S - p.pad_l;
        __syncthreads();                                 // the previous tile has been consumed (also orders ws)
        for (int i = t; i < G::FIH * G::FIW * kCVc; i += kDwT) {
            const int pix = i >> 2;
            const int r = pix / G::FIW, c = pix - r * G::FIW;
            const int iy = iy0 + r, ix = ix0 + c;
            const bool ok = cv_ok && iy >= 0 && iy < p.H && ix >= 0 && ix < p.W;
            dw_cp_async16(&xs[pix * kPS + cvl], ok ? xb + ((long long)iy * p.W + ix) * p.C : xb, ok ? 16 : 0);
        }
        dw_cp_async_wait_all();
        if (PRE) {                                       // BN0 + swish once per staged element, in place (own copies only)
            for (int i = t; i < G::FIH * G::FIW * kCVc; i += kDwT) {
                const int pix = i >> 2;
                const int r = pix / G::FIW, c = pix - r * G::FIW;
                const int iy = iy0 + r, ix = ix0 + c;
                if (cv_ok && iy >= 0 && iy < p.H && ix >= 0 && ix < p.W)      // padding stays zero AFTER the activation
                    xs[pix * kPS + cvl] = f4swish(f4fma(xs[pix * kPS + cvl], isc, ish));
            }
        }
        __syncthreads();
        constexpr int NCOL = 3 * S + K;
        for (int item = t; item < G::TOY * (G::TOX / 4) * kCVc; item += kDwT) {
            const int sp = item >> 2;
            const int oyl = sp / (G::TOX / 4), oxl0 = (sp - oyl * (G::TOX / 4)) * 4;
            const int oy = oy0 + oyl;
            if (oy >= p.Ho || ox0 + oxl0 >= p.Wo || !cv_ok) continue;
            float4 acc[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[i] = f4zero();
#pragma unroll
            for (int ky = 0; ky < K; ++ky) {
                float4 wrow[K];
#pragma unroll
                for (int kx = 0; kx < K; ++kx) wrow[kx] = ws[(ky * K + kx) * kCVc + cvl];
                const float4* xr = xs + ((oyl * S + ky) * G::FIW + oxl0 * S) * kPS + cvl;
#pragma unroll
                for (int j = 0; j < NCOL; ++j) {
                    const float4 v = xr[j * kPS];
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const int kx = j - i * S;
                        if (kx >= 0 && kx < K) acc[i] = f4fma(v, wrow[kx], acc[i]);
                    }
                }
            }
            float* zo = zb + ((long long)oy * p.Wo + ox0 + oxl0) * p.C;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                if (ox0 + oxl0 + i >= p.Wo) break;
                st4(zo + (long long)i * p.C, acc[i]);
                se = f4add(se, f4swish(f4fma(acc[i], sc1, sh1)));
            }
        }
    }
    // squeeze-excite partial sums: lanes sharing a channel vector -> one value per warp -> one atomic per CTA
    se = cv_group_sum(se);
    __syncthreads();
    if ((t & 31) < 4) red[(t >> 5) * kCVc + (t & 3)] = se;
    __syncthreads();
    if (t < 4 && cv_ok) {
        float4 s = f4zero();
#pragma unroll
        for (int w = 0; w < kDwT / 32; ++w) s = f4add(s, red[w * kCVc + t]);
        float* o = p.se_sum + (long long)b * p.C + cq;
        atomicAdd(o + 0, p.se_alpha * s.x); atomicAdd(o + 1, p.se_alpha * s.y);
        atomicAdd(o + 2, p.se_alpha * s.z); atomicAdd(o + 3, p.se_alpha * s.w);
    }
}

// ------------------------------------------------------------------------------------------------------------------
// backward
// ------------------------------------------------------------------------------------------------------------------
template <int K, int S, bool PRE, bool SMALL>
__global__ void __launch_bounds__((DwGeo<K, S, SMALL>::NT), (DwGeo<K, S, SMALL>::NT == 256 ? 1 : 2))
dw_bwd_fused_kernel(const effdet_dw_bwd_args p, const int tiles_x, const int ntiles, const int tiles_per_cta) {
    using G = DwGeo<K, S, SMALL>;
    constexpr int kDwT = G::NT;
    constexpr int KK = K * K;
    constexpr int NQ = KK + 4;                           // reduced quantities: dW taps, dgamma1, dbeta1, dgamma0, dbeta0
    extern __shared__ __align__(16) float4 dwsm[];
    float4* gs = dwsm;                                   // dq, then dz1 of the touched outputs   [GH*GW][kPS]
    float4* z1s = gs + G::GH * G::GW * kPS;              // raw z1 of the same outputs            [GH*GW][kPS]
    float4* as = z1s + G::GH * G::GW * kPS;              // sigmoid(bn0(z0)) (PRE) or a0 = x      [BIH*BIW][kPS]
    float4* zs = as + G::BIH * G::BIW * kPS;             // raw z0 (PRE only)            [BIH*BIW][kPS]
    float4* ws = zs + (PRE ? G::BIH * G::BIW * kPS : 0); // [KK][kCVc]
    float4* red = ws + KK * kCVc;                        // [NQ][4 warps][kCVc]
    const int t = threadIdx.x;
    const int cvl = t & 3;
    const int cvecs = p.C / 4;
    const int cv = blockIdx.x * kCVc + cvl;
    const bool cv_ok = cv < cvecs;
    const int b = blockIdx.z;
    const int cq = cv_ok ? cv * 4 : 0;
    // per-channel constants live in shared memory, not in 40 registers: the 5x5 kernels already carry 25 float4
    // weight-gradient accumulators per thread and spilled them when these stayed in registers
    float4* cst = red + NQ * (kDwT / 32) * kCVc;         // [10][kCVc]: sc1 sh1 mu1 rs1 gate dmean/HW sc0 sh0 mu0 rs0
    if (t < 10 * kCVc) {
        const int q = t >> 2, c4 = (blockIdx.x * kCVc + (t & 3)) * 4;
        float4 v = f4zero();
        if (c4 < p.C) {
            const float* src = q == 0 ? p.scale1 : q == 1 ? p.shift1 : q == 2 ? p.mean1 : q == 3 ? p.rstd1
                             : q == 4 ? p.gate + (long long)b * p.C : q == 5 ? p.dmean + (long long)b * p.C
                             : q == 6 ? p.scale0 : q == 7 ? p.shift0 : q == 8 ? p.mean0 : p.rstd0;
            if (q < 6 || PRE) v = ldg4(src + c4);
            if (q == 5) v = f4scale(v, p.inv_hw);
        }
        cst[t] = v;
    }
#define DWC(q_) cst[(q_) * kCVc + cvl]
    for (int i = t; i < KK * kCVc; i += kDwT) ws[i] = cv_ok ? ldg4(p.w_kkc + (long long)(i >> 2) * p.C + cq) : f4zero();
    const float* dqb = p.dq + (long long)b * p.Ho * p.Wo * p.C + cq;
    const float* z1b = p.z1 + (long long)b * p.Ho * p.Wo * p.C + cq;
    const float* xb = p.x + (long long)b * p.H * p.W * p.C + cq;
    float* dxb = p.dx + (long long)b * p.H * p.W * p.C + cq;

    float4 dW[KK];
#pragma unroll
    for (int i = 0; i < KK; ++i) dW[i] = f4zero();
    float4 sg1 = f4zero(), sb1 = f4zero(), sg0 = f4zero(), sb0 = f4zero();

    const int tile_end = min(ntiles, (int)(blockIdx.y + 1) * tiles_per_cta);
    for (int tile = blockIdx.y * tiles_per_cta; tile < tile_end; ++tile) {
        const int ty = tile / tiles_x, tx = tile - ty * tiles_x;
        const int cy0 = ty * G::TCY, cx0 = tx * G::TCX;          // first cell (= output coordinate) of the tile
        __syncthreads();
        // ---- stage the raw operands: every 16-byte copy of the tile is in flight before anything waits ---------------
        for (int i = t; i < G::GH * G::GW * kCVc; i += kDwT) {
            const int pix = i >> 2;
            const int r = pix / G::GW, c = pix - r * G::GW;
            const int oy = cy0 + r + G::DMIN, ox = cx0 + c + G::DMIN;
            const bool ok = cv_ok && oy >= 0 && oy < p.Ho && ox >= 0 && ox < p.Wo;
            const long long off = ok ? ((long long)oy * p.Wo + ox) * p.C : 0;
            dw_cp_async16(&gs[pix * kPS + cvl], dqb + off, ok ? 16 : 0);
            dw_cp_async16(&z1s[pix * kPS + cvl], z1b + off, ok ? 16 : 0);
        }
        for (int i = t; i < G::BIH * G::BIW * kCVc; i += kDwT) {
            const int pix = i >> 2;
            const int r = pix / G::BIW, c = pix - r * G::BIW;
            const int iy = cy0 * S + r, ix = cx0 * S + c;
            const bool ok = cv_ok && iy < p.H && ix < p.W;
            dw_cp_async16(PRE ? &zs[pix * kPS + cvl] : &as[pix * kPS + cvl], ok ? xb + ((long long)iy * p.W + ix) * p.C : xb,
                          ok ? 16 : 0);
        }
        dw_cp_async_wait_all();
        // ---- dz1 in place of dq (each thread transforms the elements it copied itself) --------------------------------
        for (int i = t; i < G::GH * G::GW * kCVc; i += kDwT) {
            const int pix = i >> 2;
            const int r = pix / G::GW, c = pix - r * G::GW;
            const int oy = cy0 + r + G::DMIN, ox = cx0 + c + G::DMIN;
            if (!(cv_ok && oy >= 0 && oy < p.Ho && ox >= 0 && ox < p.Wo)) continue;     // zero-filled: contributes nothing
            const float4 g = f4fma(gs[pix * kPS + cvl], DWC(4), DWC(5));              // SE product rule: d(a1*gate) + d(mean)
            const float4 z = z1s[pix * kPS + cvl];
            const float4 sc1 = DWC(0);
            const float4 du = f4mul(g, f4swish_grad(f4fma(z, sc1, DWC(1))));
            const bool owned = r + G::DMIN >= 0 && r + G::DMIN < G::TCY && c + G::DMIN >= 0 && c + G::DMIN < G::TCX;
            if (owned) {                                                       // each output is counted by exactly one tile
                sg1 = f4fma(du, f4mul(f4sub(z, DWC(2)), DWC(3)), sg1);
                sb1 = f4add(sb1, du);
            }
            gs[pix * kPS + cvl] = f4mul(du, sc1);
        }
        // ---- activated a0 next to the raw z0 (BN0 backward needs both) --------------------------------------------------
        if (PRE) {
            for (int i = t; i < G::BIH * G::BIW * kCVc; i += kDwT) {
                const int pix = i >> 2;
                const int r = pix / G::BIW, c = pix - r * G::BIW;
                const int iy = cy0 * S + r, ix = cx0 * S + c;
                const bool ok = cv_ok && iy < p.H && ix < p.W;
                float4 sg = f4zero();                       // sigmoid(bn0(z0)): a0 = u*sg and swish'(u) both follow from it
                if (ok) {
                    const float4 q = f4fma(zs[pix * kPS + cvl], DWC(6), DWC(7));
                    sg = make_float4(fsigmoid(q.x), fsigmoid(q.y), fsigmoid(q.z), fsigmoid(q.w));
                }
                as[pix * kPS + cvl] = sg;
            }
        }
        __syncthreads();
        // ---- strips of 4 cells: data gradient, weight gradient, BN0 backward ------------------------------------------
        for (int item = t; item < G::TCY * (G::TCX / 4) * kCVc; item += kDwT) {
            const int sp = item >> 2;
            const int al = sp / (G::TCX / 4), bl0 = (sp - al * (G::TCX / 4)) * 4;
            if ((cy0 + al) * S >= p.H || (cx0 + bl0) * S >= p.W || !cv_ok) continue;
#pragma unroll
            for (int py = 0; py < S; ++py) {
#pragma unroll
                for (int px = 0; px < S; ++px) {
                    float4 da[4], a0[4];
                    const int arow = (al * S + py) * G::BIW + bl0 * S + px;
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        da[i] = f4zero();
                        a0[i] = as[(arow + i * S) * kPS + cvl];
                        if (PRE)                              // staged: sigmoid(u) and raw z0 -> a0 = u * sigmoid(u)
                            a0[i] = f4mul(f4fma(zs[(arow + i * S) * kPS + cvl], DWC(6), DWC(7)), a0[i]);   // out of image: sigmoid staged as 0
                    }
#pragma unroll
                    for (int ky = 0; ky < K; ++ky) {
                        if ((py + G::PT - ky) % S != 0) continue;                  // compile-time after unrolling
                        const int dy = (py + G::PT - ky) / S;
                        float4 gw[4 + G::DMAX - G::DMIN];
                        const float4* gr = gs + ((al + dy - G::DMIN) * G::GW + bl0) * kPS + cvl;
#pragma unroll
                        for (int j = 0; j < 4 + G::DMAX - G::DMIN; ++j) gw[j] = gr[j * kPS];
#pragma unroll
                        for (int kx = 0; kx < K; ++kx) {
                            if ((px + G::PT - kx) % S != 0) continue;
                            const int dx = (px + G::PT - kx) / S;
                            const float4 w = ws[(ky * K + kx) * kCVc + cvl];
#pragma unroll
                            for (int i = 0; i < 4; ++i) {
                                const float4 g = gw[i + dx - G::DMIN];
                                da[i] = f4fma(g, w, da[i]);
                                dW[ky * K + kx] = f4fma(a0[i], g, dW[ky * K + kx]);
                            }
                        }
                    }
                    const int iy = (cy0 + al) * S + py;
                    if (iy >= p.H) continue;
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const int ix = (cx0 + bl0 + i) * S + px;
                        if (ix >= p.W) break;
                        float4 out = da[i];
                        if (PRE) {
                            const float4 z = zs[(arow + i * S) * kPS + cvl];
                            const float4 sc0 = DWC(6);
                            const float4 sg = as[(arow + i * S) * kPS + cvl], uu = f4fma(z, sc0, DWC(7));   // swish'(u) = s * (1 + u * (1 - s))
                            const float4 sp = make_float4(sg.x * (1.f + uu.x * (1.f - sg.x)), sg.y * (1.f + uu.y * (1.f - sg.y)),
                                                          sg.z * (1.f + uu.z * (1.f - sg.z)), sg.w * (1.f + uu.w * (1.f - sg.w)));
                            const float4 du = f4mul(da[i], sp);
                            sg0 = f4fma(du, f4mul(f4sub(z, DWC(8)), DWC(9)), sg0);
                            sb0 = f4add(sb0, du);
                            out = f4mul(du, sc0);
                        }
                        if (p.dx_planes) {                    // bf16 hi/lo planes: the operand format of the expand conv's
                            const __nv_bfloat162 h0 = __floats2bfloat162_rn(out.x, out.y), h1 = __floats2bfloat162_rn(out.z, out.w);
                            const __nv_bfloat162 l0 = __floats2bfloat162_rn(out.x - __low2float(h0), out.y - __high2float(h0));
                            const __nv_bfloat162 l1 = __floats2bfloat162_rn(out.z - __low2float(h1), out.w - __high2float(h1));
                            const long long e = (((long long)b * p.H + iy) * p.W + ix) * p.C + cq;   // tensor-core gradients
                            __nv_bfloat16* pl = reinterpret_cast<__nv_bfloat16*>(p.dx_planes);
                            *reinterpret_cast<uint2*>(pl + e) =
                                make_uint2(*reinterpret_cast<const uint32_t*>(&h0), *reinterpret_cast<const uint32_t*>(&h1));
                            *reinterpret_cast<uint2*>(pl + (long long)p.B * p.H * p.W * p.C + e) =
                                make_uint2(*reinterpret_cast<const uint32_t*>(&l0), *reinterpret_cast<const uint32_t*>(&l1));
                        } else {
                            st4(dxb + ((long long)iy * p.W + ix) * p.C, out);
                        }
                    }
                }
            }
        }
    }
    // ---- per-channel reductions: lanes -> warps (shuffles) -> CTA (shared memory) -> global atomics --------------------
    __syncthreads();
    const int warp = t >> 5, lane = t & 31;
#pragma unroll
    for (int q = 0; q < NQ; ++q) {
        float4 v = q < KK ? dW[q] : (q == KK ? sg1 : (q == KK + 1 ? sb1 : (q == KK + 2 ? sg0 : sb0)));
        v = cv_group_sum(v);
        if (lane < 4) red[(q * (kDwT / 32) + warp) * kCVc + lane] = v;
    }
    __syncthreads();
    for (int i = t; i < NQ * kCVc; i += kDwT) {
        const int q = i >> 2, c4 = i & 3;
        const int ccv = blockIdx.x * kCVc + c4;
        if (ccv >= cvecs) continue;
        if (!PRE && q >= KK + 2) continue;
        float4 s = f4zero();
#pragma unroll
        for (int w = 0; w < kDwT / 32; ++w) s = f4add(s, red[(q * (kDwT / 32) + w) * kCVc + c4]);
        const int c = ccv * 4;
        if (q < KK) {
            float* o = p.dw + (long long)c * KK + q;
            atomicAdd(o, s.x); atomicAdd(o + KK, s.y); atomicAdd(o + 2 * KK, s.z); atomicAdd(o + 3 * KK, s.w);
        } else {
            float* o = (q == KK ? p.dgamma1 : (q == KK + 1 ? p.dbeta1 : (q == KK + 2 ? p.dgamma0 : p.dbeta0))) + c;
            atomicAdd(o, s.x); atomicAdd(o + 1, s.y); atomicAdd(o + 2, s.z); atomicAdd(o + 3, s.w);
        }
    }
}

#undef DWC

template <int K, int S, bool PRE, bool SMALL>
static size_t dw_fwd_smem() {
    using G = DwGeo<K, S, SMALL>;
    constexpr int kDwT = G::NT;
    return (size_t)(G::FIH * G::FIW * kPS + K * K * kCVc + (kDwT / 32) * kCVc) * sizeof(float4);
}
template <int K, int S, bool PRE, bool SMALL>
static size_t dw_bwd_smem() {
    using G = DwGeo<K, S, SMALL>;
    constexpr int kDwT = G::NT;
    return (size_t)(2 * G::GH * G::GW * kPS + (PRE ? 2 : 1) * G::BIH * G::BIW * kPS + K * K * kCVc +
                    (K * K + 4) * (kDwT / 32) * kCVc + 10 * kCVc) * sizeof(float4);
}

// tiles per CTA: keep >= ~6 waves of CTAs in the grid, but let a CTA amortise its reductions over up to 8 tiles.
// tests/test_benchmark_plans.py (_dw_plan) mirrors this and the tile grids of both launchers.
static int pick_tiles_per_cta(long long ntiles, long long other) {
    long long tpc = (ntiles * other) / (148ll * 6 * 3);
    if (tpc < 1) tpc = 1;
    if (tpc > 8) tpc = 8;
    if (tpc > ntiles) tpc = ntiles;
    return (int)tpc;
}

__global__ void pack_dw_weight_kernel(const float* __restrict__ w, float* __restrict__ o, int C, int kk) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;  // output index [tap][c]
    if (i >= C * kk) return;
    const int c = i % C, tap = i / C;
    o[i] = __ldg(w + c * kk + tap);
}

}  // namespace effdet

using namespace effdet;

static int dw_fused_geometry_ok(const char* who, int k, int stride, int pad_t, int pad_l, int C, int B) {
    EFFDET_REQUIRE((k == 3 || k == 5) && (stride == 1 || stride == 2), "%s: k=%d stride=%d unsupported", who, k, stride);
    const int pt = stride == 1 ? (k - 1) / 2 : (k == 3 ? 0 : 1);
    EFFDET_REQUIRE(pad_t == pt && pad_l == pt,
                   "%s: pads (%d,%d) differ from the reference's static padding (%d) for k=%d stride=%d", who, pad_t, pad_l, pt,
                   k, stride);
    EFFDET_REQUIRE(C > 0 && C % 4 == 0 && B > 0 && B <= 65535, "%s: bad shape (C must be a multiple of 4)", who);
    return EFFDET_OK;
}

extern "C" int effdet_dwconv_fwd_fused(const effdet_dw_fwd_args* a, int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(a && a->x && a->w_kkc && a->scale && a->shift && a->z && a->se_sum, "dwconv_fwd_fused: null tensor");
    EFFDET_REQUIRE((a->in_scale == nullptr) == (a->in_shift == nullptr), "dwconv_fwd_fused: in_scale/in_shift come together");
    EFFDET_REQUIRE(aligned16(a->x) && aligned16(a->w_kkc) && aligned16(a->scale) && aligned16(a->shift) && aligned16(a->z) &&
                       aligned16(a->in_scale) && aligned16(a->in_shift) && aligned16(a->se_sum),
                   "dwconv_fwd_fused: alignment");
    int s = dw_fused_geometry_ok("dwconv_fwd_fused", a->k, a->stride, a->pad_t, a->pad_l, a->C, a->B);
    if (s) return s;
    EFFDET_REQUIRE(a->H > 0 && a->W > 0 && a->Ho > 0 && a->Wo > 0 && (a->Ho - 1) * a->stride + a->k - a->pad_t <= a->H + a->k &&
                       (a->Wo - 1) * a->stride + a->k - a->pad_l <= a->W + a->k,
                   "dwconv_fwd_fused: bad output size");
    EFFDET_DEVICE(device);
    cudaStream_t st = (cudaStream_t)stream;
    const int chunks = cdiv(a->C / 4, kCVc);
#define EFFDET_DWF(K_, S_, PRE_, SM_)                                                                                     \
    do {                                                                                                                  \
        using G = DwGeo<K_, S_, SM_>;                                                                                     \
        const int tiles_x = cdiv(a->Wo, G::TOX), tiles_y = cdiv(a->Ho, G::TOY);                                           \
        const int ntiles = tiles_x * tiles_y;                                                                             \
        const int tpc = pick_tiles_per_cta(ntiles, (long long)chunks * a->B);                                             \
        const size_t smem = dw_fwd_smem<K_, S_, PRE_, SM_>();                                                             \
        cudaError_t e = cudaFuncSetAttribute(dw_fwd_fused_kernel<K_, S_, PRE_, SM_>,                                      \
                                             cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);                     \
        if (e != cudaSuccess) return fail(EFFDET_ERR_LAUNCH, "dwconv_fwd_fused: smem opt-in: %s", cudaGetErrorString(e)); \
        dw_fwd_fused_kernel<K_, S_, PRE_, SM_><<<dim3(chunks, cdiv(ntiles, tpc), a->B), G::NT, smem, st>>>(*a, tiles_x, ntiles, tpc); \
    } while (0)
#define EFFDET_DWF_KS(PRE_, SM_)                                                                                          \
    do {                                                                                                                  \
        if (a->k == 3 && a->stride == 1) EFFDET_DWF(3, 1, PRE_, SM_);                                                     \
        else if (a->k == 3) EFFDET_DWF(3, 2, PRE_, SM_);                                                                  \
        else if (a->stride == 1) EFFDET_DWF(5, 1, PRE_, SM_);                                                             \
        else EFFDET_DWF(5, 2, PRE_, SM_);                                                                                 \
    } while (0)
    const bool small = a->Ho <= 8 && a->Wo <= 8;             // late stages: the whole map fits a small tile
    if (a->in_scale) { if (small) EFFDET_DWF_KS(true, true); else EFFDET_DWF_KS(true, false); }
    else { if (small) EFFDET_DWF_KS(false, true); else EFFDET_DWF_KS(false, false); }
#undef EFFDET_DWF_KS
#undef EFFDET_DWF
    return launch_status("dw_fwd_fused_kernel");
}

extern "C" int effdet_dwconv_bwd_fused(const effdet_dw_bwd_args* a, int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(a && a->dq && a->z1 && a->gate && a->dmean && a->scale1 && a->shift1 && a->mean1 && a->rstd1 && a->x &&
                       a->w_kkc && (a->dx || a->dx_planes) && a->dw && a->dgamma1 && a->dbeta1,
                   "dwconv_bwd_fused: null tensor");
    EFFDET_REQUIRE(!a->dx_planes || (a->C % 8 == 0 && aligned16(a->dx_planes)), "dwconv_bwd_fused: dx_planes needs C %% 8 == 0");
    const bool pre = a->scale0 != nullptr;
    EFFDET_REQUIRE(!pre || (a->shift0 && a->mean0 && a->rstd0 && a->dgamma0 && a->dbeta0), "dwconv_bwd_fused: BN0 tensors come together");
    EFFDET_REQUIRE(aligned16(a->dq) && aligned16(a->z1) && aligned16(a->gate) && aligned16(a->dmean) && aligned16(a->x) &&
                       aligned16(a->w_kkc) && aligned16(a->dx) && aligned16(a->scale1) && aligned16(a->shift1) &&
                       aligned16(a->mean1) && aligned16(a->rstd1) && aligned16(a->scale0) && aligned16(a->shift0) &&
                       aligned16(a->mean0) && aligned16(a->rstd0),
                   "dwconv_bwd_fused: alignment");
    int s = dw_fused_geometry_ok("dwconv_bwd_fused", a->k, a->stride, a->pad_t, a->pad_l, a->C, a->B);
    if (s) return s;
    EFFDET_REQUIRE(a->H > 0 && a->W > 0 && a->Ho > 0 && a->Wo > 0 && a->Ho <= cdiv(a->H, a->stride) && a->Wo <= cdiv(a->W, a->stride),
                   "dwconv_bwd_fused: bad output size");
    EFFDET_DEVICE(device);
    cudaStream_t st = (cudaStream_t)stream;
    const int chunks = cdiv(a->C / 4, kCVc);
#define EFFDET_DWB(K_, S_, PRE_, SM_)                                                                                     \
    do {                                                                                                                  \
        using G = DwGeo<K_, S_, SM_>;                                                                                     \
        const int tiles_x = cdiv(cdiv(a->W, S_), G::TCX), tiles_y = cdiv(cdiv(a->H, S_), G::TCY);                         \
        const int ntiles = tiles_x * tiles_y;                                                                             \
        const int tpc = pick_tiles_per_cta(ntiles, (long long)chunks * a->B);                                             \
        const size_t smem = dw_bwd_smem<K_, S_, PRE_, SM_>();                                                             \
        cudaError_t e = cudaFuncSetAttribute(dw_bwd_fused_kernel<K_, S_, PRE_, SM_>,                                      \
                                             cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);                     \
        if (e != cudaSuccess) return fail(EFFDET_ERR_LAUNCH, "dwconv_bwd_fused: smem opt-in: %s", cudaGetErrorString(e)); \
        dw_bwd_fused_kernel<K_, S_, PRE_, SM_><<<dim3(chunks, cdiv(ntiles, tpc), a->B), G::NT, smem, st>>>(*a, tiles_x, ntiles, tpc); \
    } while (0)
#define EFFDET_DWB_KS(PRE_, SM_)                                                                                          \
    do {                                                                                                                  \
        if (a->k == 3 && a->stride == 1) EFFDET_DWB(3, 1, PRE_, SM_);                                                     \
        else if (a->k == 3) EFFDET_DWB(3, 2, PRE_, SM_);                                                                  \
        else if (a->stride == 1) EFFDET_DWB(5, 1, PRE_, SM_);                                                             \
        else EFFDET_DWB(5, 2, PRE_, SM_);                                                                                 \
    } while (0)
    const bool small = cdiv(a->H, a->stride) <= 8 && cdiv(a->W, a->stride) <= 8;
    if (pre) { if (small) EFFDET_DWB_KS(true, true); else EFFDET_DWB_KS(true, false); }
    else { if (small) EFFDET_DWB_KS(false, true); else EFFDET_DWB_KS(false, false); }
#undef EFFDET_DWB_KS
#undef EFFDET_DWB
    return launch_status("dw_bwd_fused_kernel");
}

extern "C" int effdet_pack_dw_weight(const float* w_c1kk, float* w_kkc, int C, int k, int device,
                                     effdet_stream_t stream) {
    EFFDET_REQUIRE(w_c1kk && w_kkc && C > 0 && (k == 3 || k == 5), "pack_dw_weight: bad arguments");
    EFFDET_DEVICE(device);
    pack_dw_weight_kernel<<<cdiv((long long)C * k * k, 256), 256, 0, (cudaStream_t)stream>>>(w_c1kk, w_kkc, C, k * k);
    return launch_status("pack_dw_weight_kernel");
}
