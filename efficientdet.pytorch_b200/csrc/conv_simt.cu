// Exact-fp32 implicit-GEMM convolution (k in {1,3}, stride 1, same padding) on the CUDA cores,
// with every per-layer element-wise op of the reference folded into the prologue / epilogue.
// This is the parity engine for the HBM-bound backbone / neck layers (SURVEY.md H2) and the
// fallback-free baseline for the head until the wgmma path takes over the 256-channel convs.
//
// Reference ops replaced: F.conv2d + bias + BN(eval) + ReLU/swish/sigmoid + residual
//   models/module.py:507-515, models/retinahead.py:109-129, models/efficientnet.py:85,96-104
// and their autograd backward (dgrad = same kernel on the rotated/transposed pack; wgrad below).
#include "common.cuh"

namespace effdet {

constexpr int kBM = 128;   // output pixels per CTA
constexpr int kBK = 16;    // reduction slice (channels of one tap)
constexpr int kNT = 256;   // threads per CTA

template <int BN, int TN>
__global__ void __launch_bounds__(kNT, 2) conv_igemm_kernel(const effdet_conv_args p, const int M, const int HW) {
    constexpr int TXN = BN / TN;        // threads along N
    constexpr int TYN = kNT / TXN;      // threads along M
    constexpr int TM = kBM / TYN;       // rows per thread
    constexpr int G = TN / 4;           // float4 column groups per thread
    constexpr int GS = BN / G;          // column distance between groups
    constexpr int B4 = (kBK * BN / 4 + kNT - 1) / kNT;  // weight float4 per thread per stage

    __shared__ __align__(16) float As[2][kBM][kBK];
    __shared__ __align__(16) float Bs[2][kBK][BN];

    const int t = threadIdx.x;
    const int tx = t % TXN, ty = t / TXN;
    const int m0 = blockIdx.x * kBM, n0 = blockIdx.y * BN;
    const int pad = p.ksize / 2;
    const int taps = p.ksize * p.ksize;
    const int kchunks = (p.Cin + kBK - 1) / kBK;
    const int KT = taps * kchunks;

    // --- A-operand rows owned by this thread for loading: rows r0 and r0+64, float4 slot kq ---
    const int kq = t & 3;
    int a_oy[2], a_ox[2], a_b[2];
    bool a_ok[2];
    long long a_off[2];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
        int m = m0 + (t >> 2) + j * 64;
        a_ok[j] = m < M;
        int mm = a_ok[j] ? m : 0;
        int b = mm / HW;
        int pix = mm - b * HW;
        a_b[j] = b;
        a_oy[j] = pix / p.W;
        a_ox[j] = pix - a_oy[j] * p.W;
        a_off[j] = (long long)b * p.x_bstride;
    }

    float4 ra[2], rb[B4];
    auto load_tile = [&](int kt) {
        const int tap = kt / kchunks;
        const int c0 = (kt - tap * kchunks) * kBK;
        const int ky = tap / p.ksize, kx = tap - ky * p.ksize;
        const int c = c0 + kq * 4;
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int iy = a_oy[j] + ky - pad, ix = a_ox[j] + kx - pad;
            const bool ok = a_ok[j] && c < p.Cin && iy >= 0 && iy < p.H && ix >= 0 && ix < p.W;
            float4 v = f4zero();
            if (ok) {
                v = ldg4(p.x + a_off[j] + ((long long)iy * p.W + ix) * p.Cin + c);
                if (p.in_scale) {                      // raw conv output -> swish(bn(.)) while the tile is staged
                    const float4 u = f4fma(v, ldg4(p.in_scale + c), ldg4(p.in_shift + c));
                    v = make_float4(swishf_(u.x), swishf_(u.y), swishf_(u.z), swishf_(u.w));
                }
                if (p.a_scale) v = f4mul(v, ldg4(p.a_scale + (long long)a_b[j] * p.Cin + c));
            }
            ra[j] = v;
        }
#pragma unroll
        for (int j = 0; j < B4; ++j) {
            const int idx = t + j * kNT;
            float4 v = f4zero();
            if (idx < kBK * BN / 4) {
                const int kr = idx / (BN / 4);
                const int n = n0 + (idx - kr * (BN / 4)) * 4;
                const int cc = c0 + kr;
                if (cc < p.Cin && n < p.Cout) v = ldg4(p.w + ((long long)tap * p.Cin + cc) * p.Cout + n);
            }
            rb[j] = v;
        }
    };
    auto store_tile = [&](int s) {
#pragma unroll
        for (int j = 0; j < 2; ++j) st4(&As[s][(t >> 2) + j * 64][kq * 4], ra[j]);
#pragma unroll
        for (int j = 0; j < B4; ++j) {
            const int idx = t + j * kNT;
            if (idx < kBK * BN / 4) {
                const int kr = idx / (BN / 4);
                st4(&Bs[s][kr][(idx - kr * (BN / 4)) * 4], rb[j]);
            }
        }
    };

    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

    load_tile(0);
    store_tile(0);
    __syncthreads();
    for (int kt = 0; kt < KT; ++kt) {
        const int s = kt & 1;
        if (kt + 1 < KT) load_tile(kt + 1);
#pragma unroll
        for (int kk = 0; kk < kBK; kk += 4) {
            float4 a[TM];
#pragma unroll
            for (int i = 0; i < TM; ++i) a[i] = *reinterpret_cast<const float4*>(&As[s][ty * TM + i][kk]);
#pragma unroll
            for (int k4 = 0; k4 < 4; ++k4) {
                float bv[TN];
#pragma unroll
                for (int g = 0; g < G; ++g) {
                    const float4 q = *reinterpret_cast<const float4*>(&Bs[s][kk + k4][g * GS + tx * 4]);
                    bv[g * 4 + 0] = q.x; bv[g * 4 + 1] = q.y; bv[g * 4 + 2] = q.z; bv[g * 4 + 3] = q.w;
                }
#pragma unroll
                for (int i = 0; i < TM; ++i) {
                    const float av = k4 == 0 ? a[i].x : (k4 == 1 ? a[i].y : (k4 == 2 ? a[i].z : a[i].w));
#pragma unroll
                    for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(av, bv[j], acc[i][j]);
                }
            }
        }
        if (kt + 1 < KT) store_tile(s ^ 1);
        __syncthreads();
    }

    // --- epilogue -------------------------------------------------------------------------------
#pragma unroll
    for (int i = 0; i < TM; ++i) {
        const int m = m0 + ty * TM + i;
        if (m >= M) continue;
        const int b = m / HW;
        const long long pix = m - b * HW;
        const float rs = p.row_scale ? __ldg(p.row_scale + b) : 1.f;
#pragma unroll
        for (int g = 0; g < G; ++g) {
            const int n = n0 + g * GS + tx * 4;
            if (n >= p.Cout) continue;
            float4 v = make_float4(acc[i][g * 4 + 0], acc[i][g * 4 + 1], acc[i][g * 4 + 2], acc[i][g * 4 + 3]);
            if (p.bias) v = f4add(v, ldg4(p.bias + n));
            const long long yo = (long long)b * p.y_bstride + pix * p.Cout + n;
            if (p.z) st4(p.z + yo, v);
            if (p.scale) v = f4fma(v, ldg4(p.scale + n), ldg4(p.shift + n));
            if (p.act == EFFDET_ACT_RELU) {
                v = make_float4(fmaxf(v.x, 0.f), fmaxf(v.y, 0.f), fmaxf(v.z, 0.f), fmaxf(v.w, 0.f));
            } else if (p.act == EFFDET_ACT_SWISH) {
                v = make_float4(swishf_(v.x), swishf_(v.y), swishf_(v.z), swishf_(v.w));
            } else if (p.act == EFFDET_ACT_SIGMOID) {
                v = make_float4(sigmoidf_(v.x), sigmoidf_(v.y), sigmoidf_(v.z), sigmoidf_(v.w));
            }
            if (p.row_scale) v = f4scale(v, rs);
            if (p.residual) v = f4add(v, ldg4(p.residual + (long long)b * p.r_bstride + pix * p.Cout + n));
            if (p.mask_src) {
                const float4 q = ldg4(p.mask_src + (long long)b * p.m_bstride + pix * p.Cout + n);
                v = make_float4(q.x > 0.f ? v.x : 0.f, q.y > 0.f ? v.y : 0.f, q.z > 0.f ? v.z : 0.f,
                                q.w > 0.f ? v.w : 0.f);
            }
            st4(p.y + yo, v);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Weight gradient: dW[c, n | tap] = sum over pixels of x[pixel+tap, c] * dy[pixel, n]
// CTA tile BC x BN of (Cin x Cout) for one tap and one slice of the pixel range; fp32 atomics
// merge the slices (and the five pyramid levels that share head weights).
// ------------------------------------------------------------------------------------------------
template <int BC, int BN, int TC, int TN>
__global__ void __launch_bounds__(kNT, 2) conv_wgrad_kernel(const effdet_wgrad_args p, const int M, const int HW,
                                                         const int chunks_per_split, const int ctiles) {
    constexpr int TXN = BN / TN;
    constexpr int GC = TC / 4 > 0 ? TC / 4 : 1, GN = TN / 4;
    constexpr int GSC = BC / GC, GSN = BN / GN;
    static_assert((BC / TC) * (BN / TN) == kNT, "thread tiling");
    static_assert(TC % 4 == 0 && TN % 4 == 0, "float4 micro tiles");
    constexpr int A4 = (kBK * BC / 4 + kNT - 1) / kNT;
    constexpr int B4 = (kBK * BN / 4 + kNT - 1) / kNT;

    __shared__ __align__(16) float As[2][kBK][BC];
    __shared__ __align__(16) float Bs[2][kBK][BN];

    const int t = threadIdx.x;
    const int tx = t % TXN, ty = t / TXN;
    const int ct = blockIdx.x % ctiles, nt = blockIdx.x / ctiles;
    const int c0 = ct * BC, n0 = nt * BN;
    const int tap = blockIdx.y;
    const int pad = p.ksize / 2;
    const int ky = tap / p.ksize, kx = tap - ky * p.ksize;
    const int nchunks = (M + kBK - 1) / kBK;
    const int ch_begin = blockIdx.z * chunks_per_split;
    const int ch_end = min(nchunks, ch_begin + chunks_per_split);
    if (ch_begin >= ch_end) return;

    float4 ra[A4], rb[B4];
    auto load_tile = [&](int ch) {
        const int mbase = ch * kBK;
#pragma unroll
        for (int j = 0; j < A4; ++j) {
            const int idx = t + j * kNT;
            float4 v = f4zero();
            if (idx < kBK * BC / 4) {
                const int r = idx / (BC / 4);
                const int c = c0 + (idx - r * (BC / 4)) * 4;
                const int m = mbase + r;
                if (m < M && c < p.Cin) {
                    const int b = m / HW;
                    const int pix = m - b * HW;
                    const int oy = pix / p.W, ox = pix - oy * p.W;
                    const int iy = oy + ky - pad, ix = ox + kx - pad;
                    if (iy >= 0 && iy < p.H && ix >= 0 && ix < p.W) {
                        v = ldg4(p.x + (long long)b * p.x_bstride + ((long long)iy * p.W + ix) * p.Cin + c);
                        if (p.in_scale) {
                            const float4 u = f4fma(v, ldg4(p.in_scale + c), ldg4(p.in_shift + c));
                            v = make_float4(swishf_(u.x), swishf_(u.y), swishf_(u.z), swishf_(u.w));
                        }
                        if (p.a_scale) v = f4mul(v, ldg4(p.a_scale + (long long)b * p.Cin + c));
                    }
                }
            }
            ra[j] = v;
        }
#pragma unroll
        for (int j = 0; j < B4; ++j) {
            const int idx = t + j * kNT;
            float4 v = f4zero();
            if (idx < kBK * BN / 4) {
                const int r = idx / (BN / 4);
                const int n = n0 + (idx - r * (BN / 4)) * 4;
                const int m = mbase + r;
                if (m < M && n < p.Cout) {
                    const int b = m / HW;
                    const long long pix = m - b * HW;
                    v = ldg4(p.dy + (long long)b * p.dy_bstride + pix * p.Cout + n);
                }
            }
            rb[j] = v;
        }
    };
    auto store_tile = [&](int s) {
#pragma unroll
        for (int j = 0; j < A4; ++j) {
            const int idx = t + j * kNT;
            if (idx < kBK * BC / 4) {
                const int r = idx / (BC / 4);
                st4(&As[s][r][(idx - r * (BC / 4)) * 4], ra[j]);
            }
        }
#pragma unroll
        for (int j = 0; j < B4; ++j) {
            const int idx = t + j * kNT;
            if (idx < kBK * BN / 4) {
                const int r = idx / (BN / 4);
                st4(&Bs[s][r][(idx - r * (BN / 4)) * 4], rb[j]);
            }
        }
    };

    float acc[TC][TN];
#pragma unroll
    for (int i = 0; i < TC; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

    load_tile(ch_begin);
    store_tile(0);
    __syncthreads();
    for (int ch = ch_begin; ch < ch_end; ++ch) {
        const int s = (ch - ch_begin) & 1;
        if (ch + 1 < ch_end) load_tile(ch + 1);
#pragma unroll
        for (int r = 0; r < kBK; ++r) {
            float av[TC], bv[TN];
#pragma unroll
            for (int g = 0; g < GC; ++g) {
                const float4 q = *reinterpret_cast<const float4*>(&As[s][r][g * GSC + ty * 4]);
                av[g * 4 + 0] = q.x; av[g * 4 + 1] = q.y; av[g * 4 + 2] = q.z; av[g * 4 + 3] = q.w;
            }
#pragma unroll
            for (int g = 0; g < GN; ++g) {
                const float4 q = *reinterpret_cast<const float4*>(&Bs[s][r][g * GSN + tx * 4]);
                bv[g * 4 + 0] = q.x; bv[g * 4 + 1] = q.y; bv[g * 4 + 2] = q.z; bv[g * 4 + 3] = q.w;
            }
#pragma unroll
            for (int i = 0; i < TC; ++i)
#pragma unroll
                for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        if (ch + 1 < ch_end) store_tile(s ^ 1);
        __syncthreads();
    }

    const int kk = p.ksize * p.ksize;
#pragma unroll
    for (int i = 0; i < TC; ++i) {
        const int c = c0 + (i / 4) * GSC + ty * 4 + (i % 4);
        if (c >= p.Cin) continue;
#pragma unroll
        for (int j = 0; j < TN; ++j) {
            const int n = n0 + (j / 4) * GSN + tx * 4 + (j % 4);
            if (n >= p.Cout) continue;
            atomicAdd(p.dw + ((long long)n * p.Cin + c) * kk + tap, acc[i][j]);
        }
    }
}

// out[n] += sum_m x[m][n]   (rows of image b start at x + b*bstride; HW rows per image)
__global__ void __launch_bounds__(kNT) colsum_kernel(const float* __restrict__ x, float* __restrict__ out,
                                                     const long long M, const int N, const int rows_per_block,
                                                     const long long HW, const long long bstride) {
    __shared__ float4 red[kNT];
    const int cvecs = N / 4;
    const RowPack rp = rowpack(cvecs, blockIdx.y);
    float4 s = f4zero();
    if (rp.active) {
        const long long r_begin = (long long)blockIdx.x * rows_per_block;
        const long long r_end = min(M, r_begin + rows_per_block);
        for (long long r = r_begin + rp.tr; r < r_end; r += rp.rows) {
            const long long b = r / HW;
            s = f4add(s, ldg4(x + b * bstride + (r - b * HW) * N + rp.cv * 4));
        }
    }
    red[threadIdx.x] = s;
    __syncthreads();
    if (rp.tr == 0 && rp.cv < cvecs && rp.tc < rp.cvb) {
        float4 acc = f4zero();
        for (int r = 0; r < rp.rows; ++r) acc = f4add(acc, red[r * rp.cvb + rp.tc]);
        float* o = out + rp.cv * 4;
        atomicAdd(o + 0, acc.x); atomicAdd(o + 1, acc.y); atomicAdd(o + 2, acc.z); atomicAdd(o + 3, acc.w);
    }
}

__global__ void pack_conv_weight_kernel(const float* __restrict__ w, float* __restrict__ wf, float* __restrict__ wd,
                                        int Cout, int Cin, int ks) {
    const int kk = ks * ks;
    const long long total = (long long)Cout * Cin * kk;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        // i enumerates the forward pack [tap][c][n] so that writes are coalesced
        const int n = (int)(i % Cout);
        const long long r = i / Cout;
        const int c = (int)(r % Cin);
        const int tap = (int)(r / Cin);
        const float v = __ldg(w + ((long long)n * Cin + c) * kk + tap);
        wf[i] = v;
        if (wd) wd[((long long)(kk - 1 - tap) * Cout + n) * Cin + c] = v;
    }
}

int conv_simt_launch(const effdet_conv_args* a, cudaStream_t st) {
    const int M = a->B * a->H * a->W, HW = a->H * a->W;
    // pick the N tile that wastes the fewest padded columns (ties -> wider tile)
    int best = 128;
    long long best_pad = (long long)cdiv(a->Cout, 128) * 128;
    for (int bn : {64, 32}) {
        long long padn = (long long)cdiv(a->Cout, bn) * bn;
        if (padn < best_pad) { best_pad = padn; best = bn; }
    }
    dim3 grid(cdiv(M, kBM), cdiv(a->Cout, best));
    if (best == 128) conv_igemm_kernel<128, 8><<<grid, kNT, 0, st>>>(*a, M, HW);
    else if (best == 64) conv_igemm_kernel<64, 4><<<grid, kNT, 0, st>>>(*a, M, HW);
    else conv_igemm_kernel<32, 4><<<grid, kNT, 0, st>>>(*a, M, HW);
    return launch_status("conv_igemm_kernel");
}

int colsum_launch(const float* x, float* out, long long M, int N, long long HW, long long bstride, cudaStream_t st) {
    EFFDET_REQUIRE(x && out && M > 0 && N > 0 && N % 4 == 0, "colsum: bad arguments");
    EFFDET_REQUIRE(aligned16(x), "colsum: x must be 16-byte aligned");
    const int cvecs = N / 4;
    const int rows = rowpack_rows(cvecs);
    // ~4 waves of blocks, at least 8 row-iterations per block
    long long rpb = (M + num_sms() * 4 - 1) / (num_sms() * 4);
    if (rpb < (long long)rows * 8) rpb = (long long)rows * 8;
    dim3 grid(cdiv(M, rpb), rowpack_chunks(cvecs));
    colsum_kernel<<<grid, kNT, 0, st>>>(x, out, M, N, (int)rpb, HW, bstride);
    return launch_status("colsum_kernel");
}

int wgrad_simt_launch(const effdet_wgrad_args* a, cudaStream_t st) {
    const int M = a->B * a->H * a->W, HW = a->H * a->W;
    const int taps = a->ksize * a->ksize;
    int BC, BN;
    if (a->Cin <= 32) { BC = 32; BN = 128; }
    else if (a->Cout <= 48) { BC = 128; BN = 32; }
    else if (a->Cin >= 128 && a->Cout >= 128) { BC = 128; BN = 128; }
    else { BC = 64; BN = 64; }
    const int ctiles = cdiv(a->Cin, BC), ntiles = cdiv(a->Cout, BN);
    const int nchunks = cdiv(M, kBK);
    // enough pixel slices for ~3 waves of CTAs, each slice at least 16 chunks long
    int splits = cdiv(num_sms() * 3, ctiles * ntiles * taps);
    if (splits < 1) splits = 1;
    if (splits > cdiv(nchunks, 16)) splits = cdiv(nchunks, 16);
    int cps = cdiv(nchunks, splits);
    splits = cdiv(nchunks, cps);
    dim3 grid(ctiles * ntiles, taps, splits);
    if (BC == 32) conv_wgrad_kernel<32, 128, 4, 4><<<grid, kNT, 0, st>>>(*a, M, HW, cps, ctiles);
    else if (BN == 32) conv_wgrad_kernel<128, 32, 4, 4><<<grid, kNT, 0, st>>>(*a, M, HW, cps, ctiles);
    else if (BC == 128) conv_wgrad_kernel<128, 128, 8, 8><<<grid, kNT, 0, st>>>(*a, M, HW, cps, ctiles);
    else conv_wgrad_kernel<64, 64, 4, 4><<<grid, kNT, 0, st>>>(*a, M, HW, cps, ctiles);
    return launch_status("conv_wgrad_kernel");
}

}  // namespace effdet

using namespace effdet;

extern "C" int effdet_pack_conv_weight(const float* w_oihw, float* w_fwd, float* w_dgrad, int Cout, int Cin, int ksize,
                                       int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(w_oihw && w_fwd && Cout > 0 && Cin > 0 && (ksize == 1 || ksize == 3), "pack_conv_weight: bad arguments");
    EFFDET_DEVICE(device);
    const long long total = (long long)Cout * Cin * ksize * ksize;
    int blocks = cdiv(total, 256);
    if (blocks > num_sms() * 8) blocks = num_sms() * 8;
    pack_conv_weight_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(w_oihw, w_fwd, w_dgrad, Cout, Cin, ksize);
    return launch_status("pack_conv_weight_kernel");
}
