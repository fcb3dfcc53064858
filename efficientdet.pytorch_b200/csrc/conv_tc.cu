// Tensor-core (wgmma) implicit-GEMM convolution for the dense 3x3 layers of head and neck:
// forward, data gradient (same kernel on the rotated/transposed weight pack) and weight
// gradient.  95 % of the model's FLOPs live here (SURVEY.md section 0 fact 3).
//   conv_tc_kernel          forward / data gradient, fp32 activations gathered and split in the kernel,
//                           every pyramid level that shares the weights in one launch
//   wgrad_tc2_multi_kernel  weight gradient fed by TMA from bf16 hi/lo planes (to_planes_kernel splits the
//                           operands that are not planes yet), every level in one launch
//   wgrad_tc_kernel         weight gradient that gathers and splits fp32 operands itself: maps with no pixel box
//
// Precision: operands stay fp32 in HBM (module API parity) and are split on the fly into
// bf16 hi + bf16 lo (x = hi + lo to 16 mantissa bits); every product is evaluated as
//   hi*hi + lo*hi + hi*lo      (three bf16 wgmma, fp32 accumulation in registers)
// which is ~2^-16 per product -- far inside north_star's 1e-3 where single-pass TF32 is not
// (SURVEY.md H1) -- at 2/3 the cost of 3xTF32.  Every kernel also has a single-pass instance (template
// argument NP = 1, the tc_single flag of the C ABI): hi*hi only, the lo halves are neither formed nor loaded.
//
// Structure per CTA (288 threads, one 128 x BN output tile):
//   warps 0-7  two warpgroups: gather the im2col A tile (128 pixels x 64 channels of one tap)
//              with 128-bit loads, split to bf16 hi/lo, store into the canonical K-major
//              SWIZZLE_128B layout; then each warpgroup issues the wgmma of its 64-row half
//              (accumulator in registers, BN/2 floats per thread) while the loads of the next
//              stage are in flight; finally the same warps run the epilogue (bias / ReLU /
//              sigmoid / ReLU-mask / residual, 128-bit stores straight into the caller's layout)
//   warp 8     TMA: weight tiles (pre-split bf16 planes) -> smem, mbarrier complete_tx
// Weight gradient: both operands are NHWC rows (pixels are the GEMM-K dimension, so they are
// MN-major operands), split-K over pixel ranges with fp32 vector reductions into a tap-major accumulator
// [taps][Cout][Cin] (for a 3x3 conv a workspace that wgrad_fold_kernel adds into the OIHW gradient, for a 1x1 conv the
// gradient itself).
#include "tc_ptx.cuh"

namespace effdet {

constexpr int kTcThreads = 288;        // two gather / MMA / epilogue warpgroups + one TMA warp
constexpr int kTcProducers = 256;      // the two warpgroups (all of the gathering weight-gradient kernel)
constexpr int kTileM = 128;     // pixels per CTA (fwd/dgrad) or output channels per CTA (wgrad)
constexpr int kTileK = 64;      // bf16 elements per 128-byte swizzled row
// Most pixel chunks (<= 64 pixels each) one weight-gradient CTA accumulates (kWgMaxPixelsPerSplit, tc_ptx.cuh).
constexpr int kWgMaxChunksPerSplit = kWgMaxPixelsPerSplit / kTileK;

// ---------------------------------------------------------------------------------------------
// forward / data-gradient kernel
// ---------------------------------------------------------------------------------------------
template <int BN, int STAGES>
struct FwdSmem {
    static constexpr int kA = kTileM * 128;   // bytes of one bf16 plane of the A tile
    static constexpr int kB = BN * 128;       // bytes of one bf16 plane of the B tile
    static constexpr int kStage = 2 * kA + 2 * kB;
    static constexpr int kChan = BN * 4;      // bias of this CTA's output channels
    static constexpr int kBytes = STAGES * kStage + 1024 /*alignment slack*/ + 256 /*barriers*/ + kChan;
};

// Several pyramid levels that share one weight tensor (RetinaHead runs the same convs on P3..P7,
// models/retinahead.py:131-132) in ONE launch: the M tiles of all levels are concatenated so the small
// levels (a handful of CTAs each) ride along with the large ones instead of paying their own latency-bound launch.
struct ConvMultiArgs {
    ConvLevel lv[kMaxLevels];
    int tile_begin[kMaxLevels + 1];
    int nlevels;
};

// NP = bf16 products per multiply-add: 3 (split precision) or 1 (hi only)
template <int BN, int STAGES, int NP>
__global__ void __launch_bounds__(kTcThreads, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap wmap, const __grid_constant__ ConvMultiArgs ma, const int kblocks) {
    using S = FwdSmem<BN, STAGES>;
    const int tile = blockIdx.x;
    int l = 0;
    while (l + 1 < ma.nlevels && tile >= ma.tile_begin[l + 1]) ++l;
    const effdet_conv_args& p = ma.lv[l].get();
    const int M = p.B * p.H * p.W, HW = p.H * p.W;
    const int m0 = (tile - ma.tile_begin[l]) * kTileM, n0 = blockIdx.y * BN;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // 1024-byte aligned AND still a shared-space pointer (LDS/STS, not generic LD/ST)
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * S::kStage);
    uint64_t* empty_bar = full_bar + STAGES;
    float* chan = reinterpret_cast<float*>(smem + STAGES * S::kStage + 256);   // [BN]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int taps = p.ksize * p.ksize, pad = p.ksize / 2;
    const int KT = taps * kblocks;
    for (int i = threadIdx.x; i < BN; i += kTcThreads) {
        const int n = n0 + i;
        chan[i] = (n < p.Cout && p.bias) ? __ldg(p.bias + n) : 0.f;
    }

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 1);
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp < 8) {
        // ---------------- producers: im2col gather + bf16 split, then wgmma on this warpgroup's 64 rows -----------------
        constexpr int NB = BN / 64;
        const int t = threadIdx.x;
        const int g = warp >> 2;             // warpgroup: rows 64g .. 64g+63 of the tile
        const int j = t & 7;                 // 16-byte chunk (8 channels) within the 64-channel row
        long long base[4];
        int oyx[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int r = i * 32 + (t >> 3);
            const int m = m0 + r;
            if (m < M) {
                const int b = m / HW;
                const int pix = m - b * HW;
                const int oy = pix / p.W;
                oyx[i] = (oy << 16) | (pix - oy * p.W);
                base[i] = (long long)b * p.x_bstride;
            } else {
                oyx[i] = -1;
                base[i] = 0;
            }
        }
        // gather one stage worth of fp32 operands into registers (4 rows x 32 bytes per thread)
        auto load_stage = [&](int kt, float4 (&v)[8]) {
            const int tap = kt / kblocks;
            const int c = (kt - tap * kblocks) * kTileK + j * 8;
            const int ky = tap / p.ksize - pad, kx = tap % p.ksize - pad;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                v[2 * i] = f4zero();
                v[2 * i + 1] = f4zero();
                if (oyx[i] >= 0 && c < p.Cin) {
                    const int iy = (oyx[i] >> 16) + ky, ix = (oyx[i] & 0xffff) + kx;
                    if (iy >= 0 && iy < p.H && ix >= 0 && ix < p.W) {
                        const float* src = p.x + base[i] + ((long long)iy * p.W + ix) * p.Cin + c;
                        v[2 * i] = ldg4(src);
                        if (c + 4 < p.Cin) v[2 * i + 1] = ldg4(src + 4);
                    }
                }
            }
        };
        float d[NB][32];
        for (int kt = 0; kt < KT; ++kt) {
            const int s = kt % STAGES;
            const uint32_t ph = (kt / STAGES) & 1;
            float4 v[8];
            load_stage(kt, v);                   // in flight while the previous stage's wgmma run
            wgmma_wait<STAGES - 1>();            // this warpgroup no longer reads stage s ...
            named_bar_sync(1, kTcProducers);     // ... nor does the other one
            if (t == 0 && kt >= STAGES) mbar_arrive(&empty_bar[s]);
            uint8_t* a_hi = smem + s * S::kStage;
            uint8_t* a_lo = a_hi + S::kA;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int r = i * 32 + (t >> 3);
                const int off = r * 128 + ((j ^ (r & 7)) << 4);
                if constexpr (NP == 3) {
                    uint4 hi, lo;
                    split8(v[2 * i], v[2 * i + 1], hi, lo);
                    *reinterpret_cast<uint4*>(a_hi + off) = hi;
                    *reinterpret_cast<uint4*>(a_lo + off) = lo;
                } else {
                    *reinterpret_cast<uint4*>(a_hi + off) = hi8(v[2 * i], v[2 * i + 1]);
                }
            }
            fence_proxy_async();
            named_bar_sync(1, kTcProducers);     // the A tile is complete
            mbar_wait(&full_bar[s], ph);         // the weight tile landed
            const uint32_t sa = smem_u32(a_hi) + g * 64 * 128;
            const uint32_t sb = smem_u32(a_hi) + 2 * S::kA;
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < kTileK / 16; ++k)
                wg_mma<NB, 0, NP>(d, sa + k * 32, sa + S::kA + k * 32, sb + k * 32, sb + S::kB + k * 32, 16, 1024, (kt | k) != 0);
            wgmma_commit();
        }
        wgmma_wait<0>();
        named_bar_sync(1, kTcProducers);         // every stage is drained: stage 0 becomes the epilogue's staging buffer
        // ---------------- epilogue ------------------------------------------------------------------------------------
        float* rows_buf = reinterpret_cast<float*>(smem);
        const int quarter = 2 * g + (warp & 1), half = (warp >> 1) & 1;   // 32-row group, 32-column chunk parity
        const int m = m0 + quarter * 32 + lane;
        const bool row_ok = m < M;
        int b = 0;
        long long pix = 0;
        if (row_ok) {
            b = m / HW;
            pix = m - b * HW;
        }
        const int ncols = min(BN, p.Cout - n0);
        const int nchunks = (ncols + 31) >> 5;
        const long long ybase = (long long)b * p.y_bstride + pix * p.Cout;
        const long long rbase = (long long)b * p.r_bstride + pix * p.Cout;
        const long long mbase = (long long)b * p.m_bstride + pix * p.Cout;
#pragma unroll
        for (int jb = 0; jb < NB; ++jb) {
            float acc[32];
            wg_rows<2>(d[jb], rows_buf, g, acc);
            const int cc = 2 * jb + half;
            if (cc >= nchunks || !row_ok) continue;
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const int nl = cc * 32 + q * 4;
                const int n = n0 + nl;
                if (n >= p.Cout) break;
                float4 v = make_float4(acc[q * 4], acc[q * 4 + 1], acc[q * 4 + 2], acc[q * 4 + 3]);
                v = f4add(v, *reinterpret_cast<const float4*>(chan + nl));
                if (p.act == EFFDET_ACT_RELU) {
                    v = make_float4(fmaxf(v.x, 0.f), fmaxf(v.y, 0.f), fmaxf(v.z, 0.f), fmaxf(v.w, 0.f));
                } else if (p.act == EFFDET_ACT_SIGMOID) {
                    v = make_float4(sigmoidf_(v.x), sigmoidf_(v.y), sigmoidf_(v.z), sigmoidf_(v.w));
                } else if (p.act == EFFDET_ACT_SWISH) {
                    v = make_float4(swishf_(v.x), swishf_(v.y), swishf_(v.z), swishf_(v.w));
                }
                if (p.residual) v = f4add(v, ldg4(p.residual + rbase + n));
                if (p.mask_src) {
                    const float4 mv = ldg4(p.mask_src + mbase + n);
                    v = make_float4(mv.x > 0.f ? v.x : 0.f, mv.y > 0.f ? v.y : 0.f, mv.z > 0.f ? v.z : 0.f, mv.w > 0.f ? v.w : 0.f);
                }
                st4(p.y + ybase + n, v);
            }
        }
    } else if (warp == 8) {
        // ---------------- TMA: weight tiles (hi plane, lo plane) ---------------------------------------
        if (lane == 0) {
            for (int kt = 0; kt < KT; ++kt) {
                const int s = kt % STAGES;
                const uint32_t ph = (kt / STAGES) & 1;
                mbar_wait(&empty_bar[s], ph ^ 1);
                uint8_t* b_hi = smem + s * S::kStage + 2 * S::kA;
                mbar_arrive_expect_tx(&full_bar[s], (NP == 3 ? 2 : 1) * S::kB);
                tma_load_3d(b_hi, &wmap, &full_bar[s], kt * kTileK, n0, 0);
                if (NP == 3) tma_load_3d(b_hi + S::kB, &wmap, &full_bar[s], kt * kTileK, n0, 1);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// weight-gradient kernel:  D[n, c | tap] += sum_pixels dy[pixel, n] * x[pixel + tap, c]
//   GEMM-M = 128 output channels, GEMM-N = BC input channels, GEMM-K = pixels (64 per stage);
//   both operands are NHWC rows (channels contiguous) = MN-major SWIZZLE_128B operands:
//   one 64-channel group of a stage = 64 pixel-rows x 128 B, groups LBO = 8192 B apart,
//   8-pixel groups SBO = 1024 B apart.
// ---------------------------------------------------------------------------------------------
template <int BC, int STAGES>
struct WgSmem {
    static constexpr int kA = kTileK * 128 * (kTileM / 64);   // one plane of the dy tile: 2 channel groups
    static constexpr int kB = kTileK * 128 * (BC / 64);       // one plane of the x tile
    static constexpr int kStage = 2 * kA + 2 * kB;
    static constexpr int kXch = STAGES * kStage + 256;        // the epilogue's lane exchange: 2 x 32 float2 per warp
    static constexpr int kBytes = kXch + 8 * 2 * 32 * 8 + 1024;
};

// gather `ngroups` channel groups (64 channels each) of 64 pixel rows into swizzled bf16 planes (NP = 1: hi plane only)
template <int NGROUPS, int NP>
__device__ __forceinline__ void wg_produce(const float* __restrict__ src, const long long bstride, const int C, const int c0,
                                           const int H, const int W, const int HW, const int M, const int mbase, const int dy,
                                           const int dx, uint8_t* hi_plane, uint8_t* lo_plane, const int t) {
    // item = (pixel row r, group g, chunk j): 64 * NGROUPS * 8 items over 128 threads
    constexpr int ITEMS = 64 * NGROUPS * 8 / kTcProducers;
    const int j = t & 7;
#pragma unroll 4
    for (int it = 0; it < ITEMS; ++it) {
        const int idx = it * kTcProducers + t;
        const int rg = idx >> 3;                   // r * NGROUPS + g  (g fastest so a warp reads contiguous channels)
        const int g = rg % NGROUPS, r = rg / NGROUPS;
        const int m = mbase + r;
        const int c = c0 + g * 64 + j * 8;
        float4 v0 = f4zero(), v1 = f4zero();
        if (m < M && c < C) {
            const int b = m / HW;
            const int pix = m - b * HW;
            const int oy = pix / W;
            const int iy = oy + dy, ix = pix - oy * W + dx;
            if (iy >= 0 && iy < H && ix >= 0 && ix < W) {
                const float* q = src + (long long)b * bstride + ((long long)iy * W + ix) * C + c;
                v0 = ldg4(q);
                if (c + 4 < C) v1 = ldg4(q + 4);
            }
        }
        if constexpr (NP == 3) {
            uint4 hi, lo;
            split8(v0, v1, hi, lo);
            const int off = g * (kTileK * 128) + r * 128 + ((j ^ (r & 7)) << 4);
            *reinterpret_cast<uint4*>(hi_plane + off) = hi;
            *reinterpret_cast<uint4*>(lo_plane + off) = lo;
        } else {
            const int off = g * (kTileK * 128) + r * 128 + ((j ^ (r & 7)) << 4);
            *reinterpret_cast<uint4*>(hi_plane + off) = hi8(v0, v1);
        }
    }
}

__device__ __forceinline__ void red_add_v4(float* p, float a, float b, float c, float d) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// Adds a warpgroup's accumulator (64 output channels from n0 x NB*64 input channels from c0) into the tap-major fp32
// accumulator acc[taps][Cout][Cin], where input channels are contiguous.  In the wgmma fragment a lane holds columns 2q,
// 2q+1 of rows r and r+8 in each 8-column block; lanes 2k and 2k+1 swap one pair so that the even lane holds 4
// consecutive columns of row r and the odd lane 4 of row r+8, and each issues one 16-byte vector reduction.
// Cin % 4 == 0, so a 4-column group lies wholly inside or wholly outside Cin.
// The swap goes through the warp's 64 float2 of shared memory (xch, two slots per lane used in turn, so one __syncwarp
// per block orders both the reuse and the read): a warp shuffle in the consumer branch of wgrad_tc2_multi_kernel makes
// ptxas serialize that kernel's wgmma (C7520).
template <int NB>
__device__ __forceinline__ void wg_red_dw(const float (&d)[NB][32], float* acc, const int n0, const int c0, const int Cout,
                                          const int Cin, const int tap, float2* xch) {
    const int w = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
    const bool odd = lane & 1;
    const int n = n0 + 16 * w + (lane >> 2) + 8 * odd;
    float* row = acc + ((long long)tap * Cout + n) * Cin + c0 + 2 * (lane & 2);
#pragma unroll
    for (int jb = 0; jb < NB; ++jb)
#pragma unroll
        for (int b = 0; b < 8; ++b) {
            const float* v = &d[jb][4 * b];      // (r, 2q), (r, 2q+1), (r+8, 2q), (r+8, 2q+1)
            float2* slot = xch + 32 * (b & 1);
            slot[lane] = odd ? make_float2(v[0], v[1]) : make_float2(v[2], v[3]);
            __syncwarp();
            const float2 t = slot[lane ^ 1];
            const float s0 = t.x, s1 = t.y;
            const float x0 = odd ? s0 : v[0], x1 = odd ? s1 : v[1], x2 = odd ? v[2] : s0, x3 = odd ? v[3] : s1;
            const int c = c0 + jb * 64 + 8 * b + 2 * (lane & 2);
            if (n < Cout && c < Cin) red_add_v4(row + jb * 64 + 8 * b, x0, x1, x2, x3);
        }
}

template <int BC, int STAGES, int NP>
__global__ void __launch_bounds__(kTcProducers, 1)
wgrad_tc_kernel(const __grid_constant__ WgradPrefix pa, float* acc, const int M, const int HW, const int chunks_per_split,
                const int ctiles) {
    using S = WgSmem<BC, STAGES>;
    const effdet_wgrad_args& p = pa.get();
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // 1024-byte aligned AND still a shared-space pointer (LDS/STS, not generic LD/ST)

    const int warp = threadIdx.x >> 5;
    const int ct = blockIdx.x % ctiles, nt = blockIdx.x / ctiles;
    const int c0 = ct * BC, n0 = nt * kTileM;
    const int tap = blockIdx.y;
    const int pad = p.ksize / 2;
    const int dy = tap / p.ksize - pad, dx = tap % p.ksize - pad;
    const int nchunks = (M + kTileK - 1) / kTileK;
    const int ch_begin = blockIdx.z * chunks_per_split;
    const int ch_end = min(nchunks, ch_begin + chunks_per_split);
    const int KT = ch_end - ch_begin;      // >= 1 by construction of the grid
    constexpr int NB = BC / 64;
    constexpr uint32_t GROUP = kTileK * 128;
    const int t = threadIdx.x, g = warp >> 2;      // warpgroup g: output channels n0 + 64g .. + 63
    float d[NB][32];
    for (int kt = 0; kt < KT; ++kt) {
        const int s = kt % STAGES;
        wgmma_wait<STAGES - 1>();
        named_bar_sync(1, kTcProducers);           // neither warpgroup still reads stage s
        uint8_t* a_hi = smem + s * S::kStage;
        uint8_t* b_hi = a_hi + 2 * S::kA;
        const int mbase = (ch_begin + kt) * kTileK;
        wg_produce<kTileM / 64, NP>(p.dy, p.dy_bstride, p.Cout, n0, p.H, p.W, HW, M, mbase, 0, 0, a_hi, a_hi + S::kA, t);
        wg_produce<BC / 64, NP>(p.x, p.x_bstride, p.Cin, c0, p.H, p.W, HW, M, mbase, dy, dx, b_hi, b_hi + S::kB, t);
        fence_proxy_async();
        named_bar_sync(1, kTcProducers);
        const uint32_t sa = smem_u32(a_hi) + g * GROUP, sb = smem_u32(b_hi);
        wg_mma_mn_steps<kTileK / 16, NP>(d, sa, sa + S::kA, sb, sb + S::kB, GROUP, kt != 0);
        wgmma_commit();
    }
    wgmma_wait<0>();
    // epilogue: row = output channel n, columns = input channels c -> vector reductions into acc[tap][n][c]
    wg_red_dw<NB>(d, acc, n0 + 64 * g, c0, p.Cout, p.Cin, tap, reinterpret_cast<float2*>(smem + S::kXch) + 64 * warp);
}

// ---------------------------------------------------------------------------------------------
// weight-gradient kernel, TMA-fed: the operands are bf16 hi/lo planes [2][B][H][W][Cpad]
// (split by to_planes_kernel, or written in that form by their producer), so the gather warps
// disappear: one thread issues 5-D tensor-map loads (channel group, x, y, image, plane) whose
// out-of-bounds zero fill IS the convolution's zero padding (the tap shift is just a coordinate
// offset); two consumer warpgroups (64 output channels each) issue the wgmma and add their
// accumulators to the tap-major accumulator with vector reductions.  A stage covers a box of
// kstage = Wb*Hb*Bb pixels (<= 64, multiple of 16).
// The pixel chunks of several pyramid levels (same weights, e.g. the five RetinaHead levels) form
// one long GEMM-K dimension, so one launch covers them all; each chunk looks up its level's tensor
// maps and pixel-box geometry.
// ---------------------------------------------------------------------------------------------
struct WgMaps {
    CUtensorMap dy[kWgMaxLevels];
    CUtensorMap x[kWgMaxLevels];
};
struct WgMultiArgs {
    WgGeom g[kWgMaxLevels];
    int chunk_begin[kWgMaxLevels + 1];
    int nlevels;
    float* acc;          // [taps][Cout][Cin]
    int Cin, Cout, ksize;
};

template <int BC, int STAGES, int NP>
__global__ void __launch_bounds__(kTcThreads, 1)
wgrad_tc2_multi_kernel(const __grid_constant__ WgMaps maps, const __grid_constant__ WgMultiArgs a, const int chunks_per_split,
                       const int ctiles) {
    using S = WgSmem<BC, STAGES>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // 1024-byte aligned AND still a shared-space pointer (LDS/STS, not generic LD/ST)
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * S::kStage);
    uint64_t* empty_bar = full_bar + STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ct = blockIdx.x % ctiles, nt = blockIdx.x / ctiles;
    const int c0 = ct * BC, n0 = nt * kTileM;
    const int tap = blockIdx.y;
    const int pad = a.ksize / 2;
    const int dy = tap / a.ksize - pad, dx = tap % a.ksize - pad;
    const int nchunks = a.chunk_begin[a.nlevels];
    const int ch_begin = blockIdx.z * chunks_per_split;
    const int ch_end = min(nchunks, ch_begin + chunks_per_split);
    const int KT = ch_end - ch_begin;

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 8);     // one arrival per consumer warp
        }
        fence_barrier_init();
    }
    __syncthreads();
    constexpr int GROUP = kTileK * 128;

    if (warp == 8) {
        if (lane == 0) {
            int l = 0;
            for (int kt = 0; kt < KT; ++kt) {
                const int s = kt % STAGES;
                const uint32_t ph = (kt / STAGES) & 1;
                const int chg = ch_begin + kt;
                while (l + 1 < a.nlevels && chg >= a.chunk_begin[l + 1]) ++l;
                const WgGeom& g = a.g[l];
                int ch = chg - a.chunk_begin[l];
                const int bx = ch % g.nbx;
                ch /= g.nbx;
                const int by = ch % g.nby;
                const int bb = ch / g.nby;
                const int x0 = bx * g.Wb, y0 = by * g.Hb, b0 = bb * g.Bb;
                const uint32_t bytes = (uint32_t)((NP == 3 ? 2 : 1) * (kTileM / 64 + BC / 64) * g.kstage * 128);
                mbar_wait(&empty_bar[s], ph ^ 1);
                mbar_arrive_expect_tx(&full_bar[s], bytes);
                uint8_t* a_hi = smem + s * S::kStage;
                uint8_t* b_hi = a_hi + 2 * S::kA;
#pragma unroll
                for (int pl = 0; pl < (NP == 3 ? 2 : 1); ++pl) {
#pragma unroll
                    for (int q = 0; q < kTileM / 64; ++q)
                        tma_load_5d(a_hi + pl * S::kA + q * GROUP, &maps.dy[l], &full_bar[s], n0 + q * 64, x0, y0, b0, pl);
#pragma unroll
                    for (int q = 0; q < BC / 64; ++q)
                        tma_load_5d(b_hi + pl * S::kB + q * GROUP, &maps.x[l], &full_bar[s], c0 + q * 64, x0 + dx, y0 + dy, b0, pl);
                }
            }
        }
    } else {
        constexpr int NB = BC / 64;
        const int wg = warp >> 2;
        float d[NB][32];
        // level by level: the pixel box, and so the number of K16 steps per stage, is fixed within a level
        for (int kt = 0, l = 0; kt < KT; ++l) {
            const int end = min(KT, a.chunk_begin[l + 1] - ch_begin);
            with_count<1, 2, 3, 4>(a.g[l].kstage / 16, [&](auto ksteps) {
                for (; kt < end; ++kt) {
                    const int s = kt % STAGES;
                    const uint32_t ph = (kt / STAGES) & 1;
                    mbar_wait(&full_bar[s], ph);
                    const uint32_t sa = smem_u32(smem + s * S::kStage) + wg * GROUP;
                    const uint32_t sb = smem_u32(smem + s * S::kStage) + 2 * S::kA;
                    wg_mma_mn_steps<ksteps, NP>(d, sa, sa + S::kA, sb, sb + S::kB, GROUP, kt != 0);
                    wgmma_commit();
                    wgmma_wait<1>();
                    if (kt > 0 && lane == 0) mbar_arrive(&empty_bar[(kt - 1) % STAGES]);
                }
            });
        }
        wgmma_wait<0>();
        wg_red_dw<NB>(d, a.acc, n0 + 64 * wg, c0, a.Cout, a.Cin, tap, reinterpret_cast<float2*>(smem + S::kXch) + 64 * warp);
    }
}

// Adds the tap-major accumulator of a 3x3 weight gradient into the OIHW gradient: dw[n][c][tap] += ws[tap][n][c].
// A CTA takes kFoldPairs consecutive (n, c) pairs, reads their 9 tap rows coalesced, transposes them through shared
// memory (stride 9, odd: no bank conflicts) and adds them to the 9 * kFoldPairs consecutive floats of dw they map to.
constexpr int kFoldPairs = 256;
__global__ void __launch_bounds__(kFoldPairs)
wgrad_fold_kernel(const float* __restrict__ ws, float* __restrict__ dw, const long long nc) {
    __shared__ float t[9 * kFoldPairs];
    const long long j0 = (long long)blockIdx.x * kFoldPairs;
    const int np = (int)min((long long)kFoldPairs, nc - j0);
    if (threadIdx.x < np)
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) t[threadIdx.x * 9 + tap] = __ldg(ws + tap * nc + j0 + threadIdx.x);
    __syncthreads();
    for (int i = threadIdx.x; i < 9 * np; i += kFoldPairs) dw[j0 * 9 + i] += t[i];
}

// ---------------------------------------------------------------------------------------------
// weight pre-split: OIHW fp32 -> bf16 planes [2][rows][taps][Kpad] (K-major, zero padded)
//   forward pack : rows = Cout, k = Cin,  W[n][c][tap]
//   dgrad pack   : rows = Cin,  k = Cout, W[n][c][taps-1-tap]   (180-degree rotation, transpose)
// ---------------------------------------------------------------------------------------------
__global__ void pack_weight_tc_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ out, int Cout, int Cin, int taps,
                                      int kpad, int dgrad) {
    const int rows = dgrad ? Cin : Cout;
    const int kdim = dgrad ? Cout : Cin;
    const long long plane = (long long)rows * taps * kpad;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < plane; i += (long long)gridDim.x * blockDim.x) {
        const int k = (int)(i % kpad);
        const long long r2 = i / kpad;
        const int tap = (int)(r2 % taps);
        const int row = (int)(r2 / taps);
        float v = 0.f;
        if (k < kdim) {
            const int n = dgrad ? k : row, c = dgrad ? row : k;
            const int st = dgrad ? (taps - 1 - tap) : tap;
            v = __ldg(w + ((long long)n * Cin + c) * taps + st);
        }
        const __nv_bfloat16 h = __float2bfloat16_rn(v);
        out[i] = h;
        out[plane + i] = __float2bfloat16_rn(v - __bfloat162float(h));
    }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(ptr);
    }
    return fn;
}

int conv_tc_kpad(int k) { return (k + kTileK - 1) / kTileK * kTileK; }

// 3-D tensor map over K-major bf16 hi/lo planes [2][rows][k]: boxes of 64 k (one 128-byte swizzled row) x box_rows rows
int kmajor_planes_map(EncodeTiledFn enc, CUtensorMap* map, const void* base, int rows, int k, int box_rows) {
    const cuuint64_t gdim[3] = {(cuuint64_t)k, (cuuint64_t)rows, 2};
    const cuuint64_t gstr[2] = {(cuuint64_t)k * 2, (cuuint64_t)rows * k * 2};
    const cuuint32_t box[3] = {(cuuint32_t)kTileK, (cuuint32_t)box_rows, 1};
    const cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), gdim, gstr, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(EFFDET_ERR_LAUNCH, "tensor map of bf16 planes [2][%d][%d] failed (%d)", rows, k, (int)r);
    return EFFDET_OK;
}

// levels share weights, bias, channels and activation (checked by the caller)
int conv_tc_launch(const effdet_conv_args* levels, int nlevels, cudaStream_t st) {
    EncodeTiledFn enc = encode_fn();
    if (!enc) return fail(EFFDET_ERR_UNSUPPORTED, "conv2d(tc): cuTensorMapEncodeTiled unavailable");
    const effdet_conv_args* a = &levels[0];
    const int taps = a->ksize * a->ksize;
    const int kpad = conv_tc_kpad(a->Cin);
    const int kblocks = kpad / kTileK;
    // 128 x 128 tiles at most: the accumulator lives in the two warpgroups' registers (64 per thread)
    const int BN = a->Cout <= 64 ? 64 : 128;
    CUtensorMap map;
    int s = kmajor_planes_map(enc, &map, a->w_tc, a->Cout, taps * kpad, BN);
    if (s) return s;
    ConvMultiArgs ma;
    memset(&ma, 0, sizeof(ma));
    ma.nlevels = nlevels;
    int tiles = 0;
    for (int l = 0; l < nlevels; ++l) {
        ma.lv[l].set(levels[l]);
        ma.tile_begin[l] = tiles;
        tiles += cdiv((long long)levels[l].B * levels[l].H * levels[l].W, kTileM);
    }
    for (int l = nlevels; l <= kMaxLevels; ++l) ma.tile_begin[l] = tiles;
    dim3 grid(tiles, cdiv(a->Cout, BN));
    if (a->tc_single) {
        if (BN == 64)
            return launch_smem("conv_tc_kernel", conv_tc_kernel<64, 4, 1>, grid, kTcThreads, FwdSmem<64, 4>::kBytes, st, map, ma, kblocks);
        return launch_smem("conv_tc_kernel", conv_tc_kernel<128, 3, 1>, grid, kTcThreads, FwdSmem<128, 3>::kBytes, st, map, ma, kblocks);
    }
    if (BN == 64) return launch_smem("conv_tc_kernel", conv_tc_kernel<64, 4, 3>, grid, kTcThreads, FwdSmem<64, 4>::kBytes, st, map, ma, kblocks);
    return launch_smem("conv_tc_kernel", conv_tc_kernel<128, 3, 3>, grid, kTcThreads, FwdSmem<128, 3>::kBytes, st, map, ma, kblocks);
}

bool wg_geometry(int B, int H, int W, WgGeom* g) {
    const int Wb = W <= 64 ? W : 64;
    if (W % Wb) return false;
    int Hb = 1;
    for (int h = 1; h <= H && Wb * h <= 64; ++h)
        if (H % h == 0) Hb = h;
    int Bb = 64 / (Wb * Hb);
    if (Bb < 1) Bb = 1;
    if (Bb > B) Bb = B;
    const int ks = Wb * Hb * Bb;
    if (ks < 16 || ks % 16) return false;
    g->Wb = Wb; g->Hb = Hb; g->Bb = Bb;
    g->nbx = W / Wb; g->nby = H / Hb; g->nbb = (B + Bb - 1) / Bb;
    g->kstage = ks;
    return true;
}

// 5-D tensor map (channel, x, y, image, plane) over bf16 hi/lo planes [2][B][H][W][pitch]; C = channel extent (<= pitch):
// channels beyond C and pixels outside the image are zero-filled by the hardware
int planes_map(EncodeTiledFn enc, CUtensorMap* map, void* base, int B, int H, int W, int C, int pitch, const WgGeom& g) {
    const cuuint64_t gdim[5] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B, 2};
    const cuuint64_t gstr[4] = {(cuuint64_t)pitch * 2, (cuuint64_t)W * pitch * 2, (cuuint64_t)H * W * pitch * 2,
                                (cuuint64_t)B * H * W * pitch * 2};
    const cuuint32_t box[5] = {64, (cuuint32_t)g.Wb, (cuuint32_t)g.Hb, (cuuint32_t)g.Bb, 1};
    const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, base, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(EFFDET_ERR_LAUNCH, "wgrad(tc): cuTensorMapEncodeTiled failed (%d)", (int)r);
    return EFFDET_OK;
}

// TMA-fed weight gradient of one shared-weight layer over all levels in one launch.  conv_api.cu has checked that every
// level has a pixel box and both operands as planes or plane workspaces, and that the tensor-map encoder is available.
int wgrad_tc2_launch(const effdet_wgrad_args* levels, int nlevels, float* acc, cudaStream_t st) {
    EncodeTiledFn enc = encode_fn();
    WgMaps maps;
    WgMultiArgs ma;
    memset(&ma, 0, sizeof(ma));
    const effdet_wgrad_args* a0 = &levels[0];
    const int cin_pad = conv_tc_kpad(a0->Cin), cout_pad = conv_tc_kpad(a0->Cout);
    int chunks = 0;
    for (int l = 0; l < nlevels; ++l) {
        const effdet_wgrad_args* a = &levels[l];
        wg_geometry(a->B, a->H, a->W, &ma.g[l]);
        ma.chunk_begin[l] = chunks;
        chunks += ma.g[l].nbx * ma.g[l].nby * ma.g[l].nbb;
    }
    for (int l = nlevels; l <= kWgMaxLevels; ++l) ma.chunk_begin[l] = chunks;
    ma.nlevels = nlevels;
    ma.acc = acc;
    ma.Cin = a0->Cin; ma.Cout = a0->Cout; ma.ksize = a0->ksize;
    for (int l = 0; l < nlevels; ++l) {
        const effdet_wgrad_args* a = &levels[l];
        const int HW = a->H * a->W;
        int s = EFFDET_OK;
        if (a->x_planes) {          // operands that already live as planes: no split pass at all
            if ((s = planes_map(enc, &maps.x[l], const_cast<void*>(a->x_planes), a->B, a->H, a->W, a->Cin, (a->Cin + 7) / 8 * 8, ma.g[l])))
                return s;
        } else {
            if ((s = to_planes_launch(a->x, a->x_bstride, nullptr, 0, a->ws_x, nullptr, a->B, HW, a->Cin, cin_pad, st))) return s;
            if ((s = planes_map(enc, &maps.x[l], a->ws_x, a->B, a->H, a->W, cin_pad, cin_pad, ma.g[l]))) return s;
        }
        if (a->dy_planes) {         // unpadded pitch: TMA zero-fills the channels beyond Cout
            if ((s = planes_map(enc, &maps.dy[l], const_cast<void*>(a->dy_planes), a->B, a->H, a->W, a->Cout, (a->Cout + 7) / 8 * 8,
                                ma.g[l])))
                return s;
        } else {                    // the split pass also accumulates the bias gradient
            if ((s = to_planes_launch(a->dy, a->dy_bstride, nullptr, 0, a->ws_dy, a->dbias, a->B, HW, a->Cout, cout_pad, st))) return s;
            if ((s = planes_map(enc, &maps.dy[l], a->ws_dy, a->B, a->H, a->W, cout_pad, cout_pad, ma.g[l]))) return s;
        }
    }
    for (int l = nlevels; l < kWgMaxLevels; ++l) { maps.dy[l] = maps.dy[0]; maps.x[l] = maps.x[0]; }
    const int taps = a0->ksize * a0->ksize;
    const int BC = a0->Cin > 64 ? 256 : 64;
    const int ctiles = cdiv(a0->Cin, BC), ntiles = cdiv(a0->Cout, kTileM);
    // split-K so that the grid is as close as possible to (but not above) two full waves of CTAs, and no CTA accumulates
    // more than kWgMaxChunksPerSplit chunks.  tests/test_planes_path_parity.py (_split_plan) mirrors this arithmetic.
    int splits = (num_sms() * 2) / (ctiles * ntiles * taps);
    if (splits < 1) splits = 1;
    if (splits > cdiv(chunks, 4)) splits = cdiv(chunks, 4);
    if (splits < cdiv(chunks, kWgMaxChunksPerSplit)) splits = cdiv(chunks, kWgMaxChunksPerSplit);
    int cps = cdiv(chunks, splits);
    splits = cdiv(chunks, cps);
    dim3 grid(ctiles * ntiles, taps, splits);
    if (a0->tc_single) {
        if (BC == 256)
            return launch_smem("wgrad_tc2_multi_kernel", wgrad_tc2_multi_kernel<256, 2, 1>, grid, kTcThreads, WgSmem<256, 2>::kBytes,
                               st, maps, ma, cps, ctiles);
        return launch_smem("wgrad_tc2_multi_kernel", wgrad_tc2_multi_kernel<64, 4, 1>, grid, kTcThreads, WgSmem<64, 4>::kBytes, st,
                           maps, ma, cps, ctiles);
    }
    if (BC == 256)
        return launch_smem("wgrad_tc2_multi_kernel", wgrad_tc2_multi_kernel<256, 2, 3>, grid, kTcThreads, WgSmem<256, 2>::kBytes, st,
                           maps, ma, cps, ctiles);
    return launch_smem("wgrad_tc2_multi_kernel", wgrad_tc2_multi_kernel<64, 4, 3>, grid, kTcThreads, WgSmem<64, 4>::kBytes, st, maps,
                       ma, cps, ctiles);
}

// weight gradient of one level from fp32 operands that the kernel gathers itself; the bias gradient is not part of it
int wgrad_tc_launch(const effdet_wgrad_args* a, float* acc, cudaStream_t st) {
    const int M = a->B * a->H * a->W, HW = a->H * a->W;
    const int taps = a->ksize * a->ksize;
    const int BC = a->Cin > 64 ? 256 : 64;
    const int ctiles = cdiv(a->Cin, BC), ntiles = cdiv(a->Cout, kTileM);
    const int nchunks = cdiv(M, kTileK);
    int splits = cdiv(num_sms() * 2, ctiles * ntiles * taps);
    if (splits < 1) splits = 1;
    if (splits > cdiv(nchunks, 8)) splits = cdiv(nchunks, 8);
    if (splits < cdiv(nchunks, kWgMaxChunksPerSplit)) splits = cdiv(nchunks, kWgMaxChunksPerSplit);
    int cps = cdiv(nchunks, splits);
    splits = cdiv(nchunks, cps);
    dim3 grid(ctiles * ntiles, taps, splits);
    WgradPrefix pa;
    pa.set(*a);
    if (a->tc_single) {
        if (BC == 256)
            return launch_smem("wgrad_tc_kernel", wgrad_tc_kernel<256, 2, 1>, grid, kTcProducers, WgSmem<256, 2>::kBytes, st, pa,
                               acc, M, HW, cps, ctiles);
        return launch_smem("wgrad_tc_kernel", wgrad_tc_kernel<64, 4, 1>, grid, kTcProducers, WgSmem<64, 4>::kBytes, st, pa, acc, M,
                           HW, cps, ctiles);
    }
    if (BC == 256)
        return launch_smem("wgrad_tc_kernel", wgrad_tc_kernel<256, 2, 3>, grid, kTcProducers, WgSmem<256, 2>::kBytes, st, pa, acc, M,
                           HW, cps, ctiles);
    return launch_smem("wgrad_tc_kernel", wgrad_tc_kernel<64, 4, 3>, grid, kTcProducers, WgSmem<64, 4>::kBytes, st, pa, acc, M, HW,
                       cps, ctiles);
}

// dw[n][c][tap] += ws[tap][n][c] for the nc = Cout * Cin (n, c) pairs of a 3x3 weight gradient
int wgrad_fold_launch(const float* ws, float* dw, long long nc, cudaStream_t st) {
    wgrad_fold_kernel<<<cdiv(nc, kFoldPairs), kFoldPairs, 0, st>>>(ws, dw, nc);
    return launch_status("wgrad_fold_kernel");
}

}  // namespace effdet

using namespace effdet;

extern "C" int effdet_conv_tc_kpad(int channels) { return conv_tc_kpad(channels); }
extern "C" int effdet_wgrad_tc_geometry_ok(int B, int H, int W) {
    WgGeom g;
    return wg_geometry(B, H, W, &g) ? 1 : 0;
}

extern "C" int effdet_pack_conv_weight_tc(const float* w_oihw, void* w_fwd, void* w_dgrad, int Cout, int Cin, int ksize,
                                          int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(w_oihw && w_fwd && Cout > 0 && Cin > 0 && (ksize == 1 || ksize == 3), "pack_conv_weight_tc: bad arguments");
    EFFDET_DEVICE(device);
    const int taps = ksize * ksize;
    cudaStream_t st = (cudaStream_t)stream;
    {
        const int kpad = conv_tc_kpad(Cin);
        const long long plane = (long long)Cout * taps * kpad;
        int blocks = cdiv(plane, 256);
        if (blocks > num_sms() * 8) blocks = num_sms() * 8;
        pack_weight_tc_kernel<<<blocks, 256, 0, st>>>(w_oihw, (__nv_bfloat16*)w_fwd, Cout, Cin, taps, kpad, 0);
        int s = launch_status("pack_weight_tc_kernel");
        if (s) return s;
    }
    if (w_dgrad) {
        const int kpad = conv_tc_kpad(Cout);
        const long long plane = (long long)Cin * taps * kpad;
        int blocks = cdiv(plane, 256);
        if (blocks > num_sms() * 8) blocks = num_sms() * 8;
        pack_weight_tc_kernel<<<blocks, 256, 0, st>>>(w_oihw, (__nv_bfloat16*)w_dgrad, Cout, Cin, taps, kpad, 1);
        return launch_status("pack_weight_tc_kernel");
    }
    return EFFDET_OK;
}
