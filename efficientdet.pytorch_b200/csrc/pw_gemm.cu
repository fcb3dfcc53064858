// Pointwise (1x1) convolution of the backbone / laterals as a persistent, warp-specialised wgmma GEMM.
//
//   y[M, Cout] = epilogue( prologue(x[M, Cin]) * W[Cin, Cout] )        M = B*H*W pixels (NHWC rows)
//
// These layers are HBM-bound (arithmetic intensity 7..80 FLOP/B, SURVEY.md 8(d)): what matters is that every SM keeps
// tens of KB of loads and stores in flight and that nothing is serialised behind anything else.  Round 1 ran them on
// the 3x3 implicit-GEMM kernel: one tile per CTA, the gather warps doubled as epilogue warps, so load, MMA and store
// phases of a CTA never overlapped.  Here a CTA is persistent over (m-tile, n-tile) units and three roles run
// concurrently, decoupled by mbarrier rings:
//
//   warp 8      TMA producer : fp32 activation boxes [128 rows x 32 channels] (SWIZZLE_128B, out-of-bounds rows / channels
//                              zero-filled by the hardware) + the bf16 hi/lo weight tile of the k-block -> ring of NS stages
//   2 warps     converters   : fp32 tile -> optional BN+swish (+ squeeze-excite gate) prologue -> bf16 hi + lo planes in the
//                              canonical K-major SWIZZLE_128B layout (x = hi + lo to 16 mantissa bits)
//   warps 0-7   consumers    : two warpgroups, one per 64-row half of the tile: 3 wgmma per K16 (lo*hi, hi*lo, hi*hi),
//                              fp32 accumulation in registers, then the epilogue (bias / BN affine / drop-connect /
//                              residual, direct 128-bit stores) while the converters already fill the next unit's planes
//
// Reference ops replaced: MBConvBlock expand / project convs and their data gradients (models/efficientnet.py:85,96-104),
// BIFPN lateral convs (models/bifpn.py:96-105).
#include "tc_ptx.cuh"

namespace effdet {

constexpr int kPwA32Half = 128 * 128;      // bytes of one fp32 half-box: 128 rows x 32 floats
constexpr int kPwA16 = 2 * 128 * 128;      // bytes of one bf16 stage: hi plane + lo plane, 128 rows x 64 bf16 each
constexpr int kPwMaxStages = 6;
constexpr int kPwBarBytes = 512;           // 17 mbarriers
constexpr int kPwChanBytes = 3 * 128 * 4;  // bias | scale | shift of the current n-tile
constexpr int kPwConv = 2;                 // converter warps: 11 warps in all leave the consumers 168 registers

struct PwParams {
    effdet_conv_args a;
    int M, HW;
    int KB;          // k-blocks of 64 input channels
    int BN;          // output channels per n-tile (64 or 128)
    int ntn;         // n-tiles
    int units;       // m-tiles * n-tiles
    int NS;          // ring stages
    int a32_halves;  // fp32 half-boxes per stage (1 when Cin <= 32)
    int bres;        // the whole packed weight (ntn x KB tiles) stays resident in shared memory: loaded once per CTA, the
                     // ring then carries activations only and is deeper (more loads in flight per SM)
    int planes;      // the A operand arrives pre-split as bf16 hi/lo planes [2][M][Cin]: TMA writes the MMA operand
                     // layout directly, no converter work (data gradients of the expand convs: the fused depthwise
                     // backward emits dz0 in this form for this kernel and for the weight gradient)
};

__device__ __forceinline__ void split4(const float4 v, uint2& hi, uint2& lo) {
    const __nv_bfloat162 h0 = __floats2bfloat162_rn(v.x, v.y), h1 = __floats2bfloat162_rn(v.z, v.w);
    const __nv_bfloat162 l0 = __floats2bfloat162_rn(v.x - __low2float(h0), v.y - __high2float(h0));
    const __nv_bfloat162 l1 = __floats2bfloat162_rn(v.z - __low2float(h1), v.w - __high2float(h1));
    hi = make_uint2(*reinterpret_cast<const uint32_t*>(&h0), *reinterpret_cast<const uint32_t*>(&h1));
    lo = make_uint2(*reinterpret_cast<const uint32_t*>(&l0), *reinterpret_cast<const uint32_t*>(&l1));
}

constexpr int kPwThreads = (9 + kPwConv) * 32;

template <int NB>            // 64-column blocks per n-tile: BN = 64 * NB
__global__ void __launch_bounds__(kPwThreads, 1)
pw_gemm_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const __grid_constant__ PwParams P) {
    constexpr int NC = kPwConv;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // 1024-byte aligned AND still a shared-space pointer (LDS/STS, not generic LD/ST)
    const effdet_conv_args& p = P.a;
    const int a32_bytes = P.planes ? kPwA16 : P.a32_halves * kPwA32Half;
    const int b_plane = P.BN * 128;
    const int stage_bytes = a32_bytes + (P.bres ? 0 : 2 * b_plane);
    uint8_t* ring = smem;
    uint8_t* bres = ring + P.NS * stage_bytes;                         // [ntn][KB][hi | lo] weight tiles (resident mode)
    uint8_t* a16 = bres + (P.bres ? P.ntn * P.KB * 2 * b_plane : 0);
    float* rows_buf = reinterpret_cast<float*>(a16 + (P.planes ? 0 : 2 * kPwA16));   // epilogue staging (wg_rows)
    uint64_t* ld_full = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(rows_buf) + kRowsBytes);
    uint64_t* ld_empty = ld_full + kPwMaxStages;
    uint64_t* a16_full = ld_empty + kPwMaxStages;
    uint64_t* a16_empty = a16_full + 2;
    uint64_t* b_full = a16_empty + 2;
    float* chan = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(ld_full) + kPwBarBytes);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < kPwMaxStages; ++s) {
            mbar_init(&ld_full[s], 1);
            mbar_init(&ld_empty[s], P.planes ? 8 : NC + 8);   // the converter warps + the 8 consumer warps
        }
        for (int s = 0; s < 2; ++s) {
            mbar_init(&a16_full[s], NC);
            mbar_init(&a16_empty[s], 8);
        }
        mbar_init(b_full, 1);
        fence_barrier_init();
        tma_prefetch_desc(&map_a);
        tma_prefetch_desc(&map_b);
    }
    __syncthreads();

    if (warp == 8) {
        // ------------------------------------------------ TMA producer ----------------------------------------------
        if (lane == 0) {
            const uint32_t btx = P.bres ? 0u : (uint32_t)(2 * b_plane);
            if (P.bres) {                                          // all weight tiles once, on their own barrier
                mbar_arrive_expect_tx(b_full, (uint32_t)(P.ntn * P.KB * 2 * b_plane));
                for (int nt = 0; nt < P.ntn; ++nt)
                    for (int kb = 0; kb < P.KB; ++kb) {
                        uint8_t* bt = bres + (nt * P.KB + kb) * 2 * b_plane;
                        tma_load_3d(bt, &map_b, b_full, kb * 64, nt * P.BN, 0);
                        tma_load_3d(bt + b_plane, &map_b, b_full, kb * 64, nt * P.BN, 1);
                    }
            }
            uint32_t it = 0;
            for (int u = blockIdx.x; u < P.units; u += gridDim.x) {
                const int mt = u / P.ntn, nt = u - mt * P.ntn;
                const int m0 = mt * 128, n0 = nt * P.BN;
                for (int kb = 0; kb < P.KB; ++kb, ++it) {
                    const int s = it % P.NS;
                    const uint32_t ph = (it / P.NS) & 1;
                    mbar_wait(&ld_empty[s], ph ^ 1);
                    uint8_t* st = ring + s * stage_bytes;
                    if (P.planes) {
                        mbar_arrive_expect_tx(&ld_full[s], (uint32_t)kPwA16 + btx);
                        tma_load_3d(st, &map_a, &ld_full[s], kb * 64, m0, 0);
                        tma_load_3d(st + kPwA16 / 2, &map_a, &ld_full[s], kb * 64, m0, 1);
                    } else {
                        const int halves = (p.Cin - kb * 64 > 32) ? 2 : 1;
                        mbar_arrive_expect_tx(&ld_full[s], (uint32_t)(halves * kPwA32Half) + btx);
                        tma_load_2d(st, &map_a, &ld_full[s], kb * 64, m0);
                        if (halves == 2) tma_load_2d(st + kPwA32Half, &map_a, &ld_full[s], kb * 64 + 32, m0);
                    }
                    if (!P.bres) {
                        tma_load_3d(st + a32_bytes, &map_b, &ld_full[s], kb * 64, n0, 0);
                        tma_load_3d(st + a32_bytes + b_plane, &map_b, &ld_full[s], kb * 64, n0, 1);
                    }
                }
            }
        }
    } else if (warp > 8) {
        // ------------------------------------------------ converters ------------------------------------------------
        constexpr int RP = 4 * NC;                             // rows per pass (8 threads per row)
        const int tid = threadIdx.x - 9 * 32;
        const int j = tid & 7, rbase = tid >> 3;
        const bool pro = p.in_scale != nullptr || p.a_scale != nullptr;
        uint32_t it = 0;
        for (int u = blockIdx.x; u < (P.planes ? 0 : P.units); u += gridDim.x) {      // planes mode: nothing to convert
            const int mt = u / P.ntn;
            const int m0 = mt * 128;
            const int b_first = m0 / P.HW;
            const bool one_image = (min(m0 + 127, P.M - 1) / P.HW) == b_first;   // the usual case: HW >> 128
            for (int kb = 0; kb < P.KB; ++kb, ++it) {
                const int s = it % P.NS;
                const uint32_t ph = (it / P.NS) & 1;
                const uint32_t sa = it & 1, pha = (it >> 1) & 1;
                mbar_wait(&ld_full[s], ph);
                mbar_wait(&a16_empty[sa], pha ^ 1);
                const uint8_t* a32 = ring + s * stage_bytes;
                uint8_t* hi_pl = a16 + sa * kPwA16;
                uint8_t* lo_pl = hi_pl + kPwA16 / 2;
                // both 32-channel halves are always written (zeros past Cin): the MMAs run all four K16 steps of the
                // block against the zero-padded weights, and stale shared memory must not reach them
                for (int h = 0; h < 2; ++h) {
                    const int c = kb * 64 + h * 32 + 4 * j;
                    const bool col_ok = c < p.Cin;
                    float4 isc = make_float4(1.f, 1.f, 1.f, 1.f), ish = f4zero(), gate = isc;
                    if (p.in_scale && col_ok) { isc = ldg4(p.in_scale + c); ish = ldg4(p.in_shift + c); }
                    if (p.a_scale && col_ok && one_image) gate = ldg4(p.a_scale + (long long)b_first * p.Cin + c);
#pragma unroll
                    for (int i = 0; i < 128 / RP; ++i) {
                        const int r = rbase + RP * i;
                        float4 v = col_ok ? *reinterpret_cast<const float4*>(a32 + h * kPwA32Half + r * 128 + ((j ^ (r & 7)) << 4))
                                          : f4zero();          // (the swish of a zero-filled column would not be zero)
                        if (pro && col_ok) {
                            if (p.in_scale) {
                                const float4 q = f4fma(v, isc, ish);
                                v = make_float4(fswish(q.x), fswish(q.y), fswish(q.z), fswish(q.w));
                            }
                            if (p.a_scale) {
                                if (!one_image) {
                                    const int m = m0 + r;
                                    gate = ldg4(p.a_scale + (long long)((m < P.M ? m : P.M - 1) / P.HW) * p.Cin + c);
                                }
                                v = f4mul(v, gate);
                            }
                        }
                        uint2 hi, lo;
                        split4(v, hi, lo);
                        const int off = r * 128 + (((h * 4 + (j >> 1)) ^ (r & 7)) << 4) + (j & 1) * 8;
                        *reinterpret_cast<uint2*>(hi_pl + off) = hi;
                        *reinterpret_cast<uint2*>(lo_pl + off) = lo;
                    }
                }
                fence_proxy_async();
                __syncwarp();
                if (lane == 0) {
                    mbar_arrive(&a16_full[sa]);
                    mbar_arrive(&ld_empty[s]);
                }
            }
        }
    } else {
        // ------------------------------------------------ consumers: wgmma + epilogue ---------------------------------------
        const int g = warp >> 2;                               // rows 64g .. 64g+63 of the tile
        const int etid = threadIdx.x;
        const int quarter = 2 * g + (warp & 1), half = (warp >> 1) & 1;
        const int r = quarter * 32 + lane;                     // row of the tile owned by this thread
        uint32_t it = 0;
        if (P.bres) mbar_wait(b_full, 0);                      // resident weights landed
        for (int u = blockIdx.x; u < P.units; u += gridDim.x) {
            const int mt = u / P.ntn, nt = u - mt * P.ntn;
            const int m0 = mt * 128, n0 = nt * P.BN;
            float d[NB][32];
            for (int kb = 0; kb < P.KB; ++kb, ++it) {
                const int s = it % P.NS;
                const uint32_t ph = (it / P.NS) & 1;
                const uint32_t sa = it & 1, pha = (it >> 1) & 1;
                mbar_wait(&ld_full[s], ph);                    // weight tile (and, in planes mode, the A planes) landed
                if (!P.planes) mbar_wait(&a16_full[sa], pha);  // converters published the bf16 planes
                const uint32_t a_hi = (P.planes ? smem_u32(ring + s * stage_bytes) : smem_u32(a16 + sa * kPwA16)) + g * 64 * 128;
                const uint32_t a_lo = a_hi + kPwA16 / 2;
                const uint32_t b_hi = P.bres ? smem_u32(bres + (nt * P.KB + kb) * 2 * b_plane)
                                             : smem_u32(ring + s * stage_bytes + a32_bytes);
                const uint32_t b_lo = b_hi + b_plane;
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k) {                  // K is zero-padded to 64 per block (weights and A planes)
                    wg_mma<NB, 0, 3>(d, a_hi + k * 32, a_lo + k * 32, b_hi + k * 32, b_lo + k * 32, 16, 1024, (kb | k) != 0);
                }
                wgmma_commit();
                wgmma_wait<1>();                               // the previous k-block's operands are no longer read
                if (kb > 0 && lane == 0) {
                    if (!P.planes) mbar_arrive(&a16_empty[(it - 1) & 1]);
                    mbar_arrive(&ld_empty[(it - 1) % P.NS]);
                }
            }
            wgmma_wait<0>();
            if (lane == 0) {
                if (!P.planes) mbar_arrive(&a16_empty[(it - 1) & 1]);
                mbar_arrive(&ld_empty[(it - 1) % P.NS]);
            }
            named_bar_sync(1, 256);                            // everybody is done with the previous unit's vectors
            for (int i = etid; i < P.BN; i += 256) {
                const int n = n0 + i;
                const bool ok = n < p.Cout;
                chan[i] = (ok && p.bias) ? __ldg(p.bias + n) : 0.f;
                chan[128 + i] = (ok && p.scale) ? __ldg(p.scale + n) : 1.f;
                chan[256 + i] = (ok && p.shift) ? __ldg(p.shift + n) : 0.f;
            }
            named_bar_sync(1, 256);
            const int ncols = min(P.BN, p.Cout - n0);
            const int nchunks = (ncols + 31) >> 5;
            const int m = m0 + r;
            const bool row_ok = m < P.M;
            int b = 0;
            long long pix = 0;
            if (row_ok) { b = m / P.HW; pix = m - (long long)b * P.HW; }
            const float rs = (row_ok && p.row_scale) ? __ldg(p.row_scale + b) : 1.f;
            const long long ybase = (long long)b * p.y_bstride + pix * p.Cout;
            const long long rbase_ = (long long)b * p.r_bstride + pix * p.Cout;
            const long long mbase = (long long)b * p.m_bstride + pix * p.Cout;
#pragma unroll
            for (int jb = 0; jb < NB; ++jb) {
                float v32[32];
                wg_rows<2>(d[jb], rows_buf, g, v32);
                const int cc = 2 * jb + half;
                if (cc >= nchunks || !row_ok) continue;
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const int nl = cc * 32 + q * 4;
                    const int n = n0 + nl;
                    if (n >= p.Cout) break;
                    float4 v = make_float4(v32[q * 4], v32[q * 4 + 1], v32[q * 4 + 2], v32[q * 4 + 3]);
                    v = f4add(v, *reinterpret_cast<const float4*>(chan + nl));
                    if (p.z) st4(p.z + ybase + n, v);
                    v = f4fma(v, *reinterpret_cast<const float4*>(chan + 128 + nl), *reinterpret_cast<const float4*>(chan + 256 + nl));
                    if (p.act == EFFDET_ACT_RELU) {
                        v = make_float4(fmaxf(v.x, 0.f), fmaxf(v.y, 0.f), fmaxf(v.z, 0.f), fmaxf(v.w, 0.f));
                    } else if (p.act == EFFDET_ACT_SIGMOID) {
                        v = make_float4(sigmoidf_(v.x), sigmoidf_(v.y), sigmoidf_(v.z), sigmoidf_(v.w));
                    } else if (p.act == EFFDET_ACT_SWISH) {
                        v = make_float4(swishf_(v.x), swishf_(v.y), swishf_(v.z), swishf_(v.w));
                    }
                    if (p.row_scale) v = f4scale(v, rs);
                    if (p.residual) v = f4add(v, ldg4(p.residual + rbase_ + n));
                    if (p.mask_src) {
                        const float4 mk = ldg4(p.mask_src + mbase + n);
                        v = make_float4(mk.x > 0.f ? v.x : 0.f, mk.y > 0.f ? v.y : 0.f, mk.z > 0.f ? v.z : 0.f,
                                        mk.w > 0.f ? v.w : 0.f);
                    }
                    st4(p.y + ybase + n, v);
                }
            }
        }
    }
}

int pw_gemm_launch(const effdet_conv_args* a, cudaStream_t st) {
    EncodeTiledFn enc = encode_fn();
    if (!enc) return fail(EFFDET_ERR_UNSUPPORTED, "conv2d(pw): cuTensorMapEncodeTiled unavailable");
    PwParams P;
    memset(&P, 0, sizeof(P));
    P.a = *a;
    P.HW = a->H * a->W;
    P.M = a->B * P.HW;
    const int kpad = conv_tc_kpad(a->Cin);
    P.KB = kpad / 64;
    P.ntn = cdiv(a->Cout, 128);
    P.BN = cdiv(cdiv(a->Cout, P.ntn), 64) * 64;
    P.ntn = cdiv(a->Cout, P.BN);
    const int mtiles = cdiv(P.M, 128);
    P.units = mtiles * P.ntn;
    P.a32_halves = a->Cin > 32 ? 2 : 1;
    P.planes = a->x_planes ? 1 : 0;
    const int a_stage = P.planes ? kPwA16 : P.a32_halves * kPwA32Half;
    const int b_all = P.ntn * P.KB * P.BN * 256;                        // every weight tile of the layer (hi + lo)
    P.bres = b_all <= 64 * 1024 ? 1 : 0;
    const int stage_bytes = a_stage + (P.bres ? 0 : P.BN * 256);
    const int fixed = (P.planes ? 0 : 2 * kPwA16) + kRowsBytes + kPwBarBytes + kPwChanBytes + 1024 + (P.bres ? b_all : 0);
    const int budget = 227 * 1024 - fixed;
    int ns = budget / stage_bytes;
    if (ns > kPwMaxStages) ns = kPwMaxStages;
    if (ns < 2) return fail(EFFDET_ERR_UNSUPPORTED, "conv2d(pw): shared memory budget");
    P.NS = ns;
    const size_t smem = (size_t)fixed + (size_t)ns * stage_bytes;

    CUtensorMap map_a, map_b;
    if (P.planes) {
        const int s = kmajor_planes_map(enc, &map_a, a->x_planes, P.M, a->Cin, 128);
        if (s) return s;
    } else {
        const cuuint64_t gdim[2] = {(cuuint64_t)a->Cin, (cuuint64_t)P.M};
        const cuuint64_t gstr[1] = {(cuuint64_t)a->Cin * 4};
        const cuuint32_t box[2] = {32, 128};
        const cuuint32_t estr[2] = {1, 1};
        CUresult r = enc(&map_a, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(a->x), gdim, gstr, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return fail(EFFDET_ERR_LAUNCH, "conv2d(pw): tensor map of x failed (%d)", (int)r);
    }
    const int s = kmajor_planes_map(enc, &map_b, a->w_tc, a->Cout, kpad, P.BN);
    if (s) return s;
    const int grid = P.units < num_sms() ? P.units : num_sms();
    if (P.BN == 128) return launch_smem("pw_gemm_kernel", pw_gemm_kernel<2>, grid, kPwThreads, smem, st, map_a, map_b, P);
    return launch_smem("pw_gemm_kernel", pw_gemm_kernel<1>, grid, kPwThreads, smem, st, map_a, map_b, P);
}

}  // namespace effdet
