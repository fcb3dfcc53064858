// Dense 3x3 / 1x1 convolution whose activations live in HBM as bf16 hi/lo planes (x ~= hi + lo, the tensor-core operand
// format) -- the RetinaHead towers end to end (models/retinahead.py:67-132; 95 % of the model's FLOPs).
//
//   conv_planes_kernel  the convolution below
//   to_planes_kernel    fp32 -> planes, for the head's first input, its output gradients and the operands of the TMA-fed
//                       weight gradient (conv_tc.cu) that are not planes yet
//
// Kept as fp32, every conv would re-split its input on the fly with eight gather warps (LDG + cvt + st.shared) and every
// weight gradient would need a separate split pass over both operands.  With the
// planes format the im2col gather IS a TMA load: a 5-D tensor map (channel, x, y, image, plane) with a pixel box of
// Wb x Hb x Bb pixels delivers, for one tap, 64 channels of 16..64 pixels as consecutive 128-byte rows in the canonical
// K-major SWIZZLE_128B layout; the tap shift is a coordinate offset and the hardware's out-of-bounds zero fill is the
// convolution's zero padding.  The kernel is a warp-specialised Hopper GEMM:
//   warp 8      TMA producer (activation boxes hi/lo + weight tile hi/lo -> mbarrier complete_tx), ring of stages
//               filled in unit order
//   warps 0-7   two consumer warpgroups in ping-pong: the CTA's units alternate between them, and each owns a whole
//               128-row tile (two 64-row accumulator sets): 3 wgmma per K16 and row half (lo*hi, hi*lo, hi*hi) with the
//               accumulator in registers (single-pass instance, NP = 1: hi*hi only, and the producer loads no lo plane),
//               then the epilogue: bias / ReLU / sigmoid / ReLU-mask / residual -> bf16 hi/lo planes (the next layer's
//               operand) and / or fp32 (head outputs, data gradient w.r.t. the BiFPN features); optional per-channel
//               column sums of what was stored (= the bias gradient of the producing layer) reduced by warp shuffles
//               into the CTA's [Cout] array (shared atomics), added to colsum once per CTA.  One warpgroup's epilogue
//               runs under the other's MMAs.
// persistent over (pixel tile, channel tile) units of all pyramid levels that share the weights.
// A ReLU forward can also write the one-bit mask its data gradient applies (y_mask: bit c % 32 of word (pixel, c / 32)
// <=> the stored value of channel c is > 0); a data gradient given mask_bits loads its words before its last MMAs
// complete, 4 bytes per 32 channels instead of 2 x 64 bytes of planes read after them.
#include "tc_ptx.cuh"

#include <limits.h>
#include <stdlib.h>

namespace effdet {

constexpr int kPlMaxLevels = 8;
// two consumer warpgroups and a producer warpgroup: ptxas budgets 168 registers per thread for 384 threads, and
// setmaxnreg moves the producer's share to the consumers (128 x 40 + 256 x 232 = 384 x 168)
constexpr int kPlThreads = 384;
constexpr int kPlProducerRegs = 40, kPlConsumerRegs = 232;
constexpr int kPlA = 128 * 128;            // one plane of the activation tile: 128 pixel rows x 64 channels (bf16)
constexpr int kPlSmemOptin = 227 * 1024;   // sm_90's dynamic shared memory per block
// BN = output channels per tile (accumulator: BN registers per consumer thread); the ring depth is what fits.  Behind
// the ring: the two warpgroups' staging buffers (wg_rows_own), the mbarriers, the two warpgroups' bias buffers, and in
// a launch with column sums the CTA's [Cout] array of them (not counted in kSmem).
template <int BN>
struct PlCfg {
    static constexpr int kStages = BN == 128 ? 3 : 4;
    static constexpr int kB = BN * 128;    // one plane of the weight tile: BN output channels x 64 input channels
    static constexpr int kStage = 2 * kPlA + 2 * kB;
    static constexpr int kSmem = kStages * kStage + kRowsBytes + 1024 + 256 + 2 * BN * 4;
};
// named barriers: 1 both consumer warpgroups (their column sums are complete), 2 + g the staging buffer and bias
// buffer of consumer warpgroup g, 4 + g its turn to consume
constexpr int kPlBarSums = 1, kPlBarRows = 2, kPlBarTurn = 4;

// bit e (0..7) set <=> the value stored as the bf16 pair (hi, lo) of channel e is > 0: sign clear and magnitude
// bits set, in hi or, where hi is zero, in lo
__device__ __forceinline__ uint32_t relu_bits8(const uint4 hi, const uint4 lo) {
    const uint32_t hw[4] = {hi.x, hi.y, hi.z, hi.w}, lw[4] = {lo.x, lo.y, lo.z, lo.w};
    uint32_t bits = 0;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
        const uint32_t hb = (hw[e >> 1] >> ((e & 1) * 16)) & 0xffffu, lb = (lw[e >> 1] >> ((e & 1) * 16)) & 0xffffu;
        const bool pos = (hb & 0x7fffu) ? !(hb & 0x8000u) : ((lb & 0x7fffu) && !(lb & 0x8000u));
        bits |= (uint32_t)pos << e;
    }
    return bits;
}

struct PlLevel {
    int B, H, W;
    WgGeom g;
    int tile_begin;                        // first pixel tile of this level
    int nboxes;                            // pixel boxes of this level
    float* y;                              // fp32 output [B][H*W][Cout] with image stride y_bstride, or NULL
    long long y_bstride;
    __nv_bfloat16* y_planes;               // bf16 hi/lo output planes [2][B*H*W][opitch], or NULL
    const __nv_bfloat16* mask_planes;      // ReLU-backward mask source [2][B*H*W][opitch] (value > 0 keeps the gradient), or NULL
    uint32_t* y_mask;                      // ReLU bits of the stored planes [B*H*W][mwords], or NULL
    const uint32_t* mask_bits;             // ReLU-backward mask as bits [B*H*W][mwords] (set keeps the gradient), or NULL
    const float* residual;                 // fp32 [B][H*W][Cout] added last, or NULL
    long long r_bstride;
};
struct PlArgs {
    PlLevel lv[kPlMaxLevels];
    int nlevels, total_tiles, ntn;
    int Cin, Cout, ksize, act, kblocks, opitch, mwords;
    const float* bias;                     // [Cout] or NULL
    float* colsum;                         // [Cout] += column sums of the stored values, or NULL
};
struct PlMaps {
    CUtensorMap x[kPlMaxLevels];
};

// one step of a warp transpose-reduce of v[0 .. 2 OFF - 1]: lanes with bit OFF set keep the upper half, the others the
// lower one, and each adds its partner's copy of the half it keeps.  A compile-time OFF keeps v in registers (a loop
// over OFF that is not unrolled indexes v at run time, which puts it in local memory).
template <int OFF>
__device__ __forceinline__ void transpose_add(float (&v)[32], const int lane) {
    const bool upper = (lane & OFF) != 0;
#pragma unroll
    for (int k = 0; k < OFF; ++k) {
        const float send = upper ? v[k] : v[k + OFF];
        const float keep = upper ? v[k + OFF] : v[k];
        v[k] = keep + __shfl_xor_sync(0xffffffffu, send, OFF);
    }
}

// NP = bf16 products per multiply-add: 3 (split precision) or 1 (hi planes only)
template <int BN, int NP>
__global__ void __launch_bounds__(kPlThreads, 1)
conv_planes_kernel(const __grid_constant__ PlMaps maps, const __grid_constant__ CUtensorMap wmap, const __grid_constant__ PlArgs P) {
    constexpr int kPlBN = BN, kPlStages = PlCfg<BN>::kStages, kPlB = PlCfg<BN>::kB, kPlStage = PlCfg<BN>::kStage;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // 1024-byte aligned AND still a shared-space pointer (LDS/STS, not generic LD/ST)
    float* rows_buf = reinterpret_cast<float*>(smem + kPlStages * kPlStage);       // epilogue staging (wg_rows_own)
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kPlStages * kPlStage + kRowsBytes);
    uint64_t* empty_bar = full_bar + kPlStages;
    float* chan_buf = reinterpret_cast<float*>(smem + kPlStages * kPlStage + kRowsBytes + 256);   // bias of the channel tile
    float* csum = chan_buf + 2 * kPlBN;                                             // the CTA's column sums [Cout]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int taps = P.ksize * P.ksize, pad = P.ksize / 2;
    const int KT = taps * P.kblocks;
    if (threadIdx.x == 0) {
        for (int s = 0; s < kPlStages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 4);     // one arrival per warp of the warpgroup that consumes the stage
        }
        fence_barrier_init();
        tma_prefetch_desc(&wmap);
    }
    if (P.colsum)
        for (int i = threadIdx.x; i < P.Cout; i += kPlThreads) csum[i] = 0.f;
    __syncthreads();

    // unit -> (level, first box of the pixel tile, first output channel)
    auto decode = [&](int unit, int& l, int& box0, int& n0) {
        const int mt = unit / P.ntn;
        n0 = (unit - mt * P.ntn) * kPlBN;
        l = 0;
        while (l + 1 < P.nlevels && mt >= P.lv[l + 1].tile_begin) ++l;
        box0 = (mt - P.lv[l].tile_begin) * (128 / P.lv[l].g.kstage);
    };

    if (warp >= 8) {
        // ---------------- TMA producer (one thread of warpgroup 2) ---------------------------------------------------------
        setmaxnreg_dec<kPlProducerRegs>();
        if (warp == 8 && lane == 0) {
            uint32_t it = 0;
            for (int unit = blockIdx.x; unit < P.total_tiles; unit += gridDim.x) {
                int l, box0, n0;
                decode(unit, l, box0, n0);
                const PlLevel& L = P.lv[l];
                const int ks = L.g.kstage, nbox = 128 / ks;
                const int nvalid = min(nbox, L.nboxes - box0);
                for (int kt = 0; kt < KT; ++kt, ++it) {
                    const int s = it % kPlStages;
                    const uint32_t ph = (it / kPlStages) & 1;
                    const int tap = kt / P.kblocks, kb = kt - tap * P.kblocks;
                    const int dy = tap / P.ksize - pad, dx = tap % P.ksize - pad;
                    mbar_wait(&empty_bar[s], ph ^ 1);
                    uint8_t* a_hi = smem + s * kPlStage;
                    uint8_t* b_hi = a_hi + 2 * kPlA;
                    mbar_arrive_expect_tx(&full_bar[s], (uint32_t)((NP == 3 ? 2 : 1) * (nvalid * ks * 128 + kPlB)));
                    for (int q = 0; q < nvalid; ++q) {
                        int ch = box0 + q;
                        const int bx = ch % L.g.nbx;
                        ch /= L.g.nbx;
                        const int by = ch % L.g.nby;
                        const int bb = ch / L.g.nby;
                        const int x0 = bx * L.g.Wb + dx, y0 = by * L.g.Hb + dy, b0 = bb * L.g.Bb;
                        tma_load_5d(a_hi + q * ks * 128, &maps.x[l], &full_bar[s], kb * 64, x0, y0, b0, 0);
                        if (NP == 3) tma_load_5d(a_hi + kPlA + q * ks * 128, &maps.x[l], &full_bar[s], kb * 64, x0, y0, b0, 1);
                    }
                    tma_load_3d(b_hi, &wmap, &full_bar[s], kt * 64, n0, 0);
                    if (NP == 3) tma_load_3d(b_hi + kPlB, &wmap, &full_bar[s], kt * 64, n0, 1);
                }
            }
        }
    } else {
        // ---------------- consumer warpgroups in ping-pong: wgmma of a whole tile, then its epilogue -----------------------
        // The CTA's k-th unit belongs to warpgroup k & 1 and fills ring slots it = k * KT .. k * KT + KT - 1.  A
        // warpgroup waits for its turn (barrier 4 + g) before it waits on the full barriers of its unit: then every
        // slot before its own has been seen full, so no full barrier it polls is two phases behind the parity it
        // asks for.  It hands the turn on as soon as its last stage has landed, so the other warpgroup's MMAs start
        // while its own last ones and its epilogue run.
        setmaxnreg_inc<kPlConsumerRegs>();
        constexpr int NB = kPlBN / 64;
        const int g = warp >> 2;
        const int half = (warp >> 1) & 1;                          // columns 32 * half .. + 31 of each 64x64 block
        const int etid = threadIdx.x & 127;
        float* rows = rows_buf + g * 32 * kRowsPitch;
        float* chan = chan_buf + g * kPlBN;
        const int nunits = (P.total_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
        int chan_n0 = -1;
        for (int k = g; k < nunits; k += 2) {
            int l, box0, n0;
            decode(blockIdx.x + k * gridDim.x, l, box0, n0);
            const PlLevel& L = P.lv[l];
            if (k > 0) named_bar_sync(kPlBarTurn + g, 256);
            float d[2][NB][32];                                    // rows 0-63 and 64-127 of the tile
            uint32_t it = (uint32_t)k * KT;
            for (int kt = 0; kt < KT; ++kt, ++it) {
                const int s = it % kPlStages;
                const uint32_t ph = (it / kPlStages) & 1;
                mbar_wait(&full_bar[s], ph);
                const uint32_t sa = smem_u32(smem + s * kPlStage);
                const uint32_t sb = sa + 2 * kPlA;
                wgmma_fence();
#pragma unroll
                for (int k16 = 0; k16 < 4; ++k16) {
#pragma unroll
                    for (int m = 0; m < 2; ++m)
                        wg_mma<NB, 0, NP>(d[m], sa + m * 64 * 128 + k16 * 32, sa + kPlA + m * 64 * 128 + k16 * 32, sb + k16 * 32,
                                          sb + kPlB + k16 * 32, 16, 1024, (kt | k16) != 0);
                }
                wgmma_commit();
                wgmma_wait<1>();                                   // the previous stage is no longer read
                if (kt > 0 && lane == 0) mbar_arrive(&empty_bar[(it - 1) % kPlStages]);
            }
            if (k + 1 < nunits) named_bar_arrive(kPlBarTurn + (g ^ 1), 256);
            const int ncols = min(kPlBN, P.Cout - n0);
            const int nchunks = (ncols + 31) >> 5;
            // under the last MMAs: the pixel of the row this thread finishes in each row half (-1 past the map), and
            // the mask words of its chunks
            int pix[2];                                            // < 2^31: B * H * W is checked on the host
            uint32_t mbits[2][NB];
#pragma unroll
            for (int m = 0; m < 2; ++m) {
                // pixel of row r: box q of the tile, position i inside the box (x fastest, then y, then image)
                const int r = m * 64 + (warp & 1) * 32 + lane;
                const int ks = L.g.kstage;
                const int q = r / ks, i = r - q * ks;
                int ch = box0 + q;
                const bool box_ok = ch < L.nboxes;
                const int bx = ch % L.g.nbx;
                ch /= L.g.nbx;
                const int by = ch % L.g.nby;
                const int bb = ch / L.g.nby;
                const int wh = L.g.Wb * L.g.Hb;
                const int bi = i / wh, rem = i - bi * wh;
                const int yy = rem / L.g.Wb, xx = rem - yy * L.g.Wb;
                const int b = bb * L.g.Bb + bi, y = by * L.g.Hb + yy, x = bx * L.g.Wb + xx;
                pix[m] = box_ok && b < L.B ? (b * L.H + y) * L.W + x : -1;
#pragma unroll
                for (int jb = 0; jb < NB; ++jb) {
                    const int cc = 2 * jb + half;
                    mbits[m][jb] = L.mask_bits && pix[m] >= 0 && cc < nchunks
                                       ? __ldg(L.mask_bits + (long long)pix[m] * P.mwords + (n0 >> 5) + cc) : 0u;
                }
            }
            wgmma_wait<0>();
            if (lane == 0) mbar_arrive(&empty_bar[(it - 1) % kPlStages]);
            if (n0 != chan_n0) {
                named_bar_sync(kPlBarRows + g, 128);
                for (int i = etid; i < kPlBN; i += 128) chan[i] = (n0 + i < P.Cout && P.bias) ? __ldg(P.bias + n0 + i) : 0.f;
                named_bar_sync(kPlBarRows + g, 128);
                chan_n0 = n0;
            }
            const long long plane = (long long)L.B * L.H * L.W * P.opitch;
            // One copy of the block epilogue, looped over the 2 x NB blocks (only the staging, which must name its
            // accumulator block statically, is unrolled): unrolled per block, the kernel's code grew past what the
            // SMs' instruction caches hold, and every launch paid for it, with or without mask, residual or sums.
#pragma unroll 1
            for (int blk = 0; blk < 2 * NB; ++blk) {
                const int m = blk / NB, jb = blk - m * NB;
                float v[32];
                uint32_t keep_bits = 0;
#pragma unroll
                for (int q = 0; q < 2 * NB; ++q)
                    if (q == blk) {
                        wg_rows_own(d[q / NB][q % NB], rows, kPlBarRows + g, v);
                        keep_bits = mbits[q / NB][q % NB];
                    }
                {
                    const int pix_ = m ? pix[1] : pix[0];                      // pixel in the planes of the row
                    const bool row_ok = pix_ >= 0;                             // ... this thread owns
                    const int cc = 2 * jb + half;
                    if (cc >= nchunks) continue;
                    const int nb = n0 + cc * 32;                        // first channel of the chunk
#pragma unroll
                    for (int k = 0; k < 32; ++k) {
                        float t = v[k] + chan[cc * 32 + k];
                        if (P.act == EFFDET_ACT_RELU) t = fmaxf(t, 0.f);
                        else if (P.act == EFFDET_ACT_SIGMOID) t = sigmoidf_(t);
                        v[k] = t;
                    }
                    if (row_ok && L.residual) {
                        const int hw = L.H * L.W, b = pix_ / hw, pixb = pix_ - b * hw;        // image, pixel inside it
#pragma unroll
                        for (int k4 = 0; k4 < 8; ++k4) {
                            if (nb + k4 * 4 >= P.Cout) break;
                            const float4 rv = ldg4(L.residual + (long long)b * L.r_bstride + (long long)pixb * P.Cout + nb + k4 * 4);
                            v[k4 * 4] += rv.x; v[k4 * 4 + 1] += rv.y; v[k4 * 4 + 2] += rv.z; v[k4 * 4 + 3] += rv.w;
                        }
                    }
                    // gradient passes where the forward activation was > 0
                    if (L.mask_bits) {
                        const uint32_t keep = keep_bits;
#pragma unroll
                        for (int k = 0; k < 32; ++k)
                            if (!((keep >> k) & 1u)) v[k] = 0.f;
                    } else if (row_ok && L.mask_planes) {
                        const __nv_bfloat16* mh = L.mask_planes + (long long)pix_ * P.opitch + nb;
#pragma unroll
                        for (int k8 = 0; k8 < 4; ++k8) {
                            if (nb + k8 * 8 >= P.Cout) break;
                            const uint32_t keep = relu_bits8(__ldg(reinterpret_cast<const uint4*>(mh + k8 * 8)),
                                                             __ldg(reinterpret_cast<const uint4*>(mh + plane + k8 * 8)));
#pragma unroll
                            for (int e = 0; e < 8; ++e)
                                if (!((keep >> e) & 1u)) v[k8 * 8 + e] = 0.f;
                        }
                    }
                    if (!row_ok) {
#pragma unroll
                        for (int k = 0; k < 32; ++k) v[k] = 0.f;
                    }
                    if (row_ok && L.y) {
                        const int hw = L.H * L.W, b = pix_ / hw, pixb = pix_ - b * hw;
                        float* yo = L.y + (long long)b * L.y_bstride + (long long)pixb * P.Cout + nb;
#pragma unroll
                        for (int k4 = 0; k4 < 8; ++k4) {
                            if (nb + k4 * 4 >= P.Cout) break;
                            st4(yo + k4 * 4, make_float4(v[k4 * 4], v[k4 * 4 + 1], v[k4 * 4 + 2], v[k4 * 4 + 3]));
                        }
                    }
                    if (row_ok && L.y_planes) {
                        __nv_bfloat16* ph = L.y_planes + (long long)pix_ * P.opitch + nb;
                        uint32_t word = 0;                             // y_mask of the chunk: channel nb + k is bit k
#pragma unroll
                        for (int k8 = 0; k8 < 4; ++k8) {
                            if (nb + k8 * 8 >= P.Cout) break;
                            uint4 hi, lo;
                            split8(make_float4(v[k8 * 8], v[k8 * 8 + 1], v[k8 * 8 + 2], v[k8 * 8 + 3]),
                                   make_float4(v[k8 * 8 + 4], v[k8 * 8 + 5], v[k8 * 8 + 6], v[k8 * 8 + 7]), hi, lo);
                            *reinterpret_cast<uint4*>(ph + k8 * 8) = hi;
                            *reinterpret_cast<uint4*>(ph + plane + k8 * 8) = lo;
                            if (L.y_mask) word |= relu_bits8(hi, lo) << (8 * k8);
                        }
                        if (L.y_mask) L.y_mask[(long long)pix_ * P.mwords + (nb >> 5)] = word;
                    }
                    if (P.colsum) {
                        // warp transpose-reduce: afterwards v[0] of lane j is the sum over the warp's 32 rows of column j
                        transpose_add<16>(v, lane);
                        transpose_add<8>(v, lane);
                        transpose_add<4>(v, lane);
                        transpose_add<2>(v, lane);
                        transpose_add<1>(v, lane);
                        if (nb + lane < P.Cout) atomicAdd(csum + nb + lane, v[0]);
                    }
                }
            }
        }
        if (P.colsum) {
            named_bar_sync(kPlBarSums, 256);                           // both warpgroups' sums are in csum
            for (int i = threadIdx.x; i < P.Cout; i += 256) atomicAdd(P.colsum + i, csum[i]);
        }
    }
}

// fp32 [B][HW][C] (image stride bstride) -> bf16 hi/lo planes [2][B*HW][pitch]; optionally multiplied by p*(1-p) of a
// second tensor (sigmoid backward, models/retinahead.py:121) and optionally reduced into per-channel column sums (the
// bias gradient) on the way -- one read of the gradient instead of three passes
__global__ void __launch_bounds__(256) to_planes_kernel(const float* __restrict__ x, long long x_bstride, const float* __restrict__ prob,
                                                        long long p_bstride, __nv_bfloat16* __restrict__ out, float* __restrict__ colsum,
                                                        int B, int HW, int C, int pitch, int rows_per_block) {
    __shared__ float red[256 * 8];
    const int cv8 = pitch / 8;
    const int cvb = cv8 < 256 ? cv8 : 256;
    const int rows = 256 / cvb;
    const int tr = threadIdx.x / cvb, tc = threadIdx.x - tr * cvb;
    const int j = blockIdx.y * cvb + tc;
    const bool active = tr < rows && j < cv8;
    const long long nrows = (long long)B * HW;
    const long long plane = nrows * pitch;
    float s[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) s[i] = 0.f;
    if (active) {
        const int c = j * 8;
        const long long r_begin = (long long)blockIdx.x * rows_per_block;
        const long long r_end = min(nrows, r_begin + rows_per_block);
        for (long long row = r_begin + tr; row < r_end; row += rows) {
            const int b = (int)(row / HW);
            const long long pix = row - (long long)b * HW;
            float4 v0 = f4zero(), v1 = f4zero();
            if (c < C) {
                const float* q = x + (long long)b * x_bstride + pix * C + c;
                v0 = ldg4(q);
                if (c + 4 < C) v1 = ldg4(q + 4);
                if (prob) {
                    const float* pp = prob + (long long)b * p_bstride + pix * C + c;
                    const float4 p0 = ldg4(pp);
                    v0 = make_float4(v0.x * p0.x * (1.f - p0.x), v0.y * p0.y * (1.f - p0.y), v0.z * p0.z * (1.f - p0.z),
                                     v0.w * p0.w * (1.f - p0.w));
                    if (c + 4 < C) {
                        const float4 p1 = ldg4(pp + 4);
                        v1 = make_float4(v1.x * p1.x * (1.f - p1.x), v1.y * p1.y * (1.f - p1.y), v1.z * p1.z * (1.f - p1.z),
                                         v1.w * p1.w * (1.f - p1.w));
                    }
                }
            }
            uint4 hi, lo;
            split8(v0, v1, hi, lo);
            *reinterpret_cast<uint4*>(out + row * pitch + c) = hi;
            *reinterpret_cast<uint4*>(out + plane + row * pitch + c) = lo;
            s[0] += v0.x; s[1] += v0.y; s[2] += v0.z; s[3] += v0.w;
            s[4] += v1.x; s[5] += v1.y; s[6] += v1.z; s[7] += v1.w;
        }
    }
    if (colsum == nullptr) return;
#pragma unroll
    for (int i = 0; i < 8; ++i) red[threadIdx.x * 8 + i] = s[i];
    __syncthreads();
    if (tr == 0 && j < cv8) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            float acc = 0.f;
            for (int rr = 0; rr < rows; ++rr) acc += red[(rr * cvb + tc) * 8 + i];
            const int c = j * 8 + i;
            if (c < C) atomicAdd(colsum + c, acc);
        }
    }
}

int to_planes_launch(const float* x, long long x_bstride, const float* prob, long long p_bstride, void* out, float* colsum,
                     int B, int HW, int C, int pitch, cudaStream_t st) {
    const int cv8 = pitch / 8;
    const int cvb = cv8 < 256 ? cv8 : 256;
    const int rows = 256 / cvb;
    const long long nrows = (long long)B * HW;
    const int ychunks = cdiv(cv8, cvb);
    long long rpb;
    if (colsum) {           // ~4 waves of blocks, at least 8 row iterations each: few atomics per column
        rpb = (nrows + num_sms() * 4 - 1) / (num_sms() * 4);
        if (rpb < (long long)rows * 8) rpb = (long long)rows * 8;
    } else {                // nothing to amortise: up to 16 blocks per SM, down to one row iteration each
        rpb = (nrows * ychunks + num_sms() * 16 - 1) / (num_sms() * 16);
        if (rpb < rows) rpb = rows;
    }
    dim3 grid(cdiv(nrows, rpb), ychunks);
    to_planes_kernel<<<grid, 256, 0, st>>>(x, x_bstride, prob, p_bstride, (__nv_bfloat16*)out, colsum, B, HW, C, pitch, (int)rpb);
    return launch_status("to_planes_kernel");
}

}  // namespace effdet

using namespace effdet;

extern "C" int effdet_to_planes(const float* x, int64_t x_bstride, const float* prob, int64_t p_bstride, void* planes,
                                float* colsum, int B, int HW, int C, int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(x && planes && B > 0 && HW > 0 && C > 0 && C % 4 == 0, "to_planes: bad arguments");
    EFFDET_REQUIRE(aligned16(x) && aligned16(prob) && aligned16(planes) && x_bstride % 4 == 0 && p_bstride % 4 == 0,
                   "to_planes: alignment");
    EFFDET_DEVICE(device);
    return to_planes_launch(x, x_bstride, prob, p_bstride, planes, colsum, B, HW, C, (C + 7) / 8 * 8, (cudaStream_t)stream);
}

extern "C" int effdet_conv_planes_multi(const effdet_conv_planes_args* levels, int nlevels, int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(levels && nlevels >= 1 && nlevels <= kPlMaxLevels, "conv_planes_multi: 1..%d levels", kPlMaxLevels);
    const effdet_conv_planes_args* a0 = &levels[0];
    EFFDET_REQUIRE(!a0->tc_single || a0->ksize == 3, "conv_planes_multi: tc_single is defined for 3x3 convolutions only (ksize %d)",
                   a0->ksize);
    for (int l = 1; l < nlevels; ++l)
        EFFDET_REQUIRE(levels[l].tc_single == a0->tc_single, "conv_planes_multi: levels disagree on tc_single");
    EFFDET_REQUIRE(a0->w_tc && (a0->ksize == 1 || a0->ksize == 3) && a0->Cin % 4 == 0 && a0->Cout % 4 == 0 && a0->Cin >= 8 &&
                       a0->Cout >= 8,
                   "conv_planes_multi: needs the bf16 weight pack, k in {1,3}, channels %% 4 == 0");
    // 128 x 128 tiles at most: the accumulator lives in the consumer warpgroups' registers (64 per thread)
    const int BN = a0->Cout <= 64 ? 64 : 128;
    const size_t smem = (BN == 64 ? PlCfg<64>::kSmem : PlCfg<128>::kSmem) + (a0->colsum ? 4 * (size_t)a0->Cout : 0);
    EFFDET_REQUIRE(smem <= kPlSmemOptin, "conv_planes_multi: column sums of %d channels do not fit in shared memory", a0->Cout);
    for (int l = 0; l < nlevels; ++l) {
        const effdet_conv_planes_args* a = &levels[l];
        EFFDET_REQUIRE(!(a->mask_planes && a->mask_bits), "conv_planes_multi: level %d passes both mask_planes and mask_bits", l);
        EFFDET_REQUIRE(!a->y_mask || (a->y_planes && a->act == EFFDET_ACT_RELU),
                       "conv_planes_multi: y_mask is written by a ReLU forward that stores planes (level %d)", l);
    }
    EncodeTiledFn enc = encode_fn();
    if (!enc) return fail(EFFDET_ERR_UNSUPPORTED, "conv_planes_multi: cuTensorMapEncodeTiled unavailable");
    EFFDET_DEVICE(device);
    PlMaps maps;
    PlArgs P;
    memset(&P, 0, sizeof(P));
    const int opitch = (a0->Cout + 7) / 8 * 8, ipitch = (a0->Cin + 7) / 8 * 8;
    int tiles = 0;
    for (int l = 0; l < nlevels; ++l) {
        const effdet_conv_planes_args* a = &levels[l];
        EFFDET_REQUIRE(a->x_planes && (a->y || a->y_planes), "conv_planes_multi: null tensor");
        EFFDET_REQUIRE(a->B > 0 && a->H > 0 && a->W > 0 && (long long)a->B * a->H * a->W <= INT_MAX,
                       "conv_planes_multi: a %dx%dx%d map has more than 2^31 - 1 pixels", a->B, a->H, a->W);
        EFFDET_REQUIRE(a->Cin == a0->Cin && a->Cout == a0->Cout && a->ksize == a0->ksize && a->act == a0->act && a->w_tc == a0->w_tc &&
                           a->bias == a0->bias && a->colsum == a0->colsum,
                       "conv_planes_multi: all levels must share weights, bias, channels and activation");
        EFFDET_REQUIRE(aligned16(a->x_planes) && aligned16(a->y) && aligned16(a->y_planes) && aligned16(a->mask_planes) &&
                           aligned16(a->residual) && a->y_bstride % 4 == 0 && a->r_bstride % 4 == 0 &&
                           (reinterpret_cast<uintptr_t>(a->y_mask) & 3u) == 0 && (reinterpret_cast<uintptr_t>(a->mask_bits) & 3u) == 0,
                       "conv_planes_multi: alignment");
        PlLevel& L = P.lv[l];
        L.B = a->B; L.H = a->H; L.W = a->W;
        if (!wg_geometry(a->B, a->H, a->W, &L.g))
            return fail(EFFDET_ERR_UNSUPPORTED, "conv_planes_multi: a %dx%dx%d map has no legal pixel box (check effdet_wgrad_tc_geometry_ok)",
                        a->B, a->H, a->W);
        L.nboxes = L.g.nbx * L.g.nby * L.g.nbb;
        L.tile_begin = tiles;
        tiles += cdiv(L.nboxes, 128 / L.g.kstage);
        L.y = a->y; L.y_bstride = a->y_bstride;
        L.y_planes = (__nv_bfloat16*)a->y_planes;
        L.mask_planes = (const __nv_bfloat16*)a->mask_planes;
        L.y_mask = (uint32_t*)a->y_mask;
        L.mask_bits = (const uint32_t*)a->mask_bits;
        L.residual = a->residual; L.r_bstride = a->r_bstride;
        int s = planes_map(enc, &maps.x[l], const_cast<void*>(a->x_planes), a->B, a->H, a->W, a->Cin, ipitch, L.g);
        if (s) return s;
    }
    for (int l = nlevels; l < kPlMaxLevels; ++l) {
        maps.x[l] = maps.x[0];
        P.lv[l].tile_begin = tiles;
    }
    const int taps = a0->ksize * a0->ksize;
    const int kpad = conv_tc_kpad(a0->Cin);
    CUtensorMap wmap;
    const int s = kmajor_planes_map(enc, &wmap, a0->w_tc, a0->Cout, taps * kpad, BN);
    if (s) return s;
    P.nlevels = nlevels;
    P.ntn = cdiv(a0->Cout, BN);
    P.total_tiles = tiles * P.ntn;
    P.Cin = a0->Cin; P.Cout = a0->Cout; P.ksize = a0->ksize; P.act = a0->act;
    P.kblocks = kpad / 64;
    P.opitch = opitch;
    P.mwords = (a0->Cout + 31) / 32;
    P.bias = a0->bias;
    P.colsum = a0->colsum;
    const int grid = P.total_tiles < num_sms() ? P.total_tiles : num_sms();
    cudaStream_t st = (cudaStream_t)stream;
    if (a0->tc_single) {
        if (BN == 64) return launch_smem("conv_planes_kernel", conv_planes_kernel<64, 1>, grid, kPlThreads, smem, st, maps, wmap, P);
        return launch_smem("conv_planes_kernel", conv_planes_kernel<128, 1>, grid, kPlThreads, smem, st, maps, wmap, P);
    }
    if (BN == 64) return launch_smem("conv_planes_kernel", conv_planes_kernel<64, 3>, grid, kPlThreads, smem, st, maps, wmap, P);
    return launch_smem("conv_planes_kernel", conv_planes_kernel<128, 3>, grid, kPlThreads, smem, st, maps, wmap, P);
}
