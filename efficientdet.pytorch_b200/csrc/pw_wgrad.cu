// Weight gradient of the 1x1 convolutions of the MBConv block (models/efficientnet.py:85 expand, :96 project; reached
// through autograd's cuDNN bwd-filter in the reference), straight from the fp32 tensors:
//     dW[n][c] += sum_m dy[m][n] * xt[m][c],      xt = swish(x*in_scale+in_shift) * a_scale[image]   (both optional)
// The TMA-fed kernel in conv_tc.cu wants both operands pre-split into bf16 hi/lo planes; for these layers that would
// cost a split pass over x (after the BN+swish+SE-gate prologue) and one over dy -- each a full read + write of an
// expanded activation -- before the GEMM read them a third time.  Here eight converter warps read the fp32 rows with 128-bit
// coalesced loads, apply the prologue in registers, split to bf16 hi/lo and write the operand tiles in the
// SWIZZLE_128B "MN-major" layout (row = pixel, 128 bytes = 64 channels) the tensor-map loads would have produced; two
// consumer warpgroups (64 output channels each) issue the bf16x3 wgmma (GEMM-K = pixels, M = output channels, N = input
// channels, accumulator in registers) and add their partials to dW with vector reductions straight from the fragments.  Every operand byte is read from HBM
// once: algorithmic bytes = 4*M*(Cin + Cout) (dy pre-split by the depthwise backward kernel: same 4 bytes / element).
#include "tc_ptx.cuh"

#include <cstring>

namespace effdet {

// Threads: warps 0-7 are the two consumer warpgroups, warps 8-15 the converters, each holding kWgUnits 32-byte units of
// a stage twice over (the loads of chunk k+1 are in flight while chunk k is converted).  512 threads leave 128
// registers per thread: no variable may spill, it would share its scoreboard with the prefetched loads.
constexpr int kWgConv = 8, kWgUnits = 3;
constexpr int kWgCT = kWgConv * 32, kWgThreads = 256 + kWgCT;

struct PwWgParams {
    const float* x;
    const float* dy;
    const uint16_t* dy_planes;      // [2][M][Cout] bf16 or NULL
    const float* in_scale;
    const float* in_shift;
    const float* a_scale;
    float* dw;
    int M, HW, Cin, Cout;
    int ntn, NX, TM;                // input-channel tiles, their width (multiple of 16, <= 128), output channels per tile (<= 128)
    int K;                          // pixels per stage: 16 .. 128, the largest whose units fit the converter threads
    int nchunks, cps;               // K-pixel chunks, chunks per split
    int NS, stage_bytes;            // ring depth, bytes per stage
    int a_plane, b_plane;           // bytes of one dy / x plane of a stage (1 or 2 groups of 64 channels)
};

__device__ __forceinline__ void red_add_v2(float* p, float a, float b) {
    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}

__device__ __forceinline__ void sts128(uint32_t addr, const uint4 v) {
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w));
}

template <int NB>            // 64-channel groups of the input-channel tile
__global__ void __launch_bounds__(kWgThreads, 1) pw_wgrad_kernel(const __grid_constant__ PwWgParams P) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);    // 1024-byte aligned, still a shared pointer
    uint8_t* ctl = smem + P.NS * P.stage_bytes;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(ctl);
    uint64_t* empty_bar = full_bar + 4;
    float* chan = reinterpret_cast<float*>(ctl + 128);          // in_scale | in_shift of this tile's channels

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tn = blockIdx.x % P.ntn, tm = blockIdx.x / P.ntn;
    const int c0 = tn * P.NX, n0 = tm * P.TM;
    const int ncur = min(P.NX, P.Cin - c0);                     // real input channels of this tile (multiple of 8)
    const int mcur = min(P.TM, P.Cout - n0);                    // real output channels
    const int ch_begin = blockIdx.y * P.cps;
    const int KT = min(P.nchunks, ch_begin + P.cps) - ch_begin;
    const int group = P.K * 128;                                // bytes of one 64-channel group of one plane

    if (threadIdx.x == 0) {
        for (int s = 0; s < P.NS; ++s) {
            mbar_init(&full_bar[s], kWgConv);
            mbar_init(&empty_bar[s], 8);     // one arrival per consumer warp
        }
        fence_barrier_init();
    }
    if (P.in_scale)
        for (int i = threadIdx.x; i < ncur; i += kWgThreads) {
            chan[i] = __ldg(P.in_scale + c0 + i);
            chan[256 + i] = __ldg(P.in_shift + c0 + i);
        }
    __syncthreads();

    if (warp >= 8) {
        // This thread's units: the same (pixel row, channel octet) of every chunk; unit i is an x unit (bit i of xmask),
        // a dy unit (bit i of ymask) or nothing.  Everything that changes from chunk to chunk is advanced by additions.
        const int nxo = ncur >> 3, nyo = mcur >> 3;
        const int UX = P.K * nxo, U = UX + P.K * nyo;
        const bool planes = P.dy_planes != nullptr;
        const uint32_t smem_a = smem_u32(smem);
        uint32_t xmask = 0, ymask = 0;
        const char* src[kWgUnits];          // first 16 bytes of the unit in chunk kt (advanced every load)
        uint32_t dst[kWgUnits];             // shared address of the hi half in stage 0
        int pix[kWgUnits];                  // global pixel of the unit in the chunk being LOADED
        int cof[kWgUnits];                  // x units: channel offset inside the tile
        const float* gate[kWgUnits];        // x units: a_scale row of the image the CONVERTED pixel belongs to
        int rem[kWgUnits];                  //          ... and the pixel's index inside that image
#pragma unroll
        for (int i = 0; i < kWgUnits; ++i) {
            const int u = threadIdx.x - 256 + i * kWgCT;
            src[i] = nullptr; dst[i] = 0; pix[i] = 0; cof[i] = 0; gate[i] = nullptr; rem[i] = 0;
            if (u < UX) {
                const int p = u / nxo, o = u - p * nxo;
                xmask |= 1u << i;
                pix[i] = ch_begin * P.K + p;
                cof[i] = o * 8;
                src[i] = reinterpret_cast<const char*>(P.x + (size_t)pix[i] * P.Cin + c0 + o * 8);
                dst[i] = smem_a + 2 * P.a_plane + (o >> 3) * group + p * 128 + (((o & 7) ^ (p & 7)) << 4);
                if (P.a_scale) {
                    const int b = pix[i] / P.HW;
                    rem[i] = pix[i] - b * P.HW;
                    gate[i] = P.a_scale + (size_t)b * P.Cin + c0 + o * 8;
                }
            } else if (u < U) {
                const int v = u - UX;
                const int p = v / nyo, o = v - p * nyo;
                ymask |= 1u << i;
                pix[i] = ch_begin * P.K + p;
                const size_t e = (size_t)pix[i] * P.Cout + n0 + o * 8;
                src[i] = planes ? reinterpret_cast<const char*>(P.dy_planes + e) : reinterpret_cast<const char*>(P.dy + e);
                dst[i] = smem_a + (o >> 3) * group + p * 128 + (((o & 7) ^ (p & 7)) << 4);
            }
        }
        const size_t step_x = (size_t)P.K * P.Cin * 4, step_y = (size_t)P.K * P.Cout * (planes ? 2 : 4);
        const size_t second_y = planes ? (size_t)P.M * P.Cout * 2 : 16;       // hi -> lo plane of dy, or the next 4 floats
        const bool have_in = P.in_scale != nullptr, have_gate = P.a_scale != nullptr;
        float4 va[2][kWgUnits], vb[2][kWgUnits];
        uint32_t okmask[2] = {0, 0};                                          // units of the buffered chunk inside the tensor
        auto load = [&](float4 (&a)[kWgUnits], float4 (&b)[kWgUnits], uint32_t& ok) {
            ok = 0;
#pragma unroll
            for (int i = 0; i < kWgUnits; ++i) {
                a[i] = b[i] = f4zero();
                const bool isx = (xmask >> i) & 1, isy = (ymask >> i) & 1;
                if ((isx || isy) && pix[i] < P.M) {
                    ok |= 1u << i;
                    a[i] = __ldg(reinterpret_cast<const float4*>(src[i]));
                    b[i] = __ldg(reinterpret_cast<const float4*>(src[i] + (isx ? (size_t)16 : second_y)));
                }
                src[i] += isx ? step_x : step_y;
                pix[i] += P.K;
            }
        };
        auto convert = [&](int kt, float4 (&a)[kWgUnits], float4 (&b)[kWgUnits], const uint32_t ok) {
            const int s = kt % P.NS;
            if (lane == 0) mbar_wait(&empty_bar[s], ((kt / P.NS) & 1) ^ 1);   // the MMAs that last read the slot are done
            __syncwarp();
            const uint32_t so = (uint32_t)s * (uint32_t)P.stage_bytes;
#pragma unroll
            for (int i = 0; i < kWgUnits; ++i) {
                uint4 hi, lo;
                if ((xmask >> i) & 1) {
                    float4 xa = a[i], xb = b[i];
                    if ((ok >> i) & 1) {
                        if (have_in) {
                            const float* cs = chan + cof[i];
                            xa = f4fma(xa, *reinterpret_cast<const float4*>(cs), *reinterpret_cast<const float4*>(cs + 256));
                            xb = f4fma(xb, *reinterpret_cast<const float4*>(cs + 4), *reinterpret_cast<const float4*>(cs + 260));
                            xa = make_float4(fswish(xa.x), fswish(xa.y), fswish(xa.z), fswish(xa.w));
                            xb = make_float4(fswish(xb.x), fswish(xb.y), fswish(xb.z), fswish(xb.w));
                        }
                        if (have_gate) {
                            xa = f4mul(xa, ldg4(gate[i]));
                            xb = f4mul(xb, ldg4(gate[i] + 4));
                        }
                    }
                    if (have_gate) {                                          // move on to the pixel of the next chunk
                        rem[i] += P.K;
                        while (rem[i] >= P.HW) { rem[i] -= P.HW; gate[i] += P.Cin; }
                    }
                    split8(xa, xb, hi, lo);
                    sts128(dst[i] + so, hi);
                    sts128(dst[i] + so + P.b_plane, lo);
                } else if ((ymask >> i) & 1) {
                    if (planes) {
                        hi = *reinterpret_cast<const uint4*>(&a[i]);
                        lo = *reinterpret_cast<const uint4*>(&b[i]);
                    } else {
                        split8(a[i], b[i], hi, lo);
                    }
                    sts128(dst[i] + so, hi);
                    sts128(dst[i] + so + P.a_plane, lo);
                }
            }
            fence_proxy_async();
            __syncwarp();
            if (lane == 0) mbar_arrive(&full_bar[s]);
        };
        // software pipeline: the loads of chunk kt+1 are in flight while chunk kt is converted
        load(va[0], vb[0], okmask[0]);
        for (int kt = 0; kt < KT; kt += 2) {
            if (kt + 1 < KT) load(va[1], vb[1], okmask[1]);
            convert(kt, va[0], vb[0], okmask[0]);
            if (kt + 1 < KT) {
                if (kt + 2 < KT) load(va[0], vb[0], okmask[0]);
                convert(kt + 1, va[1], vb[1], okmask[1]);
            }
        }
    } else {
        // consumer warpgroup g: output channels n0 + 64g .. + 63.  A dy tile of at most 64 channels keeps ONE group in
        // shared memory; warpgroup 1 then multiplies the same group again and its rows are never stored.
        const int g = warp >> 2, w = warp & 3;
        const uint32_t a_off = P.a_plane > group ? (uint32_t)(g * group) : 0u;
        float d[NB][32];
        with_count<1, 2, 4, 8>(P.K / 16, [&](auto ksteps) {         // P.K is 16, 32, 64 or 128 pixels
            for (int kt = 0; kt < KT; ++kt) {
                const int s = kt % P.NS;
                const uint32_t ph = (kt / P.NS) & 1;
                mbar_wait(&full_bar[s], ph);
                const uint32_t a_hi = smem_u32(smem + (size_t)s * P.stage_bytes) + a_off;
                const uint32_t b_hi = smem_u32(smem + (size_t)s * P.stage_bytes) + 2 * P.a_plane;
                wg_mma_mn_steps<ksteps, 3>(d,a_hi, a_hi + P.a_plane, b_hi, b_hi + P.b_plane, group, kt != 0);
                wgmma_commit();
                wgmma_wait<1>();                               // the previous stage is no longer read
                if (kt > 0 && lane == 0) mbar_arrive(&empty_bar[(kt - 1) % P.NS]);
            }
            wgmma_wait<0>();
        });
        // fragment element i: output channel 16w + lane/4 + 8*((i>>1)&1), input channels 8*(i>>2) + 2*(lane&3) + {0,1}
#pragma unroll
        for (int jb = 0; jb < NB; ++jb)
#pragma unroll
            for (int i = 0; i < 32; i += 2) {
                const int r = 64 * g + 16 * w + (lane >> 2) + 8 * ((i >> 1) & 1);
                const int c = 64 * jb + 8 * (i >> 2) + 2 * (lane & 3);
                if (r < mcur && c < ncur) red_add_v2(P.dw + (size_t)(n0 + r) * P.Cin + c0 + c, d[jb][i], d[jb][i + 1]);
            }
    }
}

int pw_wgrad_launch(const effdet_wgrad_args* a, cudaStream_t st) {
    PwWgParams P;
    memset(&P, 0, sizeof(P));
    P.x = a->x;
    P.dy = a->dy;
    P.dy_planes = reinterpret_cast<const uint16_t*>(a->dy_planes);
    P.in_scale = a->in_scale;
    P.in_shift = a->in_shift;
    P.a_scale = a->a_scale;
    P.dw = a->dw;
    P.HW = a->H * a->W;
    P.M = a->B * P.HW;
    P.Cin = a->Cin;
    P.Cout = a->Cout;
    // balanced tiles: input channels in pieces of <= 128 (multiple of 16), output channels in pieces of <= 128 (multiple
    // of 8).  Every output-channel tile reads x again, every input-channel tile reads dy again -- wide tiles keep that small;
    // 128 x 128 is what the consumer warpgroups' registers hold.
    P.ntn = cdiv(a->Cin, 128);
    P.NX = cdiv(cdiv(a->Cin, P.ntn), 16) * 16;
    P.ntn = cdiv(a->Cin, P.NX);
    int ntm = cdiv(a->Cout, 128);
    P.TM = cdiv(cdiv(a->Cout, ntm), 8) * 8;
    ntm = cdiv(a->Cout, P.TM);
    const int tiles = P.ntn * ntm;
    const int octs = (P.NX < a->Cin ? P.NX : a->Cin) / 8 + P.TM / 8;
    const int capacity = kWgCT * kWgUnits;                       // units one stage may hold
    P.K = 128;
    while (P.K > 16 && P.K * octs > capacity) P.K >>= 1;
    if (P.K * octs > capacity) return fail(EFFDET_ERR_UNSUPPORTED, "wgrad(pw): tile does not fit");   // (octs <= 32: 16 * 32 = 512 always fits)
    P.nchunks = cdiv(P.M, P.K);
    // split-K: one wave of CTAs, more when a CTA would accumulate more than kWgMaxPixelsPerSplit pixels (then whole
    // waves).  tests/test_benchmark_plans.py (_pw_plan) mirrors this arithmetic.
    int splits = num_sms() / tiles;
    if (splits < 1) splits = 1;
    const int need = cdiv(P.nchunks, kWgMaxPixelsPerSplit / P.K);
    if (splits < need) splits = cdiv(need * tiles, num_sms()) * num_sms() / tiles;
    if (splits > P.nchunks) splits = P.nchunks;
    P.cps = cdiv(P.nchunks, splits);
    splits = cdiv(P.nchunks, P.cps);
    const int group = P.K * 128;
    P.a_plane = cdiv(P.TM, 64) * group;
    P.b_plane = cdiv(P.NX, 64) * group;
    P.stage_bytes = 2 * P.a_plane + 2 * P.b_plane;
    P.NS = (200 * 1024) / P.stage_bytes;
    if (P.NS > 4) P.NS = 4;
    const size_t smem = (size_t)P.NS * P.stage_bytes + 128 + 2 * 256 * sizeof(float) + 1024;
    if (P.NX > 64) return launch_smem("pw_wgrad_kernel", pw_wgrad_kernel<2>, dim3(tiles, splits), kWgThreads, smem, st, P);
    return launch_smem("pw_wgrad_kernel", pw_wgrad_kernel<1>, dim3(tiles, splits), kWgThreads, smem, st, P);
}

}  // namespace effdet
