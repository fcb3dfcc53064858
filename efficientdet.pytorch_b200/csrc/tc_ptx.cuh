// PTX wrappers shared by the wgmma / TMA kernels (conv_tc.cu, conv_planes.cu, pw_gemm.cu): mbarrier, TMA loads and
// stores, warpgroup MMA and its shared-memory descriptors.  sm_90a.
#pragma once
#include "common.cuh"

#include <cuda.h>
#include <cuda_bf16.h>
#include <stddef.h>
#include <type_traits>

namespace effdet {

// Most pixels (GEMM-K) one weight-gradient CTA accumulates in its wgmma fp32 accumulator: 64 chunks of 64 pixels.  That
// accumulation's error grows linearly with the K range it covers (H100, bf16x3, whole-tensor norm-relative: 4.5e-6 at
// <= 768 pixels, 1.0e-5 at 2 752, 1.9e-5 at 5 504, 3.8e-5 at 10 944), so longer ranges are split further and added by
// atomics.  Both weight-gradient launchers read it: conv_tc.cu and pw_wgrad.cu.
constexpr int kWgMaxPixelsPerSplit = 4096;

// ---------------------------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    const uint32_t a = smem_u32(bar);
    uint32_t done;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(a), "r"(parity)
            : "memory");
    } while (!done);
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}

__device__ __forceinline__ void tma_load_5d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3, int c4) {
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
        : "memory");
}

// ---- warpgroup MMA (sm_90a wgmma.mma_async) ---------------------------------------------------------------------------
// A warpgroup (4 consecutive warps starting at a multiple of 4) owns a 64-row slice of the 128-row tile and accumulates
// it in registers, one float[32] per 64x64 block.  Element i of a block held by thread (warp w of the group, lane l):
//   row 16*w + l/4 + 8*((i>>1)&1),  column 8*(i>>2) + 2*(l&3) + (i&1).

// Shared-memory matrix descriptor, SWIZZLE_128B (cute::GMMA::DescriptorSm90):
//   bits [0,14) start >> 4 | [16,30) LBO >> 4 | [32,46) SBO >> 4 | [62,64) layout = 1 (128B swizzle)
__device__ __forceinline__ uint64_t gmma_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return (uint64_t)((smem_addr >> 4) & 0x3FFF) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) |
           ((uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32) | (1ull << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// D[64 x 64NB] (+)= A[64x16] * B[16 x 64NB] in ONE wgmma (m64n64k16, m64n128k16 or m64n256k16), bf16 inputs from shared
// memory, fp32 accumulation in registers.  The accumulator of an m64nNk16 is the NB 64x64 blocks above side by side:
// registers 32j .. 32j+31 of the instruction are d[j].  MN = 0: K-major operands, MN = 1: MN-major operands (A and B).
#define EFFDET_WG_D8(a, o) "+f"(a[o]), "+f"(a[o + 1]), "+f"(a[o + 2]), "+f"(a[o + 3]), "+f"(a[o + 4]), "+f"(a[o + 5]), \
                           "+f"(a[o + 6]), "+f"(a[o + 7])
#define EFFDET_WG_D32(a) EFFDET_WG_D8(a, 0), EFFDET_WG_D8(a, 8), EFFDET_WG_D8(a, 16), EFFDET_WG_D8(a, 24)
template <int MN>
__device__ __forceinline__ void wgmma_bf16(float (&d)[1][32], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
        "}, %32, %33, p, 1, 1, %35, %35;\n\t}"
        : EFFDET_WG_D32(d[0])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate), "n"(MN)
        : "memory");
}
template <int MN>
__device__ __forceinline__ void wgmma_bf16(float (&d)[2][32], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
        "}, %64, %65, p, 1, 1, %67, %67;\n\t}"
        : EFFDET_WG_D32(d[0]), EFFDET_WG_D32(d[1])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate), "n"(MN)
        : "memory");
}
template <int MN>
__device__ __forceinline__ void wgmma_bf16(float (&d)[4][32], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
        "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
        "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
        "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
        "}, %128, %129, p, 1, 1, %131, %131;\n\t}"
        : EFFDET_WG_D32(d[0]), EFFDET_WG_D32(d[1]), EFFDET_WG_D32(d[2]), EFFDET_WG_D32(d[3])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate), "n"(MN)
        : "memory");
}
#undef EFFDET_WG_D32
#undef EFFDET_WG_D8
// One K16 step over all NB*64 columns with P bf16 products per multiply-add (P = 3 is the default, bf16x3 precision;
// P = 1 is EFFDET_B200_PRECISION=bf16 on the dense 3x3 convs), one full-width wgmma per product:
//   P = 3  split precision, lo*hi + hi*lo + hi*hi (x ~= hi + lo), every accumulator element sums them in that order
//   P = 1  single pass, hi*hi only (the lo planes are not read)
// a_*: this warpgroup's 64-row slice.  The descriptor locates the B operand's 64-column blocks: 8 * sbo bytes apart
// for K-major operands (64 rows of 128 bytes), lbo bytes apart for MN-major ones.
template <int NB, int MN, int P>
__device__ __forceinline__ void wg_mma(float (&d)[NB][32], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo,
                                       uint32_t lbo, uint32_t sbo, uint32_t accumulate) {
    static_assert(P == 1 || P == 3, "one or three bf16 products per multiply-add");
    if constexpr (P == 3) {
        const uint64_t dah = gmma_desc(a_hi, lbo, sbo), dal = gmma_desc(a_lo, lbo, sbo);
        const uint64_t dbh = gmma_desc(b_hi, lbo, sbo), dbl = gmma_desc(b_lo, lbo, sbo);
        wgmma_bf16<MN>(d, dal, dbh, accumulate);
        wgmma_bf16<MN>(d, dah, dbl, 1);
        wgmma_bf16<MN>(d, dah, dbh, 1);
    } else {
        wgmma_bf16<MN>(d, gmma_desc(a_hi, lbo, sbo), gmma_desc(b_hi, lbo, sbo), accumulate);
    }
}
// KS K16 steps of one stage of MN-major operands (the weight gradients: GEMM-K = pixel rows, a K16 step is two 8-row
// groups, SBO = 1024 bytes apart; 64-channel groups `group` bytes apart), fully unrolled, P products per multiply-add.
template <int KS, int P, int NB>
__device__ __forceinline__ void wg_mma_mn_steps(float (&d)[NB][32], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo,
                                                uint32_t group, uint32_t accumulate) {
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < KS; ++k) {
        const uint32_t ko = k * 2 * 1024;
        wg_mma<NB, 1, P>(d, a_hi + ko, a_lo + ko, b_hi + ko, b_lo + ko, group, 1024, accumulate | k);
    }
}
// Calls f(std::integral_constant<int, n>()) for the one count among KS... that equals n: a warp-uniform branch into one
// body per count, so that the K16 steps of a stage (a runtime count) are fully unrolled.  ptxas has to see every
// wgmma of a loop over stages in straight-line code; with a runtime trip count or a branch between the wgmma groups
// of consecutive stages it fences the accumulator registers (C7519) or serialises the wgmma (C7520).  So the branch
// goes around the whole loop over stages.
template <int... KS, class F>
__device__ __forceinline__ void with_count(const int n, F&& f) {
    (void)((n == KS && (f(std::integral_constant<int, KS>()), true)) || ...);
}

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
// per-thread register count of the calling warpgroup, lowered or raised at run time (all its warps execute it)
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}
// counts the calling warp towards named barrier `id` without waiting for it; threads in bar.sync complete it
__device__ __forceinline__ void named_bar_arrive(int id, int nthreads) {
    asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// Row layout of an accumulator block for the epilogues: thread (warp w of warpgroup g, lane l) receives row
// (w & 1) * 32 + l of g's 64x64 block, columns (w >> 1) * 32 .. + 31.  The NWG warpgroups of the CTA take turns on one
// 64 x kRowsPitch staging buffer; named barrier 1 spans all of them, 2 + g one warpgroup.
constexpr int kRowsPitch = 68;                      // floats per staged row: 16-byte rows, conflict-free row reads
constexpr int kRowsBytes = 64 * kRowsPitch * 4;
template <int NWG>
__device__ __forceinline__ void wg_rows(const float (&d)[32], float* buf, const int g, float (&out)[32]) {
    const int w = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
#pragma unroll 1
    for (int turn = 0; turn < NWG; ++turn) {
        named_bar_sync(1, NWG * 128);
        if (turn != g) continue;
#pragma unroll
        for (int i = 0; i < 32; i += 2) {
            const int row = 16 * w + (lane >> 2) + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + 2 * (lane & 3);
            *reinterpret_cast<float2*>(buf + row * kRowsPitch + col) = make_float2(d[i], d[i + 1]);
        }
        named_bar_sync(2 + g, 128);
        const float* src = buf + ((w & 1) * 32 + lane) * kRowsPitch + (w >> 1) * 32;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const float4 v = *reinterpret_cast<const float4*>(src + 4 * q);
            out[4 * q] = v.x; out[4 * q + 1] = v.y; out[4 * q + 2] = v.z; out[4 * q + 3] = v.w;
        }
    }
}
// The same row layout for a warpgroup whose epilogue runs out of phase with the other's (conv_planes_kernel's
// ping-pong schedule): each warpgroup owns a 32 x kRowsPitch buffer (two of them take kRowsBytes) and named barrier
// `bar`, and passes the 64x64 block through it in two halves of 32 rows.  Warps 2h, 2h+1 of the group write half h,
// warps h, h+2 read it.
__device__ __forceinline__ void wg_rows_own(const float (&d)[32], float* buf, const int bar, float (&out)[32]) {
    const int w = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
#pragma unroll 1
    for (int h = 0; h < 2; ++h) {
        named_bar_sync(bar, 128);                   // the previous half has been read
        if ((w >> 1) == h) {
#pragma unroll
            for (int i = 0; i < 32; i += 2) {
                const int row = 16 * (w & 1) + (lane >> 2) + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + 2 * (lane & 3);
                *reinterpret_cast<float2*>(buf + row * kRowsPitch + col) = make_float2(d[i], d[i + 1]);
            }
        }
        named_bar_sync(bar, 128);
        if ((w & 1) == h) {
            const float* src = buf + lane * kRowsPitch + (w >> 1) * 32;
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const float4 v = *reinterpret_cast<const float4*>(src + 4 * q);
                out[4 * q] = v.x; out[4 * q + 1] = v.y; out[4 * q + 2] = v.z; out[4 * q + 3] = v.w;
            }
        }
    }
}

// split 8 consecutive fp32 values into 8 bf16 "hi" and 8 bf16 "lo" (x ~= hi + lo), 16 bytes each
__device__ __forceinline__ void split8(const float4 a, const float4 b, uint4& hi, uint4& lo) {
    const float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    uint32_t h[4], l[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const __nv_bfloat162 hh = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
        const float r0 = f[2 * i] - __low2float(hh), r1 = f[2 * i + 1] - __high2float(hh);
        const __nv_bfloat162 ll = __floats2bfloat162_rn(r0, r1);
        h[i] = *reinterpret_cast<const uint32_t*>(&hh);
        l[i] = *reinterpret_cast<const uint32_t*>(&ll);
    }
    hi = make_uint4(h[0], h[1], h[2], h[3]);
    lo = make_uint4(l[0], l[1], l[2], l[3]);
}
// the "hi" half of split8 alone (round to nearest bf16), for the single-pass kernels
__device__ __forceinline__ uint4 hi8(const float4 a, const float4 b) {
    const __nv_bfloat162 h0 = __floats2bfloat162_rn(a.x, a.y), h1 = __floats2bfloat162_rn(a.z, a.w);
    const __nv_bfloat162 h2 = __floats2bfloat162_rn(b.x, b.y), h3 = __floats2bfloat162_rn(b.z, b.w);
    return make_uint4(*reinterpret_cast<const uint32_t*>(&h0), *reinterpret_cast<const uint32_t*>(&h1),
                      *reinterpret_cast<const uint32_t*>(&h2), *reinterpret_cast<const uint32_t*>(&h3));
}


// ---- additions for the persistent pointwise GEMM (pw_gemm.cu) -------------------------------------------------------
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_fn();      // cuTensorMapEncodeTiled through the runtime's driver entry point table (conv_tc.cu)
int conv_tc_kpad(int k);
// 3-D tensor map over K-major bf16 hi/lo planes [2][rows][k] (the weight packs, the x planes of a 1x1 conv): boxes of
// 64 k x box_rows rows, SWIZZLE_128B (conv_tc.cu)
int kmajor_planes_map(EncodeTiledFn enc, CUtensorMap* map, const void* base, int rows, int k, int box_rows);
// fp32 [B][HW][C] (image stride x_bstride) -> bf16 hi/lo planes [2][B*HW][pitch] with zero padded channels; optionally
// times p*(1-p) of prob, optionally accumulating the per-channel column sums into colsum (conv_planes.cu)
int to_planes_launch(const float* x, long long x_bstride, const float* prob, long long p_bstride, void* out, float* colsum,
                     int B, int HW, int C, int pitch, cudaStream_t st);

// Opts the kernel in to `smem` bytes of dynamic shared memory (the tensor-core kernels need more than the default
// 48 KB), launches it and returns the launch status under `name`.
template <class... P, class... A>
int launch_smem(const char* name, void (*kernel)(P...), dim3 grid, int threads, size_t smem, cudaStream_t st, const A&... args) {
    const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return fail(EFFDET_ERR_LAUNCH, "%s: smem opt-in: %s", name, cudaGetErrorString(e));
    kernel<<<grid, threads, smem, st>>>(args...);
    return launch_status(name);
}

// A kernel's copy of an ABI argument struct: its bytes up to the trailing tc_single, which selects the kernel instance
// instead of being read on the device.  So the parameter blocks keep the layout they had before the field was appended.
template <class T, size_t N>
struct alignas(8) ArgsPrefix {
    unsigned char raw[N];
    __host__ __device__ const T& get() const { return *reinterpret_cast<const T*>(raw); }
    void set(const T& a) { memcpy(raw, &a, N); }
};
using ConvLevel = ArgsPrefix<effdet_conv_args, offsetof(effdet_conv_args, tc_single)>;
using WgradPrefix = ArgsPrefix<effdet_wgrad_args, offsetof(effdet_wgrad_args, tc_single)>;

// pyramid levels one launch of conv_tc_kernel / wgrad_tc2_multi_kernel covers (conv_tc.cu)
constexpr int kMaxLevels = 8;
constexpr int kWgMaxLevels = 8;

// Pixel boxes of the TMA-fed kernels: a [B,H,W,*] map is tiled into boxes of Wb x Hb x Bb = kstage pixels (16..64, a
// multiple of 16) that one tensor-map load turns into kstage consecutive 128-byte rows of shared memory (conv_tc.cu)
struct WgGeom {
    int Wb, Hb, Bb;          // pixel box
    int nbx, nby, nbb;       // boxes per image row / column / batch
    int kstage;              // pixels per box
};
bool wg_geometry(int B, int H, int W, WgGeom* g);
int planes_map(EncodeTiledFn enc, CUtensorMap* map, void* base, int B, int H, int W, int C, int pitch, const WgGeom& g);

}  // namespace effdet
