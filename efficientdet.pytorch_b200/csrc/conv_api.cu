// The dense-convolution entry points effdet_conv2d{,_multi} and effdet_conv2d_wgrad{,_multi}: every level of a call is
// validated before any device work, then the routing policy picks the kernels; their launchers take validated arguments.
#include "tc_ptx.cuh"

namespace effdet {

int pw_gemm_launch(const effdet_conv_args* a, cudaStream_t st);                        // pw_gemm.cu
int conv_tc_launch(const effdet_conv_args* levels, int nlevels, cudaStream_t st);      // conv_tc.cu
int conv_simt_launch(const effdet_conv_args* a, cudaStream_t st);                      // conv_simt.cu
int pw_wgrad_launch(const effdet_wgrad_args* a, cudaStream_t st);                      // pw_wgrad.cu
int wgrad_tc2_launch(const effdet_wgrad_args* levels, int nlevels, float* acc, cudaStream_t st);   // conv_tc.cu
int wgrad_tc_launch(const effdet_wgrad_args* a, float* acc, cudaStream_t st);                      // conv_tc.cu
int wgrad_fold_launch(const float* ws, float* dw, long long nc, cudaStream_t st);                  // conv_tc.cu
int wgrad_simt_launch(const effdet_wgrad_args* a, cudaStream_t st);                    // conv_simt.cu
int colsum_launch(const float* x, float* out, long long M, int N, long long HW, long long bstride, cudaStream_t st);  // conv_simt.cu

// ---- routing policy: what each kernel takes beyond the checks below ------------------------------------------------
// persistent pointwise GEMM: 1x1 convs with a tensor-core weight pack
static bool pw_gemm_eligible(const effdet_conv_args* a) {
    if (a->ksize != 1 || a->w_tc == nullptr || a->Cin < 8 || a->Cout < 8) return false;
    if (a->x_planes) return a->Cin % 8 == 0 && !a->in_scale && !a->a_scale;
    return a->x_bstride == (long long)a->H * a->W * a->Cin;     // x must be one dense [M, Cin] matrix for the 2-D tensor map
}

// tensor-core implicit GEMM: the 3x3 convs of neck and head; the MBConv prologue / epilogue inputs go to the CUDA cores
static bool conv_tc_eligible(const effdet_conv_args* a) {
    return a->w_tc != nullptr && a->ksize == 3 && a->Cout >= 16 && !a->a_scale && !a->z && !a->scale && !a->shift &&
           !a->row_scale && !a->in_scale;
}

// pointwise weight gradient: 1x1, no bias, operands converted in the kernel, no split passes
static bool pw_wgrad_eligible(const effdet_wgrad_args* a) {
    if (a->ksize != 1 || a->precision != 1 || a->dbias || a->x_planes || !a->x) return false;
    if (a->Cin % 8 || a->Cout % 8 || a->Cin < 8 || a->Cout < 8) return false;
    const long long HW = (long long)a->H * a->W;
    if (a->x_bstride != HW * a->Cin) return false;
    if (!a->dy_planes && (!a->dy || a->dy_bstride != HW * a->Cout)) return false;
    return (long long)a->B * HW < (1ll << 31) - 64;
}

// the tensor-core weight gradients have no input prologue: those convs go to the CUDA-core kernel
static bool wgrad_tc_eligible(const effdet_wgrad_args* a) {
    return a->precision == 1 && a->Cin >= 16 && a->Cout >= 16 && !a->a_scale && !a->in_scale;
}

// the TMA-fed one also needs both operands as planes (given, or split into the workspaces) and a pixel box
static bool wgrad_tma_eligible(const effdet_wgrad_args* a) {
    WgGeom g;
    return wgrad_tc_eligible(a) && (a->ws_x || a->x_planes) && (a->ws_dy || a->dy_planes) &&
           wg_geometry(a->B, a->H, a->W, &g) && encode_fn();
}

static int conv_level(const effdet_conv_args* a, cudaStream_t st) {
    if (pw_gemm_eligible(a)) return pw_gemm_launch(a, st);
    if (conv_tc_eligible(a)) return conv_tc_launch(a, 1, st);
    return conv_simt_launch(a, st);
}

// the bias gradient comes from the dy split pass on the TMA-fed route, from a column sum on the others; the tensor-core
// kernels add into acc ([taps][Cout][Cin]), the others into dw
static int wgrad_level(const effdet_wgrad_args* a, float* acc, cudaStream_t st) {
    if (pw_wgrad_eligible(a)) return pw_wgrad_launch(a, st);
    if (wgrad_tma_eligible(a)) return wgrad_tc2_launch(a, 1, acc, st);
    if (a->dy_planes || a->x_planes)                  // the other kernels read fp32 operands only
        return fail(EFFDET_ERR_UNSUPPORTED, "wgrad: dy_planes given but the TMA-fed tensor-core kernel cannot take this shape or "
                                            "input prologue (check effdet_wgrad_tc_geometry_ok first)");
    const int s = wgrad_tc_eligible(a) ? wgrad_tc_launch(a, acc, st) : wgrad_simt_launch(a, st);
    if (s || !a->dbias) return s;
    return colsum_launch(a->dy, a->dbias, (long long)a->B * a->H * a->W, a->Cout, (long long)a->H * a->W, a->dy_bstride, st);
}

// ---- validation of one level, and of what it shares with the first level of the call --------------------------------
static int check_conv_level(const effdet_conv_args* a, const effdet_conv_args* first) {
    EFFDET_REQUIRE(a && (a->x || a->x_planes) && a->w && a->y, "conv2d: null tensor");
    EFFDET_REQUIRE(!a->x_planes || (pw_gemm_eligible(a) && aligned16(a->x_planes)),
                   "conv2d: x_planes is only understood by the tensor-core 1x1 path (Cin %% 8 == 0, no input prologue)");
    EFFDET_REQUIRE(a->ksize == 1 || a->ksize == 3, "conv2d: ksize %d not in {1,3}", a->ksize);
    EFFDET_REQUIRE(!a->tc_single || a->w_tc, "conv2d: tc_single needs the tensor-core weight pack w_tc (the exact-fp32 path has one product)");
    EFFDET_REQUIRE(!a->tc_single || a->ksize == 3, "conv2d: tc_single is defined for 3x3 convolutions only (ksize %d)", a->ksize);
    EFFDET_REQUIRE(a->Cin % 4 == 0 && a->Cout % 4 == 0, "conv2d: Cin=%d Cout=%d must be multiples of 4", a->Cin, a->Cout);
    EFFDET_REQUIRE(a->B > 0 && a->H > 0 && a->W > 0, "conv2d: empty shape");
    EFFDET_REQUIRE((a->scale == nullptr) == (a->shift == nullptr), "conv2d: scale/shift must come together");
    EFFDET_REQUIRE((a->in_scale == nullptr) == (a->in_shift == nullptr) && (!a->in_scale || a->ksize == 1),
                   "conv2d: in_scale/in_shift must come together (1x1 convs only: zero padding is applied after the activation)");
    EFFDET_REQUIRE(aligned16(a->in_scale) && aligned16(a->in_shift), "conv2d: in_scale/in_shift must be 16-byte aligned");
    EFFDET_REQUIRE(aligned16(a->x) && aligned16(a->w) && aligned16(a->y) && aligned16(a->z) && aligned16(a->bias) &&
                       aligned16(a->residual) && aligned16(a->mask_src) && aligned16(a->a_scale),
                   "conv2d: pointers must be 16-byte aligned");
    EFFDET_REQUIRE(a->x_bstride % 4 == 0 && a->y_bstride % 4 == 0 && a->r_bstride % 4 == 0 && a->m_bstride % 4 == 0,
                   "conv2d: batch strides must be multiples of 4 elements");
    EFFDET_REQUIRE((long long)a->B * a->H * a->W < (1ll << 31), "conv2d: B*H*W too large");
    EFFDET_REQUIRE(a->Cin == first->Cin && a->Cout == first->Cout && a->ksize == first->ksize && a->act == first->act &&
                       a->w == first->w && a->w_tc == first->w_tc && a->bias == first->bias,
                   "conv2d_multi: all levels must share weights, bias, channels and activation");
    EFFDET_REQUIRE(a->tc_single == first->tc_single, "conv2d_multi: levels disagree on tc_single");
    return EFFDET_OK;
}

static int check_wgrad_level(const effdet_wgrad_args* a, const effdet_wgrad_args* first) {
    EFFDET_REQUIRE(a && (a->x || a->x_planes) && (a->dy || a->dy_planes) && a->dw, "wgrad: null tensor");
    EFFDET_REQUIRE(!a->dy_planes || (a->precision == 1 && !a->dbias && aligned16(a->dy_planes) && (a->ws_x || a->x_planes)),
                   "wgrad: dy_planes needs precision 1, no dbias and the ws_x workspace (or x_planes)");
    EFFDET_REQUIRE(!a->x_planes || (a->precision == 1 && !a->a_scale && !a->in_scale && aligned16(a->x_planes) &&
                                    (a->ws_dy || a->dy_planes)),
                   "wgrad: x_planes needs precision 1 and no input prologue");
    EFFDET_REQUIRE(a->ksize == 1 || a->ksize == 3, "wgrad: ksize %d not in {1,3}", a->ksize);
    EFFDET_REQUIRE(!a->tc_single || a->precision == 1, "wgrad: tc_single needs precision 1 (the exact-fp32 path has one product)");
    EFFDET_REQUIRE(!a->tc_single || a->ksize == 3, "wgrad: tc_single is defined for 3x3 convolutions only (ksize %d)", a->ksize);
    EFFDET_REQUIRE(a->Cin % 4 == 0 && a->Cout % 4 == 0, "wgrad: channels must be multiples of 4");
    EFFDET_REQUIRE(a->B > 0 && a->H > 0 && a->W > 0, "wgrad: empty shape");
    EFFDET_REQUIRE(aligned16(a->x) && aligned16(a->dy) && aligned16(a->dw) && aligned16(a->a_scale) && aligned16(a->in_scale) &&
                       aligned16(a->in_shift) && aligned16(a->ws_dw),
                   "wgrad: pointers must be 16-byte aligned");
    EFFDET_REQUIRE((a->in_scale == nullptr) == (a->in_shift == nullptr) && (!a->in_scale || a->ksize == 1),
                   "wgrad: in_scale/in_shift must come together (1x1 convs only)");
    EFFDET_REQUIRE(a->x_bstride % 4 == 0 && a->dy_bstride % 4 == 0, "wgrad: batch strides must be multiples of 4");
    EFFDET_REQUIRE((long long)a->B * a->H * a->W < (1ll << 31), "wgrad: B*H*W too large");
    EFFDET_REQUIRE(a->dw == first->dw && a->dbias == first->dbias && a->Cin == first->Cin && a->Cout == first->Cout &&
                       a->ksize == first->ksize,
                   "conv2d_wgrad_multi: all levels must share dw, dbias, channels and ksize");
    EFFDET_REQUIRE(a->tc_single == first->tc_single, "conv2d_wgrad_multi: levels disagree on tc_single");
    return EFFDET_OK;
}

// ---- one call: every level checked, then one launch for all levels or one per level --------------------------------
static int conv2d(const effdet_conv_args* levels, int nlevels, int device, cudaStream_t st) {
    EFFDET_REQUIRE(nlevels >= 1 && nlevels <= kMaxLevels, "conv2d_multi: 1..%d levels", kMaxLevels);
    for (int l = 0; l < nlevels; ++l)
        if (const int s = check_conv_level(levels + l, levels)) return s;
    EFFDET_DEVICE(device);
    bool one = true;
    for (int l = 0; l < nlevels; ++l) one = one && conv_tc_eligible(&levels[l]);
    if (one) return conv_tc_launch(levels, nlevels, st);
    int s = EFFDET_OK;
    for (int l = 0; l < nlevels && !s; ++l) s = conv_level(&levels[l], st);
    return s;
}

static int conv2d_wgrad(const effdet_wgrad_args* levels, int nlevels, int device, cudaStream_t st) {
    EFFDET_REQUIRE(nlevels >= 1, "conv2d_wgrad_multi: no levels");
    for (int l = 0; l < nlevels; ++l)
        if (const int s = check_wgrad_level(levels + l, levels)) return s;
    // the tensor-core kernels reduce into a tap-major [taps][Cout][Cin] accumulator: dw itself for a 1x1 conv, the first
    // level's ws_dw for a 3x3 one, which is cleared here and folded into dw after the launches
    const effdet_wgrad_args* a0 = levels;
    bool tc3 = false;
    for (int l = 0; l < nlevels; ++l) tc3 = tc3 || (a0->ksize == 3 && wgrad_tc_eligible(&levels[l]));
    EFFDET_REQUIRE(!tc3 || a0->ws_dw, "wgrad: a 3x3 tensor-core weight gradient needs the ws_dw workspace (4*9*Cout*Cin bytes)");
    EFFDET_DEVICE(device);
    const long long nc = (long long)a0->Cout * a0->Cin;
    float* acc = tc3 ? static_cast<float*>(a0->ws_dw) : a0->dw;
    if (tc3) {
        const cudaError_t e = cudaMemsetAsync(acc, 0, 9 * nc * sizeof(float), st);
        if (e != cudaSuccess) return fail(EFFDET_ERR_LAUNCH, "wgrad: clearing ws_dw: %s", cudaGetErrorString(e));
    }
    bool one = nlevels > 1 && nlevels <= kWgMaxLevels;      // one level keeps its own route, the pointwise kernel included
    for (int l = 0; l < nlevels; ++l) one = one && wgrad_tma_eligible(&levels[l]);
    int s = EFFDET_OK;
    if (one)
        s = wgrad_tc2_launch(levels, nlevels, acc, st);
    else
        for (int l = 0; l < nlevels && !s; ++l) s = wgrad_level(&levels[l], acc, st);
    if (s || !tc3) return s;
    return wgrad_fold_launch(acc, a0->dw, nc, st);
}

}  // namespace effdet

extern "C" int effdet_conv2d(const effdet_conv_args* a, int device, effdet_stream_t stream) {
    return effdet::conv2d(a, 1, device, (cudaStream_t)stream);
}
extern "C" int effdet_conv2d_multi(const effdet_conv_args* levels, int nlevels, int device, effdet_stream_t stream) {
    return effdet::conv2d(levels, nlevels, device, (cudaStream_t)stream);
}
extern "C" int effdet_conv2d_wgrad(const effdet_wgrad_args* a, int device, effdet_stream_t stream) {
    return effdet::conv2d_wgrad(a, 1, device, (cudaStream_t)stream);
}
extern "C" int effdet_conv2d_wgrad_multi(const effdet_wgrad_args* levels, int nlevels, int device, effdet_stream_t stream) {
    return effdet::conv2d_wgrad(levels, nlevels, device, (cudaStream_t)stream);
}
