// SURVEY.md section 8(f) rank 1 -- the step that directly follows backward in the reference's loop:
//   torch.nn.utils.clip_grad_norm_(model.parameters(), 0.1); optimizer.step()   (train.py:115-118, AdamW train.py:268)
// as two multi-tensor launches over all ~280 parameter tensors instead of ~1400 small ATen kernels and a host sync:
//   1. global sum of squares of every gradient            (one fp32 accumulator, atomics per CTA)
//   2. clip coefficient min(1, max_norm / (norm + 1e-6)) read from device memory + decoupled-weight-decay Adam update
// Chunk tables (tensor index, element offset) are built once on the host; every CTA owns one chunk.
#include "common.cuh"

namespace effdet {

__global__ void __launch_bounds__(256) multi_sumsq_kernel(const unsigned long long* __restrict__ g_ptrs,
                                                          const long long* __restrict__ numels,
                                                          const int* __restrict__ chunk_tensor,
                                                          const long long* __restrict__ chunk_off, int chunk,
                                                          float* __restrict__ norm_sq) {
    __shared__ float red[8];
    const int t = chunk_tensor[blockIdx.x];
    const long long off = chunk_off[blockIdx.x];
    const float* g = reinterpret_cast<const float*>(g_ptrs[t]);
    long long n = numels[t] - off;
    if (n > chunk) n = chunk;
    float s = 0.f;
    for (long long i = threadIdx.x; i < n; i += blockDim.x) {
        const float v = __ldg(g + off + i);
        s = fmaf(v, v, s);
    }
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        float tot = 0.f;
        for (int i = 0; i < 8; ++i) tot += red[i];
        atomicAdd(norm_sq, tot);
    }
}

// The clip + AdamW update of one chunk, shared by the kernel with host-side lr / bias corrections and the one that
// reads them from device memory.  kZeroGrad: the gradient buffer is an accumulator that the step empties
// (optimizer.zero_grad() after optimizer.step(), train.py:117-118); otherwise write_clipped_grad says whether the
// clipped gradient is written back, as clip_grad_norm_ does.
// omb1 / omb2: 1 - beta1 / 1 - beta2 in fp32.
template <bool kZeroGrad>
__device__ __forceinline__ void clip_adamw_chunk(float* p, float* g, float* m, float* v, long long n,
                                                 const float* __restrict__ norm_sq, float max_norm, float lr,
                                                 float beta1, float beta2, float omb1, float omb2, float eps,
                                                 float weight_decay, float bias_c1, float bias_c2,
                                                 int write_clipped_grad) {
    // clip_grad_norm_: coef = max_norm / (total_norm + 1e-6), clamped to 1
    float coef = 1.f;
    if (max_norm > 0.f) coef = fminf(max_norm / (sqrtf(__ldg(norm_sq)) + 1e-6f), 1.f);
    const float step_size = lr / bias_c1;
    const float inv_sqrt_c2 = rsqrtf(bias_c2);
    for (long long i = threadIdx.x; i < n; i += blockDim.x) {
        const float gi = g[i] * coef;
        float pi = p[i];
        pi *= (1.f - lr * weight_decay);                       // decoupled weight decay (AdamW)
        const float mi = beta1 * m[i] + omb1 * gi;
        const float vi = beta2 * v[i] + omb2 * gi * gi;
        const float denom = sqrtf(vi) * inv_sqrt_c2 + eps;
        pi -= step_size * (mi / denom);
        p[i] = pi;
        m[i] = mi;
        v[i] = vi;
        if (kZeroGrad)
            g[i] = 0.f;
        else if (write_clipped_grad)
            g[i] = gi;
    }
}

__global__ void __launch_bounds__(256) multi_clip_adamw_kernel(
    const unsigned long long* __restrict__ p_ptrs, const unsigned long long* __restrict__ g_ptrs,
    const unsigned long long* __restrict__ m_ptrs, const unsigned long long* __restrict__ v_ptrs,
    const long long* __restrict__ numels, const int* __restrict__ chunk_tensor, const long long* __restrict__ chunk_off,
    int chunk, const float* __restrict__ norm_sq, float max_norm, float lr, float beta1, float beta2, float eps,
    float weight_decay, float bias_c1, float bias_c2, int write_clipped_grad) {
    const int t = chunk_tensor[blockIdx.x];
    const long long off = chunk_off[blockIdx.x];
    float* p = reinterpret_cast<float*>(p_ptrs[t]) + off;
    float* g = reinterpret_cast<float*>(g_ptrs[t]) + off;
    float* m = reinterpret_cast<float*>(m_ptrs[t]) + off;
    float* v = reinterpret_cast<float*>(v_ptrs[t]) + off;
    long long n = numels[t] - off;
    if (n > chunk) n = chunk;
    clip_adamw_chunk<false>(p, g, m, v, n, norm_sq, max_norm, lr, beta1, beta2, 1.f - beta1, 1.f - beta2, eps,
                            weight_decay, bias_c1, bias_c2, write_clipped_grad);
}

// Gradient accumulation of one micro-step: acc_t += g_t, skipped as a whole when the step's loss is exactly zero
// (train.py:111-113 `if bool(loss == 0): continue`).  CTA 0 also writes the optimizer gate of the step.
__global__ void __launch_bounds__(256) multi_accumulate_kernel(
    const unsigned long long* __restrict__ acc_ptrs, const unsigned long long* __restrict__ g_ptrs,
    const long long* __restrict__ numels, const int* __restrict__ chunk_tensor, const long long* __restrict__ chunk_off,
    int chunk, const float* __restrict__ loss, const int* __restrict__ update_requested, int* __restrict__ gate) {
    const bool live = __ldg(loss) != 0.f;
    if (gate != nullptr && blockIdx.x == 0 && threadIdx.x == 0) *gate = (live && __ldg(update_requested) != 0) ? 1 : 0;
    if (!live) return;
    const int t = chunk_tensor[blockIdx.x];
    const long long off = chunk_off[blockIdx.x];
    float* acc = reinterpret_cast<float*>(acc_ptrs[t]) + off;
    const float* g = reinterpret_cast<const float*>(g_ptrs[t]) + off;
    long long n = numels[t] - off;
    if (n > chunk) n = chunk;
    for (long long i = threadIdx.x; i < n; i += blockDim.x) acc[i] += __ldg(g + i);
}

// Clip + AdamW with the learning rate, the step count and the gate in device memory, so that a replayed CUDA graph
// follows the schedule and the bias corrections of the real step.  Gate closed: nothing is read or written beyond the
// gate.  Gate open: the update of the host-argument kernel, bias corrections 1 - beta^(step+1) in fp64 rounded to
// fp32 (what the host computes for effdet_multi_clip_adamw), 1 - beta rounded from fp64 as torch.optim.AdamW does
// (1.f - 0.999f is 1.3e-5 off), accumulators zeroed, and the counter advanced once by
// the last CTA to take a ticket -- every other CTA has read the counter before taking its ticket.
__global__ void __launch_bounds__(256) multi_clip_adamw_dev_kernel(
    const unsigned long long* __restrict__ p_ptrs, const unsigned long long* __restrict__ g_ptrs,
    const unsigned long long* __restrict__ m_ptrs, const unsigned long long* __restrict__ v_ptrs,
    const long long* __restrict__ numels, const int* __restrict__ chunk_tensor, const long long* __restrict__ chunk_off,
    int chunk, const float* __restrict__ norm_sq, float max_norm, const float* __restrict__ lr_dev, long long* step,
    const int* __restrict__ gate, unsigned int* ticket, double beta1, double beta2, float eps, float weight_decay) {
    if (__ldg(gate) == 0) return;
    __shared__ float bias_c[2];
    if (threadIdx.x == 0) {
        const long long s = *step;
        __threadfence();                                       // the read above completes before the ticket
        if (atomicAdd(ticket, 1u) == gridDim.x - 1) {
            *ticket = 0u;
            *step = s + 1;
        }
        const double k = static_cast<double>(s + 1);
        bias_c[0] = static_cast<float>(1.0 - pow(beta1, k));
        bias_c[1] = static_cast<float>(1.0 - pow(beta2, k));
    }
    __syncthreads();
    const int t = chunk_tensor[blockIdx.x];
    const long long off = chunk_off[blockIdx.x];
    long long n = numels[t] - off;
    if (n > chunk) n = chunk;
    clip_adamw_chunk<true>(reinterpret_cast<float*>(p_ptrs[t]) + off, reinterpret_cast<float*>(g_ptrs[t]) + off,
                           reinterpret_cast<float*>(m_ptrs[t]) + off, reinterpret_cast<float*>(v_ptrs[t]) + off, n,
                           norm_sq, max_norm, __ldg(lr_dev), static_cast<float>(beta1), static_cast<float>(beta2),
                           static_cast<float>(1.0 - beta1), static_cast<float>(1.0 - beta2), eps, weight_decay,
                           bias_c[0], bias_c[1], 0);
}

// Exponential moving average of the weights (Tan et al. 2020, section 5.1): e = e - w * (e - s) per element, each
// operation rounded on its own (TF's assign_moving_average: variable - (variable - value) * (1 - decay)), with the
// decay ramp of TF's ExponentialMovingAverage(decay, num_updates) in fp64 and w = 1 - d rounded once to fp32.  The
// counter advances once per launch by the last CTA to take a ticket, as in multi_clip_adamw_dev_kernel.
__global__ void __launch_bounds__(256) multi_ema_kernel(
    const unsigned long long* __restrict__ ema_ptrs, const unsigned long long* __restrict__ src_ptrs,
    const long long* __restrict__ numels, const int* __restrict__ chunk_tensor, const long long* __restrict__ chunk_off,
    int chunk, double decay, int ramp, long long* updates, const int* __restrict__ gate, unsigned int* ticket) {
    if (gate != nullptr && __ldg(gate) == 0) return;
    __shared__ float w_s;
    if (threadIdx.x == 0) {
        const long long u = *updates;
        __threadfence();                                       // the read above completes before the ticket
        if (atomicAdd(ticket, 1u) == gridDim.x - 1) {
            *ticket = 0u;
            *updates = u + 1;
        }
        const double k = static_cast<double>(u + 1);
        const double d = ramp ? fmin(decay, (1.0 + k) / (10.0 + k)) : decay;
        w_s = static_cast<float>(1.0 - d);
    }
    __syncthreads();
    const float w = w_s;
    const int t = chunk_tensor[blockIdx.x];
    const long long off = chunk_off[blockIdx.x];
    float* __restrict__ e = reinterpret_cast<float*>(ema_ptrs[t]) + off;
    const float* __restrict__ s = reinterpret_cast<const float*>(src_ptrs[t]) + off;
    long long n = numels[t] - off;
    if (n > chunk) n = chunk;
    // kUnroll elements per thread and pass, all loaded before any is stored: one load pair per thread in flight
    // leaves a 65536-element chunk latency-bound
    constexpr int kUnroll = 8;
    for (long long i0 = threadIdx.x; i0 < n; i0 += kUnroll * blockDim.x) {
        float ev[kUnroll], sv[kUnroll];
#pragma unroll
        for (int j = 0; j < kUnroll; ++j) {
            const long long i = i0 + j * blockDim.x;
            if (i < n) {
                ev[j] = e[i];
                sv[j] = __ldg(s + i);
            }
        }
#pragma unroll
        for (int j = 0; j < kUnroll; ++j) {
            const long long i = i0 + j * blockDim.x;
            if (i < n) e[i] = __fsub_rn(ev[j], __fmul_rn(w, __fsub_rn(ev[j], sv[j])));
        }
    }
}

}  // namespace effdet

using namespace effdet;

extern "C" int effdet_multi_sumsq(const uint64_t* g_ptrs, const int64_t* numels, const int32_t* chunk_tensor,
                                  const int64_t* chunk_off, int nchunks, int chunk, float* norm_sq, int device,
                                  effdet_stream_t stream) {
    EFFDET_REQUIRE(g_ptrs && numels && chunk_tensor && chunk_off && norm_sq && nchunks > 0 && chunk > 0,
                   "multi_sumsq: bad arguments");
    EFFDET_DEVICE(device);
    multi_sumsq_kernel<<<nchunks, 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const unsigned long long*>(g_ptrs), reinterpret_cast<const long long*>(numels), chunk_tensor,
        reinterpret_cast<const long long*>(chunk_off), chunk, norm_sq);
    return launch_status("multi_sumsq_kernel");
}

extern "C" int effdet_multi_clip_adamw(const uint64_t* p_ptrs, const uint64_t* g_ptrs, const uint64_t* m_ptrs,
                                       const uint64_t* v_ptrs, const int64_t* numels, const int32_t* chunk_tensor,
                                       const int64_t* chunk_off, int nchunks, int chunk, const float* norm_sq,
                                       float max_norm, float lr, float beta1, float beta2, float eps, float weight_decay,
                                       float bias_c1, float bias_c2, int write_clipped_grad, int device,
                                       effdet_stream_t stream) {
    EFFDET_REQUIRE(p_ptrs && g_ptrs && m_ptrs && v_ptrs && numels && chunk_tensor && chunk_off && norm_sq && nchunks > 0 &&
                       chunk > 0,
                   "multi_clip_adamw: bad arguments");
    EFFDET_REQUIRE(bias_c1 > 0.f && bias_c2 > 0.f, "multi_clip_adamw: bias corrections must be positive");
    EFFDET_DEVICE(device);
    multi_clip_adamw_kernel<<<nchunks, 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const unsigned long long*>(p_ptrs), reinterpret_cast<const unsigned long long*>(g_ptrs),
        reinterpret_cast<const unsigned long long*>(m_ptrs), reinterpret_cast<const unsigned long long*>(v_ptrs),
        reinterpret_cast<const long long*>(numels), chunk_tensor, reinterpret_cast<const long long*>(chunk_off), chunk,
        norm_sq, max_norm, lr, beta1, beta2, eps, weight_decay, bias_c1, bias_c2, write_clipped_grad);
    return launch_status("multi_clip_adamw_kernel");
}

extern "C" int effdet_multi_accumulate(const uint64_t* acc_ptrs, const uint64_t* g_ptrs, const int64_t* numels,
                                       const int32_t* chunk_tensor, const int64_t* chunk_off, int nchunks, int chunk,
                                       const float* loss, const int32_t* update_requested, int32_t* gate, int device,
                                       effdet_stream_t stream) {
    EFFDET_REQUIRE(acc_ptrs && g_ptrs && numels && chunk_tensor && chunk_off && loss && nchunks > 0 && chunk > 0,
                   "multi_accumulate: bad arguments");
    EFFDET_REQUIRE((gate == nullptr) == (update_requested == nullptr),
                   "multi_accumulate: gate and update_requested are given together or not at all");
    EFFDET_DEVICE(device);
    multi_accumulate_kernel<<<nchunks, 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const unsigned long long*>(acc_ptrs), reinterpret_cast<const unsigned long long*>(g_ptrs),
        reinterpret_cast<const long long*>(numels), chunk_tensor, reinterpret_cast<const long long*>(chunk_off), chunk,
        loss, update_requested, gate);
    return launch_status("multi_accumulate_kernel");
}

extern "C" int effdet_multi_clip_adamw_dev(const uint64_t* p_ptrs, const uint64_t* g_ptrs, const uint64_t* m_ptrs,
                                           const uint64_t* v_ptrs, const int64_t* numels, const int32_t* chunk_tensor,
                                           const int64_t* chunk_off, int nchunks, int chunk, const float* norm_sq,
                                           float max_norm, const float* lr, int64_t* step, const int32_t* gate,
                                           uint32_t* ticket, double beta1, double beta2, float eps, float weight_decay,
                                           int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(p_ptrs && g_ptrs && m_ptrs && v_ptrs && numels && chunk_tensor && chunk_off && norm_sq && lr && step &&
                       gate && ticket && nchunks > 0 && chunk > 0,
                   "multi_clip_adamw_dev: bad arguments");
    EFFDET_REQUIRE(beta1 >= 0.0 && beta1 < 1.0 && beta2 >= 0.0 && beta2 < 1.0,
                   "multi_clip_adamw_dev: betas must lie in [0, 1) (got %g, %g)", beta1, beta2);
    EFFDET_DEVICE(device);
    multi_clip_adamw_dev_kernel<<<nchunks, 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const unsigned long long*>(p_ptrs), reinterpret_cast<const unsigned long long*>(g_ptrs),
        reinterpret_cast<const unsigned long long*>(m_ptrs), reinterpret_cast<const unsigned long long*>(v_ptrs),
        reinterpret_cast<const long long*>(numels), chunk_tensor, reinterpret_cast<const long long*>(chunk_off), chunk,
        norm_sq, max_norm, lr, reinterpret_cast<long long*>(step), gate, ticket, beta1, beta2, eps, weight_decay);
    return launch_status("multi_clip_adamw_dev_kernel");
}

extern "C" int effdet_multi_ema(const uint64_t* ema_ptrs, const uint64_t* src_ptrs, const int64_t* numels,
                                const int32_t* chunk_tensor, const int64_t* chunk_off, int nchunks, int chunk,
                                double decay, int ramp, int64_t* updates, const int32_t* gate, uint32_t* ticket,
                                int device, effdet_stream_t stream) {
    EFFDET_REQUIRE(ema_ptrs && src_ptrs && numels && chunk_tensor && chunk_off && updates && ticket && nchunks > 0 &&
                       chunk > 0,
                   "multi_ema: bad arguments");
    EFFDET_REQUIRE(decay >= 0.0 && decay <= 1.0, "multi_ema: decay must lie in [0, 1] (got %g)", decay);
    EFFDET_DEVICE(device);
    multi_ema_kernel<<<nchunks, 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const unsigned long long*>(ema_ptrs), reinterpret_cast<const unsigned long long*>(src_ptrs),
        reinterpret_cast<const long long*>(numels), chunk_tensor, reinterpret_cast<const long long*>(chunk_off), chunk,
        decay, ramp, reinterpret_cast<long long*>(updates), gate, ticket);
    return launch_status("multi_ema_kernel");
}
