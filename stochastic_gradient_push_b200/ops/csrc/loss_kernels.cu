// Fused softmax cross-entropy + top-1 / top-5 accuracy (forward) and its gradient (backward).
//
// The reference computes, every iteration, nn.CrossEntropyLoss (log_softmax + nll_loss kernels),
// then `accuracy(output, target, topk=(1, 5))` (topk + transpose + eq + 2 x sum + mul, ~10
// launches) and reads the three scalars back with three `.item()` host syncs
// (/root/reference/gossip_sgd.py:372-373, 394-399, 192-198).  Here one launch produces all three
// numbers on the device (mean loss, prec@1 %, prec@5 %) plus the per-row log-sum-exp the backward
// kernel needs; the training step copies the 12 bytes to a pinned ring without a host sync.
//
//   forward : one warp per row:  m = max_j z_j ; lse = m + log sum_j exp(z_j - m)
//             loss_i = lse - z_t ; rank_i = #{ j : z_j > z_t }   (top-k hit <=> rank < k)
//             out[0] += loss_i / B ; out[1] += 100/B [rank == 0] ; out[2] += 100/B [rank < 5]
//   backward: dz_ij = g * (exp(z_ij - lse_i) - [j == t_i]) / B
//
// Label smoothing eps (torch.nn.functional.cross_entropy(label_smoothing=eps), mean reduction):
//   forward : loss_i = lse_i - (1 - eps) z_t - (eps / C) sum_j z_j   (sum_j z_j: one more per-lane
//             accumulator in the same pass, so each logit is still read once)
//   backward: dz_ij = g * (exp(z_ij - lse_i) - (1 - eps)[j == t_i] - eps / C) / B
// SMOOTH is a template parameter: eps == 0 launches the SMOOTH = false kernels, whose code is the
// unsmoothed kernels' instruction for instruction (no 0 * sum_j z_j, which is NaN for inf logits).
// A row whose target is out of range adds no loss and gets a zero gradient either way.
//
// Two targets (mixup / CutMix, ops/batch_mix.py): row i's partner is row B-1-i (the flipped
// batch), with target b = t_{B-1-i} and the mix weight lam read from the device mix state
// (mix[0], written by an H2D copy each step: a captured graph never re-captures):
//   forward : loss_i = lse_i - (1 - eps)(lam z_a + (1 - lam) z_b) - (eps / C) sum_j z_j
//             (one more logit read per row); prec@1 / prec@5 count against the row's own target a
//   backward: dz_ij = g * (exp(z_ij - lse_i) - (1 - eps)(lam [j == a] + (1 - lam)[j == b]) - eps / C) / B
// MIX is a template parameter next to SMOOTH: without a mix state the MIX = false kernels run,
// whose code is the one-target kernels' (the mix pointer is a trailing, unused argument).  A row
// whose target or partner target is out of range adds no loss and gets a zero gradient; its
// accuracy still counts against its own target.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace {

constexpr int XE_THREADS = 256;                 // 8 rows per CTA

template <typename T> __device__ __forceinline__ float to_f(T v);
template <> __device__ __forceinline__ float to_f<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

__device__ __forceinline__ float warp_max(float v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xFFFFFFFFu, v, o));
    return v;
}
__device__ __forceinline__ float warp_sum(float v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
    return v;
}

// One warp over row z (lane-strided): lse = log sum_j exp(z_j) by the online softmax, above = #{ j : z_j > zt }
// (the row's rank: top-k hit <=> above < k) and, with SMOOTH, sum_j z_j -- each logit read once.  Shared by
// the training forward and the evaluation accumulate kernel, so both count hits the same way.
template <typename T, bool SMOOTH>
__device__ __forceinline__ void xent_row_scan(const T* z, int C, float zt, int lane, float& lse, float& above,
                                              float& sum_z)
{
    float m = -INFINITY, s = 0.f, ab = 0.f, sz = 0.f;
    for (int j = lane; j < C; j += 32) {
        const float v = to_f<T>(z[j]);
        const float mn = fmaxf(m, v);
        s = s * __expf(m - mn) + __expf(v - mn);
        m = mn;
        ab += (v > zt) ? 1.f : 0.f;
        if (SMOOTH) sz += v;
    }
    const float mw = warp_max(m);
    s = warp_sum(s * __expf(m - mw));
    above = warp_sum(ab);
    sum_z = SMOOTH ? warp_sum(sz) : sz;
    lse = mw + __logf(s);
}

template <typename T, bool SMOOTH, bool MIX>
__global__ void __launch_bounds__(XE_THREADS)
xent_fwd_kernel(const T* __restrict__ logits, const long long* __restrict__ target, float* __restrict__ lse_out,
                float* __restrict__ out3, int B, int C, float eps, const float* __restrict__ mix)
{
    __shared__ float s_acc[3];
    if (threadIdx.x < 3) s_acc[threadIdx.x] = 0.f;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * (XE_THREADS / 32) + (threadIdx.x >> 5);
    if (row < B) {
        const T* z = logits + (size_t)row * C;
        long long t = target[row];
        const bool valid = t >= 0 && t < C;
        if (!valid) t = 0;
        const float zt = to_f<T>(z[t]);
        float zb = 0.f;
        bool valid_b = true;
        if (MIX) {
            long long tb = target[B - 1 - row];
            valid_b = tb >= 0 && tb < C;
            if (!valid_b) tb = 0;
            zb = to_f<T>(z[tb]);
        }
        // online softmax: one pass for max + sum, rank counted in the same pass
        float lse, above, sum_z;
        xent_row_scan<T, SMOOTH>(z, C, zt, lane, lse, above, sum_z);
        if (lane == 0) {
            lse_out[row] = lse;
            if (valid) {
                const float inv_b = 1.f / (float)B;
                if (MIX) {
                    const float lam = mix[0];
                    const float zm = lam * zt + (1.f - lam) * zb;
                    const float loss = SMOOTH ? lse - (1.f - eps) * zm - eps * (sum_z / (float)C) : lse - zm;
                    if (valid_b) atomicAdd(&s_acc[0], loss * inv_b);
                } else {
                    const float loss = SMOOTH ? lse - (1.f - eps) * zt - eps * (sum_z / (float)C) : lse - zt;
                    atomicAdd(&s_acc[0], loss * inv_b);
                }
                if (above < 0.5f) atomicAdd(&s_acc[1], 100.f * inv_b);
                if (above < 4.5f) atomicAdd(&s_acc[2], 100.f * inv_b);
            }
        }
    }
    __syncthreads();
    if (threadIdx.x < 3) atomicAdd(out3 + threadIdx.x, s_acc[threadIdx.x]);
}

// Evaluation: plain cross-entropy, forward only, summed over batches into a persistent device accumulator
// acc = [loss sum (fp64 bits), top-1 hits, top-5 hits, valid rows].  A row whose target is outside [0, C)
// adds to none of the four.  No lse is stored.
template <typename T>
__global__ void __launch_bounds__(XE_THREADS)
xent_eval_kernel(const T* __restrict__ logits, const long long* __restrict__ target,
                 unsigned long long* __restrict__ acc, int B, int C)
{
    __shared__ double s_loss;
    __shared__ unsigned int s_cnt[3];
    if (threadIdx.x == 0) s_loss = 0.0;
    if (threadIdx.x < 3) s_cnt[threadIdx.x] = 0u;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * (XE_THREADS / 32) + (threadIdx.x >> 5);
    if (row < B) {
        const long long t = target[row];
        if (t >= 0 && t < C) {                              // (warp-uniform)
            const T* z = logits + (size_t)row * C;
            const float zt = to_f<T>(z[t]);
            float lse, above, sum_z;
            xent_row_scan<T, false>(z, C, zt, lane, lse, above, sum_z);
            if (lane == 0) {
                atomicAdd(&s_loss, (double)(lse - zt));
                if (above < 0.5f) atomicAdd(&s_cnt[0], 1u);
                if (above < 4.5f) atomicAdd(&s_cnt[1], 1u);
                atomicAdd(&s_cnt[2], 1u);
            }
        }
    }
    __syncthreads();
    if (threadIdx.x == 0 && s_cnt[2] != 0u) atomicAdd(reinterpret_cast<double*>(acc), s_loss);
    if (threadIdx.x < 3 && s_cnt[threadIdx.x] != 0u) atomicAdd(acc + 1 + threadIdx.x, (unsigned long long)s_cnt[threadIdx.x]);
}

template <typename T, bool SMOOTH, bool MIX>
__global__ void __launch_bounds__(XE_THREADS)
xent_bwd_kernel(const T* __restrict__ logits, const long long* __restrict__ target, const float* __restrict__ lse,
                const float* __restrict__ grad_out, T* __restrict__ dlogits, int B, int C, float eps,
                const float* __restrict__ mix)
{
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * (XE_THREADS / 32) + (threadIdx.x >> 5);
    if (row >= B) return;
    const float g = grad_out[0] / (float)B;
    const T* z = logits + (size_t)row * C;
    T* dz = dlogits + (size_t)row * C;
    const long long t = target[row];
    bool valid = t >= 0 && t < C;
    const float l = lse[row];
    const float eps_c = SMOOTH ? eps / (float)C : 0.f;        // smoothed target mass of every class
    const float hit = SMOOTH ? 1.f - eps + eps_c : 1.f;       // ... and of the target class
    if (MIX) {
        const long long tb = target[B - 1 - row];
        valid = valid && tb >= 0 && tb < C;
        const float lam = mix[0];
        const float wa = SMOOTH ? (1.f - eps) * lam : lam;                // target mass of class a
        const float wb = SMOOTH ? (1.f - eps) * (1.f - lam) : 1.f - lam;  // ... and of class b
        for (int j = lane; j < C; j += 32) {
            float q = eps_c;
            if (j == t) q += wa;
            if (j == tb) q += wb;
            const float p = __expf(to_f<T>(z[j]) - l) - q;
            dz[j] = from_f<T>(valid ? g * p : 0.f);
        }
        return;
    }
    for (int j = lane; j < C; j += 32) {
        float p = __expf(to_f<T>(z[j]) - l);
        if (j == t) p -= hit;
        else if (SMOOTH) p -= eps_c;
        dz[j] = from_f<T>(valid ? g * p : 0.f);
    }
}

}  // namespace

extern "C" {

// dtype: 0 = bf16 logits, 1 = fp32 logits; out3 must be zeroed by the caller (same stream);
// eps = label smoothing in [0, 1] (checked by the caller), 0 = plain cross-entropy;
// mix = device mix state (mix[0] = lam, partner row B-1-i), nullptr = one target per row
cudaError_t xent_launch_fwd(int dtype, const void* logits, const long long* target, float* lse, float* out3, int B,
                            int C, float eps, const float* mix, cudaStream_t st)
{
    const int grid = (B + XE_THREADS / 32 - 1) / (XE_THREADS / 32);
    const bool smooth = eps != 0.f;
    if (dtype == 0) {
        auto k = mix ? (smooth ? xent_fwd_kernel<__nv_bfloat16, true, true> : xent_fwd_kernel<__nv_bfloat16, false, true>)
                     : (smooth ? xent_fwd_kernel<__nv_bfloat16, true, false> : xent_fwd_kernel<__nv_bfloat16, false, false>);
        k<<<grid, XE_THREADS, 0, st>>>((const __nv_bfloat16*)logits, target, lse, out3, B, C, eps, mix);
    } else {
        auto k = mix ? (smooth ? xent_fwd_kernel<float, true, true> : xent_fwd_kernel<float, false, true>)
                     : (smooth ? xent_fwd_kernel<float, true, false> : xent_fwd_kernel<float, false, false>);
        k<<<grid, XE_THREADS, 0, st>>>((const float*)logits, target, lse, out3, B, C, eps, mix);
    }
    return cudaGetLastError();
}

// acc: [4] 8-byte device words, see xent_eval_kernel; B >= 1
cudaError_t xent_launch_eval(int dtype, const void* logits, const long long* target, unsigned long long* acc, int B,
                             int C, cudaStream_t st)
{
    const int grid = (B + XE_THREADS / 32 - 1) / (XE_THREADS / 32);
    if (dtype == 0)
        xent_eval_kernel<__nv_bfloat16><<<grid, XE_THREADS, 0, st>>>((const __nv_bfloat16*)logits, target, acc, B, C);
    else
        xent_eval_kernel<float><<<grid, XE_THREADS, 0, st>>>((const float*)logits, target, acc, B, C);
    return cudaGetLastError();
}

cudaError_t xent_launch_bwd(int dtype, const void* logits, const long long* target, const float* lse,
                            const float* grad_out, void* dlogits, int B, int C, float eps, const float* mix,
                            cudaStream_t st)
{
    const int grid = (B + XE_THREADS / 32 - 1) / (XE_THREADS / 32);
    const bool smooth = eps != 0.f;
    if (dtype == 0) {
        auto k = mix ? (smooth ? xent_bwd_kernel<__nv_bfloat16, true, true> : xent_bwd_kernel<__nv_bfloat16, false, true>)
                     : (smooth ? xent_bwd_kernel<__nv_bfloat16, true, false> : xent_bwd_kernel<__nv_bfloat16, false, false>);
        k<<<grid, XE_THREADS, 0, st>>>((const __nv_bfloat16*)logits, target, lse, grad_out, (__nv_bfloat16*)dlogits,
                                       B, C, eps, mix);
    } else {
        auto k = mix ? (smooth ? xent_bwd_kernel<float, true, true> : xent_bwd_kernel<float, false, true>)
                     : (smooth ? xent_bwd_kernel<float, true, false> : xent_bwd_kernel<float, false, false>);
        k<<<grid, XE_THREADS, 0, st>>>((const float*)logits, target, lse, grad_out, (float*)dlogits, B, C, eps, mix);
    }
    return cudaGetLastError();
}

}  // extern "C"
