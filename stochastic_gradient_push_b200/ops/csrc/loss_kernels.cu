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
//
// Knowledge distillation (teacher logits u, same shape and dtype as z; alpha in (0, 1], temperature T > 0):
//   loss_i = (1 - alpha) CE_eps(z_i, .) + alpha T^2 KL( softmax(u_i / T) || softmax(z_i / T) )
//   forward : one pass over z and u keeps three online log-sum-exps, lse of z, lseT of z / T and lseU of
//             u / T, and the KL numerator num = sum_j exp(u_j / T - m_u) (u_j - z_j) / T rescaled with the
//             softmax sum s_u, so KL = num / s_u - lseU + lseT; the rank count and sum_j z_j as above.
//             The three lse go to lse_out[row], lse_out[B + row], lse_out[2 B + row].
//   backward: dz_ij = g * ((1 - alpha) dCE_ij + alpha T (exp(z_ij / T - lseT_i) - exp(u_ij / T - lseU_i))) / B
// DISTILL is a template parameter next to SMOOTH and MIX: without teacher logits the DISTILL = false kernels
// run, whose code is the kernels' above (the teacher pointer, alpha and T are trailing, unused arguments).
// Row validity and accuracy are as above: an invalid row adds no loss (neither term) and gets a zero gradient.
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

// The distillation forward's row scan: one warp over student row z and teacher row u, each logit of both read
// once.  Besides xent_row_scan's lse, rank and sum_j z_j it keeps lseT = log sum_j exp(z_j / T) (sharing z's
// running max: max_j z_j / T = m / T for T > 0), lseU = log sum_j exp(u_j / T) and the KL numerator
// num = sum_j exp(u_j / T - m_u) (u_j - z_j) / T, rescaled with s_u as m_u grows.  Returns
// kl = KL(softmax(u / T) || softmax(z / T)) = num / s_u - lseU + lseT.
template <typename T, bool SMOOTH>
__device__ __forceinline__ void distill_row_scan(const T* z, const T* u, int C, float zt, float inv_t, int lane,
                                                 float& lse, float& lse_t, float& lse_u, float& kl, float& above,
                                                 float& sum_z)
{
    float m = -INFINITY, s = 0.f, st = 0.f, mu = -INFINITY, su = 0.f, num = 0.f, ab = 0.f, sz = 0.f;
    for (int j = lane; j < C; j += 32) {
        const float v = to_f<T>(z[j]);
        const float w = to_f<T>(u[j]) * inv_t;
        const float mn = fmaxf(m, v);
        s = s * __expf(m - mn) + __expf(v - mn);
        st = st * __expf((m - mn) * inv_t) + __expf((v - mn) * inv_t);
        m = mn;
        const float mun = fmaxf(mu, w);
        const float r = __expf(mu - mun), e = __expf(w - mun);
        su = su * r + e;
        num = num * r + e * (w - v * inv_t);
        mu = mun;
        ab += (v > zt) ? 1.f : 0.f;
        if (SMOOTH) sz += v;
    }
    const float mw = warp_max(m);
    s = warp_sum(s * __expf(m - mw));
    st = warp_sum(st * __expf((m - mw) * inv_t));
    const float muw = warp_max(mu);
    const float r = __expf(mu - muw);
    su = warp_sum(su * r);
    num = warp_sum(num * r);
    above = warp_sum(ab);
    sum_z = SMOOTH ? warp_sum(sz) : sz;
    lse = mw + __logf(s);
    lse_t = mw * inv_t + __logf(st);
    lse_u = muw + __logf(su);
    kl = num / su - lse_u + lse_t;
}

template <typename T, bool SMOOTH, bool MIX, bool DISTILL>
__global__ void __launch_bounds__(XE_THREADS)
xent_fwd_kernel(const T* __restrict__ logits, const long long* __restrict__ target, float* __restrict__ lse_out,
                float* __restrict__ out3, int B, int C, float eps, const float* __restrict__ mix,
                const T* __restrict__ teacher, float alpha, float temp)
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
        float lse, above, sum_z, lse_t = 0.f, lse_u = 0.f, kl = 0.f;
        const float inv_t = DISTILL ? 1.f / temp : 1.f;
        if (DISTILL)
            distill_row_scan<T, SMOOTH>(z, teacher + (size_t)row * C, C, zt, inv_t, lane, lse, lse_t, lse_u, kl,
                                        above, sum_z);
        else
            xent_row_scan<T, SMOOTH>(z, C, zt, lane, lse, above, sum_z);
        if (lane == 0) {
            lse_out[row] = lse;
            if (DISTILL) {
                lse_out[B + row] = lse_t;
                lse_out[2 * B + row] = lse_u;
            }
            if (valid) {
                const float inv_b = 1.f / (float)B;
                if (MIX) {
                    const float lam = mix[0];
                    const float zm = lam * zt + (1.f - lam) * zb;
                    float loss = SMOOTH ? lse - (1.f - eps) * zm - eps * (sum_z / (float)C) : lse - zm;
                    if (DISTILL) loss = (1.f - alpha) * loss + alpha * (temp * temp) * kl;
                    if (valid_b) atomicAdd(&s_acc[0], loss * inv_b);
                } else {
                    float loss = SMOOTH ? lse - (1.f - eps) * zt - eps * (sum_z / (float)C) : lse - zt;
                    if (DISTILL) loss = (1.f - alpha) * loss + alpha * (temp * temp) * kl;
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

// the distillation gradient of one logit from its cross-entropy gradient p (before the g / B factor):
// (1 - alpha) p + alpha T (exp(z / T - lseT) - exp(u / T - lseU))
__device__ __forceinline__ float distill_grad(float p, float v, float w, float alpha, float temp, float inv_t,
                                              float lse_t, float lse_u)
{
    return (1.f - alpha) * p + (alpha * temp) * (__expf(v * inv_t - lse_t) - __expf(w * inv_t - lse_u));
}

template <typename T, bool SMOOTH, bool MIX, bool DISTILL>
__global__ void __launch_bounds__(XE_THREADS)
xent_bwd_kernel(const T* __restrict__ logits, const long long* __restrict__ target, const float* __restrict__ lse,
                const float* __restrict__ grad_out, T* __restrict__ dlogits, int B, int C, float eps,
                const float* __restrict__ mix, const T* __restrict__ teacher, float alpha, float temp)
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
    const T* u = DISTILL ? teacher + (size_t)row * C : nullptr;
    const float inv_t = DISTILL ? 1.f / temp : 1.f;
    const float lse_t = DISTILL ? lse[B + row] : 0.f, lse_u = DISTILL ? lse[2 * B + row] : 0.f;
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
            const float v = to_f<T>(z[j]);
            float p = __expf(v - l) - q;
            if (DISTILL) p = distill_grad(p, v, to_f<T>(u[j]), alpha, temp, inv_t, lse_t, lse_u);
            dz[j] = from_f<T>(valid ? g * p : 0.f);
        }
        return;
    }
    for (int j = lane; j < C; j += 32) {
        const float v = to_f<T>(z[j]);
        float p = __expf(v - l);
        if (j == t) p -= hit;
        else if (SMOOTH) p -= eps_c;
        if (DISTILL) p = distill_grad(p, v, to_f<T>(u[j]), alpha, temp, inv_t, lse_t, lse_u);
        dz[j] = from_f<T>(valid ? g * p : 0.f);
    }
}

// the <SMOOTH, MIX> instantiation of the forward / backward kernel for one dtype and DISTILL flag
template <typename T, bool DISTILL>
auto xent_fwd_pick(bool smooth, bool mix)
{
    return mix ? (smooth ? xent_fwd_kernel<T, true, true, DISTILL> : xent_fwd_kernel<T, false, true, DISTILL>)
               : (smooth ? xent_fwd_kernel<T, true, false, DISTILL> : xent_fwd_kernel<T, false, false, DISTILL>);
}
template <typename T, bool DISTILL>
auto xent_bwd_pick(bool smooth, bool mix)
{
    return mix ? (smooth ? xent_bwd_kernel<T, true, true, DISTILL> : xent_bwd_kernel<T, false, true, DISTILL>)
               : (smooth ? xent_bwd_kernel<T, true, false, DISTILL> : xent_bwd_kernel<T, false, false, DISTILL>);
}

template <typename T>
void xent_fwd(const void* logits, const long long* target, float* lse, float* out3, int B, int C, float eps,
              const float* mix, const void* teacher, float alpha, float temp, cudaStream_t st)
{
    const int grid = (B + XE_THREADS / 32 - 1) / (XE_THREADS / 32);
    const bool smooth = eps != 0.f;
    auto k = teacher ? xent_fwd_pick<T, true>(smooth, mix != nullptr) : xent_fwd_pick<T, false>(smooth, mix != nullptr);
    k<<<grid, XE_THREADS, 0, st>>>((const T*)logits, target, lse, out3, B, C, eps, mix, (const T*)teacher, alpha,
                                   temp);
}

template <typename T>
void xent_bwd(const void* logits, const long long* target, const float* lse, const float* grad_out, void* dlogits,
              int B, int C, float eps, const float* mix, const void* teacher, float alpha, float temp, cudaStream_t st)
{
    const int grid = (B + XE_THREADS / 32 - 1) / (XE_THREADS / 32);
    const bool smooth = eps != 0.f;
    auto k = teacher ? xent_bwd_pick<T, true>(smooth, mix != nullptr) : xent_bwd_pick<T, false>(smooth, mix != nullptr);
    k<<<grid, XE_THREADS, 0, st>>>((const T*)logits, target, lse, grad_out, (T*)dlogits, B, C, eps, mix,
                                   (const T*)teacher, alpha, temp);
}

}  // namespace

extern "C" {

// dtype: 0 = bf16 logits, 1 = fp32 logits; out3 must be zeroed by the caller (same stream);
// eps = label smoothing in [0, 1] (checked by the caller), 0 = plain cross-entropy;
// mix = device mix state (mix[0] = lam, partner row B-1-i), nullptr = one target per row;
// teacher = teacher logits of the logits' shape and dtype, nullptr = no distillation (alpha and temp unused);
// with a teacher, alpha in (0, 1] and temp > 0 (checked by the caller), and lse holds 3 B floats (else B)
cudaError_t xent_launch_fwd(int dtype, const void* logits, const long long* target, float* lse, float* out3, int B,
                            int C, float eps, const float* mix, const void* teacher, float alpha, float temp,
                            cudaStream_t st)
{
    if (dtype == 0)
        xent_fwd<__nv_bfloat16>(logits, target, lse, out3, B, C, eps, mix, teacher, alpha, temp, st);
    else
        xent_fwd<float>(logits, target, lse, out3, B, C, eps, mix, teacher, alpha, temp, st);
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
                            const void* teacher, float alpha, float temp, cudaStream_t st)
{
    if (dtype == 0)
        xent_bwd<__nv_bfloat16>(logits, target, lse, grad_out, dlogits, B, C, eps, mix, teacher, alpha, temp, st);
    else
        xent_bwd<float>(logits, target, lse, grad_out, dlogits, B, C, eps, mix, teacher, alpha, temp, st);
    return cudaGetLastError();
}

}  // extern "C"
