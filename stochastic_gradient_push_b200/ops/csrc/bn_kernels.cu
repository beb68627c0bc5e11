// Fused NHWC BatchNorm (+residual add) (+ReLU), training forward and backward,
// for sm_90a.  The framework's native channels-last BatchNorm + separate ReLU / add
// kernels take most of the ResNet-50 step at batch 256, far more than the tensor-core
// convolutions: these kernels are memory-bound, so the fix is fewer passes over HBM.
//
//   forward :  stats (1 read of x)  ->  finalize (C threads)  ->  apply
//              y = relu(x*scale + shift [+ res])   (1 read of x [+res], 1 write)
//   backward:  reduce (dy, x [,y]) -> finalize -> dx = c1*dz - c2*x + c3
//              the ReLU mask is recomputed from x*scale+shift (no mask tensor, no
//              extra read); with a residual the mask comes from the saved output
//              and dz is written once because it IS the residual branch's grad.
//   stochastic depth (DROP): the BN output of a residual block is scaled per sample before the add,
//              y = relu((x*scale + shift)*s[row / HW] + res); the backward reduces s*dz and forms
//              dx from s*dz, the residual-branch gradient dz stays unscaled
//   precise statistics: the finalize adds the batch statistics to an fp64 accumulator
//              instead of the running update; one commit launch per pass writes
//              running = fp32(sum / K) for every layer (GossipTrainer.update_bn)
//
// Layout: x is [M, C] row-major (M = N*H*W, NHWC), C % 8 == 0, C <= 2048.
// One thread owns 8 channels and strides over rows, so per-channel constants
// live in registers and every global access is a full 16-byte vector.  bf16:
// 8 consecutive channels, one vector.  fp32 (SPLIT map): channels [4cv, 4cv+4)
// and [C/2+4cv, C/2+4cv+4), two vectors that each continue the neighbouring
// lane's, so every warp access covers whole 128-byte lines (8 consecutive fp32
// channels would be 32 B per lane: each access would use half of every sector
// and the second one would fetch the same sectors from L2 again).
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdlib.h>

#include "vec_io.cuh"

#define BN_THREADS 256
#define BN_VEC 8
#define BN_UNROLL 4
// rows in flight per thread and tensor.  A thread's vector is 8 channels = 16 B of bf16 but 32 B
// of fp32 (8 registers per load), so fp32 uses half the unroll: the same bytes in flight and the
// same register footprint as bf16.  (With the bf16 unroll the fp32 instantiations spilled 250-460
// bytes per thread under their 64 / 80-register caps.)
template <typename T> struct Unroll {
    static constexpr int N = sizeof(T) == 4 ? 2 : 4;        // stats / apply / dx
    static constexpr int RED = sizeof(T) == 4 ? 1 : 2;      // backward reduce (up to 3 tensors)
};

namespace {

// thread -> (channels, row lane) mapping shared by all kernels.  SPLIT: the fp32 map above
// (element i < 4 is channel off + i, element i >= 4 is channel off + h + i - 4).
template <bool SPLIT>
struct Map {
    int tpr;        // threads per row  = C / 8
    int rpi;        // rows per CTA iteration = 256 / tpr
    int cv;         // this thread's channel-vector index
    int rl;         // this thread's row lane
    int off;        // first channel of the thread's first half
    int h;          // channel distance from the first half to the second (4: consecutive)
    bool active;
    __device__ __forceinline__ Map(int C) {
        tpr = C / BN_VEC;
        rpi = BN_THREADS / tpr;
        cv = threadIdx.x % tpr;
        rl = threadIdx.x / tpr;
        off = SPLIT ? cv * 4 : cv * BN_VEC;
        h = SPLIT ? C / 2 : 4;
        active = rl < rpi;
    }
};

// block reduce of 2 x 8 per-thread accumulators across the row lanes that share
// a channel vector, then one partial row per CTA: partial[blockIdx][2][C]
template <bool SPLIT>
__device__ __forceinline__ void reduce_store_partials(const Map<SPLIT>& mp, const F8& a, const F8& b,
                                                      float* __restrict__ partial, int C)
{
    __shared__ float sm[BN_THREADS * 16];
    float* mine = sm + threadIdx.x * 16;
#pragma unroll
    for (int i = 0; i < 8; ++i) { mine[i] = mp.active ? a.v[i] : 0.f; mine[8 + i] = mp.active ? b.v[i] : 0.f; }
    __syncthreads();
    if (threadIdx.x < mp.tpr) {
        float acc[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) acc[i] = 0.f;
        for (int r = 0; r < mp.rpi; ++r) {
            const float* o = sm + (r * mp.tpr + threadIdx.x) * 16;
#pragma unroll
            for (int i = 0; i < 16; ++i) acc[i] += o[i];
        }
        // thread threadIdx.x stands for channel vector cv = threadIdx.x (row lane 0)
        const unsigned off = SPLIT ? threadIdx.x * 4 : threadIdx.x * BN_VEC;
        float* out = partial + (size_t)blockIdx.x * 2 * C + off;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int j = i < 4 ? i : mp.h + i - 4;
            out[j] = acc[i]; out[C + j] = acc[8 + i];
        }
    }
}

}  // namespace

// ---------------------------------------------------------------------------
// forward: statistics
// ---------------------------------------------------------------------------
template <typename T, bool SPLIT = false>
__global__ void __launch_bounds__(BN_THREADS, 4)
bn_stats_kernel(const T* __restrict__ x, float* __restrict__ partial, long long M, int C)
{
    const Map<SPLIT> mp(C);
    F8 s, q;
#pragma unroll
    for (int i = 0; i < 8; ++i) { s.v[i] = 0.f; q.v[i] = 0.f; }
    if (mp.active) {
        const long long stride = (long long)gridDim.x * mp.rpi;
        long long r = (long long)blockIdx.x * mp.rpi + mp.rl;
        const T* base = x + mp.off;
        // shifted sums: accumulate (x - K) with K = x[row 0] so that
        // var = E[(x-K)^2] - E[x-K]^2 does not cancel when |mean| >> std
        const F8 k = Io<T>::load(base, mp.h);
        if (blockIdx.x == 0 && mp.rl == 0) {
            float* krow = partial + (size_t)gridDim.x * 2 * C + mp.off;
#pragma unroll
            for (int i = 0; i < 8; ++i) krow[i < 4 ? i : mp.h + i - 4] = k.v[i];
        }
        constexpr int UN = Unroll<T>::N;
        for (; r + (UN - 1) * stride < M; r += UN * stride) {
            typename Io<T>::raw_t raw[UN];
#pragma unroll
            for (int u = 0; u < UN; ++u) raw[u] = Io<T>::load_raw(base + (r + u * stride) * C, mp.h);
#pragma unroll
            for (int u = 0; u < UN; ++u) {
                const F8 d = Io<T>::decode(raw[u]);
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const float c = d.v[i] - k.v[i];
                    s.v[i] += c; q.v[i] = fmaf(c, c, q.v[i]);
                }
            }
        }
        for (; r < M; r += stride) {
            const F8 d = Io<T>::load(base + r * C, mp.h);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float c = d.v[i] - k.v[i];
                s.v[i] += c; q.v[i] = fmaf(c, c, q.v[i]);
            }
        }
    }
    reduce_store_partials(mp, s, q, partial, C);
}

// Finalize kernels: a CTA owns 32 channels; its 1024 threads are 32 partial-row
// lanes x 32 channels, so the G (<= 592) partial rows are summed with ~G/128
// dependent steps per thread instead of G (a one-thread-per-channel loop over G
// L2-latency-bound loads took ~78 us per launch -- longer than the streaming
// kernels it finalises).
#define BN_FIN_THREADS 1024
#define BN_FIN_ILP 10          // rows per lane in flight (G <= 592 -> 19 rows per lane: two batches)

__device__ __forceinline__ void sum_partials(const float* __restrict__ partial, int G, int C,
                                             float& s_out, float& q_out, bool& owner, int& ch)
{
    __shared__ float sm_s[32][33];
    __shared__ float sm_q[32][33];
    const int cl = threadIdx.x & 31;
    const int lane = threadIdx.x >> 5;
    ch = blockIdx.x * 32 + cl;
    // All of a lane's rows are requested before any is consumed: the partials sit in L2, each
    // dependent load is an L2 round trip, and a two-deep loop made these 106 launches per step
    // latency-bound.
    float s0 = 0.f, s1 = 0.f, q0 = 0.f, q1 = 0.f;
    if (ch < C) {
        for (int g0 = lane; g0 < G; g0 += 32 * BN_FIN_ILP) {
            float sv[BN_FIN_ILP], qv[BN_FIN_ILP];
#pragma unroll
            for (int u = 0; u < BN_FIN_ILP; ++u) {
                const int g = g0 + 32 * u;
                const bool ok = g < G;
                sv[u] = ok ? partial[(size_t)g * 2 * C + ch] : 0.f;
                qv[u] = ok ? partial[(size_t)g * 2 * C + C + ch] : 0.f;
            }
#pragma unroll
            for (int u = 0; u < BN_FIN_ILP; u += 2) {
                s0 += sv[u]; q0 += qv[u];
                s1 += sv[u + 1]; q1 += qv[u + 1];
            }
        }
    }
    sm_s[lane][cl] = s0 + s1;
    sm_q[lane][cl] = q0 + q1;
    __syncthreads();
    owner = (lane == 0) && (ch < C);
    float s = 0.f, q = 0.f;
    if (owner) {
#pragma unroll
        for (int l = 0; l < 32; ++l) { s += sm_s[l][cl]; q += sm_q[l][cl]; }
    }
    s_out = s;
    q_out = q;
}

// acc (accumulate mode, precise BatchNorm statistics): acc[c] += mu, acc[C + c] += unbiased variance, the
// fp32 values the running update would blend in; the running buffers and nbt are then left alone
__global__ void __launch_bounds__(BN_FIN_THREADS)
bn_stats_finalize_kernel(const float* __restrict__ partial, int G, long long M, int C,
                         const float* __restrict__ gamma, const float* __restrict__ beta,
                         float* running_mean, float* running_var, long long* nbt, double* acc,
                         float momentum, float eps,
                         float* __restrict__ mean, float* __restrict__ invstd,
                         float* __restrict__ scale, float* __restrict__ shift)
{
    float s, q; bool owner; int c;
    sum_partials(partial, G, C, s, q, owner, c);
    if (blockIdx.x == 0 && threadIdx.x == 0 && nbt != nullptr && acc == nullptr) *nbt += 1;
    if (!owner) return;
    const float k = partial[(size_t)G * 2 * C + c];          // the shift K = x[row 0]
    const float inv_m = 1.f / (float)M;
    const float ds = s * inv_m;
    const float mu = k + ds;
    const float var = fmaxf(fmaf(-ds, ds, q * inv_m), 0.f);
    const float is = rsqrtf(var + eps);
    mean[c] = mu;
    invstd[c] = is;
    const float sc = gamma[c] * is;
    scale[c] = sc;
    shift[c] = fmaf(-mu, sc, beta[c]);
    const float unbiased = (M > 1) ? var * ((float)M / (float)(M - 1)) : var;
    if (acc != nullptr) {
        acc[c] += (double)mu;
        acc[C + c] += (double)unbiased;
    } else if (running_mean != nullptr) {
        running_mean[c] = fmaf(momentum, mu - running_mean[c], running_mean[c]);
        running_var[c] = fmaf(momentum, unbiased - running_var[c], running_var[c]);
    }
}

// ---------------------------------------------------------------------------
// precise BatchNorm statistics: running = fp32(acc / K) for every layer, ONE launch per pass.  The table
// is the kernel's __grid_constant__ parameter (as in accum_kernels.cu), one thread per channel; a row holds
// the prefix of its first channel, so a thread finds its layer by a binary search over the table.
// ---------------------------------------------------------------------------
#define BN_COMMIT_THREADS 256
#define BN_COMMIT_MAX_SEGS 1000           // 1000 x 32 B + the header fits the 32,764-byte parameter space

struct BnCommitSeg {                      // 32 bytes
    const double* acc;                    // [2C]: sum of the batch means, then of the unbiased variances
    float* rmean;
    float* rvar;
    int C;
    int c0;                               // flat index of the layer's first channel
};

struct BnCommitTable {
    int nseg;
    int total;
    BnCommitSeg seg[BN_COMMIT_MAX_SEGS];
};

static_assert(sizeof(BnCommitSeg) == 32, "BnCommitSeg layout");
static_assert(sizeof(BnCommitTable) <= 32764, "the commit table must fit the kernel parameter space");

__global__ void __launch_bounds__(BN_COMMIT_THREADS)
bn_stats_commit_kernel(const __grid_constant__ BnCommitTable tab, double k)
{
    const int i = blockIdx.x * BN_COMMIT_THREADS + threadIdx.x;
    if (i >= tab.total) return;
    int lo = 0, hi = tab.nseg - 1;        // the last layer whose first channel is <= i
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (tab.seg[mid].c0 <= i) lo = mid; else hi = mid - 1;
    }
    const BnCommitSeg& sg = tab.seg[lo];
    const int c = i - sg.c0;
    sg.rmean[c] = __double2float_rn(__ddiv_rn(sg.acc[c], k));
    sg.rvar[c] = __double2float_rn(__ddiv_rn(sg.acc[sg.C + c], k));
}

// eval mode: scale/shift from the running statistics
__global__ void bn_eval_coeff_kernel(int C, const float* __restrict__ gamma, const float* __restrict__ beta,
                                     const float* __restrict__ running_mean,
                                     const float* __restrict__ running_var, float eps,
                                     float* __restrict__ scale, float* __restrict__ shift)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    const float sc = gamma[c] * rsqrtf(running_var[c] + eps);
    scale[c] = sc;
    shift[c] = fmaf(-running_mean[c], sc, beta[c]);
}

// ---------------------------------------------------------------------------
// forward: apply   y = act(x*scale + shift [+ res])
// MASK: also mask[M, C/8], bit i of byte j = (y[row, 8j+i] > 0) -- the ReLU mask of a residual block's
// output for the next block's conv1 dgrad (MODE 3 of conv1x1_kernels.cu), 1/32 of y's fp32 bytes.
// With the SPLIT map a byte's 8 channels belong to two neighbouring lanes (C % 16 == 0): the even
// lane of a pair stores the byte of their first halves, the odd lane the byte of their second halves.
// ---------------------------------------------------------------------------
// DROP (stochastic depth, with RELU && ADD): y = relu((x*scale + shift)*s[row / hw] + res), s the residual
// branch's per-sample scale [M / hw]; the mask is still that of y.
template <typename T, bool RELU, bool ADD, bool MASK, bool SPLIT, bool DROP>
__device__ __forceinline__ void
bn_apply_body(const T* __restrict__ x, const T* __restrict__ res, const float* __restrict__ scale,
              const float* __restrict__ shift, T* __restrict__ y, uint8_t* __restrict__ mask, long long M, int C,
              const float* __restrict__ sdrop, int hw)
{
    const Map<SPLIT> mp(C);
    if (!mp.active) return;
    const F8 sc = load_c8(scale + mp.off, mp.h);
    const F8 sh = load_c8(shift + mp.off, mp.h);
    const long long stride = (long long)gridDim.x * mp.rpi;
    const long long off = mp.off;
    constexpr int UN = Unroll<T>::N;
    for (long long r = (long long)blockIdx.x * mp.rpi + mp.rl; r < M; r += UN * stride) {
        typename Io<T>::raw_t dr[UN], ar[UN];
#pragma unroll
        for (int u = 0; u < UN; ++u) {
            const long long rr = r + u * stride;
            if (rr < M) {
                dr[u] = Io<T>::load_raw(x + rr * C + off, mp.h);
                if (ADD) ar[u] = Io<T>::load_raw(res + rr * C + off, mp.h);
            }
        }
#pragma unroll
        for (int u = 0; u < UN; ++u) {
            const long long rr = r + u * stride;
            if (rr < M) {
                const F8 d = Io<T>::decode(dr[u]);
                F8 a;
                if (ADD) a = Io<T>::decode(ar[u]);
                const float sr = DROP ? __ldg(sdrop + (int)rr / hw) : 1.f;
                F8 o;
                uint32_t bits = 0;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    float v = fmaf(d.v[i], sc.v[i], sh.v[i]);
                    if (DROP) v = fmaf(v, sr, a.v[i]);
                    else if (ADD) v += a.v[i];
                    if (RELU) v = fmaxf(v, 0.f);
                    o.v[i] = v;
                    if (MASK) {     // the sign of y as stored (bf16 rounds the tiniest positives to 0)
                        const float vs = sizeof(T) == 2 ? __bfloat162float(__float2bfloat16_rn(v)) : v;
                        bits |= (vs > 0.f ? 1u : 0u) << i;
                    }
                }
                Io<T>::store(y + rr * C + off, o, mp.h);
                if (MASK && !SPLIT) mask[rr * (C / BN_VEC) + mp.cv] = (uint8_t)bits;
                if (MASK && SPLIT) {      // both lanes of a pair are on this row
                    const uint32_t pb = __shfl_xor_sync(3u << (threadIdx.x & 30), bits, 1);
                    const bool odd = mp.cv & 1;
                    const uint32_t byte = odd ? (pb >> 4) | (bits & 0xf0u) : (bits & 0x0fu) | (pb << 4);
                    mask[rr * (C / BN_VEC) + (odd ? C / 16 : 0) + (mp.cv >> 1)] = (uint8_t)byte;
                }
            }
        }
    }
}

template <typename T, bool RELU, bool ADD, bool MASK = false, bool SPLIT = false>
__global__ void __launch_bounds__(BN_THREADS, (sizeof(T) == 4 && ADD) ? 3 : 4)     // fp32 + residual: 80 registers
bn_apply_kernel(const T* __restrict__ x, const T* __restrict__ res, const float* __restrict__ scale,
                const float* __restrict__ shift, T* __restrict__ y, uint8_t* __restrict__ mask, long long M, int C)
{
    bn_apply_body<T, RELU, ADD, MASK, SPLIT, false>(x, res, scale, shift, y, mask, M, C, nullptr, 1);
}

// 3 CTAs per SM for both dtypes: with the per-row scale the bf16 kernel spilled under a 64-register cap
template <typename T, bool MASK, bool SPLIT>
__global__ void __launch_bounds__(BN_THREADS, 3)
bn_apply_drop_kernel(const T* __restrict__ x, const T* __restrict__ res, const float* __restrict__ scale,
                     const float* __restrict__ shift, T* __restrict__ y, uint8_t* __restrict__ mask, long long M,
                     int C, const float* __restrict__ sdrop, int hw)
{
    bn_apply_body<T, true, true, MASK, SPLIT, true>(x, res, scale, shift, y, mask, M, C, sdrop, hw);
}

// ---------------------------------------------------------------------------
// backward: reduce   partial[.][0] = sum dz ; partial[.][1] = sum dz * xhat
// MODE 0: dz = dy            MODE 1: dz = dy * (x*scale+shift > 0)
// MODE 2: dz = dy * (y > 0), dz is also written (gradient of the residual branch)
// DROP (MODE 2): dz is written unscaled, the partials are those of s[row / hw] * dz, the BN output's gradient
// ---------------------------------------------------------------------------
template <typename T, int MODE, bool SPLIT, bool DROP>
__device__ __forceinline__ void
bn_bwd_reduce_body(const T* __restrict__ dy, const T* __restrict__ x, const T* __restrict__ y,
                   const float* __restrict__ scale, const float* __restrict__ shift,
                   const float* __restrict__ mean, const float* __restrict__ invstd,
                   float* __restrict__ partial, T* __restrict__ dz_out, long long M, int C,
                   const float* __restrict__ sdrop, int hw)
{
    const Map<SPLIT> mp(C);
    F8 s, q;
#pragma unroll
    for (int i = 0; i < 8; ++i) { s.v[i] = 0.f; q.v[i] = 0.f; }
    if (mp.active) {
        const long long off = mp.off;
        const F8 mu = load_c8(mean + off, mp.h);
        const F8 is = load_c8(invstd + off, mp.h);
        F8 sc, sh;
        if (MODE == 1) { sc = load_c8(scale + off, mp.h); sh = load_c8(shift + off, mp.h); }
        const long long stride = (long long)gridDim.x * mp.rpi;
        // DROP: one row in flight per tensor (bf16 spilled at two under the 80-register cap)
        constexpr int UN = DROP ? 1 : Unroll<T>::RED;
        for (long long r = (long long)blockIdx.x * mp.rpi + mp.rl; r < M; r += UN * stride) {
            typename Io<T>::raw_t gr[UN], xr[UN], yr[UN];
            float srv[UN];
#pragma unroll
            for (int u = 0; u < UN; ++u) {
                const long long rr = r + u * stride;
                if (rr < M) {
                    if (DROP) srv[u] = __ldg(sdrop + (int)rr / hw);
                    gr[u] = Io<T>::load_raw(dy + rr * C + off, mp.h);
                    xr[u] = Io<T>::load_raw(x + rr * C + off, mp.h);
                    if (MODE == 2) yr[u] = Io<T>::load_raw(y + rr * C + off, mp.h);
                }
            }
#pragma unroll
            for (int u = 0; u < UN; ++u) {
                const long long rr = r + u * stride;
                if (rr < M) {
                    const F8 g = Io<T>::decode(gr[u]);
                    const F8 d = Io<T>::decode(xr[u]);
                    F8 o;
                    if (MODE == 2) o = Io<T>::decode(yr[u]);
                    const float sr = DROP ? srv[u] : 1.f;
                    F8 dz;
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        float gz = g.v[i];
                        if (MODE == 1) gz = (fmaf(d.v[i], sc.v[i], sh.v[i]) > 0.f) ? gz : 0.f;
                        if (MODE == 2) gz = (o.v[i] > 0.f) ? gz : 0.f;
                        dz.v[i] = gz;
                        if (DROP) gz *= sr;
                        s.v[i] += gz;
                        q.v[i] = fmaf(gz, (d.v[i] - mu.v[i]) * is.v[i], q.v[i]);
                    }
                    if (MODE == 2) Io<T>::store(dz_out + rr * C + off, dz, mp.h);
                }
            }
        }
    }
    reduce_store_partials(mp, s, q, partial, C);
}

template <typename T, int MODE, bool SPLIT = false>
__global__ void __launch_bounds__(BN_THREADS, 3)
bn_bwd_reduce_kernel(const T* __restrict__ dy, const T* __restrict__ x, const T* __restrict__ y,
                     const float* __restrict__ scale, const float* __restrict__ shift,
                     const float* __restrict__ mean, const float* __restrict__ invstd,
                     float* __restrict__ partial, T* __restrict__ dz_out, long long M, int C)
{
    bn_bwd_reduce_body<T, MODE, SPLIT, false>(dy, x, y, scale, shift, mean, invstd, partial, dz_out, M, C, nullptr, 1);
}

template <typename T, bool SPLIT>
__global__ void __launch_bounds__(BN_THREADS, 3)
bn_bwd_reduce_drop_kernel(const T* __restrict__ dy, const T* __restrict__ x, const T* __restrict__ y,
                          const float* __restrict__ mean, const float* __restrict__ invstd,
                          float* __restrict__ partial, T* __restrict__ dz_out, long long M, int C,
                          const float* __restrict__ sdrop, int hw)
{
    bn_bwd_reduce_body<T, 2, SPLIT, true>(dy, x, y, nullptr, nullptr, mean, invstd, partial, dz_out, M, C, sdrop, hw);
}

// per-channel: grad_gamma, grad_beta and the dx coefficients
//   dx = scale*(dz - sdz/M - xhat*sdzx/M) = c1*dz - c2*x + c3
__global__ void __launch_bounds__(BN_FIN_THREADS)
bn_bwd_finalize_kernel(const float* __restrict__ partial, int G, long long M, int C,
                       const float* __restrict__ scale, const float* __restrict__ mean,
                       const float* __restrict__ invstd,
                       float* __restrict__ grad_gamma, float* __restrict__ grad_beta,
                       float* __restrict__ c2, float* __restrict__ c3)
{
    float s, q; bool owner; int c;
    sum_partials(partial, G, C, s, q, owner, c);
    if (!owner) return;
    grad_beta[c] = s;
    grad_gamma[c] = q;
    const float inv_m = 1.f / (float)M;
    const float k1 = s * inv_m, k2 = q * inv_m;
    const float a = invstd[c] * k2;          // xhat*k2 = x*a - mean*a
    const float sc = scale[c];
    c2[c] = sc * a;
    c3[c] = sc * (mean[c] * a - k1);
}

// MODE 0/2: dz given directly (dy, or the dz written by the reduce kernel)
// MODE 1  : dz = dy * (x*scale+shift > 0) recomputed
// DROP (MODE 0): dx = c1*(s[row / hw]*dz) - c2*x + c3 for the unscaled residual-branch gradient dz
template <typename T, int MODE, bool SPLIT, bool DROP>
__device__ __forceinline__ void
bn_bwd_dx_body(const T* __restrict__ dz_in, const T* __restrict__ x, const float* __restrict__ scale,
               const float* __restrict__ shift, const float* __restrict__ c2,
               const float* __restrict__ c3, T* __restrict__ dx, long long M, int C,
               const float* __restrict__ sdrop, int hw)
{
    // fp32 MODE 1 reads the shift from shared memory at each row: 4 x 8 constants in registers
    // next to 2 x 2 x 8 loads in flight do not fit its 80-register cap (they spilled)
    constexpr bool SH_SMEM = MODE == 1 && sizeof(T) == 4;
    __shared__ float sh_s[SH_SMEM ? 2048 : 1];
    if (SH_SMEM) {
        for (int c = threadIdx.x; c < C; c += BN_THREADS) sh_s[c] = shift[c];
        __syncthreads();
    }
    const Map<SPLIT> mp(C);
    if (!mp.active) return;
    const long long off = mp.off;
    const F8 k1 = load_c8(scale + off, mp.h);
    const F8 k2 = load_c8(c2 + off, mp.h);
    const F8 k3 = load_c8(c3 + off, mp.h);
    F8 sh;
    if (MODE == 1 && !SH_SMEM) sh = load_c8(shift + off, mp.h);
    const long long stride = (long long)gridDim.x * mp.rpi;
    constexpr int UN = Unroll<T>::N;
    for (long long r = (long long)blockIdx.x * mp.rpi + mp.rl; r < M; r += UN * stride) {
        typename Io<T>::raw_t gr[UN], xr[UN];
#pragma unroll
        for (int u = 0; u < UN; ++u) {
            const long long rr = r + u * stride;
            if (rr < M) {
                gr[u] = Io<T>::load_raw(dz_in + rr * C + off, mp.h);
                xr[u] = Io<T>::load_raw(x + rr * C + off, mp.h);
            }
        }
#pragma unroll
        for (int u = 0; u < UN; ++u) {
            const long long rr = r + u * stride;
            if (rr < M) {
                const F8 g = Io<T>::decode(gr[u]);
                const F8 d = Io<T>::decode(xr[u]);
                if (SH_SMEM) sh = load_c8(sh_s + off, mp.h);
                const float sr = DROP ? __ldg(sdrop + (int)rr / hw) : 1.f;
                F8 o;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    float gz = g.v[i];
                    if (MODE == 1) gz = (fmaf(d.v[i], k1.v[i], sh.v[i]) > 0.f) ? gz : 0.f;
                    if (DROP) gz *= sr;
                    o.v[i] = fmaf(k1.v[i], gz, fmaf(-k2.v[i], d.v[i], k3.v[i]));
                }
                Io<T>::store(dx + rr * C + off, o, mp.h);
            }
        }
    }
}

template <typename T, int MODE, bool SPLIT = false>
__global__ void __launch_bounds__(BN_THREADS, 3)
bn_bwd_dx_kernel(const T* __restrict__ dz_in, const T* __restrict__ x, const float* __restrict__ scale,
                 const float* __restrict__ shift, const float* __restrict__ c2,
                 const float* __restrict__ c3, T* __restrict__ dx, long long M, int C)
{
    bn_bwd_dx_body<T, MODE, SPLIT, false>(dz_in, x, scale, shift, c2, c3, dx, M, C, nullptr, 1);
}

template <typename T, bool SPLIT>
__global__ void __launch_bounds__(BN_THREADS, 3)
bn_bwd_dx_drop_kernel(const T* __restrict__ dz_in, const T* __restrict__ x, const float* __restrict__ scale,
                      const float* __restrict__ c2, const float* __restrict__ c3, T* __restrict__ dx, long long M,
                      int C, const float* __restrict__ sdrop, int hw)
{
    bn_bwd_dx_body<T, 0, SPLIT, true>(dz_in, x, scale, nullptr, c2, c3, dx, M, C, sdrop, hw);
}

// ---------------------------------------------------------------------------
// launchers (C linkage; dtype: 0 = bf16, 1 = fp32)
// ---------------------------------------------------------------------------
static inline int bn_grid(long long M, int C, int per_sm, int unroll = BN_UNROLL)
{
    const int tpr = C / BN_VEC;
    const int rpi = BN_THREADS / tpr;
    long long iters = (M + rpi - 1) / rpi;
    long long g = (iters + unroll - 1) / unroll;
    const long long cap = 132LL * per_sm;
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (int)g;
}

// fp32 channel map: 1 = SPLIT (default), 0 = the consecutive map of the bf16 kernels with the launch
// sizing it had.  SGP_B200_BN_F32_MAP=0 selects 0 at start-up; bn_f32_map() switches at run time.
static int g_bn_f32_map = -1;

static bool f32_split()
{
    if (g_bn_f32_map < 0) {
        const char* e = getenv("SGP_B200_BN_F32_MAP");
        g_bn_f32_map = (e != nullptr && e[0] == '0') ? 0 : 1;
    }
    return g_bn_f32_map == 1;
}

extern "C" {

// returns the map in use; value >= 0 selects a map for the launches that follow
int bn_f32_map(int value)
{
    const int cur = f32_split() ? 1 : 0;
    if (value >= 0) g_bn_f32_map = value ? 1 : 0;
    return cur;
}

int bn_supported(long long M, int C) { return (C % BN_VEC == 0) && (C / BN_VEC <= BN_THREADS) && M > 0; }

int bn_partial_rows(long long M, int C) { return bn_grid(M, C, 4); }

// the backward reduce kernel holds 3 CTAs per SM (80 registers): a grid of 4 per SM
// would run as 1.33 waves with an idle tail (ncu: 4.4 TB/s vs 5.9 TB/s for its siblings)
int bn_partial_rows_bwd(long long M, int C) { return bn_grid(M, C, 3); }

cudaError_t bn_launch_stats(int dtype, const void* x, float* partial, long long M, int C, int G,
                            cudaStream_t st)
{
    if (dtype == 0) bn_stats_kernel<__nv_bfloat16><<<G, BN_THREADS, 0, st>>>((const __nv_bfloat16*)x, partial, M, C);
    else if (f32_split()) bn_stats_kernel<float, true><<<G, BN_THREADS, 0, st>>>((const float*)x, partial, M, C);
    else            bn_stats_kernel<float><<<G, BN_THREADS, 0, st>>>((const float*)x, partial, M, C);
    return cudaGetLastError();
}

cudaError_t bn_launch_stats_finalize(const float* partial, int G, long long M, int C, const float* gamma,
                                     const float* beta, float* rmean, float* rvar, long long* nbt, double* acc,
                                     float momentum, float eps, float* mean, float* invstd,
                                     float* scale, float* shift, cudaStream_t st)
{
    bn_stats_finalize_kernel<<<(C + 31) / 32, BN_FIN_THREADS, 0, st>>>(partial, G, M, C, gamma, beta, rmean, rvar,
                                                              nbt, acc, momentum, eps, mean, invstd, scale, shift);
    return cudaGetLastError();
}

int bn_commit_max_segs() { return BN_COMMIT_MAX_SEGS; }

// rows: host int64 [nseg, 4] = (acc address, running_mean address, running_var address, C >= 1),
// 1 <= nseg <= BN_COMMIT_MAX_SEGS, fewer than 2^31 channels in all; k >= 1.  One launch.
cudaError_t bn_launch_stats_commit(const long long* rows, int nseg, double k, cudaStream_t st)
{
    if (nseg < 1 || nseg > BN_COMMIT_MAX_SEGS || !(k >= 1.0)) return cudaErrorInvalidValue;
    BnCommitTable tab;
    long long total = 0;
    for (int i = 0; i < nseg; ++i) {
        const long long* r = rows + 4 * i;
        if (r[3] < 1) return cudaErrorInvalidValue;
        tab.seg[i].acc = reinterpret_cast<const double*>(r[0]);
        tab.seg[i].rmean = reinterpret_cast<float*>(r[1]);
        tab.seg[i].rvar = reinterpret_cast<float*>(r[2]);
        tab.seg[i].C = (int)r[3];
        tab.seg[i].c0 = (int)total;
        total += r[3];
        if (total > 0x7fffffffLL) return cudaErrorInvalidValue;
    }
    tab.nseg = nseg;
    tab.total = (int)total;
    bn_stats_commit_kernel<<<(unsigned)((total + BN_COMMIT_THREADS - 1) / BN_COMMIT_THREADS), BN_COMMIT_THREADS, 0,
                             st>>>(tab, k);
    return cudaGetLastError();
}

cudaError_t bn_launch_eval_coeff(int C, const float* gamma, const float* beta, const float* rmean,
                                 const float* rvar, float eps, float* scale, float* shift, cudaStream_t st)
{
    bn_eval_coeff_kernel<<<(C + 127) / 128, 128, 0, st>>>(C, gamma, beta, rmean, rvar, eps, scale, shift);
    return cudaGetLastError();
}

#define BN_APPLY(T, R, A, S) bn_apply_kernel<T, R, A, false, S><<<G, BN_THREADS, 0, st>>>( \
    (const T*)x, (const T*)res, scale, shift, (T*)y, nullptr, M, C)

// mask (nullable; relu && add only): the 1-bit ReLU mask [M, C/8] of y (fp32 split map: C % 16 == 0).
// G <= 0: the default grid
cudaError_t bn_launch_apply(int dtype, int relu, int add, const void* x, const void* res,
                            const float* scale, const float* shift, void* y, uint8_t* mask, long long M, int C,
                            int G, cudaStream_t st)
{
    const bool split = dtype == 1 && f32_split();
    if (G <= 0) G = bn_grid(M, C, (dtype == 1 && add) ? 6 : 8);   // fp32 + residual holds 3 CTAs/SM: 2 waves
    if (mask != nullptr) {
        if (!(relu && add) || (split && C % 16 != 0)) return cudaErrorInvalidValue;
        if (dtype == 0) bn_apply_kernel<__nv_bfloat16, true, true, true><<<G, BN_THREADS, 0, st>>>(
            (const __nv_bfloat16*)x, (const __nv_bfloat16*)res, scale, shift, (__nv_bfloat16*)y, mask, M, C);
        else if (split) bn_apply_kernel<float, true, true, true, true><<<G, BN_THREADS, 0, st>>>(
            (const float*)x, (const float*)res, scale, shift, (float*)y, mask, M, C);
        else bn_apply_kernel<float, true, true, true><<<G, BN_THREADS, 0, st>>>(
            (const float*)x, (const float*)res, scale, shift, (float*)y, mask, M, C);
        return cudaGetLastError();
    }
    if (dtype == 0) {
        if (relu && add) BN_APPLY(__nv_bfloat16, true, true, false);
        else if (relu)   BN_APPLY(__nv_bfloat16, true, false, false);
        else if (add)    BN_APPLY(__nv_bfloat16, false, true, false);
        else             BN_APPLY(__nv_bfloat16, false, false, false);
    } else if (split) {
        if (relu && add) BN_APPLY(float, true, true, true);
        else if (relu)   BN_APPLY(float, true, false, true);
        else if (add)    BN_APPLY(float, false, true, true);
        else             BN_APPLY(float, false, false, true);
    } else {
        if (relu && add) BN_APPLY(float, true, true, false);
        else if (relu)   BN_APPLY(float, true, false, false);
        else if (add)    BN_APPLY(float, false, true, false);
        else             BN_APPLY(float, false, false, false);
    }
    return cudaGetLastError();
}

#define BN_APPLY_DROP(T, MK, S) bn_apply_drop_kernel<T, MK, S><<<G, BN_THREADS, 0, st>>>( \
    (const T*)x, (const T*)res, scale, shift, (T*)y, mask, M, C, sdrop, hw)

// stochastic depth: bn_launch_apply with relu and a residual, the BN output scaled by sdrop[row / hw]
// (sdrop: fp32 [M / hw], M < 2^31); mask nullable as there
cudaError_t bn_launch_apply_drop(int dtype, const void* x, const void* res, const float* scale, const float* shift,
                                 void* y, uint8_t* mask, const float* sdrop, int hw, long long M, int C, int G,
                                 cudaStream_t st)
{
    const bool split = dtype == 1 && f32_split();
    if (hw < 1 || M % hw != 0 || M >= (1LL << 31) || (mask != nullptr && split && C % 16 != 0))
        return cudaErrorInvalidValue;
    if (G <= 0) G = bn_grid(M, C, 6);           // 3 CTAs/SM resident -> 2 waves
    if (dtype == 0) { if (mask) BN_APPLY_DROP(__nv_bfloat16, true, false); else BN_APPLY_DROP(__nv_bfloat16, false, false); }
    else if (split) { if (mask) BN_APPLY_DROP(float, true, true); else BN_APPLY_DROP(float, false, true); }
    else            { if (mask) BN_APPLY_DROP(float, true, false); else BN_APPLY_DROP(float, false, false); }
    return cudaGetLastError();
}

#define BN_RED(T, MODE, S) bn_bwd_reduce_kernel<T, MODE, S><<<G, BN_THREADS, 0, st>>>( \
    (const T*)dy, (const T*)x, (const T*)y, scale, shift, mean, invstd, partial, (T*)dz, M, C)

cudaError_t bn_launch_bwd_reduce(int dtype, int mode, const void* dy, const void* x, const void* y,
                                 const float* scale, const float* shift, const float* mean,
                                 const float* invstd, float* partial, void* dz, long long M, int C,
                                 int G, cudaStream_t st)
{
    if (dtype == 0) {
        if (mode == 0) BN_RED(__nv_bfloat16, 0, false); else if (mode == 1) BN_RED(__nv_bfloat16, 1, false);
        else BN_RED(__nv_bfloat16, 2, false);
    } else if (f32_split()) {
        if (mode == 0) BN_RED(float, 0, true); else if (mode == 1) BN_RED(float, 1, true); else BN_RED(float, 2, true);
    } else {
        if (mode == 0) BN_RED(float, 0, false); else if (mode == 1) BN_RED(float, 1, false); else BN_RED(float, 2, false);
    }
    return cudaGetLastError();
}

#define BN_RED_DROP(T, S) bn_bwd_reduce_drop_kernel<T, S><<<G, BN_THREADS, 0, st>>>( \
    (const T*)dy, (const T*)x, (const T*)y, mean, invstd, partial, (T*)dz, M, C, sdrop, hw)

// stochastic depth: bn_launch_bwd_reduce MODE 2 (residual + ReLU) with the partials of sdrop[row / hw] * dz
cudaError_t bn_launch_bwd_reduce_drop(int dtype, const void* dy, const void* x, const void* y, const float* mean,
                                      const float* invstd, float* partial, void* dz, const float* sdrop, int hw,
                                      long long M, int C, int G, cudaStream_t st)
{
    if (hw < 1 || M % hw != 0 || M >= (1LL << 31)) return cudaErrorInvalidValue;
    if (dtype == 0) BN_RED_DROP(__nv_bfloat16, false);
    else if (f32_split()) BN_RED_DROP(float, true);
    else BN_RED_DROP(float, false);
    return cudaGetLastError();
}

cudaError_t bn_launch_bwd_finalize(const float* partial, int G, long long M, int C, const float* scale,
                                   const float* mean, const float* invstd, float* ggamma, float* gbeta,
                                   float* c2, float* c3, cudaStream_t st)
{
    bn_bwd_finalize_kernel<<<(C + 31) / 32, BN_FIN_THREADS, 0, st>>>(partial, G, M, C, scale, mean, invstd,
                                                            ggamma, gbeta, c2, c3);
    return cudaGetLastError();
}

#define BN_DX(T, MODE, S) bn_bwd_dx_kernel<T, MODE, S><<<G, BN_THREADS, 0, st>>>( \
    (const T*)dz, (const T*)x, scale, shift, c2, c3, (T*)dx, M, C)

// G <= 0: the default grid
cudaError_t bn_launch_bwd_dx(int dtype, int mode, const void* dz, const void* x, const float* scale,
                             const float* shift, const float* c2, const float* c3, void* dx,
                             long long M, int C, int G, cudaStream_t st)
{
    if (G <= 0) G = bn_grid(M, C, 6);      // 3 CTAs/SM resident -> exactly 2 waves
    if (dtype == 0)       { if (mode == 1) BN_DX(__nv_bfloat16, 1, false); else BN_DX(__nv_bfloat16, 0, false); }
    else if (f32_split()) { if (mode == 1) BN_DX(float, 1, true); else BN_DX(float, 0, true); }
    else                  { if (mode == 1) BN_DX(float, 1, false); else BN_DX(float, 0, false); }
    return cudaGetLastError();
}

#define BN_DX_DROP(T, S) bn_bwd_dx_drop_kernel<T, S><<<G, BN_THREADS, 0, st>>>( \
    (const T*)dz, (const T*)x, scale, c2, c3, (T*)dx, M, C, sdrop, hw)

// stochastic depth: bn_launch_bwd_dx MODE 0 with dx = c1*(sdrop[row / hw]*dz) - c2*x + c3
cudaError_t bn_launch_bwd_dx_drop(int dtype, const void* dz, const void* x, const float* scale, const float* c2,
                                  const float* c3, void* dx, const float* sdrop, int hw, long long M, int C, int G,
                                  cudaStream_t st)
{
    if (hw < 1 || M % hw != 0 || M >= (1LL << 31)) return cudaErrorInvalidValue;
    if (G <= 0) G = bn_grid(M, C, 6);
    if (dtype == 0) BN_DX_DROP(__nv_bfloat16, false);
    else if (f32_split()) BN_DX_DROP(float, true);
    else BN_DX_DROP(float, false);
    return cudaGetLastError();
}

}  // extern "C"
