// NHWC max-pooling for sm_90a (forward + backward).
//
// The framework's channels-last max-pool pair keeps int64 argmax indices, 8 bytes per
// output element, and its backward is a scatter.  Here:
//   forward : one thread = 8 channels of one output pixel, 16-byte loads of the
//             <= k*k window, writes y and a 1-BYTE window-local argmax code;
//   backward: a GATHER -- one thread = 8 channels of one INPUT pixel, visits the
//             <= ceil(k/s)^2 windows that contain it and sums dy where the stored
//             code names this pixel (first max wins, like the framework) --
//             no atomics, every dx element written exactly once.
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

#include "vec_io.cuh"

#define POOL_THREADS 256

template <typename T>
__global__ void __launch_bounds__(POOL_THREADS)
maxpool_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, uint8_t* __restrict__ code,
                   int N, int H, int W, int C, int OH, int OW, int k, int s, int p)
{
    const int cvn = C / 8;
    const long long total = (long long)N * OH * OW * cvn;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
         t += (long long)gridDim.x * blockDim.x) {
        const int cv = (int)(t % cvn);
        long long pix = t / cvn;
        const int ow = (int)(pix % OW); pix /= OW;
        const int oh = (int)(pix % OH);
        const int n = (int)(pix / OH);
        const int h0 = oh * s - p, w0 = ow * s - p;
        F8 best;
        int bi[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) { best.v[i] = -INFINITY; bi[i] = 0; }
        for (int kh = 0; kh < k; ++kh) {
            const int ih = h0 + kh;
            if (ih < 0 || ih >= H) continue;
            for (int kw = 0; kw < k; ++kw) {
                const int iw = w0 + kw;
                if (iw < 0 || iw >= W) continue;
                const F8 v = Io<T>::load_cached(x + (((long long)n * H + ih) * W + iw) * C + cv * 8);
                const int c = kh * k + kw;
#pragma unroll
                for (int i = 0; i < 8; ++i)
                    if (v.v[i] > best.v[i]) { best.v[i] = v.v[i]; bi[i] = c; }
            }
        }
        const long long o = (((long long)n * OH + oh) * OW + ow) * C + cv * 8;
        Io<T>::store(y + o, best);
        uint2 packed;
        packed.x = (uint32_t)bi[0] | ((uint32_t)bi[1] << 8) | ((uint32_t)bi[2] << 16) | ((uint32_t)bi[3] << 24);
        packed.y = (uint32_t)bi[4] | ((uint32_t)bi[5] << 8) | ((uint32_t)bi[6] << 16) | ((uint32_t)bi[7] << 24);
        *reinterpret_cast<uint2*>(code + o) = packed;
    }
}

template <typename T>
__global__ void __launch_bounds__(POOL_THREADS)
maxpool_bwd_kernel(const T* __restrict__ dy, const uint8_t* __restrict__ code, T* __restrict__ dx,
                   int N, int H, int W, int C, int OH, int OW, int k, int s, int p)
{
    const int cvn = C / 8;
    const long long total = (long long)N * H * W * cvn;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
         t += (long long)gridDim.x * blockDim.x) {
        const int cv = (int)(t % cvn);
        long long pix = t / cvn;
        const int iw = (int)(pix % W); pix /= W;
        const int ih = (int)(pix % H);
        const int n = (int)(pix / H);
        F8 acc;
#pragma unroll
        for (int i = 0; i < 8; ++i) acc.v[i] = 0.f;
        // windows (oh, ow) with oh*s - p <= ih <= oh*s - p + k - 1
        int oh_lo = (ih + p - k + 1 + s - 1) / s; if (ih + p - k + 1 < 0) oh_lo = 0;
        int oh_hi = (ih + p) / s; if (oh_hi > OH - 1) oh_hi = OH - 1;
        int ow_lo = (iw + p - k + 1 + s - 1) / s; if (iw + p - k + 1 < 0) ow_lo = 0;
        int ow_hi = (iw + p) / s; if (ow_hi > OW - 1) ow_hi = OW - 1;
        for (int oh = oh_lo; oh <= oh_hi; ++oh) {
            const int kh = ih + p - oh * s;
            for (int ow = ow_lo; ow <= ow_hi; ++ow) {
                const int kw = iw + p - ow * s;
                const uint32_t mine = (uint32_t)(kh * k + kw);
                const long long o = (((long long)n * OH + oh) * OW + ow) * C + cv * 8;
                const uint2 cd = __ldg(reinterpret_cast<const uint2*>(code + o));
                const F8 g = Io<T>::load_cached(dy + o);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    if (((cd.x >> (8 * i)) & 0xffu) == mine) acc.v[i] += g.v[i];
                    if (((cd.y >> (8 * i)) & 0xffu) == mine) acc.v[4 + i] += g.v[4 + i];
                }
            }
        }
        Io<T>::store(dx + (((long long)n * H + ih) * W + iw) * C + cv * 8, acc);
    }
}

static inline int pool_grid(long long total)
{
    long long g = (total + POOL_THREADS - 1) / POOL_THREADS;
    if (g > 132LL * 16) g = 132LL * 16;
    if (g < 1) g = 1;
    return (int)g;
}

extern "C" {

cudaError_t pool_launch_fwd(int dtype, const void* x, void* y, uint8_t* code, int N, int H, int W, int C,
                            int OH, int OW, int k, int s, int p, cudaStream_t st)
{
    const int G = pool_grid((long long)N * OH * OW * (C / 8));
    if (dtype == 0)
        maxpool_fwd_kernel<__nv_bfloat16><<<G, POOL_THREADS, 0, st>>>(
            (const __nv_bfloat16*)x, (__nv_bfloat16*)y, code, N, H, W, C, OH, OW, k, s, p);
    else
        maxpool_fwd_kernel<float><<<G, POOL_THREADS, 0, st>>>(
            (const float*)x, (float*)y, code, N, H, W, C, OH, OW, k, s, p);
    return cudaGetLastError();
}

cudaError_t pool_launch_bwd(int dtype, const void* dy, const uint8_t* code, void* dx, int N, int H, int W,
                            int C, int OH, int OW, int k, int s, int p, cudaStream_t st)
{
    const int G = pool_grid((long long)N * H * W * (C / 8));
    if (dtype == 0)
        maxpool_bwd_kernel<__nv_bfloat16><<<G, POOL_THREADS, 0, st>>>(
            (const __nv_bfloat16*)dy, code, (__nv_bfloat16*)dx, N, H, W, C, OH, OW, k, s, p);
    else
        maxpool_bwd_kernel<float><<<G, POOL_THREADS, 0, st>>>(
            (const float*)dy, code, (float*)dx, N, H, W, C, OH, OW, k, s, p);
    return cudaGetLastError();
}

}  // extern "C"
