// Batch mixing (mixup / CutMix) fused into the stage -> static input copy of the training step.
//
// The trainer copies every step's batch from its staging buffer (host layout, NCHW fp32) into the
// static input buffer the captured graph reads (NHWC fp32, or bf16 for the compute twin).  That
// copy reads each input byte once and writes it once; mixing row i with its partner row B-1-i
// (the flipped batch) fits inside it at the same traffic: one CTA column handles the row PAIR
// (i, B-1-i), so each thread reads both rows' values of a pixel and writes both mixed values.
//
// Mix state (device fp32, filled by an H2D copy per step, so a captured graph never re-captures):
//   mix[0] = lam, mix[1] = mode (0 = plain copy, 1 = mixup, 2 = CutMix),
//   mix[2..5] = CutMix box rows [y0, y1) and columns [x0, x1)
//   mixup : out_i = fmaf(lam, x_i, (1 - lam) * x_j)   (fp32; (1 - lam) and its product rounded
//           to fp32 first, then one fused multiply-add) -- the formula the Python oracle reproduces
//   CutMix: out_i = x_j inside the box, x_i outside (a select: bit-exact)
//   odd B : the middle row is its own partner (mixup: x up to rounding, CutMix: x unchanged)
// Layouts: any 4-d tensor whose pixel (h, w) sits at h * W * sp + w * sp (NCHW and NHWC both do),
// so the generic kernel serves NCHW / NHWC sources and destinations; the trainer's NCHW -> NHWC
// 3-channel case has a vectorised kernel (batch_mix_nchw3_kernel).
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace {

constexpr int MIX_THREADS = 256;
constexpr int MIX_PIX_PER_THREAD = 4;           // pixels per thread (grid-stride), sizes grid.x

template <typename T> __device__ __forceinline__ T mix_out(float v);
template <> __device__ __forceinline__ float mix_out<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 mix_out<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

template <typename TO>
__global__ void __launch_bounds__(MIX_THREADS)
batch_mix_kernel(const float* __restrict__ src, TO* __restrict__ dst, const float* __restrict__ mix, int B, int C,
                 int H, int W, long long s_n, int s_c, int s_p, long long d_n, int d_c, int d_p)
{
    const int i = blockIdx.y;
    const int j = B - 1 - i;
    const float lam = mix[0];
    const float om = 1.f - lam;
    const int mode = (int)mix[1];
    const int y0 = (int)mix[2], y1 = (int)mix[3], x0 = (int)mix[4], x1 = (int)mix[5];
    const float* si = src + (size_t)i * s_n;
    const float* sj = src + (size_t)j * s_n;
    TO* di = dst + (size_t)i * d_n;
    TO* dj = dst + (size_t)j * d_n;
    const int HW = H * W;
    for (int p = blockIdx.x * MIX_THREADS + threadIdx.x; p < HW; p += gridDim.x * MIX_THREADS) {
        bool box = false;
        if (mode == 2) {
            const int y = p / W, x = p - y * W;
            box = y >= y0 && y < y1 && x >= x0 && x < x1;
        }
        for (int c = 0; c < C; ++c) {
            const float a = si[c * s_c + p * s_p];
            const float b = sj[c * s_c + p * s_p];
            float oa = a, ob = b;
            if (mode == 1) {
                oa = fmaf(lam, a, om * b);
                ob = fmaf(lam, b, om * a);
            } else if (box) {
                oa = b;
                ob = a;
            }
            di[c * d_c + p * d_p] = mix_out<TO>(oa);
            if (j != i) dj[c * d_c + p * d_p] = mix_out<TO>(ob);
        }
    }
}

// The trainer's case: 3-channel NCHW fp32 source, NHWC destination, H * W a multiple of 4 and
// 16-byte aligned rows.  Each thread takes 4 consecutive pixels: one float4 load per channel plane
// and row, and 12 contiguous output values per row (3 x 16 B for fp32, 3 x 8 B for bf16), so
// every load and store is a full vector instead of the generic kernel's stride-3 scalar stores.
template <typename TO> struct Vec12;
template <> struct Vec12<float> {
    static __device__ __forceinline__ void store(float* d, const float (&v)[12])
    {
        float4* d4 = reinterpret_cast<float4*>(d);
        d4[0] = make_float4(v[0], v[1], v[2], v[3]);
        d4[1] = make_float4(v[4], v[5], v[6], v[7]);
        d4[2] = make_float4(v[8], v[9], v[10], v[11]);
    }
};
template <> struct Vec12<__nv_bfloat16> {
    static __device__ __forceinline__ void store(__nv_bfloat16* d, const float (&v)[12])
    {
        uint2* d2 = reinterpret_cast<uint2*>(d);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            __nv_bfloat162 lo = __floats2bfloat162_rn(v[4 * k], v[4 * k + 1]);
            __nv_bfloat162 hi = __floats2bfloat162_rn(v[4 * k + 2], v[4 * k + 3]);
            d2[k] = make_uint2(*reinterpret_cast<uint32_t*>(&lo), *reinterpret_cast<uint32_t*>(&hi));
        }
    }
};

template <typename TO>
__global__ void __launch_bounds__(MIX_THREADS)
batch_mix_nchw3_kernel(const float* __restrict__ src, TO* __restrict__ dst, const float* __restrict__ mix, int B,
                       int H, int W)
{
    const int i = blockIdx.y;
    const int j = B - 1 - i;
    const float lam = mix[0];
    const float om = 1.f - lam;
    const int mode = (int)mix[1];
    const int y0 = (int)mix[2], y1 = (int)mix[3], x0 = (int)mix[4], x1 = (int)mix[5];
    const int HW = H * W;
    const float* si = src + (size_t)i * 3 * HW;
    const float* sj = src + (size_t)j * 3 * HW;
    TO* di = dst + (size_t)i * 3 * HW;
    TO* dj = dst + (size_t)j * 3 * HW;
    for (int p = 4 * (blockIdx.x * MIX_THREADS + threadIdx.x); p < HW; p += 4 * gridDim.x * MIX_THREADS) {
        float a[12], b[12];                          // [pixel][channel], the NHWC order
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float4 va = *reinterpret_cast<const float4*>(si + c * HW + p);
            const float4 vb = *reinterpret_cast<const float4*>(sj + c * HW + p);
            a[c] = va.x; a[3 + c] = va.y; a[6 + c] = va.z; a[9 + c] = va.w;
            b[c] = vb.x; b[3 + c] = vb.y; b[6 + c] = vb.z; b[9 + c] = vb.w;
        }
        float oa[12], ob[12];
        if (mode == 1) {
#pragma unroll
            for (int k = 0; k < 12; ++k) {
                oa[k] = fmaf(lam, a[k], om * b[k]);
                ob[k] = fmaf(lam, b[k], om * a[k]);
            }
        } else {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                bool box = false;
                if (mode == 2) {
                    const int y = (p + q) / W, x = p + q - y * W;
                    box = y >= y0 && y < y1 && x >= x0 && x < x1;
                }
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    oa[3 * q + c] = box ? b[3 * q + c] : a[3 * q + c];
                    ob[3 * q + c] = box ? a[3 * q + c] : b[3 * q + c];
                }
            }
        }
        Vec12<TO>::store(di + 3 * p, oa);
        if (j != i) Vec12<TO>::store(dj + 3 * p, ob);
    }
}

}  // namespace

extern "C" {

// out_dtype: 0 = bf16, 1 = fp32 destination; src fp32.  Strides in elements: per row (n), per
// channel (c) and per pixel (p).  mix = device fp32 [lam, mode, y0, y1, x0, x1].  src and dst must
// not overlap (checked by the caller).
cudaError_t batch_mix_launch(int out_dtype, const float* src, void* dst, const float* mix, int B, int C, int H,
                             int W, long long s_n, int s_c, int s_p, long long d_n, int d_c, int d_p,
                             cudaStream_t st)
{
    const int HW = H * W;
    const int per_cta = MIX_THREADS * MIX_PIX_PER_THREAD;
    const dim3 grid((HW + per_cta - 1) / per_cta, (B + 1) / 2);
    const bool vec3 = C == 3 && HW % 4 == 0 && s_p == 1 && s_c == HW && s_n == 3LL * HW && d_c == 1 && d_p == 3 &&
                      d_n == 3LL * HW && (reinterpret_cast<uintptr_t>(src) & 15) == 0 &&
                      (reinterpret_cast<uintptr_t>(dst) & 15) == 0;
    if (vec3) {                                      // one thread per 4 pixels: the same grid covers them
        if (out_dtype == 0)
            batch_mix_nchw3_kernel<__nv_bfloat16><<<grid, MIX_THREADS, 0, st>>>(src, (__nv_bfloat16*)dst, mix, B, H, W);
        else
            batch_mix_nchw3_kernel<float><<<grid, MIX_THREADS, 0, st>>>(src, (float*)dst, mix, B, H, W);
        return cudaGetLastError();
    }
    if (out_dtype == 0)
        batch_mix_kernel<__nv_bfloat16><<<grid, MIX_THREADS, 0, st>>>(src, (__nv_bfloat16*)dst, mix, B, C, H, W, s_n,
                                                                      s_c, s_p, d_n, d_c, d_p);
    else
        batch_mix_kernel<float><<<grid, MIX_THREADS, 0, st>>>(src, (float*)dst, mix, B, C, H, W, s_n, s_c, s_p, d_n,
                                                              d_c, d_p);
    return cudaGetLastError();
}

}  // extern "C"
