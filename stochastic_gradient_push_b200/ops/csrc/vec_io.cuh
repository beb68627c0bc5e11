// 16-byte vector I/O helpers shared by the NHWC activation kernels (BatchNorm,
// max-pool): one thread owns 8 channels; bf16 loads stay packed in 4 registers
// until they are decoded.  An fp32 thread's 8 channels are two 16-byte halves
// h floats apart: h = 4 is 8 consecutive channels, the BatchNorm kernels' split
// map passes h = C/2 so that each half of a warp's accesses is contiguous.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

namespace {

struct F8 { float v[8]; };

template <typename T> struct Io;

template <> struct Io<__nv_bfloat16> {
    typedef uint4 raw_t;      // loads stay packed (4 regs) until they are consumed
    static __device__ __forceinline__ raw_t load_raw(const __nv_bfloat16* p, int = 4) {
        uint4 r;
        asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                     : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
        return r;
    }
    static __device__ __forceinline__ F8 load(const __nv_bfloat16* p, int = 4) { return decode(load_raw(p)); }
    // read-only path WITH L1 allocation: for data that neighbouring threads re-read
    // (pooling windows overlap); the streaming loads above bypass L1 on purpose
    static __device__ __forceinline__ F8 load_cached(const __nv_bfloat16* p) {
        return decode(__ldg(reinterpret_cast<const uint4*>(p)));
    }
    static __device__ __forceinline__ F8 decode(const raw_t& r) {
        F8 o;
        const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            o.v[2 * i]     = __uint_as_float(w[i] << 16);
            o.v[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
        }
        return o;
    }
    static __device__ __forceinline__ void store(__nv_bfloat16* p, const F8& f, int = 4) {
        uint32_t w[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            __nv_bfloat162 h = __floats2bfloat162_rn(f.v[2 * i], f.v[2 * i + 1]);
            w[i] = *reinterpret_cast<uint32_t*>(&h);
        }
        asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};"
                     :: "l"(p), "r"(w[0]), "r"(w[1]), "r"(w[2]), "r"(w[3]) : "memory");
    }
};

template <> struct Io<float> {
    typedef F8 raw_t;
    static __device__ __forceinline__ raw_t load_raw(const float* p, int h = 4) { return load(p, h); }
    static __device__ __forceinline__ F8 load_cached(const float* p) {
        F8 o;
        const float4 a = __ldg(reinterpret_cast<const float4*>(p));
        const float4 b = __ldg(reinterpret_cast<const float4*>(p + 4));
        o.v[0] = a.x; o.v[1] = a.y; o.v[2] = a.z; o.v[3] = a.w;
        o.v[4] = b.x; o.v[5] = b.y; o.v[6] = b.z; o.v[7] = b.w;
        return o;
    }
    static __device__ __forceinline__ F8 decode(const raw_t& r) { return r; }
    static __device__ __forceinline__ F8 load(const float* p, int h = 4) {
        F8 o;
        asm volatile("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                     : "=f"(o.v[0]), "=f"(o.v[1]), "=f"(o.v[2]), "=f"(o.v[3]) : "l"(p));
        asm volatile("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                     : "=f"(o.v[4]), "=f"(o.v[5]), "=f"(o.v[6]), "=f"(o.v[7]) : "l"(p + h));
        return o;
    }
    static __device__ __forceinline__ void store(float* p, const F8& f, int h = 4) {
        asm volatile("st.global.v4.f32 [%0], {%1,%2,%3,%4};"
                     :: "l"(p), "f"(f.v[0]), "f"(f.v[1]), "f"(f.v[2]), "f"(f.v[3]) : "memory");
        asm volatile("st.global.v4.f32 [%0], {%1,%2,%3,%4};"
                     :: "l"(p + h), "f"(f.v[4]), "f"(f.v[5]), "f"(f.v[6]), "f"(f.v[7]) : "memory");
    }
};

__device__ __forceinline__ F8 load_c8(const float* p, int h = 4) {   // per-channel constants
    F8 o;
    const float4 a = *reinterpret_cast<const float4*>(p);
    const float4 b = *reinterpret_cast<const float4*>(p + h);
    o.v[0] = a.x; o.v[1] = a.y; o.v[2] = a.z; o.v[3] = a.w;
    o.v[4] = b.x; o.v[5] = b.y; o.v[6] = b.z; o.v[7] = b.w;
    return o;
}


}  // namespace
