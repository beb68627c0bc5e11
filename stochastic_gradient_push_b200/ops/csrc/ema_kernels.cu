// Exponential moving average of a model's weights and BatchNorm statistics (ops/model_ema.py):
//
//     e <- fmaf(w_t, s - e, e),   w_t = 1 - d_t,   one fp32 w_t per launch
//
// over every tracked tensor in ONE launch.  The sources s (fp32 or bf16) are described by a segment
// table built once by ModelEma (source pointer, numel, offset into the flat fp32 EMA buffer, dtype);
// a parameter arena is one segment, each BatchNorm running statistic another.  The work is a flat
// list of (segment, chunk) items that a persistent grid strides over, so a hundred tiny BatchNorm
// segments cost a hundred small items, not a hundred CTAs.
//
// The decay lives on the device ([decay, warmup, count, done_ctas], EmaState): with warm-up
// d_t = min(decay, (1 + t) / (10 + t)), t = updates already applied (TensorFlow's
// ExponentialMovingAverage(num_updates) rule).  Every CTA reads the same row; the last CTA to finish
// advances the counter, so a captured launch replayed N times advances it N times.
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

#define EMA_THREADS 256
#define EMA_CHUNK 8192          // elements per work item (a multiple of every vector width)
#define EMA_UNROLL 4            // independent 16-byte EMA loads in flight per thread
#define EMA_CTAS_PER_SM 3       // the whole grid is resident: 3 x 256 threads at <= 80 registers, no spills

namespace {

struct EmaSeg {                 // one row of the int64 [nseg, 4] table built by ModelEma
    long long src;              // source address
    long long numel;
    long long off;              // element offset of the segment in the EMA buffer (64-aligned)
    long long bf16;             // source dtype: 0 = fp32, 1 = bf16
};

struct EmaState {               // the fp32 [4] row of ModelEma; count / done_ctas hold uint32 bits
    float decay;
    float warmup;
    unsigned int count;
    unsigned int done_ctas;
};

__device__ __forceinline__ float ema_decay(const EmaState* st) {
    const float d = st->decay;
    if (st->warmup == 0.0f) return d;
    const float t = (float)st->count;
    return fminf(d, (1.0f + t) / (10.0f + t));
}

__device__ __forceinline__ float ema_lerp(float e, float s, float w) { return fmaf(w, s - e, e); }

__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(__nv_bfloat16 v) { return __bfloat162float(v); }

// one 16-byte source vector: 4 fp32 or 8 bf16 elements
template <typename T> struct SrcVec;
template <> struct SrcVec<float> {
    static constexpr int V = 4;
    typedef float4 raw_t;
    static __device__ __forceinline__ void decode(const raw_t& r, float* f) {
        f[0] = r.x; f[1] = r.y; f[2] = r.z; f[3] = r.w;
    }
};
template <> struct SrcVec<__nv_bfloat16> {
    static constexpr int V = 8;
    typedef uint4 raw_t;
    static __device__ __forceinline__ void decode(const raw_t& r, float* f) {
        const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            f[2 * i]     = __uint_as_float(w[i] << 16);
            f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
        }
    }
};

// e[0, n) <- lerp toward s[0, n): a scalar head up to the source's 16-byte boundary, 16-byte vectors
// over the body when the EMA side is aligned there too, a scalar tail.  Any n and any alignment.
template <typename T>
__device__ __forceinline__ void ema_span(const T* __restrict__ s, float* __restrict__ e, long long n, float w) {
    typedef SrcVec<T> SV;
    constexpr int V = SV::V;
    constexpr int U = EMA_UNROLL * 4 / V;      // source vectors per batch: the batch covers EMA_UNROLL float4 of e
    const int tid = threadIdx.x;
    const uintptr_t mis = reinterpret_cast<uintptr_t>(s) & 15;
    const long long head = mis ? min(n, (long long)((16 - mis) / sizeof(T))) : 0;
    for (long long i = tid; i < head; i += EMA_THREADS) e[i] = ema_lerp(e[i], to_f32(s[i]), w);
    s += head;
    e += head;
    n -= head;
    long long body = 0;
    if ((reinterpret_cast<uintptr_t>(e) & 15) == 0) {
        const long long nv = n / V;
        const typename SV::raw_t* sv = reinterpret_cast<const typename SV::raw_t*>(s);
        float4* ev = reinterpret_cast<float4*>(e);
        for (long long v0 = tid; v0 < nv; v0 += U * EMA_THREADS) {
            typename SV::raw_t r[U];
            float4 cur[U][V / 4];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const long long v = v0 + (long long)u * EMA_THREADS;
                if (v < nv) {
                    r[u] = __ldg(sv + v);
#pragma unroll
                    for (int q = 0; q < V / 4; ++q) cur[u][q] = ev[v * (V / 4) + q];
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const long long v = v0 + (long long)u * EMA_THREADS;
                if (v < nv) {
                    float f[V];
                    SV::decode(r[u], f);
#pragma unroll
                    for (int q = 0; q < V / 4; ++q) {
                        float4 o = cur[u][q];
                        o.x = ema_lerp(o.x, f[4 * q + 0], w);
                        o.y = ema_lerp(o.y, f[4 * q + 1], w);
                        o.z = ema_lerp(o.z, f[4 * q + 2], w);
                        o.w = ema_lerp(o.w, f[4 * q + 3], w);
                        ev[v * (V / 4) + q] = o;
                    }
                }
            }
        }
        body = nv * V;
    }
    for (long long i = body + tid; i < n; i += EMA_THREADS) e[i] = ema_lerp(e[i], to_f32(s[i]), w);
}

__global__ void __launch_bounds__(EMA_THREADS, EMA_CTAS_PER_SM)
ema_update_kernel(const EmaSeg* __restrict__ segs, const int2* __restrict__ items, int nitems,
                  float* __restrict__ ema, EmaState* st)
{
    const float w = 1.0f - ema_decay(st);
    for (int it = blockIdx.x; it < nitems; it += gridDim.x) {
        const int2 item = items[it];
        const EmaSeg sg = segs[item.x];
        const long long start = (long long)item.y * EMA_CHUNK;
        const long long n = min((long long)EMA_CHUNK, sg.numel - start);
        float* e = ema + sg.off + start;
        if (sg.bf16)
            ema_span(reinterpret_cast<const __nv_bfloat16*>(sg.src) + start, e, n, w);
        else
            ema_span(reinterpret_cast<const float*>(sg.src) + start, e, n, w);
    }
    // every thread of this CTA has read the decay row; the last CTA of the grid advances the counter
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        if (atomicAdd(&st->done_ctas, 1u) == gridDim.x - 1) {
            st->count += 1u;
            st->done_ctas = 0u;
            __threadfence();
        }
    }
}

}  // namespace

extern "C" {

int sgp_ema_chunk() { return EMA_CHUNK; }

// segs: device EmaSeg[nseg]; items: device int2[nitems] of (segment, chunk); state: device EmaState.
// grid = min(nitems, EMA_CTAS_PER_SM * num_sms), at least 1 (an empty table still advances the counter)
cudaError_t sgp_launch_ema_update(const void* segs, const void* items, int nitems, float* ema, void* state,
                                  int num_sms, cudaStream_t stream)
{
    int grid = EMA_CTAS_PER_SM * num_sms;
    if (nitems < grid) grid = nitems;
    if (grid < 1) grid = 1;
    ema_update_kernel<<<grid, EMA_THREADS, 0, stream>>>(reinterpret_cast<const EmaSeg*>(segs),
                                                       reinterpret_cast<const int2*>(items), nitems, ema,
                                                       reinterpret_cast<EmaState*>(state));
    return cudaGetLastError();
}

}  // extern "C"
