// Gradient accumulation for GossipTrainer(accumulation_steps=k) (parallel/trainer.py):
//
//     dst[i] <- dst[i] + float(src[i])      over a list of (dst, src) pairs, ONE launch per table
//
// dst is fp32 and src fp32 or bf16: one fp32 rounding per element, so the result is bit-identical to
// dst.add_(src.float()) and the bf16 micro-gradients of the compute twin are summed in fp32.
//
// The sources are autograd's fresh gradients: their addresses change with every eager step and are
// fixed only inside a captured graph.  So the segment table is not a device buffer but the kernel's
// own __grid_constant__ parameter (up to 32,764 bytes of parameters since CUDA 12.1 on sm_70+): a
// capture bakes it into the kernel node, an eager step simply passes new pointers.  A list longer
// than one table is split over several launches.
//
// The work is a flat list of (segment, chunk) items that a persistent grid strides over, as in
// ema_kernels.cu; each row of the table holds the prefix of its first chunk, so the segment of an
// item is a binary search over the table, uniform across the CTA.
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

#define ACC_THREADS 256
#define ACC_CHUNK 8192          // elements per work item (a multiple of every vector width)
#define ACC_UNROLL 4            // independent 16-byte dst loads in flight per thread
#define ACC_CTAS_PER_SM 3       // the whole grid is resident: 3 x 256 threads at <= 80 registers, no spills
#define ACC_MAX_SEGS 1000       // rows per table: 1000 x 32 B + 8 B header fits the parameter space

namespace {

struct AccSeg {                 // 32 bytes
    float* dst;
    const void* src;
    long long numel;
    int chunk0;                 // index of the segment's first item
    int bf16;                   // source dtype: 0 = fp32, 1 = bf16
};

struct AccTable {
    int nseg;
    int nitems;
    AccSeg seg[ACC_MAX_SEGS];
};

static_assert(sizeof(AccSeg) == 32, "AccSeg layout");
static_assert(sizeof(AccTable) <= 32764, "the segment table must fit the 32,764-byte kernel parameter space");

template <typename T> struct SrcVec;
template <> struct SrcVec<float> {              // one 16-byte source vector: 4 fp32
    static constexpr int V = 4;
    typedef float4 raw_t;
    static __device__ __forceinline__ void decode(const raw_t& r, float* f) {
        f[0] = r.x; f[1] = r.y; f[2] = r.z; f[3] = r.w;
    }
};
template <> struct SrcVec<__nv_bfloat16> {      // or 8 bf16
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

__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(__nv_bfloat16 v) { return __bfloat162float(v); }

// d[0, n) += s[0, n): a scalar head up to the source's 16-byte boundary, 16-byte vectors over the body
// when dst is aligned there too, a scalar tail.  Any n and any alignment.
template <typename T>
__device__ __forceinline__ void acc_span(const T* __restrict__ s, float* __restrict__ d, long long n) {
    typedef SrcVec<T> SV;
    constexpr int V = SV::V;
    constexpr int U = ACC_UNROLL * 4 / V;       // source vectors per batch: the batch covers ACC_UNROLL float4 of d
    const int tid = threadIdx.x;
    const uintptr_t mis = reinterpret_cast<uintptr_t>(s) & 15;
    const long long head = mis ? min(n, (long long)((16 - mis) / sizeof(T))) : 0;
    for (long long i = tid; i < head; i += ACC_THREADS) d[i] = d[i] + to_f32(s[i]);
    s += head;
    d += head;
    n -= head;
    long long body = 0;
    if ((reinterpret_cast<uintptr_t>(d) & 15) == 0) {
        const long long nv = n / V;
        const typename SV::raw_t* sv = reinterpret_cast<const typename SV::raw_t*>(s);
        float4* dv = reinterpret_cast<float4*>(d);
        for (long long v0 = tid; v0 < nv; v0 += U * ACC_THREADS) {
            typename SV::raw_t r[U];
            float4 cur[U][V / 4];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const long long v = v0 + (long long)u * ACC_THREADS;
                if (v < nv) {
                    r[u] = __ldg(sv + v);
#pragma unroll
                    for (int q = 0; q < V / 4; ++q) cur[u][q] = dv[v * (V / 4) + q];
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const long long v = v0 + (long long)u * ACC_THREADS;
                if (v < nv) {
                    float f[V];
                    SV::decode(r[u], f);
#pragma unroll
                    for (int q = 0; q < V / 4; ++q) {
                        float4 o = cur[u][q];
                        o.x = o.x + f[4 * q + 0];
                        o.y = o.y + f[4 * q + 1];
                        o.z = o.z + f[4 * q + 2];
                        o.w = o.w + f[4 * q + 3];
                        dv[v * (V / 4) + q] = o;
                    }
                }
            }
        }
        body = nv * V;
    }
    for (long long i = body + tid; i < n; i += ACC_THREADS) d[i] = d[i] + to_f32(s[i]);
}

__global__ void __launch_bounds__(ACC_THREADS, ACC_CTAS_PER_SM)
grad_accumulate_kernel(const __grid_constant__ AccTable tab)
{
    for (int it = blockIdx.x; it < tab.nitems; it += gridDim.x) {
        int lo = 0, hi = tab.nseg - 1;          // the last segment whose first item is <= it
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (tab.seg[mid].chunk0 <= it) lo = mid; else hi = mid - 1;
        }
        const AccSeg& sg = tab.seg[lo];
        const long long start = (long long)(it - sg.chunk0) * ACC_CHUNK;
        const long long n = min((long long)ACC_CHUNK, sg.numel - start);
        float* d = sg.dst + start;
        if (sg.bf16)
            acc_span(reinterpret_cast<const __nv_bfloat16*>(sg.src) + start, d, n);
        else
            acc_span(reinterpret_cast<const float*>(sg.src) + start, d, n);
    }
}

}  // namespace

extern "C" {

int sgp_accum_chunk() { return ACC_CHUNK; }
int sgp_accum_max_segs() { return ACC_MAX_SEGS; }

// rows: host int64 [nseg, 4] = (dst address, src address, numel > 0, bf16), 1 <= nseg <= ACC_MAX_SEGS,
// and fewer than 2^31 chunks in all.  One launch, grid = min(items, ACC_CTAS_PER_SM * num_sms).
cudaError_t sgp_launch_grad_accumulate(const long long* rows, int nseg, int num_sms, cudaStream_t stream)
{
    if (nseg < 1 || nseg > ACC_MAX_SEGS) return cudaErrorInvalidValue;
    AccTable tab;
    long long items = 0;
    for (int i = 0; i < nseg; ++i) {
        const long long* r = rows + 4 * i;
        if (r[2] < 1) return cudaErrorInvalidValue;
        tab.seg[i].dst = reinterpret_cast<float*>(r[0]);
        tab.seg[i].src = reinterpret_cast<const void*>(r[1]);
        tab.seg[i].numel = r[2];
        tab.seg[i].chunk0 = (int)items;
        tab.seg[i].bf16 = (int)r[3];
        items += (r[2] + ACC_CHUNK - 1) / ACC_CHUNK;
        if (items > 0x7fffffffLL) return cudaErrorInvalidValue;
    }
    tab.nseg = nseg;
    tab.nitems = (int)items;
    int grid = ACC_CTAS_PER_SM * num_sms;
    if (items < grid) grid = (int)items;
    grad_accumulate_kernel<<<grid, ACC_THREADS, 0, stream>>>(tab);
    return cudaGetLastError();
}

}  // extern "C"
