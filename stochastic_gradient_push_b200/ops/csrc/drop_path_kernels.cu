// Stochastic depth (Huang et al. 2016): the per-sample residual-branch scales of one training forward, drawn
// on the device so that a captured graph draws fresh masks at every replay.
//
//   out[l][n] = u24(seed, rank, draw, l, n) < thresh[l] ? keep_scale[l] : 0
//
// u24 is the top 24 bits of a counter-based hash (splitmix64's finaliser chained over the five keys), so a
// value depends on nothing but its keys and ops/oracle.py reproduces every bit.  `draw` is an int64 in device
// memory that the launch reads and then increments: replays of a captured graph advance it, a capture does not.
// thresh[l] = round((1 - p_l) 2^24) and keep_scale[l] = fp32(1 / (1 - p_l)) are computed once on the host.
#include <cuda_runtime.h>
#include <stdint.h>

#define DP_THREADS 256
#define DP_MAX_BLOCKS 256

struct DropPathTable {
    int L;
    int n;
    uint32_t thresh[DP_MAX_BLOCKS];
    float keep_scale[DP_MAX_BLOCKS];
};

static_assert(sizeof(DropPathTable) <= 4096, "the drop-path table must fit the kernel parameter space");

__device__ __forceinline__ uint64_t dp_mix64(uint64_t z)
{
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// one CTA: 16 x 256 values for ResNet-50 at batch 256
__global__ void __launch_bounds__(DP_THREADS)
drop_path_draw_kernel(const __grid_constant__ DropPathTable tab, unsigned long long seed, unsigned long long rank,
                      long long* __restrict__ counter, float* __restrict__ out)
{
    const unsigned long long draw = (unsigned long long)*counter;
    const uint64_t base = dp_mix64(dp_mix64(dp_mix64(seed) ^ rank) ^ draw);
    const int total = tab.L * tab.n;
    for (int i = threadIdx.x; i < total; i += DP_THREADS) {
        const int l = i / tab.n, n = i - l * tab.n;
        const uint32_t u = (uint32_t)(dp_mix64(base ^ (((uint64_t)l << 32) | (uint32_t)n)) >> 40);
        out[i] = u < tab.thresh[l] ? tab.keep_scale[l] : 0.f;
    }
    __syncthreads();                      // every thread has read the counter
    if (threadIdx.x == 0) *counter = (long long)(draw + 1);
}

extern "C" {

int drop_path_max_blocks() { return DP_MAX_BLOCKS; }

// thresh[L] in [0, 2^24], keep_scale[L] (host arrays), 1 <= L <= DP_MAX_BLOCKS, n >= 1, L * n < 2^31;
// out: fp32 [L, n] on the device; counter: one int64 on the device
cudaError_t drop_path_launch_draw(const unsigned int* thresh, const float* keep_scale, int L, int n,
                                  unsigned long long seed, unsigned long long rank, long long* counter, float* out,
                                  cudaStream_t st)
{
    if (L < 1 || L > DP_MAX_BLOCKS || n < 1 || (long long)L * n >= (1LL << 31)) return cudaErrorInvalidValue;
    DropPathTable tab;
    tab.L = L;
    tab.n = n;
    for (int l = 0; l < L; ++l) {
        if (thresh[l] > (1u << 24)) return cudaErrorInvalidValue;
        tab.thresh[l] = thresh[l];
        tab.keep_scale[l] = keep_scale[l];
    }
    drop_path_draw_kernel<<<1, DP_THREADS, 0, st>>>(tab, seed, rank, counter, out);
    return cudaGetLastError();
}

}  // extern "C"
