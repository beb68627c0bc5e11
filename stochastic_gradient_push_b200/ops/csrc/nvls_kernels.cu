// NVLS (NVSwitch multicast) collectives fused with the optimizer -- sm_90a, multimem.* PTX.
//
// The buffers live in VMM symmetric memory with a multicast mapping (csrc/vmm_symm.cpp): a load
// from the multicast address can be REDUCED INSIDE THE SWITCH over all GPUs
// (multimem.ld_reduce.add), a store to it lands in EVERY GPU (multimem.st).
//
//   sgp_nvls_allreduce_sgd_kernel   AllReduce-SGD (the reference's DistributedDataParallel baseline,
//       gossip_sgd.py:179-180) as ONE kernel, two-shot with a sharded optimizer step:
//         barrier-in   every rank's gradients are final (per-CTA flags, as sgp_allreduce_sgd_kernel)
//         reduce       rank r owns chunks [r*S, (r+1)*S): ONE multimem.ld_reduce per 16 bytes returns
//                      the sum over all ranks (instead of n-1 P2P reads per element);
//                      multimem.st of zeros clears that slice of every rank's gradient buffer
//         update       SGD-momentum on the owned slice only (momentum is touched 1/world-th)
//         all-gather   multimem.st of the new parameters into every replica (bit-identical)
//         barrier-out  every slice has landed everywhere before the next forward reads it
//       per-GPU NVLink traffic ~ 2 x 4n bytes instead of (world-1) x 4n for the one-shot P2P kernel.
//   MODE 0 of the same kernel is a plain in-place all-reduce (hierarchical mode: the local-node
//       gradient average, gossip/distributed.py:556-562) -- reduced slice scaled and multicast back.
//   sgp_nvls_bcast_kernel           root -> all: multimem.st broadcast of a flat buffer (the
//       local-node parameter broadcast, gossip/distributed.py:282-296) + release/acquire flags.
#include "sgp_common.cuh"

namespace {

__device__ __forceinline__ float4 mc_ld_reduce_f32x4(const float* mc) {
    float4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(mc) : "memory");
    return v;
}
// 8 bf16 values summed over the ranks with fp32 accumulation inside the switch
__device__ __forceinline__ uint4 mc_ld_reduce_bf16x8(const __nv_bfloat16* mc) {
    uint4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(mc) : "memory");
    return v;
}
__device__ __forceinline__ void mc_st_f32x4(float* mc, float4 v) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};"
                 :: "l"(mc), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void mc_st_b32x4(void* mc, uint4 v) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};"
                 :: "l"(mc), "f"(__uint_as_float(v.x)), "f"(__uint_as_float(v.y)), "f"(__uint_as_float(v.z)),
                    "f"(__uint_as_float(v.w)) : "memory");
}

__device__ __forceinline__ void sgd1n(float& x, float g, float& m, float lr, float mu, float wd, float nesterov) {
    const float d = fmaf(wd, x, g);
    m = fmaf(mu, m, d);
    const float upd = (nesterov != 0.f) ? fmaf(mu, m, d) : m;
    x = fmaf(-lr, upd, x);
}

}  // namespace

struct NvlsArgs {
    float*               z;          // this rank's parameters (local view)
    float*               z_mc;       // multicast view of the parameter buffers
    void*                g_mc;       // multicast view of the gradient buffers (fp32 or bf16)
    float*               m;          // momentum (local; only the owned slice is used)
    SgpSignalPad* const* pads;       // [world] signal pads (unicast peer views)
    SgpState*            st;
    const SgpHyper*      hyper;
    long long            n;          // elements, multiple of SGP_CHUNK
    int                  rank, world;
    unsigned long long   timeout_ns;
    int                  grad_bf16;
    float                scale;      // MODE 0: factor applied to the sum (1/world for a mean)
};

// MODE 1: fused AllReduce-SGD.  MODE 0: in-place all-reduce of the gradient buffers (fp32).
template <int MODE>
__global__ void __launch_bounds__(SGP_THREADS, 2)
sgp_nvls_allreduce_kernel(const NvlsArgs a)
{
    __shared__ int s_ok;
    SgpState* st = a.st;
    const uint32_t step = *((volatile uint32_t*)&st->step);
    const int tid = threadIdx.x, b = blockIdx.x;
    SgpSignalPad* mypad = a.pads[a.rank];

    // ---- barrier-in: this rank's gradients were produced by earlier kernels on this stream ----
    if (tid == 0) {
        s_ok = 1;
        __threadfence_system();
        st_release_sys(&mypad->pub_seq[b], step + 1u);
    }
    __syncthreads();
    if (tid < a.world && tid != a.rank)
        if (!spin_wait_geq(&a.pads[tid]->pub_seq[b], step + 1u, st, a.timeout_ns, SGP_ERR_TIMEOUT_PUB)) s_ok = 0;
    __syncthreads();

    if (s_ok) {
        const long long nchunks = a.n / SGP_CHUNK;
        const long long per = (nchunks + a.world - 1) / a.world;       // chunks owned by one rank
        const long long c_lo = per * a.rank;
        const long long c_hi = (c_lo + per < nchunks) ? c_lo + per : nchunks;
        const SgpHyper hp = *a.hyper;
        const float gscale = (MODE == 1) ? hp.grad_scale / (float)a.world : a.scale;
        for (long long c = c_lo + b; c < c_hi; c += gridDim.x) {
            const long long base = c * SGP_CHUNK + (long long)tid * SGP_VEC;
            if (a.grad_bf16) {
                // 8 bf16 per request: a thread covers two consecutive float4 of its chunk quarter
                // (thread layout: 16 bytes of bf16 = 8 elements -> use half the threads per sweep)
#pragma unroll
                for (int u = 0; u < SGP_UNROLL / 2; ++u) {
                    const long long i = c * SGP_CHUNK + ((long long)u * SGP_THREADS + tid) * 8;
                    const __nv_bfloat16* gp = reinterpret_cast<const __nv_bfloat16*>(a.g_mc) + i;
                    const uint4 raw = mc_ld_reduce_bf16x8(gp);
                    mc_st_b32x4(const_cast<__nv_bfloat16*>(gp), make_uint4(0u, 0u, 0u, 0u));     // clear everywhere
                    const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
                    float g[8];
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        g[2 * e] = __uint_as_float(w[e] << 16) * gscale;
                        g[2 * e + 1] = __uint_as_float(w[e] & 0xffff0000u) * gscale;
                    }
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        float4 xv = *reinterpret_cast<const float4*>(a.z + i + 4 * h);
                        float4 mv = *reinterpret_cast<const float4*>(a.m + i + 4 * h);
                        sgd1n(xv.x, g[4 * h + 0], mv.x, hp.lr, hp.momentum, hp.weight_decay, hp.nesterov);
                        sgd1n(xv.y, g[4 * h + 1], mv.y, hp.lr, hp.momentum, hp.weight_decay, hp.nesterov);
                        sgd1n(xv.z, g[4 * h + 2], mv.z, hp.lr, hp.momentum, hp.weight_decay, hp.nesterov);
                        sgd1n(xv.w, g[4 * h + 3], mv.w, hp.lr, hp.momentum, hp.weight_decay, hp.nesterov);
                        *reinterpret_cast<float4*>(a.m + i + 4 * h) = mv;
                        mc_st_f32x4(a.z_mc + i + 4 * h, xv);
                    }
                }
            } else {
                float4 g[SGP_UNROLL];
#pragma unroll
                for (int u = 0; u < SGP_UNROLL; ++u) {
                    const long long i = base + (long long)u * SGP_THREADS * SGP_VEC;
                    g[u] = mc_ld_reduce_f32x4(reinterpret_cast<const float*>(a.g_mc) + i);
                }
#pragma unroll
                for (int u = 0; u < SGP_UNROLL; ++u) {
                    const long long i = base + (long long)u * SGP_THREADS * SGP_VEC;
                    float* gp = reinterpret_cast<float*>(a.g_mc) + i;
                    const float4 gv = make_float4(g[u].x * gscale, g[u].y * gscale, g[u].z * gscale, g[u].w * gscale);
                    if (MODE == 0) {
                        mc_st_f32x4(gp, gv);                               // the all-reduced value, everywhere
                    } else {
                        mc_st_f32x4(gp, make_float4(0.f, 0.f, 0.f, 0.f)); // consumed: clear it everywhere
                        float4 xv = *reinterpret_cast<const float4*>(a.z + i);
                        float4 mv = *reinterpret_cast<const float4*>(a.m + i);
                        sgd1n(xv.x, gv.x, mv.x, hp.lr, hp.momentum, hp.weight_decay, hp.nesterov);
                        sgd1n(xv.y, gv.y, mv.y, hp.lr, hp.momentum, hp.weight_decay, hp.nesterov);
                        sgd1n(xv.z, gv.z, mv.z, hp.lr, hp.momentum, hp.weight_decay, hp.nesterov);
                        sgd1n(xv.w, gv.w, mv.w, hp.lr, hp.momentum, hp.weight_decay, hp.nesterov);
                        *reinterpret_cast<float4*>(a.m + i) = mv;
                        mc_st_f32x4(a.z_mc + i, xv);                       // all-gather of the new parameters
                    }
                }
            }
        }
    }

    // ---- barrier-out: every rank's slice has been multicast before anybody moves on ----
    __syncthreads();
    if (tid == 0) {
        __threadfence_system();
        const uint32_t prev = atomicAdd(&st->done_ctas, 1u);
        if (prev == gridDim.x - 1) {
            __threadfence_system();
            for (int r = 0; r < a.world; ++r)
                if (r != a.rank) st_release_sys(&a.pads[r]->ack_seq[a.rank], step + 1u);
            for (int r = 0; r < a.world; ++r)
                if (r != a.rank)
                    spin_wait_geq(&mypad->ack_seq[r], step + 1u, st, a.timeout_ns, SGP_ERR_TIMEOUT_ACK);
            *((volatile uint32_t*)&st->done_ctas) = 0u;
            *((volatile uint32_t*)&st->step) = step + 1u;
            __threadfence();
        }
    }
}

// root -> everyone: dst_mc[i] = src[i] (multimem.st), then flags.  Non-root ranks launch the same
// kernel with one CTA: it only waits for the root's flag (so the broadcast is stream-ordered
// before whatever they enqueue next).
__global__ void __launch_bounds__(SGP_THREADS)
sgp_nvls_bcast_kernel(float* dst_mc, const float* __restrict__ src, long long n, SgpSignalPad* const* pads,
                      SgpState* st, int rank, int world, int root, unsigned long long timeout_ns)
{
    const uint32_t epoch = st->bar_epoch + 1u;
    if (rank == root) {
        // every receiver must have ARRIVED (its earlier kernels -- e.g. its own optimizer step on
        // the same parameters -- are complete) before the root overwrites its memory
        __shared__ int s_ok;
        if (threadIdx.x == 0) s_ok = 1;
        __syncthreads();
        if ((int)threadIdx.x < world && (int)threadIdx.x != root)
            if (!spin_wait_geq(&pads[root]->bar_seq[threadIdx.x], epoch, st, timeout_ns, SGP_ERR_TIMEOUT_BAR))
                s_ok = 0;
        __syncthreads();
        if (!s_ok) return;
        const long long n4 = n / 4;
        for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4;
             i += (long long)gridDim.x * blockDim.x)
            mc_st_f32x4(dst_mc + 4 * i, reinterpret_cast<const float4*>(src)[i]);
        __syncthreads();
        if (threadIdx.x == 0) {
            __threadfence_system();
            const uint32_t prev = atomicAdd(&st->done_ctas, 1u);
            if (prev == gridDim.x - 1) {
                __threadfence_system();
                for (int r = 0; r < world; ++r)
                    if (r != rank) st_release_sys(&pads[r]->bar_seq[root], epoch);
                *((volatile uint32_t*)&st->done_ctas) = 0u;
                st->bar_epoch = epoch;
                __threadfence();
            }
        }
    } else if (blockIdx.x == 0 && threadIdx.x == 0) {
        __threadfence_system();
        st_release_sys(&pads[root]->bar_seq[rank], epoch);            // "I am here, overwrite me"
        spin_wait_geq(&pads[rank]->bar_seq[root], epoch, st, timeout_ns, SGP_ERR_TIMEOUT_BAR);
        st->bar_epoch = epoch;
        __threadfence();
    }
}

extern "C" {

cudaError_t sgp_launch_nvls_allreduce(const NvlsArgs* a, int fused_sgd, int grid, cudaStream_t stream)
{
    if (fused_sgd) sgp_nvls_allreduce_kernel<1><<<grid, SGP_THREADS, 0, stream>>>(*a);
    else           sgp_nvls_allreduce_kernel<0><<<grid, SGP_THREADS, 0, stream>>>(*a);
    return cudaGetLastError();
}

cudaError_t sgp_launch_nvls_bcast(float* dst_mc, const float* src, long long n, SgpSignalPad* const* pads,
                                  SgpState* st, int rank, int world, int root, unsigned long long timeout_ns,
                                  int grid, cudaStream_t stream)
{
    sgp_nvls_bcast_kernel<<<(rank == root) ? grid : 1, SGP_THREADS, 0, stream>>>(dst_mc, src, n, pads, st, rank,
                                                                                world, root, timeout_ns);
    return cudaGetLastError();
}

int sgp_nvls_max_grid(int device)
{
    int sms = 0, per_sm = 0;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess) return 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, sgp_nvls_allreduce_kernel<1>, SGP_THREADS, 0)
        != cudaSuccess) return 0;
    return sms * per_sm;
}

}  // extern "C"
