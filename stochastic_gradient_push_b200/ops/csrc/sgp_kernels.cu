// sm_90a gossip kernels: fused SGD + push-sum mix over NVSwitch peer memory.
//
// Replaces, in ONE launch per training step, the reference's K1-K9 elementwise
// swarm (ps_numerator / unbias / residual add / pre-scale / flatten / scale /
// accumulate / unflatten / optimizer.step; gossip/distributed.py:298-455,
// gossip/gossiper.py:125-219, gossip_sgd.py:389) and its N1-N3 NCCL broadcasts.
//
//   sgp_step_kernel    phase 1: x = z*w ; SGD-momentum ; (+residual) ; publish
//                      phase 2: acquire in-neighbours' flags ; weighted P2P
//                               loads ; push-sum weight update ; de-bias ; store
//   sgp_step_pipe_kernel   the same full step, warp-specialised: a producer warp feeds phase 2
//                      through a TMA ring while the consumers run phase 1 (SGP / D-PSGD hot path)
//   sgp_gather_kernel, sgp_gather_tma_kernel
//                      Overlap-SGP: residual = sum_k w_k * outbox_k  (side stream)
//   sgp_gather_wait_kernel, sgp_gather_ack_kernel
//                      the same gather on a copy engine: flag wait before, bookkeeping after
//   sgp_probe_kernel   AD-PSGD passive poll ("has my partner published?")
//   sgp_bilat_decide_kernel, sgp_bilat_ctl_kernel   AD-PSGD round state machine
//   sgp_allreduce_sgd  AR-SGD comparator: one-shot P2P all-reduce fused with SGD (+ sgp_zero_kernel)
//   sgp_barrier_kernel device-side barrier over the signal pads
//   sgp_scale_kernel   flat x *= w  /  x /= w  (ps_numerator / unbias API parity)
//   sgp_peer_reduce_kernel   dst = scale * sum of flat buffers on peer devices
//   sgp_snapshot_kernel, sgp_consensus_kernel, sgp_consensus_finalize_kernel
//                      consensus distance and the push-sum average model
//   sgp_slowmo_kernel  SlowMo: exact average + slow-momentum update
//   sgp_lars_norms_kernel, sgp_lars_trust_kernel   LARS trust ratios for the step kernels
//
// What several kernels share is written once, ahead of the kernels:
//   phase1_chunk       phase 1 of both step kernels for one chunk (sgd4, store_z)
//   TmaRing            the single-producer TMA ring of the gather, consensus and SlowMo kernels
//   clamped_segments, wait_pub_flags, pub_flags_visible, wait_outbox_acks, outbox_acks_ok,
//   gather_epilogue    the flag / ack protocol
// and, ahead of the launchers, for_each_step_variant (the legal instantiations of the step
// kernels), ensure_dynamic_smem (per-device shared-memory opt-in) and flat_grid.
#include "sgp_common.cuh"

#include <type_traits>

namespace {

struct RowInfo {
    int   n_in, n_out;
    int   in[SGP_MAX_PEERS];
    int   out[SGP_MAX_PEERS];
    float self_w;
    float in_w[SGP_MAX_PEERS];
};

__device__ __forceinline__ void load_row(const SgpArgs& a, uint32_t step_like, RowInfo& r) {
    const uint32_t row = (step_like + a.st->phase_base) % (uint32_t)a.period;
    const int*   t = a.table  + row * SGP_TABLE_ROW;
    const float* w = a.wtable + row * SGP_WTABLE_ROW;
    r.n_in = t[0];
    r.n_out = t[1];
#pragma unroll
    for (int k = 0; k < SGP_MAX_PEERS; ++k) {
        r.in[k]   = t[2 + k];
        r.out[k]  = t[2 + SGP_MAX_PEERS + k];
        r.in_w[k] = w[1 + k];
    }
    r.self_w = w[0];
}

__device__ __forceinline__ float4 fma4(float4 a, float s, float4 b) {
    return make_float4(fmaf(a.x, s, b.x), fmaf(a.y, s, b.y), fmaf(a.z, s, b.z), fmaf(a.w, s, b.w));
}
__device__ __forceinline__ float4 mul4(float4 a, float s) {
    return make_float4(a.x * s, a.y * s, a.z * s, a.w * s);
}

// SGD with momentum on the four lanes of the push-sum numerator (torch.optim.SGD semantics,
// dampening 0): d = g + wd*x ; m = mu*m + d ; x -= lr * (nesterov ? d + mu*m : m), with the
// hyper-parameters as one row h = {lr, mu, wd, nesterov}.
// LARS (SGP_F_LARS): d = t * (g + wd*x), t the trust ratio of the element's tensor.  t == 1 (LARS
// disabled, zero norms) multiplies exactly, so those elements get the bits of the plain update
template <bool LARS>
__device__ __forceinline__ void sgd4(float4& xv, const float4& gv, float4& mv, const float4& h, float t) {
#define SGP_SGD_LANE(e)                                                        \
    {                                                                          \
        float d = fmaf(h.z, xv.e, gv.e);                                       \
        if constexpr (LARS) d = t * d;                                         \
        mv.e = fmaf(h.y, mv.e, d);                                             \
        const float upd = (h.w != 0.f) ? fmaf(h.y, mv.e, d) : mv.e;            \
        xv.e = fmaf(-h.x, upd, xv.e);                                          \
    }
    SGP_SGD_LANE(x) SGP_SGD_LANE(y) SGP_SGD_LANE(z) SGP_SGD_LANE(w)
#undef SGP_SGD_LANE
}
__device__ __forceinline__ float4 hyper_row(const SgpHyper& h) {
    return make_float4(h.lr, h.momentum, h.weight_decay, h.nesterov);
}

// SGP_F_GROUPS: the group rows {lr, momentum, weight_decay, nesterov} go to shared memory once
// per CTA (threads [0, groups) copy one row each; the caller synchronises).  A 16-byte access
// never straddles a 64-float block, so one block_group byte serves all four lanes of a float4
__device__ __forceinline__ void load_group_rows(const SgpArgs& a, float4* s_rows, int tid) {
    if (tid < a.groups) s_rows[tid] = hyper_row(a.hyper_groups[tid]);
}
__device__ __forceinline__ uint32_t block_group_of(const SgpArgs& a, long long i) {
    return __ldg(a.block_group + (i / SGP_GROUP_BLOCK));
}
// trust ratio of the tensor that owns the 64-float block of element i (written by
// sgp_lars_trust_kernel earlier on the stream, so the read-only path is safe)
__device__ __forceinline__ float lars_trust_of(const SgpArgs& a, long long i) {
    return __ldg(a.lars_trust + __ldg(a.block_tensor + (i / SGP_GROUP_BLOCK)));
}

// Last-CTA bookkeeping shared by the kernels: returns true in thread 0 of the
// CTA that finishes last.
__device__ __forceinline__ bool cta_done_is_last(SgpState* st) {
    __threadfence();
    const uint32_t prev = atomicAdd(&st->done_ctas, 1u);
    if (prev == gridDim.x - 1) {
        __threadfence();
        return true;
    }
    return false;
}

// ---- chunk decomposition ----------------------------------------------------
// CTA b of a grid owns chunks b, b + G, b + 2G, ... of `nchunks`: how many that is
__device__ __forceinline__ long long cta_chunks(long long nchunks, int b) {
    return (nchunks > b) ? (nchunks - 1 - b) / gridDim.x + 1 : 0;
}
// Thread `tid` makes SGP_UNROLL 16-byte accesses to chunk c, SGP_THREADS * SGP_VEC elements apart:
// chunk_base is the first one's element, chunk_elem(base, u) the u-th one's
__device__ __forceinline__ long long chunk_base(long long c, int tid) {
    return c * SGP_CHUNK + (long long)tid * SGP_VEC;
}
__device__ __forceinline__ long long chunk_elem(long long base, int u) {
    return base + (long long)u * SGP_THREADS * SGP_VEC;
}
// de-biased parameters and, with SGP_F_SHADOW, their bf16 copy
__device__ __forceinline__ void store_z(const SgpArgs& a, uint32_t flags, long long i, const float4& zv) {
    st_f4(reinterpret_cast<float4*>(a.z + i), zv);
    if (flags & SGP_F_SHADOW) st_u2(reinterpret_cast<uint2*>(a.shadow + i), f4_to_bf16x4(zv));
}

// ---- phase 1 of the step kernels, one chunk -----------------------------------
// All SGP_UNROLL loads first, then per access: x = z * wmul ; SGD (clearing the gradient with
// SGP_F_ZERO_GRAD) ; + rscale * residual ; publish ; z = x / w1.
// MSG_BF16: publish Q(x) = bf16(x) and keep what was not sent, c = x - (1 - self_w) Q(x), in z.
// FULL_STEP (sgp_step_pipe_kernel: always PHASE1 | PUBLISH | PHASE2, never FOLD_RES) compiles the
// residual fold, the test of SGP_F_PUBLISH and the z store out; rscale, inv_w1 and write_z are
// then unused.  Ranks of one job may run either step kernel, so both must get these bits.
template <bool MSG_BF16, bool GROUPS, bool LARS, bool FULL_STEP>
__device__ __forceinline__ void phase1_chunk(
    const SgpArgs& a, const uint32_t flags, const long long c, const int tid, const SgpHyper& hp,
    const bool do_sgd, const float4* s_rows, const float wmul, const float self_w,
    typename std::conditional<MSG_BF16, __nv_bfloat16, float>::type* my_out, const uint64_t pol_first,
    const uint64_t pol_last, const float rscale, const float inv_w1, const bool write_z)
{
    const bool fold = !FULL_STEP && (flags & SGP_F_FOLD_RES);
    const long long base = chunk_base(c, tid);
    float4 x[SGP_UNROLL], g[SGP_UNROLL], m[SGP_UNROLL], r[SGP_UNROLL];
    uint32_t grp[SGP_UNROLL];
    float tr[SGP_UNROLL];
#pragma unroll
    for (int u = 0; u < SGP_UNROLL; ++u) {
        const long long i = chunk_elem(base, u);
        x[u] = ld_once_f4(reinterpret_cast<const float4*>(a.z + i), pol_first);
        if (do_sgd) {
            if (flags & SGP_F_GRAD_BF16)
                g[u] = bf16x4_to_f4(ld_once_u2(reinterpret_cast<const uint2*>(
                           reinterpret_cast<const __nv_bfloat16*>(a.g) + i), pol_first));
            else
                g[u] = ld_once_f4(reinterpret_cast<const float4*>(
                           reinterpret_cast<const float*>(a.g) + i), pol_first);
            if (a.g2 != nullptr) {
                const float4 h = ld_once_f4(reinterpret_cast<const float4*>(a.g2 + i), pol_first);
                g[u].x += h.x; g[u].y += h.y; g[u].z += h.z; g[u].w += h.w;
            }
            m[u] = ld_once_f4(reinterpret_cast<const float4*>(a.m + i), pol_first);
            if constexpr (GROUPS) grp[u] = block_group_of(a, i);
            if constexpr (LARS) tr[u] = lars_trust_of(a, i);
        }
        if (fold) r[u] = ld_once_f4(reinterpret_cast<const float4*>(a.residual + i), pol_first);
    }
#pragma unroll
    for (int u = 0; u < SGP_UNROLL; ++u) {
        const long long i = chunk_elem(base, u);
        float4 xv = mul4(x[u], wmul);               // numerator (exact if w == 1)
        if (do_sgd) {
            const float4 gv = mul4(g[u], hp.grad_scale);
            float4 mv = m[u];
            float t = 1.f;
            if constexpr (LARS) t = tr[u];
            if constexpr (GROUPS) sgd4<LARS>(xv, gv, mv, s_rows[grp[u]], t);
            else                  sgd4<LARS>(xv, gv, mv, hyper_row(hp), t);
            st_f4(reinterpret_cast<float4*>(a.m + i), mv);
            if (flags & SGP_F_ZERO_GRAD) {
                if (flags & SGP_F_GRAD_BF16)
                    st_u2(reinterpret_cast<uint2*>(
                              reinterpret_cast<__nv_bfloat16*>(a.g) + i), make_uint2(0u, 0u));
                else
                    st_f4(reinterpret_cast<float4*>(reinterpret_cast<float*>(a.g) + i),
                          make_float4(0.f, 0.f, 0.f, 0.f));
                if (a.g2 != nullptr)
                    st_f4(reinterpret_cast<float4*>(a.g2 + i), make_float4(0.f, 0.f, 0.f, 0.f));
            }
        }
        if (fold)      // (rscale: 1 after a gather kernel, the edge weight after a DMA gather)
            xv = fma4(r[u], rscale, xv);
        if constexpr (MSG_BF16) {
            const uint2 q = f4_to_bf16x4(xv);
            st_hint_u2(reinterpret_cast<uint2*>(my_out + i), q, pol_last);
            st_hint_f4(reinterpret_cast<float4*>(a.z + i), fma4(bf16x4_to_f4(q), self_w - 1.f, xv), pol_last);
        } else if (FULL_STEP || (flags & SGP_F_PUBLISH)) {   // keep the outbox in L2 for phase 2 / peers
            st_hint_f4(reinterpret_cast<float4*>(my_out + i), xv, pol_last);
        }
        if (!FULL_STEP && write_z) store_z(a, flags, i, mul4(xv, inv_w1));
    }
}

// ---- mbarrier / bulk-copy (TMA) helpers ---------------------------------------
#define SGP_TMA_BYTES  (SGP_CHUNK * 4)      // one 4096-float chunk = 16 KB per stage

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;"
                 :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}"
        :: "r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes,
                                            uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
        :: "r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// ---- single-producer TMA ring ---------------------------------------------------
// The snapshot readers (TMA gather, consensus, SlowMo) should saturate NVLink from few SMs.
// Register-staged loads need ~300 CTAs of in-flight 16-byte requests to cover the ~2 us NVLink
// latency; here thread 0 of the CTA keeps a ring of SGP_RING_STAGES x 16 KB bulk copies
// (cp.async.bulk, global[peer] -> shared, mbarrier complete_tx) in flight, i.e. ~100 KB per CTA
// instead of ~16 KB, and the whole CTA only touches a chunk once it has landed in shared memory.
// The CTA's work is a sequence of items 0, 1, 2, ..., one fp32 chunk each; item i uses stage
// i % STAGES, and `src_of(item)` gives the chunk's global address.
#define SGP_RING_STAGES 6
#define SGP_RING_SMEM   (SGP_RING_STAGES * SGP_TMA_BYTES + SGP_RING_STAGES * 8 + 64)

struct TmaRing {
    float*    data;                                   // [STAGES][CHUNK]
    uint64_t* full;                                   // [STAGES] "the stage's copy has landed"

    // smem: the kernel's dynamic shared memory (SGP_RING_SMEM bytes, 128-byte aligned)
    __device__ __forceinline__ explicit TmaRing(unsigned char* smem)
        : data(reinterpret_cast<float*>(smem)),
          full(reinterpret_cast<uint64_t*>(smem + SGP_RING_STAGES * SGP_TMA_BYTES)) {}

    // thread 0, followed by a block barrier before anything else touches the ring
    __device__ __forceinline__ void init() const {
        for (int i = 0; i < SGP_RING_STAGES; ++i) mbar_init(&full[i], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __device__ __forceinline__ void issue(long long item, const float* src) const {
        const int stage = (int)(item % SGP_RING_STAGES);
        mbar_expect_tx(&full[stage], SGP_TMA_BYTES);
        tma_load_1d(data + (size_t)stage * SGP_CHUNK, src, SGP_TMA_BYTES, &full[stage]);
    }
    // thread 0: start the first STAGES items
    template <class SrcOf>
    __device__ __forceinline__ void fill(long long items, SrcOf&& src_of) const {
        for (long long i = 0; i < items && i < SGP_RING_STAGES; ++i) issue(i, src_of(i));
    }
    // every thread: wait until `item` has landed; returns its chunk
    __device__ __forceinline__ const float4* wait(long long item) const {
        const int stage = (int)(item % SGP_RING_STAGES);
        mbar_wait(&full[stage], (uint32_t)((item / SGP_RING_STAGES) & 1));
        return reinterpret_cast<const float4*>(data + (size_t)stage * SGP_CHUNK);
    }
    // every thread, after its last read of `item`: once the whole block is done with the stage,
    // thread 0 refills it with item + STAGES
    template <class SrcOf>
    __device__ __forceinline__ void refill(long long item, long long items, SrcOf&& src_of) const {
        __syncthreads();
        if (threadIdx.x == 0 && item + SGP_RING_STAGES < items) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic reads -> async write
            issue(item + SGP_RING_STAGES, src_of(item + SGP_RING_STAGES));
        }
    }
};

// Factors of the weighted running mean over the ranks' snapshots (consensus, SlowMo):
// f[j] = w_j / W_j with W_j = w_0 + .. + w_j, so that zbar_j = zbar_{j-1} + f[j] (z_j - zbar_{j-1}).
// One thread; the same operations in the same order wherever it is called, so every kernel and
// every rank forms zbar with the same bits
__device__ __forceinline__ void running_mean_factors(const SgpArgs& a, float* f) {
    float wsum = 0.f;
    for (int j = 0; j < a.world; ++j) {
        const float wj = ld_relaxed_sys_f32(&a.pads[j]->snap_w);
        wsum += wj;
        f[j] = wj / wsum;
    }
}

// ---- flag / ack protocol ----------------------------------------------------------
// pub_seq counts segments within a step, so at most SGP_SEQ_STRIDE - 1 of them
__device__ __forceinline__ int clamped_segments(const SgpArgs& a) {
    int segs = a.segments < 1 ? 1 : a.segments;
    if (segs > SGP_SEQ_STRIDE - 1) segs = SGP_SEQ_STRIDE - 1;
    return segs;
}

// The whole block waits until ALL pub_grid publish flags of every in-neighbour of `row` have
// reached `want` (block-parallel poll, heartbeat timeout).  Returns false in every thread when a
// wait gave up.  Its first barrier also orders what thread 0 initialised before the call
__device__ __forceinline__ bool wait_pub_flags(const SgpArgs& a, const RowInfo& row, uint32_t want, int pub_grid) {
    __shared__ int s_ok;
    if (threadIdx.x == 0) s_ok = 1;
    __syncthreads();
    for (int k = 0; k < row.n_in; ++k) {
        const int j = row.in[k];
        if (j < 0) continue;
        const SgpSignalPad* pj = a.pads[j];
        for (int f = threadIdx.x; f < pub_grid; f += blockDim.x)
            if (!spin_wait_geq(&pj->pub_seq[f], want, a.st, a.timeout_ns, SGP_ERR_TIMEOUT_PUB))
                s_ok = 0;
    }
    __syncthreads();
    return s_ok != 0;
}

// The same question without waiting: one look at every flag.  Returns the answer in every thread;
// ends with a barrier, so it may be called again at once
__device__ __forceinline__ bool pub_flags_visible(const SgpArgs& a, const RowInfo& row, uint32_t want, int pub_grid) {
    __shared__ int s_all;
    if (threadIdx.x == 0) s_all = 1;
    __syncthreads();
    for (int k = 0; k < row.n_in; ++k) {
        const int j = row.in[k];
        if (j < 0) continue;
        for (int f = threadIdx.x; f < pub_grid; f += blockDim.x)
            if ((int32_t)(ld_acquire_sys(&a.pads[j]->pub_seq[f]) - want) < 0) s_all = 0;
    }
    __syncthreads();
    const bool all = s_all != 0;
    __syncthreads();
    return all;
}

// WAR fence of the outbox: outbox[step & 1] was last read at step - 2 by that step's
// out-neighbours, and may be overwritten once each of them has acked (ack_seq >= step - 1).
// That holds from step ack_from + 2 on (outbox_was_read); before, there is nothing to wait for.
// One thread: wait_outbox_acks spins (heartbeat timeout -> false), outbox_acks_ok looks once
__device__ __forceinline__ bool outbox_was_read(const SgpArgs& a, uint32_t step) {
    return step >= a.st->ack_from + 2u;
}
__device__ __forceinline__ bool wait_outbox_acks(const SgpArgs& a, uint32_t step) {
    RowInfo prev;
    load_row(a, step - 2u, prev);
    int ok = 1;
    for (int k = 0; k < prev.n_out; ++k) {
        const int o = prev.out[k];
        if (o == a.rank || o < 0) continue;
        ok &= spin_wait_geq(&a.pads[a.rank]->ack_seq[o], step - 1u, a.st, a.timeout_ns,
                            SGP_ERR_TIMEOUT_ACK) ? 1 : 0;
    }
    return ok != 0;
}
__device__ __forceinline__ bool outbox_acks_ok(const SgpArgs& a, uint32_t step) {
    RowInfo prev;
    load_row(a, step - 2u, prev);
    bool ok = true;
    for (int k = 0; k < prev.n_out; ++k) {
        const int o = prev.out[k];
        if (o < 0 || o == a.rank) continue;
        if ((int32_t)(ld_acquire_sys(&a.pads[a.rank]->ack_seq[o]) - (step - 1u)) < 0) ok = false;
    }
    return ok;
}

// End of a gather of step s, one thread: the residual's push-sum weight, the factor the next
// publish folds it with, and the acks that release the in-neighbours' outboxes.  ok = false (a
// publish flag never came) leaves an empty residual.
// dma: a copy engine brought the raw outbox of the single in-neighbour, so the factor is that
// edge's weight; otherwise a gather kernel already applied the weights and resets done_ctas
__device__ __forceinline__ void gather_epilogue(const SgpArgs& a, const RowInfo& row, uint32_t s, bool ok, bool dma) {
    float wr = 0.f, scale = dma ? 0.f : 1.f;
    for (int k = 0; k < row.n_in; ++k) {
        const int j = row.in[k];
        if (j < 0) continue;
        if (dma) scale = row.in_w[k];               // (single in-neighbour: enforced by the host)
        wr = fmaf(row.in_w[k], ld_relaxed_sys_f32(&a.pads[j]->psw[s & 1u]), wr);
        if (j != a.rank) st_release_sys(&a.pads[j]->ack_seq[a.rank], s + 1u);
    }
    *((volatile float*)&a.st->res_weight) = ok ? wr : 0.f;
    *((volatile float*)&a.st->res_scale) = (ok || !dma) ? scale : 0.f;
    if (!dma) *((volatile uint32_t*)&a.st->done_ctas) = 0u;
    __threadfence();
}

}  // namespace

// ---------------------------------------------------------------------------
// Fused step kernel.  MSG_BF16 (SGP_F_MSG_BF16): bf16 messages, full synchronous step only
// (PHASE1 | PUBLISH | PHASE2; the launcher rejects every other mode): phase 1 publishes Q(x) and
// keeps c = x - (1 - self_w) Q(x) in z, phase 2 mixes c + sum_k in_w[k] Q(x_k).
// GROUPS (SGP_F_GROUPS): per-parameter-group SGD, see load_group_rows / block_group_of.
// LARS (SGP_F_LARS, only with GROUPS): per-tensor trust ratio, see lars_trust_of.
// ---------------------------------------------------------------------------
template <bool MSG_BF16, bool GROUPS, bool LARS>
__global__ void __launch_bounds__(SGP_THREADS, 2)
sgp_step_kernel(const SgpArgs a)
{
    using Msg = typename std::conditional<MSG_BF16, __nv_bfloat16, float>::type;
    __shared__ float s_wn;        // new push-sum weight
    __shared__ int   s_ok;

    SgpState* st = a.st;
    const uint32_t step   = *((volatile uint32_t*)&st->step);
    const uint32_t parity = step & 1u;
    // AD-PSGD: the mode bits come from the device-side round state machine (what the preceding
    // sgp_bilat_decide_kernel decided); nothing to do -> the whole grid exits at once
    const bool from_state = (a.flags & SGP_F_FROM_STATE) != 0;
    const uint32_t flags  = from_state
        ? ((a.flags & (SGP_F_SHADOW | SGP_F_GRAD_BF16)) | *((volatile uint32_t*)&st->bilat_cmd))
        : a.flags;
    if (from_state && (flags & (SGP_F_PHASE1 | SGP_F_PHASE2)) == 0u) return;
    const int      tid    = threadIdx.x;
    const int      b      = blockIdx.x;
    const long long nchunks = a.n / SGP_CHUNK;

    RowInfo row;
    load_row(a, step, row);

    const float w0 = *((volatile float*)&st->ps_weight[parity]);
    const float wmul = (flags & SGP_F_IN_NUMER) ? 1.f : w0;   // z -> numerator factor
    const float wres = (flags & SGP_F_FOLD_RES) ? *((volatile float*)&st->res_weight) : 0.f;
    const float rscale = (flags & SGP_F_FOLD_RES) ? *((volatile float*)&st->res_scale) : 1.f;
    const float w1 = w0 + wres;                    // weight of the published numerator

    SgpSignalPad* mypad = a.pads[a.rank];
    Msg* my_out = a.outboxes ? (reinterpret_cast<Msg*>(a.outboxes[a.rank]) + (size_t)parity * a.n) : nullptr;

    const SgpHyper hp = *a.hyper;
    const uint64_t pol_first = l2_evict_first_policy();
    const uint64_t pol_last = l2_evict_last_policy();
    const bool do_sgd = (flags & SGP_F_SGD) && (hp.do_sgd != 0.f);
    const float4* s_rows = nullptr;
    if constexpr (GROUPS) {
        __shared__ float4 s_group_rows[SGP_MAX_GROUPS];
        load_group_rows(a, s_group_rows, tid);
        __syncthreads();
        s_rows = s_group_rows;
    }

    // Work decomposition: this CTA owns chunks b, b+G, b+2G, ...; they are cut into
    // K contiguous SEGMENTS.  For each segment the CTA runs phase 1 (local update +
    // publish, HBM-bound), releases a per-CTA progress counter
    //        pub_seq[b] = step * SGP_SEQ_STRIDE + seg + 1
    // and immediately runs phase 2 (pull + mix, NVLink-bound) on the same segment.
    // CTAs sharing an SM drift apart, so one CTA's NVLink phase overlaps another's
    // HBM phase and the kernel approaches max(HBM time, NVLink time) instead of
    // their sum; the own-term re-read of phase 2 always hits L2.
    const long long my_chunks = cta_chunks(nchunks, b);
    const int K = clamped_segments(a);
    const uint32_t seq_base = step * (uint32_t)SGP_SEQ_STRIDE;

    if ((flags & SGP_F_PHASE1) && (flags & SGP_F_PUBLISH) && outbox_was_read(a, step)) {
        if (tid == 0) s_ok = wait_outbox_acks(a, step) ? 1 : 0;      // before overwriting outbox[parity]
        __syncthreads();
    }

    const float inv_w1 = 1.f / w1;
    const bool write_z = !(flags & SGP_F_PHASE2) && !(flags & SGP_F_KEEP_Z);
    // overlap publish keeps the self-loop share locally (w <- self_w * w1); a
    // snapshot-only publish (AD-PSGD) leaves the weight alone
    float w_next = ((flags & SGP_F_PUBLISH) && !(flags & SGP_F_KEEP_Z)) ? row.self_w * w1 : w1;
    float inv_wn = 1.f;
    bool pull_ok = true;
    const Msg* peer_out[SGP_MAX_PEERS];
#pragma unroll
    for (int k = 0; k < SGP_MAX_PEERS; ++k)
        peer_out[k] = ((flags & SGP_F_PHASE2) && k < row.n_in && row.in[k] >= 0)
                          ? reinterpret_cast<const Msg*>(a.outboxes[row.in[k]]) + (size_t)parity * a.n : nullptr;

    for (int seg = 0; seg < K; ++seg) {
        const long long it_lo = my_chunks * seg / K;
        const long long it_hi = my_chunks * (seg + 1) / K;

        // ---------------- phase 1: local update + publish ------------------
        if (flags & SGP_F_PHASE1) {
            for (long long it = it_lo; it < it_hi; ++it)
                phase1_chunk<MSG_BF16, GROUPS, LARS, false>(a, flags, b + it * gridDim.x, tid, hp, do_sgd, s_rows,
                                                            wmul, row.self_w, my_out, pol_first, pol_last,
                                                            rscale, inv_w1, write_z);
            if (flags & SGP_F_PUBLISH) {
                __syncthreads();
                if (tid == 0) {
                    if (seg == 0) st_relaxed_sys_f32(&mypad->psw[parity], w1);  // same value from every CTA
                    __threadfence_system();
                    st_release_sys(&mypad->pub_seq[b], seq_base + (uint32_t)seg + 1u);
                }
            }
        }

        // ---------------- phase 2: pull + mix ------------------------------
        if (flags & SGP_F_PHASE2) {
            if (tid == 0) {
                int ok = 1;
                float wn = row.self_w * w1;
                for (int k = 0; k < row.n_in; ++k) {
                    const int j = row.in[k];
                    if (j < 0) continue;
                    const SgpSignalPad* pj = a.pads[j];
                    ok &= spin_wait_geq(&pj->pub_seq[b], seq_base + (uint32_t)seg + 1u, st,
                                        a.timeout_ns, SGP_ERR_TIMEOUT_PUB) ? 1 : 0;
                    if (seg == 0) wn = fmaf(row.in_w[k], ld_relaxed_sys_f32(&pj->psw[parity]), wn);
                }
                if (seg == 0) s_wn = wn;
                s_ok = ok;
            }
            __syncthreads();
            if (seg == 0) {
                w_next = s_wn;
                inv_wn = 1.f / s_wn;
            }
            pull_ok = pull_ok && (s_ok != 0);
            if (pull_ok) {
                for (long long it = it_lo; it < it_hi; ++it) {
                    const long long c = b + it * gridDim.x;
                    const long long base = chunk_base(c, tid);
                    float4 acc[SGP_UNROLL];
                    float4 pv[SGP_UNROLL];
#pragma unroll
                    for (int u = 0; u < SGP_UNROLL; ++u) {
                        const long long i = chunk_elem(base, u);
                        if constexpr (MSG_BF16) {
                            // own term: c, kept in z by phase 1 (already carries the self weight)
                            acc[u] = ld_once_f4(reinterpret_cast<const float4*>(a.z + i), pol_first);
                        } else {
                            // own term: the snapshot this CTA just published (L2-resident),
                            // or (AD-PSGD) the live parameters, which may already carry
                            // newer local SGD updates
                            const float* own = (flags & SGP_F_SELF_FROM_Z) ? a.z : my_out;
                            acc[u] = mul4(ld_once_f4(reinterpret_cast<const float4*>(own + i), pol_first),
                                          (flags & SGP_F_SELF_FROM_Z) ? row.self_w * w0 : row.self_w);
                        }
                    }
                    // peer loads: all UNROLL requests of one peer in flight together
                    for (int k = 0; k < row.n_in; ++k) {
                        const Msg* po = peer_out[k];
                        if (po == nullptr) continue;
#pragma unroll
                        for (int u = 0; u < SGP_UNROLL; ++u) {
                            const long long i = chunk_elem(base, u);
                            if constexpr (MSG_BF16)
                                pv[u] = bf16x4_to_f4(ld_stream_u2(reinterpret_cast<const uint2*>(po + i)));
                            else
                                pv[u] = ld_stream_f4(reinterpret_cast<const float4*>(po + i));
                        }
                        const float wk = row.in_w[k];
#pragma unroll
                        for (int u = 0; u < SGP_UNROLL; ++u) acc[u] = fma4(pv[u], wk, acc[u]);
                    }
#pragma unroll
                    for (int u = 0; u < SGP_UNROLL; ++u) {
                        const long long i = chunk_elem(base, u);
                        const float4 zv = mul4(acc[u], inv_wn);
                        store_z(a, flags, i, zv);
                    }
                }
            }
            else if (!(flags & SGP_F_SELF_FROM_Z) && (flags & SGP_F_PHASE1)) {
                // an in-neighbour timed out: "every in-message of this round was lost" -- de-bias the
                // numerator this CTA published (a valid push-sum state) instead of leaving the
                // pre-SGD parameters behind; the sticky status word makes the host raise.  With bf16
                // messages the numerator this rank still holds is c (it sent the rest), carrying the
                // weight self_w * w1 -- see sgp_step_pipe_kernel
                const float inv_own = MSG_BF16 ? 1.f / (row.self_w * w1) : 1.f / w1;
                const float* own;
                if constexpr (MSG_BF16) own = a.z; else own = my_out;
                for (long long it = it_lo; it < it_hi; ++it) {
                    const long long c = b + it * gridDim.x;
                    const long long base = chunk_base(c, tid);
#pragma unroll
                    for (int u = 0; u < SGP_UNROLL; ++u) {
                        const long long i = chunk_elem(base, u);
                        const float4 zv = mul4(ld_once_f4(reinterpret_cast<const float4*>(own + i), pol_first),
                                               inv_own);
                        store_z(a, flags, i, zv);
                    }
                }
            }
            __syncthreads();     // s_ok / s_wn are rewritten by the next segment
        }
    }

    // ---------------- epilogue: last CTA publishes state + acks ------------
    __syncthreads();
    if (tid == 0 && cta_done_is_last(st)) {
        if (flags & SGP_F_PHASE2) {
            for (int k = 0; k < row.n_in; ++k) {
                const int j = row.in[k];
                if (j < 0 || j == a.rank) continue;
                st_release_sys(&a.pads[j]->ack_seq[a.rank], step + 1u);
            }
        }
        const bool rotate = !(flags & SGP_F_NO_ROTATE);
        *((volatile float*)&st->ps_weight[rotate ? (parity ^ 1u) : parity]) = w_next;
        if (flags & SGP_F_FOLD_RES) *((volatile float*)&st->res_weight) = 0.f;
        *((volatile uint32_t*)&st->done_ctas) = 0u;
        if (rotate) *((volatile uint32_t*)&st->step) = step + 1u;
        if (from_state) {                       // bilateral round bookkeeping
            if (rotate) {                       // round complete
                st->bilat_published = 0u;
                st->bilat_round += 1u;
            } else if (flags & SGP_F_PUBLISH) {
                st->bilat_published = 1u;       // snapshot is out; the pull follows in a later launch
            }
            st->bilat_cmd = 0u;
        }
        __threadfence();
    }
}

// ---------------------------------------------------------------------------
// Overlap-SGP gather: residual = sum_k in_w[k] * outbox_k[parity]   (side stream)
// Runs after the local publish kernel of the same step, i.e. st->step == s+1.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(SGP_THREADS, 2)
sgp_gather_kernel(const SgpArgs a, const int pub_grid)
{
    SgpState* st = a.st;
    const uint32_t s      = *((volatile uint32_t*)&st->step) - 1u;
    const uint32_t parity = s & 1u;
    const int tid = threadIdx.x;
    const long long nchunks = a.n / SGP_CHUNK;

    RowInfo row;
    load_row(a, s, row);
    const bool ok = wait_pub_flags(a, row, s * (uint32_t)SGP_SEQ_STRIDE + (uint32_t)clamped_segments(a), pub_grid);

    if (ok) {
        const float* peer_out[SGP_MAX_PEERS];
#pragma unroll
        for (int k = 0; k < SGP_MAX_PEERS; ++k)
            peer_out[k] = (k < row.n_in && row.in[k] >= 0)
                              ? a.outboxes[row.in[k]] + (size_t)parity * a.n : nullptr;
        for (long long c = blockIdx.x; c < nchunks; c += gridDim.x) {
            const long long base = chunk_base(c, tid);
            float4 acc[SGP_UNROLL], pv[SGP_UNROLL];
#pragma unroll
            for (int u = 0; u < SGP_UNROLL; ++u) acc[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int k = 0; k < row.n_in; ++k) {
                const float* po = peer_out[k];
                if (po == nullptr) continue;
#pragma unroll
                for (int u = 0; u < SGP_UNROLL; ++u)
                    pv[u] = ld_stream_f4(reinterpret_cast<const float4*>(po + chunk_elem(base, u)));
#pragma unroll
                for (int u = 0; u < SGP_UNROLL; ++u) acc[u] = fma4(pv[u], row.in_w[k], acc[u]);
            }
#pragma unroll
            for (int u = 0; u < SGP_UNROLL; ++u)
                st_f4(reinterpret_cast<float4*>(a.residual + chunk_elem(base, u)), acc[u]);
        }
    }

    __syncthreads();
    if (tid == 0 && cta_done_is_last(st)) gather_epilogue(a, row, s, ok, false);
}

// ---------------------------------------------------------------------------
// Overlap-SGP gather, TMA variant.  The gather runs on a side stream next to the
// forward/backward pass, so it should saturate NVLink from as FEW SMs as possible: the peers'
// chunks come through the TmaRing; items are (chunk, in-peer) pairs, peer fastest.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(SGP_THREADS, 1)
sgp_gather_tma_kernel(const SgpArgs a, const int pub_grid)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const TmaRing ring(smem_raw);

    SgpState* st = a.st;
    const uint32_t s      = *((volatile uint32_t*)&st->step) - 1u;
    const uint32_t parity = s & 1u;
    const int tid = threadIdx.x;
    const long long nchunks = a.n / SGP_CHUNK;

    RowInfo row;
    load_row(a, s, row);

    if (tid == 0) ring.init();
    const bool ok = wait_pub_flags(a, row, s * (uint32_t)SGP_SEQ_STRIDE + (uint32_t)clamped_segments(a), pub_grid);

    const int n_in = row.n_in;
    const long long items = ok ? cta_chunks(nchunks, blockIdx.x) * n_in : 0;     // (chunk, in-peer) pairs, peer fastest
    const auto src_of = [&](long long item) -> const float* {
        const long long it = item / n_in;
        const int k = (int)(item - it * n_in);
        const long long c = blockIdx.x + it * gridDim.x;
        return a.outboxes[row.in[k]] + (size_t)parity * a.n + c * SGP_CHUNK;
    };
    if (tid == 0) ring.fill(items, src_of);

    float4 acc[SGP_UNROLL];
    for (long long item = 0; item < items; ++item) {
        const long long it = item / n_in;
        const int k = (int)(item - it * n_in);
        const float4* src = ring.wait(item);
        const float wk = row.in_w[k];
#pragma unroll
        for (int u = 0; u < SGP_UNROLL; ++u) {
            const float4 v = src[tid + u * SGP_THREADS];
            acc[u] = (k == 0) ? mul4(v, wk) : fma4(v, wk, acc[u]);
        }
        if (k == n_in - 1) {
            const long long c = blockIdx.x + it * gridDim.x;
            float4* dst = reinterpret_cast<float4*>(a.residual + c * SGP_CHUNK);
#pragma unroll
            for (int u = 0; u < SGP_UNROLL; ++u) st_f4(dst + tid + u * SGP_THREADS, acc[u]);
        }
        ring.refill(item, items, src_of);
    }

    __syncthreads();
    if (tid == 0 && cta_done_is_last(st)) gather_epilogue(a, row, s, ok, false);
}

// ---------------------------------------------------------------------------
// Fused step kernel, warp-specialised + TMA-fed variant (the SGP / D-PSGD hot path).
//
// sgp_step_kernel pulls the peers' outboxes with register-staged 16-byte loads: every
// consumer thread has 4 x 16 B in flight and the CTA alternates between an HBM-bound phase 1
// and an NVLink-bound phase 2, so its time is close to the sum of the two.  Here the two phases run on different warps of the same CTA:
//
//   warps 0-7 (consumers)  for seg = 0..K:   phase 1 of segment `seg`   (SGD + publish, HBM)
//                                            phase 2 of segment `seg-1` (mix + de-bias)
//                          phase 2 reads the peers' data from SHARED MEMORY, where it has
//                          been landing while phase 1 of the next segment was streaming HBM
//   warp 8 lane 0 (producer) per segment: acquire the in-neighbours' publish flags, then keep
//                          a ring of PIPE_STAGES x 16 KB bulk copies (cp.async.bulk,
//                          peer global -> shared, mbarrier complete_tx) in flight over NVLink
//
// so the NVLink stream starts as soon as the first segment of the peer is published and
// never waits for a consumer register to free up; the consumers never wait for NVLink
// latency.  Flags, outbox layout, acks and the last-CTA epilogue are those of
// sgp_step_kernel (gather / probe / the old kernel interoperate with it); the grid must be
// the same on all ranks (flags are matched by CTA index).
//
// (Tried and rejected, round 2: splitting the consumers into a phase-1 group and a phase-2 group of
// four warps each so that both streams run concurrently inside a CTA -- 0.298 ms vs 0.254 ms for
// this version on 2 GPUs: four warps per stream no longer cover the HBM / shared-memory latencies.)
//
// A timed-out flag wait does not leave stale parameters behind: the producer marks the CTA
// failed, completes its barriers without data, and the consumers de-bias their own published
// numerator instead (z = x_own / w1, i.e. "every in-message of this round was lost" -- a valid
// push-sum state); the sticky status word makes the host raise at its next poll.
//
// MSG_BF16 (SGP_F_MSG_BF16): the outbox holds Q(x) = bf16(x) and each ring stage one 8 KB bf16
// chunk.  Phase 1 keeps c = x - (1 - self_w) Q(x) in z (overwritten by phase 2 anyway) and phase 2
// computes c + sum_k in_w[k] Q(x_k): the sender loses exactly what its out-neighbours receive, so
// sum_i x_i is conserved for any column-stochastic schedule.  On a timed-out in-neighbour the
// consumers de-bias c over self_w * w1 (the weight the rank keeps when every in-message is lost):
// c is what this rank still holds after sending, so the fallback stays a valid push-sum state.
// That needs self_w > 0, which every mixing of this project has (1 / (peers + 1) for uniform).
// ---------------------------------------------------------------------------
#define PIPE_STAGES    4
#define PIPE_CONSUMERS SGP_THREADS                 // 256: the chunk decomposition of sgp_step_kernel
#define PIPE_THREADS   (PIPE_CONSUMERS + 32)
#define PIPE_SMEM      (PIPE_STAGES * SGP_TMA_BYTES + 2 * PIPE_STAGES * 8 + 64)

// 9 warps x 2 CTAs per SM: the register file is split over 4 sub-partitions (16 K registers
// each), so 18 warps only fit at <= 102 registers per thread -- __launch_bounds__(288, 2) makes
// ptxas pick 96.  (At 112 registers the kernel runs one CTA per SM.)
// GROUPS (SGP_F_GROUPS) and LARS (SGP_F_LARS): as in sgp_step_kernel.
template <bool MSG_BF16, bool GROUPS, bool LARS>
__global__ void __launch_bounds__(PIPE_THREADS, 2)
sgp_step_pipe_kernel(const SgpArgs a)
{
    using Msg = typename std::conditional<MSG_BF16, __nv_bfloat16, float>::type;
    constexpr uint32_t MSG_BYTES = SGP_CHUNK * sizeof(Msg);                    // one chunk per stage
    extern __shared__ __align__(128) unsigned char smem_raw[];
    unsigned char* ring = smem_raw;                                            // [STAGES][MSG_BYTES]
    uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + PIPE_STAGES * SGP_TMA_BYTES);
    uint64_t* empty = full + PIPE_STAGES;
    uint64_t* wbar = empty + PIPE_STAGES;            // new push-sum weight is known
    __shared__ float s_wn;
    __shared__ int   s_ok;                            // WAR fence outcome (consumers)
    __shared__ volatile int s_fail;                   // producer: an in-neighbour timed out

    SgpState* st = a.st;
    const uint32_t step   = *((volatile uint32_t*)&st->step);
    const uint32_t parity = step & 1u;
    const uint32_t flags  = a.flags;
    const int      tid    = threadIdx.x;
    const int      warp   = tid >> 5;
    const int      b      = blockIdx.x;
    const long long nchunks = a.n / SGP_CHUNK;

    RowInfo row;
    load_row(a, step, row);

    const float w0 = *((volatile float*)&st->ps_weight[parity]);
    const float wmul = (flags & SGP_F_IN_NUMER) ? 1.f : w0;
    const float w1 = w0;                              // (no residual fold in the synchronous step)

    SgpSignalPad* mypad = a.pads[a.rank];
    Msg* my_out = reinterpret_cast<Msg*>(a.outboxes[a.rank]) + (size_t)parity * a.n;

    const long long my_chunks = cta_chunks(nchunks, b);
    const int K = clamped_segments(a);
    const uint32_t seq_base = step * (uint32_t)SGP_SEQ_STRIDE;

    // compacted in-neighbour list (table entries < 0 are holes)
    int n_in = 0;
    int in_rank[SGP_MAX_PEERS];
    float in_w[SGP_MAX_PEERS];
#pragma unroll
    for (int k = 0; k < SGP_MAX_PEERS; ++k)
        if (k < row.n_in && row.in[k] >= 0) { in_rank[n_in] = row.in[k]; in_w[n_in] = row.in_w[k]; ++n_in; }

    if (tid == 0) {
        for (int i = 0; i < PIPE_STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], PIPE_CONSUMERS / 32); }
        mbar_init(wbar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        s_fail = 0;
        s_ok = 1;
    }
    const float4* s_rows = nullptr;
    if constexpr (GROUPS) {
        __shared__ float4 s_group_rows[SGP_MAX_GROUPS];
        load_group_rows(a, s_group_rows, tid);
        s_rows = s_group_rows;
    }
    __syncthreads();

    if (warp == PIPE_CONSUMERS / 32) {
        // ============================ producer ============================
        if ((tid & 31) == 0) {
            int stage = 0;
            uint32_t phase = 0;
            bool ok = true;
            float wn = row.self_w * w1;
            for (int seg = 0; seg < K; ++seg) {
                for (int k = 0; k < n_in && ok; ++k) {
                    const SgpSignalPad* pj = a.pads[in_rank[k]];
                    ok = spin_wait_geq(&pj->pub_seq[b], seq_base + (uint32_t)seg + 1u, st, a.timeout_ns,
                                       SGP_ERR_TIMEOUT_PUB);
                    if (ok && seg == 0) wn = fmaf(in_w[k], ld_relaxed_sys_f32(&pj->psw[parity]), wn);
                }
                if (!ok) s_fail = 1;
                if (seg == 0) {
                    s_wn = ok ? wn : row.self_w * w1;
                    __threadfence_block();
                    mbar_arrive(wbar);
                }
                const long long it_lo = my_chunks * seg / K, it_hi = my_chunks * (seg + 1) / K;
                for (long long it = it_lo; it < it_hi; ++it) {
                    const long long c = b + it * gridDim.x;
                    for (int k = 0; k < n_in; ++k) {
                        mbar_wait(&empty[stage], phase ^ 1u);
                        if (ok) {
                            const Msg* src = reinterpret_cast<const Msg*>(a.outboxes[in_rank[k]]) +
                                             (size_t)parity * a.n + c * SGP_CHUNK;
                            mbar_expect_tx(&full[stage], MSG_BYTES);
                            tma_load_1d(ring + (size_t)stage * MSG_BYTES, src, MSG_BYTES, &full[stage]);
                        } else {
                            mbar_arrive(&full[stage]);           // nothing will land: release the consumers
                        }
                        if (++stage == PIPE_STAGES) { stage = 0; phase ^= 1u; }
                    }
                }
            }
        }
        __syncwarp();
    } else {
        // ============================ consumers ============================
        const SgpHyper hp = *a.hyper;
        const uint64_t pol_first = l2_evict_first_policy();
        const uint64_t pol_last = l2_evict_last_policy();
        const bool do_sgd = (flags & SGP_F_SGD) && (hp.do_sgd != 0.f);
        const int lane = tid & 31;

        if (outbox_was_read(a, step)) {
            if (tid == 0) s_ok = wait_outbox_acks(a, step) ? 1 : 0;      // before overwriting outbox[parity]
            asm volatile("bar.sync 1, %0;" :: "n"(PIPE_CONSUMERS) : "memory");
        }

        int cstage = 0;
        uint32_t cphase = 0;
        float inv_wn = 1.f;
        const float inv_w1 = 1.f / w1;

        for (int seg = 0; seg <= K; ++seg) {
            // ---------------- phase 1 of segment `seg`: local update + publish ----------------
            if (seg < K) {
                const long long it_lo = my_chunks * seg / K, it_hi = my_chunks * (seg + 1) / K;
                for (long long it = it_lo; it < it_hi; ++it)
                    phase1_chunk<MSG_BF16, GROUPS, LARS, true>(a, flags, b + it * gridDim.x, tid, hp, do_sgd, s_rows,
                                                               wmul, row.self_w, my_out, pol_first, pol_last,
                                                               1.f, inv_w1, false);
                asm volatile("bar.sync 1, %0;" :: "n"(PIPE_CONSUMERS) : "memory");
                if (tid == 0) {
                    if (seg == 0) st_relaxed_sys_f32(&mypad->psw[parity], w1);
                    __threadfence_system();
                    st_release_sys(&mypad->pub_seq[b], seq_base + (uint32_t)seg + 1u);
                }
            }
            // ---------------- phase 2 of segment `seg - 1`: mix + de-bias ----------------
            if (seg >= 1) {
                const int ps = seg - 1;
                if (ps == 0) {
                    mbar_wait(wbar, 0);
                    inv_wn = 1.f / s_wn;
                }
                const long long it_lo = my_chunks * ps / K, it_hi = my_chunks * (ps + 1) / K;
                for (long long it = it_lo; it < it_hi; ++it) {
                    const long long c = b + it * gridDim.x;
                    const long long base = chunk_base(c, tid);
                    float4 acc[SGP_UNROLL];
#pragma unroll
                    for (int u = 0; u < SGP_UNROLL; ++u) {
                        const long long i = chunk_elem(base, u);
                        if constexpr (MSG_BF16)      // c already carries the self weight
                            acc[u] = ld_once_f4(reinterpret_cast<const float4*>(a.z + i), pol_first);   // L2 hit
                        else
                            acc[u] = mul4(ld_once_f4(reinterpret_cast<const float4*>(my_out + i), pol_first),   // L2 hit
                                          row.self_w);
                    }
                    for (int k = 0; k < n_in; ++k) {
                        mbar_wait(&full[cstage], cphase);
                        const unsigned char* stage_p = ring + (size_t)cstage * MSG_BYTES;
                        const float wk = in_w[k];
#pragma unroll
                        for (int u = 0; u < SGP_UNROLL; ++u) {
                            float4 v;
                            if constexpr (MSG_BF16)
                                v = bf16x4_to_f4(reinterpret_cast<const uint2*>(stage_p)[tid + u * SGP_THREADS]);
                            else
                                v = reinterpret_cast<const float4*>(stage_p)[tid + u * SGP_THREADS];
                            acc[u] = fma4(v, wk, acc[u]);
                        }
                        __syncwarp();
                        if (lane == 0) mbar_arrive(&empty[cstage]);     // this warp is done with the stage
                        if (++cstage == PIPE_STAGES) { cstage = 0; cphase ^= 1u; }
                    }
                    const bool failed = s_fail != 0;           // (rare: re-read the own numerator)
#pragma unroll
                    for (int u = 0; u < SGP_UNROLL; ++u) {
                        const long long i = chunk_elem(base, u);
                        float4 zv;
                        if constexpr (MSG_BF16)    // own numerator c (still in z) over the weight kept
                            zv = failed ? mul4(ld_once_f4(reinterpret_cast<const float4*>(a.z + i), pol_first),
                                               inv_w1 / row.self_w)
                                        : mul4(acc[u], inv_wn);
                        else
                            zv = failed
                                ? mul4(ld_once_f4(reinterpret_cast<const float4*>(my_out + i), pol_first), inv_w1)
                                : mul4(acc[u], inv_wn);
                        store_z(a, flags, i, zv);
                    }
                }
            }
        }
    }

    // ---------------- epilogue: last CTA publishes state + acks ------------
    __syncthreads();
    if (tid == 0 && cta_done_is_last(st)) {
        for (int k = 0; k < n_in; ++k)
            if (in_rank[k] != a.rank) st_release_sys(&a.pads[in_rank[k]]->ack_seq[a.rank], step + 1u);
        *((volatile float*)&st->ps_weight[parity ^ 1u]) = s_wn;
        *((volatile uint32_t*)&st->done_ctas) = 0u;
        *((volatile uint32_t*)&st->step) = step + 1u;
        __threadfence();
    }
}

// ---------------------------------------------------------------------------
// AD-PSGD passive poll: did the in-neighbour of the current round publish?
// ---------------------------------------------------------------------------
__global__ void sgp_probe_kernel(const SgpArgs a, const int pub_grid, uint32_t* host_flag)
{
    SgpState* st = a.st;
    const uint32_t step = *((volatile uint32_t*)&st->step);
    RowInfo row;
    load_row(a, step, row);
    const uint32_t all = pub_flags_visible(a, row, step * (uint32_t)SGP_SEQ_STRIDE + (uint32_t)clamped_segments(a),
                                           pub_grid) ? 1u : 0u;
    if (threadIdx.x == 0) {
        // may outbox[step&1] be overwritten?  (the publish kernel would otherwise
        // spin on these acks; the host checks first so no kernel ever waits)
        const uint32_t acks_ok = (!outbox_was_read(a, step) || outbox_acks_ok(a, step)) ? 1u : 0u;
        st->bilat_done = all;
        if (host_flag) {
            ((volatile uint32_t*)host_flag)[0] = all;
            ((volatile uint32_t*)host_flag)[1] = acks_ok;
        }
        __threadfence_system();
    }
}

// ---------------------------------------------------------------------------
// Overlap-SGP gather on the COPY ENGINES (one in-neighbour per step).  A gather kernel on the side
// stream -- even the 32-CTA TMA one -- holds SMs while the forward pass starts: persistent
// one-CTA-per-SM kernels (the wgmma GEMMs) and 2-CTA/SM tile loops then wait for "their" SM, and
// the overlap costs more than it hides.  With a single in-neighbour the residual is just a copy of the peer's
// outbox, so:
//     sgp_gather_wait_kernel   ONE CTA: wait for the in-neighbour's publish flags of this step
//     cudaMemcpyAsync          peer outbox -> residual, 100 MB over NVLink on a DMA engine: zero SMs
//     sgp_gather_ack_kernel    ONE thread: residual weight / scale (= the edge weight; applied when
//                              the next publish folds the residual), ack the outbox to its owner
// ---------------------------------------------------------------------------
__global__ void sgp_gather_wait_kernel(const SgpArgs a, const int pub_grid)
{
    SgpState* st = a.st;
    const uint32_t s = *((volatile uint32_t*)&st->step) - 1u;
    RowInfo row;
    load_row(a, s, row);
    // (a timeout is left in st->status, where sgp_gather_ack_kernel finds it)
    wait_pub_flags(a, row, s * (uint32_t)SGP_SEQ_STRIDE + (uint32_t)clamped_segments(a), pub_grid);
}

__global__ void sgp_gather_ack_kernel(const SgpArgs a)
{
    SgpState* st = a.st;
    const uint32_t s = *((volatile uint32_t*)&st->step) - 1u;
    RowInfo row;
    load_row(a, s, row);
    const bool ok = *((volatile uint32_t*)&st->status) == SGP_OK;
    __threadfence_system();                         // the DMA copy before this kernel has completed
    gather_epilogue(a, row, s, ok, true);
}

// ---------------------------------------------------------------------------
// AD-PSGD round state machine, device side.  One CTA decides what the NEXT worker launch
// (sgp_step_kernel with SGP_F_FROM_STATE) does, from flags only:
//   * active ranks publish their snapshot unconditionally, passive ranks only once their
//     partner's snapshot of this round is visible (gossip/gossiper.py:290-316);
//   * nobody publishes before the readers of round r-2 released the outbox half;
//   * the pull (x <- 1/2 (x_now + x_partner), ack, advance) runs once both snapshots are out;
//   * waiting for the partner is BOUNDED (max_wait_ns, ~50 us): if it does not show up the
//     launch pair does nothing (or only publishes) and the daemon simply enqueues the next
//     pair -- no kernel ever spins for long, no host synchronisation per poll;
//   * a rank only STARTS a round while it has budget (rounds per applied gradient) and gossip
//     is enabled; a round whose snapshot is already out is always completed.
// host_fb (pinned, optional): [0] = decided bits, [1] = rounds completed, [2] = status word.
// ---------------------------------------------------------------------------
__global__ void sgp_bilat_decide_kernel(const SgpArgs a, const int pub_grid, const int passive,
                                        const unsigned long long max_wait_ns, uint32_t* host_fb)
{
    __shared__ int s_stop;
    __shared__ uint32_t s_published, s_may_start;
    SgpState* st = a.st;
    const uint32_t step = *((volatile uint32_t*)&st->step);
    RowInfo row;
    load_row(a, step, row);
    const uint32_t want = step * (uint32_t)SGP_SEQ_STRIDE + (uint32_t)clamped_segments(a);
    // bilat_budget / bilat_enabled are rewritten asynchronously (sgp_bilat_ctl_kernel on the
    // training stream): ONE thread samples them and the whole CTA uses that sample, so that every
    // thread takes the same branch around the barrier loop below
    if (threadIdx.x == 0) {
        s_published = *((volatile uint32_t*)&st->bilat_published);
        s_may_start = ((*((volatile uint32_t*)&st->bilat_enabled) != 0u) &&
                       (*((volatile uint32_t*)&st->bilat_budget) != 0u)) ? 1u : 0u;
    }
    __syncthreads();
    const uint32_t published = s_published;
    const bool may_start = s_may_start != 0u;
    const bool engaged = published != 0u || may_start;

    int ready = 0;
    if (engaged) {
        const unsigned long long t0 = globaltimer_ns();
        while (true) {
            ready = pub_flags_visible(a, row, want, pub_grid) ? 1 : 0;
            // ONE thread decides whether to stop (the deadline must not be evaluated per thread:
            // threads straddling it would leave the barrier loop at different iterations)
            if (threadIdx.x == 0) s_stop = (ready != 0) || (globaltimer_ns() - t0 > max_wait_ns);
            __syncthreads();
            const int stop = s_stop;
            __syncthreads();                  // s_stop is rewritten by the next iteration
            if (stop) break;
            __nanosleep(500);
        }
    }
    if (threadIdx.x != 0) return;
    const bool acks_ok = !outbox_was_read(a, step) || outbox_acks_ok(a, step);
    const bool do_publish = !published && may_start && acks_ok && (ready || !passive);
    const bool do_pull = ready && (published || do_publish);
    uint32_t cmd = 0u;
    if (do_publish && do_pull)
        cmd = SGP_F_PHASE1 | SGP_F_PUBLISH | SGP_F_KEEP_Z | SGP_F_PHASE2 | SGP_F_SELF_FROM_Z;
    else if (do_publish)
        cmd = SGP_F_PHASE1 | SGP_F_PUBLISH | SGP_F_KEEP_Z | SGP_F_NO_ROTATE;
    else if (do_pull)
        cmd = SGP_F_PHASE2 | SGP_F_PUBLISH | SGP_F_SELF_FROM_Z;
    if (do_publish) {                          // starting a round consumes budget
        // (compare-and-swap: a budget that sgp_bilat_ctl_kernel rewrote in the meantime wins)
        const uint32_t bud = *((volatile uint32_t*)&st->bilat_budget);
        if (bud != 0xFFFFFFFFu && bud > 0u) atomicCAS(&st->bilat_budget, bud, bud - 1u);
    }
    st->bilat_cmd = cmd;
    st->bilat_done = (uint32_t)ready;
    __threadfence();
    if (host_fb) {
        ((volatile uint32_t*)host_fb)[0] = cmd;
        ((volatile uint32_t*)host_fb)[1] = st->bilat_round + (do_pull ? 1u : 0u);
        ((volatile uint32_t*)host_fb)[2] = st->status;
        __threadfence_system();
    }
}

// budget < 0 / enabled < 0: leave the field alone.  budget == INT_MAX: unbounded
__global__ void sgp_bilat_ctl_kernel(SgpState* st, int budget, int enabled)
{
    if (budget >= 0) st->bilat_budget = (budget == 0x7FFFFFFF) ? 0xFFFFFFFFu : (uint32_t)budget;
    if (enabled >= 0) st->bilat_enabled = (uint32_t)enabled;
    __threadfence();
}

// ---------------------------------------------------------------------------
// AR-SGD comparator: one-shot P2P all-reduce of the (symmetric) gradient
// buffers fused with the SGD update.  Every rank sums in rank order, so the
// replicas stay bit-identical.  pub_seq doubles as the "gradients ready"
// barrier, ack_seq as the "done reading" barrier.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(SGP_THREADS, 2)
sgp_allreduce_sgd_kernel(const SgpArgs a, void* const* grad_peers)
{
    __shared__ int s_ok;
    SgpState* st = a.st;
    const uint32_t step = *((volatile uint32_t*)&st->step);
    const int tid = threadIdx.x, b = blockIdx.x;
    const uint32_t flags = a.flags;
    const long long nchunks = a.n / SGP_CHUNK;
    SgpSignalPad* mypad = a.pads[a.rank];
    const SgpHyper hp = *a.hyper;
    const uint64_t pol_first = l2_evict_first_policy();

    // gradients of this rank were produced by earlier kernels on this stream
    if (tid == 0) {
        s_ok = 1;
        __threadfence_system();
        st_release_sys(&mypad->pub_seq[b], step + 1u);
    }
    __syncthreads();
    if (tid < a.world && tid != a.rank)
        if (!spin_wait_geq(&a.pads[tid]->pub_seq[b], step + 1u, st, a.timeout_ns,
                           SGP_ERR_TIMEOUT_PUB))
            s_ok = 0;
    __syncthreads();

    if (s_ok) {
        const float inv_world = hp.grad_scale / (float)a.world;
        for (long long c = b; c < nchunks; c += gridDim.x) {
            const long long base = chunk_base(c, tid);
            float4 acc[SGP_UNROLL];
#pragma unroll
            for (int u = 0; u < SGP_UNROLL; ++u) acc[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int r = 0; r < a.world; ++r) {
                float4 gv[SGP_UNROLL];
#pragma unroll
                for (int u = 0; u < SGP_UNROLL; ++u) {
                    const long long i = chunk_elem(base, u);
                    if (flags & SGP_F_GRAD_BF16) {
                        uint2 raw;
                        const uint2* p = reinterpret_cast<const uint2*>(
                            reinterpret_cast<const __nv_bfloat16*>(grad_peers[r]) + i);
                        asm volatile("ld.global.L1::no_allocate.v2.u32 {%0,%1}, [%2];"
                                     : "=r"(raw.x), "=r"(raw.y) : "l"(p));
                        gv[u] = bf16x4_to_f4(raw);
                    } else {
                        gv[u] = ld_stream_f4(reinterpret_cast<const float4*>(
                            reinterpret_cast<const float*>(grad_peers[r]) + i));
                    }
                }
#pragma unroll
                for (int u = 0; u < SGP_UNROLL; ++u) {
                    acc[u].x += gv[u].x; acc[u].y += gv[u].y;
                    acc[u].z += gv[u].z; acc[u].w += gv[u].w;
                }
            }
#pragma unroll
            for (int u = 0; u < SGP_UNROLL; ++u) {
                const long long i = chunk_elem(base, u);
                float4 xv = ld_once_f4(reinterpret_cast<const float4*>(a.z + i), pol_first);
                float4 mv = ld_once_f4(reinterpret_cast<const float4*>(a.m + i), pol_first);
                const float4 gv = mul4(acc[u], inv_world);
                sgd4<false>(xv, gv, mv, hyper_row(hp), 1.f);
                st_f4(reinterpret_cast<float4*>(a.m + i), mv);
                store_z(a, flags, i, xv);
            }
        }
    }

    __syncthreads();
    if (tid == 0 && cta_done_is_last(st)) {
        // tell every peer we are done with its gradients, then wait until every
        // peer is done with ours (the next backward overwrites them)
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

// after the all-reduce the caller's gradient buffer is cleared by this rank
__global__ void __launch_bounds__(SGP_THREADS)
sgp_zero_kernel(float4* p, long long n16)
{
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n16;
         i += (long long)gridDim.x * blockDim.x)
        p[i] = make_float4(0.f, 0.f, 0.f, 0.f);
}

// ---------------------------------------------------------------------------
// Device barrier across ranks (model.block())
// ---------------------------------------------------------------------------
__global__ void sgp_barrier_kernel(SgpSignalPad* const* pads, SgpState* st, int rank, int world,
                                   unsigned long long timeout_ns)
{
    const uint32_t epoch = st->bar_epoch + 1u;
    const int t = threadIdx.x;
    __threadfence_system();
    if (t < world) st_release_sys(&pads[t]->bar_seq[rank], epoch);   // tell everyone
    if (t < world)
        spin_wait_geq(&pads[rank]->bar_seq[t], epoch, st, timeout_ns, SGP_ERR_TIMEOUT_BAR);
    __syncthreads();
    if (t == 0) { st->bar_epoch = epoch; __threadfence(); }
}

// ---------------------------------------------------------------------------
// x *= s  or  x /= s  over a flat buffer (ps_numerator / unbias parity path)
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(SGP_THREADS)
sgp_scale_kernel(float* x, long long n, const float* scalar, int invert, __nv_bfloat16* shadow)
{
    const float s = invert ? (1.f / *scalar) : *scalar;
    const long long n4 = n / 4;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4;
         i += (long long)gridDim.x * blockDim.x) {
        float4 v = reinterpret_cast<float4*>(x)[i];
        v = mul4(v, s);
        reinterpret_cast<float4*>(x)[i] = v;
        if (shadow) reinterpret_cast<uint2*>(shadow)[i] = f4_to_bf16x4(v);
    }
}

// ---------------------------------------------------------------------------
// dst = scale * sum_k srcs[k]   over flat fp32 buffers that may live on PEER devices of the same
// process (single-process multi-GPU replicas): the reference's reduce_add_coalesced
// (gossip/distributed.py:523-549, N10) as one kernel of 16-byte P2P loads on the master GPU.
// ---------------------------------------------------------------------------
struct SgpPtrList { const float* p[SGP_MAX_RANKS]; int n; };

__global__ void __launch_bounds__(SGP_THREADS)
sgp_peer_reduce_kernel(float* __restrict__ dst, const SgpPtrList srcs, long long n4, float scale)
{
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4;
         i += (long long)gridDim.x * blockDim.x) {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int k = 0; k < srcs.n; ++k) {
            const float4 v = ld_stream_f4(reinterpret_cast<const float4*>(srcs.p[k]) + i);
            acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
        reinterpret_cast<float4*>(dst)[i] = mul4(acc, scale);
    }
}

// ---------------------------------------------------------------------------
// Consensus distance and push-sum average model (a collective of every rank; the launcher
// brackets each step with sgp_barrier_kernel):
//
//   barrier   nobody still reads an outbox
//   sgp_snapshot_kernel            outbox words [0, n) <- z (fp32), pad.snap_w <- w
//   barrier
//   sgp_consensus_kernel<FULL>     per element, over every rank's snapshot (TMA ring, items are
//                                  (chunk, rank) pairs, rank fastest, so each peer byte crosses
//                                  NVLink once): weighted running mean zbar and unweighted
//                                  Welford mean m / M2, then sum_j (z_j - zbar)^2 = M2 + n (m - zbar)^2
//                                  (one pass; sum z^2 - n zbar^2 would cancel catastrophically
//                                  exactly when the ranks agree).  Per-thread sums in fp64, CTA
//                                  and grid reductions in a fixed order; the last CTA stores the
//                                  rank's partials into its symmetric slot.
//                                  slice (FULL = false): rank r covers chunks [rC/n, (r+1)C/n)
//                                  full: every rank covers everything, writes zbar and its own
//                                  |z_r - zbar|^2
//   barrier
//   sgp_consensus_finalize_kernel  sum the ranks' slots in rank order -> result (identical bits
//                                  on every rank)
//   barrier   nobody still reads a snapshot / slot when the next step overwrites them
//
// zbar is accumulated as the weighted running mean zbar_j = zbar_{j-1} + (w_j / W_j)(z_j - zbar_{j-1})
// (W_j = w_0 + .. + w_j) rather than as (sum_j w_j z_j) / W: the same quantity up to fp32 rounding,
// but identical replicas give zbar == z exactly, whatever the weights, so their distance is 0.
// The snapshot never touches pub_seq / ack_seq / psw: the next gossip step publishes with the
// sequence numbers it would have used anyway.
// ---------------------------------------------------------------------------
#define SGP_CONS_SLOT   4      // doubles per rank: [sum_j (z_j - zbar)^2, |zbar|^2, |z_rank - zbar|^2, -]

__global__ void __launch_bounds__(SGP_THREADS)
sgp_snapshot_kernel(const SgpArgs a)
{
    float4* dst = reinterpret_cast<float4*>(a.outboxes[a.rank]);
    const float4* src = reinterpret_cast<const float4*>(a.z);
    const long long n4 = a.n / 4;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4;
         i += (long long)gridDim.x * blockDim.x)
        dst[i] = src[i];
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        const uint32_t step = *((volatile uint32_t*)&a.st->step);
        *((volatile float*)&a.pads[a.rank]->snap_w) = *((volatile float*)&a.st->ps_weight[step & 1u]);
    }
}

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    return v;
}

template <bool FULL>
__global__ void __launch_bounds__(SGP_THREADS, 2)
sgp_consensus_kernel(const SgpArgs a, double* const* partials, double* scratch, float* avg_out)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const TmaRing ring(smem_raw);
    __shared__ float  s_f[SGP_MAX_RANKS];              // w_j / W_j   (weighted running mean)
    __shared__ float  s_inv[SGP_MAX_RANKS];            // 1 / (j + 1) (Welford)
    __shared__ double s_red[3][SGP_THREADS / 32];
    __shared__ int    s_last;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int world = a.world;
    const long long nchunks = a.n / SGP_CHUNK;
    const long long lo = FULL ? 0 : nchunks * a.rank / world;
    const long long hi = FULL ? nchunks : nchunks * (a.rank + 1) / world;

    if (tid == 0) {
        running_mean_factors(a, s_f);
        for (int j = 0; j < world; ++j) s_inv[j] = 1.f / (float)(j + 1);
        ring.init();
    }
    __syncthreads();

    const long long items = cta_chunks(hi - lo, blockIdx.x) * world;     // (chunk, rank) pairs, rank fastest
    const auto src_of = [&](long long item) -> const float* {
        const long long it = item / world;
        const int j = (int)(item - it * world);
        const long long c = lo + blockIdx.x + it * gridDim.x;
        return a.outboxes[j] + c * SGP_CHUNK;
    };
    if (tid == 0) ring.fill(items, src_of);

    float4 zb[SGP_UNROLL], mu[SGP_UNROLL], m2[SGP_UNROLL], own[SGP_UNROLL];
    double acc_d = 0.0, acc_n = 0.0, acc_o = 0.0;
    const double nd = (double)world;
    for (long long item = 0; item < items; ++item) {
        const long long it = item / world;
        const int j = (int)(item - it * world);
        const float4* src = ring.wait(item);
        const float fj = s_f[j], ij = s_inv[j];
#pragma unroll
        for (int u = 0; u < SGP_UNROLL; ++u) {
            const float4 v = src[tid + u * SGP_THREADS];
            // (full mode needs no Welford terms: its distance is sum_r |z_r - zbar|^2, each rank
            // contributing its own term)
            if (j == 0) {
                zb[u] = v;
                if (!FULL) { mu[u] = v; m2[u] = make_float4(0.f, 0.f, 0.f, 0.f); }
            } else {
#define SGP_CONS_UPD(e)                                              \
                {                                                    \
                    zb[u].e = fmaf(fj, v.e - zb[u].e, zb[u].e);      \
                    if (!FULL) {                                     \
                        const float d = v.e - mu[u].e;               \
                        mu[u].e = fmaf(d, ij, mu[u].e);              \
                        m2[u].e = fmaf(d, v.e - mu[u].e, m2[u].e);   \
                    }                                                \
                }
                SGP_CONS_UPD(x) SGP_CONS_UPD(y) SGP_CONS_UPD(z) SGP_CONS_UPD(w)
#undef SGP_CONS_UPD
            }
            if (FULL && j == a.rank) own[u] = v;
        }
        if (j == world - 1) {
            const long long c = lo + blockIdx.x + it * gridDim.x;
#pragma unroll
            for (int u = 0; u < SGP_UNROLL; ++u) {
#define SGP_CONS_ACC(e)                                                                 \
                {                                                                       \
                    acc_n = fma((double)zb[u].e, (double)zb[u].e, acc_n);               \
                    if (FULL) {                                                         \
                        const double o = (double)own[u].e - (double)zb[u].e;            \
                        acc_o = fma(o, o, acc_o);                                       \
                    } else {                                                            \
                        const double dm = (double)mu[u].e - (double)zb[u].e;            \
                        acc_d += fma(nd * dm, dm, (double)m2[u].e);                     \
                    }                                                                   \
                }
                SGP_CONS_ACC(x) SGP_CONS_ACC(y) SGP_CONS_ACC(z) SGP_CONS_ACC(w)
#undef SGP_CONS_ACC
                if (FULL)
                    st_f4(reinterpret_cast<float4*>(avg_out + c * SGP_CHUNK) + tid + u * SGP_THREADS, zb[u]);
            }
        }
        ring.refill(item, items, src_of);
    }

    // CTA reduction in a fixed order (shuffle tree, then warps 0..7), then the grid: the last CTA
    // sums the CTA partials in CTA order
    acc_d = warp_sum_f64(acc_d);
    acc_n = warp_sum_f64(acc_n);
    acc_o = warp_sum_f64(acc_o);
    if (lane == 0) { s_red[0][warp] = acc_d; s_red[1][warp] = acc_n; s_red[2][warp] = acc_o; }
    __syncthreads();
    unsigned int* counter = reinterpret_cast<unsigned int*>(scratch + (size_t)SGP_MAX_CTAS * SGP_CONS_SLOT);
    if (tid == 0) {
        double t[3] = {0.0, 0.0, 0.0};
        for (int q = 0; q < 3; ++q)
            for (int w = 0; w < SGP_THREADS / 32; ++w) t[q] += s_red[q][w];
        double* mine = scratch + (size_t)blockIdx.x * SGP_CONS_SLOT;
        mine[0] = t[0]; mine[1] = t[1]; mine[2] = t[2];
        __threadfence();
        s_last = atomicAdd(counter, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (tid == 0 && s_last) {
        __threadfence();
        double t[3] = {0.0, 0.0, 0.0};
        for (unsigned int b = 0; b < gridDim.x; ++b)
            for (int q = 0; q < 3; ++q) t[q] += ((volatile double*)scratch)[(size_t)b * SGP_CONS_SLOT + q];
        volatile double* slot = partials[a.rank];
        slot[0] = t[0];
        slot[1] = t[1];
        slot[2] = t[2];
        *((volatile unsigned int*)counter) = 0u;
        __threadfence_system();
    }
}

// result[0] = distance_sq, result[1] = |zbar|^2, result[2 + r] = |z_r - zbar|^2 (full mode; 0 in
// slice mode).  Every rank sums the same slots in the same order.  NaN after a timed-out barrier.
__global__ void sgp_consensus_finalize_kernel(const SgpArgs a, double* const* partials, double* result, int full)
{
    if (threadIdx.x != 0) return;
    double d = 0.0, nrm = 0.0;
    for (int r = 0; r < a.world; ++r) {
        const volatile double* p = partials[r];
        const double own = p[2];
        d += full ? own : p[0];
        if (!full) nrm += p[1];
        result[2 + r] = full ? own : 0.0;
    }
    if (full) nrm = ((const volatile double*)partials[0])[1];
    const bool ok = *((volatile uint32_t*)&a.st->status) == SGP_OK;
    result[0] = ok ? d / (double)a.world : __longlong_as_double(0x7ff8000000000000ll);
    result[1] = ok ? nrm : __longlong_as_double(0x7ff8000000000000ll);
}

// ---------------------------------------------------------------------------
// SlowMo (slow momentum over periodic exact averaging; Wang et al., ICLR 2020), a collective of
// every rank bracketed by device barriers like the consensus collective:
//
//   barrier | sgp_snapshot_kernel | barrier | sgp_slowmo_kernel | barrier
//
// sgp_slowmo_kernel reads every rank's snapshot through the TMA ring of sgp_consensus_kernel
// ((chunk, rank) items, rank fastest; every rank covers every chunk) and forms zbar with the same
// weighted running mean, in the same rank order, so zbar -- and the update -- has the same bits
// on every rank.  Per element, with gamma = lr:
//
//   init:   x_prev <- zbar ; u <- 0 ; z <- zbar
//   else:   u <- beta u + (x_prev - zbar) / gamma ; x_new <- x_prev - alpha gamma u ;
//           x_prev <- x_new ; z <- x_new
//
// (plus the bf16 shadow of z), then both push-sum weight slots <- 1.  After a timed-out barrier
// (sticky status != OK) nothing is written: the host raises at poll().  pub_seq / ack_seq / psw
// and the step counter are not touched, so the next gossip step publishes as it would have; the
// closing barrier keeps that publish from overwriting a snapshot a slower rank still reads.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(SGP_THREADS, 2)
sgp_slowmo_kernel(const SgpArgs a, float* u, float* x_prev, float lr, float alpha, float beta, int init)
{
    if (*((volatile uint32_t*)&a.st->status) != SGP_OK) return;

    extern __shared__ __align__(128) unsigned char smem_raw[];
    const TmaRing ring(smem_raw);
    __shared__ float s_f[SGP_MAX_RANKS];              // w_j / W_j   (weighted running mean)

    const int tid = threadIdx.x;
    const int world = a.world;
    const long long nchunks = a.n / SGP_CHUNK;

    if (tid == 0) {
        running_mean_factors(a, s_f);
        ring.init();
        if (blockIdx.x == 0) {
            *((volatile float*)&a.st->ps_weight[0]) = 1.f;
            *((volatile float*)&a.st->ps_weight[1]) = 1.f;
        }
    }
    __syncthreads();

    const long long items = cta_chunks(nchunks, blockIdx.x) * world;     // (chunk, rank) pairs, rank fastest
    const auto src_of = [&](long long item) -> const float* {
        const long long it = item / world;
        const int j = (int)(item - it * world);
        const long long c = blockIdx.x + it * gridDim.x;
        return a.outboxes[j] + c * SGP_CHUNK;
    };
    if (tid == 0) ring.fill(items, src_of);

    const uint64_t pol_first = l2_evict_first_policy();
    const float alr = alpha * lr;
    float4 zb[SGP_UNROLL];
    for (long long item = 0; item < items; ++item) {
        const long long it = item / world;
        const int j = (int)(item - it * world);
        const float4* src = ring.wait(item);
        const float fj = s_f[j];
#pragma unroll
        for (int k = 0; k < SGP_UNROLL; ++k) {
            const float4 v = src[tid + k * SGP_THREADS];
            if (j == 0) {
                zb[k] = v;
            } else {
                zb[k].x = fmaf(fj, v.x - zb[k].x, zb[k].x);
                zb[k].y = fmaf(fj, v.y - zb[k].y, zb[k].y);
                zb[k].z = fmaf(fj, v.z - zb[k].z, zb[k].z);
                zb[k].w = fmaf(fj, v.w - zb[k].w, zb[k].w);
            }
        }
        ring.refill(item, items, src_of);
        if (j == world - 1) {
            const long long c = blockIdx.x + it * gridDim.x;
#pragma unroll
            for (int k = 0; k < SGP_UNROLL; ++k) {
                const long long i4 = c * (SGP_CHUNK / 4) + tid + k * SGP_THREADS;
                float4 xn = zb[k], un = make_float4(0.f, 0.f, 0.f, 0.f);
                if (!init) {
                    const float4 up = ld_once_f4(reinterpret_cast<const float4*>(u) + i4, pol_first);
                    const float4 xp = ld_once_f4(reinterpret_cast<const float4*>(x_prev) + i4, pol_first);
#define SGP_SLOWMO_UPD(e)                                                   \
                    un.e = fmaf(beta, up.e, __fdiv_rn(xp.e - zb[k].e, lr)); \
                    xn.e = fmaf(-alr, un.e, xp.e);
                    SGP_SLOWMO_UPD(x) SGP_SLOWMO_UPD(y) SGP_SLOWMO_UPD(z) SGP_SLOWMO_UPD(w)
#undef SGP_SLOWMO_UPD
                }
                st_hint_f4(reinterpret_cast<float4*>(u) + i4, un, pol_first);
                st_hint_f4(reinterpret_cast<float4*>(x_prev) + i4, xn, pol_first);
                st_f4(reinterpret_cast<float4*>(a.z) + i4, xn);
                if (a.shadow)
                    st_u2(reinterpret_cast<uint2*>(a.shadow) + i4, f4_to_bf16x4(xn));
            }
        }
    }
}

// ---------------------------------------------------------------------------
// LARS (SGP_F_LARS): per-tensor trust ratios, computed right before each SGD launch.
//
// sgp_lars_norms_kernel: grid-stride over the host-built tile table.  A tile is <= SGP_LARS_TILE
// elements of ONE tensor; the CTA reads its x = z * wmul and g^ = grad_scale * (g [+ g2]) exactly
// as phase 1 of the step kernels does (same fp32 operations), and writes the tile's sum x^2 and
// sum g^2 in fp64 to lars_partials[tile].  Each thread owns fixed elements of the tile, the warps
// reduce with a fixed shuffle tree and thread 0 adds the warps in order: no atomics, so the
// partials -- and the trust ratios -- are bit-identical from run to run and for any grid.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(SGP_THREADS)
sgp_lars_norms_kernel(const SgpArgs a)
{
    __shared__ double s_x[SGP_THREADS / 32], s_g[SGP_THREADS / 32];
    const SgpState* st = a.st;
    const uint32_t parity = *((volatile const uint32_t*)&st->step) & 1u;
    const float w0 = *((volatile const float*)&st->ps_weight[parity]);
    const float wmul = (a.flags & SGP_F_IN_NUMER) ? 1.f : w0;    // as phase 1
    const float gscale = a.hyper->grad_scale;
    const bool g_bf16 = (a.flags & SGP_F_GRAD_BF16) != 0;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    static_assert(SGP_LARS_TILE == SGP_THREADS * SGP_VEC * SGP_UNROLL, "one pass per tile");

    for (int t = blockIdx.x; t < a.lars_ntiles; t += gridDim.x) {
        const SgpLarsTile tile = a.lars_tiles[t];
        float4 xv[SGP_UNROLL], gv[SGP_UNROLL];
#pragma unroll
        for (int u = 0; u < SGP_UNROLL; ++u) {
            // tile.start is a multiple of 64 and j of 4, so every float4 is aligned and stays
            // inside the arena (lanes past tile.count are masked below)
            const int j = (u * SGP_THREADS + tid) * SGP_VEC;
            const long long i = tile.start + j;
            xv[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            gv[u] = xv[u];
            if (j < tile.count) {
                xv[u] = __ldg(reinterpret_cast<const float4*>(a.z + i));
                if (g_bf16)
                    gv[u] = bf16x4_to_f4(__ldg(reinterpret_cast<const uint2*>(
                                reinterpret_cast<const __nv_bfloat16*>(a.g) + i)));
                else
                    gv[u] = __ldg(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(a.g) + i));
                if (a.g2 != nullptr) {
                    const float4 h = __ldg(reinterpret_cast<const float4*>(a.g2 + i));
                    gv[u].x += h.x; gv[u].y += h.y; gv[u].z += h.z; gv[u].w += h.w;
                }
            }
        }
        double sx = 0.0, sg = 0.0;
#pragma unroll
        for (int u = 0; u < SGP_UNROLL; ++u) {
            const int j = (u * SGP_THREADS + tid) * SGP_VEC;
            const float4 x = mul4(xv[u], wmul), g = mul4(gv[u], gscale);
            const float xs[4] = {x.x, x.y, x.z, x.w}, gs[4] = {g.x, g.y, g.z, g.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                if (j + k < tile.count) {
                    sx = fma((double)xs[k], (double)xs[k], sx);
                    sg = fma((double)gs[k], (double)gs[k], sg);
                }
            }
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            sx += __shfl_down_sync(0xffffffffu, sx, off);
            sg += __shfl_down_sync(0xffffffffu, sg, off);
        }
        if (lane == 0) { s_x[warp] = sx; s_g[warp] = sg; }
        __syncthreads();
        if (tid == 0) {
            double tx = 0.0, tg = 0.0;
#pragma unroll
            for (int w = 0; w < SGP_THREADS / 32; ++w) { tx += s_x[w]; tg += s_g[w]; }
            a.lars_partials[2 * (long long)t] = tx;
            a.lars_partials[2 * (long long)t + 1] = tg;
        }
        __syncthreads();
    }
}

// sgp_lars_trust_kernel: one warp per tensor.  Lane l adds the tensor's tile partials l, l+32, ...
// in order and a fixed shuffle tree combines the lanes (deterministic); lane 0 writes the sums to
// lars_sumsq and the trust ratio
//     t = eta |x| / (|g^| + wd |x| + eps)   if LARS is on for the tensor and |x| > 0 and |g^| > 0,
//     t = 1                                 otherwise,
// in fp64, rounded once to fp32.  wd is the weight decay of the tensor's group, read from the
// device rows at every launch (so a change reaches a captured graph).
__global__ void __launch_bounds__(SGP_THREADS)
sgp_lars_trust_kernel(const SgpArgs a)
{
    const int t = (int)((blockIdx.x * (unsigned)SGP_THREADS + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (t >= a.lars_tensors) return;                  // (whole warps)
    const int k0 = a.lars_tile_first[t], k1 = a.lars_tile_first[t + 1];
    double sx = 0.0, sg = 0.0;
    for (int k = k0 + lane; k < k1; k += 32) {
        sx += a.lars_partials[2 * (long long)k];
        sg += a.lars_partials[2 * (long long)k + 1];
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        sx += __shfl_down_sync(0xffffffffu, sx, off);
        sg += __shfl_down_sync(0xffffffffu, sg, off);
    }
    if (lane == 0) {
        a.lars_sumsq[2 * t] = sx;
        a.lars_sumsq[2 * t + 1] = sg;
        float tr = 1.f;
        if (a.lars_enabled[t] != 0 && sx > 0.0 && sg > 0.0) {
            const double nx = sqrt(sx), ng = sqrt(sg);
            const int grp = a.block_group[a.lars_tiles[k0].start / SGP_GROUP_BLOCK];
            const double wd = (double)a.hyper_groups[grp].weight_decay;
            tr = (float)((double)a.lars_eta * nx / (ng + wd * nx + (double)a.lars_eps));
        }
        a.lars_trust[t] = tr;
    }
}

// ---------------------------------------------------------------------------
// launchers
// ---------------------------------------------------------------------------
// bf16 messages are implemented for the full synchronous step only
static bool msg_bf16_mode_ok(unsigned int flags)
{
    if (!(flags & SGP_F_MSG_BF16)) return true;
    const unsigned int full = SGP_F_PHASE1 | SGP_F_PUBLISH | SGP_F_PHASE2;
    const unsigned int partial = SGP_F_FOLD_RES | SGP_F_NO_ROTATE | SGP_F_KEEP_Z | SGP_F_SELF_FROM_Z |
                                 SGP_F_FROM_STATE;
    return (flags & full) == full && (flags & partial) == 0u;
}

// The instantiations of the two step kernels: MSG_BF16 is free, LARS needs GROUPS.  Whatever has
// to know every variant (launch, shared-memory opt-in, occupancy, preloading) goes through
// for_each_step_variant, so a new variant is one more line here.
template <bool MSG_BF16, bool GROUPS, bool LARS>
struct StepVariant {
    static constexpr auto step = &sgp_step_kernel<MSG_BF16, GROUPS, LARS>;
    static constexpr auto pipe = &sgp_step_pipe_kernel<MSG_BF16, GROUPS, LARS>;
    // (lars_ok: SGP_F_LARS only comes with SGP_F_GROUPS)
    static bool selected_by(unsigned int flags) {
        return MSG_BF16 == ((flags & SGP_F_MSG_BF16) != 0u) && LARS == ((flags & SGP_F_LARS) != 0u) &&
               GROUPS == ((flags & (SGP_F_GROUPS | SGP_F_LARS)) != 0u);
    }
};

template <class F>
static void for_each_step_variant(F&& f)
{
    f(StepVariant<false, false, false>{});
    f(StepVariant<true, false, false>{});
    f(StepVariant<false, true, false>{});
    f(StepVariant<true, true, false>{});
    f(StepVariant<false, true, true>{});
    f(StepVariant<true, true, true>{});
}

// f(variant) -> cudaError_t for the variant that `flags` selects
template <class F>
static cudaError_t with_step_variant(unsigned int flags, F&& f)
{
    cudaError_t e = cudaErrorInvalidValue;
    for_each_step_variant([&](auto v) { if (v.selected_by(flags)) e = f(v); });
    return e;
}

// Opt Kernel in to `bytes` of dynamic shared memory (and, with max_carveout, to the large
// shared-memory carve-out) on the current device.  The attribute belongs to the device's context
// and one process can drive several devices, so it is set once per kernel AND device.
template <auto Kernel>
static cudaError_t ensure_dynamic_smem(int bytes, bool max_carveout = false)
{
    static bool configured[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    const bool remember = dev >= 0 && dev < 64;
    if (remember && configured[dev]) return cudaSuccess;
    cudaError_t e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess && max_carveout)
        e = cudaFuncSetAttribute(Kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (e == cudaSuccess && remember) configured[dev] = true;
    return e;
}

// Co-resident CTAs of a step kernel: the minimum over its variants, because the ranks of a job
// share one grid whatever variant each of them launches.
// pipe: two CTAs x 64 KB per SM need the large shared-memory carve-out (the default one fits a
// single CTA).  The bf16 ring uses half of each stage but asks for the same PIPE_SMEM, so the
// occupancy stays that of the fp32 kernel
static int step_resident_ctas(int device, bool pipe)
{
    int sms = 0, per_sm = 1 << 30;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess) return 0;
    for_each_step_variant([&](auto v) {
        int n = 0;
        cudaError_t e = pipe ? ensure_dynamic_smem<v.pipe>(PIPE_SMEM, true) : cudaSuccess;
        if (e == cudaSuccess)
            e = pipe ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, v.pipe, PIPE_THREADS, PIPE_SMEM)
                     : cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, v.step, SGP_THREADS, 0);
        if (e != cudaSuccess) n = 0;
        if (n < per_sm) per_sm = n;
    });
    return sms * per_sm;
}

// grid of the flat grid-stride kernels over n_vec 16-byte accesses
static int flat_grid(long long n_vec)
{
    long long grid = (n_vec + SGP_THREADS - 1) / SGP_THREADS;
    if (grid > 132 * 8) grid = 132 * 8;
    if (grid < 1) grid = 1;
    return (int)grid;
}

// SGP_F_GROUPS needs the group table, the block map and 1..SGP_MAX_GROUPS groups
static bool groups_ok(const SgpArgs* args)
{
    if (!(args->flags & SGP_F_GROUPS)) return true;
    return args->hyper_groups && args->block_group && args->groups >= 1 && args->groups <= SGP_MAX_GROUPS;
}

// SGP_F_LARS needs SGP_F_GROUPS (the rows give each tensor's weight decay) and every LARS buffer
static bool lars_ok(const SgpArgs* args)
{
    if (!(args->flags & SGP_F_LARS)) return true;
    return (args->flags & SGP_F_GROUPS) && groups_ok(args) && args->block_tensor && args->lars_trust &&
           args->lars_enabled && args->lars_tiles && args->lars_tile_first && args->lars_partials &&
           args->lars_sumsq && args->lars_tensors >= 1 && args->lars_tensors <= SGP_LARS_MAX_TENSORS &&
           args->lars_ntiles >= args->lars_tensors;
}

extern "C" {

cudaError_t sgp_launch_step(const SgpArgs* args, int grid, cudaStream_t stream)
{
    if (!msg_bf16_mode_ok(args->flags) || !groups_ok(args) || !lars_ok(args)) return cudaErrorInvalidValue;
    return with_step_variant(args->flags, [&](auto v) {
        v.step<<<grid, SGP_THREADS, 0, stream>>>(*args);
        return cudaGetLastError();
    });
}

cudaError_t sgp_launch_step_pipe(const SgpArgs* args, int grid, cudaStream_t stream)
{
    if (!msg_bf16_mode_ok(args->flags) || !groups_ok(args) || !lars_ok(args)) return cudaErrorInvalidValue;
    return with_step_variant(args->flags, [&](auto v) {
        const cudaError_t e = ensure_dynamic_smem<v.pipe>(PIPE_SMEM, true);
        if (e != cudaSuccess) return e;
        v.pipe<<<grid, PIPE_THREADS, PIPE_SMEM, stream>>>(*args);
        return cudaGetLastError();
    });
}

int sgp_max_resident_ctas_pipe(int device) { return step_resident_ctas(device, true); }
int sgp_max_resident_ctas(int device) { return step_resident_ctas(device, false); }

// the two LARS kernels (see sgp_lars_norms_kernel): any grid >= 1 gives the same bits
cudaError_t sgp_launch_lars_norms(const SgpArgs* args, int grid, cudaStream_t stream)
{
    if (!lars_ok(args) || !(args->flags & SGP_F_LARS) || grid < 1) return cudaErrorInvalidValue;
    sgp_lars_norms_kernel<<<grid, SGP_THREADS, 0, stream>>>(*args);
    return cudaGetLastError();
}

cudaError_t sgp_launch_lars_trust(const SgpArgs* args, cudaStream_t stream)
{
    if (!lars_ok(args) || !(args->flags & SGP_F_LARS)) return cudaErrorInvalidValue;
    const int warps_per_cta = SGP_THREADS / 32;
    const int grid = (args->lars_tensors + warps_per_cta - 1) / warps_per_cta;
    sgp_lars_trust_kernel<<<grid, SGP_THREADS, 0, stream>>>(*args);
    return cudaGetLastError();
}

cudaError_t sgp_launch_gather(const SgpArgs* args, int grid, int pub_grid, cudaStream_t stream)
{
    if (args->flags & SGP_F_MSG_BF16) return cudaErrorInvalidValue;
    sgp_gather_kernel<<<grid, SGP_THREADS, 0, stream>>>(*args, pub_grid);
    return cudaGetLastError();
}

cudaError_t sgp_launch_gather_tma(const SgpArgs* args, int grid, int pub_grid, cudaStream_t stream)
{
    if (args->flags & SGP_F_MSG_BF16) return cudaErrorInvalidValue;
    const cudaError_t e = ensure_dynamic_smem<sgp_gather_tma_kernel>(SGP_RING_SMEM);
    if (e != cudaSuccess) return e;
    sgp_gather_tma_kernel<<<grid, SGP_THREADS, SGP_RING_SMEM, stream>>>(*args, pub_grid);
    return cudaGetLastError();
}

cudaError_t sgp_launch_probe(const SgpArgs* args, int pub_grid, uint32_t* host_flag,
                             cudaStream_t stream)
{
    sgp_probe_kernel<<<1, SGP_THREADS, 0, stream>>>(*args, pub_grid, host_flag);
    return cudaGetLastError();
}

cudaError_t sgp_launch_gather_wait(const SgpArgs* args, int pub_grid, cudaStream_t stream)
{
    sgp_gather_wait_kernel<<<1, SGP_THREADS, 0, stream>>>(*args, pub_grid);
    return cudaGetLastError();
}

cudaError_t sgp_launch_gather_ack(const SgpArgs* args, cudaStream_t stream)
{
    sgp_gather_ack_kernel<<<1, 1, 0, stream>>>(*args);
    return cudaGetLastError();
}

cudaError_t sgp_launch_bilat_decide(const SgpArgs* args, int pub_grid, int passive,
                                    unsigned long long max_wait_ns, uint32_t* host_fb, cudaStream_t stream)
{
    sgp_bilat_decide_kernel<<<1, SGP_THREADS, 0, stream>>>(*args, pub_grid, passive, max_wait_ns, host_fb);
    return cudaGetLastError();
}

cudaError_t sgp_launch_bilat_ctl(SgpState* st, int budget, int enabled, cudaStream_t stream)
{
    sgp_bilat_ctl_kernel<<<1, 1, 0, stream>>>(st, budget, enabled);
    return cudaGetLastError();
}

cudaError_t sgp_launch_allreduce_sgd(const SgpArgs* args, void* const* grad_peers, int grid,
                                     cudaStream_t stream)
{
    sgp_allreduce_sgd_kernel<<<grid, SGP_THREADS, 0, stream>>>(*args, grad_peers);
    return cudaGetLastError();
}

cudaError_t sgp_launch_peer_reduce(float* dst, const float* const* srcs, int nsrc, long long n, float scale,
                                   cudaStream_t stream)
{
    if (nsrc < 1 || nsrc > SGP_MAX_RANKS || (n & 3)) return cudaErrorInvalidValue;
    SgpPtrList l;
    l.n = nsrc;
    for (int k = 0; k < nsrc; ++k) l.p[k] = srcs[k];
    const long long n4 = n / 4;
    sgp_peer_reduce_kernel<<<flat_grid(n4), SGP_THREADS, 0, stream>>>(dst, l, n4, scale);
    return cudaGetLastError();
}

cudaError_t sgp_launch_zero(void* p, long long bytes, cudaStream_t stream)
{
    const long long n16 = bytes / 16;
    sgp_zero_kernel<<<flat_grid(n16), SGP_THREADS, 0, stream>>>(reinterpret_cast<float4*>(p), n16);
    return cudaGetLastError();
}

cudaError_t sgp_launch_barrier(SgpSignalPad* const* pads, SgpState* st, int rank, int world,
                               unsigned long long timeout_ns, cudaStream_t stream)
{
    sgp_barrier_kernel<<<1, SGP_MAX_RANKS, 0, stream>>>(pads, st, rank, world, timeout_ns);
    return cudaGetLastError();
}

cudaError_t sgp_launch_scale(float* x, long long n, const float* scalar, int invert,
                             __nv_bfloat16* shadow, cudaStream_t stream)
{
    sgp_scale_kernel<<<flat_grid(n / 4), SGP_THREADS, 0, stream>>>(x, n, scalar, invert, shadow);
    return cudaGetLastError();
}

cudaError_t sgp_launch_snapshot(const SgpArgs* args, cudaStream_t stream)
{
    if (!args->outboxes || (args->n & 3)) return cudaErrorInvalidValue;
    sgp_snapshot_kernel<<<flat_grid(args->n / 4), SGP_THREADS, 0, stream>>>(*args);
    return cudaGetLastError();
}

// scratch: SGP_MAX_CTAS * SGP_CONS_SLOT doubles of CTA partials + one zeroed 32-bit counter
cudaError_t sgp_launch_consensus(const SgpArgs* args, double* const* partials, double* scratch, float* avg_out,
                                 int full, int grid, cudaStream_t stream)
{
    if (!args->outboxes || grid < 1 || grid > SGP_MAX_CTAS || (full && !avg_out)) return cudaErrorInvalidValue;
    const cudaError_t e = full ? ensure_dynamic_smem<sgp_consensus_kernel<true>>(SGP_RING_SMEM)
                               : ensure_dynamic_smem<sgp_consensus_kernel<false>>(SGP_RING_SMEM);
    if (e != cudaSuccess) return e;
    if (full)
        sgp_consensus_kernel<true><<<grid, SGP_THREADS, SGP_RING_SMEM, stream>>>(*args, partials, scratch, avg_out);
    else
        sgp_consensus_kernel<false><<<grid, SGP_THREADS, SGP_RING_SMEM, stream>>>(*args, partials, scratch, avg_out);
    return cudaGetLastError();
}

cudaError_t sgp_launch_consensus_finalize(const SgpArgs* args, double* const* partials, double* result, int full,
                                          cudaStream_t stream)
{
    sgp_consensus_finalize_kernel<<<1, 32, 0, stream>>>(*args, partials, result, full);
    return cudaGetLastError();
}

cudaError_t sgp_launch_slowmo(const SgpArgs* args, float* u, float* x_prev, float lr, float alpha, float beta,
                              int init, int grid, cudaStream_t stream)
{
    if (!args->outboxes || !u || !x_prev || grid < 1 || grid > SGP_MAX_CTAS) return cudaErrorInvalidValue;
    const cudaError_t e = ensure_dynamic_smem<sgp_slowmo_kernel>(SGP_RING_SMEM);
    if (e != cudaSuccess) return e;
    sgp_slowmo_kernel<<<grid, SGP_THREADS, SGP_RING_SMEM, stream>>>(*args, u, x_prev, lr, alpha, beta, init);
    return cudaGetLastError();
}

// Load every gossip kernel into the current device's context now.  Under lazy module loading a
// kernel is loaded at its first launch, and loading can wait for the whole device.  A process that
// drives several ranks (one GPU each, or virtual ranks sharing one GPU) would then wait for one
// rank's spinning gossip kernel whose in-neighbour's publish it has not launched yet.
cudaError_t sgp_preload_kernels()
{
    cudaError_t e = cudaSuccess;
    const auto load = [&](const void* kernel) {
        cudaFuncAttributes attr;
        if (e == cudaSuccess) e = cudaFuncGetAttributes(&attr, kernel);
    };
    for_each_step_variant([&](auto v) { load((const void*)v.step); load((const void*)v.pipe); });
    const void* kernels[] = {
        (const void*)sgp_gather_kernel, (const void*)sgp_gather_tma_kernel,
        (const void*)sgp_lars_norms_kernel, (const void*)sgp_lars_trust_kernel,
        (const void*)sgp_probe_kernel, (const void*)sgp_gather_wait_kernel,
        (const void*)sgp_gather_ack_kernel, (const void*)sgp_bilat_decide_kernel, (const void*)sgp_bilat_ctl_kernel,
        (const void*)sgp_allreduce_sgd_kernel, (const void*)sgp_zero_kernel, (const void*)sgp_barrier_kernel,
        (const void*)sgp_scale_kernel, (const void*)sgp_peer_reduce_kernel, (const void*)sgp_snapshot_kernel,
        (const void*)sgp_consensus_kernel<false>, (const void*)sgp_consensus_kernel<true>,
        (const void*)sgp_consensus_finalize_kernel, (const void*)sgp_slowmo_kernel};
    for (const void* k : kernels) load(k);
    return e;
}

}  // extern "C"
