// 1x1 convolution (NHWC) as a wgmma GEMM with the BatchNorm statistics (forward) or the
// skip-branch gradient accumulation (backward) fused into the epilogue -- sm_90a (Hopper).
//
//   Y[M, N] = X[M, K] . W[N, K]^T        M = batch*H*W, K = C_in, N = C_out, bf16 in / fp32 acc
//
// In a bottleneck ResNet two of the three convolutions of every block are 1x1 and
// every one of them feeds a training-mode BatchNorm, whose first pass re-reads the
// whole activation just to get per-channel mean / variance.  At batch 256 these
// GEMMs are HBM-bound (K is 64..2048 and M is up to 802,816), so the kernel is
// organised around the epilogue, not the MMA:
//
//   warp 8     TMA producer   X tiles -> 128B-swizzled smem ring (cp.async.bulk.tensor, mbarrier
//                             complete_tx).  The CTA's W block [BN, K] is loaded ONCE and stays
//                             resident whenever it fits next to a >= 3-deep X ring (K*BN <= 64K
//                             elements); otherwise W tiles travel through the ring with X.
//   warps 0-7  two warpgroups, each: wgmma.mma_async m64 x BN x 16 (bf16) / x 8 (tf32) on rows
//                             [64g, 64g+64) of the 128-row tile, fp32 accumulators in registers,
//                             then the epilogue.  Each warp owns the 16 tile rows its accumulator
//                             fragment holds end to end: registers -> bf16 -> its own 2 KB
//                             swizzled slab -> its own TMA store (box 64 x 16), then the
//                             statistics of exactly those rows are read back from the slab (lane =
//                             channel pair): n / shifted sum / shifted sum of squares of the
//                             ROUNDED outputs (what BatchNorm will read).  No CTA-wide barrier in
//                             the loop; slabs recycle through the issuing lane's bulk-group counter.
//
// The grid is persistent: CTA (nb, j) owns output-channel block nb for its whole life
// and walks the row tiles j, j + ctas_per_n, ...; its statistics therefore stay in
// registers until the end: each warp keeps (n, K, sum(y-K), sum((y-K)^2)) with its
// own shift K (its first output row), the eight warps are merged in shared memory into one
// (n, mean, M2) row per CTA, and c1_stats_finalize_kernel merges the rows (one per CTA, at most
// one per SM) with the pairwise (Chan) update and emits mean / invstd / scale / shift and the
// running-statistics update, exactly what bn_stats_finalize_kernel does for the stand-alone
// statistics pass.
//
// Three epilogue modes share the producer / MMA pipeline:
//   MODE 0  Y = X.W^T
//   MODE 1  + the BatchNorm statistics above (forward of conv + BN: no separate statistics pass)
//   MODE 2  Y = X.W^T + R, R's 2 KB slab prefetched by TMA one sub-tile ahead (own mbarrier per
//           slab), summed in fp32 before the single bf16 rounding.  Used as the dgrad of the first
//           convolution of a residual block with R = the skip-branch gradient, which replaces
//           autograd's read-read-write accumulation pass over the block's widest tensor.
//   MODE 3  MODE 2 + the backward reduction of the BatchNorm (+ residual + ReLU) that produced this
//           dgrad's input X' in the previous block:  dz = mask ? X.W^T + R : 0 is stored, and per
//           channel sum(dz) and sum(dz * (x' - mean) * invstd) are accumulated, x' being the BN's
//           input (a second TMA slab stream shaped like R), mean / invstd from its coefficients and
//           mask its 1-bit ReLU mask [M, N/8] (plain loads).  The statistics are read back from the
//           stored (rounded) slab like MODE 1's and merged into partial[ctas_per_n][2][N], the layout
//           bn_bwd_finalize_kernel consumes; the stand-alone reduce pass over dy / x' / out is gone.
//
// Timing: benchmarks/conv1x1_bench.py.
//
// Reference call site: torchvision Bottleneck conv1/conv3 + BatchNorm2d in the reference
// gossip_sgd.py (models.resnet50()).

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

namespace {

constexpr int BM = 128;                 // rows per tile: two warpgroups x wgmma M = 64
constexpr int ROW_BYTES = 128;          // one k-block row == one 128-byte swizzle row: 64 bf16 or 32 fp32
constexpr int A_BYTES = BM * ROW_BYTES; // 16 KB
constexpr int SLAB_BYTES = 16 * 128;    // one warp's store slab: 16 rows x 128 B (64 bf16 / 32 fp32), 2 KB
// Element-type dependent tile geometry.  F32 = fp32 activations / weights multiplied on the tensor
// cores as TF32 (wgmma .tf32 reads fp32 words from shared memory and uses their top 19
// bits: the same arithmetic as the reference's cuDNN TF32 convolutions), fp32 accumulate, fp32 out.
template <bool F32> struct Elt {
    static constexpr int BYTES = F32 ? 4 : 2;
    static constexpr int BK = ROW_BYTES / BYTES;      // elements per k-block: 32 / 64
    static constexpr int MMA_K = 32 / BYTES;          // 8 (tf32) / 16 (bf16): 32 bytes of K per instruction
    static constexpr int COLS = ROW_BYTES / BYTES;    // output columns per store slab: 32 / 64
};
constexpr int kMmaWarps = 8;            // two warpgroups: MMA + epilogue
constexpr int kThreads = kMmaWarps * 32 + 32;   // + the producer warp
constexpr int MAX_STAGES = 8;
constexpr int SMEM_LIMIT = 227 * 1024;  // opt-in dynamic shared memory per CTA on sm_90
constexpr int SMEM_FIXED = 1024 + 512;  // alignment slack + barriers

// cute::TMA::CacheHintSm90 encodings
constexpr uint64_t L2_EVICT_NORMAL = 0x1000000000000000ull;
constexpr uint64_t L2_EVICT_FIRST = 0x12F0000000000000ull;
constexpr uint64_t L2_EVICT_LAST = 0x14F0000000000000ull;

// ---------------------------------------------------------------------------
// PTX helpers
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ bool mbar_try(uint64_t* bar, uint32_t parity)
{
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// A protocol bug must not hang the GPU: after ~2 s of spinning the kernel traps.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity)
{
    if (mbar_try(bar, parity)) return;
    unsigned long long t0 = 0;
    for (uint32_t spins = 1;; ++spins) {
        if (mbar_try(bar, parity)) return;
        if ((spins & 0xFFFu) == 0) {
            unsigned long long now;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
            if (t0 == 0) t0 = now;
            else if (now - t0 > 2000000000ull) __trap();
        }
    }
}

__device__ __forceinline__ void tma_load_2d(const CUtensorMap* tm, uint64_t* bar, void* dst, int c0, int c1,
                                            uint64_t hint)
{
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
        " [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(smem_u32(dst)),
        "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(hint)
        : "memory");
}
__device__ __forceinline__ void tma_load_2d_s(const CUtensorMap* tm, uint32_t bar_smem, uint32_t dst_smem, int c0,
                                              int c1, uint64_t hint)
{
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
        " [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(dst_smem),
        "l"(reinterpret_cast<uint64_t>(tm)), "r"(bar_smem), "r"(c0), "r"(c1), "l"(hint)
        : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* tm, uint32_t src_smem, int c0, int c1)
{
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                     reinterpret_cast<uint64_t>(tm)),
                 "r"(src_smem), "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* tm)
{
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tm)) : "memory");
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait()
{
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across wgmma issue and wait
template <int R> __device__ __forceinline__ void fence_operands(float (&d)[R])
{
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// K-major operand tile, rows of 128 B (64 bf16 / 32 fp32) in the TMA 128B-swizzle layout, 8-row
// groups 1024 B apart.  (cute::GMMA::GmmaDescriptor: start>>4 [0,14), LBO>>4 [16,30) (unused for a
// swizzled K-major operand), SBO>>4 [32,46), layout SWIZZLE_128B = 1 at [62,64).)
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr)
{
    return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}

// D[64 x N] (+)= A[64 x K-step] . B[N x K-step]^T, both operands K-major in shared memory, fp32
// accumulators in registers; issued by one warpgroup.  bf16: k16 per instruction; tf32: k8.
__device__ __forceinline__ void wgmma_bf16(float (&d)[32], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
        " %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31},"
        " %32, %33, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_bf16(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
        " %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
        " %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47,"
        " %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63},"
        " %64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_bf16(float (&d)[128], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
        " %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
        " %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47,"
        " %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63,"
        " %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79,"
        " %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95,"
        " %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111,"
        " %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127},"
        " %128, %129, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
          "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
          "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
          "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
          "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
          "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
          "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
          "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
          "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_tf32(float (&d)[32], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
        " %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31},"
        " %32, %33, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
        " %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
        " %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47,"
        " %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63},"
        " %64, %65, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_tf32(float (&d)[128], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
        " %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
        " %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47,"
        " %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63,"
        " %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79,"
        " %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95,"
        " %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111,"
        " %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127},"
        " %128, %129, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
          "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
          "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
          "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
          "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
          "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
          "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
          "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
          "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}

__device__ __forceinline__ uint32_t pack_bf16(uint32_t lo_f32, uint32_t hi_f32)
{
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(__uint_as_float(hi_f32)), "f"(__uint_as_float(lo_f32)));
    return r;
}

// ---------------------------------------------------------------------------
// the GEMM
// ---------------------------------------------------------------------------
struct C1Plan {            // host-computed shared-memory plan (bytes are multiples of 1024)
    int stages;            // depth of the X (or X+W) ring, 2..MAX_STAGES
    int resident;          // 1: this CTA's whole W block [BN, K] is loaded once and stays in smem
    int nbuf;              // store slabs per epilogue warp (2 or 1)
    int x_hint_first;      // 1: X tiles are read by one CTA only -> L2 evict_first
};

// MODES 4 / 5 (c1_gemm_eval_kernel): eval-mode BatchNorm of the live parameters and running statistics,
// Y = act(acc * s[c] + t[c] (+ R)) with s = gamma * rsqrt(running_var + eps), t = beta - running_mean * s
struct C1Eval {
    const float* gamma;
    const float* beta;
    const float* mean;
    const float* var;
    float eps;
    int relu;
};

// MODE 0: Y = X.W^T          MODE 1: + BatchNorm statistics of Y          MODE 2: Y = X.W^T + R
// MODE 3: dz = mask ? X.W^T + R : 0, + BatchNorm backward reduction against bn_x (tm_b), coef, mask
// MODE 4: Y = act(X.W^T * s + t)                                           MODE 5: Y = act(X.W^T * s + t + R)
// (one body for all kernels; ev is read by MODES 4 / 5 only)
// DROP (MODE 3, stochastic depth): the previous block's BN output was scaled by sdrop[row / hw] before the
// residual add, so the reduction is that of sdrop[row / hw] * dz; dz itself is stored unscaled
template <int BN, int MODE, bool F32, bool DROP = false>
__device__ __forceinline__ void
c1_gemm_body(const CUtensorMap& tm_x, const CUtensorMap& tm_w, const CUtensorMap& tm_y, const CUtensorMap& tm_r,
             const CUtensorMap& tm_b, int M, int N, int K, float* __restrict__ partial,
             const float* __restrict__ coef, const uint8_t* __restrict__ mask, const C1Plan& plan, const C1Eval& ev,
             const float* __restrict__ sdrop = nullptr, int hw = 1)
{
    constexpr bool STATS = MODE == 1;
    constexpr bool RES = MODE == 2 || MODE == 3 || MODE == 5;
    constexpr bool BNR = MODE == 3;
    constexpr bool EVAL = MODE >= 4;
    constexpr int BK = Elt<F32>::BK;
    constexpr int MMA_K = Elt<F32>::MMA_K;
    constexpr int COLS = Elt<F32>::COLS;
    constexpr int B_BYTES = BN * ROW_BYTES;
    constexpr int NS = BN / COLS;             // store-slab wide sub-tiles per tile (64 bf16 / 32 fp32 columns)
    constexpr int G8 = COLS / 8;              // 8-column accumulator groups per sub-tile
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));

    const int warp = threadIdx.x >> 5;        // warp-uniform
    const int lane = threadIdx.x & 31;
    const int n_blocks = N / BN;
    const int ctas_per_n = gridDim.x / n_blocks;
    const int nb = blockIdx.x % n_blocks;
    const int j = blockIdx.x / n_blocks;
    const int m_tiles = (M + BM - 1) / BM;
    const int k_blocks = (K + BK - 1) / BK;
    const int stages = plan.stages;
    const bool resident = plan.resident != 0;
    const int nbuf = plan.nbuf;

    // [ resident W : k_blocks x B_BYTES ][ ring : stages x (X tile [+ W tile]) ][ store slabs ]
    // [ MODE 3: bn_x slabs, 8 warps x 2 | MODES 4 / 5: (s, t) of the BN columns ][ barriers ]
    uint8_t* sW = smem;
    uint8_t* ring = sW + (resident ? k_blocks * B_BYTES : 0);
    const int stage_bytes = A_BYTES + (resident ? 0 : B_BYTES);
    uint8_t* sO = ring + stages * stage_bytes;
    uint8_t* sB = sO + 8 * nbuf * SLAB_BYTES;
    uint64_t* full = reinterpret_cast<uint64_t*>(sB + (BNR ? 16 * SLAB_BYTES : 0) + (EVAL ? BN * 8 : 0));
    uint64_t* empty = full + MAX_STAGES;
    uint64_t* wfull = empty + MAX_STAGES;    // resident W landed
    uint64_t* rbar0 = wfull + 1;             // MODE 2: residual slab landed, [8 warps][2 slots]

    if (warp == kMmaWarps && lane == 0) {
        tma_prefetch_desc(&tm_x);
        tma_prefetch_desc(&tm_w);
        tma_prefetch_desc(&tm_y);
        for (int i = 0; i < stages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], kMmaWarps); }
        mbar_init(wfull, 1);
        if (RES) { tma_prefetch_desc(&tm_r); for (int i = 0; i < 16; ++i) mbar_init(&rbar0[i], 1); }
        if (BNR) tma_prefetch_desc(&tm_b);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (EVAL) {
        // the CTA's channel block never changes: (s, t) once per launch, from the live tensors
        float2* st = reinterpret_cast<float2*>(sB);
        for (int c = (int)threadIdx.x; c < BN; c += kThreads) {
            const int ch = nb * BN + c;
            const float sc = __ldg(ev.gamma + ch) * rsqrtf(__ldg(ev.var + ch) + ev.eps);
            st[c] = make_float2(sc, fmaf(-__ldg(ev.mean + ch), sc, __ldg(ev.beta + ch)));
        }
    }
    __syncthreads();

    if (warp == kMmaWarps) {
        // ===================== TMA producer =====================
        if (lane == 0) {
            if (resident) {
                mbar_expect_tx(wfull, (uint32_t)(k_blocks * B_BYTES));
                for (int kb = 0; kb < k_blocks; ++kb)
                    tma_load_2d(&tm_w, wfull, sW + kb * B_BYTES, kb * BK, nb * BN, L2_EVICT_LAST);
            }
            const uint64_t x_hint = plan.x_hint_first ? L2_EVICT_FIRST : L2_EVICT_NORMAL;
            int stage = 0;
            uint32_t phase = 0;
            for (int mt = j; mt < m_tiles; mt += ctas_per_n) {
                for (int kb = 0; kb < k_blocks; ++kb) {
                    mbar_wait(&empty[stage], phase ^ 1);
                    mbar_expect_tx(&full[stage], (uint32_t)stage_bytes);
                    uint8_t* dst = ring + stage * stage_bytes;
                    tma_load_2d(&tm_x, &full[stage], dst, kb * BK, mt * BM, x_hint);
                    if (!resident) tma_load_2d(&tm_w, &full[stage], dst + A_BYTES, kb * BK, nb * BN, L2_EVICT_LAST);
                    if (++stage == stages) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        // ===================== MMA + epilogue =====================
        // Warpgroup g multiplies rows [64g, 64g+64) of every tile with the whole W block.  In the
        // accumulator layout of wgmma warp q of the group holds rows [16q, 16q+16) of that half:
        // d[4c + i] is row lane/4 + 8*(i/2), column 8c + 2*(lane%4) + i%2.  Each warp then carries
        // its 16 rows end to end: registers -> bf16 -> its own 2 KB swizzled slab -> its own TMA
        // store (box 64 x 16) -> statistics of exactly those rows read back from the slab.  No
        // CTA-wide barrier in the loop; slabs recycle through the issuing lane's bulk-group counter.
        // While a tile drains, the producer keeps the ring filling with the next tile's X.
        const int g = warp >> 2;
        const int e = warp;                                                // 0..7: this warp's 16 rows
        const int row0 = 64 * g + 16 * (warp & 3);                         // first tile row of this warp
        const uint32_t slab0 = smem_u32(sO) + (uint32_t)(e * nbuf * SLAB_BYTES);
        const uint32_t rd_off = (uint32_t)((lane & 3) * 4);                // this lane's bf16 pair in a row
        const int rd_chunk = lane >> 2;
        const int r0 = lane >> 2;                                          // accumulator rows r0, r0 + 8
        const uint32_t wr_off = (uint32_t)(r0 * 128);
        float acc[BN / 2];
        int slot = 0;
        float cnt = 0.f;
        float k0[NS], k1[NS], s0[NS], s1[NS], q0[NS], q1[NS];
#pragma unroll
        for (int s = 0; s < NS; ++s) { k0[s] = k1[s] = s0[s] = s1[s] = q0[s] = q1[s] = 0.f; }
        bool have_k = false;
        int stage = 0;
        uint32_t phase = 0;
        // MODE 2: the residual slab of sub-tile i+1 is fetched (TMA, own mbarrier per slab) while
        // sub-tile i is converted; the sum is formed in fp32 in place and stored from the same slab.
        const uint32_t rbar = smem_u32(rbar0 + e * 2);
        uint32_t rphase = 0;                                     // bit b: parity of slab b's barrier
        const int tile_step = ctas_per_n;
        // MODE 3: the bn_x slab of the same rows / columns lands on the residual slab's barrier
        const uint32_t bslab0 = smem_u32(sB) + (uint32_t)(e * 2 * SLAB_BYTES);
        constexpr uint32_t R_TX = (BNR ? 2 : 1) * SLAB_BYTES;
        if (RES && lane == 0) {
            const int mt0 = j;
            if (mt0 < m_tiles && M - mt0 * BM - row0 > 0) {
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(rbar), "r"(R_TX)
                             : "memory");
                tma_load_2d_s(&tm_r, rbar, slab0, nb * BN, mt0 * BM + row0, L2_EVICT_FIRST);
                if (BNR) tma_load_2d_s(&tm_b, rbar, bslab0, nb * BN, mt0 * BM + row0, L2_EVICT_FIRST);
            }
        }
        if (resident) mbar_wait(wfull, 0);
        for (int mt = j; mt < m_tiles; mt += tile_step) {
            // ---- MMA: one commit group per k-block; a stage is released once its group retired ----
            int prev = -1;
            for (int kb = 0; kb < k_blocks; ++kb) {
                mbar_wait(&full[stage], phase);
                const uint8_t* a_ptr = ring + stage * stage_bytes;
                const uint8_t* b_ptr = resident ? sW + kb * B_BYTES : a_ptr + A_BYTES;
                const uint64_t a_desc = gmma_desc_sw128(smem_u32(a_ptr + g * (A_BYTES / 2)));
                const uint64_t b_desc = gmma_desc_sw128(smem_u32(b_ptr));
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < BK / MMA_K; ++k) {     // +32 B per MMA_K inside the swizzle row
                    if (F32) wgmma_tf32(acc, a_desc + (uint64_t)(k * 2), b_desc + (uint64_t)(k * 2),
                                        (uint32_t)((kb | k) != 0));
                    else wgmma_bf16(acc, a_desc + (uint64_t)(k * 2), b_desc + (uint64_t)(k * 2),
                                    (uint32_t)((kb | k) != 0));
                }
                wgmma_commit();
                wgmma_wait<1>();
                if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty[prev]); }
                prev = stage;
                if (++stage == stages) { stage = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
            fence_operands(acc);
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[prev]);

            // ---- epilogue ----
            const int nrows = min(16, M - mt * BM - row0);         // rows of this slab that exist (<= 0: none)
            float srow = 1.f;                                      // DROP: lane l < 16 holds row l's scale
            if (DROP && nrows > 0) {
                const int gr = mt * BM + row0 + (lane & 15);
                srow = gr < M ? __ldg(sdrop + gr / hw) : 0.f;
            }
#pragma unroll
            for (int s = 0; s < NS; ++s) {
                const uint32_t slab = slab0 + (uint32_t)(slot * SLAB_BYTES);
                if (!RES) {
                    if (lane == 0) {                               // the store that last used this slab has read it
                        if (nbuf == 2) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
                        else asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                    }
                    __syncwarp();
                }
                // MODE 3: this lane's mask bits of rows r0 and r0 + 8, one byte per 8-column group c:
                // bit 2*(lane%4) + i%2 of byte c is element d[4c + i].  Issued before the slab wait.
                uint32_t mk[2][2] = {{0u, 0u}, {0u, 0u}};     // [row r0 / r0 + 8][bytes 0-3 / 4-7]
                if (BNR && nrows > 0) {
                    const size_t pitch = (size_t)(N / 8);
                    const uint8_t* mp = mask + (size_t)(mt * BM + row0 + r0) * pitch + (nb * BN + s * COLS) / 8;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        if (r0 + 8 * h < nrows) {
                            if (F32) {
                                mk[h][0] = __ldg(reinterpret_cast<const unsigned int*>(mp + 8 * h * pitch));
                            } else {
                                const uint2 v = __ldg(reinterpret_cast<const uint2*>(mp + 8 * h * pitch));
                                mk[h][0] = v.x; mk[h][1] = v.y;
                            }
                        }
                    }
                }
                if (RES && nrows > 0) {
                    const uint32_t bar = rbar + (uint32_t)(slot * 8);
                    const uint32_t par = (rphase >> slot) & 1u;
                    while (true) {
                        uint32_t ok;
                        asm volatile(
                            "{\n\t.reg .pred p;\n\t"
                            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                            "selp.u32 %0, 1, 0, p;\n\t}"
                            : "=r"(ok) : "r"(bar), "r"(par) : "memory");
                        if (ok) break;
                    }
                    rphase ^= 1u << slot;
                }
                if (!RES || nrows > 0) {
#pragma unroll
                    for (int c = 0; c < G8; ++c) {
                        const float* d = acc + 4 * (s * G8 + c);
                        // 16-byte chunk of the 128-byte row and byte offset in it; rows r0 and r0 + 8
                        // share the swizzle phase (row & 7), so the second address is + 1024
                        const uint32_t chunk = F32 ? (uint32_t)(2 * c + ((lane & 3) >> 1)) : (uint32_t)c;
                        const uint32_t addr = slab + wr_off + ((chunk ^ (uint32_t)(r0 & 7)) << 4) +
                                              (F32 ? (uint32_t)((lane & 1) * 8) : rd_off);
                        // MODE 3 keep bits of d[0..3] (c is a compile-time index)
                        const uint32_t msh = (uint32_t)(8 * (c & 3) + 2 * (lane & 3));
                        const uint32_t mlo = mk[0][c >> 2] >> msh, mhi = mk[1][c >> 2] >> msh;
                        float4 st = make_float4(0.f, 0.f, 0.f, 0.f);   // MODES 4 / 5: (s, t) of both columns
                        if (EVAL)
                            st = *reinterpret_cast<const float4*>(sB + 8 * (s * COLS + 8 * c + 2 * (lane & 3)));
                        if (F32) {
                            float v0 = d[0], v1 = d[1], v2 = d[2], v3 = d[3];
                            if (EVAL) {
                                v0 = fmaf(v0, st.x, st.y); v1 = fmaf(v1, st.z, st.w);
                                v2 = fmaf(v2, st.x, st.y); v3 = fmaf(v3, st.z, st.w);
                            }
                            if (RES) {
                                float a0, a1, a2, a3;
                                asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(a0), "=f"(a1) : "r"(addr) : "memory");
                                asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(a2), "=f"(a3) : "r"(addr + 1024u)
                                             : "memory");
                                v0 += a0; v1 += a1; v2 += a2; v3 += a3;
                            }
                            if (EVAL && ev.relu) {                 // (a NaN stays NaN, as in torch.relu)
                                v0 = v0 < 0.f ? 0.f : v0; v1 = v1 < 0.f ? 0.f : v1;
                                v2 = v2 < 0.f ? 0.f : v2; v3 = v3 < 0.f ? 0.f : v3;
                            }
                            if (BNR) {
                                v0 = (mlo & 1u) ? v0 : 0.f; v1 = (mlo & 2u) ? v1 : 0.f;
                                v2 = (mhi & 1u) ? v2 : 0.f; v3 = (mhi & 2u) ? v3 : 0.f;
                            }
                            asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(v0), "f"(v1) : "memory");
                            asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr + 1024u), "f"(v2), "f"(v3)
                                         : "memory");
                        } else {
                            float v0 = d[0], v1 = d[1], v2 = d[2], v3 = d[3];
                            if (EVAL) {
                                v0 = fmaf(v0, st.x, st.y); v1 = fmaf(v1, st.z, st.w);
                                v2 = fmaf(v2, st.x, st.y); v3 = fmaf(v3, st.z, st.w);
                            }
                            if (RES) {
                                uint32_t a, b;
                                asm volatile("ld.shared.b32 %0, [%1];" : "=r"(a) : "r"(addr) : "memory");
                                asm volatile("ld.shared.b32 %0, [%1];" : "=r"(b) : "r"(addr + 1024u) : "memory");
                                v0 += __uint_as_float(a << 16); v1 += __uint_as_float(a & 0xFFFF0000u);
                                v2 += __uint_as_float(b << 16); v3 += __uint_as_float(b & 0xFFFF0000u);
                            }
                            if (EVAL && ev.relu) {
                                v0 = v0 < 0.f ? 0.f : v0; v1 = v1 < 0.f ? 0.f : v1;
                                v2 = v2 < 0.f ? 0.f : v2; v3 = v3 < 0.f ? 0.f : v3;
                            }
                            if (BNR) {
                                v0 = (mlo & 1u) ? v0 : 0.f; v1 = (mlo & 2u) ? v1 : 0.f;
                                v2 = (mhi & 1u) ? v2 : 0.f; v3 = (mhi & 2u) ? v3 : 0.f;
                            }
                            asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr),
                                         "r"(pack_bf16(__float_as_uint(v0), __float_as_uint(v1))) : "memory");
                            asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr + 1024u),
                                         "r"(pack_bf16(__float_as_uint(v2), __float_as_uint(v3))) : "memory");
                        }
                    }
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic writes -> TMA reads
                __syncwarp();
                if (lane == 0) {
                    if (nrows > 0) tma_store_2d(&tm_y, slab, nb * BN + s * COLS, mt * BM + row0);
                    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                    if (RES) {                                     // fetch the next residual slab
                        const int nmt = (s + 1 < NS) ? mt : mt + tile_step;
                        const int ns = (s + 1 < NS) ? s + 1 : 0;
                        if (nmt < m_tiles && M - nmt * BM - row0 > 0) {
                            asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");   // other slab is free
                            const uint32_t nbar = rbar + (uint32_t)((slot ^ 1) * 8);
                            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(nbar),
                                         "r"(R_TX)
                                         : "memory");
                            tma_load_2d_s(&tm_r, nbar, slab0 + (uint32_t)((slot ^ 1) * SLAB_BYTES), nb * BN + ns * COLS,
                                          nmt * BM + row0, L2_EVICT_FIRST);
                            // (its previous contents were read back by every lane before the __syncwarp above)
                            if (BNR)
                                tma_load_2d_s(&tm_b, nbar, bslab0 + (uint32_t)((slot ^ 1) * SLAB_BYTES),
                                              nb * BN + ns * COLS, nmt * BM + row0, L2_EVICT_FIRST);
                        }
                    }
                }
                if (BNR && nrows > 0) {
                    // lane = channel (fp32) / channel pair (bf16), as in MODE 1: dz from the stored slab,
                    // x' from the bn_x slab at the same swizzled offset
                    const uint32_t rd = slab + rd_off;
                    const uint32_t rb = bslab0 + (uint32_t)(slot * SLAB_BYTES) + rd_off;
                    const int ch = nb * BN + s * COLS + (F32 ? lane : 2 * lane);
                    const float mu0 = __ldg(coef + ch), is0 = __ldg(coef + N + ch);
                    const float mu1 = F32 ? 0.f : __ldg(coef + ch + 1), is1 = F32 ? 0.f : __ldg(coef + N + ch + 1);
                    auto acc_row = [&](int r) {
                        const uint32_t o = (uint32_t)(r * 128 + ((rd_chunk ^ (r & 7)) << 4));
                        uint32_t u, b;
                        asm volatile("ld.shared.b32 %0, [%1];" : "=r"(u) : "r"(rd + o));
                        asm volatile("ld.shared.b32 %0, [%1];" : "=r"(b) : "r"(rb + o));
                        const float sr = DROP ? __shfl_sync(0xffffffffu, srow, r) : 1.f;
                        float g0 = F32 ? __uint_as_float(u) : __uint_as_float(u << 16);
                        if (DROP) g0 *= sr;
                        const float x0 = F32 ? __uint_as_float(b) : __uint_as_float(b << 16);
                        s0[s] += g0; q0[s] = fmaf(g0, (x0 - mu0) * is0, q0[s]);
                        if (!F32) {
                            float g1 = __uint_as_float(u & 0xFFFF0000u);
                            if (DROP) g1 *= sr;
                            const float x1 = __uint_as_float(b & 0xFFFF0000u);
                            s1[s] += g1; q1[s] = fmaf(g1, (x1 - mu1) * is1, q1[s]);
                        }
                    };
                    if (nrows == 16) {
#pragma unroll
                        for (int r = 0; r < 16; ++r) acc_row(r);
                    } else {
                        for (int r = 0; r < nrows; ++r) acc_row(r);
                    }
                }
                if (STATS && nrows > 0) {
                    const uint32_t rd = slab + rd_off;
                    if (!have_k) {
                        uint32_t u;
                        asm volatile("ld.shared.b32 %0, [%1];" : "=r"(u) : "r"(rd + (uint32_t)(rd_chunk << 4)));
                        k0[s] = F32 ? __uint_as_float(u) : __uint_as_float(u << 16);
                        k1[s] = __uint_as_float(u & 0xFFFF0000u);
                    }
                    if (nrows == 16) {
#pragma unroll
                        for (int r8 = 0; r8 < 16; r8 += 8) {
                            uint32_t u[8];
#pragma unroll
                            for (int i = 0; i < 8; ++i)
                                asm volatile("ld.shared.b32 %0, [%1];" : "=r"(u[i])
                                             : "r"(rd + (uint32_t)((r8 + i) * 128 + ((rd_chunk ^ i) << 4))));
#pragma unroll
                            for (int i = 0; i < 8; ++i) {
                                const float d0 = (F32 ? __uint_as_float(u[i]) : __uint_as_float(u[i] << 16)) - k0[s];
                                s0[s] += d0; q0[s] = fmaf(d0, d0, q0[s]);
                                if (!F32) {          // fp32: one channel per lane; bf16: a channel pair
                                    const float d1 = __uint_as_float(u[i] & 0xFFFF0000u) - k1[s];
                                    s1[s] += d1; q1[s] = fmaf(d1, d1, q1[s]);
                                }
                            }
                        }
                    } else {
                        for (int r = 0; r < nrows; ++r) {
                            uint32_t u;
                            asm volatile("ld.shared.b32 %0, [%1];" : "=r"(u)
                                         : "r"(rd + (uint32_t)(r * 128 + ((rd_chunk ^ (r & 7)) << 4))));
                            const float d0 = (F32 ? __uint_as_float(u) : __uint_as_float(u << 16)) - k0[s];
                            s0[s] += d0; q0[s] = fmaf(d0, d0, q0[s]);
                            if (!F32) {
                                const float d1 = __uint_as_float(u & 0xFFFF0000u) - k1[s];
                                s1[s] += d1; q1[s] = fmaf(d1, d1, q1[s]);
                            }
                        }
                    }
                }
                slot = (slot + 1) & (nbuf - 1);      // nbuf is 1 or 2
            }
            if (nrows > 0) { cnt += (float)nrows; have_k = true; }
        }
        if (STATS) {
            // Merge the eight warps' partials (each with its own shift) into ONE row per CTA,
            // partial[j][field][N] with fields = n, mean, M2 (Chan et al.), so the finalize kernel
            // reads one row per CTA.  Every X load has landed and been consumed, so the ring is
            // free to serve as scratch.
            asm volatile("bar.sync 1, %0;" ::"n"(kMmaWarps * 32) : "memory");
            float4* sc = reinterpret_cast<float4*>(ring);
#pragma unroll
            for (int s = 0; s < NS; ++s) {
                if (F32) {
                    sc[e * BN + s * COLS + lane] = make_float4(cnt, k0[s], s0[s], q0[s]);
                } else {
                    sc[e * BN + s * COLS + 2 * lane] = make_float4(cnt, k0[s], s0[s], q0[s]);
                    sc[e * BN + s * COLS + 2 * lane + 1] = make_float4(cnt, k1[s], s1[s], q1[s]);
                }
            }
            asm volatile("bar.sync 1, %0;" ::"n"(kMmaWarps * 32) : "memory");
            const int t = (int)threadIdx.x;
            if (t < BN) {
                float n_tot = 0.f, m_sum = 0.f;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const float4 v = sc[i * BN + t];
                    n_tot += v.x;
                    m_sum += fmaf(v.x, v.y, v.z);                  // n*K + sum(y-K)
                }
                const float mu = n_tot > 0.f ? m_sum / n_tot : 0.f;
                float m2 = 0.f;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const float4 v = sc[i * BN + t];
                    if (v.x > 0.f) {
                        const float ds = v.z / v.x;                // mean_i - K_i
                        const float d = v.y + ds - mu;
                        m2 += fmaxf(fmaf(-v.z, ds, v.w), 0.f) + v.x * d * d;
                    }
                }
                float* p = partial + (size_t)j * 3 * N + nb * BN + t;
                p[0] = n_tot;
                p[N] = mu;
                p[2 * (size_t)N] = m2;
            }
        }
        if (BNR) {
            // the eight warps' (sum dz, sum dz*xhat) merged into partial[j][2][N] (ring as scratch, as above)
            asm volatile("bar.sync 1, %0;" ::"n"(kMmaWarps * 32) : "memory");
            float2* sc = reinterpret_cast<float2*>(ring);
#pragma unroll
            for (int s = 0; s < NS; ++s) {
                if (F32) {
                    sc[e * BN + s * COLS + lane] = make_float2(s0[s], q0[s]);
                } else {
                    sc[e * BN + s * COLS + 2 * lane] = make_float2(s0[s], q0[s]);
                    sc[e * BN + s * COLS + 2 * lane + 1] = make_float2(s1[s], q1[s]);
                }
            }
            asm volatile("bar.sync 1, %0;" ::"n"(kMmaWarps * 32) : "memory");
            const int t = (int)threadIdx.x;
            if (t < BN) {
                float a = 0.f, b = 0.f;
#pragma unroll
                for (int i = 0; i < 8; ++i) { const float2 v = sc[i * BN + t]; a += v.x; b += v.y; }
                float* p = partial + (size_t)j * 2 * N + nb * BN + t;
                p[0] = a;
                p[N] = b;
            }
        }
        if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    }
}

template <int BN, int MODE, bool F32>
__global__ void __launch_bounds__(kThreads, 1)
c1_gemm_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_w,
               const __grid_constant__ CUtensorMap tm_y, const __grid_constant__ CUtensorMap tm_r,
               const __grid_constant__ CUtensorMap tm_b, int M, int N, int K, float* __restrict__ partial,
               const float* __restrict__ coef, const uint8_t* __restrict__ mask, const C1Plan plan)
{
    static_assert(MODE >= 0 && MODE <= 3, "MODES 4 / 5 are c1_gemm_eval_kernel");
    c1_gemm_body<BN, MODE, F32>(tm_x, tm_w, tm_y, tm_r, tm_b, M, N, K, partial, coef, mask, plan, C1Eval{});
}

// MODE 3 with the stochastic-depth scale sdrop[row / hw] of the BatchNorm being reduced
template <int BN, bool F32>
__global__ void __launch_bounds__(kThreads, 1)
c1_gemm_drop_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_w,
                    const __grid_constant__ CUtensorMap tm_y, const __grid_constant__ CUtensorMap tm_r,
                    const __grid_constant__ CUtensorMap tm_b, int M, int N, int K, float* __restrict__ partial,
                    const float* __restrict__ coef, const uint8_t* __restrict__ mask, const C1Plan plan,
                    const float* __restrict__ sdrop, int hw)
{
    c1_gemm_body<BN, 3, F32, true>(tm_x, tm_w, tm_y, tm_r, tm_b, M, N, K, partial, coef, mask, plan, C1Eval{},
                                   sdrop, hw);
}

// MODE 4 (no residual) / MODE 5 (+ R through tm_r, as MODE 2): the eval-mode conv + BatchNorm (+ R) (+ ReLU)
template <int BN, int MODE, bool F32>
__global__ void __launch_bounds__(kThreads, 1)
c1_gemm_eval_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_w,
                    const __grid_constant__ CUtensorMap tm_y, const __grid_constant__ CUtensorMap tm_r, int M, int N,
                    int K, const C1Plan plan, const C1Eval ev)
{
    static_assert(MODE == 4 || MODE == 5, "eval modes only");
    c1_gemm_body<BN, MODE, F32>(tm_x, tm_w, tm_y, tm_r, tm_r, M, N, K, nullptr, nullptr, nullptr, plan, ev);
}

// ---------------------------------------------------------------------------
// statistics finalize: merge the R per-CTA rows (n, mean, M2) per channel (Chan et al.),
// then the same outputs as bn_stats_finalize_kernel (accumulate mode included: acc != nullptr adds
// mu / the unbiased variance to acc in fp64 and leaves the running buffers and nbt alone).
// 1024 threads = 32 row lanes x 32 channels.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(1024, 1)
c1_stats_finalize_kernel(const float* __restrict__ partial, int R, int C, const float* __restrict__ gamma,
                         const float* __restrict__ beta, float* running_mean, float* running_var, long long* nbt,
                         double* acc, float momentum, float eps, float* __restrict__ mean,
                         float* __restrict__ invstd, float* __restrict__ scale, float* __restrict__ shift)
{
    __shared__ float sm_a[32][33];
    __shared__ float sm_b[32][33];
    __shared__ float sm_mu[32];
    const int cl = threadIdx.x & 31;
    const int lane = threadIdx.x >> 5;
    const int ch = blockIdx.x * 32 + cl;
    const bool live = ch < C;
    if (blockIdx.x == 0 && threadIdx.x == 0 && nbt != nullptr && acc == nullptr) *nbt += 1;

    // every row of this lane is loaded up front (R <= 160 -> at most 5 rows per lane per batch), so
    // the kernel pays one L2 round trip instead of one per row
    constexpr int ILP = 5;
    float n_sum = 0.f, m_sum = 0.f;
    float nv[ILP], mv[ILP], qv[ILP];
#pragma unroll
    for (int u = 0; u < ILP; ++u) {
        const int r = lane + 32 * u;
        const bool ok = live && r < R;
        const int at = r * 3 * C + ch;                 // R * 3 * C < 2^20: 32-bit indexing
        nv[u] = ok ? partial[at] : 0.f;
        mv[u] = ok ? partial[at + C] : 0.f;
        qv[u] = ok ? partial[at + 2 * C] : 0.f;
        n_sum += nv[u];
        m_sum = fmaf(nv[u], mv[u], m_sum);
    }
    if (live)
        for (int r = lane + 32 * ILP; r < R; r += 32) {            // (only on parts with > 160 SMs)
            const float* p = partial + (size_t)r * 3 * C + ch;
            n_sum += p[0];
            m_sum = fmaf(p[0], p[C], m_sum);
        }
    sm_a[lane][cl] = n_sum;
    sm_b[lane][cl] = m_sum;
    __syncthreads();
    if (lane == 0) {
        float n = 0.f, m = 0.f;
#pragma unroll 4
        for (int l = 0; l < 32; ++l) { n += sm_a[l][cl]; m += sm_b[l][cl]; }
        sm_mu[cl] = (n > 0.f) ? m / n : 0.f;
        sm_a[0][cl] = n;
    }
    __syncthreads();
    const float mu = sm_mu[cl];
    const float n_tot = sm_a[0][cl];
    __syncthreads();

    // M2 = sum_p [ M2_p + n_p (mean_p - mu)^2 ]
    float m2 = 0.f;
#pragma unroll
    for (int u = 0; u < ILP; ++u) {
        const float d = mv[u] - mu;
        m2 += qv[u] + nv[u] * d * d;
    }
    if (live)
        for (int r = lane + 32 * ILP; r < R; r += 32) {
            const float* p = partial + (size_t)r * 3 * C + ch;
            const float d = p[C] - mu;
            m2 += p[2 * (size_t)C] + p[0] * d * d;
        }
    sm_b[lane][cl] = m2;
    __syncthreads();
    if (lane != 0 || !live) return;
    float tot = 0.f;
#pragma unroll 4
    for (int l = 0; l < 32; ++l) tot += sm_b[l][cl];
    const float var = (n_tot > 0.f) ? tot / n_tot : 0.f;
    const float is = rsqrtf(var + eps);
    mean[ch] = mu;
    invstd[ch] = is;
    const float sc = gamma[ch] * is;
    scale[ch] = sc;
    shift[ch] = fmaf(-mu, sc, beta[ch]);
    const float unbiased = (n_tot > 1.f) ? var * (n_tot / (n_tot - 1.f)) : var;
    if (acc != nullptr) {
        acc[ch] += (double)mu;
        acc[C + ch] += (double)unbiased;
    } else if (running_mean != nullptr) {
        running_mean[ch] = fmaf(momentum, mu - running_mean[ch], running_mean[ch]);
        running_var[ch] = fmaf(momentum, unbiased - running_var[ch], running_var[ch]);
    }
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn()
{
    static EncodeTiledFn fn = nullptr;
    if (fn == nullptr) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

// row-major [rows, cols] bf16 / fp32 matrix, box = [box_rows, 128 bytes of columns], 128B swizzle.  wide_promotion:
// let L2 fetch 256 B per request -- right for operand tiles whose rows are consumed whole, wrong
// for the 128 B-per-row output / residual slabs (ncu: +21 % DRAM reads on the residual stream).
bool make_map(CUtensorMap* tm, const void* base, long long rows, int cols, int box_rows, bool wide_promotion,
              bool f32)
{
    EncodeTiledFn fn = encode_fn();
    if (fn == nullptr) return false;
    const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)cols * (f32 ? 4 : 2)};
    const cuuint32_t box[2] = {f32 ? 32u : 64u, (cuuint32_t)box_rows};     // 128 bytes wide
    const cuuint32_t estr[2] = {1u, 1u};
    return fn(tm, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2,
              const_cast<void*>(base), dims, strides, box, estr,
              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
              wide_promotion ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B : CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Tile width: the widest BLOCK_N dividing N unless a narrower one shortens the critical path
// (waves of row tiles per CTA x BLOCK_N) by more than 10 % -- that only happens when M is small.
bool c1_f32_prefer_resident()
{
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("SGP_B200_C1_F32_RESIDENT");
        v = e ? atoi(e) : 1;
    }
    return v != 0;
}

int bn_override()        // SGP_B200_C1_BN=64|128|256 forces a tile width (benchmarking)
{
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("SGP_B200_C1_BN");
        v = e ? atoi(e) : 0;
    }
    return v;
}

// can the CTA's whole W block stay resident next to a >= 3-deep X ring and one slab per epilogue warp?
bool fits_resident(int bn, int K, bool f32)
{
    const int bk = f32 ? Elt<true>::BK : Elt<false>::BK;
    const int k_blocks = (K + bk - 1) / bk;
    return SMEM_LIMIT - SMEM_FIXED - 8 * SLAB_BYTES - k_blocks * bn * ROW_BYTES >= 3 * A_BYTES;
}

// MODE 3 (bn_reduce) runs at most 128 wide: at 256 its 128 accumulators per thread plus the reduction
// state exceed the 168 registers a 288-thread CTA gets, and the kernel spills.
int pick_bn(long long M, int N, int K, int num_sms, bool f32, bool bn_reduce)
{
    const long long m_tiles = (M + BM - 1) / BM;
    int best = 0;
    long long best_cost = 0;
    const int cap = bn_reduce ? 128 : 256;
    const int force = bn_override();
    if (force >= 64 && force <= cap && N % force == 0) return force;
    // fp32 operands are twice as wide: prefer the widest tile whose W block stays resident (a
    // non-resident 256-wide tile re-streams 3x the bytes of X per row tile through L2)
    int bn_max = cap;
    if (f32 && c1_f32_prefer_resident())
        for (int bn = cap; bn >= 128; bn >>= 1)      // (a 64-wide tile re-reads X once per 64 channels)
            if (N % bn == 0 && fits_resident(bn, K, true)) { bn_max = bn; break; }
    for (int bn = bn_max; bn >= 64; bn >>= 1) {
        if (N % bn) continue;
        long long per = num_sms / (N / bn);
        if (per < 1) per = 1;
        const long long cost = ((m_tiles + per - 1) / per) * bn;
        if (best == 0 || cost * 10 < best_cost * 9) { best = bn; best_cost = cost; }
    }
    return best;
}

void grid_shape(long long M, int N, int K, int num_sms, bool f32, bool bn_reduce, int& bn, int& ctas_per_n,
                int& grid)
{
    bn = pick_bn(M, N, K, num_sms, f32, bn_reduce);
    const int n_blocks = N / bn;
    const long long m_tiles = (M + BM - 1) / BM;
    long long per = num_sms / n_blocks;
    if (per < 1) per = 1;
    if (per > m_tiles) per = m_tiles;
    ctas_per_n = (int)per;
    grid = n_blocks * ctas_per_n;
}

// Shared-memory plan.  W stays resident when the CTA's [BN, K] block plus a >= 3-deep X ring
// fits (then every row tile costs one 16 KB X load instead of X + W); the store slabs shrink
// from 2 to 1 per warp if that is what makes it fit.  MODE 3 adds 8 x 2 bn_x slabs, MODES 4 / 5 (eval_bn)
// the BN x 8 bytes of (s, t).
C1Plan make_plan(int bn, int K, int n_blocks, bool residual, bool bn_reduce, bool f32, int& smem_bytes,
                 bool eval_bn = false)
{
    const int bk = f32 ? Elt<true>::BK : Elt<false>::BK;
    const int k_blocks = (K + bk - 1) / bk;
    const int b_bytes = bn * ROW_BYTES;
    const int extra = bn_reduce ? 16 * SLAB_BYTES : eval_bn ? bn * 8 : 0;
    residual = residual || bn_reduce;
    C1Plan p;
    p.x_hint_first = n_blocks == 1;
    p.resident = 0;
    p.nbuf = 2;
    for (int nbuf = 2; nbuf >= (residual ? 2 : 1) && !p.resident; --nbuf) {   // MODE 2/3 double-buffer their slabs
        const int ring = SMEM_LIMIT - SMEM_FIXED - extra - 8 * nbuf * SLAB_BYTES - k_blocks * b_bytes;
        if (ring >= 3 * A_BYTES) { p.resident = 1; p.nbuf = nbuf; }
    }
    const int stage_bytes = A_BYTES + (p.resident ? 0 : b_bytes);
    const int ring = SMEM_LIMIT - SMEM_FIXED - extra - 8 * p.nbuf * SLAB_BYTES - (p.resident ? k_blocks * b_bytes : 0);
    p.stages = ring / stage_bytes;
    if (p.stages > MAX_STAGES) p.stages = MAX_STAGES;
    smem_bytes = SMEM_FIXED + (p.resident ? k_blocks * b_bytes : 0) + p.stages * stage_bytes +
                 8 * p.nbuf * SLAB_BYTES + extra;
    return p;
}

template <int BN, bool F32>
cudaError_t launch(const CUtensorMap& tx, const CUtensorMap& tw, const CUtensorMap& ty, const CUtensorMap& tr,
                   const CUtensorMap& tb, int M, int N, int K, float* partial, const float* coef,
                   const uint8_t* mask, int mode, int grid, cudaStream_t st, const float* sdrop, int hw)
{
    constexpr int M3 = BN <= 128 ? 3 : 0;           // (no 256-wide MODE 3: see pick_bn)
    if (mode == 3 && M3 != 3) return cudaErrorInvalidValue;
    const bool drop = sdrop != nullptr;             // (MODE 3 only)
    auto kern = mode == 1 ? c1_gemm_kernel<BN, 1, F32>
              : mode == 2 ? c1_gemm_kernel<BN, 2, F32>
              : mode == 3 ? c1_gemm_kernel<BN, M3, F32> : c1_gemm_kernel<BN, 0, F32>;
    auto dkern = c1_gemm_drop_kernel<BN <= 128 ? BN : 128, F32>;
    const int slot = drop ? 4 : mode;
    static bool configured[5][64] = {};            // function attributes are per device (and per instantiation)
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64 || !configured[slot][dev]) {
        cudaError_t e = drop ? cudaFuncSetAttribute(dkern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT)
                             : cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT);
        if (e != cudaSuccess) return e;
        if (dev >= 0 && dev < 64) configured[slot][dev] = true;
    }
    int smem = 0;
    const C1Plan plan = make_plan(BN, K, N / BN, mode == 2, mode == 3, F32, smem);
    if (plan.stages < 2) return cudaErrorInvalidValue;
    if (drop) dkern<<<grid, kThreads, smem, st>>>(tx, tw, ty, tr, tb, M, N, K, partial, coef, mask, plan, sdrop, hw);
    else kern<<<grid, kThreads, smem, st>>>(tx, tw, ty, tr, tb, M, N, K, partial, coef, mask, plan);
    return cudaGetLastError();
}

template <int BN, bool F32>
cudaError_t launch_eval(const CUtensorMap& tx, const CUtensorMap& tw, const CUtensorMap& ty, const CUtensorMap& tr,
                        int M, int N, int K, bool residual, const C1Eval& ev, int grid, cudaStream_t st)
{
    auto kern = residual ? c1_gemm_eval_kernel<BN, 5, F32> : c1_gemm_eval_kernel<BN, 4, F32>;
    static bool configured[2][64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64 || !configured[residual][dev]) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT);
        if (e != cudaSuccess) return e;
        if (dev >= 0 && dev < 64) configured[residual][dev] = true;
    }
    int smem = 0;
    const C1Plan plan = make_plan(BN, K, N / BN, residual, false, F32, smem, true);
    if (plan.stages < 2) return cudaErrorInvalidValue;
    kern<<<grid, kThreads, smem, st>>>(tx, tw, ty, tr, M, N, K, plan, ev);
    return cudaGetLastError();
}

}  // namespace

extern "C" {

// shapes the kernel covers: 16-byte row pitch (K % 8 == 0 for bf16, K % 4 == 0 for fp32), N % 64 == 0,
// M < 2^31
int c1_supported(long long M, int N, int K, int f32)
{
    const int kq = f32 ? 4 : 8;
    return M >= 1 && M < (1ll << 31) && N >= 64 && N % 64 == 0 && K >= 8 && K % kq == 0;
}

// launch plan for a shape (host logic only; exercised by the CPU tests):
// out = {BLOCK_N, grid, ctas_per_n, stages, resident, nbuf, dynamic smem bytes}
void c1_describe_plan(long long M, int N, int K, int num_sms, int residual, int bn_reduce, int f32, int* out)
{
    int bn, per, grid, smem = 0;
    grid_shape(M, N, K, num_sms, f32 != 0, bn_reduce != 0, bn, per, grid);
    const C1Plan p = make_plan(bn, K, N / bn, residual != 0, bn_reduce != 0, f32 != 0, smem);
    out[0] = bn; out[1] = grid; out[2] = per; out[3] = p.stages; out[4] = p.resident; out[5] = p.nbuf;
    out[6] = smem;
}

// number of partial-statistics rows c1_launch_gemm writes for this shape (bn_reduce: in MODE 3)
int c1_partial_rows(long long M, int N, int K, int num_sms, int bn_reduce, int f32)
{
    int bn, per, grid;
    grid_shape(M, N, K, num_sms, f32 != 0, bn_reduce != 0, bn, per, grid);
    return per;              // one merged partial row per CTA
}

// y[M,N] = x[M,K] . w[N,K]^T [+ residual[M,N]]; all operands bf16 (f32 == 0) or all fp32 with TF32
// tensor-core math (f32 != 0); partial (nullable) = [c1_partial_rows][3][N] fp32 statistics of y.
// partial and residual are mutually exclusive, except in MODE 3 (mask != nullptr): then residual,
// bn_x ([M, N], y's dtype), coef (mean [N], invstd [N]) and mask ([M, N/8] bytes) are all given,
// y = dz and partial = [c1_partial_rows][2][N] (sum dz, sum dz * xhat).
static cudaError_t gemm(const void* x, const void* w, void* y, long long M, int N, int K, float* partial,
                        const void* residual, const void* bn_x, const float* coef, const uint8_t* mask,
                        int num_sms, int f32, cudaStream_t st, const float* sdrop, int hw)
{
    if (!c1_supported(M, N, K, f32)) return cudaErrorInvalidValue;
    if (mask ? !(partial && residual && bn_x && coef) : (partial && residual)) return cudaErrorInvalidValue;
    const int mode = mask ? 3 : partial ? 1 : (residual ? 2 : 0);
    const bool f = f32 != 0;
    int bn, per, grid;
    grid_shape(M, N, K, num_sms, f, mode == 3, bn, per, grid);
    CUtensorMap tx, tw, ty, tr, tb;
    if (!make_map(&tx, x, M, K, BM, true, f) || !make_map(&tw, w, N, K, bn, true, f) ||
        !make_map(&ty, y, M, N, 16, false, f) || !make_map(&tr, residual ? residual : y, M, N, 16, false, f) ||
        !make_map(&tb, bn_x ? bn_x : y, M, N, 16, false, f))
        return cudaErrorInvalidValue;
    if (f) {
        switch (bn) {
        case 256: return launch<256, true>(tx, tw, ty, tr, tb, (int)M, N, K, partial, coef, mask, mode, grid, st, sdrop, hw);
        case 128: return launch<128, true>(tx, tw, ty, tr, tb, (int)M, N, K, partial, coef, mask, mode, grid, st, sdrop, hw);
        default: return launch<64, true>(tx, tw, ty, tr, tb, (int)M, N, K, partial, coef, mask, mode, grid, st, sdrop, hw);
        }
    }
    switch (bn) {
    case 256: return launch<256, false>(tx, tw, ty, tr, tb, (int)M, N, K, partial, coef, mask, mode, grid, st, sdrop, hw);
    case 128: return launch<128, false>(tx, tw, ty, tr, tb, (int)M, N, K, partial, coef, mask, mode, grid, st, sdrop, hw);
    default: return launch<64, false>(tx, tw, ty, tr, tb, (int)M, N, K, partial, coef, mask, mode, grid, st, sdrop, hw);
    }
}

cudaError_t c1_launch_gemm(const void* x, const void* w, void* y, long long M, int N, int K, float* partial,
                           const void* residual, const void* bn_x, const float* coef, const uint8_t* mask,
                           int num_sms, int f32, cudaStream_t st)
{
    return gemm(x, w, y, M, N, K, partial, residual, bn_x, coef, mask, num_sms, f32, st, nullptr, 1);
}

// stochastic depth: c1_launch_gemm in MODE 3 (all of partial, residual, bn_x, coef, mask given) for a BatchNorm
// whose output was scaled by sdrop[row / hw] (fp32 [M / hw]) before the residual add: dz is stored as there,
// partial holds (sum sdrop * dz, sum sdrop * dz * xhat)
cudaError_t c1_launch_gemm_bn_reduce_drop(const void* x, const void* w, void* y, long long M, int N, int K,
                                          float* partial, const void* residual, const void* bn_x, const float* coef,
                                          const uint8_t* mask, const float* sdrop, int hw, int num_sms, int f32,
                                          cudaStream_t st)
{
    if (!mask || !sdrop || hw < 1 || M % hw != 0) return cudaErrorInvalidValue;
    return gemm(x, w, y, M, N, K, partial, residual, bn_x, coef, mask, num_sms, f32, st, sdrop, hw);
}

// eval-mode conv + BatchNorm: y = act(x . w^T * s + t [+ residual]), s = gamma * rsqrt(var + eps),
// t = beta - mean * s per output channel, computed by each CTA from the live fp32 [N] tensors at every
// launch (a captured graph follows in-place parameter swaps).  Same plan and grid as MODE 0 / MODE 2.
cudaError_t c1_launch_gemm_bn_eval(const void* x, const void* w, void* y, long long M, int N, int K,
                                   const void* residual, const float* gamma, const float* beta, const float* mean,
                                   const float* var, float eps, int relu, int num_sms, int f32, cudaStream_t st)
{
    if (!c1_supported(M, N, K, f32)) return cudaErrorInvalidValue;
    const bool f = f32 != 0;
    int bn, per, grid;
    grid_shape(M, N, K, num_sms, f, false, bn, per, grid);
    CUtensorMap tx, tw, ty, tr;
    if (!make_map(&tx, x, M, K, BM, true, f) || !make_map(&tw, w, N, K, bn, true, f) ||
        !make_map(&ty, y, M, N, 16, false, f) || !make_map(&tr, residual ? residual : y, M, N, 16, false, f))
        return cudaErrorInvalidValue;
    const C1Eval ev{gamma, beta, mean, var, eps, relu ? 1 : 0};
    const bool r = residual != nullptr;
    if (f) {
        switch (bn) {
        case 256: return launch_eval<256, true>(tx, tw, ty, tr, (int)M, N, K, r, ev, grid, st);
        case 128: return launch_eval<128, true>(tx, tw, ty, tr, (int)M, N, K, r, ev, grid, st);
        default: return launch_eval<64, true>(tx, tw, ty, tr, (int)M, N, K, r, ev, grid, st);
        }
    }
    switch (bn) {
    case 256: return launch_eval<256, false>(tx, tw, ty, tr, (int)M, N, K, r, ev, grid, st);
    case 128: return launch_eval<128, false>(tx, tw, ty, tr, (int)M, N, K, r, ev, grid, st);
    default: return launch_eval<64, false>(tx, tw, ty, tr, (int)M, N, K, r, ev, grid, st);
    }
}

cudaError_t c1_launch_stats_finalize(const float* partial, int R, int C, const float* gamma, const float* beta,
                                     float* rmean, float* rvar, long long* nbt, double* acc, float momentum,
                                     float eps, float* mean, float* invstd, float* scale, float* shift,
                                     cudaStream_t st)
{
    c1_stats_finalize_kernel<<<(C + 31) / 32, 1024, 0, st>>>(partial, R, C, gamma, beta, rmean, rvar, nbt, acc,
                                                            momentum, eps, mean, invstd, scale, shift);
    return cudaGetLastError();
}

}  // extern "C"
