// ResNet stem convolution (C_in = 3 -> C_out = 64, 7x7, stride 2, pad 3), NHWC bf16,
// forward and weight-gradient, as implicit GEMMs on the tensor cores.
//
// Why a dedicated kernel: with 3 input channels the library falls back to generic
// kernels (ncu launch list, batch 256: fprop 1.48 ms, wgrad 0.77 ms per step) although
// the layer only moves ~0.5 GB (ideal ~0.1 ms).  K = 7*7*3 = 147 is too short for the
// big wgmma tiles to matter -- the op is bandwidth/issue bound -- so this uses warp-
// level mma.sync.m16n8k16 (bf16 in, fp32 accumulate) with the im2col gather done on the
// fly from a shared-memory copy of the input patch:
//
//   tile   = 8 x 16 output pixels (128 GEMM rows) x 64 channels, one warp per output row
//   patch  = 21 x 37 x 3 input window of the tile, zero-filled outside the image
//   A[p,k] = patch[2*pr + k/21][6*pc + k%21]      (k = (kh*7+kw)*3+ci, 21 = 7*3)
//   fprop : Y[128 x 64]   = A[128 x 160] * W^T[160 x 64]     (K padded 147 -> 160 with zeros)
//   wgrad : dW[64 x 160] += dY^T[64 x 128] * A[128 x 160]    per tile, accumulated in
//           registers over the CTA's tiles, then one fp32 atomicAdd per element
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

#define ST_THREADS 256
#define ST_TH 8            // output rows per tile
#define ST_TW 16           // output cols per tile
#define ST_PR (2 * ST_TH + 5)        // 21 patch rows
#define ST_PC (2 * ST_TW + 5)        // 37 patch cols
#define ST_PITCH 112                 // patch row pitch in elements (37*3 = 111 -> 112)
#define ST_K 147
#define ST_KP 160                    // K padded to 10 mma k-steps
#define ST_CO 64
#define ST_WPITCH 168                // weight row pitch in smem (bank-conflict padding)
// forward-only K layout: every kh row (7*3 = 21 taps) is padded to 24, so that the k pairs
// an mma register holds (2m, 2m+1) are ADJACENT, 4-byte aligned elements of the patch
// (32-bit shared loads instead of two 16-bit loads + a pack).  7 * 24 = 168 -> 176 (11 steps)
#define ST_KF 176
#define ST_WFPITCH 184

namespace {

__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4],
                                               const uint32_t (&b)[2]) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 "
        "{%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

__device__ __forceinline__ uint32_t pack2(uint16_t lo, uint16_t hi) {
    return (uint32_t)lo | ((uint32_t)hi << 16);
}

// k -> offset inside the patch relative to the pixel's top-left element, or -1 (padding)
__device__ __forceinline__ void fill_koff(int16_t* koff) {
    for (int k = threadIdx.x; k < ST_KP; k += ST_THREADS)
        koff[k] = (k < ST_K) ? (int16_t)((k / 21) * ST_PITCH + (k % 21)) : (int16_t)-1;
}

// The input window of a tile is fetched in two halves so that global-memory latency hides
// behind the previous tile's math: `patch_fetch` issues the loads into registers (one tile
// AHEAD), `patch_commit` writes them to shared memory once the current tile is done.
#define ST_PATCH_ELEMS (ST_PR * ST_PITCH)                                  // 2352
#define ST_PATCH_PER_THREAD ((ST_PATCH_ELEMS + ST_THREADS - 1) / ST_THREADS)   // 10

struct TileCoord { int n, oh0, ow0; };

__device__ __forceinline__ TileCoord tile_coord(long long t, int tiles_h, int tiles_w) {
    TileCoord c;
    c.ow0 = (int)(t % tiles_w) * ST_TW;
    c.oh0 = (int)((t / tiles_w) % tiles_h) * ST_TH;
    c.n = (int)(t / ((long long)tiles_w * tiles_h));
    return c;
}

__device__ __forceinline__ void patch_fetch(uint16_t (&reg)[ST_PATCH_PER_THREAD],
                                            const uint16_t* __restrict__ x, TileCoord tc, int H, int W)
{
    const int ih0 = 2 * tc.oh0 - 3, iw0 = 2 * tc.ow0 - 3;
#pragma unroll
    for (int i = 0; i < ST_PATCH_PER_THREAD; ++i) {
        const int e = threadIdx.x + i * ST_THREADS;
        const int r = e / ST_PITCH, c = e - r * ST_PITCH;       // c = col*3 + ci
        const int ih = ih0 + r, iw = iw0 + c / 3;
        uint16_t v = 0;
        if (e < ST_PATCH_ELEMS && c < ST_PC * 3 && ih >= 0 && ih < H && iw >= 0 && iw < W)
            v = x[((size_t)(tc.n * H + ih) * W + iw) * 3 + (c % 3)];
        reg[i] = v;
    }
}

__device__ __forceinline__ void patch_commit(uint16_t* patch, const uint16_t (&reg)[ST_PATCH_PER_THREAD])
{
#pragma unroll
    for (int i = 0; i < ST_PATCH_PER_THREAD; ++i) {
        const int e = threadIdx.x + i * ST_THREADS;
        if (e < ST_PATCH_ELEMS) patch[e] = reg[i];
    }
}

}  // namespace

// ---------------------------------------------------------------------------
// forward
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(ST_THREADS, 2)
stem_fwd_kernel(const uint16_t* __restrict__ x, const uint16_t* __restrict__ w,
                uint16_t* __restrict__ y, int N, int H, int W, int OH, int OW)
{
    __shared__ __align__(16) uint16_t s_w[ST_CO * ST_WFPITCH];       // [co][kh*24 + kw*3+ci]  23.0 KB
    __shared__ __align__(16) uint16_t s_patch[ST_PR * ST_PITCH + 8]; //                          4.6 KB
    __shared__ __align__(16) uint16_t s_out[ST_TH * ST_TW * ST_CO];  // [pix][co]               16.0 KB
    __shared__ int16_t s_koff[ST_KF];                                // even k -> patch offset

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int gid = lane >> 2, tig = lane & 3;

    for (int e = tid; e < ST_CO * ST_WFPITCH; e += ST_THREADS) {
        const int co = e / ST_WFPITCH, k = e - co * ST_WFPITCH;
        const int kh = k / 24, r = k - kh * 24;
        s_w[e] = (kh < 7 && r < 21) ? w[co * ST_K + kh * 21 + r] : (uint16_t)0;   // pads are ZERO
    }
    for (int k = tid; k < ST_KF; k += ST_THREADS)       // padded taps read finite neighbours (x 0)
        s_koff[k] = (k < 168) ? (int16_t)((k / 24) * ST_PITCH + (k % 24)) : (int16_t)0;
    if (tid < 8) s_patch[ST_PR * ST_PITCH + tid] = 0;

    const int tiles_w = (OW + ST_TW - 1) / ST_TW, tiles_h = (OH + ST_TH - 1) / ST_TH;
    const long long n_tiles = (long long)N * tiles_h * tiles_w;

    uint16_t pre[ST_PATCH_PER_THREAD];
    if ((long long)blockIdx.x < n_tiles) patch_fetch(pre, x, tile_coord(blockIdx.x, tiles_h, tiles_w), H, W);

    for (long long t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const TileCoord tc = tile_coord(t, tiles_h, tiles_w);
        const int n = tc.n, oh0 = tc.oh0, ow0 = tc.ow0;
        __syncthreads();                      // previous tile's smem fully consumed
        patch_commit(s_patch, pre);
        __syncthreads();
        if (t + gridDim.x < n_tiles)          // next tile's loads fly during this tile's math
            patch_fetch(pre, x, tile_coord(t + gridDim.x, tiles_h, tiles_w), H, W);

        // warp `warp` owns output row pr = warp: pixels (pr, pc = gid) and (pr, gid + 8)
        float acc[8][4];
#pragma unroll
        for (int j = 0; j < 8; ++j) { acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f; }
        const uint16_t* p0 = s_patch + (2 * warp) * ST_PITCH + 6 * gid;      // even offsets only
        const uint16_t* p1 = p0 + 6 * 8;
#pragma unroll 2
        for (int ks = 0; ks < ST_KF / 16; ++ks) {
            const int k0 = ks * 16 + tig * 2;
            const int o0 = s_koff[k0], o2 = s_koff[k0 + 8];
            uint32_t a[4];
            a[0] = *reinterpret_cast<const uint32_t*>(p0 + o0);
            a[1] = *reinterpret_cast<const uint32_t*>(p1 + o0);
            a[2] = *reinterpret_cast<const uint32_t*>(p0 + o2);
            a[3] = *reinterpret_cast<const uint32_t*>(p1 + o2);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const uint16_t* wr = s_w + (j * 8 + gid) * ST_WFPITCH + k0;
                uint32_t b[2];
                b[0] = *reinterpret_cast<const uint32_t*>(wr);
                b[1] = *reinterpret_cast<const uint32_t*>(wr + 8);
                mma_bf16_16816(acc[j], a, b);
            }
        }

        // stage the warp's 16 pixels x 64 channels as bf16, then 16-byte coalesced stores
        uint16_t* so = s_out + warp * ST_TW * ST_CO;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int ch = j * 8 + tig * 2;
            __nv_bfloat162 v0 = __floats2bfloat162_rn(acc[j][0], acc[j][1]);
            __nv_bfloat162 v1 = __floats2bfloat162_rn(acc[j][2], acc[j][3]);
            *reinterpret_cast<uint32_t*>(so + gid * ST_CO + ch) = *reinterpret_cast<uint32_t*>(&v0);
            *reinterpret_cast<uint32_t*>(so + (gid + 8) * ST_CO + ch) = *reinterpret_cast<uint32_t*>(&v1);
        }
        __syncwarp();
        const int oh = oh0 + warp;
        if (oh < OH) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int pc = i * 4 + (lane >> 3), part = lane & 7;     // 8 x 16 B per pixel
                const int ow = ow0 + pc;
                if (ow < OW) {
                    const uint4 v = *reinterpret_cast<const uint4*>(so + pc * ST_CO + part * 8);
                    *reinterpret_cast<uint4*>(y + (((size_t)n * OH + oh) * OW + ow) * ST_CO + part * 8) = v;
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------
// weight gradient: dw_acc[co][k] (fp32, zero-initialised) += sum over pixels
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(ST_THREADS, 2)
stem_wgrad_kernel(const uint16_t* __restrict__ x, const uint16_t* __restrict__ dy,
                  float* __restrict__ dw_acc, int N, int H, int W, int OH, int OW)
{
    __shared__ __align__(16) uint16_t s_patch[ST_PR * ST_PITCH];
    __shared__ __align__(16) uint16_t s_dyT[ST_CO * (ST_TH * ST_TW + 8)];   // [co][pixel], pitch 136
    __shared__ int16_t s_koff[ST_KP];
    constexpr int DP = ST_TH * ST_TW + 8;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int gid = lane >> 2, tig = lane & 3;
    fill_koff(s_koff);

    // warp -> (m-tile of 16 output channels, 10 consecutive n-tiles of 8 k-indices)
    const int mt = warp & 3, nt0 = (warp >> 2) * 10;
    float acc[10][4];
#pragma unroll
    for (int j = 0; j < 10; ++j) { acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f; }

    const int tiles_w = (OW + ST_TW - 1) / ST_TW, tiles_h = (OH + ST_TH - 1) / ST_TH;
    const long long n_tiles = (long long)N * tiles_h * tiles_w;

    // register prefetch of the NEXT tile (input patch + the 4 x 16 B of dy this thread stages)
    uint16_t pre[ST_PATCH_PER_THREAD];
    uint4 dpre[4];
    auto dy_fetch = [&](TileCoord tc) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int e = tid + i * ST_THREADS;
            const int p = e >> 3, part = e & 7;
            const int oh = tc.oh0 + p / ST_TW, ow = tc.ow0 + p % ST_TW;
            dpre[i] = make_uint4(0u, 0u, 0u, 0u);
            if (oh < OH && ow < OW)
                dpre[i] = *reinterpret_cast<const uint4*>(
                    dy + (((size_t)tc.n * OH + oh) * OW + ow) * ST_CO + part * 8);
        }
    };
    if ((long long)blockIdx.x < n_tiles) {
        const TileCoord tc0 = tile_coord(blockIdx.x, tiles_h, tiles_w);
        patch_fetch(pre, x, tc0, H, W);
        dy_fetch(tc0);
    }

    for (long long t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        __syncthreads();
        patch_commit(s_patch, pre);
        // dy tile, transposed to [co][pixel] so two consecutive pixels share a 32-bit word
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int e = tid + i * ST_THREADS;
            const int p = e >> 3, part = e & 7;
            const uint16_t* h = reinterpret_cast<const uint16_t*>(&dpre[i]);
#pragma unroll
            for (int q = 0; q < 8; ++q) s_dyT[(part * 8 + q) * DP + p] = h[q];
        }
        __syncthreads();
        if (t + gridDim.x < n_tiles) {
            const TileCoord tn = tile_coord(t + gridDim.x, tiles_h, tiles_w);
            patch_fetch(pre, x, tn, H, W);
            dy_fetch(tn);
        }

        // GEMM K dimension = the tile's 128 pixels, 16 per step (one output row per step)
#pragma unroll 1
        for (int ks = 0; ks < ST_TH; ++ks) {
            const int p0 = ks * 16 + tig * 2;                    // pixel index of a0 / b0
            uint32_t a[4];
            const uint16_t* d0 = s_dyT + (mt * 16 + gid) * DP + p0;
            const uint16_t* d1 = d0 + 8 * DP;
            a[0] = *reinterpret_cast<const uint32_t*>(d0);
            a[1] = *reinterpret_cast<const uint32_t*>(d1);
            a[2] = *reinterpret_cast<const uint32_t*>(d0 + 8);
            a[3] = *reinterpret_cast<const uint32_t*>(d1 + 8);
            // im2col rows for pixels (ks, tig*2), (ks, tig*2+1), (ks, tig*2+8), (ks, tig*2+9)
            const int rowb = (2 * ks) * ST_PITCH;
            const int pb0 = rowb + 6 * (tig * 2), pb1 = pb0 + 6, pb2 = pb0 + 48, pb3 = pb0 + 54;
#pragma unroll
            for (int j = 0; j < 10; ++j) {
                const int o = s_koff[(nt0 + j) * 8 + gid];
                uint32_t b[2];
                if (o >= 0) {
                    b[0] = pack2(s_patch[pb0 + o], s_patch[pb1 + o]);
                    b[1] = pack2(s_patch[pb2 + o], s_patch[pb3 + o]);
                } else {
                    b[0] = b[1] = 0u;
                }
                mma_bf16_16816(acc[j], a, b);
            }
        }
    }

    // one atomic per accumulator element: rows = output channel, cols = k index
#pragma unroll
    for (int j = 0; j < 10; ++j) {
        const int k = (nt0 + j) * 8 + tig * 2;
        const int co = mt * 16 + gid;
        if (k < ST_K)     { atomicAdd(dw_acc + co * ST_K + k, acc[j][0]);
                            atomicAdd(dw_acc + (co + 8) * ST_K + k, acc[j][2]); }
        if (k + 1 < ST_K) { atomicAdd(dw_acc + co * ST_K + k + 1, acc[j][1]);
                            atomicAdd(dw_acc + (co + 8) * ST_K + k + 1, acc[j][3]); }
    }
}

// ===========================================================================
// fp32 activations / weights, TF32 tensor-core math (mma.sync.m16n8k8.tf32): the
// precision-matched flagship path (the reference's cuDNN runs this layer in TF32 too, with
// generic kernels).
// Same tiling as the bf16 kernels; fp32 words in shared memory, so no pair-packing tricks:
//   fprop : Y[128 x 64] = A[128 x 152] * W^T[152 x 64]      (K 147 -> 152 = 19 k-steps of 8)
//   wgrad : dW[64 x 152] += dY^T[64 x 128] * A[128 x 152]   (K = the tile's 128 pixels)
// ===========================================================================
#define ST_K32 152                    // K padded to 19 mma k-steps of 8
#define ST_W32PITCH 156               // == 28 (mod 32): B-fragment loads are bank-conflict free

namespace {

__device__ __forceinline__ void mma_tf32_1688(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    asm volatile(
        "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 "
        "{%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

__device__ __forceinline__ void patch_fetch_f32(float (&reg)[ST_PATCH_PER_THREAD], const float* __restrict__ x,
                                                TileCoord tc, int H, int W)
{
    const int ih0 = 2 * tc.oh0 - 3, iw0 = 2 * tc.ow0 - 3;
#pragma unroll
    for (int i = 0; i < ST_PATCH_PER_THREAD; ++i) {
        const int e = threadIdx.x + i * ST_THREADS;
        const int r = e / ST_PITCH, c = e - r * ST_PITCH;       // c = col*3 + ci
        const int ih = ih0 + r, iw = iw0 + c / 3;
        float v = 0.f;
        if (e < ST_PATCH_ELEMS && c < ST_PC * 3 && ih >= 0 && ih < H && iw >= 0 && iw < W)
            v = __ldg(x + ((size_t)(tc.n * H + ih) * W + iw) * 3 + (c % 3));
        reg[i] = v;
    }
}

__device__ __forceinline__ void patch_commit_f32(float* patch, const float (&reg)[ST_PATCH_PER_THREAD])
{
#pragma unroll
    for (int i = 0; i < ST_PATCH_PER_THREAD; ++i) {
        const int e = threadIdx.x + i * ST_THREADS;
        if (e < ST_PATCH_ELEMS) patch[e] = reg[i];
    }
}

}  // namespace

// dynamic shared memory: [ s_w : 64 x 156 fp32 ][ s_patch : 21 x 112 (+8) fp32 ][ koff : 152 int16 ]
#define ST_F32_FWD_SMEM (ST_CO * ST_W32PITCH * 4 + (ST_PATCH_ELEMS + 8) * 4 + ST_K32 * 2 + 16)

__global__ void __launch_bounds__(ST_THREADS, 2)
stem_fwd_tf32_kernel(const float* __restrict__ x, const float* __restrict__ w, float* __restrict__ y,
                     int N, int H, int W, int OH, int OW)
{
    extern __shared__ __align__(16) unsigned char st_smem[];
    float* s_w = reinterpret_cast<float*>(st_smem);                             // [co][k], pads ZERO
    float* s_patch = s_w + ST_CO * ST_W32PITCH;
    int16_t* s_koff = reinterpret_cast<int16_t*>(s_patch + ST_PATCH_ELEMS + 8);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int gid = lane >> 2, tig = lane & 3;

    for (int e = tid; e < ST_CO * ST_W32PITCH; e += ST_THREADS) {
        const int co = e / ST_W32PITCH, k = e - co * ST_W32PITCH;
        s_w[e] = (k < ST_K) ? w[co * ST_K + k] : 0.f;
    }
    for (int k = tid; k < ST_K32; k += ST_THREADS)          // padded taps read a finite word (x 0)
        s_koff[k] = (k < ST_K) ? (int16_t)((k / 21) * ST_PITCH + (k % 21)) : (int16_t)0;
    if (tid < 8) s_patch[ST_PATCH_ELEMS + tid] = 0.f;

    const int tiles_w = (OW + ST_TW - 1) / ST_TW, tiles_h = (OH + ST_TH - 1) / ST_TH;
    const long long n_tiles = (long long)N * tiles_h * tiles_w;

    float pre[ST_PATCH_PER_THREAD];
    if ((long long)blockIdx.x < n_tiles) patch_fetch_f32(pre, x, tile_coord(blockIdx.x, tiles_h, tiles_w), H, W);

    for (long long t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const TileCoord tc = tile_coord(t, tiles_h, tiles_w);
        __syncthreads();                      // previous tile's patch fully consumed
        patch_commit_f32(s_patch, pre);
        __syncthreads();
        if (t + gridDim.x < n_tiles)          // next tile's loads fly during this tile's math
            patch_fetch_f32(pre, x, tile_coord(t + gridDim.x, tiles_h, tiles_w), H, W);

        // warp `warp` owns output row pr = warp: pixels (pr, gid) and (pr, gid + 8)
        float acc[8][4];
#pragma unroll
        for (int j = 0; j < 8; ++j) { acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f; }
        const float* p0 = s_patch + (2 * warp) * ST_PITCH + 6 * gid;
        const float* p1 = p0 + 6 * 8;
#pragma unroll 2
        for (int ks = 0; ks < ST_K32 / 8; ++ks) {
            const int k0 = ks * 8 + tig;
            const int o0 = s_koff[k0], o1 = s_koff[k0 + 4];
            uint32_t a[4];
            a[0] = __float_as_uint(p0[o0]);
            a[1] = __float_as_uint(p1[o0]);
            a[2] = __float_as_uint(p0[o1]);
            a[3] = __float_as_uint(p1[o1]);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float* wr = s_w + (j * 8 + gid) * ST_W32PITCH + k0;
                uint32_t b[2];
                b[0] = __float_as_uint(wr[0]);
                b[1] = __float_as_uint(wr[4]);
                mma_tf32_1688(acc[j], a, b);
            }
        }

        // C fragment: (pixel gid | gid+8, channels j*8 + 2*tig, +1): four adjacent lanes fill one
        // 32-byte sector, so the fragments are stored directly (no staging tile)
        const int oh = tc.oh0 + warp;
        if (oh < OH) {
            const int ow_a = tc.ow0 + gid, ow_b = ow_a + 8;
            float* ya = y + (((size_t)tc.n * OH + oh) * OW + ow_a) * ST_CO + 2 * tig;
            float* yb = ya + (size_t)8 * ST_CO;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                if (ow_a < OW) *reinterpret_cast<float2*>(ya + j * 8) = make_float2(acc[j][0], acc[j][1]);
                if (ow_b < OW) *reinterpret_cast<float2*>(yb + j * 8) = make_float2(acc[j][2], acc[j][3]);
            }
        }
    }
}

// weight gradient, fp32 / TF32: dw_acc[co][k] (fp32, zero-initialised) += sum over pixels
#define ST_DP32 132                   // dY^T row pitch (128 pixels + 4): == 4 (mod 32)
__global__ void __launch_bounds__(ST_THREADS, 2)
stem_wgrad_tf32_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dw_acc,
                       int N, int H, int W, int OH, int OW)
{
    __shared__ __align__(16) float s_patch[ST_PATCH_ELEMS];
    __shared__ __align__(16) float s_dyT[ST_CO * ST_DP32];       // [co][pixel ^ swz(co)]
    __shared__ int16_t s_koff[ST_KP];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int gid = lane >> 2, tig = lane & 3;
    fill_koff(s_koff);

    // warp -> (m-tile of 16 output channels, 10 consecutive n-tiles of 8 k-indices)
    const int mt = warp & 3, nt0 = (warp >> 2) * 10;
    float acc[10][4];
#pragma unroll
    for (int j = 0; j < 10; ++j) { acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f; }

    const int tiles_w = (OW + ST_TW - 1) / ST_TW, tiles_h = (OH + ST_TH - 1) / ST_TH;
    const long long n_tiles = (long long)N * tiles_h * tiles_w;

    // register prefetch of the NEXT tile: input patch + the 8 x 16 B of dy this thread stages
    float pre[ST_PATCH_PER_THREAD];
    float4 dpre[8];
    auto dy_fetch = [&](TileCoord tc) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int e = tid + i * ST_THREADS;
            const int p = e >> 4, part = e & 15;                  // 16 x 16 B per pixel
            const int oh = tc.oh0 + p / ST_TW, ow = tc.ow0 + p % ST_TW;
            dpre[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (oh < OH && ow < OW)
                dpre[i] = __ldg(reinterpret_cast<const float4*>(
                    dy + (((size_t)tc.n * OH + oh) * OW + ow) * ST_CO + part * 4));
        }
    };
    if ((long long)blockIdx.x < n_tiles) {
        const TileCoord tc0 = tile_coord(blockIdx.x, tiles_h, tiles_w);
        patch_fetch_f32(pre, x, tc0, H, W);
        dy_fetch(tc0);
    }

    // A-fragment rows of this warp: co = mt*16 + gid (swizzle 2*mt) and co + 8 (swizzle 2*mt + 1)
    const int swz_lo = (mt * 2) & 7, swz_hi = (mt * 2 + 1) & 7;
    const float* d_lo = s_dyT + (mt * 16 + gid) * ST_DP32;
    const float* d_hi = d_lo + 8 * ST_DP32;

    for (long long t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        __syncthreads();
        patch_commit_f32(s_patch, pre);
        // dy tile transposed to [co][pixel]; the pixel index is XOR-swizzled with (co >> 3) & 7 so
        // that the 16 lanes that write 16 different channel quads of one pixel hit 16 banks
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int e = tid + i * ST_THREADS;
            const int p = e >> 4, part = e & 15;
            const float v[4] = {dpre[i].x, dpre[i].y, dpre[i].z, dpre[i].w};
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int co = part * 4 + q;
                s_dyT[co * ST_DP32 + (p ^ ((co >> 3) & 7))] = v[q];
            }
        }
        __syncthreads();
        if (t + gridDim.x < n_tiles) {
            const TileCoord tn = tile_coord(t + gridDim.x, tiles_h, tiles_w);
            patch_fetch_f32(pre, x, tn, H, W);
            dy_fetch(tn);
        }

        // GEMM K dimension = the tile's 128 pixels, 8 per step (half an output row per step)
#pragma unroll 1
        for (int ks = 0; ks < 2 * ST_TH; ++ks) {
            const int pix = ks * 8 + tig;                        // pixel of a0/a1/b0; +4: a2/a3/b1
            uint32_t a[4];
            a[0] = __float_as_uint(d_lo[pix ^ swz_lo]);
            a[1] = __float_as_uint(d_hi[pix ^ swz_hi]);
            a[2] = __float_as_uint(d_lo[(pix + 4) ^ swz_lo]);
            a[3] = __float_as_uint(d_hi[(pix + 4) ^ swz_hi]);
            // im2col rows of pixels (pr, pc) and (pr, pc + 4)
            const int pb0 = (2 * (ks >> 1)) * ST_PITCH + 6 * ((ks & 1) * 8 + tig), pb1 = pb0 + 24;
#pragma unroll
            for (int j = 0; j < 10; ++j) {
                const int o = s_koff[(nt0 + j) * 8 + gid];
                uint32_t b[2];
                if (o >= 0) {
                    b[0] = __float_as_uint(s_patch[pb0 + o]);
                    b[1] = __float_as_uint(s_patch[pb1 + o]);
                } else {
                    b[0] = b[1] = 0u;
                }
                mma_tf32_1688(acc[j], a, b);
            }
        }
    }

    // one atomic per accumulator element: rows = output channel, cols = k index
#pragma unroll
    for (int j = 0; j < 10; ++j) {
        const int k = (nt0 + j) * 8 + tig * 2;
        const int co = mt * 16 + gid;
        if (k < ST_K)     { atomicAdd(dw_acc + co * ST_K + k, acc[j][0]);
                            atomicAdd(dw_acc + (co + 8) * ST_K + k, acc[j][2]); }
        if (k + 1 < ST_K) { atomicAdd(dw_acc + co * ST_K + k + 1, acc[j][1]);
                            atomicAdd(dw_acc + (co + 8) * ST_K + k + 1, acc[j][3]); }
    }
}

extern "C" {

cudaError_t stem_launch_fwd_f32(const void* x, const void* w, void* y, int N, int H, int W, int OH, int OW,
                                cudaStream_t st)
{
    const long long tiles = (long long)N * ((OH + ST_TH - 1) / ST_TH) * ((OW + ST_TW - 1) / ST_TW);
    int grid = 132 * 2;
    if (tiles < grid) grid = (int)tiles;
    static bool configured[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64 || !configured[dev]) {
        cudaError_t e = cudaFuncSetAttribute(stem_fwd_tf32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             ST_F32_FWD_SMEM);
        if (e != cudaSuccess) return e;
        if (dev >= 0 && dev < 64) configured[dev] = true;
    }
    stem_fwd_tf32_kernel<<<grid, ST_THREADS, ST_F32_FWD_SMEM, st>>>((const float*)x, (const float*)w, (float*)y,
                                                                    N, H, W, OH, OW);
    return cudaGetLastError();
}

cudaError_t stem_launch_wgrad_f32(const void* x, const void* dy, float* dw_acc, int N, int H, int W,
                                  int OH, int OW, cudaStream_t st)
{
    const long long tiles = (long long)N * ((OH + ST_TH - 1) / ST_TH) * ((OW + ST_TW - 1) / ST_TW);
    int grid = 132 * 2;
    if (tiles < grid) grid = (int)tiles;
    stem_wgrad_tf32_kernel<<<grid, ST_THREADS, 0, st>>>((const float*)x, (const float*)dy, dw_acc, N, H, W, OH, OW);
    return cudaGetLastError();
}

cudaError_t stem_launch_fwd(const void* x, const void* w, void* y, int N, int H, int W, int OH, int OW,
                            cudaStream_t st)
{
    const long long tiles = (long long)N * ((OH + ST_TH - 1) / ST_TH) * ((OW + ST_TW - 1) / ST_TW);
    int grid = 132 * 2;
    if (tiles < grid) grid = (int)tiles;
    stem_fwd_kernel<<<grid, ST_THREADS, 0, st>>>((const uint16_t*)x, (const uint16_t*)w, (uint16_t*)y,
                                                 N, H, W, OH, OW);
    return cudaGetLastError();
}

cudaError_t stem_launch_wgrad(const void* x, const void* dy, float* dw_acc, int N, int H, int W,
                              int OH, int OW, cudaStream_t st)
{
    const long long tiles = (long long)N * ((OH + ST_TH - 1) / ST_TH) * ((OW + ST_TW - 1) / ST_TW);
    int grid = 132 * 2;
    if (tiles < grid) grid = (int)tiles;
    stem_wgrad_kernel<<<grid, ST_THREADS, 0, st>>>((const uint16_t*)x, (const uint16_t*)dy, dw_acc,
                                                   N, H, W, OH, OW);
    return cudaGetLastError();
}

}  // extern "C"
