// Training-time image augmentation of uint8 shard batches (data/shards.py, GpuAugment with
// auto_augment='ta_wide' / 'ra' / 'imagenet' and / or random_erase > 0): one launch per batch, one CTA per
// image.
//
//   stage 1  crop   bilinear RandomResizedCrop + flip of the stored [S, S, 3] image with the affine
//                   map GpuAugment builds (F.affine_grid + F.grid_sample(bilinear, border,
//                   align_corners=False)), rounded half-to-even and clamped to uint8 -- the quantised
//                   image torchvision's uint8 pipeline hands the augmentation policy -- into shared memory
//   chain    every op of the row but the last non-Identity one, left to right, each on the uint8
//                   result of the one before (RandAugment / AutoAugment): its reduction (stage 2), then
//                   its uint8 result materialised in shared memory -- in place for the pointwise ops;
//                   geometric ops and Sharpness read other pixels, so they write their result into this
//                   image's slice of dst (3 out^2 bytes of the 12 / 6 out^2 the final stage overwrites),
//                   and the CTA reads it back with coherent L2 loads.  Identity entries are skipped.
//   stage 2  reduce only for the op that needs one: per-channel min / max (AutoContrast), per-channel
//                   256-bin histogram and equalisation LUT (Equalize), the sum of the floored grayscale
//                   image (Contrast); the tables are re-initialised after each op that used them
//   stage 3  output per element: the last op (reading shared memory), normalisation
//                   (v - 255 mean) * 1 / (255 std) in fp32, 0 inside the erase box, NHWC fp32 / bf16
//                   stores of 16 bytes
//
// Per-op arithmetic follows torchvision.transforms.v2.functional on uint8 tensors: fp32 products,
// blends as fmaf(1 - r, other, r * v) (torch's add_(other, alpha) is one fused multiply-add on the CPU
// and on CUDA), truncation back to uint8 after clamping, grayscale 0.2989 r + 0.587 g + 0.114 b
// floored.  Geometric ops sample nearest (round half to even) through torchvision's inverse affine
// matrix, precomputed on the host and rescaled as its _affine_grid does, with fill 0.
//
// Per-image parameter row (fp32, AUG_ROW_ONE_OP floats for one op, AUG_ROW for a chain of up to
// AUG_MAX_OPS ops; filled on the host -- data/shards.py GpuAugment.kernel_rows):
//   [0..5]   crop theta  (x_in = t0 x + t1 y + t2, y_in = t3 x + t4 y + t5 in grid_sample coordinates)
//   [6..14]  op 1:
//     [6]      op id (0 Identity, 1 ShearX, 2 ShearY, 3 TranslateX, 4 TranslateY, 5 Rotate, 6 Brightness,
//              7 Color, 8 Contrast, 9 Sharpness, 10 Posterize, 11 Solarize, 12 AutoContrast, 13 Equalize,
//              14 Invert)
//     [7], [8] op scalars: Brightness factor; Color / Contrast ratio r and 1 - r; Sharpness 1 - factor in
//              [8]; Posterize bit mask; Solarize threshold
//     [9..14]  geometric ops: gx = a xc + b yc + c, gy = d xc + e yc + f, with (xc, yc) the output pixel
//              relative to the image centre and (gx, gy) in grid_sample coordinates
//   [15..18] erase box rows [y0, y1) and columns [x0, x1); y1 = y0 means no box
//   chain rows only: op k = 2..AUG_MAX_OPS at [19 + 9 (k - 2) ..], laid out as op 1's [6..14]; 0 = Identity
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace {

constexpr int AUG_THREADS = 1024;
constexpr int AUG_ROW_ONE_OP = 24;
constexpr int AUG_MAX_OPS = 4;
constexpr int AUG_CHAIN_COL = 19;                // op 2's columns in a chain row; 9 per op
constexpr int AUG_ROW = 48;                      // AUG_CHAIN_COL + 9 (AUG_MAX_OPS - 1), padded to 4 floats
constexpr int AUG_TABLE_INTS = 3 * 256 + 16;     // histogram / LUT, then min[3], max[3], gray sum

enum {
    OP_IDENTITY = 0, OP_SHEAR_X, OP_SHEAR_Y, OP_TRANSLATE_X, OP_TRANSLATE_Y, OP_ROTATE, OP_BRIGHTNESS, OP_COLOR,
    OP_CONTRAST, OP_SHARPNESS, OP_POSTERIZE, OP_SOLARIZE, OP_AUTOCONTRAST, OP_EQUALIZE, OP_INVERT
};

struct AugNorm {
    float mean[3];   // 255 * mean, fp32
    float inv[3];    // 1 / (255 * std), fp32
};

__host__ __device__ constexpr size_t aug_image_bytes(int out) { return ((size_t)out * out * 3 + 15) / 16 * 16; }
__host__ __device__ constexpr size_t aug_smem_bytes(int out)
{
    return aug_image_bytes(out) + AUG_TABLE_INTS * sizeof(int);
}

// F.affine_grid's base coordinate (align_corners=False): linspace(-1, 1, n)[k] * (n - 1) / n, with
// ATen's linspace (start + step * k below the midpoint, end - step * (n - 1 - k) above it)
__device__ __forceinline__ float base_coord(int k, int n)
{
    if (n == 1) return 0.f;
    const float step = 2.f / (float)(n - 1);
    const float v = k < n / 2 ? -1.f + step * (float)k : 1.f - step * (float)(n - 1 - k);
    return v * (float)(n - 1) / (float)n;
}

__device__ __forceinline__ float gray_floor(float r, float g, float b)
{
    return floorf(fmaf(0.114f, b, fmaf(0.587f, g, r * 0.2989f)));
}

__device__ __forceinline__ int clamp_trunc(float v) { return (int)fminf(fmaxf(v, 0.f), 255.f); }

// the uint8 value of channel c at (y, x) after the op
__device__ __forceinline__ int ta_value(const uint8_t* img, const int* tab, int out, int op, float p0, float p1,
                                        const float* m, float xc_base, int y, int x, int c)
{
    const int pix = y * out + x;
    const int u = img[pix * 3 + c];
    switch (op) {
    case OP_SHEAR_X: case OP_SHEAR_Y: case OP_TRANSLATE_X: case OP_TRANSLATE_Y: case OP_ROTATE: {
        const float xc = (float)x - xc_base, yc = (float)y - xc_base;
        const float gx = xc * m[0] + yc * m[1] + m[2];
        const float gy = xc * m[3] + yc * m[4] + m[5];
        const float ix = rintf(((gx + 1.f) * (float)out - 1.f) * 0.5f);
        const float iy = rintf(((gy + 1.f) * (float)out - 1.f) * 0.5f);
        if (!(ix >= 0.f && ix < (float)out && iy >= 0.f && iy < (float)out)) return 0;
        return img[((int)iy * out + (int)ix) * 3 + c];
    }
    case OP_BRIGHTNESS:
        return clamp_trunc((float)u * p0);
    case OP_COLOR: {
        const uint8_t* q = img + pix * 3;
        const float g = gray_floor((float)q[0], (float)q[1], (float)q[2]);
        return clamp_trunc(fmaf(p1, g, (float)u * p0));
    }
    case OP_CONTRAST:
        return clamp_trunc(fmaf(p1, __int_as_float(tab[3 * 256 + 6]), (float)u * p0));
    case OP_SHARPNESS: {
        if (y == 0 || x == 0 || y == out - 1 || x == out - 1) return u;
        int n = 0;
#pragma unroll
        for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
            for (int dx = -1; dx <= 1; ++dx) n += img[(pix + dy * out + dx) * 3 + c];
        n += 4 * u;                                   // (sum of the 8 neighbours + 5 u) / 13
        // conv2d with the 1/13, 5/13 kernel then round(): n / 13 is never within 1/26 of a tie, so the
        // fp32 convolution rounds to the nearest integer of the exact quotient
        const int blur = (2 * n + 13) / 26;
        return clamp_trunc(fmaf(p1, (float)(blur - u), (float)u));
    }
    case OP_POSTERIZE:
        return u & (int)p0;
    case OP_SOLARIZE:
        return (float)u >= p0 ? 255 - u : u;
    case OP_AUTOCONTRAST: {
        float lo = (float)tab[3 * 256 + c], hi = (float)tab[3 * 256 + 3 + c];
        float inv_scale = (hi - lo) * (1.f / 255.f);
        if (hi == lo) { lo = 0.f; inv_scale = 1.f; }
        return clamp_trunc(((float)u - lo) / inv_scale);
    }
    case OP_EQUALIZE:
        return tab[c * 256 + u];
    case OP_INVERT:
        return 255 - u;
    default:
        return u;
    }
}

template <typename T> struct AugStore;
template <> struct AugStore<float> {
    static constexpr int V = 4;
    static __device__ __forceinline__ void vec(float* d, const float (&v)[V])
    {
        *reinterpret_cast<float4*>(d) = make_float4(v[0], v[1], v[2], v[3]);
    }
    static __device__ __forceinline__ void one(float* d, float v) { *d = v; }
};
template <> struct AugStore<__nv_bfloat16> {
    static constexpr int V = 8;
    static __device__ __forceinline__ void vec(__nv_bfloat16* d, const float (&v)[V])
    {
        uint32_t w[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            __nv_bfloat162 h = __floats2bfloat162_rn(v[2 * k], v[2 * k + 1]);
            w[k] = *reinterpret_cast<uint32_t*>(&h);
        }
        *reinterpret_cast<uint4*>(d) = make_uint4(w[0], w[1], w[2], w[3]);
    }
    static __device__ __forceinline__ void one(__nv_bfloat16* d, float v) { *d = __float2bfloat16_rn(v); }
};

__device__ __forceinline__ void init_tables(int* tab, int tid)
{
    if (tid < AUG_TABLE_INTS) {
        int init = 0;
        if (tid >= 3 * 256 && tid < 3 * 256 + 3) init = 255;          // running minimum
        tab[tid] = init;
    }
}

__device__ __forceinline__ bool uses_tables(int op)
{
    return op == OP_AUTOCONTRAST || op == OP_CONTRAST || op == OP_EQUALIZE;
}

// op k's 9 columns (id, two scalars, six matrix entries) in a parameter row
__device__ __forceinline__ const float* op_cols(const float* row, int k)
{
    return k == 0 ? row + 6 : row + AUG_CHAIN_COL + 9 * (k - 1);
}

// stage 2: the reduction op needs, into tab (initialised, and img final, at entry; both final at exit)
__device__ __forceinline__ void aug_reduce(const uint8_t* img, int* tab, int npix, int op, int tid)
{
    if (op == OP_AUTOCONTRAST || op == OP_CONTRAST || op == OP_EQUALIZE) {
        int lo[3] = {255, 255, 255}, hi[3] = {0, 0, 0}, gsum = 0;
        for (int p = tid; p < npix; p += AUG_THREADS) {
            const uint8_t* q = img + p * 3;
            if (op == OP_EQUALIZE) {
#pragma unroll
                for (int c = 0; c < 3; ++c) atomicAdd(&tab[c * 256 + q[c]], 1);
            } else if (op == OP_CONTRAST) {
                gsum += (int)gray_floor((float)q[0], (float)q[1], (float)q[2]);
            } else {
#pragma unroll
                for (int c = 0; c < 3; ++c) { lo[c] = min(lo[c], (int)q[c]); hi[c] = max(hi[c], (int)q[c]); }
            }
        }
        if (op == OP_CONTRAST) {
            gsum = __reduce_add_sync(0xffffffffu, gsum);                // exact: < 2^24 for out <= 256
            if ((tid & 31) == 0) atomicAdd(&tab[3 * 256 + 6], gsum);
        } else if (op == OP_AUTOCONTRAST) {
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                lo[c] = (int)__reduce_min_sync(0xffffffffu, (unsigned)lo[c]);
                hi[c] = (int)__reduce_max_sync(0xffffffffu, (unsigned)hi[c]);
            }
            if ((tid & 31) == 0) {
#pragma unroll
                for (int c = 0; c < 3; ++c) { atomicMin(&tab[3 * 256 + c], lo[c]); atomicMax(&tab[3 * 256 + 3 + c], hi[c]); }
            }
        }
        __syncthreads();
        if (op == OP_CONTRAST && tid == 0) {
            // torch.mean of the floored grayscale image: the integer sum is exact in fp32, then / N
            tab[3 * 256 + 6] = __float_as_int((float)tab[3 * 256 + 6] / (float)npix);
        } else if (op == OP_EQUALIZE && tid < 3) {
            // torchvision's equalize: step = (N - count of the last non-empty bin) // 255; lut[0] = 0,
            // lut[k] = min((cdf[k - 1] + step // 2) // step, 255); step == 0 leaves the channel as is
            int* h = tab + tid * 256;
            int last = 255;
            while (last > 0 && h[last] == 0) --last;
            const int step = (npix - h[last]) / 255;
            int cum = 0;
            for (int k = 0; k < 256; ++k) {
                const int cnt = h[k];
                h[k] = step == 0 ? k : (k == 0 ? 0 : min((cum + step / 2) / step, 255));
                cum += cnt;
            }
        }
        __syncthreads();
    }
}

template <typename TO>
__global__ void __launch_bounds__(AUG_THREADS, 1)
gpu_augment_kernel(const uint8_t* __restrict__ src, const float* __restrict__ rows, TO* __restrict__ dst, int S,
                   int out, AugNorm norm, int row_len, int vec_ok)
{
    extern __shared__ __align__(16) uint8_t smem[];
    uint8_t* img = smem;
    int* tab = reinterpret_cast<int*>(smem + aug_image_bytes(out));
    const int b = blockIdx.x;
    const int tid = threadIdx.x;
    const float* row = rows + (size_t)b * row_len;
    const uint8_t* in = src + (size_t)b * S * S * 3;
    const int npix = out * out;

    init_tables(tab, tid);

    // ---- stage 1: bilinear crop (grid_sample, border padding) -> rounded uint8 in shared memory ----
    {
        const float t0 = row[0], t1 = row[1], t2 = row[2], t3 = row[3], t4 = row[4], t5 = row[5];
        for (int p = tid; p < npix; p += AUG_THREADS) {
            const int y = p / out, x = p - y * out;
            const float bx = base_coord(x, out), by = base_coord(y, out);
            float ix = ((bx * t0 + by * t1 + t2) + 1.f) * (float)S;
            float iy = ((bx * t3 + by * t4 + t5) + 1.f) * (float)S;
            ix = fminf(fmaxf((ix - 1.f) / 2.f, 0.f), (float)(S - 1));
            iy = fminf(fmaxf((iy - 1.f) / 2.f, 0.f), (float)(S - 1));
            const float x0f = floorf(ix), y0f = floorf(iy);
            const int x0 = (int)x0f, y0 = (int)y0f;
            const float x1f = x0f + 1.f, y1f = y0f + 1.f;
            const float w_nw = (x1f - ix) * (y1f - iy), w_ne = (ix - x0f) * (y1f - iy);
            const float w_sw = (x1f - ix) * (iy - y0f), w_se = (ix - x0f) * (iy - y0f);
            const bool xin = x0 + 1 < S, yin = y0 + 1 < S;
            const uint8_t* q = in + ((size_t)y0 * S + x0) * 3;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                float acc = 0.f;
                acc += (float)q[c] * w_nw;
                if (xin) acc += (float)q[3 + c] * w_ne;
                if (yin) acc += (float)q[S * 3 + c] * w_sw;
                if (xin && yin) acc += (float)q[S * 3 + 3 + c] * w_se;
                img[p * 3 + c] = (uint8_t)fminf(fmaxf(rintf(acc), 0.f), 255.f);
            }
        }
    }
    __syncthreads();

    // ---- the chain: every op before the last non-Identity one, each materialised as uint8 in img ----
    const float xc_base = 0.5f * (float)(out - 1);
    const int nel = npix * 3;
    int last = 0;
    if (row_len == AUG_ROW) {
        for (int k = 1; k < AUG_MAX_OPS; ++k)
            if ((int)op_cols(row, k)[0] != OP_IDENTITY) last = k;
    }
    for (int k = 0; k < last; ++k) {
        const float* q = op_cols(row, k);
        const int op = (int)q[0];
        if (op == OP_IDENTITY) continue;                                // block-uniform
        aug_reduce(img, tab, npix, op, tid);
        const float p0 = q[1], p1 = q[2];
        const float* m = q + 3;
        if (op <= OP_ROTATE || op == OP_SHARPNESS) {
            // reads other pixels: stage the result in this image's slice of dst, which only the final
            // stage writes, then read it back through L2 (ld.global.cg: coherent with this CTA's stores)
            uint8_t* stage = reinterpret_cast<uint8_t*>(dst + (size_t)b * nel);
            auto at = [&](int e) -> uint32_t {
                const int p = e / 3, c = e - 3 * p;
                const int y = p / out, x = p - y * out;
                return (uint32_t)ta_value(img, tab, out, op, p0, p1, m, xc_base, y, x, c);
            };
            if (vec_ok) {                                               // nel % 4 == 0, dst 16-byte aligned
                uint32_t* st32 = reinterpret_cast<uint32_t*>(stage);
                for (int w = tid; w < nel / 4; w += AUG_THREADS) {
                    const int e = 4 * w;
                    st32[w] = at(e) | at(e + 1) << 8 | at(e + 2) << 16 | at(e + 3) << 24;
                }
                __syncthreads();
                for (int w = tid; w < nel / 4; w += AUG_THREADS)
                    reinterpret_cast<uint32_t*>(img)[w] = __ldcg(st32 + w);
            } else {
                for (int e = tid; e < nel; e += AUG_THREADS) stage[e] = (uint8_t)at(e);
                __syncthreads();
                for (int e = tid; e < nel; e += AUG_THREADS) img[e] = __ldcg(stage + e);
            }
        } else {
            // pointwise: each thread rewrites whole pixels it alone reads
            for (int p = tid; p < npix; p += AUG_THREADS) {
                const int y = p / out, x = p - y * out;
                int v[3];
#pragma unroll
                for (int c = 0; c < 3; ++c) v[c] = ta_value(img, tab, out, op, p0, p1, m, xc_base, y, x, c);
#pragma unroll
                for (int c = 0; c < 3; ++c) img[p * 3 + c] = (uint8_t)v[c];
            }
        }
        __syncthreads();
        if (uses_tables(op)) {
            init_tables(tab, tid);
            __syncthreads();
        }
    }

    // ---- stage 2: the last op's reduction ----
    const float* q = op_cols(row, last);
    const int op = (int)q[0];
    aug_reduce(img, tab, npix, op, tid);

    // ---- stage 3: last op, normalisation, erase, store ----
    const float p0 = q[1], p1 = q[2];
    const float* m = q + 3;                           // block-uniform loads, served by L1
    const int ey0 = (int)row[15], ey1 = (int)row[16], ex0 = (int)row[17], ex1 = (int)row[18];
    TO* o = dst + (size_t)b * nel;
    constexpr int V = AugStore<TO>::V;
    auto value = [&](int e) -> float {
        const int p = e / 3, c = e - 3 * p;
        const int y = p / out, x = p - y * out;
        if (y >= ey0 && y < ey1 && x >= ex0 && x < ex1) return 0.f;
        const int u = ta_value(img, tab, out, op, p0, p1, m, xc_base, y, x, c);
        // (selects, not norm.mean[c]: a run-time index into the parameter struct puts it on the stack)
        const float mc = c == 0 ? norm.mean[0] : (c == 1 ? norm.mean[1] : norm.mean[2]);
        const float ic = c == 0 ? norm.inv[0] : (c == 1 ? norm.inv[1] : norm.inv[2]);
        return ((float)u - mc) * ic;
    };
    if (vec_ok) {
        for (int e = tid * V; e < nel; e += AUG_THREADS * V) {
            float v[V];
#pragma unroll
            for (int k = 0; k < V; ++k) v[k] = value(e + k);
            AugStore<TO>::vec(o + e, v);
        }
    } else {
        for (int e = tid; e < nel; e += AUG_THREADS) AugStore<TO>::one(o + e, value(e));
    }
}

template <typename TO>
cudaError_t launch_typed(const uint8_t* src, const float* rows, int row_len, void* dst, int B, int S, int out,
                         AugNorm norm, cudaStream_t st)
{
    static bool attr_set[64] = {};
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    const size_t smem = aug_smem_bytes(out);
    if (dev < 64 && !attr_set[dev]) {
        int optin = 0;
        e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
        if (e != cudaSuccess) return e;
        e = cudaFuncSetAttribute(gpu_augment_kernel<TO>, cudaFuncAttributeMaxDynamicSharedMemorySize, optin);
        if (e != cudaSuccess) return e;
        attr_set[dev] = true;
    }
    const size_t nel = (size_t)out * out * 3;
    const int vec_ok = (nel % AugStore<TO>::V == 0) && (reinterpret_cast<uintptr_t>(dst) % 16 == 0);
    gpu_augment_kernel<TO><<<B, AUG_THREADS, smem, st>>>(src, rows, (TO*)dst, S, out, norm, row_len, vec_ok);
    return cudaGetLastError();
}

}  // namespace

extern "C" {

int sgp_augment_row() { return AUG_ROW; }
int sgp_augment_row_one_op() { return AUG_ROW_ONE_OP; }
long long sgp_augment_smem_bytes(int out) { return (long long)aug_smem_bytes(out); }

// src: uint8 [B, S, S, 3]; rows: fp32 [B, row_len] on the device, row_len AUG_ROW_ONE_OP (one op) or
// AUG_ROW (a chain); dst: [B, out, out, 3] (NHWC), fp32 (out_dtype 1) or bf16 (0); mean / inv: the 3
// normalisation constants each.
cudaError_t sgp_launch_augment(const uint8_t* src, const float* rows, int row_len, void* dst, int out_dtype, int B,
                               int S, int out, const float* mean, const float* inv, cudaStream_t st)
{
    if (B <= 0) return cudaSuccess;
    if (row_len != AUG_ROW_ONE_OP && row_len != AUG_ROW) return cudaErrorInvalidValue;
    AugNorm norm;
    for (int c = 0; c < 3; ++c) { norm.mean[c] = mean[c]; norm.inv[c] = inv[c]; }
    if (out_dtype == 0) return launch_typed<__nv_bfloat16>(src, rows, row_len, dst, B, S, out, norm, st);
    return launch_typed<float>(src, rows, row_len, dst, B, S, out, norm, st);
}

}  // extern "C"
