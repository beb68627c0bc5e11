// torch bindings for the fused NHWC BatchNorm kernels (bn_kernels.cu)
#include <torch/extension.h>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <cuda_runtime.h>

#include <atomic>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

namespace py = pybind11;

extern "C" {
int bn_supported(long long M, int C);
int bn_partial_rows(long long M, int C);
int bn_partial_rows_bwd(long long M, int C);
int bn_f32_map(int value);
cudaError_t bn_launch_stats(int dtype, const void* x, float* partial, long long M, int C, int G, cudaStream_t st);
cudaError_t bn_launch_stats_finalize(const float* partial, int G, long long M, int C, const float* gamma,
                                     const float* beta, float* rmean, float* rvar, long long* nbt, double* acc,
                                     float momentum, float eps, float* mean, float* invstd,
                                     float* scale, float* shift, cudaStream_t st);
int bn_commit_max_segs();
cudaError_t bn_launch_stats_commit(const long long* rows, int nseg, double k, cudaStream_t st);
cudaError_t bn_launch_eval_coeff(int C, const float* gamma, const float* beta, const float* rmean,
                                 const float* rvar, float eps, float* scale, float* shift, cudaStream_t st);
cudaError_t bn_launch_apply(int dtype, int relu, int add, const void* x, const void* res,
                            const float* scale, const float* shift, void* y, uint8_t* mask, long long M, int C,
                            int G, cudaStream_t st);
cudaError_t bn_launch_bwd_reduce(int dtype, int mode, const void* dy, const void* x, const void* y,
                                 const float* scale, const float* shift, const float* mean,
                                 const float* invstd, float* partial, void* dz, long long M, int C,
                                 int G, cudaStream_t st);
cudaError_t bn_launch_bwd_finalize(const float* partial, int G, long long M, int C, const float* scale,
                                   const float* mean, const float* invstd, float* ggamma, float* gbeta,
                                   float* c2, float* c3, cudaStream_t st);
cudaError_t bn_launch_bwd_dx(int dtype, int mode, const void* dz, const void* x, const float* scale,
                             const float* shift, const float* c2, const float* c3, void* dx,
                             long long M, int C, int G, cudaStream_t st);
cudaError_t bn_launch_apply_drop(int dtype, const void* x, const void* res, const float* scale, const float* shift,
                                 void* y, uint8_t* mask, const float* sdrop, int hw, long long M, int C, int G,
                                 cudaStream_t st);
cudaError_t bn_launch_bwd_reduce_drop(int dtype, const void* dy, const void* x, const void* y, const float* mean,
                                      const float* invstd, float* partial, void* dz, const float* sdrop, int hw,
                                      long long M, int C, int G, cudaStream_t st);
cudaError_t bn_launch_bwd_dx_drop(int dtype, const void* dz, const void* x, const float* scale, const float* c2,
                                  const float* c3, void* dx, const float* sdrop, int hw, long long M, int C, int G,
                                  cudaStream_t st);
int drop_path_max_blocks();
cudaError_t drop_path_launch_draw(const unsigned int* thresh, const float* keep_scale, int L, int n,
                                  unsigned long long seed, unsigned long long rank, long long* counter, float* out,
                                  cudaStream_t st);
}

extern std::atomic<long long> g_sgp_kernel_launches;       // bindings.cpp

#define BN_CHECK(expr)                                                                   \
    do {                                                                                 \
        if (std::strstr(#expr, "_launch_") != nullptr) ++g_sgp_kernel_launches;          \
        cudaError_t _e = (expr);                                                         \
        if (_e != cudaSuccess)                                                           \
            throw std::runtime_error(std::string(#expr) + ": " + cudaGetErrorString(_e)); \
    } while (0)

static int dtype_code(const torch::Tensor& t)
{
    if (t.scalar_type() == torch::kBFloat16) return 0;
    if (t.scalar_type() == torch::kFloat32) return 1;
    throw std::runtime_error("fused BN supports bf16 / fp32 activations");
}

// x must be NHWC-dense: a 4-D channels_last tensor or a 2-D [M, C] matrix
static void nhwc_dims(const torch::Tensor& x, long long& M, int& C)
{
    if (x.dim() == 4) {
        TORCH_CHECK(x.is_contiguous(at::MemoryFormat::ChannelsLast), "fused BN needs channels_last input");
        C = (int)x.size(1);
        M = x.numel() / C;
    } else {
        TORCH_CHECK(x.dim() == 2 && x.is_contiguous());
        C = (int)x.size(1);
        M = x.size(0);
    }
}

static bool bn_can_fuse(const torch::Tensor& x)
{
    if (!x.is_cuda()) return false;
    if (x.scalar_type() != torch::kBFloat16 && x.scalar_type() != torch::kFloat32) return false;
    if (x.dim() == 4) { if (!x.is_contiguous(at::MemoryFormat::ChannelsLast)) return false; }
    else if (!(x.dim() == 2 && x.is_contiguous())) return false;
    const int C = (int)x.size(1);
    return bn_supported(x.numel() / C, C) != 0;
}

// acc (training only): a contiguous fp64 [2C] tensor on x's device, or None.  Given, the finalize adds the
// batch mean and unbiased variance to acc[0:C] and acc[C:2C] and leaves the running buffers and nbt alone
// (precise BatchNorm statistics, ops/fused_bn.py precise_bn_stats)
static double* bn_acc_ptr(const c10::optional<torch::Tensor>& acc, const torch::Tensor& x, int C)
{
    if (!acc.has_value() || !acc->defined()) return nullptr;
    TORCH_CHECK(acc->is_cuda() && acc->get_device() == x.get_device() && acc->scalar_type() == torch::kFloat64 &&
                    acc->is_contiguous() && acc->numel() == 2 * (int64_t)C,
                "acc must be a contiguous fp64 [2C] tensor on x's device");
    return acc->data_ptr<double>();
}

// branch_scale (stochastic depth): a contiguous fp32 [n] tensor on x's device, one value per sample of x, whose
// M rows are n samples of hw = M / n rows each (4-D x: n = x.size(0)); or None.  Returns its pointer and sets hw.
static const float* branch_scale_ptr(const c10::optional<torch::Tensor>& s, const torch::Tensor& x, long long M,
                                     int& hw)
{
    hw = 1;
    if (!s.has_value() || !s->defined()) return nullptr;
    TORCH_CHECK(s->is_cuda() && s->get_device() == x.get_device() && s->scalar_type() == torch::kFloat32 &&
                    s->is_contiguous() && s->dim() == 1 && s->numel() >= 1 && M % s->numel() == 0 &&
                    (x.dim() != 4 || s->numel() == x.size(0)) && M < (1LL << 31),
                "branch_scale must be a contiguous fp32 [N] tensor on x's device, one value per sample");
    hw = (int)(M / s->numel());
    return s->data_ptr<float>();
}

// returns (y, mean, invstd, scale, shift)
static std::vector<torch::Tensor> bn_forward(torch::Tensor x, c10::optional<torch::Tensor> residual,
                                             torch::Tensor gamma, torch::Tensor beta,
                                             c10::optional<torch::Tensor> running_mean,
                                             c10::optional<torch::Tensor> running_var,
                                             c10::optional<torch::Tensor> num_batches_tracked,
                                             bool training, double momentum, double eps, bool relu,
                                             c10::optional<torch::Tensor> acc,
                                             c10::optional<torch::Tensor> branch_scale)
{
    long long M; int C;
    nhwc_dims(x, M, C);
    TORCH_CHECK(bn_supported(M, C), "unsupported channel count ", C);
    TORCH_CHECK(gamma.scalar_type() == torch::kFloat32 && beta.scalar_type() == torch::kFloat32);
    const int dt = dtype_code(x);
    c10::cuda::CUDAGuard guard(x.get_device());
    auto st = at::cuda::getCurrentCUDAStream();
    auto fopt = torch::TensorOptions().dtype(torch::kFloat32).device(x.device());
    auto y = torch::empty_like(x);
    auto coef = torch::empty({4, C}, fopt);      // mean, invstd, scale, shift
    float* mean = coef.data_ptr<float>();
    float* invstd = mean + C; float* scale = mean + 2 * C; float* shift = mean + 3 * C;
    const bool has_res = residual.has_value() && residual->defined();
    if (has_res) TORCH_CHECK(residual->sizes() == x.sizes() && residual->scalar_type() == x.scalar_type()
                             && residual->strides() == x.strides());
    double* accp = bn_acc_ptr(acc, x, C);
    TORCH_CHECK(training || accp == nullptr, "bn_forward: acc needs training mode");
    if (training) {
        const int G = bn_partial_rows(M, C);
        auto partial = torch::empty({G + 1, 2, C}, fopt);   // last row carries the shift K
        BN_CHECK(bn_launch_stats(dt, x.data_ptr(), partial.data_ptr<float>(), M, C, G, st));
        float* rm = nullptr; float* rv = nullptr; long long* nbt = nullptr;
        if (running_mean.has_value() && running_mean->defined()) {
            rm = running_mean->data_ptr<float>();
            rv = running_var->data_ptr<float>();
        }
        if (num_batches_tracked.has_value() && num_batches_tracked->defined())
            nbt = reinterpret_cast<long long*>(num_batches_tracked->data_ptr<int64_t>());
        BN_CHECK(bn_launch_stats_finalize(partial.data_ptr<float>(), G, M, C, gamma.data_ptr<float>(),
                                          beta.data_ptr<float>(), rm, rv, nbt, accp, (float)momentum,
                                          (float)eps, mean, invstd, scale, shift, st));
    } else {
        TORCH_CHECK(running_mean.has_value() && running_var.has_value());
        BN_CHECK(bn_launch_eval_coeff(C, gamma.data_ptr<float>(), beta.data_ptr<float>(),
                                      running_mean->data_ptr<float>(), running_var->data_ptr<float>(),
                                      (float)eps, scale, shift, st));
    }
    int hw;
    const float* sdrop = branch_scale_ptr(branch_scale, x, M, hw);
    if (sdrop != nullptr) {
        TORCH_CHECK(has_res && relu && training, "bn_forward: branch_scale needs a residual, relu and training mode");
        BN_CHECK(bn_launch_apply_drop(dt, x.data_ptr(), residual->data_ptr(), scale, shift, y.data_ptr(), nullptr,
                                      sdrop, hw, M, C, 0, st));
        return {y, coef};
    }
    BN_CHECK(bn_launch_apply(dt, relu ? 1 : 0, has_res ? 1 : 0, x.data_ptr(),
                             has_res ? residual->data_ptr() : nullptr, scale, shift, y.data_ptr(), nullptr,
                             M, C, 0, st));
    return {y, coef};
}

// returns (dx, dres or undefined, grad_gamma, grad_beta).  branch_scale (residual + relu only): the forward's
// per-sample scale s of the BN output; dres = dy * (y > 0) unscaled, the BN's gradient is s * dres
static std::vector<torch::Tensor> bn_backward(torch::Tensor dy, torch::Tensor x,
                                              c10::optional<torch::Tensor> y, torch::Tensor coef,
                                              bool relu, bool add, c10::optional<torch::Tensor> branch_scale)
{
    long long M; int C;
    nhwc_dims(x, M, C);
    const int dt = dtype_code(x);
    TORCH_CHECK(dy.scalar_type() == x.scalar_type());
    if (dy.strides() != x.strides()) dy = dy.contiguous(x.dim() == 4 ? at::MemoryFormat::ChannelsLast
                                                                     : at::MemoryFormat::Contiguous);
    c10::cuda::CUDAGuard guard(x.get_device());
    auto st = at::cuda::getCurrentCUDAStream();
    auto fopt = torch::TensorOptions().dtype(torch::kFloat32).device(x.device());
    const float* mean = coef.data_ptr<float>();
    const float* invstd = mean + C; const float* scale = mean + 2 * C; const float* shift = mean + 3 * C;
    const int mode = add ? 2 : (relu ? 1 : 0);
    TORCH_CHECK(!add || relu, "residual add without ReLU is plain autograd (not fused)");
    if (mode == 2) TORCH_CHECK(y.has_value() && y->defined() && y->strides() == x.strides());
    const int G = bn_partial_rows_bwd(M, C);
    auto partial = torch::empty({G, 2, C}, fopt);
    auto grads = torch::empty({4, C}, fopt);    // grad_gamma, grad_beta, c2, c3
    float* gg = grads.data_ptr<float>();
    torch::Tensor dz;
    if (mode == 2) dz = torch::empty_like(x);
    int hw;
    const float* sdrop = branch_scale_ptr(branch_scale, x, M, hw);
    if (sdrop != nullptr) {
        TORCH_CHECK(mode == 2, "bn_backward: branch_scale needs a residual and relu");
        BN_CHECK(bn_launch_bwd_reduce_drop(dt, dy.data_ptr(), x.data_ptr(), y->data_ptr(), mean, invstd,
                                           partial.data_ptr<float>(), dz.data_ptr(), sdrop, hw, M, C, G, st));
        BN_CHECK(bn_launch_bwd_finalize(partial.data_ptr<float>(), G, M, C, scale, mean, invstd,
                                        gg, gg + C, gg + 2 * C, gg + 3 * C, st));
        auto dx = torch::empty_like(x);
        BN_CHECK(bn_launch_bwd_dx_drop(dt, dz.data_ptr(), x.data_ptr(), scale, gg + 2 * C, gg + 3 * C, dx.data_ptr(),
                                       sdrop, hw, M, C, 0, st));
        return {dx, dz, grads.select(0, 0), grads.select(0, 1)};
    }
    BN_CHECK(bn_launch_bwd_reduce(dt, mode, dy.data_ptr(), x.data_ptr(),
                                  mode == 2 ? y->data_ptr() : nullptr, scale, shift, mean, invstd,
                                  partial.data_ptr<float>(), mode == 2 ? dz.data_ptr() : nullptr,
                                  M, C, G, st));
    BN_CHECK(bn_launch_bwd_finalize(partial.data_ptr<float>(), G, M, C, scale, mean, invstd,
                                    gg, gg + C, gg + 2 * C, gg + 3 * C, st));
    auto dx = torch::empty_like(x);
    BN_CHECK(bn_launch_bwd_dx(dt, mode == 1 ? 1 : 0, mode == 2 ? dz.data_ptr() : dy.data_ptr(),
                              x.data_ptr(), scale, shift, gg + 2 * C, gg + 3 * C, dx.data_ptr(),
                              M, C, 0, st));
    return {dx, dz, grads.select(0, 0), grads.select(0, 1)};
}

// bn_backward's finalize + dx passes for a dz whose reduction partial[G][2][C] (sum dz, sum dz * xhat)
// was produced elsewhere (the MODE 3 dgrad epilogue); returns (dx, grad_gamma, grad_beta).  branch_scale: as in
// bn_backward (the partials are then those of s * dz)
static std::vector<torch::Tensor> bn_backward_from_partials(torch::Tensor dz, torch::Tensor x, torch::Tensor coef,
                                                            torch::Tensor partial,
                                                            c10::optional<torch::Tensor> branch_scale)
{
    long long M; int C;
    nhwc_dims(x, M, C);
    const int dt = dtype_code(x);
    TORCH_CHECK(dz.scalar_type() == x.scalar_type() && dz.sizes() == x.sizes() && dz.strides() == x.strides());
    TORCH_CHECK(partial.scalar_type() == torch::kFloat32 && partial.is_contiguous() && partial.dim() == 3 &&
                partial.size(1) == 2 && partial.size(2) == C);
    c10::cuda::CUDAGuard guard(x.get_device());
    auto st = at::cuda::getCurrentCUDAStream();
    const float* mean = coef.data_ptr<float>();
    const float* invstd = mean + C; const float* scale = mean + 2 * C; const float* shift = mean + 3 * C;
    auto grads = torch::empty({4, C}, torch::TensorOptions().dtype(torch::kFloat32).device(x.device()));
    float* gg = grads.data_ptr<float>();
    BN_CHECK(bn_launch_bwd_finalize(partial.data_ptr<float>(), (int)partial.size(0), M, C, scale, mean, invstd,
                                    gg, gg + C, gg + 2 * C, gg + 3 * C, st));
    auto dx = torch::empty_like(x);
    int hw;
    const float* sdrop = branch_scale_ptr(branch_scale, x, M, hw);
    if (sdrop != nullptr)
        BN_CHECK(bn_launch_bwd_dx_drop(dt, dz.data_ptr(), x.data_ptr(), scale, gg + 2 * C, gg + 3 * C, dx.data_ptr(),
                                       sdrop, hw, M, C, 0, st));
    else
        BN_CHECK(bn_launch_bwd_dx(dt, 0, dz.data_ptr(), x.data_ptr(), scale, shift, gg + 2 * C, gg + 3 * C,
                                  dx.data_ptr(), M, C, 0, st));
    return {dx, grads.select(0, 0), grads.select(0, 1)};
}

// running_mean[l] = fp32(acc[l][0:C] / k), running_var[l] = fp32(acc[l][C:2C] / k) for every layer l: one
// launch per BN_COMMIT_MAX_SEGS layers on the current stream (precise BatchNorm statistics).  acc[l]: contiguous
// fp64 [2C]; running_mean[l], running_var[l]: contiguous fp32 [C], all on one device; k >= 1.
static void bn_stats_commit(const std::vector<torch::Tensor>& acc, const std::vector<torch::Tensor>& running_mean,
                            const std::vector<torch::Tensor>& running_var, int64_t k)
{
    auto fail = [](size_t i, const char* what) {
        throw std::runtime_error("bn_stats_commit: layer " + std::to_string(i) + ": " + what);
    };
    if (acc.size() != running_mean.size() || acc.size() != running_var.size())
        throw std::runtime_error("bn_stats_commit: acc, running_mean and running_var must have the same length");
    if (k < 1) throw std::runtime_error("bn_stats_commit: k must be >= 1");
    if (acc.empty()) return;
    const auto device = acc[0].device();
    std::vector<long long> rows;
    rows.reserve(4 * acc.size());
    for (size_t i = 0; i < acc.size(); ++i) {
        const torch::Tensor& a = acc[i];
        const torch::Tensor& m = running_mean[i];
        const torch::Tensor& v = running_var[i];
        const int64_t C = m.numel();
        if (!(a.is_cuda() && m.is_cuda() && v.is_cuda() && a.device() == device && m.device() == device &&
              v.device() == device))
            fail(i, "every tensor must be a CUDA tensor on the first acc's device");
        if (!(a.scalar_type() == torch::kFloat64 && a.is_contiguous() && a.numel() == 2 * C && C >= 1))
            fail(i, "acc must be a contiguous fp64 [2C] tensor");
        if (!(m.scalar_type() == torch::kFloat32 && v.scalar_type() == torch::kFloat32 && m.is_contiguous() &&
              v.is_contiguous() && v.numel() == C))
            fail(i, "running_mean and running_var must be contiguous fp32 [C] tensors");
        rows.insert(rows.end(), {(long long)reinterpret_cast<uintptr_t>(a.data_ptr()),
                                 (long long)reinterpret_cast<uintptr_t>(m.data_ptr()),
                                 (long long)reinterpret_cast<uintptr_t>(v.data_ptr()), (long long)C});
    }
    c10::cuda::CUDAGuard guard(device);
    const auto st = at::cuda::getCurrentCUDAStream();
    const long long nseg = (long long)rows.size() / 4, per = bn_commit_max_segs();
    for (long long b = 0; b < nseg; b += per)
        BN_CHECK(bn_launch_stats_commit(rows.data() + 4 * b, (int)std::min(per, nseg - b), (double)k, st));
}

// ---------------------------------------------------------------------------
// The streaming BN kernels one launch at a time (kernel tests and benchmarks/bn_bandwidth.py).
// coef is bn_forward's [4, C] (mean, invstd, scale, shift), c23 a [2, C] (c2, c3); G <= 0 is the
// grid bn_forward / bn_backward launch.
// ---------------------------------------------------------------------------
static void bn_kernel_args(const torch::Tensor& x, const torch::Tensor& coef, long long& M, int& C)
{
    nhwc_dims(x, M, C);
    TORCH_CHECK(x.is_cuda() && bn_supported(M, C), "unsupported tensor for the BN kernels");
    TORCH_CHECK(coef.is_cuda() && coef.scalar_type() == torch::kFloat32 && coef.is_contiguous() &&
                coef.dim() == 2 && coef.size(1) == C);
}

static void same_layout(const torch::Tensor& t, const torch::Tensor& x)
{
    TORCH_CHECK(t.scalar_type() == x.scalar_type() && t.sizes() == x.sizes() && t.strides() == x.strides(),
                "operands must match x's dtype, shape and layout");
}

// partial[G + 1][2][C]: per-CTA shifted sums and the shift row
static torch::Tensor bn_kernel_stats(torch::Tensor x, int G)
{
    long long M; int C;
    nhwc_dims(x, M, C);
    TORCH_CHECK(x.is_cuda() && bn_supported(M, C), "unsupported tensor for the BN kernels");
    c10::cuda::CUDAGuard guard(x.get_device());
    if (G <= 0) G = bn_partial_rows(M, C);
    auto partial = torch::empty({G + 1, 2, C}, x.options().dtype(torch::kFloat32));
    BN_CHECK(bn_launch_stats(dtype_code(x), x.data_ptr(), partial.data_ptr<float>(), M, C, G,
                             at::cuda::getCurrentCUDAStream()));
    return partial;
}

static torch::Tensor bn_kernel_apply(torch::Tensor x, c10::optional<torch::Tensor> residual, torch::Tensor coef,
                                     bool relu, c10::optional<torch::Tensor> mask, int G)
{
    long long M; int C;
    bn_kernel_args(x, coef, M, C);
    TORCH_CHECK(coef.size(0) >= 4);
    const bool has_res = residual.has_value() && residual->defined();
    const bool has_mask = mask.has_value() && mask->defined();
    if (has_res) same_layout(*residual, x);
    if (has_mask) TORCH_CHECK(mask->is_cuda() && mask->scalar_type() == torch::kUInt8 && mask->is_contiguous() &&
                              mask->numel() == M * (C / 8), "mask must be [M, C/8] uint8");
    c10::cuda::CUDAGuard guard(x.get_device());
    auto y = torch::empty_like(x);
    const float* cf = coef.data_ptr<float>();
    BN_CHECK(bn_launch_apply(dtype_code(x), relu ? 1 : 0, has_res ? 1 : 0, x.data_ptr(),
                             has_res ? residual->data_ptr() : nullptr, cf + 2 * C, cf + 3 * C, y.data_ptr(),
                             has_mask ? mask->data_ptr<uint8_t>() : nullptr, M, C, G,
                             at::cuda::getCurrentCUDAStream()));
    return y;
}

// returns (partial[G][2][C], dz or undefined); mode 2 needs y and writes dz
static std::vector<torch::Tensor> bn_kernel_reduce(int mode, torch::Tensor dy, torch::Tensor x,
                                                   c10::optional<torch::Tensor> y, torch::Tensor coef, int G)
{
    long long M; int C;
    bn_kernel_args(x, coef, M, C);
    TORCH_CHECK(coef.size(0) >= 4 && mode >= 0 && mode <= 2);
    same_layout(dy, x);
    if (mode == 2) { TORCH_CHECK(y.has_value() && y->defined()); same_layout(*y, x); }
    c10::cuda::CUDAGuard guard(x.get_device());
    if (G <= 0) G = bn_partial_rows_bwd(M, C);
    auto partial = torch::empty({G, 2, C}, x.options().dtype(torch::kFloat32));
    torch::Tensor dz;
    if (mode == 2) dz = torch::empty_like(x);
    const float* cf = coef.data_ptr<float>();
    BN_CHECK(bn_launch_bwd_reduce(dtype_code(x), mode, dy.data_ptr(), x.data_ptr(),
                                  mode == 2 ? y->data_ptr() : nullptr, cf + 2 * C, cf + 3 * C, cf, cf + C,
                                  partial.data_ptr<float>(), mode == 2 ? dz.data_ptr() : nullptr, M, C, G,
                                  at::cuda::getCurrentCUDAStream()));
    return {partial, dz};
}

static torch::Tensor bn_kernel_dx(int mode, torch::Tensor dz, torch::Tensor x, torch::Tensor coef,
                                  torch::Tensor c23, int G)
{
    long long M; int C;
    bn_kernel_args(x, coef, M, C);
    bn_kernel_args(x, c23, M, C);
    TORCH_CHECK(coef.size(0) >= 4 && c23.size(0) == 2 && (mode == 0 || mode == 1));
    same_layout(dz, x);
    c10::cuda::CUDAGuard guard(x.get_device());
    auto dx = torch::empty_like(x);
    const float* cf = coef.data_ptr<float>();
    const float* k = c23.data_ptr<float>();
    BN_CHECK(bn_launch_bwd_dx(dtype_code(x), mode, dz.data_ptr(), x.data_ptr(), cf + 2 * C, cf + 3 * C, k, k + C,
                              dx.data_ptr(), M, C, G, at::cuda::getCurrentCUDAStream()));
    return dx;
}

// ---------------------------------------------------------------------------
// NHWC max-pool
// ---------------------------------------------------------------------------
extern "C" {
cudaError_t pool_launch_fwd(int dtype, const void* x, void* y, uint8_t* code, int N, int H, int W, int C,
                            int OH, int OW, int k, int s, int p, cudaStream_t st);
cudaError_t pool_launch_bwd(int dtype, const void* dy, const uint8_t* code, void* dx, int N, int H, int W,
                            int C, int OH, int OW, int k, int s, int p, cudaStream_t st);
}

static bool pool_can_fuse(const torch::Tensor& x, int k, int s, int p)
{
    return x.is_cuda() && x.dim() == 4 && x.is_contiguous(at::MemoryFormat::ChannelsLast)
        && (x.scalar_type() == torch::kBFloat16 || x.scalar_type() == torch::kFloat32)
        && x.size(1) % 8 == 0 && k >= 1 && k <= 11 && s >= 1 && p >= 0 && 2 * p <= k;
}

// returns (y, code)
static std::vector<torch::Tensor> maxpool_forward(torch::Tensor x, int k, int s, int p)
{
    TORCH_CHECK(pool_can_fuse(x, k, s, p));
    const int N = (int)x.size(0), C = (int)x.size(1), H = (int)x.size(2), W = (int)x.size(3);
    const int OH = (H + 2 * p - k) / s + 1, OW = (W + 2 * p - k) / s + 1;
    c10::cuda::CUDAGuard guard(x.get_device());
    auto y = torch::empty({N, C, OH, OW}, x.options().memory_format(at::MemoryFormat::ChannelsLast));
    auto code = torch::empty({N, OH, OW, C}, x.options().dtype(torch::kUInt8));
    BN_CHECK(pool_launch_fwd(dtype_code(x), x.data_ptr(), y.data_ptr(), code.data_ptr<uint8_t>(),
                             N, H, W, C, OH, OW, k, s, p, at::cuda::getCurrentCUDAStream()));
    return {y, code};
}

static torch::Tensor maxpool_backward(torch::Tensor dy, torch::Tensor code, int H, int W, int k, int s, int p)
{
    const int N = (int)dy.size(0), C = (int)dy.size(1), OH = (int)dy.size(2), OW = (int)dy.size(3);
    if (!dy.is_contiguous(at::MemoryFormat::ChannelsLast)) dy = dy.contiguous(at::MemoryFormat::ChannelsLast);
    c10::cuda::CUDAGuard guard(dy.get_device());
    auto dx = torch::empty({N, C, H, W}, dy.options().memory_format(at::MemoryFormat::ChannelsLast));
    BN_CHECK(pool_launch_bwd(dtype_code(dy), dy.data_ptr(), code.data_ptr<uint8_t>(), dx.data_ptr(),
                             N, H, W, C, OH, OW, k, s, p, at::cuda::getCurrentCUDAStream()));
    return dx;
}

// ---------------------------------------------------------------------------
// ResNet stem convolution (3 -> 64, 7x7 / 2, pad 3), NHWC bf16
// ---------------------------------------------------------------------------
extern "C" {
cudaError_t stem_launch_fwd(const void* x, const void* w, void* y, int N, int H, int W, int OH, int OW,
                            cudaStream_t st);
cudaError_t stem_launch_wgrad(const void* x, const void* dy, float* dw_acc, int N, int H, int W,
                              int OH, int OW, cudaStream_t st);
cudaError_t stem_launch_fwd_f32(const void* x, const void* w, void* y, int N, int H, int W, int OH, int OW,
                                cudaStream_t st);
cudaError_t stem_launch_wgrad_f32(const void* x, const void* dy, float* dw_acc, int N, int H, int W,
                                  int OH, int OW, cudaStream_t st);
}

static bool stem_can_fuse(const torch::Tensor& x, const torch::Tensor& w)
{
    // bf16 (mma.sync bf16) or fp32 operands (mma.sync TF32), same dtype for both
    return x.is_cuda() && x.dim() == 4 && x.size(1) == 3
        && (x.scalar_type() == torch::kBFloat16 || x.scalar_type() == torch::kFloat32)
        && x.is_contiguous(at::MemoryFormat::ChannelsLast)
        && w.dim() == 4 && w.size(0) == 64 && w.size(1) == 3 && w.size(2) == 7 && w.size(3) == 7
        && w.scalar_type() == x.scalar_type() && w.is_contiguous(at::MemoryFormat::ChannelsLast)
        && x.size(2) >= 7 && x.size(3) >= 7;
}

static torch::Tensor stem_forward(torch::Tensor x, torch::Tensor w)
{
    TORCH_CHECK(stem_can_fuse(x, w), "stem_forward: unsupported tensors");
    const int N = (int)x.size(0), H = (int)x.size(2), W = (int)x.size(3);
    const int OH = (H + 6 - 7) / 2 + 1, OW = (W + 6 - 7) / 2 + 1;
    c10::cuda::CUDAGuard guard(x.get_device());
    auto y = torch::empty({N, 64, OH, OW}, x.options().memory_format(at::MemoryFormat::ChannelsLast));
    if (x.scalar_type() == torch::kFloat32)
        BN_CHECK(stem_launch_fwd_f32(x.data_ptr(), w.data_ptr(), y.data_ptr(), N, H, W, OH, OW,
                                     at::cuda::getCurrentCUDAStream()));
    else
        BN_CHECK(stem_launch_fwd(x.data_ptr(), w.data_ptr(), y.data_ptr(), N, H, W, OH, OW,
                                 at::cuda::getCurrentCUDAStream()));
    return y;
}

// returns dW as an fp32 [64, 3, 7, 7] tensor in channels_last layout
static torch::Tensor stem_wgrad(torch::Tensor x, torch::Tensor dy)
{
    TORCH_CHECK((x.scalar_type() == torch::kBFloat16 || x.scalar_type() == torch::kFloat32) &&
                x.is_contiguous(at::MemoryFormat::ChannelsLast));
    TORCH_CHECK(dy.scalar_type() == x.scalar_type() && dy.size(1) == 64);
    if (!dy.is_contiguous(at::MemoryFormat::ChannelsLast)) dy = dy.contiguous(at::MemoryFormat::ChannelsLast);
    const int N = (int)x.size(0), H = (int)x.size(2), W = (int)x.size(3);
    const int OH = (int)dy.size(2), OW = (int)dy.size(3);
    c10::cuda::CUDAGuard guard(x.get_device());
    auto acc = torch::zeros({64, 7, 7, 3}, x.options().dtype(torch::kFloat32));
    if (x.scalar_type() == torch::kFloat32)
        BN_CHECK(stem_launch_wgrad_f32(x.data_ptr(), dy.data_ptr(), acc.data_ptr<float>(), N, H, W, OH, OW,
                                       at::cuda::getCurrentCUDAStream()));
    else
        BN_CHECK(stem_launch_wgrad(x.data_ptr(), dy.data_ptr(), acc.data_ptr<float>(), N, H, W, OH, OW,
                                   at::cuda::getCurrentCUDAStream()));
    return acc.permute({0, 3, 1, 2});
}

// ---------------------------------------------------------------------------
// 1x1 convolution as a wgmma GEMM, BatchNorm statistics fused into its epilogue
// (conv1x1_kernels.cu)
// ---------------------------------------------------------------------------
extern "C" {
int c1_supported(long long M, int N, int K, int f32);
int c1_partial_rows(long long M, int N, int K, int num_sms, int bn_reduce, int f32);
void c1_describe_plan(long long M, int N, int K, int num_sms, int residual, int bn_reduce, int f32, int* out);
cudaError_t c1_launch_gemm(const void* x, const void* w, void* y, long long M, int N, int K, float* partial,
                           const void* residual, const void* bn_x, const float* coef, const uint8_t* mask,
                           int num_sms, int f32, cudaStream_t st);
cudaError_t c1_launch_stats_finalize(const float* partial, int R, int C, const float* gamma, const float* beta,
                                     float* rmean, float* rvar, long long* nbt, double* acc, float momentum,
                                     float eps, float* mean, float* invstd, float* scale, float* shift,
                                     cudaStream_t st);
cudaError_t c1_launch_gemm_bn_eval(const void* x, const void* w, void* y, long long M, int N, int K,
                                   const void* residual, const float* gamma, const float* beta, const float* mean,
                                   const float* var, float eps, int relu, int num_sms, int f32, cudaStream_t st);
cudaError_t c1_launch_gemm_bn_reduce_drop(const void* x, const void* w, void* y, long long M, int N, int K,
                                          float* partial, const void* residual, const void* bn_x, const float* coef,
                                          const uint8_t* mask, const float* sdrop, int hw, int num_sms, int f32,
                                          cudaStream_t st);
}

// x: NHWC bf16 / fp32 activation (4-D channels_last) or [M, K] matrix; w: [N, K, 1, 1] or [N, K], rows
// contiguous, same dtype as x (fp32 operands are multiplied as TF32, fp32 accumulate)
static bool conv1x1_can_fuse(const torch::Tensor& x, const torch::Tensor& w)
{
    if (!x.is_cuda() || !w.is_cuda() || x.scalar_type() != w.scalar_type() ||
        (x.scalar_type() != torch::kBFloat16 && x.scalar_type() != torch::kFloat32))
        return false;
    if (x.dim() == 4) { if (!x.is_contiguous(at::MemoryFormat::ChannelsLast)) return false; }
    else if (!(x.dim() == 2 && x.is_contiguous())) return false;
    if (w.dim() == 4) { if (w.size(2) != 1 || w.size(3) != 1) return false; }
    else if (w.dim() != 2) return false;
    const int K = (int)x.size(1), N = (int)w.size(0);
    if (w.size(1) != K || w.stride(1) != 1 || w.stride(0) != K) return false;
    if ((reinterpret_cast<uintptr_t>(x.data_ptr()) | reinterpret_cast<uintptr_t>(w.data_ptr())) & 15) return false;
    return c1_supported(x.numel() / K, N, K, x.scalar_type() == torch::kFloat32) != 0;
}

static torch::Tensor conv1x1_alloc_out(const torch::Tensor& x, int N)
{
    if (x.dim() == 4)
        return torch::empty({x.size(0), N, x.size(2), x.size(3)},
                            x.options().memory_format(at::MemoryFormat::ChannelsLast));
    return torch::empty({x.size(0), N}, x.options());
}

// host-side launch plan of the GEMM for a shape (no GPU needed)
// (bn_reduce: the MODE 3 dgrad + BatchNorm backward reduction, which implies a residual)
static py::dict conv1x1_plan(long long M, int N, int K, int num_sms, bool residual, bool f32, bool bn_reduce)
{
    TORCH_CHECK(c1_supported(M, N, K, f32), "unsupported GEMM shape");
    int v[7];
    c1_describe_plan(M, N, K, num_sms, residual ? 1 : 0, bn_reduce ? 1 : 0, f32 ? 1 : 0, v);
    py::dict d;
    d["block_n"] = v[0]; d["grid"] = v[1]; d["ctas_per_n"] = v[2]; d["stages"] = v[3];
    d["resident_w"] = v[4] != 0; d["store_slabs"] = v[5]; d["smem_bytes"] = v[6];
    d["partial_rows"] = c1_partial_rows(M, N, K, num_sms, bn_reduce ? 1 : 0, f32 ? 1 : 0);
    return d;
}

static int sm_count() { return at::cuda::getCurrentDeviceProperties()->multiProcessorCount; }

// num_sms: the SM count the persistent grid is planned for; <= 0 is the device's own.  A smaller value
// gives every CTA more row tiles (tests of the cross-tile state reach it at small M).
static int plan_sms(int num_sms) { return num_sms > 0 ? num_sms : sm_count(); }

// y = x . w^T [+ residual] (residual: same shape / layout as y, added in fp32 in the epilogue).
// with_stats: also run the statistics epilogue into a scratch buffer (benchmarking the GEMM alone)
static torch::Tensor conv1x1_forward(torch::Tensor x, torch::Tensor w, bool with_stats,
                                     c10::optional<torch::Tensor> residual, int num_sms)
{
    TORCH_CHECK(conv1x1_can_fuse(x, w), "conv1x1_forward: unsupported tensors");
    const int K = (int)x.size(1), N = (int)w.size(0);
    const long long M = x.numel() / K;
    c10::cuda::CUDAGuard guard(x.get_device());
    auto y = conv1x1_alloc_out(x, N);
    const bool has_res = residual.has_value() && residual->defined();
    TORCH_CHECK(!(has_res && with_stats));
    const int f32 = x.scalar_type() == torch::kFloat32 ? 1 : 0;
    if (has_res)
        TORCH_CHECK(residual->is_cuda() && residual->scalar_type() == x.scalar_type() &&
                    residual->sizes() == y.sizes() && residual->strides() == y.strides() &&
                    (reinterpret_cast<uintptr_t>(residual->data_ptr()) & 15) == 0,
                    "conv1x1_forward: residual must match the output's shape and layout");
    const int sms = plan_sms(num_sms);
    torch::Tensor partial;
    if (with_stats)
        partial = torch::empty({c1_partial_rows(M, N, K, sms, 0, f32), 3, N},
                               torch::TensorOptions().dtype(torch::kFloat32).device(x.device()));
    BN_CHECK(c1_launch_gemm(x.data_ptr(), w.data_ptr(), y.data_ptr(), M, N, K,
                            with_stats ? partial.data_ptr<float>() : nullptr,
                            has_res ? residual->data_ptr() : nullptr, nullptr, nullptr, nullptr, sms, f32,
                            at::cuda::getCurrentCUDAStream()));
    return y;
}

// MODE 3: dz = mask ? x . w^T + residual : 0 and the backward reduction of the BatchNorm (+ residual
// + ReLU) whose input was bn_x, output mask `mask` ([M, N/8] uint8) and coefficients `coef` ([4, N]:
// mean, invstd, scale, shift).  Returns (dz, partial[R][2][N]) for bn_backward_from_partials.
// branch_scale: that BatchNorm's stochastic-depth scale (bn_forward); the partials are then those of s * dz
static std::vector<torch::Tensor> conv1x1_dgrad_bn_reduce(torch::Tensor x, torch::Tensor w, torch::Tensor residual,
                                                          torch::Tensor bn_x, torch::Tensor coef, torch::Tensor mask,
                                                          int num_sms, c10::optional<torch::Tensor> branch_scale)
{
    TORCH_CHECK(conv1x1_can_fuse(x, w), "conv1x1_dgrad_bn_reduce: unsupported tensors");
    const int K = (int)x.size(1), N = (int)w.size(0);
    const long long M = x.numel() / K;
    c10::cuda::CUDAGuard guard(x.get_device());
    auto y = conv1x1_alloc_out(x, N);
    for (const torch::Tensor* t : {&residual, &bn_x})
        TORCH_CHECK(t->is_cuda() && t->scalar_type() == x.scalar_type() && t->sizes() == y.sizes() &&
                    t->strides() == y.strides() && (reinterpret_cast<uintptr_t>(t->data_ptr()) & 15) == 0,
                    "conv1x1_dgrad_bn_reduce: residual / bn_x must match the output's shape and layout");
    TORCH_CHECK(coef.is_cuda() && coef.scalar_type() == torch::kFloat32 && coef.is_contiguous() &&
                coef.dim() == 2 && coef.size(1) == N && coef.size(0) >= 2);
    TORCH_CHECK(mask.is_cuda() && mask.scalar_type() == torch::kUInt8 && mask.is_contiguous() &&
                mask.numel() == M * (N / 8) && (reinterpret_cast<uintptr_t>(mask.data_ptr()) & 15) == 0,
                "conv1x1_dgrad_bn_reduce: mask must be [M, N/8] uint8");
    const int f32 = x.scalar_type() == torch::kFloat32 ? 1 : 0;
    const int sms = plan_sms(num_sms);
    auto partial = torch::empty({c1_partial_rows(M, N, K, sms, 1, f32), 2, N},
                                torch::TensorOptions().dtype(torch::kFloat32).device(x.device()));
    int hw;
    const float* sdrop = branch_scale_ptr(branch_scale, y, M, hw);
    if (sdrop != nullptr)
        BN_CHECK(c1_launch_gemm_bn_reduce_drop(x.data_ptr(), w.data_ptr(), y.data_ptr(), M, N, K,
                                               partial.data_ptr<float>(), residual.data_ptr(), bn_x.data_ptr(),
                                               coef.data_ptr<float>(), mask.data_ptr<uint8_t>(), sdrop, hw, sms, f32,
                                               at::cuda::getCurrentCUDAStream()));
    else
        BN_CHECK(c1_launch_gemm(x.data_ptr(), w.data_ptr(), y.data_ptr(), M, N, K, partial.data_ptr<float>(),
                                residual.data_ptr(), bn_x.data_ptr(), coef.data_ptr<float>(), mask.data_ptr<uint8_t>(),
                                sms, f32, at::cuda::getCurrentCUDAStream()));
    return {y, partial};
}

// training-mode  out = act(bn(conv1x1(x, w)) [+ residual]);  returns (conv output, out, coef).
// mask (optional, residual + relu only): filled with out's 1-bit ReLU mask, [M, N/8] uint8
// acc (optional): accumulate mode of the statistics finalize, as in bn_forward
static std::vector<torch::Tensor> conv1x1_bn_forward(torch::Tensor x, torch::Tensor w,
                                                     c10::optional<torch::Tensor> residual,
                                                     torch::Tensor gamma, torch::Tensor beta,
                                                     c10::optional<torch::Tensor> running_mean,
                                                     c10::optional<torch::Tensor> running_var,
                                                     c10::optional<torch::Tensor> num_batches_tracked,
                                                     double momentum, double eps, bool relu,
                                                     c10::optional<torch::Tensor> mask, int num_sms,
                                                     c10::optional<torch::Tensor> acc,
                                                     c10::optional<torch::Tensor> branch_scale)
{
    TORCH_CHECK(conv1x1_can_fuse(x, w), "conv1x1_bn_forward: unsupported tensors");
    const int K = (int)x.size(1), N = (int)w.size(0);
    const long long M = x.numel() / K;
    TORCH_CHECK(bn_supported(M, N), "unsupported channel count ", N);
    TORCH_CHECK(gamma.scalar_type() == torch::kFloat32 && beta.scalar_type() == torch::kFloat32);
    c10::cuda::CUDAGuard guard(x.get_device());
    auto st = at::cuda::getCurrentCUDAStream();
    auto fopt = torch::TensorOptions().dtype(torch::kFloat32).device(x.device());
    auto yraw = conv1x1_alloc_out(x, N);
    const bool has_res = residual.has_value() && residual->defined();
    if (has_res) TORCH_CHECK(residual->sizes() == yraw.sizes() && residual->scalar_type() == yraw.scalar_type()
                             && residual->strides() == yraw.strides());
    const int sms = plan_sms(num_sms);
    const int f32 = x.scalar_type() == torch::kFloat32 ? 1 : 0;
    const bool has_mask = mask.has_value() && mask->defined();
    if (has_mask)
        TORCH_CHECK(has_res && relu && mask->is_cuda() && mask->scalar_type() == torch::kUInt8 &&
                    mask->is_contiguous() && mask->numel() == M * (N / 8),
                    "conv1x1_bn_forward: mask must be [M, N/8] uint8 (residual + relu only)");
    double* accp = bn_acc_ptr(acc, x, N);
    const int R = c1_partial_rows(M, N, K, sms, 0, f32);
    auto partial = torch::empty({R, 3, N}, fopt);
    BN_CHECK(c1_launch_gemm(x.data_ptr(), w.data_ptr(), yraw.data_ptr(), M, N, K, partial.data_ptr<float>(),
                            nullptr, nullptr, nullptr, nullptr, sms, f32, st));
    auto coef = torch::empty({4, N}, fopt);      // mean, invstd, scale, shift
    float* mean = coef.data_ptr<float>();
    float* rm = nullptr; float* rv = nullptr; long long* nbt = nullptr;
    if (running_mean.has_value() && running_mean->defined()) {
        rm = running_mean->data_ptr<float>();
        rv = running_var->data_ptr<float>();
    }
    if (num_batches_tracked.has_value() && num_batches_tracked->defined())
        nbt = reinterpret_cast<long long*>(num_batches_tracked->data_ptr<int64_t>());
    BN_CHECK(c1_launch_stats_finalize(partial.data_ptr<float>(), R, N, gamma.data_ptr<float>(),
                                      beta.data_ptr<float>(), rm, rv, nbt, accp, (float)momentum, (float)eps,
                                      mean, mean + N, mean + 2 * N, mean + 3 * N, st));
    auto out = torch::empty_like(yraw);
    int hw;
    const float* sdrop = branch_scale_ptr(branch_scale, yraw, M, hw);
    if (sdrop != nullptr) {
        TORCH_CHECK(has_res && relu, "conv1x1_bn_forward: branch_scale needs a residual and relu");
        BN_CHECK(bn_launch_apply_drop(f32, yraw.data_ptr(), residual->data_ptr(), mean + 2 * N, mean + 3 * N,
                                      out.data_ptr(), has_mask ? mask->data_ptr<uint8_t>() : nullptr, sdrop, hw, M, N,
                                      0, st));
        return {yraw, out, coef};
    }
    BN_CHECK(bn_launch_apply(f32, relu ? 1 : 0, has_res ? 1 : 0, yraw.data_ptr(),
                             has_res ? residual->data_ptr() : nullptr, mean + 2 * N, mean + 3 * N,
                             out.data_ptr(), has_mask ? mask->data_ptr<uint8_t>() : nullptr, M, N, 0, st));
    return {yraw, out, coef};
}

// eval-mode  out = act(bn(conv1x1(x, w)) [+ residual]) with the running statistics, in ONE launch: the
// BatchNorm affine map (from gamma, beta, mean, var as they are at launch time), the residual add and the
// ReLU run in the GEMM epilogue (MODES 4 / 5).  Nothing is updated.
static torch::Tensor conv1x1_bn_eval(torch::Tensor x, torch::Tensor w, torch::Tensor gamma, torch::Tensor beta,
                                     torch::Tensor mean, torch::Tensor var, double eps, bool relu,
                                     c10::optional<torch::Tensor> residual, int num_sms)
{
    TORCH_CHECK(conv1x1_can_fuse(x, w), "conv1x1_bn_eval: unsupported tensors");
    const int K = (int)x.size(1), N = (int)w.size(0);
    const long long M = x.numel() / K;
    for (const torch::Tensor* t : {&gamma, &beta, &mean, &var})
        TORCH_CHECK(t->is_cuda() && t->get_device() == x.get_device() && t->scalar_type() == torch::kFloat32 &&
                        t->is_contiguous() && t->numel() == N,
                    "conv1x1_bn_eval: gamma, beta, mean and var must be contiguous fp32 [N] tensors on x's device");
    c10::cuda::CUDAGuard guard(x.get_device());
    auto y = conv1x1_alloc_out(x, N);
    const bool has_res = residual.has_value() && residual->defined();
    if (has_res)
        TORCH_CHECK(residual->is_cuda() && residual->scalar_type() == x.scalar_type() &&
                        residual->sizes() == y.sizes() && residual->strides() == y.strides() &&
                        (reinterpret_cast<uintptr_t>(residual->data_ptr()) & 15) == 0,
                    "conv1x1_bn_eval: residual must match the output's shape and layout");
    BN_CHECK(c1_launch_gemm_bn_eval(x.data_ptr(), w.data_ptr(), y.data_ptr(), M, N, K,
                                    has_res ? residual->data_ptr() : nullptr, gamma.data_ptr<float>(),
                                    beta.data_ptr<float>(), mean.data_ptr<float>(), var.data_ptr<float>(), (float)eps,
                                    relu ? 1 : 0, plan_sms(num_sms), x.scalar_type() == torch::kFloat32 ? 1 : 0,
                                    at::cuda::getCurrentCUDAStream()));
    return y;
}

// ---------------------------------------------------------------------------
// fused softmax cross-entropy + top-1 / top-5 accuracy (csrc/loss_kernels.cu)
// ---------------------------------------------------------------------------
extern "C" {
cudaError_t xent_launch_fwd(int dtype, const void* logits, const long long* target, float* lse, float* out3, int B,
                            int C, float eps, const float* mix, cudaStream_t st);
cudaError_t xent_launch_eval(int dtype, const void* logits, const long long* target, unsigned long long* acc, int B,
                             int C, cudaStream_t st);
cudaError_t xent_launch_bwd(int dtype, const void* logits, const long long* target, const float* lse,
                            const float* grad_out, void* dlogits, int B, int C, float eps, const float* mix,
                            cudaStream_t st);
cudaError_t batch_mix_launch(int out_dtype, const float* src, void* dst, const float* mix, int B, int C, int H,
                             int W, long long s_n, int s_c, int s_p, long long d_n, int d_c, int d_p,
                             cudaStream_t st);
}

// torch.nn.functional.cross_entropy accepts label_smoothing in [0, 1]; so do the kernels
static float xent_check_smoothing(double label_smoothing)
{
    TORCH_CHECK(label_smoothing >= 0.0 && label_smoothing <= 1.0, "label_smoothing must be in [0, 1]");
    return (float)label_smoothing;
}

static bool xent_can_fuse(const torch::Tensor& logits, const torch::Tensor& target)
{
    return logits.is_cuda() && target.is_cuda() && logits.dim() == 2 && logits.is_contiguous() &&
           (logits.scalar_type() == torch::kFloat32 || logits.scalar_type() == torch::kBFloat16) &&
           target.dim() == 1 && target.scalar_type() == torch::kInt64 && target.is_contiguous() &&
           target.size(0) == logits.size(0) && logits.size(0) > 0 && logits.size(1) > 0;
}

// mixup / CutMix state (ops/batch_mix.py): fp32 [lam, mode, y0, y1, x0, x1] on the logits' device;
// None = one target per row (the MIX = false kernels)
static const float* xent_mix_ptr(const c10::optional<torch::Tensor>& mix, const torch::Tensor& logits)
{
    if (!mix.has_value() || !mix->defined()) return nullptr;
    TORCH_CHECK(mix->is_cuda() && mix->get_device() == logits.get_device() && mix->scalar_type() == torch::kFloat32 &&
                    mix->is_contiguous() && mix->numel() >= 6,
                "mix must be the fp32 device mix state [lam, mode, y0, y1, x0, x1] on the logits' device");
    return mix->data_ptr<float>();
}

// returns (metrics[3] = mean loss (label-smoothed when label_smoothing > 0), prec@1 %, prec@5 %; lse[B]);
// with mix: the two-target loss lam CE(z_i, t_i) + (1 - lam) CE(z_i, t_{B-1-i})
static std::vector<torch::Tensor> xent_forward(torch::Tensor logits, torch::Tensor target, double label_smoothing,
                                               c10::optional<torch::Tensor> mix)
{
    TORCH_CHECK(xent_can_fuse(logits, target), "xent_forward: unsupported tensors");
    const float eps = xent_check_smoothing(label_smoothing);
    const float* mixp = xent_mix_ptr(mix, logits);
    c10::cuda::CUDAGuard guard(logits.get_device());
    auto st = at::cuda::getCurrentCUDAStream();
    auto fopt = torch::TensorOptions().dtype(torch::kFloat32).device(logits.device());
    const int B = (int)logits.size(0), C = (int)logits.size(1);
    auto out3 = torch::empty({3}, fopt);
    auto lse = torch::empty({B}, fopt);
    BN_CHECK(cudaMemsetAsync(out3.data_ptr(), 0, 3 * sizeof(float), st));
    BN_CHECK(xent_launch_fwd(dtype_code(logits), logits.data_ptr(),
                             reinterpret_cast<const long long*>(target.data_ptr<int64_t>()),
                             lse.data_ptr<float>(), out3.data_ptr<float>(), B, C, eps, mixp, st));
    return {out3, lse};
}

static torch::Tensor xent_backward(torch::Tensor logits, torch::Tensor target, torch::Tensor lse,
                                   torch::Tensor grad_out, double label_smoothing, c10::optional<torch::Tensor> mix)
{
    TORCH_CHECK(xent_can_fuse(logits, target) && lse.is_cuda() && lse.scalar_type() == torch::kFloat32 &&
                grad_out.is_cuda() && grad_out.scalar_type() == torch::kFloat32 && grad_out.numel() == 1);
    const float eps = xent_check_smoothing(label_smoothing);
    const float* mixp = xent_mix_ptr(mix, logits);
    c10::cuda::CUDAGuard guard(logits.get_device());
    auto dl = torch::empty_like(logits);
    BN_CHECK(xent_launch_bwd(dtype_code(logits), logits.data_ptr(),
                             reinterpret_cast<const long long*>(target.data_ptr<int64_t>()), lse.data_ptr<float>(),
                             grad_out.data_ptr<float>(), dl.data_ptr(), (int)logits.size(0), (int)logits.size(1), eps,
                             mixp, at::cuda::getCurrentCUDAStream()));
    return dl;
}

// evaluation: adds the plain cross-entropy sum and the top-1 / top-5 / valid-row counts of this batch to acc,
// an int64 [4] device tensor: [loss sum as fp64 bits, top-1 hits, top-5 hits, rows with a target in [0, C)]
static void xent_eval_accumulate(torch::Tensor logits, torch::Tensor target, torch::Tensor acc)
{
    TORCH_CHECK(xent_can_fuse(logits, target), "xent_eval_accumulate: unsupported tensors");
    TORCH_CHECK(acc.is_cuda() && acc.get_device() == logits.get_device() && acc.scalar_type() == torch::kInt64 &&
                    acc.is_contiguous() && acc.numel() == 4,
                "xent_eval_accumulate: acc must be a contiguous int64 [4] tensor on the logits' device");
    c10::cuda::CUDAGuard guard(logits.get_device());
    BN_CHECK(xent_launch_eval(dtype_code(logits), logits.data_ptr(),
                              reinterpret_cast<const long long*>(target.data_ptr<int64_t>()),
                              reinterpret_cast<unsigned long long*>(acc.data_ptr<int64_t>()), (int)logits.size(0),
                              (int)logits.size(1), at::cuda::getCurrentCUDAStream()));
}

// ---------------------------------------------------------------------------
// mixup / CutMix inside the stage -> static input copy (csrc/mix_kernels.cu)
// ---------------------------------------------------------------------------
// NCHW or NHWC dense: pixel (h, w) at h * W * sp + w * sp
static bool mix_layout_ok(const torch::Tensor& t)
{
    return t.dim() == 4 && (t.is_contiguous() || t.is_contiguous(at::MemoryFormat::ChannelsLast));
}

// out <- src with row i mixed with row B-1-i as the device mix state says (mode 0 = plain copy)
static void batch_mix(torch::Tensor src, torch::Tensor out, torch::Tensor mix)
{
    TORCH_CHECK(src.is_cuda() && src.scalar_type() == torch::kFloat32 && mix_layout_ok(src),
                "batch_mix: src must be a 4-d NCHW or NHWC fp32 CUDA tensor");
    TORCH_CHECK(out.is_cuda() && out.get_device() == src.get_device() &&
                    (out.scalar_type() == torch::kFloat32 || out.scalar_type() == torch::kBFloat16) &&
                    mix_layout_ok(out) && out.sizes() == src.sizes(),
                "batch_mix: out must be a 4-d NCHW or NHWC fp32 / bf16 tensor of src's shape on its device");
    TORCH_CHECK(mix.is_cuda() && mix.get_device() == src.get_device() && mix.scalar_type() == torch::kFloat32 &&
                    mix.is_contiguous() && mix.numel() >= 6,
                "batch_mix: mix must be the fp32 device mix state [lam, mode, y0, y1, x0, x1]");
    const long long B = src.size(0), C = src.size(1), H = src.size(2), W = src.size(3);
    TORCH_CHECK(C * H * W < (1LL << 31), "batch_mix: one image must have fewer than 2^31 elements");
    const char* s0 = (const char*)src.data_ptr();
    const char* o0 = (const char*)out.data_ptr();
    TORCH_CHECK(o0 + out.nbytes() <= s0 || s0 + src.nbytes() <= o0, "batch_mix: src and out must not overlap");
    if (B == 0 || H * W == 0 || C == 0) return;
    c10::cuda::CUDAGuard guard(src.get_device());
    BN_CHECK(batch_mix_launch(dtype_code(out), src.data_ptr<float>(), out.data_ptr(), mix.data_ptr<float>(), (int)B,
                              (int)C, (int)H, (int)W, src.stride(0), (int)src.stride(1), (int)src.stride(3),
                              out.stride(0), (int)out.stride(1), (int)out.stride(3),
                              at::cuda::getCurrentCUDAStream()));
}

// ---------------------------------------------------------------------------
// stochastic depth: the per-sample residual-branch scales of one training forward (csrc/drop_path_kernels.cu)
// ---------------------------------------------------------------------------
// returns a fresh fp32 [L, n] tensor on counter's device; thresh[l] in [0, 2^24] and keep_scale[l] per block;
// counter: a contiguous int64 [1] CUDA tensor, read and incremented by the launch
static torch::Tensor drop_path_draw(torch::Tensor counter, int64_t seed, int64_t rank,
                                    const std::vector<int64_t>& thresh, const std::vector<double>& keep_scale,
                                    int64_t n)
{
    TORCH_CHECK(counter.is_cuda() && counter.scalar_type() == torch::kInt64 && counter.is_contiguous() &&
                    counter.numel() == 1,
                "drop_path_draw: counter must be a contiguous int64 [1] CUDA tensor");
    const int64_t L = (int64_t)thresh.size();
    TORCH_CHECK(L >= 1 && L <= drop_path_max_blocks() && (int64_t)keep_scale.size() == L,
                "drop_path_draw: thresh and keep_scale must have the same length, 1 to ", drop_path_max_blocks());
    TORCH_CHECK(n >= 1 && L * n < (1LL << 31), "drop_path_draw: bad sample count ", n);
    std::vector<unsigned int> th((size_t)L);
    std::vector<float> ks((size_t)L);
    for (int64_t l = 0; l < L; ++l) {
        TORCH_CHECK(thresh[l] >= 0 && thresh[l] <= (1LL << 24), "drop_path_draw: thresh must be in [0, 2^24]");
        th[l] = (unsigned int)thresh[l];
        ks[l] = (float)keep_scale[l];
    }
    c10::cuda::CUDAGuard guard(counter.get_device());
    auto out = torch::empty({L, n}, counter.options().dtype(torch::kFloat32));
    BN_CHECK(drop_path_launch_draw(th.data(), ks.data(), (int)L, (int)n, (unsigned long long)seed,
                                   (unsigned long long)rank, reinterpret_cast<long long*>(counter.data_ptr<int64_t>()),
                                   out.data_ptr<float>(), at::cuda::getCurrentCUDAStream()));
    return out;
}

void bind_bn(py::module& mod)
{
    mod.def("drop_path_draw", &drop_path_draw, py::arg("counter"), py::arg("seed"), py::arg("rank"),
            py::arg("thresh"), py::arg("keep_scale"), py::arg("n"));
    mod.attr("DROP_PATH_MAX_BLOCKS") = drop_path_max_blocks();
    mod.def("xent_can_fuse", &xent_can_fuse);
    mod.def("xent_forward", &xent_forward, py::arg("logits"), py::arg("target"), py::arg("label_smoothing") = 0.0,
            py::arg("mix") = py::none());
    mod.def("xent_backward", &xent_backward, py::arg("logits"), py::arg("target"), py::arg("lse"),
            py::arg("grad_out"), py::arg("label_smoothing") = 0.0, py::arg("mix") = py::none());
    mod.def("xent_eval_accumulate", &xent_eval_accumulate, py::arg("logits"), py::arg("target"), py::arg("acc"));
    mod.def("batch_mix", &batch_mix, py::arg("src"), py::arg("out"), py::arg("mix"));
    mod.def("conv1x1_can_fuse", &conv1x1_can_fuse);
    mod.def("conv1x1_plan", &conv1x1_plan, py::arg("M"), py::arg("N"), py::arg("K"), py::arg("num_sms") = 132,
            py::arg("residual") = false, py::arg("f32") = false, py::arg("bn_reduce") = false);
    mod.def("conv1x1_forward", &conv1x1_forward, py::arg("x"), py::arg("w"), py::arg("with_stats") = false,
            py::arg("residual") = py::none(), py::kw_only(), py::arg("num_sms") = 0);
    mod.def("conv1x1_bn_forward", &conv1x1_bn_forward, py::arg("x"), py::arg("w"), py::arg("residual"),
            py::arg("gamma"), py::arg("beta"), py::arg("running_mean"), py::arg("running_var"),
            py::arg("num_batches_tracked"), py::arg("momentum"), py::arg("eps"), py::arg("relu"),
            py::arg("mask") = py::none(), py::kw_only(), py::arg("num_sms") = 0, py::arg("acc") = py::none(),
            py::arg("branch_scale") = py::none());
    mod.def("conv1x1_dgrad_bn_reduce", &conv1x1_dgrad_bn_reduce, py::arg("x"), py::arg("w"), py::arg("residual"),
            py::arg("bn_x"), py::arg("coef"), py::arg("mask"), py::kw_only(), py::arg("num_sms") = 0,
            py::arg("branch_scale") = py::none());
    mod.def("conv1x1_bn_eval", &conv1x1_bn_eval, py::arg("x"), py::arg("w"), py::arg("gamma"), py::arg("beta"),
            py::arg("mean"), py::arg("var"), py::arg("eps"), py::arg("relu"), py::arg("residual") = py::none(),
            py::kw_only(), py::arg("num_sms") = 0);
    mod.def("stem_can_fuse", &stem_can_fuse);
    mod.def("stem_forward", &stem_forward);
    mod.def("stem_wgrad", &stem_wgrad);
    mod.def("pool_can_fuse", &pool_can_fuse);
    mod.def("maxpool_forward", &maxpool_forward);
    mod.def("maxpool_backward", &maxpool_backward);
    mod.def("bn_can_fuse", &bn_can_fuse);
    mod.def("bn_forward", &bn_forward, py::arg("x"), py::arg("residual"), py::arg("gamma"), py::arg("beta"),
            py::arg("running_mean"), py::arg("running_var"), py::arg("num_batches_tracked"), py::arg("training"),
            py::arg("momentum"), py::arg("eps"), py::arg("relu"), py::arg("acc") = py::none(),
            py::arg("branch_scale") = py::none());
    mod.def("bn_stats_commit", &bn_stats_commit, py::arg("acc"), py::arg("running_mean"), py::arg("running_var"),
            py::arg("k"), "running = fp32(acc / k) for every BatchNorm layer: one launch per BN_COMMIT_MAX_SEGS layers");
    mod.attr("BN_COMMIT_MAX_SEGS") = bn_commit_max_segs();
    mod.def("bn_backward", &bn_backward, py::arg("dy"), py::arg("x"), py::arg("y"), py::arg("coef"), py::arg("relu"),
            py::arg("add"), py::arg("branch_scale") = py::none());
    mod.def("bn_backward_from_partials", &bn_backward_from_partials, py::arg("dz"), py::arg("x"), py::arg("coef"),
            py::arg("partial"), py::arg("branch_scale") = py::none());
    mod.def("bn_f32_map", &bn_f32_map, py::arg("value") = -1,
            "fp32 BatchNorm channel map: returns the one in use (1 = split, 0 = consecutive); "
            "value >= 0 selects one for the launches that follow");
    mod.def("bn_kernel_stats", &bn_kernel_stats, py::arg("x"), py::arg("G") = 0);
    mod.def("bn_kernel_apply", &bn_kernel_apply, py::arg("x"), py::arg("residual"), py::arg("coef"),
            py::arg("relu"), py::arg("mask") = py::none(), py::arg("G") = 0);
    mod.def("bn_kernel_reduce", &bn_kernel_reduce, py::arg("mode"), py::arg("dy"), py::arg("x"), py::arg("y"),
            py::arg("coef"), py::arg("G") = 0);
    mod.def("bn_kernel_dx", &bn_kernel_dx, py::arg("mode"), py::arg("dz"), py::arg("x"), py::arg("coef"),
            py::arg("c23"), py::arg("G") = 0);
}
