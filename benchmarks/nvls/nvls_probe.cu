// NVLS feasibility probe: ONE process, all visible GPUs.  Creates a multicast object over the
// devices (cuMulticastCreate / AddDevice / BindMem), maps unicast + multicast views, then checks
// multimem.ld_reduce (in-switch sum) and multimem.st (in-switch broadcast) from a kernel, and
// whether the handles can be exported as POSIX file descriptors (what the multi-process
// rendezvous needs).   nvcc -arch=sm_90a -o nvls_probe nvls_probe.cu -lcuda
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <vector>

#define CK(x) do { CUresult r_ = (x); if (r_ != CUDA_SUCCESS) { const char* s_ = nullptr; cuGetErrorString(r_, &s_); \
    printf("FAIL %s -> %d (%s)\n", #x, (int)r_, s_ ? s_ : "?"); return 1; } } while (0)

__global__ void fill(float* p, float v, size_t n) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = v + (float)(i & 7);
}
__global__ void mc_reduce(const float* mc, float* out, size_t n4) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
        float4 v;
        asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                     : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(mc + 4 * i) : "memory");
        reinterpret_cast<float4*>(out)[i] = v;
    }
}
__global__ void mc_store(float* mc, float v, size_t n4) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x)
        asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};"
                     :: "l"(mc + 4 * i), "f"(v), "f"(v + 1.f), "f"(v + 2.f), "f"(v + 3.f) : "memory");
}

int main() {
    CK(cuInit(0));
    int ndev = 0;
    CK(cuDeviceGetCount(&ndev));
    printf("devices: %d\n", ndev);
    if (ndev < 2) { printf("need >= 2 GPUs\n"); return 0; }
    std::vector<CUdevice> dev(ndev);
    for (int d = 0; d < ndev; ++d) {
        CK(cuDeviceGet(&dev[d], d));
        int mc = 0, fab = 0, posix = 0;
        cuDeviceGetAttribute(&mc, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, dev[d]);
        cuDeviceGetAttribute(&fab, CU_DEVICE_ATTRIBUTE_HANDLE_TYPE_FABRIC_SUPPORTED, dev[d]);
        cuDeviceGetAttribute(&posix, CU_DEVICE_ATTRIBUTE_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR_SUPPORTED, dev[d]);
        printf("dev %d: multicast_supported=%d fabric_handles=%d posix_fd_handles=%d\n", d, mc, fab, posix);
        cudaSetDevice(d);
        cudaFree(0);
        for (int p = 0; p < ndev; ++p) if (p != d) cudaDeviceEnablePeerAccess(p, 0);
    }
    const size_t want = 64ull << 20;
    CUmulticastObjectProp mprop = {};
    mprop.numDevices = (unsigned)ndev;
    mprop.size = want;
    mprop.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    size_t gran = 0;
    CK(cuMulticastGetGranularity(&gran, &mprop, CU_MULTICAST_GRANULARITY_RECOMMENDED));
    const size_t size = (want + gran - 1) / gran * gran;
    mprop.size = size;
    printf("multicast granularity %zu, size %zu\n", gran, size);
    CUmemGenericAllocationHandle mc;
    CK(cuMulticastCreate(&mc, &mprop));
    for (int d = 0; d < ndev; ++d) CK(cuMulticastAddDevice(mc, dev[d]));
    int fd = -1;
    CUresult er = cuMemExportToShareableHandle(&fd, mc, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0);
    printf("export multicast object as POSIX fd: rc=%d fd=%d\n", (int)er, fd);

    std::vector<CUmemGenericAllocationHandle> mem(ndev);
    std::vector<CUdeviceptr> uc(ndev), mcva(ndev);
    for (int d = 0; d < ndev; ++d) {
        CUmemAllocationProp ap = {};
        ap.type = CU_MEM_ALLOCATION_TYPE_PINNED;
        ap.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
        ap.location.id = d;
        ap.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
        size_t ag = 0;
        CK(cuMemGetAllocationGranularity(&ag, &ap, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED));
        if (d == 0) printf("alloc granularity %zu\n", ag);
        CK(cuMemCreate(&mem[d], size, &ap, 0));
        int mfd = -1;
        er = cuMemExportToShareableHandle(&mfd, mem[d], CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0);
        if (d == 0) printf("export memory handle as POSIX fd: rc=%d fd=%d\n", (int)er, mfd);
        CK(cuMulticastBindMem(mc, 0, mem[d], 0, size, 0));
        CK(cuMemAddressReserve(&uc[d], size, gran, 0, 0));
        CK(cuMemMap(uc[d], size, 0, mem[d], 0));
        std::vector<CUmemAccessDesc> acc(ndev);
        for (int p = 0; p < ndev; ++p) { acc[p].location.type = CU_MEM_LOCATION_TYPE_DEVICE; acc[p].location.id = p; acc[p].flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE; }
        CK(cuMemSetAccess(uc[d], size, acc.data(), ndev));
    }
    // one multicast VA (the mapping is per process; every device of the process gets access)
    CUdeviceptr mva;
    CK(cuMemAddressReserve(&mva, size, gran, 0, 0));
    CK(cuMemMap(mva, size, 0, mc, 0));
    {
        std::vector<CUmemAccessDesc> acc(ndev);
        for (int p = 0; p < ndev; ++p) { acc[p].location.type = CU_MEM_LOCATION_TYPE_DEVICE; acc[p].location.id = p; acc[p].flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE; }
        CK(cuMemSetAccess(mva, size, acc.data(), ndev));
    }
    const size_t n = size / 4;
    for (int d = 0; d < ndev; ++d) { cudaSetDevice(d); fill<<<296, 256>>>((float*)uc[d], 1.0f + d, n); cudaDeviceSynchronize(); }
    cudaSetDevice(0);
    float* out = nullptr;
    cudaMalloc(&out, size);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    mc_reduce<<<296, 256>>>((const float*)mva, out, n / 4);
    cudaError_t ce = cudaDeviceSynchronize();
    printf("multimem.ld_reduce kernel: %s\n", cudaGetErrorString(ce));
    if (ce != cudaSuccess) return 1;
    float h[8];
    cudaMemcpy(h, out, sizeof(h), cudaMemcpyDeviceToHost);
    float expect0 = 0.f;
    for (int d = 0; d < ndev; ++d) expect0 += 1.0f + d;
    printf("ld_reduce[0..3] = %.1f %.1f %.1f %.1f (expect %.1f %.1f ...)\n", h[0], h[1], h[2], h[3], expect0, expect0 + ndev);
    for (int it = 0; it < 3; ++it) {
        cudaEventRecord(e0);
        mc_reduce<<<296, 256>>>((const float*)mva, out, n / 4);
        cudaEventRecord(e1);
        cudaDeviceSynchronize();
        float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
        printf("ld_reduce %zu MB over %d GPUs: %.3f ms -> %.1f GB/s of reduced output\n", size >> 20, ndev, ms, size / ms / 1e6);
    }
    mc_store<<<296, 256>>>((float*)mva, 42.f, n / 4);
    ce = cudaDeviceSynchronize();
    printf("multimem.st kernel: %s\n", cudaGetErrorString(ce));
    for (int d = 0; d < ndev; ++d) {
        cudaSetDevice(d);
        cudaDeviceSynchronize();
        cudaMemcpy(h, (void*)uc[d], sizeof(h), cudaMemcpyDeviceToHost);
        printf("after multimem.st, dev %d sees %.1f %.1f %.1f %.1f\n", d, h[0], h[1], h[2], h[3]);
    }
    cudaSetDevice(0);
    for (int it = 0; it < 3; ++it) {
        cudaEventRecord(e0);
        mc_store<<<296, 256>>>((float*)mva, 1.f, n / 4);
        cudaEventRecord(e1);
        cudaDeviceSynchronize();
        float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
        printf("multimem.st %zu MB to %d GPUs: %.3f ms -> %.1f GB/s\n", size >> 20, ndev, ms, size / ms / 1e6);
    }
    printf("NVLS PROBE OK\n");
    return 0;
}
