// Symmetric memory through the CUDA virtual-memory-management API, with an NVSwitch MULTICAST view.
//
// The cudaMalloc + cudaIpc* rendezvous of bindings.cpp::symm_alloc cannot host a multicast object
// (VERDICT r1).  This allocator does what NVLS needs:
//
//   every rank   cuMemCreate (POSIX-fd exportable physical memory on its GPU), map it
//   exchange     the POSIX fds are passed between the ranks' processes over abstract unix-domain
//                sockets (SCM_RIGHTS; `FdChannel` below -- pidfd_getfd is refused with EPERM inside
//                containers), then
//                cuMemImportFromShareableHandle'd; no fabric handles / IMEX daemon needed
//   unicast      every peer's allocation is mapped (cuMemAddressReserve / cuMemMap / cuMemSetAccess):
//                plain P2P loads / stores / cp.async.bulk over NVLink work as before
//   multicast    symmetric rank 0 creates the multicast object (cuMulticastCreate), everyone adds
//                its device and binds its physical memory (cuMulticastBindMem), then maps the
//                object: stores to that address land in EVERY GPU (multimem.st), loads can be
//                reduced inside the switch (multimem.ld_reduce)
//
// libcuda is not linked (the extension must import on CPU-only hosts): every driver entry point is
// resolved through cudaGetDriverEntryPoint at first use.
#include <torch/extension.h>
#include <c10/cuda/CUDAGuard.h>
#include <cuda.h>
#include <cuda_runtime.h>

#include <poll.h>
#include <sys/socket.h>
#include <sys/time.h>
#include <sys/syscall.h>
#include <sys/un.h>
#include <unistd.h>

#include <algorithm>
#include <cerrno>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

namespace py = pybind11;

namespace {

template <typename Fn> Fn drv(const char* name)
{
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess ||
        p == nullptr)
        throw std::runtime_error(std::string("driver entry point unavailable: ") + name);
    return reinterpret_cast<Fn>(p);
}

#define DRV(name) static auto name##_ = drv<decltype(&name)>(#name)

void ck(CUresult r, const char* what)
{
    if (r == CUDA_SUCCESS) return;
    static auto get_str = drv<decltype(&cuGetErrorString)>("cuGetErrorString");
    const char* s = nullptr;
    get_str(r, &s);
    throw std::runtime_error(std::string(what) + " failed: " + (s ? s : "unknown CUDA driver error") + " (" +
                             std::to_string((int)r) + ")");
}

size_t round_up(size_t x, size_t g) { return (x + g - 1) / g * g; }

CUmemAllocationProp alloc_prop(int device)
{
    CUmemAllocationProp p;
    std::memset(&p, 0, sizeof(p));
    p.type = CU_MEM_ALLOCATION_TYPE_PINNED;
    p.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    p.location.id = device;
    p.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    return p;
}

// `fd` as usable in this process: a same-process handle is dup'ed; a foreign (pid, fd) pair is
// first tried with pidfd_getfd (works on hosts that allow it); the portable path is FdChannel,
// where the owner SENDS the descriptor and `fd` is already ours (pid == 0).
int steal_fd(int pid, int fd)
{
    if (pid == 0 || pid == (int)getpid()) return dup(fd);
    const int pidfd = (int)syscall(SYS_pidfd_open, pid, 0);
    if (pidfd < 0) throw std::runtime_error("pidfd_open failed (errno " + std::to_string(errno) + ")");
    const int got = (int)syscall(SYS_pidfd_getfd, pidfd, fd, 0);
    const int err = errno;
    close(pidfd);
    if (got < 0) throw std::runtime_error("pidfd_getfd failed (errno " + std::to_string(err) +
                                          "): cannot import the peer's memory handle");
    return got;
}

sockaddr_un abstract_addr(const std::string& name, socklen_t& len)
{
    sockaddr_un a;
    std::memset(&a, 0, sizeof(a));
    a.sun_family = AF_UNIX;
    if (name.size() + 1 >= sizeof(a.sun_path)) throw std::runtime_error("socket name too long");
    std::memcpy(a.sun_path + 1, name.data(), name.size());          // leading NUL: abstract namespace
    len = (socklen_t)(offsetof(sockaddr_un, sun_path) + 1 + name.size());
    return a;
}

struct Mapping {                 // one mapped range; unmapped + released with the last tensor using it
    CUdeviceptr va = 0;
    size_t size = 0;
    CUmemGenericAllocationHandle handle = 0;
    bool own_handle = false;
    ~Mapping()
    {
        try {
            DRV(cuMemUnmap); DRV(cuMemAddressFree); DRV(cuMemRelease);
            if (va) { cuMemUnmap_(va, size); cuMemAddressFree_(va, size); }
            if (own_handle && handle) cuMemRelease_(handle);
        } catch (...) {}
    }
};

torch::Tensor tensor_over(std::shared_ptr<Mapping> m, size_t nbytes, int device)
{
    // target_device: the mapping may point at a PEER's physical memory (or at a multicast object);
    // without it from_blob asks the driver where the memory lives and refuses "cuda:1 != cuda:0"
    auto opts = torch::TensorOptions().dtype(torch::kUInt8).device(torch::kCUDA, device);
    return torch::for_blob(reinterpret_cast<void*>(m->va), {(int64_t)nbytes})
        .deleter([m](void*) mutable { m.reset(); })
        .options(opts)
        .target_device(c10::Device(c10::kCUDA, (c10::DeviceIndex)device))
        .make_tensor();
}

std::shared_ptr<Mapping> map_handle(CUmemGenericAllocationHandle h, size_t size, size_t align, int device, bool own)
{
    DRV(cuMemAddressReserve); DRV(cuMemMap); DRV(cuMemSetAccess);
    auto m = std::make_shared<Mapping>();
    m->size = size;
    m->handle = h;
    m->own_handle = own;
    ck(cuMemAddressReserve_(&m->va, size, align, 0, 0), "cuMemAddressReserve");
    ck(cuMemMap_(m->va, size, 0, h, 0), "cuMemMap");
    CUmemAccessDesc acc;
    std::memset(&acc, 0, sizeof(acc));
    acc.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    acc.location.id = device;
    acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    ck(cuMemSetAccess_(m->va, size, &acc, 1), "cuMemSetAccess");
    return m;
}

}  // namespace

// ---------------------------------------------------------------------------
// capability probe
// ---------------------------------------------------------------------------
static py::dict vmm_caps(int device)
{
    py::dict d;
    int mc = 0, posix = 0, fabric = 0;
    try {
        DRV(cuDeviceGet); DRV(cuDeviceGetAttribute);
        c10::cuda::CUDAGuard guard(device);
        cudaFree(0);
        CUdevice dev;
        ck(cuDeviceGet_(&dev, device), "cuDeviceGet");
        cuDeviceGetAttribute_(&mc, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, dev);
        cuDeviceGetAttribute_(&posix, CU_DEVICE_ATTRIBUTE_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR_SUPPORTED, dev);
        cuDeviceGetAttribute_(&fabric, CU_DEVICE_ATTRIBUTE_HANDLE_TYPE_FABRIC_SUPPORTED, dev);
    } catch (const std::exception& e) {
        d["error"] = std::string(e.what());
    }
    d["multicast"] = mc != 0;
    d["posix_fd"] = posix != 0;
    d["fabric"] = fabric != 0;
    return d;
}

// size a symmetric allocation must have so that it can also be bound to a multicast object
static int64_t vmm_padded_size(int64_t nbytes, int device, int world)
{
    DRV(cuMemGetAllocationGranularity); DRV(cuMulticastGetGranularity);
    CUmemAllocationProp p = alloc_prop(device);
    size_t g = 0;
    ck(cuMemGetAllocationGranularity_(&g, &p, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED), "cuMemGetAllocationGranularity");
    size_t mg = g;
    if (world > 1) {
        CUmulticastObjectProp mp;
        std::memset(&mp, 0, sizeof(mp));
        mp.numDevices = (unsigned)world;
        mp.size = round_up((size_t)nbytes, g);
        mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
        if (cuMulticastGetGranularity_(&mg, &mp, CU_MULTICAST_GRANULARITY_MINIMUM) != CUDA_SUCCESS) mg = g;
    }
    return (int64_t)round_up((size_t)nbytes, mg > g ? mg : g);
}

// ---------------------------------------------------------------------------
// VmmBuffer: this rank's physical allocation + the views mapped so far
// ---------------------------------------------------------------------------
class VmmBuffer {
public:
    VmmBuffer(int64_t nbytes, int device, int world) : device_(device), world_(world)
    {
        c10::cuda::CUDAGuard guard(device);
        cudaFree(0);
        DRV(cuMemCreate); DRV(cuMemExportToShareableHandle);
        size_ = (size_t)vmm_padded_size(nbytes, device, world);
        nbytes_ = (size_t)nbytes;
        CUmemAllocationProp p = alloc_prop(device);
        ck(cuMemCreate_(&handle_, size_, &p, 0), "cuMemCreate");
        ck(cuMemExportToShareableHandle_(&fd_, handle_, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0),
           "cuMemExportToShareableHandle");
        local_map_ = map_handle(handle_, size_, size_ >= (2u << 20) ? (2u << 20) : 0, device, /*own=*/true);
        cudaMemset(reinterpret_cast<void*>(local_map_->va), 0, size_);
        cudaDeviceSynchronize();
    }
    ~VmmBuffer()
    {
        if (fd_ >= 0) close(fd_);
        if (mc_fd_ >= 0) close(mc_fd_);
        if (have_mc_ && !mc_map_) {          // created / imported but never bound + mapped
            try { DRV(cuMemRelease); cuMemRelease_(mc_); } catch (...) {}
        }
    }

    int fd() const { return fd_; }
    int pid() const { return (int)getpid(); }
    int64_t size() const { return (int64_t)size_; }
    torch::Tensor local() { return tensor_over(local_map_, nbytes_, device_); }

    // map the allocation of a peer process (its pid + the fd number it exported)
    torch::Tensor open_peer(int pid, int fd)
    {
        c10::cuda::CUDAGuard guard(device_);
        DRV(cuMemImportFromShareableHandle);
        const int mine = steal_fd(pid, fd);
        CUmemGenericAllocationHandle h;
        CUresult r = cuMemImportFromShareableHandle_(&h, reinterpret_cast<void*>((uintptr_t)mine),
                                                     CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR);
        close(mine);
        ck(r, "cuMemImportFromShareableHandle");
        auto m = map_handle(h, size_, size_ >= (2u << 20) ? (2u << 20) : 0, device_, /*own=*/true);
        return tensor_over(m, nbytes_, device_);
    }

    // --- multicast: symmetric rank 0 creates, everyone imports / adds / binds / maps ---------
    int mc_create()
    {
        c10::cuda::CUDAGuard guard(device_);
        DRV(cuMulticastCreate); DRV(cuMemExportToShareableHandle);
        CUmulticastObjectProp mp;
        std::memset(&mp, 0, sizeof(mp));
        mp.numDevices = (unsigned)world_;
        mp.size = size_;
        mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
        ck(cuMulticastCreate_(&mc_, &mp), "cuMulticastCreate");
        ck(cuMemExportToShareableHandle_(&mc_fd_, mc_, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0),
           "cuMemExportToShareableHandle(multicast)");
        have_mc_ = true;
        return mc_fd_;
    }
    void mc_import(int pid, int fd)
    {
        c10::cuda::CUDAGuard guard(device_);
        DRV(cuMemImportFromShareableHandle);
        const int mine = steal_fd(pid, fd);
        CUresult r = cuMemImportFromShareableHandle_(&mc_, reinterpret_cast<void*>((uintptr_t)mine),
                                                     CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR);
        close(mine);
        ck(r, "cuMemImportFromShareableHandle(multicast)");
        have_mc_ = true;
    }
    void mc_add_device()
    {
        c10::cuda::CUDAGuard guard(device_);
        DRV(cuMulticastAddDevice); DRV(cuDeviceGet);
        TORCH_CHECK(have_mc_, "no multicast object");
        CUdevice dev;
        ck(cuDeviceGet_(&dev, device_), "cuDeviceGet");
        ck(cuMulticastAddDevice_(mc_, dev), "cuMulticastAddDevice");
    }
    // call after EVERY rank has added its device
    torch::Tensor mc_bind_and_map()
    {
        c10::cuda::CUDAGuard guard(device_);
        DRV(cuMulticastBindMem);
        TORCH_CHECK(have_mc_, "no multicast object");
        ck(cuMulticastBindMem_(mc_, 0, handle_, 0, size_, 0), "cuMulticastBindMem");
        mc_map_ = map_handle(mc_, size_, size_ >= (2u << 20) ? (2u << 20) : 0, device_, /*own=*/true);
        return tensor_over(mc_map_, nbytes_, device_);
    }

private:
    int device_, world_;
    size_t size_ = 0, nbytes_ = 0;
    CUmemGenericAllocationHandle handle_ = 0, mc_ = 0;
    bool have_mc_ = false;
    int fd_ = -1, mc_fd_ = -1;
    std::shared_ptr<Mapping> local_map_, mc_map_;
};

// ---------------------------------------------------------------------------
// FdChannel: pass file descriptors between the ranks of one host (SCM_RIGHTS over abstract
// unix-domain sockets).  Every rank listens on "<job>.<rank>"; send() connects to the peer's name and
// ships (sender rank, tag, fd); recv() accepts one connection.  Sends never block on the receiver
// (the kernel queues the connection and the message), so "everybody sends, then everybody
// receives" cannot deadlock.
// ---------------------------------------------------------------------------
class FdChannel {
public:
    FdChannel(const std::string& job, int rank, int world) : job_(job), rank_(rank)
    {
        sock_ = socket(AF_UNIX, SOCK_STREAM, 0);
        if (sock_ < 0) throw std::runtime_error("socket() failed");
        socklen_t len;
        sockaddr_un a = abstract_addr(job + "." + std::to_string(rank), len);
        if (bind(sock_, reinterpret_cast<sockaddr*>(&a), len) != 0 || listen(sock_, world * 8 + 8) != 0) {
            const int e = errno;
            close(sock_);
            throw std::runtime_error("bind/listen on the fd channel failed (errno " + std::to_string(e) + ")");
        }
    }
    ~FdChannel() { if (sock_ >= 0) close(sock_); }

    void send(int peer, int tag, int fd)
    {
        const int c = socket(AF_UNIX, SOCK_STREAM, 0);
        if (c < 0) throw std::runtime_error("socket() failed");
        socklen_t len;
        sockaddr_un a = abstract_addr(job_ + "." + std::to_string(peer), len);
        int tries = 0;
        while (connect(c, reinterpret_cast<sockaddr*>(&a), len) != 0) {
            if (++tries > 2000) { close(c); throw std::runtime_error("fd channel: cannot reach rank " + std::to_string(peer)); }
            usleep(5000);                    // the peer has not bound its socket yet
        }
        int payload[2] = {rank_, tag};
        iovec iov = {payload, sizeof(payload)};
        char ctrl[CMSG_SPACE(sizeof(int))];
        std::memset(ctrl, 0, sizeof(ctrl));
        msghdr msg;
        std::memset(&msg, 0, sizeof(msg));
        msg.msg_iov = &iov;
        msg.msg_iovlen = 1;
        msg.msg_control = ctrl;
        msg.msg_controllen = sizeof(ctrl);
        cmsghdr* cm = CMSG_FIRSTHDR(&msg);
        cm->cmsg_level = SOL_SOCKET;
        cm->cmsg_type = SCM_RIGHTS;
        cm->cmsg_len = CMSG_LEN(sizeof(int));
        std::memcpy(CMSG_DATA(cm), &fd, sizeof(int));
        const ssize_t n = sendmsg(c, &msg, 0);
        const int e = errno;
        close(c);
        if (n != (ssize_t)sizeof(payload)) throw std::runtime_error("fd channel: sendmsg failed (errno " + std::to_string(e) + ")");
    }

    // -> (sender rank, tag, fd usable in this process)
    // (a rank that never sends -- crashed, or stuck before its rendezvous -- surfaces as an
    // exception after `timeout_s`, not as a hang; the GIL is released while waiting)
    py::tuple recv(double timeout_s)
    {
        int c = -1;
        {
            py::gil_scoped_release nogil;
            pollfd pf;
            pf.fd = sock_;
            pf.events = POLLIN;
            pf.revents = 0;
            const int ms = timeout_s <= 0 ? -1 : (int)std::min(timeout_s * 1e3, 2.0e9);
            int r;
            do { r = poll(&pf, 1, ms); } while (r < 0 && errno == EINTR);
            if (r > 0) c = accept(sock_, nullptr, nullptr);
            else if (r == 0) c = -2;
        }
        if (c == -2) throw std::runtime_error("fd channel: timed out waiting for a peer's descriptor");
        if (c < 0) throw std::runtime_error("fd channel: accept failed");
        timeval tv;
        tv.tv_sec = 30;
        tv.tv_usec = 0;
        setsockopt(c, SOL_SOCKET, SO_RCVTIMEO, &tv, sizeof(tv));
        int payload[2] = {-1, -1};
        iovec iov = {payload, sizeof(payload)};
        char ctrl[CMSG_SPACE(sizeof(int))];
        msghdr msg;
        std::memset(&msg, 0, sizeof(msg));
        msg.msg_iov = &iov;
        msg.msg_iovlen = 1;
        msg.msg_control = ctrl;
        msg.msg_controllen = sizeof(ctrl);
        const ssize_t n = recvmsg(c, &msg, MSG_WAITALL);
        close(c);
        int fd = -1;
        for (cmsghdr* cm = CMSG_FIRSTHDR(&msg); cm != nullptr; cm = CMSG_NXTHDR(&msg, cm))
            if (cm->cmsg_level == SOL_SOCKET && cm->cmsg_type == SCM_RIGHTS) std::memcpy(&fd, CMSG_DATA(cm), sizeof(int));
        if (n != (ssize_t)sizeof(payload) || fd < 0) throw std::runtime_error("fd channel: no descriptor received");
        return py::make_tuple(payload[0], payload[1], fd);
    }

private:
    std::string job_;
    int rank_;
    int sock_ = -1;
};

static void close_fd(int fd) { if (fd >= 0) close(fd); }

void bind_vmm(py::module& mod)
{
    py::class_<FdChannel, std::shared_ptr<FdChannel>>(mod, "FdChannel")
        .def(py::init<const std::string&, int, int>(), py::arg("job"), py::arg("rank"), py::arg("world"))
        .def("send", &FdChannel::send, py::call_guard<py::gil_scoped_release>())
        .def("recv", &FdChannel::recv, py::arg("timeout_s") = 300.0);
    mod.def("close_fd", &close_fd);
    mod.def("vmm_caps", &vmm_caps, "multicast / handle-type capabilities of a device");
    mod.def("vmm_padded_size", &vmm_padded_size);
    py::class_<VmmBuffer, std::shared_ptr<VmmBuffer>>(mod, "VmmBuffer")
        .def(py::init<int64_t, int, int>(), py::arg("nbytes"), py::arg("device"), py::arg("world"))
        .def("fd", &VmmBuffer::fd)
        .def("pid", &VmmBuffer::pid)
        .def("size", &VmmBuffer::size)
        .def("local", &VmmBuffer::local)
        .def("open_peer", &VmmBuffer::open_peer)
        .def("mc_create", &VmmBuffer::mc_create)
        .def("mc_import", &VmmBuffer::mc_import)
        .def("mc_add_device", &VmmBuffer::mc_add_device)
        .def("mc_bind_and_map", &VmmBuffer::mc_bind_and_map);
}
