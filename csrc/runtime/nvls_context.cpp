#include "runtime/nvls_context.h"

#include <unistd.h>

#include <algorithm>
#include <cstring>
#include <stdexcept>

namespace ssb {

namespace {

// The driver API is reached through cudaGetDriverEntryPoint so the extension does not link libcuda (the build /
// CPU-test container has no driver; importing the module there must keep working).
template <typename Fn>
Fn driver_fn(const char* name) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint(name, &ptr, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess || !ptr)
        throw std::runtime_error(std::string("NVLS: driver entry point not available: ") + name);
    return reinterpret_cast<Fn>(ptr);
}

#define DRV(name) driver_fn<decltype(&name)>(#name)

void cu_check(CUresult r, const char* what) {
    if (r == CUDA_SUCCESS) return;
    const char* msg = nullptr;
    try {
        DRV(cuGetErrorString)(r, &msg);
    } catch (...) {
    }
    throw std::runtime_error(std::string("NVLS: ") + what + " failed: " + (msg ? msg : "unknown driver error") + " (" +
                             std::to_string((int)r) + ")");
}

#define CUDA_RT(expr)                                                                                      \
    do {                                                                                                   \
        cudaError_t _e = (expr);                                                                           \
        if (_e != cudaSuccess)                                                                             \
            throw std::runtime_error(std::string("CUDA error: ") + cudaGetErrorString(_e) + " at " #expr); \
    } while (0)

size_t round_up_sz(size_t x, size_t m) { return (x + m - 1) / m * m; }

CUmemAllocationProp device_alloc_prop(int dev) {
    CUmemAllocationProp prop;
    memset(&prop, 0, sizeof(prop));
    prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
    prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    prop.location.id = dev;
    prop.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;   // required to bind to a shared multicast object
    return prop;
}

}  // namespace

bool NvlsContext::supported() {
    int dev = 0, flag = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return false;
    try {
        CUdevice cudev;
        if (DRV(cuDeviceGet)(&cudev, dev) != CUDA_SUCCESS) return false;
        if (DRV(cuDeviceGetAttribute)(&flag, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, cudev) != CUDA_SUCCESS) return false;
    } catch (...) {
        return false;
    }
    return flag != 0;
}

namespace {

void check_team(int dp, int rank, int64_t arena_numel) {
    if (dp < 2 || dp > 8) throw std::runtime_error("NvlsContext: dp must be in [2, 8]");
    if (rank < 0 || rank >= dp) throw std::runtime_error("NvlsContext: rank must be in [0, dp)");
    // the kernels work in float4 chunks (ParamArena keeps a multiple of 32 floats)
    if (arena_numel <= 0 || arena_numel % 4 != 0) throw std::runtime_error("NvlsContext: arena_numel must be a positive multiple of 4");
}

int64_t pad_numel(int64_t arena_numel) { return (arena_numel + 63) / 64 * 64; }   // 256-byte multiple

size_t alloc_bytes(int64_t numel_pad) { return ((size_t)2 * numel_pad + 64) * sizeof(float); }   // W | G | 2 x 32 flag words

}  // namespace

NvlsContext::NvlsContext(int dp, int rank, int64_t arena_numel, float /*lr: unused, see nvls_context.h*/, int devices)
    : dp_(dp), rank_(rank), devices_(devices == 0 ? dp : devices), arena_numel_(arena_numel) {
    check_team(dp, rank, arena_numel);
    if (devices_ < 1 || devices_ > dp_) throw std::runtime_error("NvlsContext: devices must be in [1, dp]");
    CUDA_RT(cudaGetDevice(&dev_));
    CUDA_RT(cudaFree(nullptr));                                  // make sure the primary context exists
    if (!supported()) throw std::runtime_error("NvlsContext: this device / driver does not support NVLink multicast");
    numel_pad_ = pad_numel(arena_numel_);
    const size_t want = alloc_bytes(numel_pad_);
    CUmulticastObjectProp mprop;
    memset(&mprop, 0, sizeof(mprop));
    mprop.numDevices = (unsigned)devices_;
    mprop.size = want;
    mprop.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    size_t g_mc = 0, g_mem = 0;
    cu_check(DRV(cuMulticastGetGranularity)(&g_mc, &mprop, CU_MULTICAST_GRANULARITY_RECOMMENDED), "cuMulticastGetGranularity");
    CUmemAllocationProp aprop = device_alloc_prop(dev_);
    cu_check(DRV(cuMemGetAllocationGranularity)(&g_mem, &aprop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED), "cuMemGetAllocationGranularity");
    gran_ = std::max(g_mc, g_mem);
    size_ = round_up_sz(want, gran_);
    CUDA_RT(cudaMalloc(&epoch_, 64));
    CUDA_RT(cudaMemset(epoch_, 0, 64));
    CUDA_RT(cudaMalloc(&cta_done_, 64));
    CUDA_RT(cudaMemset(cta_done_, 0, 64));
}

NvlsContext::NvlsContext(int dp, int rank, int64_t arena_numel, Local)
    : dp_(dp), rank_(rank), devices_(dp), arena_numel_(arena_numel) {
    check_team(dp, rank, arena_numel);
    CUDA_RT(cudaGetDevice(&dev_));
    numel_pad_ = pad_numel(arena_numel_);
    size_ = alloc_bytes(numel_pad_);
    CUDA_RT(cudaMalloc(&local_mem_, size_));
    CUDA_RT(cudaMemset(local_mem_, 0, size_));
    uc_ptr_ = reinterpret_cast<CUdeviceptr>(local_mem_);
    CUDA_RT(cudaMalloc(&epoch_, 64));
    CUDA_RT(cudaMemset(epoch_, 0, 64));
    CUDA_RT(cudaMalloc(&cta_done_, 64));
    CUDA_RT(cudaMemset(cta_done_, 0, 64));
    CUDA_RT(cudaDeviceSynchronize());
}

std::unique_ptr<NvlsContext> NvlsContext::local(int dp, int rank, int64_t arena_numel) {
    return std::unique_ptr<NvlsContext>(new NvlsContext(dp, rank, arena_numel, Local{}));
}

void NvlsContext::open_local(const std::vector<const NvlsContext*>& team) {
    if (!is_local()) throw std::runtime_error("NvlsContext::open_local: not a local team member (NvlsContext::local)");
    if ((int)team.size() != dp_ || team[rank_] != this)
        throw std::runtime_error("NvlsContext::open_local: the team must list dp members in rank order, this one at its rank");
    std::vector<NvlsMember> views;
    for (int m = 0; m < dp_; ++m) {
        const NvlsContext* c = team[m];
        if (c == nullptr || !c->is_local() || c->dp_ != dp_ || c->rank_ != m || c->arena_numel_ != arena_numel_ || c->dev_ != dev_)
            throw std::runtime_error("NvlsContext::open_local: member " + std::to_string(m) +
                                     " is not a local context of this team's size, rank, arena and device");
        views.push_back({c->weights(), c->grads(), c->flag_in(), c->flag_out()});
    }
    if (team_ == nullptr) CUDA_RT(cudaMalloc(&team_, sizeof(NvlsMember) * 8));
    CUDA_RT(cudaMemcpy(team_, views.data(), sizeof(NvlsMember) * views.size(), cudaMemcpyHostToDevice));
}

NvlsContext::~NvlsContext() {
    cudaDeviceSynchronize();
    if (local_mem_ != nullptr) {
        cudaFree(local_mem_);
        cudaFree(team_);
        cudaFree(epoch_);
        cudaFree(cta_done_);
        return;
    }
    try {
        if (mc_ptr_) {
            DRV(cuMemUnmap)(mc_ptr_, size_);
            DRV(cuMemAddressFree)(mc_ptr_, size_);
        }
        if (uc_ptr_) {
            DRV(cuMemUnmap)(uc_ptr_, size_);
            DRV(cuMemAddressFree)(uc_ptr_, size_);
        }
        if (bound_) {
            CUdevice cudev;
            if (DRV(cuDeviceGet)(&cudev, dev_) == CUDA_SUCCESS) DRV(cuMulticastUnbind)(mc_, cudev, 0, size_);
        }
        if (have_mem_) DRV(cuMemRelease)(mem_);
        if (have_mc_) DRV(cuMemRelease)(mc_);
    } catch (...) {
    }
    cudaFree(epoch_);
    cudaFree(cta_done_);
}

int NvlsContext::export_fd() {
    if (is_local()) throw std::runtime_error("NvlsContext: a local team member has no multicast object");
    if (have_mc_) throw std::runtime_error("NvlsContext: multicast object already present");
    CUmulticastObjectProp mprop;
    memset(&mprop, 0, sizeof(mprop));
    mprop.numDevices = (unsigned)devices_;
    mprop.size = size_;
    mprop.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    cu_check(DRV(cuMulticastCreate)(&mc_, &mprop), "cuMulticastCreate");
    have_mc_ = true;
    int fd = -1;
    cu_check(DRV(cuMemExportToShareableHandle)(&fd, mc_, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0),
             "cuMemExportToShareableHandle(multicast)");
    return fd;
}

void NvlsContext::import_fd(int fd) {
    if (is_local()) throw std::runtime_error("NvlsContext: a local team member has no multicast object");
    if (have_mc_) throw std::runtime_error("NvlsContext: multicast object already present");
    cu_check(DRV(cuMemImportFromShareableHandle)(&mc_, reinterpret_cast<void*>(static_cast<uintptr_t>(fd)),
                                                 CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR),
             "cuMemImportFromShareableHandle(multicast)");
    have_mc_ = true;
}

void NvlsContext::add_device() {
    if (!have_mc_) throw std::runtime_error("NvlsContext::add_device before export_fd / import_fd");
    CUdevice cudev;
    cu_check(DRV(cuDeviceGet)(&cudev, dev_), "cuDeviceGet");
    cu_check(DRV(cuMulticastAddDevice)(mc_, cudev), "cuMulticastAddDevice");
}

void NvlsContext::bind_and_map() {
    if (!have_mc_) throw std::runtime_error("NvlsContext::bind_and_map before export_fd / import_fd");
    CUmemAllocationProp aprop = device_alloc_prop(dev_);
    cu_check(DRV(cuMemCreate)(&mem_, size_, &aprop, 0), "cuMemCreate");
    have_mem_ = true;
    cu_check(DRV(cuMulticastBindMem)(mc_, 0, mem_, 0, size_, 0), "cuMulticastBindMem");
    bound_ = true;
    CUmemAccessDesc acc;
    memset(&acc, 0, sizeof(acc));
    acc.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    acc.location.id = dev_;
    acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    // unicast view of this replica's physical memory
    cu_check(DRV(cuMemAddressReserve)(&uc_ptr_, size_, gran_, 0, 0), "cuMemAddressReserve(unicast)");
    cu_check(DRV(cuMemMap)(uc_ptr_, size_, 0, mem_, 0), "cuMemMap(unicast)");
    cu_check(DRV(cuMemSetAccess)(uc_ptr_, size_, &acc, 1), "cuMemSetAccess(unicast)");
    // multicast view: stores / reductions issued here reach every replica's copy
    cu_check(DRV(cuMemAddressReserve)(&mc_ptr_, size_, gran_, 0, 0), "cuMemAddressReserve(multicast)");
    cu_check(DRV(cuMemMap)(mc_ptr_, size_, 0, mc_, 0), "cuMemMap(multicast)");
    cu_check(DRV(cuMemSetAccess)(mc_ptr_, size_, &acc, 1), "cuMemSetAccess(multicast)");
    CUDA_RT(cudaMemset(reinterpret_cast<void*>(uc_ptr_), 0, size_));
    CUDA_RT(cudaDeviceSynchronize());
}

NvlsParams NvlsContext::params() const {
    if (is_local() ? team_ == nullptr : (!mc_ptr_ || !uc_ptr_))
        throw std::runtime_error(is_local() ? "NvlsContext::params before open_local" : "NvlsContext::params before bind_and_map");
    NvlsParams p{};
    float* uc = reinterpret_cast<float*>(uc_ptr_);
    p.W_uc = uc; p.G_uc = uc + numel_pad_;
    p.flag_in_uc = flag_in(); p.flag_out_uc = flag_out();
    if (is_local()) {
        p.team = team_;                                        // W_mc / G_mc / flag_*_mc stay null: the replay transport
    } else {
        float* mc = reinterpret_cast<float*>(mc_ptr_);
        p.W_mc = mc; p.G_mc = mc + numel_pad_;
        uint32_t* fmc = reinterpret_cast<uint32_t*>(mc + 2 * numel_pad_);
        p.flag_in_mc = fmc; p.flag_out_mc = fmc + 32;
    }
    p.epoch = epoch_;
    p.cta_done = cta_done_;
    // the arena, not the padded allocation: the owners also read and write the caller's momentum / EMA arenas at the
    // same offsets, and those hold arena_numel floats
    p.numel = arena_numel_;
    p.dp = dp_; p.rank = rank_;
    p.lr = nullptr;
    return p;
}

}  // namespace ssb
