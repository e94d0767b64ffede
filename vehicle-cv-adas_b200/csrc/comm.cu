// comm.cu -- optional multi-GPU gather of the per-batch detection / track records over NCCL, driven from C.
//
// (No reference counterpart: the reference is single-GPU, SURVEY 8e.  BASELINE configs[4] asks for an NCCL gather of boxes.)
// Frames / streams are independent, so nothing is exchanged on the data path; what consumers of configs[4] need is every rank's
// fixed-size record block per batch.  A per-step torch.distributed.all_gather from Python would cost interpreter / host-sync
// time every step.  Here each step is ONE library call that returns immediately:
// the caller's records are staged into a pinned ring slot, copied to the device and all-gathered (ncclAllGather) on a private
// side stream with its own communicator (ncclCommInitRank) -- nothing on the detectors' streams waits for it.
// NCCL is bound at run time (dlopen of the libnccl.so.2 the process already loaded through torch, else the system one), so the
// library has no link-time dependency on it.
#include "common.h"
#include "../../include/adas_b200.h"
#include <dlfcn.h>
#include <string.h>
#include <mutex>

namespace adas {
struct NcclId { char internal[128]; };
typedef void* NcclComm;
struct NcclApi {
    int (*GetUniqueId)(NcclId*) = nullptr;
    int (*CommInitRank)(NcclComm*, int, NcclId, int) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, NcclComm, cudaStream_t) = nullptr;
    int (*CommDestroy)(NcclComm) = nullptr;
    int (*CommCount)(NcclComm, int*) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
    bool ok = false;
};
static NcclApi g_nccl;
static std::mutex g_nccl_mu;

static int nccl_bind() {
    std::lock_guard<std::mutex> lk(g_nccl_mu);
    if (g_nccl.ok) return 0;
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);          // the copy torch brought in, if any
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    ADAS_CHECK(h != nullptr, "NCCL is not available in this process (%s)", dlerror());
    g_nccl.GetUniqueId = (int (*)(NcclId*))dlsym(h, "ncclGetUniqueId");
    g_nccl.CommInitRank = (int (*)(NcclComm*, int, NcclId, int))dlsym(h, "ncclCommInitRank");
    g_nccl.AllGather = (int (*)(const void*, void*, size_t, int, NcclComm, cudaStream_t))dlsym(h, "ncclAllGather");
    g_nccl.CommDestroy = (int (*)(NcclComm))dlsym(h, "ncclCommDestroy");
    g_nccl.CommCount = (int (*)(NcclComm, int*))dlsym(h, "ncclCommCount");
    g_nccl.GetErrorString = (const char* (*)(int))dlsym(h, "ncclGetErrorString");
    ADAS_CHECK(g_nccl.GetUniqueId && g_nccl.CommInitRank && g_nccl.AllGather && g_nccl.CommDestroy && g_nccl.CommCount && g_nccl.GetErrorString,
               "libnccl does not export the expected entry points");
    g_nccl.ok = true;
    return 0;
}
#define ADAS_NCCL(call)                                                                                   \
    do {                                                                                                  \
        int _r = (call);                                                                                  \
        if (_r != 0) { adas::set_error("%s:%d NCCL error %d (%s) in %s", __FILE__, __LINE__, _r, g_nccl.GetErrorString(_r), #call); return 1; } \
    } while (0)
}  // namespace adas

using namespace adas;

static constexpr int COMM_SLOTS = 4;
struct adas_comm {
    int device = 0, rank = 0, world = 1;
    size_t bytes = 0;
    NcclComm comm = nullptr;
    cudaStream_t st = nullptr;
    uint8_t* h_slot[COMM_SLOTS] = {nullptr, nullptr, nullptr, nullptr};     // pinned staging ring
    uint8_t* d_slot[COMM_SLOTS] = {nullptr, nullptr, nullptr, nullptr};     // device send ring
    cudaEvent_t ev[COMM_SLOTS] = {nullptr, nullptr, nullptr, nullptr};
    uint8_t* d_all = nullptr;                                               // [world * bytes] last gathered block
    long long n = 0;
};

extern "C" {

int adas_comm_unique_id(uint8_t id[128]) {
    if (nccl_bind()) return 1;
    NcclId u;
    ADAS_NCCL(g_nccl.GetUniqueId(&u));
    memcpy(id, u.internal, 128);
    return 0;
}

int adas_comm_create(int device, int rank, int world, const uint8_t id[128], int64_t bytes_per_rank, adas_comm** out) {
    ADAS_CHECK(out != nullptr && id != nullptr && world >= 1 && rank >= 0 && rank < world && bytes_per_rank > 0, "adas_comm_create: bad arguments");
    if (nccl_bind()) return 1;
    ADAS_CUDA(cudaSetDevice(device));
    adas_comm* c = new adas_comm();
    c->device = device; c->rank = rank; c->world = world; c->bytes = (size_t)bytes_per_rank;
    ADAS_CUDA(cudaStreamCreateWithFlags(&c->st, cudaStreamNonBlocking));
    for (int i = 0; i < COMM_SLOTS; ++i) {
        ADAS_CUDA(cudaHostAlloc(&c->h_slot[i], c->bytes, cudaHostAllocDefault));
        ADAS_CUDA(cudaMalloc(&c->d_slot[i], c->bytes));
        ADAS_CUDA(cudaEventCreateWithFlags(&c->ev[i], cudaEventDisableTiming));
    }
    ADAS_CUDA(cudaMalloc(&c->d_all, c->bytes * (size_t)world));
    NcclId u;
    memcpy(u.internal, id, 128);
    ADAS_NCCL(g_nccl.CommInitRank(&c->comm, world, u, rank));
    *out = c;
    return 0;
}

int adas_comm_destroy(adas_comm* c) {
    if (!c) return 0;
    cudaSetDevice(c->device);
    if (c->st) cudaStreamSynchronize(c->st);
    if (c->comm && g_nccl.ok) g_nccl.CommDestroy(c->comm);
    for (int i = 0; i < COMM_SLOTS; ++i) { if (c->h_slot[i]) cudaFreeHost(c->h_slot[i]); cudaFree(c->d_slot[i]); if (c->ev[i]) cudaEventDestroy(c->ev[i]); }
    cudaFree(c->d_all);
    if (c->st) cudaStreamDestroy(c->st);
    delete c;
    return 0;
}

// One step's record block of this rank (host memory, `bytes_per_rank` bytes): staged, uploaded and all-gathered asynchronously.
int adas_comm_all_gather(adas_comm* c, const void* host_src) {
    ADAS_CHECK(c != nullptr && host_src != nullptr, "adas_comm_all_gather: bad arguments");
    ADAS_CUDA(cudaSetDevice(c->device));
    const int k = (int)(c->n % COMM_SLOTS);
    if (c->n >= COMM_SLOTS) ADAS_CUDA(cudaEventSynchronize(c->ev[k]));      // the gather that last used this slot (4 steps ago) is done
    memcpy(c->h_slot[k], host_src, c->bytes);
    ADAS_CUDA(cudaMemcpyAsync(c->d_slot[k], c->h_slot[k], c->bytes, cudaMemcpyHostToDevice, c->st));
    ADAS_NCCL(g_nccl.AllGather(c->d_slot[k], c->d_all, c->bytes, 1 /* ncclUint8 */, c->comm, c->st));
    ADAS_CUDA(cudaEventRecord(c->ev[k], c->st));
    c->n += 1;
    return 0;
}

int adas_comm_sync(adas_comm* c) {
    ADAS_CHECK(c != nullptr, "adas_comm_sync: null communicator");
    ADAS_CUDA(cudaSetDevice(c->device));
    ADAS_CUDA(cudaStreamSynchronize(c->st));
    return 0;
}

// copies the last gathered block ([world, bytes_per_rank]) to host memory (synchronous)
int adas_comm_read(adas_comm* c, void* host_dst) {
    ADAS_CHECK(c != nullptr && host_dst != nullptr, "adas_comm_read: bad arguments");
    ADAS_CUDA(cudaSetDevice(c->device));
    ADAS_CUDA(cudaMemcpyAsync(host_dst, c->d_all, c->bytes * (size_t)c->world, cudaMemcpyDeviceToHost, c->st));
    ADAS_CUDA(cudaStreamSynchronize(c->st));
    return 0;
}

int adas_comm_info(adas_comm* c, int* nranks, int64_t* gathers) {
    ADAS_CHECK(c != nullptr, "adas_comm_info: null communicator");
    int n = 0;
    ADAS_NCCL(g_nccl.CommCount(c->comm, &n));
    if (nranks) *nranks = n;
    if (gathers) *gathers = c->n;
    return 0;
}

}  // extern "C"
