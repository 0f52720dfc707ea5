// nccl_vrf.cu — the path's ONE exchange step for hosts that run one process per GPU: the min-reduction of the VRF nonce
// candidate over the ranks (SURVEY.md §8e; north_star: "NCCL used only for the final min-reduction of the VRF nonce
// candidate").  bench.py does this through torch.distributed; a Go / C host calls the four functions below.  NCCL's
// ncclMin is per element, not lexicographic over a 32-byte key with an index tie-break, so the reduction is an
// all-gather of one 64-byte record per rank (384 B on 8 GPUs — latency, not bandwidth) and a local arg-min.
// libnccl is loaded at first use (dlopen): the label / verify / k2pow paths do not depend on it.
#include <dlfcn.h>

#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/b200post.h"
#include "engine.h"
#include "host_hash.h"

using namespace b200post;

namespace {

typedef struct ncclComm *ncclComm_t;
struct NcclId { char bytes[128]; };
typedef int (*fn_get_id)(NcclId *);
typedef int (*fn_init_rank)(ncclComm_t *, int, NcclId, int);
typedef int (*fn_all_gather)(const void *, void *, size_t, int, ncclComm_t, cudaStream_t);
typedef int (*fn_destroy)(ncclComm_t);
typedef const char *(*fn_errstr)(int);

struct Nccl {
    void *lib = nullptr;
    fn_get_id get_id = nullptr; fn_init_rank init_rank = nullptr; fn_all_gather all_gather = nullptr; fn_destroy destroy = nullptr;
    fn_errstr errstr = nullptr;
};

Nccl *nccl() {
    static Nccl n;
    static std::once_flag once;
    std::call_once(once, [] {
        // An NCCL already in the process (e.g. the one a PyTorch host bundles) is reused; otherwise the system's is loaded,
        // privately.  The loader de-duplicates by soname, so a host that also loads another libnccl.so.2 must load it FIRST.
        n.lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
        for (const char *name : {"libnccl.so.2", "libnccl.so"}) {
            if (n.lib) break;
            n.lib = dlopen(name, RTLD_NOW | RTLD_LOCAL);
        }
        if (!n.lib) return;
        n.get_id = (fn_get_id)dlsym(n.lib, "ncclGetUniqueId");
        n.init_rank = (fn_init_rank)dlsym(n.lib, "ncclCommInitRank");
        n.all_gather = (fn_all_gather)dlsym(n.lib, "ncclAllGather");
        n.destroy = (fn_destroy)dlsym(n.lib, "ncclCommDestroy");
        n.errstr = (fn_errstr)dlsym(n.lib, "ncclGetErrorString");
    });
    if (!n.lib || !n.get_id || !n.init_rank || !n.all_gather || !n.destroy) { set_error("libnccl.so.2 not loadable"); return nullptr; }
    return &n;
}

int nccl_fail(const char *what, int rc) {
    Nccl *n = nccl();
    set_error(std::string(what) + ": " + (n && n->errstr ? n->errstr(rc) : "NCCL error " + std::to_string(rc)));
    return B200POST_ERR_CUDA;
}

struct Record { uint32_t found, pad; uint64_t index; uint8_t label32[32]; uint8_t fill[16]; };   // 64 bytes
static_assert(sizeof(Record) == 64, "one NCCL element block per rank");

}  // namespace

struct b200post_vrf_comm {
    ncclComm_t comm = nullptr;
    int dev = 0, world = 0, rank = 0;
    Stream stream;
    DeviceBuffer<Record> d_send, d_recv;
    std::vector<Record> host;
};

extern "C" {

int b200post_vrf_comm_unique_id(uint8_t out128[128]) {
    Nccl *n = nccl();
    if (!n || !out128) return n ? B200POST_ERR_INVALID_ARGUMENT : B200POST_ERR_UNSUPPORTED;
    NcclId id;
    const int rc = n->get_id(&id);
    if (rc) return nccl_fail("ncclGetUniqueId", rc);
    memcpy(out128, id.bytes, 128);
    return B200POST_OK;
}

int b200post_vrf_comm_init(uint32_t provider, int rank, int world, const uint8_t id128[128], b200post_vrf_comm **out) {
    if (!out || !id128 || world < 1 || rank < 0 || rank >= world) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    *out = nullptr;
    if (int rc = device_engine(provider)) return rc;
    Nccl *n = nccl();                  // loaded only once a device is there to use it
    if (!n) return B200POST_ERR_UNSUPPORTED;
    if (cudaSetDevice((int)provider) != cudaSuccess) { set_error("cudaSetDevice failed"); return B200POST_ERR_CUDA; }
    b200post_vrf_comm *c = new b200post_vrf_comm;
    c->dev = (int)provider; c->world = world; c->rank = rank;
    c->host.resize((size_t)world);
    NcclId id;
    memcpy(id.bytes, id128, 128);
    int rc = n->init_rank(&c->comm, world, id, rank);
    if (rc) { delete c; return nccl_fail("ncclCommInitRank", rc); }
    if (c->stream.create(cudaStreamNonBlocking) != cudaSuccess || c->d_send.resize(1) != cudaSuccess ||
        c->d_recv.resize((size_t)world) != cudaSuccess) {
        set_error("CUDA allocation for the VRF exchange failed");
        n->destroy(c->comm);
        delete c;
        return B200POST_ERR_CUDA;
    }
    *out = c;
    return B200POST_OK;
}

int b200post_vrf_comm_min(b200post_vrf_comm *c, const b200post_vrf_nonce *mine, b200post_vrf_nonce *best) {
    if (!c || !mine || !best) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    Nccl *n = nccl();
    if (!n) return B200POST_ERR_UNSUPPORTED;
    if (cudaSetDevice(c->dev) != cudaSuccess) { set_error("cudaSetDevice failed"); return B200POST_ERR_CUDA; }
    Record r{};
    r.found = mine->found; r.index = mine->index; memcpy(r.label32, mine->label32, 32);
    if (cudaMemcpyAsync(c->d_send.get(), &r, sizeof r, cudaMemcpyHostToDevice, c->stream.get()) != cudaSuccess) { set_error("H2D failed"); return B200POST_ERR_CUDA; }
    const int rc = n->all_gather(c->d_send.get(), c->d_recv.get(), sizeof(Record), 1 /* ncclUint8 */, c->comm, c->stream.get());
    if (rc) return nccl_fail("ncclAllGather", rc);
    if (cudaMemcpyAsync(c->host.data(), c->d_recv.get(), sizeof(Record) * (size_t)c->world, cudaMemcpyDeviceToHost, c->stream.get()) != cudaSuccess ||
        cudaStreamSynchronize(c->stream.get()) != cudaSuccess) { set_error("VRF exchange failed"); return B200POST_ERR_CUDA; }
    memset(best, 0, sizeof *best);
    for (const Record &x : c->host)
        if (x.found && (!best->found || vrf_less(x.label32, x.index, best->label32, best->index))) {
            best->found = 1; best->index = x.index; memcpy(best->label32, x.label32, 32);
        }
    return B200POST_OK;
}

void b200post_vrf_comm_free(b200post_vrf_comm *c) {
    if (!c) return;
    Nccl *n = nccl();
    cudaSetDevice(c->dev);
    if (n && c->comm) n->destroy(c->comm);
    delete c;   // frees the buffers and the stream on c->dev
}

}  // extern "C"
