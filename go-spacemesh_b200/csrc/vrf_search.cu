// vrf_search.cu — the VRF nonce of a POST from its stored labels (include/b200post_setup.h, b200post_search_vrf_nonce):
// the counterpart of postcli -searchForNonce (recalled, unpinned), for POST data whose files were written by
// file-range sessions on several machines, none of which saw every label.
//
// The arg-min of label32 (big-endian) is decided by its first 16 bytes, and those are exactly what postdata_N.bin
// holds.  So instead of recomputing every label (ROMix speed), the files are streamed through the GPU at 16 B per label
// (storage speed): a reader thread fills pinned staging one chunk ahead, the H2D copy runs on its own stream, and per
// chunk K8 reduces the chunk to one small record (lowest prefix, its two lowest positions, how many hold it).  The host
// folds the records; only the two lowest positions at the final lowest prefix have their label32 recomputed.
#include <algorithm>
#include <cstring>
#include <future>
#include <string>
#include <utility>
#include <vector>

#include "../../include/b200post_setup.h"
#include "engine.h"
#include "host_hash.h"
#include "postdata_io.h"
#include "setup_internal.h"

namespace b200post {
namespace {

constexpr uint64_t kMaxChunk = 1ull << 26;   // 1 GiB of staging per buffer
constexpr int kTpb = 256;

// a stored label as two big-endian 64-bit halves, so that (hi, lo) orders like the bytes
struct Key { uint64_t hi, lo; };

// one per chunk, copied back to the host
struct ChunkMin {
    uint64_t hi, lo;          // the smallest stored 16-byte prefix of the chunk
    uint32_t index;           // its lowest position in the chunk
    uint32_t n_ties;          // positions holding that prefix, all of them counted
    uint32_t next;            // the lowest of them above index (~0u: none)
};

struct CtaMin { uint64_t hi, lo; uint32_t index, pad; };

__device__ __forceinline__ Key load_key(const uint4 v) {
    return Key{((uint64_t)__byte_perm(v.x, 0, 0x0123) << 32) | __byte_perm(v.y, 0, 0x0123),
                ((uint64_t)__byte_perm(v.z, 0, 0x0123) << 32) | __byte_perm(v.w, 0, 0x0123)};
}

__device__ __forceinline__ bool less3(uint64_t ah, uint64_t al, uint32_t ai, uint64_t bh, uint64_t bl, uint32_t bi) {
    return ah != bh ? ah < bh : al != bl ? al < bl : ai < bi;
}

// warp-shuffle arg-min of (hi, lo, index), then across the CTA through shared memory; the result is in thread 0
__device__ __forceinline__ void cta_argmin(uint64_t &h, uint64_t &l, uint32_t &i) {
    __shared__ CtaMin warp_min[kTpb / 32];
    for (int d = 16; d; d >>= 1) {
        const uint64_t oh = __shfl_down_sync(0xffffffffu, h, d), ol = __shfl_down_sync(0xffffffffu, l, d);
        const uint32_t oi = __shfl_down_sync(0xffffffffu, i, d);
        if (less3(oh, ol, oi, h, l, i)) { h = oh; l = ol; i = oi; }
    }
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) warp_min[warp] = CtaMin{h, l, i, 0};
    __syncthreads();
    if (warp == 0) {
        const bool live = lane < blockDim.x / 32;
        h = live ? warp_min[lane].hi : ~0ull; l = live ? warp_min[lane].lo : ~0ull; i = live ? warp_min[lane].index : ~0u;
        for (int d = 16; d; d >>= 1) {
            const uint64_t oh = __shfl_down_sync(0xffffffffu, h, d), ol = __shfl_down_sync(0xffffffffu, l, d);
            const uint32_t oi = __shfl_down_sync(0xffffffffu, i, d);
            if (less3(oh, ol, oi, h, l, i)) { h = oh; l = ol; i = oi; }
        }
    }
    __syncthreads();   // warp_min may be reused by the caller's next reduction
}

// K8a: arg-min of the chunk's stored prefixes (lowest position on ties).  Each thread keeps its own minimum over a
// grid-stride walk (positions ascend per thread, so a strict comparison keeps the lowest; a thread's first label is
// always taken, so an all-ones prefix gets its real position, not the empty ~0u); each CTA writes one partial; the
// last CTA to finish reduces the partials into the chunk's record and re-arms the counter.
__global__ void __launch_bounds__(kTpb) stored_min_kernel(const uint4 *__restrict__ labels, uint32_t count, CtaMin *__restrict__ partial,
                                                         uint32_t *__restrict__ done, ChunkMin *__restrict__ rec) {
    uint64_t h = ~0ull, l = ~0ull;
    uint32_t idx = ~0u;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x) {
        const Key k = load_key(__ldcs(labels + i));
        if (idx == ~0u || k.hi < h || (k.hi == h && k.lo < l)) { h = k.hi; l = k.lo; idx = i; }
    }
    cta_argmin(h, l, idx);
    __shared__ bool last;
    if (threadIdx.x == 0) {
        partial[blockIdx.x] = CtaMin{h, l, idx, 0};
        __threadfence();
        last = atomicAdd(done, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    h = ~0ull; l = ~0ull; idx = ~0u;
    for (uint32_t c = threadIdx.x; c < gridDim.x; c += blockDim.x) {
        const uint64_t ph = __ldcg(&partial[c].hi), pl = __ldcg(&partial[c].lo);
        const uint32_t pi = __ldcg(&partial[c].index);
        if (less3(ph, pl, pi, h, l, idx)) { h = ph; l = pl; idx = pi; }
    }
    cta_argmin(h, l, idx);
    if (threadIdx.x == 0) {
        rec->hi = h; rec->lo = l; rec->index = idx; rec->n_ties = 0; rec->next = ~0u;
        *done = 0;
    }
}

// K8b: a second pass over the same device-resident chunk counts the positions whose prefix equals the minimum and keeps
// the lowest above K8a's index (two distinct real labels cannot share 128 bits, so more than one means damaged data:
// index is damaged, or index holds the real label and next is the lowest copy of it)
__global__ void __launch_bounds__(kTpb) stored_tie_kernel(const uint4 *__restrict__ labels, uint32_t count, ChunkMin *__restrict__ rec) {
    const uint64_t mh = rec->hi, ml = rec->lo;
    const uint32_t first = rec->index;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x) {
        const Key k = load_key(__ldcs(labels + i));
        if (k.hi == mh && k.lo == ml) {
            atomicAdd(&rec->n_ties, 1u);
            if (i != first) atomicMin(&rec->next, i);
        }
    }
}

// Streams chunks of stored labels through K8: staging(b) -> H2D on the copy stream -> K8a, K8b and the record's D2H
// on the kernel stream.  Buffer b is reused two chunks later: the copy into d_labels_[b] waits for the kernels of the
// chunk before, and the reader waits (wait_copied) for the copy out of staging(b) before refilling it.
class StoredScan {
public:
    ~StoredScan() {
        if (dev_ < 0) return;
        cudaSetDevice(dev_);   // the members free themselves on the scan's device, after its work
        if (copy_.get()) cudaStreamSynchronize(copy_.get());
        if (kern_.get()) cudaStreamSynchronize(kern_.get());
    }
    int init(const DeviceEngine *e, uint64_t chunk) {
        dev_ = e->device();
        CUDA_TRY(cudaSetDevice(dev_));
        grid_ = (uint32_t)e->prop().multiProcessorCount * 4;
        CUDA_TRY(copy_.create(cudaStreamNonBlocking));
        CUDA_TRY(kern_.create(cudaStreamNonBlocking));
        CUDA_TRY(d_partial_.resize(grid_));
        CUDA_TRY(d_done_.resize(1));
        CUDA_TRY(cudaMemsetAsync(d_done_.get(), 0, sizeof(uint32_t), kern_.get()));
        for (int b = 0; b < 2; b++) {
            CUDA_TRY(h_labels_[b].resize(chunk * 16));
            CUDA_TRY(d_labels_[b].resize(chunk * 16));
            CUDA_TRY(d_rec_[b].resize(1));
            CUDA_TRY(h_rec_[b].resize(1));
            CUDA_TRY(copied_[b].create(cudaEventDisableTiming));
            CUDA_TRY(scanned_[b].create(cudaEventDisableTiming));
        }
        return B200POST_OK;
    }
    uint8_t *staging(int b) { return h_labels_[b].get(); }
    // staging(b) may be refilled (callable from the reader thread)
    int wait_copied(int b) {
        CUDA_TRY(cudaSetDevice(dev_));
        CUDA_TRY(cudaEventSynchronize(copied_[b].get()));
        return B200POST_OK;
    }
    int submit(int b, uint32_t count) {
        CUDA_TRY(cudaSetDevice(dev_));
        CUDA_TRY(cudaStreamWaitEvent(copy_.get(), scanned_[b].get(), 0));
        CUDA_TRY(cudaMemcpyAsync(d_labels_[b].get(), h_labels_[b].get(), (size_t)count * 16, cudaMemcpyHostToDevice, copy_.get()));
        CUDA_TRY(cudaEventRecord(copied_[b].get(), copy_.get()));
        CUDA_TRY(cudaStreamWaitEvent(kern_.get(), copied_[b].get(), 0));
        const uint4 *labels = reinterpret_cast<const uint4 *>(d_labels_[b].get());
        const uint32_t grid = std::min<uint32_t>(grid_, (count + kTpb - 1) / kTpb);
        stored_min_kernel<<<grid, kTpb, 0, kern_.get()>>>(labels, count, d_partial_.get(), d_done_.get(), d_rec_[b].get());
        stored_tie_kernel<<<grid, kTpb, 0, kern_.get()>>>(labels, count, d_rec_[b].get());
        g_launches += 2;
        CUDA_TRY(cudaGetLastError());
        CUDA_TRY(cudaMemcpyAsync(h_rec_[b].get(), d_rec_[b].get(), sizeof(ChunkMin), cudaMemcpyDeviceToHost, kern_.get()));
        CUDA_TRY(cudaEventRecord(scanned_[b].get(), kern_.get()));
        return B200POST_OK;
    }
    int collect(int b, ChunkMin *out) {
        CUDA_TRY(cudaSetDevice(dev_));
        CUDA_TRY(cudaEventSynchronize(scanned_[b].get()));
        *out = *h_rec_[b].get();
        return B200POST_OK;
    }

private:
    int dev_ = -1;
    uint32_t grid_ = 0;
    Stream copy_, kern_;
    PinnedBuffer<uint8_t> h_labels_[2];
    DeviceBuffer<uint8_t> d_labels_[2];
    DeviceBuffer<CtaMin> d_partial_;
    DeviceBuffer<uint32_t> d_done_;
    DeviceBuffer<ChunkMin> d_rec_[2];
    PinnedBuffer<ChunkMin> h_rec_[2];
    Event copied_[2], scanned_[2];
};

// the running minimum across chunks and files; next is the lowest position at the prefix above index (~0: none)
struct Running {
    bool any = false;
    uint64_t hi = 0, lo = 0, index = 0, next = ~0ull, n_ties = 0;
    void fold(const ChunkMin &r, uint64_t first) {
        const bool less = !any || r.hi < hi || (r.hi == hi && r.lo < lo);
        if (less) {
            any = true; hi = r.hi; lo = r.lo; index = first + r.index; n_ties = 0;
            next = r.next == ~0u ? ~0ull : first + r.next;
        } else if (r.hi != hi || r.lo != lo) {
            return;
        } else {
            next = std::min(next, first + r.index);   // chunks arrive in ascending order: above index
        }
        n_ties += r.n_ties;
    }
};

}  // namespace

int stored_vrf_search(const std::string &dir, b200post_post_metadata *md, const b200post_vrf_search_opts &o, b200post_vrf_nonce *out,
                      const volatile int *cancel) {
    memset(out, 0, sizeof *out);
    const uint64_t batch = o.compute_batch_size ? o.compute_batch_size : 1ull << 20;
    uint64_t chunk = o.chunk_labels ? o.chunk_labels : 1ull << 22;
    if (o.provider_id < 0 && o.provider_id != B200POST_PROVIDER_ALL) return fail(B200POST_ERR_INVALID_ARGUMENT, "invalid provider id");
    if (chunk > kMaxChunk) return fail(B200POST_ERR_INVALID_ARGUMENT, "chunk_labels above 2^26");

    // ---- metadata and files, on the host before any device is touched
    if (int rc = check_layout(*md)) return rc;
    const Layout lay(*md);
    if (int rc = check_post_files(dir, lay, 0, lay.n_files - 1)) return rc;
    const uint64_t N = md->scrypt_n, num_labels = lay.num_labels;

    // ---- device: the scan runs on one (it is bound by storage, not by the GPU)
    std::vector<uint32_t> devs;
    if (int rc = provider_devices(o.provider_id, &devs)) return rc;
    DeviceEngine *e;
    if (int rc = device_engine(devs[0], &e)) return rc;
    chunk = std::min(chunk, num_labels);

    Running best;
    {
        PostDataReader reader(dir, lay.per_file);
        StoredScan scan;
        int rc = scan.init(e, chunk);
        if (rc) return rc;
        const uint64_t n_chunks = (num_labels + chunk - 1) / chunk;
        auto count_of = [&](uint64_t k) { return std::min<uint64_t>(chunk, num_labels - k * chunk); };
        // the reader: chunk k into staging(k & 1), once the chunk two back has left it
        auto load = [&](uint64_t k) -> std::pair<int, std::string> {
            int r = scan.wait_copied((int)(k & 1));
            if (!r) r = reader.read(k * chunk, count_of(k), scan.staging((int)(k & 1)));
            return {r, r ? last_error() : ""};
        };
        std::future<std::pair<int, std::string>> next = std::async(std::launch::async, load, (uint64_t)0);
        for (uint64_t k = 0; k < n_chunks; k++) {
            const int b = (int)(k & 1);
            const auto got = next.get();
            if (got.first) return fail(got.first, got.second);
            if (cancel && *cancel) return fail(B200POST_ERR_CANCELLED, "cancelled");
            if ((rc = scan.submit(b, (uint32_t)count_of(k)))) return rc;
            if (k + 1 < n_chunks) next = std::async(std::launch::async, load, k + 1);
            if (k > 0) {
                ChunkMin r;
                if ((rc = scan.collect(b ^ 1, &r))) return rc;
                best.fold(r, (k - 1) * chunk);
                if (o.progress) __atomic_fetch_add(o.progress, count_of(k - 1), __ATOMIC_RELAXED);
            }
        }
        ChunkMin r;
        if ((rc = scan.collect((int)((n_chunks - 1) & 1), &r))) return rc;
        best.fold(r, (n_chunks - 1) * chunk);
        if (o.progress) __atomic_fetch_add(o.progress, count_of(n_chunks - 1), __ATOMIC_RELAXED);
    }

    // ---- the label32 of the two lowest positions at the lowest prefix, recomputed; a stored prefix it does not reproduce
    // is damage.  index first: if it is damaged it is the lowest damaged position, else next is the lowest copy of it.
    uint8_t prefix[16];
    for (int j = 0; j < 8; j++) { prefix[j] = (uint8_t)(best.hi >> (56 - 8 * j)); prefix[8 + j] = (uint8_t)(best.lo >> (56 - 8 * j)); }
    std::vector<uint64_t> pos{best.index};
    if (best.next != ~0ull) pos.push_back(best.next);
    uint8_t commitment[32], best32[32];
    commitment_bytes(md->node_id, md->commitment_atx_id, commitment);
    uint64_t best_index = 0;
    for (size_t j = 0; j < pos.size(); j++) {
        uint8_t l32[32];
        if (int rc = label32_at(e, commitment, N, pos[j], l32)) return rc;
        if (memcmp(l32, prefix, 16))
            return fail(B200POST_ERR_LABEL_MISMATCH, "the stored label at index " + std::to_string(pos[j]) +
                                                         " differs from its recomputation: the POST data is damaged");
        if (j == 0 || memcmp(l32, best32, 32) < 0) { memcpy(best32, l32, 32); best_index = pos[j]; }
    }
    if (best.n_ties > pos.size())
        return fail(B200POST_ERR_LABEL_MISMATCH, std::to_string(best.n_ties) + " stored labels share the smallest 16-byte prefix: the POST data is damaged");

    return settle_nonce(dir, md, best_index, best32, o.provider_id, batch, out, nullptr, cancel);
}

// The rule of an init: below the threshold, or the past-the-end search.
int settle_nonce(const std::string &dir, b200post_post_metadata *md, uint64_t best_index, const uint8_t best32[32], int64_t provider_id,
                 uint64_t batch, b200post_vrf_nonce *out, bool *past_end, const volatile int *cancel) {
    const uint64_t num_labels = (uint64_t)md->num_units * md->labels_per_unit;
    uint8_t diff[32], commitment[32];
    vrf_difficulty(num_labels, diff);
    commitment_bytes(md->node_id, md->commitment_atx_id, commitment);
    const bool below = memcmp(best32, diff, 32) < 0;
    if (past_end) *past_end = !below;
    if (below) {
        md->has_nonce = 1; md->nonce = best_index; memcpy(md->nonce_value, best32, 32); md->last_position = 0;
    } else {
        // a recorded nonce is replaced, so the search starts at numLabels; without one it resumes a stopped search.
        // The marker stays set until the search ends, so a stopped search is finished by the next search or session.
        if (md->has_nonce) md->last_position = 0;
        md->has_nonce = 0; md->vrf_scan_pending = 1;
        if (int rc = search_past_end(dir, md, num_labels, provider_id, batch, commitment, diff, cancel)) return rc;
    }
    md->vrf_scan_pending = 0;
    if (int rc = save_post_metadata(dir, *md)) return rc;
    out->found = 1; out->index = md->nonce; memcpy(out->label32, md->nonce_value, 32);
    return B200POST_OK;
}

}  // namespace b200post

using namespace b200post;

extern "C" {

void b200post_default_vrf_search_opts(b200post_vrf_search_opts *o) {
    if (!o) return;
    memset(o, 0, sizeof *o);
    o->provider_id = 0; o->compute_batch_size = 1ull << 20; o->chunk_labels = 1ull << 22; o->progress = nullptr;
}

int b200post_search_vrf_nonce(const char *data_dir, const b200post_vrf_search_opts *o, b200post_vrf_nonce *out, const volatile int *cancel) {
    if (!data_dir || !o || !out) return fail(B200POST_ERR_INVALID_ARGUMENT, "invalid argument");
    b200post_post_metadata md;
    if (int rc = load_post_metadata(data_dir, &md)) return rc;
    return stored_vrf_search(data_dir, &md, *o, out, cancel);
}

}  // extern "C"
