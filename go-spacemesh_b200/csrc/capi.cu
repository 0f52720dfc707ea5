// capi.cu — extern "C" surface of libb200post.so (declared in include/b200post.h, include/post_compat.h).
#include <algorithm>
#include <chrono>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/b200post.h"
#include "../../include/b200post_verify.h"
#include "../../include/post_compat.h"
#include "engine.h"
#include "host_hash.h"
#include "randomx_engine.h"

using namespace b200post;

namespace {

// N is a power of two in [2, 2^20]: one scratchpad is 128*N bytes (128 MiB at the cap) and a warp's
// region (N * 4 KiB) must stay within 4 GiB for the kernels' 32-bit in-region addressing.
bool valid_n(uint64_t n) { return n >= 2 && n <= (1ull << 20) && (n & (n - 1)) == 0; }

void fill_nonce(b200post_vrf_nonce *dst, const VrfResult &r) {
    if (!dst) return;
    memset(dst, 0, sizeof *dst);
    dst->found = r.found ? 1 : 0;
    if (r.found) { dst->index = r.index; memcpy(dst->label32, r.label32, 32); }
}

int range_common(uint32_t provider, const uint8_t *commitment, uint64_t n, uint64_t start, uint64_t count,
                 uint8_t *out_host, uint8_t *out_dev, const uint8_t *vrf_difficulty, b200post_vrf_nonce *nonce,
                 const volatile int *cancel) {
    if (!commitment || !valid_n(n) || (vrf_difficulty && !nonce) || (count && start + (count - 1) < start)) {
        set_error("invalid argument (commitment NULL, N not a power of two in [2, 2^20], missing nonce out, or index overflow)");
        return B200POST_ERR_INVALID_ARGUMENT;
    }
    DeviceEngine *e;
    if (int rc = device_engine(provider, &e)) return rc;
    VrfResult vr;
    const int rc = e->labels_range(commitment, n, start, count, out_host, out_dev, vrf_difficulty, &vr, cancel);
    if (rc == B200POST_OK) fill_nonce(nonce, vr);
    return rc;
}

}  // namespace

extern "C" {

int b200post_providers(b200post_provider *out, int max) {
    const int n = device_count();
    for (int i = 0; i < n && out && i < max; i++) {
        cudaDeviceProp p;
        if (cudaGetDeviceProperties(&p, i) != cudaSuccess) continue;
        memset(&out[i], 0, sizeof out[i]);
        out[i].id = (uint32_t)i;
        out[i].device_class = B200POST_DEVICE_CLASS_GPU;
        strncpy(out[i].model, p.name, sizeof(out[i].model) - 1);
        out[i].hbm_bytes = p.totalGlobalMem;
        out[i].sm_count = (uint32_t)p.multiProcessorCount;
        out[i].cc_major = (uint32_t)p.major; out[i].cc_minor = (uint32_t)p.minor;
    }
    return n;
}

const char *b200post_last_error(void) { return last_error(); }

int b200post_set_option(const char *key, int64_t value) {
    if (!key) return B200POST_ERR_INVALID_ARGUMENT;
    Options &o = options();
    const std::string k(key);
    if (k == "romix_variant" && value >= 0 && value <= 5) { o.romix_variant = value; return B200POST_OK; }
    if (k == "rotate_mask" && value >= 0 && value <= 1 && romix_mask_supported((int)value)) { o.rotate_mask = value; return B200POST_OK; }
    if (k == "tpb" && (value == 64 || value == 128 || value == 256 || value == 512)) { o.tpb = value; return B200POST_OK; }
    if (k == "dr_unroll" && (value == 1 || value == 4)) { o.dr_unroll = value; return B200POST_OK; }
    if (k == "ctas_per_sm" && value >= 0 && value <= 32) { o.ctas_per_sm = value; return B200POST_OK; }
    if (k == "max_scratch_mib" && value >= 0) { o.max_scratch_mib = value; return B200POST_OK; }
    if (k == "speculate_next" && (value == 0 || value == 1)) { o.speculate_next = value; return B200POST_OK; }
    if (k == "debug_corrupt_next_batch" && (value == 0 || value == 1)) { o.debug_corrupt_next_batch = value; return B200POST_OK; }
    if (k == "debug_corrupt_check_all" && (value == 0 || value == 1)) { o.debug_corrupt_check_all = value; return B200POST_OK; }
    if (k == "lowlat_max_labels" && value >= 0 && value <= (1 << 20)) { o.lowlat_max_labels = value; return B200POST_OK; }
    if (k == "rx_vm_mode" && value >= 0 && value <= 3) { o.rx_vm_mode = value; return B200POST_OK; }
    if (k == "rx_vms_per_sm" && value >= 0 && value <= 4096) { o.rx_vms_per_sm = value; return B200POST_OK; }
    if (k == "debug_skip_phase" && value >= 0 && value <= 3) { o.debug_skip_phase = value; return B200POST_OK; }
    set_error("unknown option or value out of range: " + k);
    return B200POST_ERR_INVALID_ARGUMENT;
}

int64_t b200post_get_option(const char *key) {
    if (!key) return -1;
    Options &o = options();
    const std::string k(key);
    if (k == "romix_variant") return o.romix_variant;
    if (k == "rotate_mask") return o.rotate_mask;
    if (k == "tpb") return o.tpb;
    if (k == "dr_unroll") return o.dr_unroll;
    if (k == "ctas_per_sm") return o.ctas_per_sm;
    if (k == "max_scratch_mib") return o.max_scratch_mib;
    if (k == "speculate_next") return o.speculate_next;
    if (k == "rx_vms_per_sm") return o.rx_vms_per_sm;
    if (k == "rx_vm_mode") return o.rx_vm_mode;
    if (k == "lowlat_max_labels") return o.lowlat_max_labels;
    if (k == "debug_skip_phase") return o.debug_skip_phase;
    return -1;
}

int b200post_labels_range(uint32_t provider, const uint8_t commitment[32], uint64_t n, uint64_t start, uint64_t count,
                          uint8_t *out16, const uint8_t *vrf_difficulty, b200post_vrf_nonce *nonce,
                          const volatile int *cancel) {
    return range_common(provider, commitment, n, start, count, out16, nullptr, vrf_difficulty, nonce, cancel);
}

int b200post_labels_range_dev(uint32_t provider, const uint8_t commitment[32], uint64_t n, uint64_t start, uint64_t count,
                              void *d_out16, const uint8_t *vrf_difficulty, b200post_vrf_nonce *nonce,
                              const volatile int *cancel) {
    if (d_out16 && ((uintptr_t)d_out16 & 15)) { set_error("d_out16 must be 16-byte aligned"); return B200POST_ERR_INVALID_ARGUMENT; }
    return range_common(provider, commitment, n, start, count, nullptr, (uint8_t *)d_out16, vrf_difficulty, nonce, cancel);
}

int b200post_labels_range_multi(const uint32_t *providers, int n_providers, const uint8_t commitment[32], uint64_t n,
                                uint64_t start, uint64_t count, uint8_t *out16, const uint8_t *vrf_difficulty,
                                b200post_vrf_nonce *nonce, const volatile int *cancel) {
    if (!providers || n_providers <= 0) { set_error("no providers given"); return B200POST_ERR_INVALID_ARGUMENT; }
    if (n_providers == 1) return b200post_labels_range(providers[0], commitment, n, start, count, out16, vrf_difficulty, nonce, cancel);
    // contiguous shards: device g gets [start + g*per, start + (g+1)*per) — keeps each device's output a
    // contiguous slice of the POST data (SURVEY.md §8e)
    const uint64_t per = (count + (uint64_t)n_providers - 1) / (uint64_t)n_providers;
    std::vector<b200post_vrf_nonce> nonces((size_t)n_providers);
    const int rc = fan_out((size_t)n_providers, [&](size_t g) {
        const uint64_t off = std::min<uint64_t>(per * (uint64_t)g, count);
        const uint64_t cnt = std::min<uint64_t>(per, count - off);
        memset(&nonces[g], 0, sizeof(b200post_vrf_nonce));
        const int r = b200post_labels_range(providers[g], commitment, n, start + off, cnt, out16 ? out16 + off * 16 : nullptr,
                                            vrf_difficulty, vrf_difficulty ? &nonces[g] : nullptr, cancel);
        if (r) set_error("provider " + std::to_string(providers[g]) + ": " + last_error());
        return r;
    });
    if (rc) return rc;
    if (vrf_difficulty && nonce) {
        memset(nonce, 0, sizeof *nonce);
        for (const b200post_vrf_nonce &c : nonces)
            if (c.found && (!nonce->found || vrf_less(c.label32, c.index, nonce->label32, nonce->index))) *nonce = c;
    }
    return B200POST_OK;
}

int b200post_labels_gather(uint32_t provider, size_t n_items, const uint8_t *commitments, const uint64_t *indices,
                           uint64_t n, uint8_t *out16) {
    if (!valid_n(n) || (n_items && (!commitments || !indices || !out16))) {
        set_error("invalid argument");
        return B200POST_ERR_INVALID_ARGUMENT;
    }
    DeviceEngine *e;
    if (int rc = device_engine(provider, &e)) return rc;
    return e->labels_gather(n_items, commitments, indices, n, out16);
}

int b200post_labels_gather_indexed(uint32_t provider, size_t n_items, size_t n_commitments, const uint8_t *commitments,
                                   const uint32_t *commitment_index, const uint64_t *indices, uint64_t n, uint8_t *out16) {
    if (!valid_n(n) || (n_items && (!commitments || !commitment_index || !indices || !out16 || !n_commitments)) ||
        n_commitments > 0xffffffffull) {
        set_error("invalid argument");
        return B200POST_ERR_INVALID_ARGUMENT;
    }
    for (size_t i = 0; i < n_items; i++)
        if (commitment_index[i] >= n_commitments) { set_error("commitment_index out of range"); return B200POST_ERR_INVALID_ARGUMENT; }
    DeviceEngine *e;
    if (int rc = device_engine(provider, &e)) return rc;
    return e->labels_gather_indexed(n_items, n_commitments, commitments, commitment_index, indices, n, out16, nullptr);
}

void b200post_commitment(const uint8_t node_id[32], const uint8_t commitment_atx_id[32], uint8_t out[32]) {
    commitment_bytes(node_id, commitment_atx_id, out);
}

void b200post_vrf_difficulty(uint64_t num_labels, uint8_t out[32]) { vrf_difficulty(num_labels, out); }

// The one-check case of b200post_verify_vrf_nonces (one path for every VRF-nonce check).  The check's own arguments are
// judged here first, so that they keep their codes before the provider and device checks of the batch call.
static int vrf_check_one(uint32_t provider, uint64_t nonce, const uint8_t node_id[32], const uint8_t commitment_atx_id[32],
                         uint32_t num_units, uint64_t labels_per_unit, uint64_t n, int *valid, uint8_t label32[32]) {
    if (!valid_n(n)) { set_error("invalid argument (N not a power of two in [2, 2^20])"); return B200POST_ERR_INVALID_ARGUMENT; }
    b200post_vrf_check c;
    memset(&c, 0, sizeof c);
    memcpy(c.node_id, node_id, 32);
    memcpy(c.commitment_atx_id, commitment_atx_id, 32);
    c.nonce = nonce; c.num_units = num_units; c.labels_per_unit = labels_per_unit; c.scrypt_n = n;
    int status = B200POST_OK;
    const int rc = b200post_verify_vrf_nonces(provider, 1, &c, &status, valid, label32);
    return rc ? rc : status;
}

int b200post_verify_vrf_nonce(uint32_t provider, uint64_t nonce, const uint8_t node_id[32],
                              const uint8_t commitment_atx_id[32], uint32_t num_units, uint64_t labels_per_unit,
                              uint64_t n, int *valid) {
    if (!node_id || !commitment_atx_id || !valid) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    *valid = 0;
    const unsigned __int128 total = (unsigned __int128)num_units * labels_per_unit;
    if (total == 0 || total > ~0ull) { set_error("num_units * labels_per_unit out of range"); return B200POST_ERR_INVALID_ARGUMENT; }
    int ok = 0;
    const int rc = vrf_check_one(provider, nonce, node_id, commitment_atx_id, num_units, labels_per_unit, n, &ok, nullptr);
    if (rc) return rc;
    *valid = ok;
    return B200POST_OK;
}

int b200post_vrf_nonce_label(uint32_t provider, uint64_t nonce, const uint8_t node_id[32], const uint8_t commitment_atx_id[32],
                             uint64_t n, uint8_t label32[32]) {
    if (!node_id || !commitment_atx_id || !label32) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    int ok = 0;
    uint8_t l32[32];
    // the label does not depend on numLabels: one label suffices for a well-formed check
    const int rc = vrf_check_one(provider, nonce, node_id, commitment_atx_id, 1, 1, n, &ok, l32);
    if (rc) return rc;
    memcpy(label32, l32, 32);
    return B200POST_OK;
}

int b200post_benchmark(uint32_t provider, uint64_t n, double seconds, double *labels_per_sec) {
    if (!labels_per_sec || !valid_n(n)) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    uint8_t commitment[32];
    memset(commitment, 0x5a, 32);
    DeviceEngine *e;
    if (int rc = device_engine(provider, &e)) return rc;
    // batches of 4 whole layers (the software pipeline needs >= 4 to run filled, and back-to-back calls continue it:
    // DeviceEngine's speculative next-layer fill); the first call allocates the scratch and is not timed
    uint64_t slots = 0;
    int rc = b200post_wave_slots(provider, n, &slots);
    if (rc) return rc;
    const uint64_t batch = std::max<uint64_t>(4 * slots, 1u << 16);
    rc = b200post_labels_range(provider, commitment, n, 0, batch, nullptr, nullptr, nullptr, nullptr);
    if (rc) return rc;
    const auto t0 = std::chrono::steady_clock::now();
    uint64_t done = 0;
    double el = 0;
    do {
        rc = b200post_labels_range(provider, commitment, n, batch + done, batch, nullptr, nullptr, nullptr, nullptr);
        if (rc) return rc;
        done += batch;
        el = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    } while (el < seconds);
    *labels_per_sec = (double)done / el;
    return B200POST_OK;
}

uint64_t b200post_launch_count(void) { return g_launches.load(); }

int b200post_romix_time(uint32_t provider, double *ms_total, uint64_t *launches, double *labels, int reset) {
    DeviceEngine *e = engine_for(provider);
    if (!e) return B200POST_ERR_NO_DEVICE;
    e->romix_time(ms_total, launches, labels, reset != 0);
    return B200POST_OK;
}

int b200post_wave_slots(uint32_t provider, uint64_t n, uint64_t *slots) {
    if (!slots || !valid_n(n)) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    DeviceEngine *e;
    if (int rc = device_engine(provider, &e)) return rc;
    *slots = e->wave_slots(n);
    return *slots ? B200POST_OK : B200POST_ERR_CUDA;
}

int b200post_timer_mark(uint32_t provider, int which) {
    DeviceEngine *e = engine_for(provider);
    return e ? e->timer_mark(which) : B200POST_ERR_NO_DEVICE;
}

double b200post_timer_elapsed_ms(uint32_t provider) {
    DeviceEngine *e = engine_for(provider);
    return e ? e->timer_elapsed_ms() : -1.0;
}

double b200post_last_call_ms(uint32_t provider) {
    DeviceEngine *e = engine_for(provider);
    return e ? e->last_call_ms() : -1.0;
}

int b200post_reference_label(const uint8_t commitment[32], uint64_t index, uint64_t n, uint8_t out32[32]) {
    if (!commitment || !out32 || !valid_n(n)) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    reference_label32(commitment, index, (uint32_t)n, out32);
    return B200POST_OK;
}

void b200post_shutdown(void) { randomx_shutdown_all(); shutdown_all(); }

// ------------------------------------------------------------------------------------------------
// libpost-compatible symbols (include/post_compat.h)
// ------------------------------------------------------------------------------------------------
struct Initializer {
    uint32_t provider;
    uint64_t n;
    uint8_t commitment[32];
    bool has_vrf;
    uint8_t vrf[32];
};

size_t get_providers_count(void) { return (size_t)device_count(); }

DeviceInfoResult get_providers(Provider *out, size_t out_len) {
    if (!out && out_len) return DeviceInfoInvalidArgument;
    const int n = device_count();
    if ((size_t)n > out_len) return DeviceInfoBufferTooSmall;
    for (int i = 0; i < n; i++) {
        cudaDeviceProp p;
        if (cudaGetDeviceProperties(&p, i) != cudaSuccess) return DeviceInfoFailed;
        memset(&out[i], 0, sizeof out[i]);
        strncpy(out[i].name, p.name, sizeof(out[i].name) - 1);
        out[i].id = (uint32_t)i;
        out[i].class_ = DeviceClassGPU;
    }
    return DeviceInfoOk;
}

Initializer *new_initializer(uint32_t provider_id, size_t n, const uint8_t *commitment, const uint8_t *vrf_difficulty) {
    if (!commitment || !valid_n(n)) { set_error("new_initializer: invalid argument"); return nullptr; }
    if (!engine_for(provider_id)) return nullptr;   // includes the CPU id: no CPU path in this library
    Initializer *i = new Initializer;
    i->provider = provider_id; i->n = n;
    memcpy(i->commitment, commitment, 32);
    i->has_vrf = vrf_difficulty != nullptr;
    if (i->has_vrf) memcpy(i->vrf, vrf_difficulty, 32);
    return i;
}

InitializeResult initialize(Initializer *init, uint64_t start, uint64_t end, uint8_t *out, uint64_t *nonce) {
    if (!init) return InitializeInvalidArgument;
    if (end < start) return InitializeInvalidLabelsRange;
    const uint64_t count = end - start + 1;   // end is inclusive
    if (count == 0) return InitializeInvalidLabelsRange;   // [0, 2^64-1] overflows
    b200post_vrf_nonce r;
    const int rc = b200post_labels_range(init->provider, init->commitment, init->n, start, count, out,
                                         init->has_vrf ? init->vrf : nullptr, init->has_vrf ? &r : nullptr, nullptr);
    if (rc == B200POST_ERR_INVALID_ARGUMENT) return InitializeInvalidArgument;
    if (rc) return InitializeError;
    if (init->has_vrf && r.found) {
        if (nonce) *nonce = r.index;
        return InitializeOk;
    }
    return InitializeOkNonceNotFound;   // also when no difficulty was given (libpost: vrf_nonce == None)
}

void free_initializer(Initializer *init) { delete init; }

}  // extern "C"
