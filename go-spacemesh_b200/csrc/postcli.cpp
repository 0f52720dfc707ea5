// postcli.cpp — `b200postcli`: a postcli-compatible initialisation CLI on top of libb200post.so.
//
// The reference deploys POST data with an init container running `postcli` (systest/cluster/nodes.go:990-999):
//   postcli -id <hex pubkey> -commitmentAtxId <hex> -datadir /data -numUnits N -labelsPerUnit L -scryptN 8192
//           -provider 4294967295 -yes
// This tool accepts the same flags (single-dash, Go `flag` style; "-flag value" or "-flag=value") and drives a
// PostSetupManager session (include/b200post_setup.h).  Differences: `-provider` takes a CUDA ordinal or
// "all"; the CPU provider id 4294967295 is refused (the library has no CPU path).
//
// `-verify` checks data already on disk instead (postcli's flags as recalled, unpinned):
//   b200postcli -verify -datadir /data [-fraction 0.2] [-fromFile 0] [-toFile N] [-seed S] [-provider 0|all]
// recomputes `-fraction` percent of each file's labels on the GPU, prints `file N offset K (label I)` for each
// reported mismatch and exits 0 when the data is valid, 1 otherwise.
//
// One POST initialised on several machines (postcli's flag names as recalled, unpinned):
//   b200postcli <init flags> -fromFile A -toFile B      writes only postdata_A.bin .. postdata_B.bin
//   b200postcli -printNumFiles -numUnits N -labelsPerUnit L [-maxFileSize S]   how many files the POST has
//   b200postcli -searchForNonce -datadir D [-provider 0|all] [-computeBatchSize B]
// The last one finds the VRF nonce of the merged files from their stored labels and writes it to the metadata.
//
// The initial proof (the proof for the zero challenge a node asks for right after initialisation) from the labels as
// the session computes them, so that the node's post-service need not read the whole POST back:
//   b200postcli <init flags> -initialProof [-nonces 288] [-k1 26] [-k2 37] [-powDifficulty <64 hex digits>]
// writes initial_post.json into the data dir (k2pow on the session's devices).  Not with -fromFile / -toFile.
// Exit codes: 0 ok, 1 error or damaged data, 2 usage, 130 stopped.
#include <signal.h>

#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <cstring>
#include <string>
#include <thread>

#include "../../include/b200post_prove.h"

static volatile int g_cancel = 0;
static void on_signal(int) { g_cancel = 1; }

static bool unhex32(const std::string &s, uint8_t out[32]) {
    if (s.size() != 64) return false;
    for (int i = 0; i < 32; i++) {
        unsigned v;
        if (sscanf(s.c_str() + 2 * i, "%2x", &v) != 1) return false;
        out[i] = (uint8_t)v;
    }
    return true;
}

static int run_verify(const std::string &datadir, const std::string &provider, double fraction, uint64_t from_file, int64_t to_file,
                      uint64_t seed) {
    b200post_verify_pos_opts o;
    b200post_default_verify_pos_opts(&o);
    o.provider_id = provider == "all" ? B200POST_PROVIDER_ALL : (int64_t)strtoull(provider.c_str(), nullptr, 10);
    if (o.provider_id == (int64_t)B200POST_CPU_PROVIDER_ID) { fprintf(stderr, "provider 4294967295 (CPU) is not served: this build has no CPU path\n"); return 2; }
    o.fraction = fraction; o.from_file = from_file; o.to_file = to_file; o.seed = seed;
    // what the progress line counts towards: the sample sizes of the checked files
    uint64_t total = 0, per_file = 0;
    b200post_post_metadata md;
    if (b200post_load_metadata(datadir.c_str(), &md) == 0 && md.max_file_size >= 16) {
        const uint64_t nl = (uint64_t)md.num_units * md.labels_per_unit;
        per_file = md.max_file_size / 16;
        const uint64_t n_files = (nl + per_file - 1) / per_file, last = to_file < 0 ? n_files - 1 : (uint64_t)to_file;
        for (uint64_t f = from_file; f <= last && f < n_files; f++) {
            uint64_t n = 0;
            if (b200post_verify_pos_sample(1, f, std::min(per_file, nl - f * per_file), fraction, nullptr, 0, &n) == 0) total += n;
        }
    }
    volatile uint64_t progress = 0;
    o.progress = &progress;
    signal(SIGINT, on_signal); signal(SIGTERM, on_signal);
    b200post_verify_pos_result r;
    volatile int done = 0;
    std::thread show([&] {
        const auto t0 = std::chrono::steady_clock::now();
        while (!done) {
            for (int k = 0; k < 20 && !done; k++) std::this_thread::sleep_for(std::chrono::milliseconds(100));
            const double el = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
            const uint64_t p = progress;
            fprintf(stderr, "\r%llu / %llu labels checked (%.1f %%), %.0f labels/s   ", (unsigned long long)p, (unsigned long long)total,
                    total ? 100.0 * p / (double)total : 0.0, el > 0 ? p / el : 0.0);
        }
        fprintf(stderr, "\n");
    });
    const int rc = b200post_verify_pos(datadir.c_str(), &o, &r, &g_cancel);
    done = 1;
    show.join();
    if (rc == B200POST_ERR_CANCELLED) { fprintf(stderr, "stopped\n"); return 130; }
    if (rc != 0 && rc != B200POST_ERR_LABEL_MISMATCH && rc != B200POST_ERR_STATE) { fprintf(stderr, "verify failed: %s (%d)\n", b200post_last_error(), rc); return 1; }
    printf("checked %llu labels in %llu files (seed %llu): %llu mismatches\n", (unsigned long long)r.labels_checked,
           (unsigned long long)r.files_checked, (unsigned long long)r.seed, (unsigned long long)r.mismatches);
    for (uint32_t i = 0; i < r.n_reported && per_file; i++)
        printf("file %llu offset %llu (label %llu)\n", (unsigned long long)(r.bad_index[i] / per_file),
               (unsigned long long)(r.bad_index[i] % per_file * 16), (unsigned long long)r.bad_index[i]);
    if (rc == B200POST_ERR_STATE) printf("%s\n", b200post_last_error());
    else if (!r.nonce_ok) printf("the VRF nonce's label does not match the metadata\n");
    if (r.argmin_checked) printf("VRF nonce is the arg-min of the data: %s\n", r.argmin_ok ? "yes" : "no");
    if (rc == 0) { printf("POST data is valid\n"); return 0; }
    printf(rc == B200POST_ERR_STATE ? "POST data is not complete\n" : "POST data is INVALID\n");
    return 1;
}

static int run_search(const std::string &datadir, const std::string &provider, uint64_t batch) {
    b200post_vrf_search_opts o;
    b200post_default_vrf_search_opts(&o);
    o.provider_id = provider == "all" ? B200POST_PROVIDER_ALL : (int64_t)strtoull(provider.c_str(), nullptr, 10);
    if (o.provider_id == (int64_t)B200POST_CPU_PROVIDER_ID) { fprintf(stderr, "provider 4294967295 (CPU) is not served: this build has no CPU path\n"); return 2; }
    o.compute_batch_size = batch;
    uint64_t total = 0;
    b200post_post_metadata md;
    if (b200post_load_metadata(datadir.c_str(), &md) == 0) total = (uint64_t)md.num_units * md.labels_per_unit;
    volatile uint64_t progress = 0;
    o.progress = &progress;
    signal(SIGINT, on_signal); signal(SIGTERM, on_signal);
    volatile int done = 0;
    std::thread show([&] {
        const auto t0 = std::chrono::steady_clock::now();
        while (!done) {
            for (int k = 0; k < 20 && !done; k++) std::this_thread::sleep_for(std::chrono::milliseconds(100));
            const double el = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
            const uint64_t p = progress;
            fprintf(stderr, "\r%llu / %llu stored labels scanned (%.1f %%), %.0f labels/s   ", (unsigned long long)p, (unsigned long long)total,
                    total ? 100.0 * p / (double)total : 0.0, el > 0 ? p / el : 0.0);
        }
        fprintf(stderr, "\n");
    });
    b200post_vrf_nonce nn;
    const int rc = b200post_search_vrf_nonce(datadir.c_str(), &o, &nn, &g_cancel);
    done = 1;
    show.join();
    if (rc == B200POST_ERR_CANCELLED) { fprintf(stderr, "stopped; run again to finish the search\n"); return 130; }
    if (rc) { fprintf(stderr, "search failed: %s (%d)\n", b200post_last_error(), rc); return 1; }
    printf("VRF nonce %llu\n", (unsigned long long)nn.index);
    return 0;
}

int main(int argc, char **argv) {
    std::string id, atx, datadir = "./post-data", provider = "0";
    uint64_t num_units = 0, labels_per_unit = 0, scrypt_n = 8192, max_file_size = 4ull << 30, batch = 1ull << 20;
    bool print_providers = false, verify = false, print_num_files = false, search = false, range = false, initial = false;
    uint32_t nonces = 288, k1 = 0, k2 = 0;
    std::string pow_difficulty;
    double fraction = 0.2;
    uint64_t from_file = 0, seed = 0;
    int64_t to_file = -1;
    for (int i = 1; i < argc; i++) {
        std::string a = argv[i], v;
        while (!a.empty() && a[0] == '-') a.erase(0, 1);
        const size_t eq = a.find('=');
        if (eq != std::string::npos) { v = a.substr(eq + 1); a = a.substr(0, eq); }
        auto val = [&]() -> std::string { if (eq != std::string::npos) return v; return i + 1 < argc ? argv[++i] : ""; };
        if (a == "id") id = val();
        else if (a == "commitmentAtxId") atx = val();
        else if (a == "datadir") datadir = val();
        else if (a == "numUnits") num_units = strtoull(val().c_str(), nullptr, 10);
        else if (a == "labelsPerUnit") labels_per_unit = strtoull(val().c_str(), nullptr, 10);
        else if (a == "scryptN") scrypt_n = strtoull(val().c_str(), nullptr, 10);
        else if (a == "maxFileSize") max_file_size = strtoull(val().c_str(), nullptr, 10);
        else if (a == "computeBatchSize") batch = strtoull(val().c_str(), nullptr, 10);
        else if (a == "provider") provider = val();
        else if (a == "printProviders") print_providers = true;
        else if (a == "yes") {}
        else if (a == "verify") verify = true;
        else if (a == "fraction") fraction = strtod(val().c_str(), nullptr);
        else if (a == "fromFile") { from_file = strtoull(val().c_str(), nullptr, 10); range = true; }
        else if (a == "toFile") { to_file = strtoll(val().c_str(), nullptr, 10); range = true; }
        else if (a == "printNumFiles") print_num_files = true;
        else if (a == "searchForNonce") search = true;
        else if (a == "seed") seed = strtoull(val().c_str(), nullptr, 10);
        else if (a == "initialProof") initial = true;
        else if (a == "nonces") nonces = (uint32_t)strtoul(val().c_str(), nullptr, 10);
        else if (a == "k1") k1 = (uint32_t)strtoul(val().c_str(), nullptr, 10);
        else if (a == "k2") k2 = (uint32_t)strtoul(val().c_str(), nullptr, 10);
        else if (a == "powDifficulty") pow_difficulty = val();
        else { fprintf(stderr, "unknown flag -%s\n", a.c_str()); return 2; }
    }
    if (print_providers) {
        b200post_provider p[16];
        const int n = b200post_providers(p, 16);
        for (int k = 0; k < n && k < 16; k++) printf("{ID: %u, Model: \"%s\", DeviceType: GPU, HBM: %llu}\n", p[k].id, p[k].model, (unsigned long long)p[k].hbm_bytes);
        return 0;
    }
    if (print_num_files) {
        const unsigned __int128 nl = (unsigned __int128)num_units * (labels_per_unit ? labels_per_unit : 512);
        if (nl == 0 || max_file_size < 16 || max_file_size % 16) { fprintf(stderr, "-numUnits, -labelsPerUnit and -maxFileSize (a multiple of 16) must be positive\n"); return 2; }
        const unsigned __int128 per_file = max_file_size / 16;
        printf("%llu\n", (unsigned long long)((nl + per_file - 1) / per_file));
        return 0;
    }
    if (verify) return run_verify(datadir, provider, fraction, from_file, to_file, seed);
    if (search) return run_search(datadir, provider, batch);
    uint8_t node_id[32], atx_id[32];
    if (!unhex32(id, node_id) || !unhex32(atx, atx_id)) { fprintf(stderr, "-id and -commitmentAtxId must be 32-byte hex strings\n"); return 2; }
    b200post_post_config cfg;
    b200post_default_post_config(&cfg);
    if (labels_per_unit) cfg.labels_per_unit = labels_per_unit;
    cfg.min_num_units = 1; cfg.max_num_units = 1u << 20;
    if (initial && range) { fprintf(stderr, "-initialProof needs the whole POST: it cannot be combined with -fromFile / -toFile\n"); return 2; }
    if (k1) cfg.k1 = k1;
    if (k2) cfg.k2 = cfg.k3 = k2;
    if (!pow_difficulty.empty() && !unhex32(pow_difficulty, cfg.pow_difficulty)) { fprintf(stderr, "-powDifficulty must be a 32-byte hex string\n"); return 2; }
    b200post_setup_opts o;
    b200post_default_setup_opts(&o);
    o.data_dir = datadir.c_str(); o.num_units = (uint32_t)num_units; o.scrypt_n = scrypt_n; o.max_file_size = max_file_size;
    o.compute_batch_size = batch;
    if (provider == "all") o.provider_id = B200POST_PROVIDER_ALL;
    else o.provider_id = (int64_t)strtoull(provider.c_str(), nullptr, 10);
    if (o.provider_id == (int64_t)B200POST_CPU_PROVIDER_ID) { fprintf(stderr, "provider 4294967295 (CPU) is not served: this build has no CPU path\n"); return 2; }

    b200post_setup_manager *mgr = nullptr;
    if (b200post_setup_manager_new(&cfg, &mgr)) { fprintf(stderr, "error: %s\n", b200post_last_error()); return 1; }
    if (int rc = b200post_setup_prepare_files(mgr, &o, node_id, atx_id, from_file, to_file)) {
        fprintf(stderr, "prepare: %s (%d)\n", b200post_last_error(), rc);
        return range && rc == B200POST_ERR_INVALID_ARGUMENT ? 2 : 1;   // a file range outside the POST is a usage error
    }
    if (initial) {
        b200post_prove_opts po{};
        po.nonces = nonces; po.pow_mode = B200POST_POW_BUILTIN;
        if (int rc = b200post_setup_request_initial_proof(mgr, &po)) {
            fprintf(stderr, "initial proof: %s (%d)\n", b200post_last_error(), rc);
            return rc == B200POST_ERR_INVALID_ARGUMENT ? 2 : 1;
        }
    }
    signal(SIGINT, on_signal); signal(SIGTERM, on_signal);
    const uint64_t per_file = o.max_file_size / 16, all = (uint64_t)o.num_units * cfg.labels_per_unit;
    const uint64_t total = range ? std::min<uint64_t>(to_file < 0 ? all : (uint64_t)(to_file + 1) * per_file, all) - from_file * per_file : all;
    std::thread progress([&] {
        const auto t0 = std::chrono::steady_clock::now();
        b200post_setup_status st;
        uint64_t first = ~0ull;
        do {
            std::this_thread::sleep_for(std::chrono::seconds(2));
            b200post_setup_get_status(mgr, &st);
            if (first == ~0ull) first = st.num_labels_written;
            const double el = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
            fprintf(stderr, "\r%llu / %llu labels (%.1f %%), %.0f labels/s   ", (unsigned long long)st.num_labels_written, (unsigned long long)total,
                    100.0 * st.num_labels_written / (double)total, el > 0 ? (st.num_labels_written - first) / el : 0.0);
        } while (st.state == B200POST_SETUP_IN_PROGRESS || st.state == B200POST_SETUP_PREPARED);
        fprintf(stderr, "\n");
    });
    const int rc = b200post_setup_start_session(mgr, &g_cancel);
    progress.join();
    if (rc == B200POST_ERR_CANCELLED) { fprintf(stderr, "stopped; run again to resume\n"); return 130; }
    if (rc) { fprintf(stderr, "init failed: %s (%d)\n", b200post_last_error(), rc); return 1; }
    b200post_post_metadata md;
    if (b200post_load_metadata(datadir.c_str(), &md) == 0) {
        if (md.vrf_scan_pending)
            printf("files %llu..%llu complete; copy every range's files and one metadata file into one directory, then search the VRF nonce "
                   "with -searchForNonce\n", (unsigned long long)from_file, (unsigned long long)(from_file + (total + per_file - 1) / per_file - 1));
        else if (md.has_nonce) printf("initialization complete; VRF nonce %llu\n", (unsigned long long)md.nonce);
    }
    if (initial) {
        b200post_proof_out proof;
        const int prc = b200post_setup_initial_proof(mgr, &proof, nullptr);
        const std::string where = datadir + (datadir.empty() || datadir.back() == '/' ? "" : "/") + "initial_post.json";
        if (prc == 0) printf("initial proof: nonce %u, written to %s\n", proof.nonce, where.c_str());
        else printf("no initial proof: %s; the post-service proves from the stored data instead\n", b200post_last_error());
    }
    b200post_setup_manager_free(mgr);
    return 0;
}
