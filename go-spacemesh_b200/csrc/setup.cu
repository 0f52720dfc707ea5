// setup.cu — POST setup sessions (include/b200post_setup.h): the host-side mirror of
// activation.PostSetupManager (activation/post.go:185-449) and of the initializer it drives
// (un-vendored spacemeshos/post `initialization.Initializer`: files, metadata, resume, VRF nonce).
// C++ because the reference's host side is compiled Go; file formats are restated from the published
// spacemeshos/post layout (ASSUMED, "parity unpinned").
#include <dirent.h>
#include <errno.h>
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/b200post_setup.h"
#include "engine.h"
#include "host_hash.h"
#include "metrics.h"
#include "setup_internal.h"

using namespace b200post;

namespace {

const char kMetaFile[] = "postdata_metadata.json";

std::string b64(const uint8_t *p, size_t n) {
    static const char T[] = "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/";
    std::string o;
    for (size_t i = 0; i < n; i += 3) {
        const uint32_t v = (p[i] << 16) | ((i + 1 < n ? p[i + 1] : 0) << 8) | (i + 2 < n ? p[i + 2] : 0);
        o += T[v >> 18]; o += T[(v >> 12) & 63];
        o += i + 1 < n ? T[(v >> 6) & 63] : '=';
        o += i + 2 < n ? T[v & 63] : '=';
    }
    return o;
}
bool unb64(const std::string &s, uint8_t *out, size_t n) {
    auto val = [](char c) -> int {
        if (c >= 'A' && c <= 'Z') return c - 'A';
        if (c >= 'a' && c <= 'z') return c - 'a' + 26;
        if (c >= '0' && c <= '9') return c - '0' + 52;
        return c == '+' ? 62 : c == '/' ? 63 : -1;
    };
    std::vector<uint8_t> buf;
    uint32_t acc = 0; int bits = 0;
    for (char c : s) {
        if (c == '=') break;
        const int v = val(c);
        if (v < 0) return false;
        acc = (acc << 6) | (uint32_t)v; bits += 6;
        if (bits >= 8) { bits -= 8; buf.push_back((uint8_t)(acc >> bits)); }
    }
    if (buf.size() != n) return false;
    memcpy(out, buf.data(), n);
    return true;
}
std::string hex(const uint8_t *p, size_t n) {
    static const char H[] = "0123456789abcdef";
    std::string o;
    for (size_t i = 0; i < n; i++) { o += H[p[i] >> 4]; o += H[p[i] & 15]; }
    return o;
}
bool unhex(const std::string &s, uint8_t *out, size_t n) {
    if (s.size() != 2 * n) return false;
    for (size_t i = 0; i < n; i++) {
        unsigned v;
        if (sscanf(s.c_str() + 2 * i, "%2x", &v) != 1) return false;
        out[i] = (uint8_t)v;
    }
    return true;
}

// minimal JSON field access for the flat object we write ourselves
bool json_raw(const std::string &doc, const char *key, std::string *out) {
    const std::string pat = std::string("\"") + key + "\"";
    size_t p = doc.find(pat);
    if (p == std::string::npos) return false;
    p = doc.find(':', p + pat.size());
    if (p == std::string::npos) return false;
    p++;
    while (p < doc.size() && isspace((unsigned char)doc[p])) p++;
    size_t e = p;
    if (p < doc.size() && doc[p] == '"') { e = doc.find('"', p + 1); if (e == std::string::npos) return false; *out = doc.substr(p + 1, e - p - 1); return true; }
    while (e < doc.size() && doc[e] != ',' && doc[e] != '}' && !isspace((unsigned char)doc[e])) e++;
    *out = doc.substr(p, e - p);
    return true;
}
bool json_u64(const std::string &doc, const char *key, uint64_t *v) {
    std::string s;
    if (!json_raw(doc, key, &s) || s.empty() || s == "null") return false;
    char *end = nullptr;
    *v = strtoull(s.c_str(), &end, 10);
    return end && *end == 0;
}

std::string path_join(const std::string &d, const std::string &f) { return d.empty() || d.back() == '/' ? d + f : d + "/" + f; }
std::string data_file(const std::string &d, uint64_t i) { return path_join(d, "postdata_" + std::to_string(i) + ".bin"); }

int io_error(const std::string &what) {
    set_error(what + ": " + strerror(errno));
    return B200POST_ERR_IO;
}

int mkdir_p(const std::string &dir) {
    std::string cur;
    for (size_t i = 0; i <= dir.size(); i++) {
        if (i == dir.size() || dir[i] == '/') {
            if (!cur.empty() && mkdir(cur.c_str(), 0755) != 0 && errno != EEXIST) return io_error("mkdir " + cur);
        }
        if (i < dir.size()) cur += dir[i];
    }
    return B200POST_OK;
}

int save_metadata(const std::string &dir, const b200post_post_metadata &m) {
    std::string j = "{\n";
    j += " \"NodeId\": \"" + b64(m.node_id, 32) + "\",\n";
    j += " \"CommitmentAtxId\": \"" + b64(m.commitment_atx_id, 32) + "\",\n";
    j += " \"LabelsPerUnit\": " + std::to_string(m.labels_per_unit) + ",\n";
    j += " \"NumUnits\": " + std::to_string(m.num_units) + ",\n";
    j += " \"MaxFileSize\": " + std::to_string(m.max_file_size) + ",\n";
    j += " \"Nonce\": " + (m.has_nonce ? std::to_string(m.nonce) : std::string("null")) + ",\n";
    j += " \"NonceValue\": " + (m.has_nonce ? "\"" + hex(m.nonce_value, 32) + "\"" : std::string("null")) + ",\n";
    j += " \"LastPosition\": " + std::to_string(m.last_position) + ",\n";
    if (m.vrf_scan_pending) j += " \"VrfScanPending\": true,\n";   // absent otherwise: such a file reads as before
    j += " \"Scrypt\": {\"N\": " + std::to_string(m.scrypt_n) + ", \"R\": " + std::to_string(m.scrypt_r) + ", \"P\": " + std::to_string(m.scrypt_p) + "}\n}\n";
    const std::string tmp = path_join(dir, std::string(kMetaFile) + ".tmp"), fin = path_join(dir, kMetaFile);
    FILE *f = fopen(tmp.c_str(), "w");
    if (!f) return io_error("open " + tmp);
    const bool ok = fwrite(j.data(), 1, j.size(), f) == j.size();
    if (fclose(f) != 0 || !ok) return io_error("write " + tmp);
    if (rename(tmp.c_str(), fin.c_str()) != 0) return io_error("rename " + tmp);
    return B200POST_OK;
}

// returns OK, or B200POST_ERR_IO with ENOENT-text "metadata file is missing" when absent
int load_metadata(const std::string &dir, b200post_post_metadata *m, bool *missing) {
    if (missing) *missing = false;
    const std::string p = path_join(dir, kMetaFile);
    FILE *f = fopen(p.c_str(), "r");
    if (!f) {
        if (errno == ENOENT) { if (missing) *missing = true; set_error("metadata file is missing"); return B200POST_ERR_IO; }
        return io_error("open " + p);
    }
    std::string doc;
    char buf[4096];
    size_t n;
    while ((n = fread(buf, 1, sizeof buf, f)) > 0) doc.append(buf, n);
    fclose(f);
    memset(m, 0, sizeof *m);
    std::string s;
    uint64_t v;
    if (!json_raw(doc, "NodeId", &s) || !unb64(s, m->node_id, 32) || !json_raw(doc, "CommitmentAtxId", &s) ||
        !unb64(s, m->commitment_atx_id, 32)) { set_error("corrupt metadata: ids"); return B200POST_ERR_IO; }
    if (json_u64(doc, "LabelsPerUnit", &v)) m->labels_per_unit = v;
    if (json_u64(doc, "NumUnits", &v)) m->num_units = (uint32_t)v;
    if (json_u64(doc, "MaxFileSize", &v)) m->max_file_size = v;
    if (json_u64(doc, "LastPosition", &v)) m->last_position = v;
    if (json_u64(doc, "N", &v)) m->scrypt_n = v;
    if (json_u64(doc, "R", &v)) m->scrypt_r = v;
    if (json_u64(doc, "P", &v)) m->scrypt_p = v;
    if (json_u64(doc, "Nonce", &v) && json_raw(doc, "NonceValue", &s) && unhex(s, m->nonce_value, 32)) { m->has_nonce = 1; m->nonce = v; }
    m->vrf_scan_pending = json_raw(doc, "VrfScanPending", &s) && s == "true";
    return B200POST_OK;
}

}  // namespace

namespace b200post {

int save_post_metadata(const std::string &dir, const b200post_post_metadata &m) { return save_metadata(dir, m); }

int compute_labels(int64_t provider_id, uint64_t N, const uint8_t commitment[32], uint64_t start, uint64_t count, uint8_t *out,
                   const uint8_t *diff, b200post_vrf_nonce *nonce, const volatile int *cancel) {
    if (nonce) memset(nonce, 0, sizeof *nonce);
    if (provider_id == B200POST_PROVIDER_ALL) {
        const int n = device_count();
        if (n == 0) { set_error("no CUDA device available"); return B200POST_ERR_NO_DEVICE; }
        std::vector<uint32_t> ids((size_t)n);
        for (int i = 0; i < n; i++) ids[(size_t)i] = (uint32_t)i;
        return b200post_labels_range_multi(ids.data(), n, commitment, N, start, count, out, diff, diff ? nonce : nullptr, cancel);
    }
    return b200post_labels_range((uint32_t)provider_id, commitment, N, start, count, out, diff, diff ? nonce : nullptr, cancel);
}

int search_past_end(const std::string &dir, b200post_post_metadata *md, uint64_t num_labels, int64_t provider_id, uint64_t batch,
                    const uint8_t commitment[32], const uint8_t diff[32], const volatile int *cancel) {
    uint64_t pos = std::max<uint64_t>(num_labels, md->last_position);
    while (!md->has_nonce) {
        if (cancel && *cancel) { set_error("cancelled"); return B200POST_ERR_CANCELLED; }
        b200post_vrf_nonce nn;
        int rc = compute_labels(provider_id, md->scrypt_n, commitment, pos, batch, nullptr, diff, &nn, cancel);
        if (rc) return rc;
        pos += batch;
        md->last_position = pos;
        if (nn.found) { md->has_nonce = 1; md->nonce = nn.index; memcpy(md->nonce_value, nn.label32, 32); }
        if ((rc = save_metadata(dir, *md))) return rc;
    }
    return B200POST_OK;
}

}  // namespace b200post

struct b200post_setup_manager {
    b200post_post_config cfg{};
    std::mutex mu;
    int32_t state = B200POST_SETUP_NOT_STARTED;
    // last prepared session
    bool have_opts = false;
    b200post_setup_opts opts{};
    std::string data_dir;
    uint8_t node_id[32] = {0};
    b200post_post_metadata meta{};
    std::atomic<uint64_t> labels_written{0};   // of the session's label range
    uint64_t num_labels = 0;
    uint64_t range_lo = 0, range_hi = 0;        // the session writes labels [range_lo, range_hi)
    bool range() const { return range_lo != 0 || range_hi != num_labels; }
};

namespace {

int fail_state(b200post_setup_manager *m, int code, const std::string &msg) {
    m->state = B200POST_SETUP_ERROR;
    set_error(msg);
    return code;
}

}  // namespace

extern "C" {

void b200post_default_post_config(b200post_post_config *cfg) {
    if (!cfg) return;
    memset(cfg, 0, sizeof *cfg);
    cfg->min_num_units = 1; cfg->max_num_units = 10; cfg->labels_per_unit = 512;   // 2 x 512 = BASELINE.json configs[0]
    cfg->k1 = 26; cfg->k2 = 37; cfg->k3 = 37;
    static const uint8_t d[4] = {0x00, 0x0d, 0xfb, 0x23};                           // config/mainnet.go:41 prefix
    memset(cfg->pow_difficulty, 0xff, 32);
    memcpy(cfg->pow_difficulty, d, 4);
}

void b200post_default_setup_opts(b200post_setup_opts *o) {
    if (!o) return;
    memset(o, 0, sizeof *o);
    o->num_units = 2; o->max_file_size = 4ull << 30; o->provider_id = B200POST_PROVIDER_UNSET;
    o->scrypt_n = 8192; o->scrypt_r = 1; o->scrypt_p = 1; o->compute_batch_size = 1ull << 20; o->self_check_every = 16;
}

int b200post_setup_manager_new(const b200post_post_config *cfg, b200post_setup_manager **out) {
    if (!cfg || !out) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    *out = new b200post_setup_manager;
    (*out)->cfg = *cfg;
    return B200POST_OK;
}

void b200post_setup_manager_free(b200post_setup_manager *m) { delete m; }

int b200post_setup_prepare_initializer(b200post_setup_manager *m, const b200post_setup_opts *o, const uint8_t node_id[32],
                                       const uint8_t commitment_atx_id[32]) {
    return b200post_setup_prepare_files(m, o, node_id, commitment_atx_id, 0, -1);
}

int b200post_setup_prepare_files(b200post_setup_manager *m, const b200post_setup_opts *o, const uint8_t node_id[32],
                                 const uint8_t commitment_atx_id[32], uint64_t from_file, int64_t to_file) {
    if (!m || !o || !node_id || !commitment_atx_id) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    std::lock_guard<std::mutex> lk(m->mu);
    if (m->state == B200POST_SETUP_PREPARED || m->state == B200POST_SETUP_IN_PROGRESS) {
        set_error("post setup session in progress");   // activation/post.go:345
        return B200POST_ERR_STATE;
    }
    // ---- option validation (initialization.NewInitializer / config.Validate upstream; errors -> state Error, post.go:362-365)
    const b200post_post_config &c = m->cfg;
    if (!o->data_dir || !*o->data_dir) return fail_state(m, B200POST_ERR_INVALID_ARGUMENT, "invalid `opts.DataDir`: empty");
    if (o->num_units < c.min_num_units) return fail_state(m, B200POST_ERR_INVALID_ARGUMENT, "invalid `opts.NumUnits`: below `cfg.MinNumUnits`");
    if (o->num_units > c.max_num_units) return fail_state(m, B200POST_ERR_INVALID_ARGUMENT, "invalid `opts.NumUnits`: above `cfg.MaxNumUnits`");
    if (c.labels_per_unit == 0) return fail_state(m, B200POST_ERR_INVALID_ARGUMENT, "invalid `cfg.LabelsPerUnit`: 0");
    if (o->compute_batch_size == 0 || o->compute_batch_size % 8) return fail_state(m, B200POST_ERR_INVALID_ARGUMENT, "invalid `opts.ComputeBatchSize`: must be a positive multiple of 8");
    if (o->scrypt_n < 2 || o->scrypt_n > (1ull << 20) || (o->scrypt_n & (o->scrypt_n - 1)) || o->scrypt_r != 1 || o->scrypt_p != 1)
        return fail_state(m, B200POST_ERR_INVALID_ARGUMENT, "invalid `opts.Scrypt`: N must be a power of two in [2, 2^20], r = p = 1");
    if (o->max_file_size < 16 || o->max_file_size % 16) return fail_state(m, B200POST_ERR_INVALID_ARGUMENT, "invalid `opts.MaxFileSize`: must be a positive multiple of 16");
    const unsigned __int128 nl = (unsigned __int128)o->num_units * c.labels_per_unit;
    if (nl > (~0ull >> 4)) return fail_state(m, B200POST_ERR_INVALID_ARGUMENT, "NumUnits * LabelsPerUnit overflows");
    if (o->provider_id < B200POST_PROVIDER_ALL || o->provider_id > 0xfffffffe) return fail_state(m, B200POST_ERR_INVALID_ARGUMENT, "invalid `opts.ProviderID`");
    const uint64_t num_labels = (uint64_t)nl, per_file = o->max_file_size / 16;
    uint64_t lo = 0, hi = num_labels, last_file = ~0ull;   // the whole POST: no bound on the resume scan (as before ranges)
    if (from_file != 0 || to_file != -1) {
        const uint64_t n_files = (num_labels + per_file - 1) / per_file;
        if (to_file < -1) return fail_state(m, B200POST_ERR_INVALID_ARGUMENT, "invalid file range: toFile < -1");
        last_file = to_file == -1 ? n_files - 1 : (uint64_t)to_file;
        if (n_files == 0 || from_file > last_file || last_file >= n_files)
            return fail_state(m, B200POST_ERR_INVALID_ARGUMENT, "invalid file range: need fromFile <= toFile < " + std::to_string(n_files) + " (the POST's files)");
        lo = from_file * per_file;
        hi = std::min<uint64_t>((last_file + 1) * per_file, num_labels);
    }

    const std::string dir = o->data_dir;
    int rc = mkdir_p(dir);
    if (rc) { m->state = B200POST_SETUP_ERROR; return rc; }

    // ---- metadata: an existing file pins identity + commitment ATX (post.go:374-377)
    b200post_post_metadata meta;
    bool missing = false;
    rc = load_metadata(dir, &meta, &missing);
    if (rc && !missing) { m->state = B200POST_SETUP_ERROR; return rc; }
    if (!missing) {
        if (memcmp(meta.node_id, node_id, 32)) return fail_state(m, B200POST_ERR_CONFIG_MISMATCH, "`NodeId` mismatch with the metadata in DataDir");
        if (meta.labels_per_unit != c.labels_per_unit) return fail_state(m, B200POST_ERR_CONFIG_MISMATCH, "`LabelsPerUnit` mismatch with the metadata in DataDir");
        if (meta.scrypt_n != o->scrypt_n) return fail_state(m, B200POST_ERR_CONFIG_MISMATCH, "`Scrypt.N` mismatch with the metadata in DataDir");
        if (meta.max_file_size != o->max_file_size) return fail_state(m, B200POST_ERR_CONFIG_MISMATCH, "`MaxFileSize` mismatch with the metadata in DataDir");
        if (meta.num_units > o->num_units) return fail_state(m, B200POST_ERR_CONFIG_MISMATCH, "`NumUnits` is smaller than the initialised data");
        meta.num_units = o->num_units;
    } else {
        memset(&meta, 0, sizeof meta);
        memcpy(meta.node_id, node_id, 32);
        memcpy(meta.commitment_atx_id, commitment_atx_id, 32);
        meta.labels_per_unit = c.labels_per_unit; meta.num_units = o->num_units; meta.max_file_size = o->max_file_size;
        meta.scrypt_n = o->scrypt_n; meta.scrypt_r = 1; meta.scrypt_p = 1;
    }

    // ---- resume point: full files from_file..k-1, then one partial file; nothing past the range is looked at
    uint64_t written = 0;
    for (uint64_t i = from_file; i <= last_file; i++) {
        struct stat st;
        if (stat(data_file(dir, i).c_str(), &st) != 0) break;
        if (st.st_size % 16 || (uint64_t)st.st_size / 16 > per_file) return fail_state(m, B200POST_ERR_CONFIG_MISMATCH, "postdata file has an unexpected size");
        written += (uint64_t)st.st_size / 16;
        if ((uint64_t)st.st_size / 16 < per_file) break;
    }
    if (written > hi - lo) return fail_state(m, B200POST_ERR_CONFIG_MISMATCH, "DataDir holds more labels than NumUnits * LabelsPerUnit");
    // a range's labels are not VRF-scanned: without a nonce, the stored data must be searched once it is merged
    // (with one, the labels are deterministic and the nonce stays right)
    const bool range = lo != 0 || hi != num_labels;
    if (range && !meta.has_nonce) meta.vrf_scan_pending = 1;

    m->opts = *o; m->data_dir = dir; m->opts.data_dir = m->data_dir.c_str();
    if (m->opts.self_check_every == 0) m->opts.self_check_every = 16;
    memcpy(m->node_id, node_id, 32);
    m->meta = meta; m->num_labels = num_labels; m->have_opts = true;
    m->range_lo = lo; m->range_hi = hi;
    m->labels_written.store(written);
    if ((rc = save_metadata(dir, m->meta))) { m->state = B200POST_SETUP_ERROR; return rc; }
    m->state = B200POST_SETUP_PREPARED;
    return B200POST_OK;
}

int b200post_setup_start_session(b200post_setup_manager *m, const volatile int *cancel) {
    if (!m) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    {
        std::lock_guard<std::mutex> lk(m->mu);
        if (m->state != B200POST_SETUP_PREPARED) { set_error("post session not prepared"); return B200POST_ERR_STATE; }   // post.go:277
        m->state = B200POST_SETUP_IN_PROGRESS;
    }
    metrics().setup_sessions_total++;
    auto finish = [&](int32_t state, int rc) { std::lock_guard<std::mutex> lk(m->mu); m->state = state; return rc; };

    const uint64_t num_labels = m->num_labels, per_file = m->opts.max_file_size / 16, batch = m->opts.compute_batch_size;
    const uint64_t lo = m->range_lo, hi = m->range_hi;
    const bool range = m->range();   // no VRF scan, no nonce, no past-the-end search: a range's arg-min is not the POST's
    uint64_t written = lo + m->labels_written.load();   // the next label to write
    const bool need_work = written < hi || (!range && (!m->meta.has_nonce || m->meta.vrf_scan_pending));
    if (need_work && m->opts.provider_id == B200POST_PROVIDER_UNSET) {
        set_error("no provider specified");
        return finish(B200POST_SETUP_ERROR, B200POST_ERR_NO_PROVIDER);
    }
    uint8_t commitment[32];
    commitment_bytes(m->meta.node_id, m->meta.commitment_atx_id, commitment);
    uint8_t diff[32];
    if (m->meta.has_nonce) memcpy(diff, m->meta.nonce_value, 32); else vrf_difficulty(num_labels, diff);

    std::vector<uint8_t> buf;
    uint64_t n_batches = 0;
    auto note_nonce = [&](const b200post_vrf_nonce &nn) -> int {
        if (!nn.found) return B200POST_OK;
        m->meta.has_nonce = 1; m->meta.nonce = nn.index; memcpy(m->meta.nonce_value, nn.label32, 32);
        memcpy(diff, nn.label32, 32);   // only a smaller label can replace it
        return save_metadata(m->data_dir, m->meta);
    };

    while (written < hi) {
        if (cancel && *cancel) { set_error("cancelled"); return finish(B200POST_SETUP_STOPPED, B200POST_ERR_CANCELLED); }
        const uint64_t file_idx = written / per_file, in_file = written % per_file;
        const uint64_t count = std::min<uint64_t>({batch, per_file - in_file, hi - written});
        buf.resize((size_t)count * 16);
        b200post_vrf_nonce nn;
        int rc = compute_labels(m->opts.provider_id, m->opts.scrypt_n, commitment, written, count, buf.data(), range ? nullptr : diff,
                                &nn, cancel);
        if (rc == B200POST_ERR_CANCELLED) return finish(B200POST_SETUP_STOPPED, rc);
        if (rc) return finish(B200POST_SETUP_ERROR, rc);
        // ErrReferenceLabelMismatch contract (activation/post.go:299-312): every self_check_every batches one label of the
        // batch is recomputed ON THE HOST CPU (reference_label.cpp: the kernels' own arithmetic header compiled for the
        // host) and compared with what the device wrote — independent of the device, its kernels' scheduling and memory.
        if (options().debug_corrupt_next_batch.exchange(0) != 0 && count) buf[((n_batches * 7) % count) * 16 + 3] ^= 0x40;   // fault injection (tests)
        if (n_batches % m->opts.self_check_every == 0) {
            uint8_t ref[32];
            uint64_t pick = written + (n_batches * 2654435761ull) % count;
            if (options().debug_corrupt_check_all.load() != 0) {
                // test hook: check the label the injected fault hit (the sampled one is elsewhere with probability 1 - 1/count)
                pick = written + (n_batches * 7) % count;
            }
            reference_label32(commitment, pick, (uint32_t)m->opts.scrypt_n, ref);
            if (memcmp(ref, buf.data() + (pick - written) * 16, 16)) {
                metrics().setup_label_mismatch_total++;
                set_error("reference label mismatch at index " + std::to_string(pick));
                return finish(B200POST_SETUP_ERROR, B200POST_ERR_LABEL_MISMATCH);
            }
        }
        n_batches++;
        const std::string path = data_file(m->data_dir, file_idx);
        const int fd = open(path.c_str(), O_WRONLY | O_CREAT, 0644);
        if (fd < 0) return finish(B200POST_SETUP_ERROR, io_error("open " + path));
        size_t done = 0;
        bool ok = lseek(fd, (off_t)(in_file * 16), SEEK_SET) >= 0;
        while (ok && done < buf.size()) {
            const ssize_t w = write(fd, buf.data() + done, buf.size() - done);
            if (w <= 0) ok = false; else done += (size_t)w;
        }
        if (!ok || close(fd) != 0) { const int rcio = io_error("write " + path); if (ok) {} else close(fd); return finish(B200POST_SETUP_ERROR, rcio); }
        written += count;
        m->labels_written.store(written - lo);
        if ((rc = note_nonce(nn))) return finish(B200POST_SETUP_ERROR, rc);
    }
    if (!range) {
        int rc;
        if (m->meta.vrf_scan_pending) {
            // some files were written by range sessions and never scanned: the nonce comes from all stored labels,
            // whatever this session's own scan recorded
            b200post_vrf_search_opts so;
            b200post_default_vrf_search_opts(&so);
            so.provider_id = m->opts.provider_id; so.compute_batch_size = batch;
            b200post_vrf_nonce nn;
            rc = stored_vrf_search(m->data_dir, &m->meta, so, &nn, cancel);
        } else {
            // "keep searching past numLabels until a VRF nonce is found" (SURVEY.md §8f.1): outputs are discarded
            rc = search_past_end(m->data_dir, &m->meta, num_labels, m->opts.provider_id, batch, commitment, diff, cancel);
        }
        if (rc == B200POST_ERR_CANCELLED) return finish(B200POST_SETUP_STOPPED, rc);
        if (rc) return finish(B200POST_SETUP_ERROR, rc);
    }
    const int rc = save_metadata(m->data_dir, m->meta);
    if (rc) return finish(B200POST_SETUP_ERROR, rc);
    return finish(B200POST_SETUP_COMPLETE, B200POST_OK);
}

int b200post_setup_get_status(b200post_setup_manager *m, b200post_setup_status *out) {
    if (!m || !out) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    std::lock_guard<std::mutex> lk(m->mu);
    out->state = m->state;
    // activation/post.go:249-264: no label count in NotStarted / Error
    out->num_labels_written = (m->state == B200POST_SETUP_NOT_STARTED || m->state == B200POST_SETUP_ERROR) ? 0 : m->labels_written.load();
    return B200POST_OK;
}

int b200post_setup_reset(b200post_setup_manager *m) {
    if (!m) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    std::lock_guard<std::mutex> lk(m->mu);
    if (m->state == B200POST_SETUP_IN_PROGRESS) { set_error("post setup session in progress"); return B200POST_ERR_STATE; }
    if (!m->have_opts) { set_error("reset: no session was prepared"); return B200POST_ERR_STATE; }
    DIR *d = opendir(m->data_dir.c_str());
    if (d) {
        while (struct dirent *e = readdir(d)) {
            const std::string name = e->d_name;
            const bool data = name.rfind("postdata_", 0) == 0 && name.size() > 13 && name.substr(name.size() - 4) == ".bin";
            if (data || name == kMetaFile) {
                if (unlink(path_join(m->data_dir, name).c_str()) != 0) { closedir(d); return io_error("unlink " + name); }
            }
        }
        closedir(d);
    }
    m->labels_written.store(0);
    memset(&m->meta, 0, sizeof m->meta);
    m->state = B200POST_SETUP_NOT_STARTED;
    return B200POST_OK;
}

int b200post_setup_commitment_atx(b200post_setup_manager *m, uint8_t out[32]) {
    if (!m || !out) return B200POST_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> lk(m->mu);
    if (!m->have_opts) { set_error("no session was prepared"); return B200POST_ERR_STATE; }
    memcpy(out, m->meta.commitment_atx_id, 32);
    return B200POST_OK;
}

int b200post_load_metadata(const char *data_dir, b200post_post_metadata *out) {
    if (!data_dir || !out) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    return load_metadata(data_dir, out, nullptr);
}

}  // extern "C"
