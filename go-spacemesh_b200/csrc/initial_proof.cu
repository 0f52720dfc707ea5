// initial_proof.cu — see initial_proof.h.  The state file is the resume point of the scan: whatever it does not
// cover is rescanned from the postdata files, so a stop, a crash or a stale state costs a read, never a wrong proof.
#include "initial_proof.h"

#include <algorithm>
#include <cerrno>
#include <cstdio>
#include <cstring>

#include "postdata_io.h"
#include "randomx_engine.h"
#include "setup_internal.h"

namespace b200post {

const char kInitialProofFile[] = "initial_post.json";
const char kInitialScanFile[] = "initial_post.scan";

namespace {

const uint8_t kZeroChallenge[32] = {0};   // shared.ZeroChallenge: the challenge of the initial proof
const uint64_t kMaxScanChunk = 1ull << 22;   // labels per scan chunk (64 MiB of pinned staging per buffer), as the prover

uint64_t fnv1a64(const std::string &s) {
    uint64_t h = 0xcbf29ce484222325ull;
    for (unsigned char c : s) { h ^= c; h *= 0x100000001b3ull; }
    return h;
}
template <class T> void put(std::string *s, T v) { s->append(reinterpret_cast<const char *>(&v), sizeof v); }
template <class T> bool get(const std::string &s, size_t *p, T *v) {
    if (*p + sizeof(T) > s.size()) return false;
    memcpy(v, s.data() + *p, sizeof(T));
    *p += sizeof(T);
    return true;
}
std::string join(const std::string &d, const char *f) { return d.empty() || d.back() == '/' ? d + f : d + "/" + f; }

}  // namespace

// Everything the scan's result depends on besides the labels: a state whose header differs is someone else's.
std::string InitialProofScan::header() const {
    std::string h("B2IPSCAN", 8);
    put<uint32_t>(&h, 1);   // layout version
    h.append(reinterpret_cast<const char *>(md_.node_id), 32);
    h.append(reinterpret_cast<const char *>(md_.commitment_atx_id), 32);
    put<uint32_t>(&h, md_.num_units);
    put<uint64_t>(&h, md_.labels_per_unit);
    put<uint64_t>(&h, md_.scrypt_n);
    put<uint32_t>(&h, cfg_.k1);
    put<uint32_t>(&h, cfg_.k2);
    put<uint32_t>(&h, opts_.nonces);
    h.append(reinterpret_cast<const char *>(cfg_.pow_difficulty), 32);
    h.append(reinterpret_cast<const char *>(kZeroChallenge), 32);
    put<uint32_t>(&h, opts_.pow_mode);
    put<uint32_t>(&h, (uint32_t)key_.size());
    h.append(key_.begin(), key_.end());
    return h;
}

// header | pows | upto | lists (count, then nonce, length, indices) | FNV-1a 64 of everything before it
int InitialProofScan::save_state() {
    std::string s = header();
    for (uint64_t p : pows_) put<uint64_t>(&s, p);
    put<uint64_t>(&s, start_ + sc_.scanned());
    put<uint32_t>(&s, (uint32_t)sc_.lists().size());
    for (const auto &kv : sc_.lists()) {
        put<uint32_t>(&s, kv.first);
        put<uint32_t>(&s, (uint32_t)kv.second.size());
        for (uint64_t i : kv.second) put<uint64_t>(&s, i);
    }
    put<uint64_t>(&s, fnv1a64(s));
    const std::string fin = join(dir_, kInitialScanFile), tmp = fin + ".tmp";
    FILE *f = fopen(tmp.c_str(), "wb");
    if (!f) { set_error("open " + tmp + ": " + strerror(errno)); return B200POST_ERR_IO; }
    const bool ok = fwrite(s.data(), 1, s.size(), f) == s.size();
    if (fclose(f) != 0 || !ok) { set_error("write " + tmp + ": " + strerror(errno)); return B200POST_ERR_IO; }
    if (rename(tmp.c_str(), fin.c_str()) != 0) { set_error("rename " + tmp + ": " + strerror(errno)); return B200POST_ERR_IO; }
    return B200POST_OK;
}

bool InitialProofScan::load_state(uint64_t written) {
    FILE *f = fopen(join(dir_, kInitialScanFile).c_str(), "rb");
    if (!f) return false;
    std::string s;
    char buf[65536];
    size_t n;
    while ((n = fread(buf, 1, sizeof buf, f)) > 0) s.append(buf, n);
    fclose(f);
    const std::string h = header();
    if (s.size() < h.size() + 8 || s.compare(0, h.size(), h) != 0) return false;
    uint64_t sum;
    memcpy(&sum, s.data() + s.size() - 8, 8);
    const std::string body = s.substr(0, s.size() - 8);
    if (fnv1a64(body) != sum) return false;
    size_t p = h.size();
    std::vector<uint64_t> pows(opts_.nonces / 16);
    for (uint64_t &v : pows) if (!get(body, &p, &v)) return false;
    uint64_t upto;
    uint32_t n_lists;
    if (!get(body, &p, &upto) || upto > written || upto > num_labels_ || !get(body, &p, &n_lists)) return false;
    HitLists lists;
    for (uint32_t i = 0; i < n_lists; i++) {
        uint32_t nonce, len;
        if (!get(body, &p, &nonce) || !get(body, &p, &len) || nonce >= opts_.nonces || len > cfg_.k2) return false;
        std::vector<uint64_t> &l = lists[nonce];
        l.resize(len);
        for (uint64_t &v : l) if (!get(body, &p, &v) || v >= upto) return false;
    }
    if (p != body.size()) return false;
    pows_ = pows; start_ = upto; restored_ = lists;
    return true;
}

int InitialProofScan::begin(const InitialProofRequest &req, const std::string &dir, const b200post_post_metadata &md,
                            const b200post_post_config &cfg, int64_t provider_id, uint64_t written, uint64_t batch,
                            const volatile int *cancel) {
    dir_ = dir; opts_ = req.opts; key_ = req.cache_key; md_ = md; cfg_ = cfg;
    opts_.pow_cache_key = key_.empty() ? nullptr : key_.data();
    opts_.pow_cache_key_len = key_.size();
    num_labels_ = (uint64_t)md.num_units * md.labels_per_unit;
    // the session's devices: the proving scan runs on the first, a BUILTIN k2pow search on all of them
    std::vector<uint32_t> devs;
    if (provider_id == B200POST_PROVIDER_ALL) for (int i = 0; i < device_count(); i++) devs.push_back((uint32_t)i);
    else devs.push_back((uint32_t)provider_id);
    if (devs.empty()) { set_error("no CUDA device available"); return B200POST_ERR_NO_DEVICE; }
    scan_dev_ = devs[0];
    if (!engine_for(scan_dev_)) return B200POST_ERR_NO_DEVICE;

    int rc;
    if (!load_state(written)) {
        start_ = 0; restored_.clear();
        if ((rc = find_pows(opts_, kZeroChallenge, md.node_id, md.num_units, cfg.pow_difficulty, devs.data(), (int)devs.size(), &pows_, cancel)))
            return rc;
        // the RandomX dataset and batch (~14 GiB per device) would otherwise stay resident and shrink every label layer
        if (opts_.pow_mode == B200POST_POW_BUILTIN) for (uint32_t d : devs) randomx_release((int)d);
        if ((rc = save_state())) return rc;   // a resumed session never searches again
    }
    const uint64_t chunk = std::min<uint64_t>({std::max<uint64_t>(batch, 1), kMaxScanChunk, num_labels_});
    if ((rc = sc_.init(scan_dev_, kZeroChallenge, opts_.nonces, pows_.data(), cfg.k1, cfg.k2, num_labels_, chunk))) return rc;
    sc_.restore(restored_);
    // the gap between the state's prefix and what is on disk, in index order, from the files
    PostDataReader reader(dir, md.max_file_size / 16);
    for (uint64_t pos = start_; pos < written;) {
        if (cancel && *cancel) { stop(); set_error("cancelled"); return B200POST_ERR_CANCELLED; }
        const uint64_t n = std::min<uint64_t>(chunk, written - pos);
        if ((rc = collect(b_)) || (rc = reader.read(pos, n, sc_.staging(b_))) || (rc = submit(b_, pos, n))) { stop(); return rc; }
        b_ ^= 1;
        pos += n;
    }
    return B200POST_OK;
}

int InitialProofScan::buffer(uint64_t count, uint8_t **dst) {
    *dst = nullptr;
    if (count > sc_.chunk()) return B200POST_OK;
    const int rc = collect(b_);   // the chunk that last used this staging buffer
    if (rc == B200POST_OK) *dst = sc_.staging(b_);
    return rc;
}

int InitialProofScan::scan(uint64_t first, uint64_t count, const uint8_t *src) {
    if (src == sc_.staging(b_)) {
        const int rc = submit(b_, first, count);
        b_ ^= 1;
        return rc;
    }
    return submit_from(src, first, count);
}

// a batch larger than one scan chunk: copied into staging and scanned in pieces
int InitialProofScan::submit_from(const uint8_t *src, uint64_t first, uint64_t count) {
    for (uint64_t off = 0; off < count;) {
        const uint64_t n = std::min<uint64_t>(sc_.chunk(), count - off);
        int rc = collect(b_);
        if (rc) return rc;
        memcpy(sc_.staging(b_), src + off * 16, (size_t)n * 16);
        if ((rc = submit(b_, first + off, n))) return rc;
        b_ ^= 1;
        off += n;
    }
    return B200POST_OK;
}

int InitialProofScan::checkpoint() {
    int rc;
    for (int k = 0; k < 2; k++) if ((rc = collect(b_ ^ k))) return rc;   // older chunk first
    return save_state();
}

// Chunks are folded in submission order, so what is folded is always a prefix of the labels.  After the first chunk
// that failed to go in or come back, nothing more is folded: a later chunk would leave a hole below upto.
int InitialProofScan::collect(int b) {
    if (failed_) { sc_.drain(); set_error("initial proof: an earlier scan chunk failed"); return B200POST_ERR_STATE; }
    const int rc = sc_.collect(b);
    failed_ = rc != B200POST_OK;
    return rc;
}

int InitialProofScan::submit(int b, uint64_t first, uint64_t count) {
    const int rc = sc_.submit(b, first, (uint32_t)count);
    failed_ = failed_ || rc != B200POST_OK;
    return rc;
}

void InitialProofScan::stop() {
    const std::string err = last_error();
    for (int k = 0; k < 2 && !failed_; k++) collect(b_ ^ k);   // older chunk first; stops at a failure
    sc_.drain();
    save_state();   // upto = the end of the folded prefix, whose hit lists are complete
    set_error(err);   // the session reports its own failure, not the state's
}

int InitialProofScan::finish(b200post_proof_out *out, b200post_proof_metadata *meta) {
    int rc = checkpoint();
    if (rc) return rc;
    if (start_ + sc_.scanned() != num_labels_) { set_error("initial proof: the scan does not cover every label"); return B200POST_ERR_STATE; }
    uint32_t nonce = 0;
    std::vector<uint64_t> idx;
    if (!pick_winner(sc_.lists(), cfg_.k2, &nonce, &idx)) { set_error(kNoProof); return B200POST_ERR_INVALID_PROOF; }
    if ((rc = write_proof(num_labels_, nonce, idx, pows_.data(), num_labels_, out))) return rc;
    memset(meta, 0, sizeof *meta);
    memcpy(meta->node_id, md_.node_id, 32);
    memcpy(meta->commitment_atx_id, md_.commitment_atx_id, 32);
    memcpy(meta->challenge, kZeroChallenge, 32);
    meta->num_units = md_.num_units; meta->labels_per_unit = md_.labels_per_unit;
    // the gate of b200post_generate_proof_checked: a proof this library's own verifier rejects is never handed out
    return gate_proof(scan_dev_, cfg_, md_.scrypt_n, opts_, *meta, out);
}

}  // namespace b200post
