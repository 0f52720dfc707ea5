// initial_proof.cu — see initial_proof.h.  The state file is the resume point of the scan: whatever it does not
// cover is rescanned from the postdata files, so a stop, a crash or a stale state costs a read, never a wrong proof.
#include "initial_proof.h"

#include <algorithm>
#include <cstring>

#include "postdata_io.h"
#include "randomx_engine.h"

namespace b200post {
namespace {

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
}  // namespace

// Everything the scan's result depends on besides the labels: a state whose header differs is someone else's.  A
// record adds the POST's file size and its own range, and carries the proof part only when it was asked for.
std::string InitialProofScan::header() const {
    std::string h(record_ ? "B2RNGREC" : "B2IPSCAN", 8);
    put<uint32_t>(&h, 1);   // layout version
    h.append(reinterpret_cast<const char *>(md_.node_id), 32);
    h.append(reinterpret_cast<const char *>(md_.commitment_atx_id), 32);
    put<uint32_t>(&h, md_.num_units);
    put<uint64_t>(&h, md_.labels_per_unit);
    put<uint64_t>(&h, md_.scrypt_n);
    if (record_) {
        put<uint64_t>(&h, md_.max_file_size);
        put<uint64_t>(&h, range_.from_file);
        put<uint64_t>(&h, range_.to_file);
        put<uint64_t>(&h, range_.lo);
        put<uint64_t>(&h, range_.hi);
        put<uint32_t>(&h, proof_);
    }
    if (proof_) h += proof_part();
    return h;
}

std::string InitialProofScan::proof_part() const {
    std::string h;
    put<uint32_t>(&h, cfg_.k1);
    put<uint32_t>(&h, cfg_.k2);
    put<uint32_t>(&h, opts_.nonces);
    h.append(reinterpret_cast<const char *>(cfg_.pow_difficulty), 32);
    h.append(reinterpret_cast<const char *>(kZeroChallenge), 32);
    put<uint32_t>(&h, opts_.pow_mode);
    put<uint32_t>(&h, (uint32_t)key_.size());
    h.append(key_.begin(), key_.end());
    if (record_ || windows_ > 1) put<uint32_t>(&h, windows_);   // absent from a one-window state: such states stay valid
    return h;
}

std::string InitialProofScan::state_path() const {
    return record_ ? range_record_path(dir_, range_.from_file, range_.to_file) : join(dir_, kInitialScanFile);
}

// header | pows | upto | lists (count, then nonce, length, indices) | a record's VRF best (found, index, label32) |
// FNV-1a 64 of everything before it.  A record without the scan has no pows and no lists.
int InitialProofScan::save_state() {
    std::string s = header();
    for (uint64_t p : pows_) put<uint64_t>(&s, p);
    put<uint64_t>(&s, upto());
    if (proof_) {
        put<uint32_t>(&s, (uint32_t)book().lists().size());
        for (const auto &kv : book().lists()) {
            put<uint32_t>(&s, kv.first);
            put<uint32_t>(&s, (uint32_t)kv.second.size());
            for (const KeptHit &k : kv.second) put<uint64_t>(&s, k.index);
        }
    }
    if (record_) {
        put<uint32_t>(&s, vrf_.found);
        put<uint64_t>(&s, vrf_.index);
        s.append(reinterpret_cast<const char *>(vrf_.label32), 32);
    }
    put<uint64_t>(&s, fnv1a64(s));
    return write_file_atomic(state_path(), s);
}

// The state in s, if it is intact, has this object's header and covers a prefix ending at or below `written`.
bool InitialProofScan::decode(const std::string &s, uint64_t written) {
    const std::string h = header();
    if (s.size() < h.size() + 8 || s.compare(0, h.size(), h) != 0) return false;
    uint64_t sum;
    memcpy(&sum, s.data() + s.size() - 8, 8);
    const std::string body = s.substr(0, s.size() - 8);
    if (fnv1a64(body) != sum) return false;
    size_t p = h.size();
    std::vector<uint64_t> pows(proof_ ? nonces() / 16 : 0);
    for (uint64_t &v : pows) if (!get(body, &p, &v)) return false;
    uint64_t upto;
    if (!get(body, &p, &upto) || upto > written || upto < range_.lo || upto > range_.hi) return false;
    HitBook restored(proof_ ? nonces() : 0, cfg_.k2, true);
    uint32_t n_lists = 0;
    if (proof_ && !get(body, &p, &n_lists)) return false;
    for (uint32_t i = 0; i < n_lists; i++) {
        uint32_t nonce, len;
        if (!get(body, &p, &nonce) || !get(body, &p, &len) || nonce >= nonces() || len > cfg_.k2) return false;
        for (uint64_t j = 0, v; j < len; j++) {
            if (!get(body, &p, &v) || v < range_.lo || v >= upto) return false;
            restored.add(nonce, v, nullptr);
        }
    }
    b200post_vrf_nonce vrf{};
    if (record_) {
        // the best may lie past upto (the labels after it were computed, then the session stopped), never past hi
        if (!get(body, &p, &vrf.found) || vrf.found > 1 || !get(body, &p, &vrf.index) || p + 32 > body.size()) return false;
        memcpy(vrf.label32, body.data() + p, 32);
        p += 32;
        if (vrf.found && (vrf.index < range_.lo || vrf.index >= range_.hi)) return false;
    }
    if (p != body.size()) return false;
    restored.advance(upto - range_.lo);
    pows_ = pows; vrf_ = vrf; upto_ = upto;
    if (proof_) book() = restored;
    return true;
}

bool InitialProofScan::load_state(uint64_t written) {
    std::string s;
    return read_file(state_path(), &s) && decode(s, written);
}

bool InitialProofScan::read_record(const std::string &s) {
    // the fields header() writes, in its order; decode() then compares the whole header as header() re-encodes it
    size_t p = 8;
    uint32_t version, proof = 0, key_len = 0;
    record_ = true;
    if (s.size() < 8 || s.compare(0, 8, "B2RNGREC") != 0 || !get(s, &p, &version) || version != 1 || p + 64 > s.size()) return false;
    memcpy(md_.node_id, s.data() + p, 32);
    memcpy(md_.commitment_atx_id, s.data() + p + 32, 32);
    p += 64;
    if (!get(s, &p, &md_.num_units) || !get(s, &p, &md_.labels_per_unit) || !get(s, &p, &md_.scrypt_n) ||
        !get(s, &p, &md_.max_file_size) || !get(s, &p, &range_.from_file) || !get(s, &p, &range_.to_file) ||
        !get(s, &p, &range_.lo) || !get(s, &p, &range_.hi) || !get(s, &p, &proof) || proof > 1)
        return false;
    proof_ = proof;
    const unsigned __int128 nl = (unsigned __int128)md_.num_units * md_.labels_per_unit;
    if (nl == 0 || nl > (~0ull >> 4) || range_.lo >= range_.hi || range_.hi > (uint64_t)nl) return false;
    num_labels_ = (uint64_t)nl;
    if (proof_) {
        if (!get(s, &p, &cfg_.k1) || !get(s, &p, &cfg_.k2) || !get(s, &p, &opts_.nonces) || p + 64 > s.size()) return false;
        memcpy(cfg_.pow_difficulty, s.data() + p, 32);
        p += 64;   // and the zero challenge
        if (!get(s, &p, &opts_.pow_mode) || !get(s, &p, &key_len) || p + key_len > s.size()) return false;
        key_.assign(s.begin() + (long)p, s.begin() + (long)(p + key_len));
        p += key_len;
        if (!get(s, &p, &windows_)) return false;
        if (cfg_.k2 == 0 || opts_.nonces == 0 || opts_.nonces % 16 || windows_ == 0 || windows_ > 4096 / std::min(opts_.nonces, 4096u) ||
            opts_.nonces > 4096)
            return false;
        opts_.windows_per_pass = windows_;
        opts_.pow_cache_key = key_.empty() ? nullptr : key_.data();
        opts_.pow_cache_key_len = key_.size();
        rule_.emplace(std::vector<std::pair<uint64_t, uint64_t>>{{range_.lo, range_.hi}}, 0, opts_.nonces, windows_, cfg_.k2);
    }
    return decode(s, range_.hi);
}

int InitialProofScan::begin(const InitialProofRequest *req, const RangeSpec *range, const std::string &dir,
                            const b200post_post_metadata &md, const b200post_post_config &cfg, int64_t provider_id, uint64_t *written,
                            uint64_t batch, const volatile int *cancel) {
    dir_ = dir; md_ = md; cfg_ = cfg;
    const Layout lay(md);
    num_labels_ = lay.num_labels;
    record_ = range != nullptr;
    proof_ = req != nullptr;
    range_ = record_ ? *range : RangeSpec{0, 0, 0, num_labels_};
    if (proof_) {
        opts_ = req->opts; key_ = req->cache_key;
        windows_ = std::max(opts_.windows_per_pass, 1u);
        opts_.pow_cache_key = key_.empty() ? nullptr : key_.data();
        opts_.pow_cache_key_len = key_.size();
    }
    // the session's devices: the proving scan runs on the first, a BUILTIN k2pow search on all of them
    std::vector<uint32_t> devs;
    int rc = provider_devices(provider_id, &devs);
    if (rc) return rc;
    scan_dev_ = devs[0];
    if ((rc = device_engine(scan_dev_))) return rc;

    if (proof_) rule_.emplace(std::vector<std::pair<uint64_t, uint64_t>>{{range_.lo, range_.hi}}, 0, opts_.nonces, windows_, cfg.k2);
    if (!load_state(*written)) {
        // a record restarts at lo with nothing in it; the whole POST's scan restarts at 0 and rescans what is on disk
        vrf_ = b200post_vrf_nonce{}; upto_ = range_.lo;
        if (proof_) {
            if ((rc = find_pows(opts_, kZeroChallenge, md.node_id, md.num_units, cfg.pow_difficulty, devs.data(), (int)devs.size(), 0,
                                nonces() / 16, &pows_, cancel)))
                return rc;
            // the RandomX dataset and batch (~14 GiB per device) would otherwise stay resident and shrink every label layer
            if (opts_.pow_mode == B200POST_POW_BUILTIN) for (uint32_t d : devs) randomx_release((int)d);
        }
        if ((rc = save_state())) return rc;   // a resumed session never searches again
    }
    if (record_) *written = upto();   // a record speaks of computed labels only: nothing is read back
    if (!proof_) return B200POST_OK;
    const uint64_t chunk = std::min<uint64_t>({std::max<uint64_t>(batch, 1), kMaxScanChunk, num_labels_});
    if ((rc = sc_.init(scan_dev_, kZeroChallenge, nonces(), pows_.data(), cfg.k1, cfg.k2, num_labels_, chunk))) return rc;
    // the gap between the state's prefix and what is on disk, in index order, from the files
    PostDataReader reader(dir, lay.per_file);
    for (uint64_t pos = upto(); pos < *written;) {
        if (cancel && *cancel) { stop(); set_error("cancelled"); return B200POST_ERR_CANCELLED; }
        const uint64_t n = std::min<uint64_t>(chunk, *written - pos);
        if ((rc = collect(b_)) || (rc = reader.read(pos, n, sc_.staging(b_))) || (rc = submit(b_, pos, n))) { stop(); return rc; }
        b_ ^= 1;
        pos += n;
    }
    return B200POST_OK;
}

int InitialProofScan::buffer(uint64_t count, uint8_t **dst) {
    *dst = nullptr;
    if (!proof_ || count > sc_.chunk()) return B200POST_OK;
    const int rc = collect(b_);   // the chunk that last used this staging buffer
    if (rc == B200POST_OK) *dst = sc_.staging(b_);
    return rc;
}

int InitialProofScan::scan(uint64_t first, uint64_t count, const uint8_t *src) {
    if (!proof_) { upto_ = first + count; return B200POST_OK; }
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
    for (int k = 0; k < 2 && proof_; k++) if ((rc = collect(b_ ^ k))) return rc;   // older chunk first
    return save_state();
}

// Chunks are folded in submission order, so what is folded is always a prefix of the labels.  After the first chunk
// that failed to go in or come back, nothing more is folded: a later chunk would leave a hole below upto.
int InitialProofScan::collect(int b) {
    if (failed_) { sc_.drain(); set_error("initial proof: an earlier scan chunk failed"); return B200POST_ERR_STATE; }
    const int rc = sc_.collect(b, &book());
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
    for (int k = 0; k < 2 && proof_ && !failed_; k++) collect(b_ ^ k);   // older chunk first; stops at a failure
    if (proof_) sc_.drain();
    save_state();   // upto = the end of the folded prefix, whose hits are all in the book
    set_error(err);   // the session reports its own failure, not the state's
}

int InitialProofScan::finish(b200post_proof_out *out, b200post_proof_metadata *meta) {
    int rc = checkpoint();
    if (rc) return rc;
    if (book().scanned() != num_labels_) { set_error("initial proof: the scan does not cover every label"); return B200POST_ERR_STATE; }
    uint32_t nonce = 0;
    std::vector<uint64_t> idx;
    if (!rule_->decide(&nonce, &idx, &rc)) return no_proof(windows_, opts_.nonces);   // the lowest window with a winner
    if ((rc = write_proof(num_labels_, nonce, idx, pows_.data(), 0, num_labels_, out))) return rc;
    memset(meta, 0, sizeof *meta);
    memcpy(meta->node_id, md_.node_id, 32);
    memcpy(meta->commitment_atx_id, md_.commitment_atx_id, 32);
    memcpy(meta->challenge, kZeroChallenge, 32);
    meta->num_units = md_.num_units; meta->labels_per_unit = md_.labels_per_unit;
    // the gate of b200post_generate_proof_checked: a proof this library's own verifier rejects is never handed out
    return gate_proof(scan_dev_, cfg_, md_.scrypt_n, opts_, *meta, out);
}

}  // namespace b200post
