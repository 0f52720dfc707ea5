// setup.cu — POST setup sessions (include/b200post_setup.h): the host-side mirror of
// activation.PostSetupManager (activation/post.go:185-449) and of the initializer it drives
// (un-vendored spacemeshos/post `initialization.Initializer`: files, metadata, resume, VRF nonce).
// C++ because the reference's host side is compiled Go.  The data directory's files are postdata_io.h's.
#include <dirent.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/b200post_prove.h"
#include "engine.h"
#include "host_hash.h"
#include "initial_proof.h"
#include "label_sums.h"
#include "metrics.h"
#include "postdata_io.h"
#include "setup_internal.h"

using namespace b200post;

namespace b200post {

int compute_labels(int64_t provider_id, uint64_t N, const uint8_t commitment[32], uint64_t start, uint64_t count, uint8_t *out,
                   const uint8_t *diff, b200post_vrf_nonce *nonce, const volatile int *cancel) {
    if (nonce) memset(nonce, 0, sizeof *nonce);
    if (provider_id == B200POST_PROVIDER_ALL) {
        std::vector<uint32_t> ids;
        if (int rc = provider_devices(provider_id, &ids)) return rc;
        return b200post_labels_range_multi(ids.data(), (int)ids.size(), commitment, N, start, count, out, diff, diff ? nonce : nullptr, cancel);
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
        if ((rc = save_post_metadata(dir, *md))) return rc;
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
    uint64_t range_from = 0, range_to = 0;      // of files [range_from, range_to]
    bool range() const { return range_lo != 0 || range_hi != num_labels; }
    // a file range's record (b200post_setup_request_range_record): asked for between prepare and start, kept by start
    bool want_record = false, record_proof = false;
    InitialProofRequest record_req;
    // the initial proof: asked for between prepare and start (b200post_setup_request_initial_proof), produced by start
    bool want_proof = false;
    InitialProofRequest proof_req;
    bool proof_done = false;                    // the last session that asked for it completed
    int proof_rc = B200POST_OK;                 // its outcome: OK, or INVALID_PROOF with proof_err
    std::string proof_err;
    b200post_proof_out proof{};
    b200post_proof_metadata proof_meta{};
    // block checksums (b200post_setup_request_checksums): asked for between prepare and start
    bool want_sums = false;
};

namespace {

int fail_state(b200post_setup_manager *m, int code, const std::string &msg) {
    m->state = B200POST_SETUP_ERROR;
    set_error(msg);
    return code;
}

// The self-check of a batch: label `pick`, recomputed on the host CPU, against the device's label16
int reference_check(const uint8_t commitment[32], uint64_t N, uint64_t pick, const uint8_t *label16) {
    uint8_t ref[32];
    reference_label32(commitment, pick, (uint32_t)N, ref);
    if (memcmp(ref, label16, 16) == 0) return B200POST_OK;
    metrics().setup_label_mismatch_total++;
    return fail(B200POST_ERR_LABEL_MISMATCH, "reference label mismatch at index " + std::to_string(pick));
}

// The sidecars (postdata_<N>.sum, DESIGN.md §3g) of a session that asked for them.  They are built from the labels
// the session computes, on its first device; labels already on disk are recomputed for them, never read back.
class SessionSums {
public:
    SessionSums(std::string dir, const b200post_post_metadata &md, uint64_t num_labels)
        : dir_(std::move(dir)), md_(md), lay_(num_labels, md.max_file_size / 16) {}

    // Before the first batch: each file of the range with labels below `written` gets a sidecar covering them.  The
    // whole blocks of a usable sidecar below the labels on disk are kept, and the rest, from the start of the block
    // that holds its end (from label 0 of the file when the sidecar is absent or unusable), is recomputed and hashed.
    // The initial-proof scan, the VRF scan and a range record never see these labels.
    int begin(int64_t provider_id, uint64_t from_file, uint64_t written, uint64_t batch, const uint8_t commitment[32],
              const volatile int *cancel) {
        std::vector<uint32_t> devs;
        if (int rc = provider_devices(provider_id, &devs)) return rc;
        if (int rc = device_engine(devs[0])) return rc;
        hasher_.reset(new BlockHasher((int)devs[0]));
        std::vector<uint8_t> buf;
        for (uint64_t f = from_file; f * lay_.per_file < written; f++) {
            const uint64_t base = f * lay_.per_file, have = std::min<uint64_t>(lay_.labels_in(f), written - base);
            PostSums old;
            const bool usable = load_post_sums(dir_, md_, f, lay_.per_file, &old);
            if (!usable) old = PostSums::of(md_, f);
            const bool whole_file = have == lay_.labels_in(f);
            if (usable && whole_file && old.covered == have) continue;   // nothing to add, nothing left open
            open_.reset(new FileSums(old, std::min(old.covered, have) / kSumBlockLabels * kSumBlockLabels));
            for (uint64_t at = open_->covered(); at < have;) {
                if (cancel && *cancel) { save(); return fail(B200POST_ERR_CANCELLED, "cancelled"); }
                const uint64_t n = std::min(batch, have - at);
                buf.resize((size_t)n * 16);
                int rc = compute_labels(provider_id, md_.scrypt_n, commitment, base + at, n, buf.data(), nullptr, nullptr, cancel);
                if (!rc) rc = self_check(commitment, base + at, n, buf.data());
                if (!rc) rc = open_->feed(*hasher_, buf.data(), n);
                if (rc) { if (rc == B200POST_ERR_CANCELLED) save(); return rc; }
                at += n;
            }
            if (int rc = save()) return rc;
            if (whole_file) open_.reset();
        }
        return B200POST_OK;
    }

    // labels [pos, pos + count) of one file, as the session writes them.  The sidecar is saved when they complete a
    // block and at the end of the file.
    int batch(uint64_t pos, const uint8_t *labels, uint64_t count) {
        const uint64_t f = pos / lay_.per_file, in_file = pos % lay_.per_file;
        if (!open_ || open_->file() != f) open_.reset(new FileSums(PostSums::of(md_, f), 0));
        if (open_->covered() != in_file) return fail(B200POST_ERR_STATE, "checksums: batch at label " + std::to_string(pos) + " does not continue the sidecar");
        bool completed = false;
        if (int rc = open_->feed(*hasher_, labels, count, &completed)) return rc;
        const bool file_end = in_file + count == lay_.labels_in(f);
        if (completed || file_end) {
            if (int rc = save()) return rc;
        }
        if (file_end) open_.reset();
        return B200POST_OK;
    }

    // the sidecar of the file the session is writing, as far as it got
    int save() { return open_ ? open_->save(*hasher_, dir_) : B200POST_OK; }

private:
    // the session's self-check applied to one recomputed piece
    int self_check(const uint8_t commitment[32], uint64_t start, uint64_t count, const uint8_t *labels) {
        const uint64_t pick = start + (n_checked_++ * 2654435761ull) % count;
        return reference_check(commitment, md_.scrypt_n, pick, labels + (pick - start) * 16);
    }

    std::string dir_;
    b200post_post_metadata md_;
    Layout lay_;
    std::unique_ptr<BlockHasher> hasher_;
    std::unique_ptr<FileSums> open_;
    uint64_t n_checked_ = 0;
};

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
    // a request belongs to one prepared session, and so does its outcome
    m->want_proof = m->proof_done = m->want_record = m->want_sums = false;
    m->proof_rc = B200POST_OK; m->proof_err.clear();
    m->proof = b200post_proof_out{}; m->proof_meta = b200post_proof_metadata{};
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
    const Layout lay((uint64_t)nl, o->max_file_size / 16);
    uint64_t lo = 0, hi = lay.num_labels, last_file = ~0ull;   // the whole POST: no bound on the resume scan (as before ranges)
    if (from_file != 0 || to_file != -1) {
        if (to_file < -1) return fail_state(m, B200POST_ERR_INVALID_ARGUMENT, "invalid file range: toFile < -1");
        last_file = to_file == -1 ? lay.n_files - 1 : (uint64_t)to_file;
        if (lay.n_files == 0 || from_file > last_file || last_file >= lay.n_files)
            return fail_state(m, B200POST_ERR_INVALID_ARGUMENT, "invalid file range: need fromFile <= toFile < " + std::to_string(lay.n_files) + " (the POST's files)");
        lo = from_file * lay.per_file;
        hi = last_file * lay.per_file + lay.labels_in(last_file);
    }

    const std::string dir = o->data_dir;
    int rc = make_dirs(dir);
    if (rc) { m->state = B200POST_SETUP_ERROR; return rc; }

    // ---- metadata: an existing file pins identity + commitment ATX (post.go:374-377)
    b200post_post_metadata meta;
    bool missing = false;
    rc = load_post_metadata(dir, &meta, &missing);
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
    if (!stored_labels(dir, lay.per_file, from_file, last_file, &written))
        return fail_state(m, B200POST_ERR_CONFIG_MISMATCH, "postdata file has an unexpected size");
    if (written > hi - lo) return fail_state(m, B200POST_ERR_CONFIG_MISMATCH, "DataDir holds more labels than NumUnits * LabelsPerUnit");
    // a range's labels are not VRF-scanned: without a nonce, the stored data must be searched once it is merged
    // (with one, the labels are deterministic and the nonce stays right)
    const bool range = lo != 0 || hi != lay.num_labels;
    if (range && !meta.has_nonce) meta.vrf_scan_pending = 1;

    m->opts = *o; m->data_dir = dir; m->opts.data_dir = m->data_dir.c_str();
    if (m->opts.self_check_every == 0) m->opts.self_check_every = 16;
    memcpy(m->node_id, node_id, 32);
    m->meta = meta; m->num_labels = lay.num_labels; m->have_opts = true;
    m->range_lo = lo; m->range_hi = hi;
    m->range_from = from_file; m->range_to = last_file;
    m->labels_written.store(written);
    if ((rc = save_post_metadata(dir, m->meta))) { m->state = B200POST_SETUP_ERROR; return rc; }
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

    const Layout lay(m->num_labels, m->opts.max_file_size / 16);
    const uint64_t batch = m->opts.compute_batch_size;
    const uint64_t lo = m->range_lo, hi = m->range_hi;
    const bool range = m->range();   // no nonce, no past-the-end search: a range's arg-min is not the POST's
    // a range with a record scans its labels for the VRF into the record, not into the metadata
    const bool record = range && m->want_record;
    uint64_t written = lo + m->labels_written.load();   // the next label to write
    // a session with checksums may have sidecars to complete even when every label is on disk
    const bool need_work = written < hi || (!range && (!m->meta.has_nonce || m->meta.vrf_scan_pending)) || m->want_sums;
    if (need_work && m->opts.provider_id == B200POST_PROVIDER_UNSET) {
        set_error("no provider specified");
        return finish(B200POST_SETUP_ERROR, B200POST_ERR_NO_PROVIDER);
    }
    uint8_t commitment[32];
    commitment_bytes(m->meta.node_id, m->meta.commitment_atx_id, commitment);
    uint8_t diff[32];
    if (m->meta.has_nonce) memcpy(diff, m->meta.nonce_value, 32); else vrf_difficulty(lay.num_labels, diff);   // numLabels of the whole POST

    // the initial proof: pows, state and the rescan of what is already on disk come before the first batch.  A record:
    // pows and record, and the session resumes at the record's prefix (labels past it are computed again).
    std::unique_ptr<InitialProofScan> ip;
    if (m->want_proof || record) {
        m->proof_done = false;
        if (m->opts.provider_id == B200POST_PROVIDER_UNSET) {
            set_error("no provider specified");
            return finish(B200POST_SETUP_ERROR, B200POST_ERR_NO_PROVIDER);
        }
        ip.reset(new InitialProofScan);
        const RangeSpec rs{m->range_from, m->range_to, lo, hi};
        const InitialProofRequest *req = record ? (m->record_proof ? &m->record_req : nullptr) : &m->proof_req;
        const int rc = ip->begin(req, record ? &rs : nullptr, m->data_dir, m->meta, m->cfg, m->opts.provider_id, &written, batch, cancel);
        if (rc == B200POST_ERR_CANCELLED) return finish(B200POST_SETUP_STOPPED, rc);
        if (rc) return finish(B200POST_SETUP_ERROR, rc);
        if (record) {
            m->labels_written.store(written - lo);   // the status counts from the resume point
            if (ip->vrf().found) memcpy(diff, ip->vrf().label32, 32);
        }
    }
    // the sidecars: completed up to the resume point before the first batch
    std::unique_ptr<SessionSums> sums;
    if (m->want_sums) {
        sums.reset(new SessionSums(m->data_dir, m->meta, lay.num_labels));
        const int rc = sums->begin(m->opts.provider_id, m->range_from, written, batch, commitment, cancel);
        if (rc) {
            if (ip) ip->stop();
            return finish(rc == B200POST_ERR_CANCELLED ? B200POST_SETUP_STOPPED : B200POST_SETUP_ERROR, rc);
        }
    }
    // from here on a stop or failure first saves the initial proof's scan state and the open sidecar
    auto end = [&](int32_t state, int rc) {
        if (ip) ip->stop();
        if (sums) {
            const std::string err = last_error();
            sums->save();   // best effort: the session's own outcome is what it reports
            set_error(err);
        }
        return finish(state, rc);
    };

    std::vector<uint8_t> buf;
    uint64_t n_batches = 0;
    auto note_nonce = [&](const b200post_vrf_nonce &nn) -> int {
        if (!nn.found) return B200POST_OK;
        m->meta.has_nonce = 1; m->meta.nonce = nn.index; memcpy(m->meta.nonce_value, nn.label32, 32);
        memcpy(diff, nn.label32, 32);   // only a smaller label can replace it
        return save_post_metadata(m->data_dir, m->meta);
    };

    while (written < hi) {
        if (cancel && *cancel) { set_error("cancelled"); return end(B200POST_SETUP_STOPPED, B200POST_ERR_CANCELLED); }
        const uint64_t file_idx = written / lay.per_file, in_file = written % lay.per_file;
        const uint64_t count = std::min<uint64_t>({batch, lay.per_file - in_file, hi - written});
        int rc;
        // with an initial proof the batch is computed into the scan's pinned staging, which the file is written from
        uint8_t *labels = nullptr;
        if (ip && (rc = ip->buffer(count, &labels))) return end(B200POST_SETUP_ERROR, rc);
        if (!labels) { buf.resize((size_t)count * 16); labels = buf.data(); }
        b200post_vrf_nonce nn;
        rc = compute_labels(m->opts.provider_id, m->opts.scrypt_n, commitment, written, count, labels, range && !record ? nullptr : diff,
                            &nn, cancel);
        if (rc == B200POST_ERR_CANCELLED) return end(B200POST_SETUP_STOPPED, rc);
        if (rc) return end(B200POST_SETUP_ERROR, rc);
        // ErrReferenceLabelMismatch contract (activation/post.go:299-312): every self_check_every batches one label of the
        // batch is recomputed ON THE HOST CPU (reference_label.cpp: the kernels' own arithmetic header compiled for the
        // host) and compared with what the device wrote — independent of the device, its kernels' scheduling and memory.
        if (options().debug_corrupt_next_batch.exchange(0) != 0 && count) labels[((n_batches * 7) % count) * 16 + 3] ^= 0x40;   // fault injection (tests)
        if (n_batches % m->opts.self_check_every == 0) {
            uint64_t pick = written + (n_batches * 2654435761ull) % count;
            if (options().debug_corrupt_check_all.load() != 0) {
                // test hook: check the label the injected fault hit (the sampled one is elsewhere with probability 1 - 1/count)
                pick = written + (n_batches * 7) % count;
            }
            if ((rc = reference_check(commitment, m->opts.scrypt_n, pick, labels + (pick - written) * 16))) return end(B200POST_SETUP_ERROR, rc);
        }
        n_batches++;
        // a record's VRF best covers every batch that its scan folds: it is noted before the batch goes to the scan
        if (record && nn.found) { ip->note_vrf(nn); memcpy(diff, nn.label32, 32); }
        if ((rc = write_labels(m->data_dir, file_idx, in_file, labels, count))) return end(B200POST_SETUP_ERROR, rc);
        if (sums && (rc = sums->batch(written, labels, count))) return end(B200POST_SETUP_ERROR, rc);
        // the scan of this batch overlaps the computation of the next one
        if (ip && (rc = ip->scan(written, count, labels))) return end(B200POST_SETUP_ERROR, rc);
        written += count;
        m->labels_written.store(written - lo);
        if (!record && (rc = note_nonce(nn))) return end(B200POST_SETUP_ERROR, rc);
        if (ip && (written % lay.per_file == 0 || written == hi) && (rc = ip->checkpoint())) return end(B200POST_SETUP_ERROR, rc);
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
            rc = search_past_end(m->data_dir, &m->meta, lay.num_labels, m->opts.provider_id, batch, commitment, diff, cancel);
        }
        if (rc == B200POST_ERR_CANCELLED) return end(B200POST_SETUP_STOPPED, rc);
        if (rc) return end(B200POST_SETUP_ERROR, rc);
    }
    int rc = save_post_metadata(m->data_dir, m->meta);
    if (rc) return end(B200POST_SETUP_ERROR, rc);
    if (ip && !record) {
        // every label is on disk and the VRF nonce is settled: decide, gate, publish.  No proof is not a failed session.
        b200post_proof_out proof{};
        b200post_proof_metadata pm{};
        rc = ip->finish(&proof, &pm);
        if (rc == B200POST_OK) rc = save_initial_proof_file(m->data_dir, pm, m->cfg, m->proof_req.opts.nonces, m->proof_req.opts.windows_per_pass, proof);
        else if (rc == B200POST_ERR_INVALID_PROOF) unlink(join(m->data_dir, kInitialProofFile).c_str());   // a stale one must not answer
        if (rc != B200POST_OK && rc != B200POST_ERR_INVALID_PROOF) return end(B200POST_SETUP_ERROR, rc);
        std::lock_guard<std::mutex> lk(m->mu);
        m->proof_done = true; m->proof_rc = rc; m->proof_err = rc ? last_error() : "";
        m->proof = proof; m->proof_meta = pm;
    }
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
            if (post_file_kind(name, nullptr) != PostFile::kNone && unlink(join(m->data_dir, name).c_str()) != 0) {
                closedir(d);
                return io_error("unlink " + name);
            }
        }
        closedir(d);
    }
    m->labels_written.store(0);
    memset(&m->meta, 0, sizeof m->meta);
    m->want_proof = m->proof_done = m->want_record = m->want_sums = false;
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
    return load_post_metadata(data_dir, out);
}

}  // extern "C"

namespace {

// the fields of an initial-proof request that the session's scan uses, checked and copied into *req
int take_proof_request(const b200post_prove_opts *opts, InitialProofRequest *req) {
    b200post_prove_opts o = *opts;
    if (o.nonces == 0) o.nonces = 16;
    if (o.nonces % 16 || o.nonces > 4096) { set_error("invalid nonce count (a positive multiple of 16, <= 4096)"); return B200POST_ERR_INVALID_ARGUMENT; }
    // the session's one pass scans windows_per_pass nonce windows (0 = 1, clamped to the group limit); max_windows is unused
    o.windows_per_pass = std::min(std::max(o.windows_per_pass, 1u), 4096 / o.nonces);
    o.max_windows = 0;
    const int rc = check_pow_mode(o);
    if (rc) return rc;
    req->cache_key.assign(o.pow_cache_key, o.pow_cache_key ? o.pow_cache_key + o.pow_cache_key_len : o.pow_cache_key);
    o.pow_cache_key = nullptr; o.pow_cache_key_len = 0;   // the copy above is the key
    req->opts = o;
    return B200POST_OK;
}

}  // namespace

extern "C" {

int b200post_setup_request_initial_proof(b200post_setup_manager *m, const b200post_prove_opts *opts) {
    if (!m || !opts) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    std::lock_guard<std::mutex> lk(m->mu);
    if (m->state != B200POST_SETUP_PREPARED) { set_error("post session not prepared"); return B200POST_ERR_STATE; }
    if (m->range()) { set_error("initial proof: a file-range session does not see the whole POST"); return B200POST_ERR_STATE; }
    const int rc = take_proof_request(opts, &m->proof_req);
    if (rc) return rc;
    m->want_proof = true;
    return B200POST_OK;
}

int b200post_setup_request_range_record(b200post_setup_manager *m, const b200post_prove_opts *proof) {
    if (!m) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    std::lock_guard<std::mutex> lk(m->mu);
    if (m->state != B200POST_SETUP_PREPARED) { set_error("post session not prepared"); return B200POST_ERR_STATE; }
    if (!m->range()) { set_error("range record: the session covers the whole POST (it finds the nonce and proof itself)"); return B200POST_ERR_STATE; }
    if (m->meta.has_nonce) { set_error("range record: the metadata already holds the VRF nonce"); return B200POST_ERR_STATE; }
    if (proof) {
        const int rc = take_proof_request(proof, &m->record_req);
        if (rc) return rc;
    }
    m->want_record = true;
    m->record_proof = proof != nullptr;
    return B200POST_OK;
}

int b200post_setup_request_checksums(b200post_setup_manager *m) {
    if (!m) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    std::lock_guard<std::mutex> lk(m->mu);
    if (m->state != B200POST_SETUP_PREPARED) { set_error("post session not prepared"); return B200POST_ERR_STATE; }
    m->want_sums = true;
    return B200POST_OK;
}

int b200post_setup_initial_proof(b200post_setup_manager *m, b200post_proof_out *out, b200post_proof_metadata *meta) {
    if (!m || !out) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    std::lock_guard<std::mutex> lk(m->mu);
    if (m->state != B200POST_SETUP_COMPLETE || !m->proof_done) {
        set_error("no initial proof: the session did not ask for one or has not completed");
        return B200POST_ERR_STATE;
    }
    if (m->proof_rc) { set_error(m->proof_err); return m->proof_rc; }
    *out = m->proof;
    if (meta) *meta = m->proof_meta;
    return B200POST_OK;
}

int b200post_load_initial_proof(const char *data_dir, const b200post_post_config *cfg, uint32_t nonces, b200post_proof_out *out,
                                b200post_proof_metadata *meta) {
    if (!data_dir || !cfg || !out) { set_error("invalid argument"); return B200POST_ERR_INVALID_ARGUMENT; }
    b200post_post_metadata md;
    const int rc = load_post_metadata(data_dir, &md);
    if (rc) return rc;
    return load_initial_proof_file(data_dir, md, *cfg, nonces ? nonces : 16, out, meta);
}

}  // extern "C"
