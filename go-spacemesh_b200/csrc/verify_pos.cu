// verify_pos.cu — checking stored POST data (include/b200post_setup.h, b200post_verify_pos): the counterpart of
// postcli -verify (spacemeshos/post verifying.VerifyPos -> post-rs verify_pos, recalled, unpinned).  The labels of a
// share of each postdata_N.bin are recomputed by the label engine and compared on the device (K3c) with the stored
// bytes, which a reader thread loads one chunk ahead of the engine.
//   fraction 100: range compare jobs over the checked files, with the VRF scan (arg-min) fused in
//   fraction < 100: per file max(1, floor(L * fraction / 100)) positions drawn from (seed, file), indexed compare jobs
#include <sys/random.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <future>
#include <memory>
#include <string>
#include <vector>

#include "../../include/b200post_setup.h"
#include "engine.h"
#include "host_hash.h"
#include "metrics.h"
#include "postdata_io.h"

using namespace b200post;

namespace {

// splitmix64: the sampler's generator (which labels a sample picks is not an interop property)
struct Rng {
    uint64_t s;
    uint64_t next() {
        uint64_t z = (s += 0x9e3779b97f4a7c15ull);
        z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
        z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
        return z ^ (z >> 31);
    }
    uint64_t below(uint64_t m) { return (uint64_t)(((unsigned __int128)next() * m) >> 64); }   // [0, m)
};

uint64_t sample_size(uint64_t labels, double fraction) {
    if (fraction >= 100.0) return labels;
    const double k = std::floor((double)labels * fraction / 100.0);
    return std::max<uint64_t>(1, std::min<uint64_t>(labels, (uint64_t)k));
}

// A file's sample is read as one sequential stream when it holds >= 1 position per 4 KiB page (256 labels), with one
// positioned read per touched page otherwise.  (The crossover is a guess; it has not been measured.)
constexpr uint64_t kDenseLabelsPerPosition = 256;
constexpr uint64_t kSeqReadLabels = 1ull << 20;   // 16 MiB per sequential read
constexpr uint64_t kMaxSampleChunk = 1ull << 22;  // positions per indexed compare job

// The k positions of one file's sample: distinct, ascending, every k-subset of [0, L) equally likely, determined by
// (seed, file).  They come out in pieces, so a check holds at most one job's worth of them:
//   k == L: every position;
//   k > L / 64 or k > kMaxSampleChunk: selection sampling (Knuth, Algorithm S), streamed from O(1) state with one
//     draw per label, which costs less than recomputing the k labels;
//   otherwise drawn whole (<= kMaxSampleChunk positions): i.i.d. draws, sorted and de-duplicated, the shortfall drawn
//     again until k distinct remain.  That set is the first k distinct values of an i.i.d. sequence, so it is uniform.
class FileSampler {
public:
    FileSampler(uint64_t seed, uint64_t file, uint64_t L, uint64_t k) : L_(L), need_(k) {
        Rng seeder{seed};
        r_.s = seeder.next() ^ Rng{file ^ 0x5350414345ull}.next();
        if (k >= L) { mode_ = ALL; return; }
        if (k > L / 64 || k > kMaxSampleChunk) { mode_ = STREAM; return; }
        mode_ = WHOLE;
        while (all_.size() < k) {
            for (uint64_t d = k - all_.size(); d; d--) all_.push_back(r_.below(L));
            std::sort(all_.begin(), all_.end());
            all_.erase(std::unique(all_.begin(), all_.end()), all_.end());
        }
    }
    // the next n positions (n <= what is left of the sample)
    void next(size_t n, uint64_t *out) {
        if (mode_ == ALL) {
            for (size_t j = 0; j < n; j++) out[j] = i_++;
        } else if (mode_ == WHOLE) {
            std::copy(all_.begin() + (ptrdiff_t)at_, all_.begin() + (ptrdiff_t)(at_ + n), out);
            at_ += n;
        } else {
            for (size_t j = 0; j < n; i_++)
                if (r_.below(L_ - i_) < need_) { out[j++] = i_; need_--; }
        }
    }

private:
    enum { ALL, STREAM, WHOLE } mode_;
    uint64_t L_, need_, i_ = 0;
    Rng r_{0};
    std::vector<uint64_t> all_;
    size_t at_ = 0;
};

// one compare job and the stored labels it checks
struct Chunk {
    uint64_t start = 0, count = 0;     // range job: global labels [start, start + count)
    std::vector<uint64_t> idx;         // indexed job: global label indices (ascending)
    std::vector<uint8_t> expect;       // count x 16 stored bytes
    int rc = B200POST_OK;
    std::string err;
};

// the next n positions of one file's sample; a compare job takes pieces of consecutive files up to kMaxSampleChunk items
struct SamplePiece { uint64_t file; size_t n; bool dense; };

struct DevResult {
    int rc = B200POST_OK;
    std::string err;
    uint64_t labels = 0, files = 0, mismatches = 0;
    std::vector<uint64_t> bad;   // lowest mismatching global indices, ascending (<= 64)
    VrfResult best;              // full check: VRF arg-min over the device's share
};

void add_progress(volatile uint64_t *p, uint64_t n) {
    if (p) __atomic_fetch_add(p, n, __ATOMIC_RELAXED);
}

// Runs the chunks of one device: a reader thread loads chunk k + 1 while the engine compares chunk k.
template <class Load>
void run_chunks(DeviceEngine *e, size_t n_chunks, Load load, const uint8_t commitment[32], uint64_t N, const uint8_t *diff,
                const b200post_verify_pos_opts &o, const volatile int *cancel, DevResult *res) {
    if (n_chunks == 0) return;
    std::future<Chunk> next = std::async(std::launch::async, load, (size_t)0);
    for (size_t k = 0; k < n_chunks; k++) {
        Chunk cur = next.get();
        if (cur.rc) { res->rc = cur.rc; res->err = cur.err; return; }
        if (k + 1 < n_chunks) next = std::async(std::launch::async, load, k + 1);
        CompareResult cmp;
        VrfResult vr;
        int rc;
        if (cur.idx.empty()) {
            rc = e->labels_compare_range(commitment, N, cur.start, cur.count, cur.expect.data(), diff, diff ? &vr : nullptr, &cmp, cancel);
        } else {
            rc = e->labels_compare_indexed(commitment, cur.idx.size(), cur.idx.data(), N, cur.expect.data(), &cmp, cancel);
        }
        if (rc != B200POST_OK && rc != B200POST_ERR_CANCELLED) {
            res->rc = rc; res->err = last_error();
            if (k + 1 < n_chunks) next.wait();
            return;
        }
        res->mismatches += cmp.mismatches;
        for (uint64_t p : cmp.first) {
            if (res->bad.size() >= CompareResult::kMaxReported) break;
            res->bad.push_back(cur.idx.empty() ? cur.start + p : cur.idx[(size_t)p]);
        }
        if (rc == B200POST_ERR_CANCELLED) {
            res->rc = rc; res->err = "cancelled";
            if (k + 1 < n_chunks) next.wait();
            return;
        }
        res->labels += cur.count;
        add_progress(o.progress, cur.count);
        if (diff && vr.found && (!res->best.found || vrf_less(vr.label32, vr.index, res->best.label32, res->best.index))) res->best = vr;
    }
}

// fraction 100: labels [lo, hi) of the POST as range compare jobs
void check_range(DeviceEngine *e, const Layout &lay, const std::string &dir, uint64_t lo, uint64_t hi, const uint8_t commitment[32],
                 uint64_t N, const uint8_t *diff, const b200post_verify_pos_opts &o, const volatile int *cancel, DevResult *res) {
    if (hi <= lo) return;
    // >= 4 layers per call keep the software pipeline filled, and consecutive calls continue it (speculative fill)
    const uint64_t wave = e->wave_slots(N);
    if (wave == 0) { res->rc = B200POST_ERR_CUDA; res->err = last_error(); return; }
    const uint64_t chunk = std::max<uint64_t>(4 * wave, std::min<uint64_t>(8 * wave, 1ull << 22));
    const size_t n_chunks = (size_t)((hi - lo + chunk - 1) / chunk);
    PostDataReader reader(dir, lay.per_file);
    auto load = [&](size_t k) {
        Chunk c;
        c.start = lo + (uint64_t)k * chunk;
        c.count = std::min<uint64_t>(chunk, hi - c.start);
        c.expect.resize((size_t)c.count * 16);
        if ((c.rc = reader.read(c.start, c.count, c.expect.data()))) c.err = last_error();
        return c;
    };
    run_chunks(e, n_chunks, load, commitment, N, diff, o, cancel, res);
}

// fraction < 100: the samples of files [f0, f1).  Small samples of consecutive files share one indexed compare job, so that
// a sparse check does not pay one pipeline fill and drain per file.  The plan needs only the sample sizes; positions are
// drawn by the loader, on the reader thread one job ahead of the engine, and dropped once their job is built.
void check_sampled(DeviceEngine *e, const Layout &lay, const std::string &dir, uint64_t f0, uint64_t f1, uint64_t seed,
                   double fraction, const uint8_t commitment[32], uint64_t N, const b200post_verify_pos_opts &o,
                   const volatile int *cancel, DevResult *res) {
    std::vector<std::vector<SamplePiece>> jobs(1);
    size_t in_job = 0;
    for (uint64_t f = f0; f < f1; f++) {
        const uint64_t L = lay.labels_in(f), k = sample_size(L, fraction);
        const bool dense = k * kDenseLabelsPerPosition >= L;
        for (uint64_t left = k; left;) {
            if (in_job == kMaxSampleChunk) { jobs.emplace_back(); in_job = 0; }
            const size_t n = (size_t)std::min<uint64_t>(left, kMaxSampleChunk - in_job);
            jobs.back().push_back({f, n, dense});
            in_job += n;
            left -= n;
        }
    }
    PostDataReader reader(dir, lay.per_file);
    std::unique_ptr<FileSampler> sampler;   // of the file the last piece came from; pieces of a file load in order
    uint64_t sampler_file = ~0ull;
    auto load = [&](size_t i) {
        Chunk c;
        for (const SamplePiece &p : jobs[i]) c.count += p.n;
        c.idx.resize((size_t)c.count);
        c.expect.resize((size_t)c.count * 16);
        std::vector<uint8_t> buf;
        std::vector<uint64_t> pos;
        size_t at = 0;   // items of the job filled so far
        for (const SamplePiece &p : jobs[i]) {
            if (p.file != sampler_file) {
                const uint64_t L = lay.labels_in(p.file);
                sampler = std::make_unique<FileSampler>(seed, p.file, L, sample_size(L, fraction));
                sampler_file = p.file;
            }
            pos.resize(p.n);
            sampler->next(p.n, pos.data());
            const uint64_t base = p.file * lay.per_file;
            uint8_t *exp = &c.expect[at * 16];
            for (size_t j = 0; j < p.n; j++) c.idx[at + j] = base + pos[j];
            size_t j = 0;
            if (p.dense) {
                // sequential reads over the span of the piece; positions are picked from memory
                buf.resize((size_t)std::min<uint64_t>(kSeqReadLabels, pos[p.n - 1] - pos[0] + 1) * 16);
                for (uint64_t s = pos[0]; j < p.n;) {
                    const uint64_t n = std::min<uint64_t>(kSeqReadLabels, pos[p.n - 1] + 1 - s);
                    if ((c.rc = reader.read(base + s, n, buf.data()))) break;
                    for (; j < p.n && pos[j] < s + n; j++) memcpy(exp + j * 16, &buf[(size_t)(pos[j] - s) * 16], 16);
                    if (j < p.n) s = pos[j];
                }
            } else {
                // one positioned read per 4 KiB page that holds positions
                buf.resize(kDenseLabelsPerPosition * 16);
                while (j < p.n) {
                    const uint64_t page = pos[j] / kDenseLabelsPerPosition;
                    size_t e2 = j;
                    while (e2 < p.n && pos[e2] / kDenseLabelsPerPosition == page) e2++;
                    if ((c.rc = reader.read_in_file(p.file, pos[j], pos[e2 - 1] + 1 - pos[j], buf.data()))) break;
                    for (size_t q = j; q < e2; q++) memcpy(exp + q * 16, &buf[(size_t)(pos[q] - pos[j]) * 16], 16);
                    j = e2;
                }
            }
            if (c.rc) { c.err = last_error(); break; }
            at += p.n;
        }
        return c;
    };
    run_chunks(e, f1 > f0 ? jobs.size() : 0, load, commitment, N, nullptr, o, cancel, res);
    if (res->rc == B200POST_OK) res->files = f1 - f0;
}

}  // namespace

extern "C" {

void b200post_default_verify_pos_opts(b200post_verify_pos_opts *o) {
    if (!o) return;
    memset(o, 0, sizeof *o);
    o->provider_id = 0; o->fraction = 0.2; o->from_file = 0; o->to_file = -1; o->seed = 0; o->progress = nullptr;
}

int b200post_verify_pos_sample(uint64_t seed, uint64_t file, uint64_t labels_in_file, double fraction, uint64_t *out,
                               uint64_t cap, uint64_t *n) {
    if (!n || labels_in_file == 0 || !(fraction > 0.0 && fraction <= 100.0)) return fail(B200POST_ERR_INVALID_ARGUMENT, "invalid argument");
    *n = sample_size(labels_in_file, fraction);
    if (!out) return B200POST_OK;
    if (cap < *n) return fail(B200POST_ERR_INVALID_ARGUMENT, "output buffer holds fewer positions than the sample");
    FileSampler(seed, file, labels_in_file, *n).next((size_t)*n, out);
    return B200POST_OK;
}

int b200post_verify_pos(const char *data_dir, const b200post_verify_pos_opts *o, b200post_verify_pos_result *out,
                        const volatile int *cancel) {
    if (!data_dir || !o || !out) return fail(B200POST_ERR_INVALID_ARGUMENT, "invalid argument");
    memset(out, 0, sizeof *out);
    if (!(o->fraction > 0.0 && o->fraction <= 100.0)) return fail(B200POST_ERR_INVALID_ARGUMENT, "invalid fraction: must be in (0, 100]");
    if (o->provider_id < 0 && o->provider_id != B200POST_PROVIDER_ALL) return fail(B200POST_ERR_INVALID_ARGUMENT, "invalid provider id");
    if (o->to_file < -1 || (o->to_file >= 0 && o->from_file > (uint64_t)o->to_file))
        return fail(B200POST_ERR_INVALID_ARGUMENT, "invalid file range: fromFile > toFile");

    // ---- metadata and files, on the host before any device is touched
    b200post_post_metadata md;
    int rc = load_post_metadata(data_dir, &md);
    if (rc || (rc = check_layout(md))) return rc;
    const Layout lay(md);
    const uint64_t N = md.scrypt_n;
    const uint64_t last = o->to_file < 0 ? lay.n_files - 1 : (uint64_t)o->to_file;
    if (last >= lay.n_files || o->from_file > last)
        return fail(B200POST_ERR_INVALID_ARGUMENT, "invalid file range: the POST has " + std::to_string(lay.n_files) + " files");
    const std::string dir = data_dir;
    if ((rc = check_post_files(dir, lay, o->from_file, last))) return rc;
    uint64_t seed = o->seed;
    while (seed == 0) {
        if (getrandom(&seed, sizeof seed, 0) != (ssize_t)sizeof seed) return fail(B200POST_ERR_IO, "getrandom failed");
    }
    out->seed = seed;

    // ---- devices
    std::vector<uint32_t> devs;
    if ((rc = provider_devices(o->provider_id, &devs))) return rc;
    std::vector<DeviceEngine *> engines;
    if ((rc = device_engines(devs.data(), (int)devs.size(), &engines))) return rc;

    uint8_t commitment[32], diff[32];
    commitment_bytes(md.node_id, md.commitment_atx_id, commitment);
    vrf_difficulty(lay.num_labels, diff);
    const bool full = o->fraction >= 100.0;
    const bool whole = full && o->from_file == 0 && last + 1 == lay.n_files;   // the fused VRF scan sees every label

    // ---- contiguous shares: of the checked label range (full check) or of the files (sampled check)
    const size_t G = engines.size();
    std::vector<DevResult> res(G);
    auto work = [&](size_t g) {
        if (full) {
            const uint64_t lo = o->from_file * lay.per_file, hi = std::min<uint64_t>((last + 1) * lay.per_file, lay.num_labels);
            const uint64_t per = (hi - lo + G - 1) / G;
            const uint64_t a = std::min<uint64_t>(hi, lo + per * g), b = std::min<uint64_t>(hi, a + per);
            check_range(engines[g], lay, dir, a, b, commitment, N, whole ? diff : nullptr, *o, cancel, &res[g]);
        } else {
            const uint64_t nf = last + 1 - o->from_file, per = (nf + G - 1) / G;
            const uint64_t a = std::min<uint64_t>(last + 1, o->from_file + per * g), b = std::min<uint64_t>(last + 1, a + per);
            check_sampled(engines[g], lay, dir, a, b, seed, o->fraction, commitment, N, *o, cancel, &res[g]);
        }
    };
    if (G == 1) work(0);
    else fan_out(G, [&](size_t g) { work(g); return B200POST_OK; });   // the parts' outcomes are in res, merged below

    // ---- merge
    int status = B200POST_OK;
    std::vector<uint64_t> bad;
    VrfResult best;
    for (size_t g = 0; g < G; g++) {
        const DevResult &r = res[g];
        if (r.rc && r.rc != B200POST_ERR_CANCELLED && status == B200POST_OK) {
            set_error(G > 1 ? "provider " + std::to_string(engines[g]->device()) + ": " + r.err : r.err);
            status = r.rc;
        }
        out->labels_checked += r.labels; out->mismatches += r.mismatches;
        bad.insert(bad.end(), r.bad.begin(), r.bad.end());
        if (r.best.found && (!best.found || vrf_less(r.best.label32, r.best.index, best.label32, best.index))) best = r.best;
    }
    out->files_checked = full ? last + 1 - o->from_file : 0;
    for (size_t g = 0; g < G && !full; g++) out->files_checked += res[g].files;
    std::sort(bad.begin(), bad.end());
    out->n_reported = (uint32_t)std::min<size_t>(bad.size(), 64);
    for (uint32_t i = 0; i < out->n_reported; i++) out->bad_index[i] = bad[i];
    metrics().post_data_labels_verified_total += out->labels_checked;
    metrics().post_data_label_mismatch_total += out->mismatches;
    if (status) return status;
    bool cancelled = false;
    for (const DevResult &r : res) cancelled |= r.rc == B200POST_ERR_CANCELLED;
    if (cancelled) { out->files_checked = 0; return fail(B200POST_ERR_CANCELLED, "cancelled"); }

    // ---- the VRF nonce: its label recomputed and compared with NonceValue; for a whole-POST check also the arg-min
    if (md.has_nonce) {
        uint8_t l32[32];
        if ((rc = label32_at(engines[0], commitment, N, md.nonce, l32))) return rc;
        out->nonce_ok = memcmp(l32, md.nonce_value, 32) == 0;
    }
    if (whole && md.has_nonce) {
        out->argmin_checked = 1;
        if (best.found)   // the smallest label below the threshold, lowest index on ties
            out->argmin_ok = best.index == md.nonce && memcmp(best.label32, md.nonce_value, 32) == 0;
        else              // none inside the POST: the search went past its end
            out->argmin_ok = md.nonce >= lay.num_labels && memcmp(md.nonce_value, diff, 32) < 0 && out->nonce_ok;
    }
    if (out->mismatches) return fail(B200POST_ERR_LABEL_MISMATCH, std::to_string(out->mismatches) + " stored labels differ from their recomputation");
    if (!md.has_nonce) {
        // the labels are what they should be, but initialisation stopped before the VRF nonce was found: not a damaged
        // POST, and not a usable one either
        return fail(B200POST_ERR_STATE, "the stored labels match, but the metadata has no VRF nonce: initialisation has not finished");
    }
    if (!out->nonce_ok) return fail(B200POST_ERR_LABEL_MISMATCH, "the VRF nonce's label differs from the metadata's NonceValue");
    return B200POST_OK;
}

}  // extern "C"
