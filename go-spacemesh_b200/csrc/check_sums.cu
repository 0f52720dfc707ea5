// check_sums.cu — checking stored POST data against its block checksums, repairing the damaged blocks, and giving
// checksums to data that has none (include/b200post_setup.h: b200post_check_sums, b200post_write_sums; DESIGN.md §3g).
//   check:  the covered labels of each file are streamed file -> pinned -> device (a reader thread loads piece k + 1
//           while the device hashes piece k) and every block's digest is compared with its postdata_<N>.sum
//   repair: a bad block is recomputed by the label engine, hashed, and written back only if it matches its checksum
//   write:  the full check of b200post_verify_pos (every label recomputed and compared, K3c) file by file; the bytes it
//           matched are hashed and a file with no mismatch gets its sidecar
#include <fcntl.h>
#include <unistd.h>

#include <algorithm>
#include <cstring>
#include <future>
#include <memory>
#include <string>
#include <vector>

#include "../../include/b200post_setup.h"
#include "engine.h"
#include "host_hash.h"
#include "label_sums.h"
#include "metrics.h"
#include "postdata_io.h"
#include "setup_internal.h"

using namespace b200post;

namespace {

constexpr uint64_t kCheckPieceLabels = 64 * kSumBlockLabels;   // 64 MiB per read and per hash launch

// global labels [start, start + count) of one file
struct Piece { uint64_t file, start, count; };

void add_progress(volatile uint64_t *p, uint64_t n) {
    if (p) __atomic_fetch_add(p, n, __ATOMIC_RELAXED);
}

// body(piece, bytes) over the pieces in order, with piece k + 1 read into the other buffer while body runs on piece k
template <class Body>
int stream_pieces(const std::string &dir, uint64_t per_file, const std::vector<Piece> &pieces, uint8_t *const buf[2],
                  const volatile int *cancel, Body body) {
    if (pieces.empty()) return B200POST_OK;
    PostDataReader reader(dir, per_file);
    struct Loaded { int rc; std::string err; };
    auto load = [&](size_t k) {
        const Piece &p = pieces[k];
        Loaded l{reader.read(p.start, p.count, buf[k & 1]), ""};
        if (l.rc) l.err = last_error();
        return l;
    };
    std::future<Loaded> next = std::async(std::launch::async, load, (size_t)0);
    for (size_t k = 0; k < pieces.size(); k++) {
        const Loaded cur = next.get();
        if (cur.rc) return fail(cur.rc, cur.err);
        if (cancel && *cancel) return fail(B200POST_ERR_CANCELLED, "cancelled");
        if (k + 1 < pieces.size()) next = std::async(std::launch::async, load, k + 1);
        const int rc = body(pieces[k], buf[k & 1]);
        if (rc) {
            if (k + 1 < pieces.size()) next.wait();
            return rc;
        }
    }
    return B200POST_OK;
}

// The host checks both calls share, in order: arguments, metadata, the file range, the files' sizes
int host_checks(const char *data_dir, int64_t provider_id, bool any_provider, uint64_t from_file, int64_t to_file,
                b200post_post_metadata *md, uint64_t *last) {
    if (provider_id < 0 ? !(any_provider && provider_id == B200POST_PROVIDER_ALL) : provider_id > 0xffffffffll)
        return fail(B200POST_ERR_INVALID_ARGUMENT, "invalid provider id");
    if (to_file < -1 || (to_file >= 0 && from_file > (uint64_t)to_file)) return fail(B200POST_ERR_INVALID_ARGUMENT, "invalid file range: fromFile > toFile");
    int rc = load_post_metadata(data_dir, md);
    if (rc || (rc = check_layout(*md))) return rc;
    const Layout lay(*md);
    *last = to_file < 0 ? lay.n_files - 1 : (uint64_t)to_file;
    if (*last >= lay.n_files || from_file > *last)
        return fail(B200POST_ERR_INVALID_ARGUMENT, "invalid file range: the POST has " + std::to_string(lay.n_files) + " files");
    return check_post_files(data_dir, lay, from_file, *last);
}

void report(b200post_sums_result *out, uint64_t first_label, uint64_t count) {
    if (out->n_reported < 64) {
        out->bad[out->n_reported].first_label = first_label;
        out->bad[out->n_reported].count = count;
        out->n_reported++;
    }
}

bool pwrite_all(int fd, const uint8_t *p, size_t n, off_t o) {
    while (n) {
        const ssize_t w = pwrite(fd, p, n, o);
        if (w <= 0) return false;
        p += w; n -= (size_t)w; o += w;
    }
    return true;
}

// One bad block: recomputed, hashed and compared with its checksum, written back, synced, read back and hashed again
int repair_block(const std::string &dir, const b200post_post_metadata &md, const Layout &lay, uint32_t provider, BlockHasher &h,
                 const uint8_t commitment[32], uint64_t file, uint64_t block, uint64_t count, const uint8_t want[32],
                 const volatile int *cancel) {
    const uint64_t first = file * lay.per_file + block * kSumBlockLabels;
    std::vector<uint8_t> labels((size_t)count * 16), back(labels.size());
    uint8_t d[32];
    int rc = compute_labels(provider, md.scrypt_n, commitment, first, count, labels.data(), nullptr, nullptr, cancel);
    if (rc || (rc = h.digests(labels.data(), count, d))) return rc;
    if (memcmp(d, want, 32))
        return fail(B200POST_ERR_LABEL_MISMATCH, "recomputed block disagrees with its checksum (file " + std::to_string(file) + ", labels [" +
                                                     std::to_string(first) + ", " + std::to_string(first + count) + "))");
    const std::string path = postdata_path(dir, file);
    const int fd = open(path.c_str(), O_RDWR);
    if (fd < 0) return io_error("open " + path);
    const off_t off = (off_t)(block * kSumBlockLabels * 16);
    const bool ok = pwrite_all(fd, labels.data(), labels.size(), off) && fdatasync(fd) == 0;
    const bool read_ok = ok && parallel_pread(fd, back.data(), back.size(), off);
    if (!ok) { rc = io_error("write " + path); close(fd); return rc; }
    close(fd);
    if (!read_ok) return fail(B200POST_ERR_IO, "read back of " + path + " failed");
    if ((rc = h.digests(back.data(), count, d))) return rc;
    if (memcmp(d, want, 32)) return fail(B200POST_ERR_IO, "the repaired block of " + path + " at label " + std::to_string(first) + " reads back damaged");
    return B200POST_OK;
}

}  // namespace

extern "C" {

void b200post_default_sums_opts(b200post_sums_opts *o) {
    if (!o) return;
    memset(o, 0, sizeof *o);
    o->provider_id = 0; o->from_file = 0; o->to_file = -1; o->progress = nullptr; o->repair = 0;
}

int b200post_check_sums(const char *data_dir, const b200post_sums_opts *o, b200post_sums_result *out, const volatile int *cancel) {
    if (!data_dir || !o || !out || o->repair > 1) return fail(B200POST_ERR_INVALID_ARGUMENT, "invalid argument");
    memset(out, 0, sizeof *out);
    b200post_post_metadata md;
    uint64_t last;
    int rc = host_checks(data_dir, o->provider_id, false, o->from_file, o->to_file, &md, &last);
    if (rc) return rc;
    const std::string dir = data_dir;
    const Layout lay(md);

    // ---- sidecars: a file without a usable one is unchecked
    std::vector<PostSums> sums(last + 1 - o->from_file);
    std::vector<Piece> pieces;
    for (uint64_t f = o->from_file; f <= last; f++) {
        PostSums &s = sums[f - o->from_file];
        if (!load_post_sums(dir, md, f, lay.labels_in(f), &s)) s = PostSums::of(md, f);
        if (s.covered) out->files_checked++; else out->files_unchecked++;
        out->labels_unchecked += lay.labels_in(f) - s.covered;
        for (uint64_t at = 0; at < s.covered; at += kCheckPieceLabels)
            pieces.push_back({f, f * lay.per_file + at, std::min(kCheckPieceLabels, s.covered - at)});
    }
    if (pieces.empty())
        return fail(B200POST_ERR_STATE, "no checksums: no label of files " + std::to_string(o->from_file) + ".." + std::to_string(last) +
                                            " is covered by a usable postdata_<N>.sum (initialise with -checksums, or run -verify "
                                            "-fraction 100 -writeSums once)");

    // ---- device
    const uint32_t dev = (uint32_t)o->provider_id;
    if ((rc = device_engine(dev))) return rc;
    BlockHasher hasher((int)dev);
    PinnedBuffer<uint8_t> pin[2];
    const uint64_t most = std::max_element(pieces.begin(), pieces.end(), [](const Piece &a, const Piece &b) { return a.count < b.count; })->count;
    for (auto &p : pin) CUDA_TRY(p.resize((size_t)most * 16));
    uint8_t *const bufs[2] = {pin[0].get(), pin[1].get()};

    // ---- stream and compare
    struct Bad { uint64_t file, block, count; };
    std::vector<Bad> bad;
    std::vector<uint8_t> dg((size_t)(kCheckPieceLabels / kSumBlockLabels) * 32);
    rc = stream_pieces(dir, lay.per_file, pieces, bufs, cancel, [&](const Piece &p, const uint8_t *bytes) -> int {
        if (int r = hasher.digests(bytes, p.count, dg.data())) return r;
        const PostSums &s = sums[p.file - o->from_file];
        const uint64_t in_file = p.start - p.file * lay.per_file, b0 = in_file / kSumBlockLabels;
        const uint64_t nb = (p.count + kSumBlockLabels - 1) / kSumBlockLabels;
        for (uint64_t b = 0; b < nb; b++) {
            if (memcmp(&dg[(size_t)b * 32], &s.digests[(size_t)(b0 + b) * 32], 32) == 0) continue;
            const uint64_t count = std::min<uint64_t>(kSumBlockLabels, s.covered - (b0 + b) * kSumBlockLabels);
            bad.push_back({p.file, b0 + b, count});
            report(out, p.start + b * kSumBlockLabels, count);
        }
        out->labels_checked += p.count;
        out->bytes_read += p.count * 16;
        out->blocks_checked += nb;
        add_progress(o->progress, p.count);
        return B200POST_OK;
    });
    out->bad_blocks = bad.size();
    metrics().sums_blocks_checked_total += out->blocks_checked;
    metrics().sums_blocks_bad_total += out->bad_blocks;
    if (rc) return rc;

    // ---- repair
    if (o->repair && !bad.empty()) {
        uint8_t commitment[32];
        commitment_bytes(md.node_id, md.commitment_atx_id, commitment);
        for (const Bad &b : bad) {
            if (cancel && *cancel) return fail(B200POST_ERR_CANCELLED, "cancelled");
            const PostSums &s = sums[b.file - o->from_file];
            rc = repair_block(dir, md, lay, dev, hasher, commitment, b.file, b.block, b.count,
                              reinterpret_cast<const uint8_t *>(&s.digests[(size_t)b.block * 32]), cancel);
            if (rc) return rc;
            out->repaired_blocks++;
            metrics().sums_blocks_repaired_total++;
        }
    }
    if (out->bad_blocks > out->repaired_blocks)
        return fail(B200POST_ERR_LABEL_MISMATCH, std::to_string(out->bad_blocks) + " blocks differ from their checksums");
    if (out->labels_unchecked)
        return fail(B200POST_ERR_STATE, std::to_string(out->labels_unchecked) + " labels of the range have no checksum: the check is incomplete");
    return B200POST_OK;
}

int b200post_write_sums(const char *data_dir, const b200post_sums_opts *o, b200post_sums_result *out, const volatile int *cancel) {
    if (!data_dir || !o || !out || o->repair) return fail(B200POST_ERR_INVALID_ARGUMENT, "invalid argument");
    memset(out, 0, sizeof *out);
    b200post_post_metadata md;
    uint64_t last;
    int rc = host_checks(data_dir, o->provider_id, true, o->from_file, o->to_file, &md, &last);
    if (rc) return rc;
    const std::string dir = data_dir;
    const Layout lay(md);
    std::vector<uint32_t> devs;
    if ((rc = provider_devices(o->provider_id, &devs))) return rc;
    std::vector<DeviceEngine *> engines;
    if ((rc = device_engines(devs.data(), (int)devs.size(), &engines))) return rc;
    uint8_t commitment[32];
    commitment_bytes(md.node_id, md.commitment_atx_id, commitment);

    // contiguous shares of the files, one per device; each device checks, hashes and saves its own files
    struct Share {
        uint64_t labels = 0, bytes = 0, blocks = 0, saved = 0, unsaved = 0;
        std::vector<uint64_t> bad;   // first labels of blocks that hold a mismatch (the lowest the compare reported)
        std::vector<uint64_t> bad_count;
    };
    const size_t G = engines.size();
    const uint64_t nf = last + 1 - o->from_file, per = (nf + G - 1) / G;
    std::vector<Share> shares(G);
    rc = fan_out(G, [&](size_t g) -> int {
        DeviceEngine *e = engines[g];
        Share &sh = shares[g];
        const uint64_t f0 = std::min(last + 1, o->from_file + per * g), f1 = std::min(last + 1, f0 + per);
        if (f0 >= f1) return B200POST_OK;
        // >= 4 layers per compare call keep the engine's pipeline filled (as verify_pos), in whole blocks
        const uint64_t wave = e->wave_slots(md.scrypt_n);
        if (wave == 0) return B200POST_ERR_CUDA;
        const uint64_t want = std::max<uint64_t>(4 * wave, std::min<uint64_t>(8 * wave, 1ull << 22));
        const uint64_t chunk = (want + kSumBlockLabels - 1) / kSumBlockLabels * kSumBlockLabels;
        std::vector<Piece> pieces;
        for (uint64_t f = f0; f < f1; f++)
            for (uint64_t at = 0; at < lay.labels_in(f); at += chunk) pieces.push_back({f, f * lay.per_file + at, std::min(chunk, lay.labels_in(f) - at)});
        CUDA_TRY(cudaSetDevice(e->device()));
        PinnedBuffer<uint8_t> pin[2];
        const uint64_t most = std::min<uint64_t>(chunk, lay.per_file);
        for (auto &p : pin) CUDA_TRY(p.resize((size_t)most * 16));
        uint8_t *const bufs[2] = {pin[0].get(), pin[1].get()};
        BlockHasher hasher(e->device());
        std::unique_ptr<FileSums> fs;
        bool clean = true;
        return stream_pieces(dir, lay.per_file, pieces, bufs, cancel, [&](const Piece &p, const uint8_t *bytes) -> int {
            const uint64_t in_file = p.start - p.file * lay.per_file;
            if (in_file == 0) { fs.reset(new FileSums(PostSums::of(md, p.file), 0)); clean = true; }
            CompareResult cmp;
            int r = e->labels_compare_range(commitment, md.scrypt_n, p.start, p.count, bytes, nullptr, nullptr, &cmp, cancel);
            if (r) return r;
            sh.labels += p.count;
            sh.bytes += p.count * 16;
            sh.blocks += (p.count + kSumBlockLabels - 1) / kSumBlockLabels;
            add_progress(o->progress, p.count);
            for (uint64_t q : cmp.first) {
                const uint64_t blk = (in_file + q) / kSumBlockLabels;
                const uint64_t first = p.file * lay.per_file + blk * kSumBlockLabels;
                if (!sh.bad.empty() && sh.bad.back() == first) continue;
                sh.bad.push_back(first);
                sh.bad_count.push_back(std::min<uint64_t>(kSumBlockLabels, lay.labels_in(p.file) - blk * kSumBlockLabels));
            }
            if (cmp.mismatches) clean = false;
            if (clean && (r = fs->feed(hasher, bytes, p.count))) return r;
            if (in_file + p.count == lay.labels_in(p.file)) {   // the file's end: a sidecar for a clean file only
                if (!clean) { sh.unsaved++; return B200POST_OK; }
                if ((r = fs->save(hasher, dir))) return r;
                sh.saved++;
            }
            return B200POST_OK;
        });
    });
    std::vector<std::pair<uint64_t, uint64_t>> bad;
    for (const Share &sh : shares) {
        out->labels_checked += sh.labels; out->bytes_read += sh.bytes; out->blocks_checked += sh.blocks;
        out->files_checked += sh.saved; out->files_unchecked += sh.unsaved;
        for (size_t i = 0; i < sh.bad.size(); i++) bad.push_back({sh.bad[i], sh.bad_count[i]});
    }
    std::sort(bad.begin(), bad.end());
    out->bad_blocks = bad.size();
    for (const auto &b : bad) report(out, b.first, b.second);
    metrics().post_data_labels_verified_total += out->labels_checked;
    metrics().sums_blocks_checked_total += out->blocks_checked;
    metrics().sums_blocks_bad_total += out->bad_blocks;
    if (rc) return rc;
    if (out->files_unchecked)
        return fail(B200POST_ERR_LABEL_MISMATCH, std::to_string(out->files_unchecked) + " files hold labels that differ from their recomputation: "
                                                     "they got no checksums");
    return B200POST_OK;
}

}  // extern "C"
