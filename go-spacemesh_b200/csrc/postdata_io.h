// postdata_io.h — the POST data directory (DESIGN.md §3f): file names, the file layout, every read and write of its files.
// The labels, the metadata and initial_post.json are encoded here; the scan state and the range records are laid out by
// InitialProofScan (initial_proof.cu).  Errors return a B200POST_* code with the text in b200post_last_error().
#pragma once
#include <sys/types.h>

#include <algorithm>
#include <cstdint>
#include <string>

#include "../../include/b200post_prove.h"

namespace b200post {

// ---- names
extern const char kMetadataFile[];       // postdata_metadata.json
extern const char kInitialProofFile[];   // initial_post.json
extern const char kInitialScanFile[];    // initial_post.scan
extern const uint8_t kZeroChallenge[32];   // shared.ZeroChallenge: the challenge of the initial proof

// dir/name, with no doubled '/'; an empty dir gives the bare name
std::string join(const std::string &dir, const std::string &name);
std::string postdata_path(const std::string &dir, uint64_t file);
std::string range_record_path(const std::string &dir, uint64_t from_file, uint64_t to_file);
std::string sums_path(const std::string &dir, uint64_t file);   // postdata_<file>.sum

// Which of the directory's files a directory entry is.  *tmp (may be NULL): the entry is the ".tmp" of one of them,
// left by an atomic write that did not finish.
enum class PostFile { kNone, kLabels, kMetadata, kInitialProof, kInitialScan, kRangeRecord, kSums };
PostFile post_file_kind(const std::string &name, bool *tmp);

// ---- layout: numLabels in files of MaxFileSize / 16 labels, the last one possibly shorter
struct Layout {
    Layout(uint64_t labels, uint64_t per_file) : num_labels(labels), per_file(per_file), n_files(per_file ? (labels + per_file - 1) / per_file : 0) {}
    // as the metadata gives it: check_layout() says whether that is usable
    explicit Layout(const b200post_post_metadata &md) : Layout((uint64_t)md.num_units * md.labels_per_unit, md.max_file_size / 16) {}
    uint64_t labels_in(uint64_t f) const { return std::min<uint64_t>(per_file, num_labels - f * per_file); }
    uint64_t num_labels, per_file, n_files;
};
// B200POST_ERR_IO "corrupt metadata: ..." unless md's label count, MaxFileSize and Scrypt.N are in range
int check_layout(const b200post_post_metadata &md);

// ---- files
int io_error(const std::string &what);   // B200POST_ERR_IO "<what>: strerror(errno)"
int make_dirs(const std::string &dir);    // mkdir -p
// bytes to path + ".tmp", then renamed over path
int write_file_atomic(const std::string &path, const std::string &bytes);
// the whole file; false with errno set by the call that failed (ENOENT when it is absent)
bool read_file(const std::string &path, std::string *bytes);

// "POST data is incomplete": files [from_file, last_file] exist with the sizes the layout implies.  Reads no label.
int check_post_files(const std::string &dir, const Layout &lay, uint64_t from_file, uint64_t last_file);
// Labels already stored from file from_file on: whole files, then at most one partial file, up to last_file.  False
// when a file holds a partial label or more than per_file labels.
bool stored_labels(const std::string &dir, uint64_t per_file, uint64_t from_file, uint64_t last_file, uint64_t *labels);
// labels [in_file, in_file + count) of one file (created when absent), in one positioned write loop
int write_labels(const std::string &dir, uint64_t file, uint64_t in_file, const uint8_t *labels, uint64_t count);

// pread of [off, off + bytes) into dst on up to 8 threads (pread is position-independent, so slices are independent)
bool parallel_pread(int fd, uint8_t *dst, size_t bytes, off_t off);

// Labels of one POST by global label index, over files of `labels_per_file` labels; keeps the last file open.
class PostDataReader {
public:
    PostDataReader(std::string dir, uint64_t labels_per_file) : dir_(std::move(dir)), per_file_(labels_per_file) {}
    ~PostDataReader();
    PostDataReader(const PostDataReader &) = delete;
    // labels [pos, pos + n) into dst (n x 16 bytes); the range may span files
    int read(uint64_t pos, uint64_t n, uint8_t *dst);
    // one positioned read of labels [in_file, in_file + n) of one file, on the calling thread
    int read_in_file(uint64_t file, uint64_t in_file, uint64_t n, uint8_t *dst);

private:
    int open_file(uint64_t file);
    std::string dir_;
    uint64_t per_file_;
    int fd_ = -1;
    uint64_t open_ = ~0ull;
};

// ---- the JSON files
int save_post_metadata(const std::string &dir, const b200post_post_metadata &m);
// B200POST_ERR_IO "metadata file is missing" when absent (*missing, may be NULL, then says so)
int load_post_metadata(const std::string &dir, b200post_post_metadata *m, bool *missing = nullptr);
// initial_post.json: the proof for the zero challenge, the POST it belongs to, K1, K2, the pow difficulty, the nonce
// count and (above 1) the nonce windows scanned
int save_initial_proof_file(const std::string &dir, const b200post_proof_metadata &pm, const b200post_post_config &cfg, uint32_t nonces,
                            uint32_t windows, const b200post_proof_out &p);
// the proof in initial_post.json if it answers the zero challenge for this POST (md), cfg and nonce count; B200POST_ERR_IO
// "no initial proof: <why>" otherwise
int load_initial_proof_file(const std::string &dir, const b200post_post_metadata &md, const b200post_post_config &cfg, uint32_t nonces,
                            b200post_proof_out *out, b200post_proof_metadata *pm);

// ---- postdata_<N>.sum (DESIGN.md §3g): BLAKE3 digests of one postdata file's labels in blocks of kSumBlockLabels,
// aligned to the file's first label.  `covered` labels [0, covered) are described: every digest covers a whole block
// except possibly the last, which covers [floor((covered - 1) / B) * B, covered).  Written only from labels computed
// on a device (or, by b200post_write_sums, from stored bytes a full recomputation has just matched), never from bytes
// read back: labels are deterministic, so no session makes a sidecar wrong, and labels past `covered` are unchecked.
constexpr uint64_t kSumBlockLabels = 1ull << 16;   // 1 MiB of labels
struct PostSums {
    uint8_t node_id[32] = {0}, commitment_atx_id[32] = {0};
    uint64_t scrypt_n = 0, labels_per_file = 0, file = 0, covered = 0;
    std::string digests;   // ceil(covered / kSumBlockLabels) x 32 bytes
    // the header of `file` of the POST md describes, covering nothing
    static PostSums of(const b200post_post_metadata &md, uint64_t file);
    uint64_t blocks() const { return (covered + kSumBlockLabels - 1) / kSumBlockLabels; }
};
int save_post_sums(const std::string &dir, const PostSums &s);
// The sidecar of `file`: true with *out filled when it is intact (magic, version, block size, checksum, length), made
// for this POST (NodeId, CommitmentAtxId, Scrypt.N, labels per file) and this file, and covers at most max_labels.
// False when it is absent or unusable.
bool load_post_sums(const std::string &dir, const b200post_post_metadata &md, uint64_t file, uint64_t max_labels, PostSums *out);

}  // namespace b200post
