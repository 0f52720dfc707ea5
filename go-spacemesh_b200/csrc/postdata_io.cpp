// postdata_io.cpp — see postdata_io.h.  The JSON files restate the published spacemeshos/post layout (ASSUMED, "parity
// unpinned"); tests/golden/post_files pins their bytes.
#include "postdata_io.h"

#include <errno.h>
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <cstdio>
#include <cstring>
#include <thread>
#include <vector>

#include "engine.h"

namespace b200post {

const char kMetadataFile[] = "postdata_metadata.json";
const char kInitialProofFile[] = "initial_post.json";
const char kInitialScanFile[] = "initial_post.scan";
const uint8_t kZeroChallenge[32] = {0};

namespace {

bool ends_with(const std::string &s, const char *suffix) {
    const size_t n = strlen(suffix);
    return s.size() >= n && s.compare(s.size() - n, n, suffix) == 0;
}

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

int no_initial_proof(const std::string &why) { return fail(B200POST_ERR_IO, "no initial proof: " + why); }

const char kShortRead[] = "POST data is incomplete (short read): initialisation not finished?";

bool pread_all(int fd, uint8_t *d, size_t n, off_t o) {
    while (n) {
        const ssize_t r = pread(fd, d, n, o);
        if (r <= 0) return false;
        d += r; n -= (size_t)r; o += r;
    }
    return true;
}

}  // namespace

std::string join(const std::string &dir, const std::string &name) { return dir.empty() || dir.back() == '/' ? dir + name : dir + "/" + name; }

std::string postdata_path(const std::string &dir, uint64_t file) { return join(dir, "postdata_" + std::to_string(file) + ".bin"); }

std::string range_record_path(const std::string &dir, uint64_t from_file, uint64_t to_file) {
    return join(dir, "range_" + std::to_string(from_file) + "_" + std::to_string(to_file) + ".rec");
}

std::string sums_path(const std::string &dir, uint64_t file) { return join(dir, "postdata_" + std::to_string(file) + ".sum"); }

PostFile post_file_kind(const std::string &name, bool *tmp) {
    const bool t = ends_with(name, ".tmp");
    if (tmp) *tmp = t;
    const std::string base = t ? name.substr(0, name.size() - 4) : name;
    if (!t && name.size() > 13 && name.rfind("postdata_", 0) == 0 && ends_with(name, ".bin")) return PostFile::kLabels;
    if (base == kMetadataFile) return PostFile::kMetadata;
    if (base == kInitialProofFile) return PostFile::kInitialProof;
    if (base == kInitialScanFile) return PostFile::kInitialScan;
    if (base.size() > 4 && base.rfind("range_", 0) == 0 && ends_with(base, ".rec")) return PostFile::kRangeRecord;
    if (base.size() > 13 && base.rfind("postdata_", 0) == 0 && ends_with(base, ".sum")) return PostFile::kSums;
    return PostFile::kNone;
}

int check_layout(const b200post_post_metadata &md) {
    const unsigned __int128 nl = (unsigned __int128)md.num_units * md.labels_per_unit;
    const uint64_t N = md.scrypt_n;
    if (nl == 0 || nl > (~0ull >> 4) || md.max_file_size < 16 || md.max_file_size % 16 || N < 2 || N > (1ull << 20) || (N & (N - 1)))
        return fail(B200POST_ERR_IO, "corrupt metadata: label count, MaxFileSize or Scrypt.N out of range");
    return B200POST_OK;
}

int io_error(const std::string &what) { return fail(B200POST_ERR_IO, what + ": " + strerror(errno)); }

int make_dirs(const std::string &dir) {
    std::string cur;
    for (size_t i = 0; i <= dir.size(); i++) {
        if (i == dir.size() || dir[i] == '/') {
            if (!cur.empty() && mkdir(cur.c_str(), 0755) != 0 && errno != EEXIST) return io_error("mkdir " + cur);
        }
        if (i < dir.size()) cur += dir[i];
    }
    return B200POST_OK;
}

int write_file_atomic(const std::string &path, const std::string &bytes) {
    const std::string tmp = path + ".tmp";
    FILE *f = fopen(tmp.c_str(), "wb");
    if (!f) return io_error("open " + tmp);
    const bool ok = fwrite(bytes.data(), 1, bytes.size(), f) == bytes.size();
    if (fclose(f) != 0 || !ok) return io_error("write " + tmp);
    if (rename(tmp.c_str(), path.c_str()) != 0) return io_error("rename " + tmp);
    return B200POST_OK;
}

bool read_file(const std::string &path, std::string *bytes) {
    FILE *f = fopen(path.c_str(), "rb");
    if (!f) return false;
    char buf[65536];
    size_t n;
    bytes->clear();
    while ((n = fread(buf, 1, sizeof buf, f)) > 0) bytes->append(buf, n);
    const bool ok = !ferror(f);
    const int err = errno;
    fclose(f);
    errno = err;
    return ok;
}

int check_post_files(const std::string &dir, const Layout &lay, uint64_t from_file, uint64_t last_file) {
    for (uint64_t f = from_file; f <= last_file; f++) {
        struct stat st;
        const std::string p = postdata_path(dir, f);
        const uint64_t want = lay.labels_in(f) * 16;
        if (stat(p.c_str(), &st) != 0) return fail(B200POST_ERR_IO, "POST data is incomplete: " + p + " is missing");
        if ((uint64_t)st.st_size != want)
            return fail(B200POST_ERR_IO, "POST data is incomplete: " + p + " holds " + std::to_string(st.st_size) + " bytes, the metadata implies " +
                                             std::to_string(want));
    }
    return B200POST_OK;
}

bool stored_labels(const std::string &dir, uint64_t per_file, uint64_t from_file, uint64_t last_file, uint64_t *labels) {
    *labels = 0;
    for (uint64_t i = from_file; i <= last_file; i++) {
        struct stat st;
        if (stat(postdata_path(dir, i).c_str(), &st) != 0) break;
        if (st.st_size % 16 || (uint64_t)st.st_size / 16 > per_file) return false;
        *labels += (uint64_t)st.st_size / 16;
        if ((uint64_t)st.st_size / 16 < per_file) break;
    }
    return true;
}

int write_labels(const std::string &dir, uint64_t file, uint64_t in_file, const uint8_t *labels, uint64_t count) {
    const std::string path = postdata_path(dir, file);
    const int fd = open(path.c_str(), O_WRONLY | O_CREAT, 0644);
    if (fd < 0) return io_error("open " + path);
    const size_t bytes = (size_t)count * 16;
    size_t done = 0;
    bool ok = lseek(fd, (off_t)(in_file * 16), SEEK_SET) >= 0;
    while (ok && done < bytes) {
        const ssize_t w = write(fd, labels + done, bytes - done);
        if (w <= 0) ok = false; else done += (size_t)w;
    }
    if (!ok) { const int rc = io_error("write " + path); close(fd); return rc; }
    if (close(fd) != 0) return io_error("write " + path);
    return B200POST_OK;
}

bool parallel_pread(int fd, uint8_t *dst, size_t bytes, off_t off) {
    const size_t kMinSlice = (size_t)4 << 20;
    const unsigned hw = std::max(1u, std::thread::hardware_concurrency());
    const size_t nt = std::min<size_t>({(size_t)8, (size_t)hw, std::max<size_t>(1, bytes / kMinSlice)});
    if (nt <= 1) return pread_all(fd, dst, bytes, off);
    std::vector<std::thread> th;
    std::vector<char> ok(nt, 0);
    const size_t per = (bytes / nt + 15) & ~(size_t)15;
    for (size_t t = 0; t < nt; t++) {
        const size_t lo = std::min(bytes, t * per), hi = t + 1 == nt ? bytes : std::min(bytes, (t + 1) * per);
        th.emplace_back([&, t, lo, hi] { ok[t] = pread_all(fd, dst + lo, hi - lo, off + (off_t)lo); });
    }
    for (auto &x : th) x.join();
    for (char c : ok) if (!c) return false;
    return true;
}

PostDataReader::~PostDataReader() { if (fd_ >= 0) close(fd_); }

int PostDataReader::open_file(uint64_t file) {
    if (file == open_) return B200POST_OK;
    if (fd_ >= 0) close(fd_);
    open_ = ~0ull;
    const std::string path = postdata_path(dir_, file);
    fd_ = open(path.c_str(), O_RDONLY);
    if (fd_ < 0) return io_error("open " + path);
    open_ = file;
    return B200POST_OK;
}

int PostDataReader::read(uint64_t pos, uint64_t n, uint8_t *dst) {
    for (uint64_t done = 0; done < n;) {
        const uint64_t file = (pos + done) / per_file_, in_file = (pos + done) % per_file_;
        if (int rc = open_file(file)) return rc;
        const uint64_t take = std::min<uint64_t>(n - done, per_file_ - in_file);
        // one thread reading into pinned memory was the proving scan's bound (6.7-7.5 GB/s): split it
        if (!parallel_pread(fd_, dst + done * 16, (size_t)take * 16, (off_t)(in_file * 16))) return fail(B200POST_ERR_IO, kShortRead);
        done += take;
    }
    return B200POST_OK;
}

int PostDataReader::read_in_file(uint64_t file, uint64_t in_file, uint64_t n, uint8_t *dst) {
    if (int rc = open_file(file)) return rc;
    return pread_all(fd_, dst, (size_t)n * 16, (off_t)(in_file * 16)) ? B200POST_OK : fail(B200POST_ERR_IO, kShortRead);
}

int save_post_metadata(const std::string &dir, const b200post_post_metadata &m) {
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
    return write_file_atomic(join(dir, kMetadataFile), j);
}

int load_post_metadata(const std::string &dir, b200post_post_metadata *m, bool *missing) {
    if (missing) *missing = false;
    const std::string p = join(dir, kMetadataFile);
    std::string doc;
    if (!read_file(p, &doc)) {
        if (errno == ENOENT) { if (missing) *missing = true; return fail(B200POST_ERR_IO, "metadata file is missing"); }
        return io_error("open " + p);
    }
    memset(m, 0, sizeof *m);
    std::string s;
    uint64_t v;
    if (!json_raw(doc, "NodeId", &s) || !unb64(s, m->node_id, 32) || !json_raw(doc, "CommitmentAtxId", &s) ||
        !unb64(s, m->commitment_atx_id, 32))
        return fail(B200POST_ERR_IO, "corrupt metadata: ids");
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

// "Windows" (the nonce windows the session scanned) is written only above 1, so a one-window file is what it was before
// windows.
int save_initial_proof_file(const std::string &dir, const b200post_proof_metadata &pm, const b200post_post_config &cfg, uint32_t nonces,
                            uint32_t windows, const b200post_proof_out &p) {
    std::string j = "{\n";
    j += " \"NodeId\": \"" + b64(pm.node_id, 32) + "\",\n";
    j += " \"CommitmentAtxId\": \"" + b64(pm.commitment_atx_id, 32) + "\",\n";
    j += " \"NumUnits\": " + std::to_string(pm.num_units) + ",\n";
    j += " \"LabelsPerUnit\": " + std::to_string(pm.labels_per_unit) + ",\n";
    j += " \"K1\": " + std::to_string(cfg.k1) + ",\n";
    j += " \"K2\": " + std::to_string(cfg.k2) + ",\n";
    j += " \"Nonces\": " + std::to_string(nonces) + ",\n";
    if (windows > 1) j += " \"Windows\": " + std::to_string(windows) + ",\n";
    j += " \"PowDifficulty\": \"" + hex(cfg.pow_difficulty, 32) + "\",\n";
    j += " \"Challenge\": \"" + b64(pm.challenge, 32) + "\",\n";
    j += " \"Nonce\": " + std::to_string(p.nonce) + ",\n";
    j += " \"Indices\": \"" + b64(p.indices, p.indices_len) + "\",\n";
    j += " \"Pow\": " + std::to_string(p.pow) + "\n}\n";
    return write_file_atomic(join(dir, kInitialProofFile), j);
}

int load_initial_proof_file(const std::string &dir, const b200post_post_metadata &md, const b200post_post_config &cfg, uint32_t nonces,
                            b200post_proof_out *out, b200post_proof_metadata *pm) {
    std::string doc;
    if (!read_file(join(dir, kInitialProofFile), &doc)) return no_initial_proof(std::string(kInitialProofFile) + " is absent");
    const uint64_t num_labels = (uint64_t)md.num_units * md.labels_per_unit;
    const size_t packed = num_labels ? ((size_t)cfg.k2 * b200post_bits_per_index(num_labels) + 7) / 8 : 0;
    b200post_proof_metadata m{};
    b200post_proof_out p{};
    uint8_t diff[32];
    std::string s;
    uint64_t units, lpu, k1, k2, nn, nonce, pow;
    if (!json_raw(doc, "NodeId", &s) || !unb64(s, m.node_id, 32) || !json_raw(doc, "CommitmentAtxId", &s) ||
        !unb64(s, m.commitment_atx_id, 32) || !json_raw(doc, "Challenge", &s) || !unb64(s, m.challenge, 32) ||
        !json_raw(doc, "PowDifficulty", &s) || !unhex(s, diff, 32) || !json_u64(doc, "NumUnits", &units) ||
        !json_u64(doc, "LabelsPerUnit", &lpu) || !json_u64(doc, "K1", &k1) || !json_u64(doc, "K2", &k2) ||
        !json_u64(doc, "Nonces", &nn) || !json_u64(doc, "Nonce", &nonce) || !json_u64(doc, "Pow", &pow) ||
        packed == 0 || packed > sizeof p.indices || !json_raw(doc, "Indices", &s) || !unb64(s, p.indices, packed))
        return no_initial_proof(std::string(kInitialProofFile) + " is unreadable");
    if (memcmp(m.node_id, md.node_id, 32) || memcmp(m.commitment_atx_id, md.commitment_atx_id, 32)) return no_initial_proof("it belongs to another identity");
    if (units != md.num_units || lpu != md.labels_per_unit || lpu != cfg.labels_per_unit) return no_initial_proof("it was made for another POST size");
    if (k1 != cfg.k1 || k2 != cfg.k2 || memcmp(diff, cfg.pow_difficulty, 32)) return no_initial_proof("it was made under another K1, K2 or pow difficulty");
    if (nn != nonces) return no_initial_proof("it was made for another nonce count");
    // a session that scanned several nonce windows may have proved with a nonce of any of them
    uint64_t windows = 1;
    if (doc.find("\"Windows\"") != std::string::npos && (!json_u64(doc, "Windows", &windows) || windows < 2 || windows > 4096 / nonces))
        return no_initial_proof(std::string(kInitialProofFile) + " is unreadable");
    if (memcmp(m.challenge, kZeroChallenge, 32) || nonce >= nonces * windows) return no_initial_proof("it does not answer the zero challenge");
    m.num_units = md.num_units; m.labels_per_unit = md.labels_per_unit;
    p.nonce = (uint32_t)nonce; p.pow = pow; p.indices_len = packed; p.labels_scanned = num_labels;
    *out = p;
    if (pm) *pm = m;
    return B200POST_OK;
}

// ---- postdata_<N>.sum: "B2PSUMS1" | version u32 | block labels u32 | NodeId | CommitmentAtxId | Scrypt.N u64 |
// labels per file u64 | file u64 | covered u64 | digests | FNV-1a 64 of everything before it (little endian)
namespace {

const char kSumsMagic[] = "B2PSUMS1";
const uint32_t kSumsVersion = 1;
const size_t kSumsHeader = 8 + 4 + 4 + 32 + 32 + 8 * 4;

uint64_t fnv1a64(const char *p, size_t n) {
    uint64_t h = 0xcbf29ce484222325ull;
    for (size_t i = 0; i < n; i++) { h ^= (unsigned char)p[i]; h *= 0x100000001b3ull; }
    return h;
}
template <class T> void put(std::string *s, T v) { s->append(reinterpret_cast<const char *>(&v), sizeof v); }
template <class T> T at(const std::string &s, size_t off) { T v; memcpy(&v, s.data() + off, sizeof v); return v; }

}  // namespace

PostSums PostSums::of(const b200post_post_metadata &md, uint64_t file) {
    PostSums s;
    memcpy(s.node_id, md.node_id, 32);
    memcpy(s.commitment_atx_id, md.commitment_atx_id, 32);
    s.scrypt_n = md.scrypt_n; s.labels_per_file = md.max_file_size / 16; s.file = file;
    return s;
}

int save_post_sums(const std::string &dir, const PostSums &s) {
    if (s.digests.size() != s.blocks() * 32) return fail(B200POST_ERR_INVALID_ARGUMENT, "sidecar: digest count does not match its coverage");
    std::string b(kSumsMagic, 8);
    put<uint32_t>(&b, kSumsVersion);
    put<uint32_t>(&b, (uint32_t)kSumBlockLabels);
    b.append(reinterpret_cast<const char *>(s.node_id), 32);
    b.append(reinterpret_cast<const char *>(s.commitment_atx_id), 32);
    put<uint64_t>(&b, s.scrypt_n);
    put<uint64_t>(&b, s.labels_per_file);
    put<uint64_t>(&b, s.file);
    put<uint64_t>(&b, s.covered);
    b += s.digests;
    put<uint64_t>(&b, fnv1a64(b.data(), b.size()));
    return write_file_atomic(sums_path(dir, s.file), b);
}

bool load_post_sums(const std::string &dir, const b200post_post_metadata &md, uint64_t file, uint64_t max_labels, PostSums *out) {
    std::string b;
    if (!read_file(sums_path(dir, file), &b) || b.size() < kSumsHeader + 8) return false;
    if (fnv1a64(b.data(), b.size() - 8) != at<uint64_t>(b, b.size() - 8)) return false;
    PostSums s = PostSums::of(md, file);
    if (b.compare(0, 8, kSumsMagic, 8) != 0 || at<uint32_t>(b, 8) != kSumsVersion || at<uint32_t>(b, 12) != kSumBlockLabels) return false;
    if (memcmp(b.data() + 16, s.node_id, 32) || memcmp(b.data() + 48, s.commitment_atx_id, 32)) return false;
    if (at<uint64_t>(b, 80) != s.scrypt_n || at<uint64_t>(b, 88) != s.labels_per_file || at<uint64_t>(b, 96) != file) return false;
    s.covered = at<uint64_t>(b, 104);
    if (s.covered > max_labels || s.covered > s.labels_per_file || b.size() != kSumsHeader + s.blocks() * 32 + 8) return false;
    s.digests = b.substr(kSumsHeader, s.blocks() * 32);
    *out = std::move(s);
    return true;
}

}  // namespace b200post
