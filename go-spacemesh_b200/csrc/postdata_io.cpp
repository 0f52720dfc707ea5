// postdata_io.cpp — see postdata_io.h.
#include "postdata_io.h"

#include <errno.h>
#include <fcntl.h>
#include <unistd.h>

#include <algorithm>
#include <cstring>
#include <thread>
#include <vector>

#include "../../include/b200post_setup.h"
#include "engine.h"

namespace b200post {

bool parallel_pread(int fd, uint8_t *dst, size_t bytes, off_t off) {
    auto read_all = [fd](uint8_t *d, size_t n, off_t o) {
        while (n) {
            const ssize_t r = pread(fd, d, n, o);
            if (r <= 0) return false;
            d += r; n -= (size_t)r; o += r;
        }
        return true;
    };
    const size_t kMinSlice = (size_t)4 << 20;
    const unsigned hw = std::max(1u, std::thread::hardware_concurrency());
    const size_t nt = std::min<size_t>({(size_t)8, (size_t)hw, std::max<size_t>(1, bytes / kMinSlice)});
    if (nt <= 1) return read_all(dst, bytes, off);
    std::vector<std::thread> th;
    std::vector<char> ok(nt, 0);
    const size_t per = (bytes / nt + 15) & ~(size_t)15;
    for (size_t t = 0; t < nt; t++) {
        const size_t lo = std::min(bytes, t * per), hi = t + 1 == nt ? bytes : std::min(bytes, (t + 1) * per);
        th.emplace_back([&, t, lo, hi] { ok[t] = read_all(dst + lo, hi - lo, off + (off_t)lo); });
    }
    for (auto &x : th) x.join();
    for (char c : ok) if (!c) return false;
    return true;
}

std::string postdata_path(const std::string &dir, uint64_t file) {
    return dir + "/postdata_" + std::to_string(file) + ".bin";
}

PostDataReader::~PostDataReader() { if (fd_ >= 0) close(fd_); }

int PostDataReader::open_file(uint64_t file) {
    if (file == open_) return B200POST_OK;
    if (fd_ >= 0) close(fd_);
    open_ = ~0ull;
    const std::string path = postdata_path(dir_, file);
    fd_ = open(path.c_str(), O_RDONLY);
    if (fd_ < 0) { set_error("open " + path + ": " + strerror(errno)); return B200POST_ERR_IO; }
    open_ = file;
    return B200POST_OK;
}

int PostDataReader::read(uint64_t pos, uint64_t n, uint8_t *dst) {
    for (uint64_t done = 0; done < n;) {
        const uint64_t file = (pos + done) / per_file_, in_file = (pos + done) % per_file_;
        if (int rc = open_file(file)) return rc;
        const uint64_t take = std::min<uint64_t>(n - done, per_file_ - in_file);
        // one thread reading into pinned memory was the proving scan's bound (6.7-7.5 GB/s): split it
        if (!parallel_pread(fd_, dst + done * 16, (size_t)take * 16, (off_t)(in_file * 16))) {
            set_error("POST data is incomplete (short read): initialisation not finished?");
            return B200POST_ERR_IO;
        }
        done += take;
    }
    return B200POST_OK;
}

int PostDataReader::read_in_file(uint64_t file, uint64_t in_file, uint64_t n, uint8_t *dst) {
    if (int rc = open_file(file)) return rc;
    size_t left = (size_t)n * 16;
    off_t o = (off_t)(in_file * 16);
    while (left) {
        const ssize_t r = pread(fd_, dst, left, o);
        if (r <= 0) { set_error("POST data is incomplete (short read): initialisation not finished?"); return B200POST_ERR_IO; }
        dst += r; left -= (size_t)r; o += r;
    }
    return B200POST_OK;
}

}  // namespace b200post
