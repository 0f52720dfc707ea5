// postdata_io.h — reading stored labels back from postdata_N.bin files (shared by the prover and the POS check).
#pragma once
#include <sys/types.h>

#include <cstdint>
#include <string>

namespace b200post {

// pread of [off, off + bytes) into dst on up to 8 threads (pread is position-independent, so slices are independent)
bool parallel_pread(int fd, uint8_t *dst, size_t bytes, off_t off);

std::string postdata_path(const std::string &dir, uint64_t file);

// Labels of one POST by global label index, over files of `labels_per_file` labels; keeps the last file open.
// Errors return B200POST_ERR_IO with the text in b200post_last_error().
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

}  // namespace b200post
