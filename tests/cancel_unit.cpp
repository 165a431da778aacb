// cancel_unit.cpp -- CPU unit test of the cancel checkpoints in csrc/vmig_tree.cpp and csrc/vmig_table.cpp (compiled and
// run by tests/test_cancel_host.py): the chunked base copy of a snapshot stops at a chunk boundary once the latch is set,
// the walk, prune and metadata replay start no step after it, and a table is never renamed into place after it.
//   usage: cancel_unit DIR
#include "vmig_tree.h"
#include "vmig_table.h"
#include "vmig_common.h"
#include <fcntl.h>
#include <unistd.h>
#include <sys/stat.h>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <thread>
#include <vector>

namespace vmig {   // the error-channel functions normally provided by vmig_engine.cu
static thread_local std::string g_err;
void set_last_error(const char* fmt, ...) { char b[1024]; va_list ap; va_start(ap, fmt); vsnprintf(b, sizeof b, fmt, ap); va_end(ap); g_err = b; }
void set_last_error_str(const std::string& s) { g_err = s; }
const char* last_error_cstr() { return g_err.c_str(); }
long env_long(const char* name, long d) { const char* v = getenv(name); return v && *v ? atol(v) : d; }
}
using namespace vmig;

#define CHECK(c) do { if (!(c)) { printf("FAIL line %d: %s   [last error: %s]\n", __LINE__, #c, last_error_cstr()); return 1; } } while (0)

static uint64_t fsize(int fd) { struct stat st; return fstat(fd, &st) == 0 ? (uint64_t)st.st_size : 0; }

// Copy `chunks` chunks of a patterned file; a helper thread, already spinning before the copy starts, sets the latch as
// soon as the output holds any byte.  The copy must stop at the next chunk boundary: ECANCELED, a whole number of
// chunks copied, fewer than all, each one byte for byte.
static int chunk_stop(const std::string& dir, bool rw_only) {
    const uint64_t chunks = 6, size = chunks * kCopyChunk;
    const std::string in = dir + "/in.bin", out = dir + "/out" + std::to_string(rw_only) + ".bin";
    {
        const int fd = open(in.c_str(), O_WRONLY | O_CREAT | O_TRUNC, 0600);
        CHECK(fd >= 0);
        std::vector<uint64_t> piece((1u << 20) / 8);
        for (uint64_t off = 0; off < size; off += 1u << 20) {
            for (size_t i = 0; i < piece.size(); i++) piece[i] = (off / 8 + i) * 0x9E3779B97F4A7C15ull;
            CHECK(pwrite(fd, piece.data(), 1u << 20, (off_t)off) == (ssize_t)(1u << 20));
        }
        close(fd);
    }
    const int ifd = open(in.c_str(), O_RDONLY), ofd = open(out.c_str(), O_RDWR | O_CREAT | O_TRUNC, 0600);
    CHECK(ifd >= 0 && ofd >= 0);
    std::atomic<int> latch{0};
    std::atomic<bool> done{false}, spinning{false};
    std::thread setter([&] {
        spinning.store(true);
        while (!done.load() && fsize(ofd) == 0) {}
        latch.store(VMIG_ECANCELED);
    });
    while (!spinning.load()) std::this_thread::yield();
    const int rc = copy_range(ifd, ofd, 0, size, false, rw_only, in, &latch);
    done.store(true); setter.join();
    const uint64_t got = fsize(ofd);
    printf("chunk stop (%s): rc=%d, %llu of %llu bytes copied\n", rw_only ? "pread/pwrite" : "copy_file_range", rc,
           (unsigned long long)got, (unsigned long long)size);
    CHECK(rc == VMIG_ECANCELED);
    CHECK(got % kCopyChunk == 0 && got >= kCopyChunk && got < size);
    std::vector<uint8_t> a(1u << 20), b(1u << 20);
    for (uint64_t off = 0; off < got; off += 1u << 20) {
        CHECK(pread(ifd, a.data(), a.size(), (off_t)off) == (ssize_t)a.size() && pread(ofd, b.data(), b.size(), (off_t)off) == (ssize_t)b.size());
        CHECK(a == b);
    }
    close(ifd); close(ofd);
    unlink(in.c_str()); unlink(out.c_str());
    return 0;
}

int main(int argc, char** argv) {
    if (argc < 2) return 2;
    const std::string dir = argv[1];
    std::atomic<int> set{VMIG_ECANCELED};

    // a latch set before the copy: nothing is copied
    {
        const std::string in = dir + "/small.bin", out = dir + "/small_out.bin";
        const int fd = open(in.c_str(), O_WRONLY | O_CREAT | O_TRUNC, 0600);
        CHECK(fd >= 0 && ftruncate(fd, 1 << 20) == 0);
        close(fd);
        const int ifd = open(in.c_str(), O_RDONLY), ofd = open(out.c_str(), O_WRONLY | O_CREAT | O_TRUNC, 0600);
        CHECK(copy_range(ifd, ofd, 0, 1 << 20, false, false, in, &set) == VMIG_ECANCELED && fsize(ofd) == 0);
        CHECK(copy_range(ifd, ofd, 0, 1 << 20, false, true, in, &set) == VMIG_ECANCELED && fsize(ofd) == 0);
        close(ifd); close(ofd);
    }
    if (chunk_stop(dir, false) || chunk_stop(dir, true)) return 1;

    // walk, prune and metadata replay start nothing once the latch is set
    const std::string tree = dir + "/tree", dst = dir + "/dst";
    CHECK(mkdir(tree.c_str(), 0755) == 0 && mkdir((tree + "/d").c_str(), 0755) == 0 && mkdir(dst.c_str(), 0755) == 0);
    CHECK(symlink("target", (tree + "/lnk").c_str()) == 0);
    CHECK(mkdir((dst + "/extra").c_str(), 0755) == 0);
    Manifest m;
    CHECK(walk_tree(tree, 4096, false, &m, &set) == VMIG_ECANCELED);
    CHECK(walk_tree(tree, 4096, false, &m) == VMIG_OK && m.symlinks.size() == 1);
    uint64_t n = 0;
    CHECK(prune_extras(dst, m, false, &n, &set) == VMIG_ECANCELED && n == 0);
    struct stat st;
    CHECK(lstat((dst + "/extra").c_str(), &st) == 0);
    CHECK(make_dirs(dst, m) == VMIG_OK);
    CHECK(replay_metadata(dst, m, default_meta_policy(0), nullptr, nullptr, nullptr, &set) == VMIG_ECANCELED);
    CHECK(lstat((dst + "/lnk").c_str(), &st) != 0);

    // a table is not written, and leaves no .tmp, once the latch is set
    BlockTable t; t.block_bytes = 4096; t.algo = 1;
    const std::string tp = dir + "/t.vmig";
    CHECK(table_store(tp, t, &set) == VMIG_ECANCELED && access(tp.c_str(), F_OK) != 0);
    CHECK(table_store(tp, t) == VMIG_OK && access(tp.c_str(), F_OK) == 0);
    printf("cancel unit ok\n");
    return 0;
}
