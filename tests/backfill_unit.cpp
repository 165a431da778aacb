// backfill_unit.cpp -- CPU unit test of copy_range() in csrc/vmig_tree.cpp, the copy that gives a snapshot file the
// blocks it shares with the base snapshot's file (compiled and run by tests/test_snapshot_host.py).  Both the
// copy_file_range path and the pread/pwrite fallback must put exactly [off, off + len) of the input at the same offsets
// of the output and nothing else; an O_DIRECT output takes whole sectors (the caller truncates); an input that ends
// early is VMIG_ESRCCHANGED.
//   usage: backfill_unit DIR [DIR2 ...]   (each DIR is tried; O_DIRECT runs where the filesystem allows it)
//          backfill_unit --large DIR      (a sparse file of 2^32 + 9 MiB + 777 bytes: one run longer than 2^32 bytes and offsets
//                                          above 2^32, through both paths; DIR needs about 5 GiB, best on tmpfs)
#include "vmig_tree.h"
#include "vmig_common.h"
#include <fcntl.h>
#include <unistd.h>
#include <sys/stat.h>
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <string>
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

static std::vector<uint8_t> pattern(size_t n, uint32_t seed) {
    std::vector<uint8_t> v(n);
    uint32_t x = seed;
    for (auto& b : v) { x = x * 1664525u + 1013904223u; b = (uint8_t)(x >> 24); }
    return v;
}
static bool put(const std::string& p, const std::vector<uint8_t>& v) {
    FILE* f = fopen(p.c_str(), "wb"); if (!f) return false;
    const bool ok = fwrite(v.data(), 1, v.size(), f) == v.size(); return fclose(f) == 0 && ok;
}
static std::vector<uint8_t> get(const std::string& p) {
    std::vector<uint8_t> v; FILE* f = fopen(p.c_str(), "rb"); if (!f) return v;
    uint8_t b[65536]; size_t n; while ((n = fread(b, 1, sizeof b, f)) > 0) v.insert(v.end(), b, b + n);
    fclose(f); return v;
}

static int run(const std::string& dir) {
    const size_t size = (3u << 20) + 123;                  // not a whole number of sectors
    const std::vector<uint8_t> base = pattern(size, 1), old = pattern(size, 2);
    const std::string in = dir + "/base.bin";
    CHECK(put(in, base));
    for (int rw_only = 0; rw_only < 2; rw_only++) {
        // the middle of the file (a run of unchanged blocks) and its tail (the short last block)
        const std::string out = dir + "/out" + std::to_string(rw_only) + ".bin";
        CHECK(put(out, old));
        const int ifd = open(in.c_str(), O_RDONLY), ofd = open(out.c_str(), O_WRONLY);
        CHECK(ifd >= 0 && ofd >= 0);
        CHECK(copy_range(ifd, ofd, 1u << 20, 1u << 20, false, rw_only != 0, in) == VMIG_OK);
        CHECK(copy_range(ifd, ofd, 3u << 20, 123, false, rw_only != 0, in) == VMIG_OK);
        CHECK(copy_range(ifd, ofd, 3u << 20, 200, false, rw_only != 0, in) == VMIG_ESRCCHANGED);   // the base is shorter
        close(ifd); close(ofd);
        std::vector<uint8_t> want = old;
        std::copy(base.begin() + (1u << 20), base.begin() + (2u << 20), want.begin() + (1u << 20));
        std::copy(base.begin() + (3u << 20), base.end(), want.begin() + (3u << 20));
        CHECK(get(out) == want);
    }
    // O_DIRECT destination, as a snapshot file written with VMIG_F_DIRECT_IO: sector-aligned buffer and lengths
    const std::string dout = dir + "/direct.bin";
    const int dfd = open(dout.c_str(), O_WRONLY | O_CREAT | O_TRUNC | O_DIRECT, 0600);
    if (dfd < 0) { printf("direct: refused by %s\n", dir.c_str()); return 0; }
    const int ifd = open(in.c_str(), O_RDONLY);
    CHECK(ifd >= 0);
    CHECK(copy_range(ifd, dfd, 0, 2u << 20, true, false, in) == VMIG_OK);
    CHECK(copy_range(ifd, dfd, 2u << 20, size - (2u << 20), true, false, in) == VMIG_OK);
    CHECK(ftruncate(dfd, (off_t)size) == 0);
    close(ifd); close(dfd);
    CHECK(get(dout) == base);
    printf("direct: ok in %s\n", dir.c_str());
    return 0;
}

// ---------------------------------------------------------------------------------------------- past 4 GiB
static const uint64_t kBig = (1ull << 32) + (9ull << 20) + 777, k4G = 1ull << 32, kMiB = 1ull << 20;

// Island bytes name their own offset and file, so bytes that landed in the wrong place cannot pass for the right ones
static void island(std::vector<uint8_t>* v, uint64_t off, uint64_t salt) {
    for (size_t i = 0; i < v->size(); i++) {
        const uint64_t o = off + i, w = (o / 8 + salt) * 0x9E3779B97F4A7C15ull;
        (*v)[i] = (uint8_t)(w >> (8 * (o % 8))) ^ (uint8_t)(w >> 56);
    }
}
static bool put_at(int fd, uint64_t off, const std::vector<uint8_t>& v) {
    size_t put = 0;
    while (put < v.size()) { const ssize_t w = pwrite(fd, v.data() + put, v.size() - put, (off_t)(off + put)); if (w <= 0) return false; put += (size_t)w; }
    return true;
}
static bool get_at(int fd, uint64_t off, std::vector<uint8_t>* v) {
    size_t got = 0;
    while (got < v->size()) { const ssize_t r = pread(fd, v->data() + got, v->size() - got, (off_t)(off + got)); if (r <= 0) return false; got += (size_t)r; }
    return true;
}
// [a, b) of the two files are equal
static bool same_range(int fa, int fb, uint64_t a, uint64_t b) {
    std::vector<uint8_t> x(4 * kMiB), y(4 * kMiB);
    for (uint64_t o = a; o < b; o += x.size()) {
        const size_t n = (size_t)std::min<uint64_t>(x.size(), b - o);
        x.resize(n); y.resize(n);
        if (!get_at(fa, o, &x) || !get_at(fb, o, &y) || x != y) { printf("differs in [%llu, %llu)\n", (unsigned long long)o, (unsigned long long)(o + n)); return false; }
    }
    return true;
}

static int run_large(const std::string& dir) {
    // the input: holes, and islands in the first blocks, either side of 2^32, at 3 GiB and over the tail
    const std::string in = dir + "/big_in.bin";
    const int ifd = open(in.c_str(), O_RDWR | O_CREAT | O_TRUNC, 0600);
    CHECK(ifd >= 0 && ftruncate(ifd, (off_t)kBig) == 0);
    const uint64_t at[][2] = {{0, 6 * kMiB}, {k4G - 5 * kMiB, 10 * kMiB}, {3ull << 30, 2 * kMiB + 4096}, {kBig - 2 * kMiB - 777, 2 * kMiB + 777}};
    for (const auto& a : at) { std::vector<uint8_t> v(a[1]); island(&v, a[0], 1); CHECK(put_at(ifd, a[0], v)); }
    const uint64_t r0 = 4 * kMiB, r1 = kBig - 4096 - 777;               // the long run: [4 MiB, the file's last 4873 bytes)
    CHECK(r1 - r0 > k4G);
    for (int rw_only = 0; rw_only < 2; rw_only++) {
        const std::string out = dir + "/big_out" + std::to_string(rw_only) + ".bin";
        const int ofd = open(out.c_str(), O_RDWR | O_CREAT | O_TRUNC, 0600);
        CHECK(ofd >= 0 && ftruncate(ofd, (off_t)kBig) == 0);
        // what the output holds outside the run, and must keep
        std::vector<uint8_t> head(r0), tail(kBig - r1);
        island(&head, 0, 2); island(&tail, r1, 2);
        CHECK(put_at(ofd, 0, head) && put_at(ofd, r1, tail));
        CHECK(copy_range(ifd, ofd, r0, r1 - r0, false, rw_only != 0, in) == VMIG_OK);
        struct stat so;
        CHECK(fstat(ofd, &so) == 0 && (uint64_t)so.st_size == kBig);
        std::vector<uint8_t> h2(head.size()), t2(tail.size());
        CHECK(get_at(ofd, 0, &h2) && h2 == head && get_at(ofd, r1, &t2) && t2 == tail);
        CHECK(same_range(ifd, ofd, r0, r1));
        // separate offsets, both above 2^32: input [2^32 + 1 MiB, +2 MiB + 5) to output [2^32 + 5 MiB + 4096, ...)
        const uint64_t so_off = k4G + kMiB, do_off = k4G + 5 * kMiB + 4096, n = 2 * kMiB + 5;
        CHECK(copy_range_at(ifd, so_off, ofd, do_off, n, false, rw_only != 0, in) == VMIG_OK);
        std::vector<uint8_t> want(n), got(n);
        island(&want, so_off, 1);
        CHECK(get_at(ofd, do_off, &got) && got == want);
        CHECK(same_range(ifd, ofd, k4G - 5 * kMiB, do_off) && same_range(ifd, ofd, do_off + n, r1));      // and nothing around it
        CHECK(get_at(ofd, 0, &h2) && h2 == head);
        // a range that ends past the input's end, above 2^32
        CHECK(copy_range(ifd, ofd, kBig - 100, 200, false, rw_only != 0, in) == VMIG_ESRCCHANGED);
        CHECK(fstat(ofd, &so) == 0 && (uint64_t)so.st_size == kBig);
        close(ofd);
        CHECK(unlink(out.c_str()) == 0);
    }
    close(ifd);
    CHECK(unlink(in.c_str()) == 0);
    printf("backfill large ok\n");
    return 0;
}

int main(int argc, char** argv) {
    if (argc < 2) return 2;
    if (std::string(argv[1]) == "--large") return argc == 3 ? run_large(argv[2]) : 2;
    for (int i = 1; i < argc; i++) if (run(argv[i])) return 1;
    printf("backfill unit ok\n");
    return 0;
}
