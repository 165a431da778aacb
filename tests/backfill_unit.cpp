// backfill_unit.cpp -- CPU unit test of copy_range() in csrc/vmig_tree.cpp, the copy that gives a snapshot file the
// blocks it shares with the base snapshot's file (compiled and run by tests/test_snapshot_host.py).  Both the
// copy_file_range path and the pread/pwrite fallback must put exactly [off, off + len) of the input at the same offsets
// of the output and nothing else; an O_DIRECT output takes whole sectors (the caller truncates); an input that ends
// early is VMIG_ESRCCHANGED.
//   usage: backfill_unit DIR [DIR2 ...]   (each DIR is tried; O_DIRECT runs where the filesystem allows it)
#include "vmig_tree.h"
#include "vmig_common.h"
#include <fcntl.h>
#include <unistd.h>
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

int main(int argc, char** argv) {
    if (argc < 2) return 2;
    for (int i = 1; i < argc; i++) if (run(argv[i])) return 1;
    printf("backfill unit ok\n");
    return 0;
}
