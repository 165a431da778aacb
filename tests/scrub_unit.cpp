// scrub_unit.cpp -- CPU unit test of the host side of vmig_scrub_store (csrc/vmig_scrub.cpp; compiled and run by
// tests/test_scrub_host.py):
//   - the table merge lists every missing, extra and resized path, not only the first;
//   - the inode grouping maps the paths of one inode, in any version, to one block range;
//   - report path escaping round-trips awkward names, and the report is sorted and written atomically;
//   - a reader fed a descriptor whose reads fail records the inode as unreadable and returns success to the pipeline;
//     an inode replaced since the walk is VMIG_ESRCCHANGED;
//   - the reader takes blocks either side of offset 2^32 of a sparse file longer than that, and its short last block.
//   usage: scrub_unit DIR
#include "vmig_scrub.h"
#include "vmig_common.h"
#include <fcntl.h>
#include <unistd.h>
#include <sys/stat.h>
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

static Entry file(const std::string& rel, uint64_t size, uint64_t ino, uint32_t bb) {
    Entry e; e.rel = rel; e.type = kFile; e.size = size; e.n_blocks = (size + bb - 1) / bb; e.dev = 7; e.ino = ino;
    return e;
}
static void finish(Manifest* m) {
    uint64_t fb = 0;
    for (auto& e : m->files) { e.first_block = fb; fb += e.n_blocks; m->bytes_total += e.size; }
    m->n_blocks = fb;
}
static void add(BlockTable* t, const std::string& rel, uint64_t size) {
    const uint64_t fb = t->hashes.size();
    t->files.push_back({rel, size, fb, 0, 0});
    for (uint64_t r = 0; r < t->blocks_of(t->files.back()); r++) t->hashes.push_back(0);
}

static int merge_and_group() {
    const uint32_t bb = 4096;
    Manifest a, b;
    a.files = {file("a", 5000, 10, bb), file("b", 10, 11, bb), file("c", 100, 12, bb), file("x", 1, 13, bb), file("z", 8192, 14, bb)};
    finish(&a);
    BlockTable ta; ta.block_bytes = bb;
    add(&ta, "a", 5000); add(&ta, "b", 20); add(&ta, "m", 3); add(&ta, "n", 4); add(&ta, "z", 8192);
    std::vector<ScrubFinding> f;
    std::vector<int64_t> ta_of;
    CHECK(scrub_merge_table(0, a, ta, &ta_of, &f) == 5);
    CHECK(f[0].kind == kScrubResized && f[0].path == "b");
    CHECK(f[1].kind == kScrubExtra && f[1].path == "c");
    CHECK(f[2].kind == kScrubMissing && f[2].path == "m");
    CHECK(f[3].kind == kScrubMissing && f[3].path == "n");
    CHECK(f[4].kind == kScrubExtra && f[4].path == "x");
    CHECK((ta_of == std::vector<int64_t>{0, -1, -1, -1, 4}));
    // version 1 holds inode 10 under another name and inode 14 under two names (a hard link inside the version)
    b.files = {file("empty", 0, 15, bb), file("moved", 5000, 10, bb), file("z", 8192, 14, bb), file("z2", 8192, 14, bb)};
    finish(&b);
    BlockTable tb; tb.block_bytes = bb;
    add(&tb, "empty", 0); add(&tb, "moved", 5000); add(&tb, "z", 8192); add(&tb, "z2", 8192);
    std::vector<int64_t> tb_of;
    f.clear();
    CHECK(scrub_merge_table(1, b, tb, &tb_of, &f) == 0);
    std::vector<ScrubInode> inodes;
    std::vector<std::vector<uint32_t>> inode_of;
    CHECK(scrub_group_inodes({&a, nullptr, &b}, {ta_of, {}, tb_of}, bb, &inodes, &inode_of) == VMIG_OK);
    CHECK(inodes.size() == 2);                                  // inode 10 and inode 14; the empty file reads nothing
    CHECK(inodes[0].ino == 10 && inodes[0].first_block == 0 && inodes[0].n_blocks == 2 && inodes[0].version == 0 && inodes[0].rel == "a");
    CHECK(inodes[1].ino == 14 && inodes[1].first_block == 2 && inodes[1].n_blocks == 2);
    CHECK((inode_of[0] == std::vector<uint32_t>{0, kNoInode, kNoInode, kNoInode, 1}));
    CHECK(inode_of[1].empty());
    CHECK((inode_of[2] == std::vector<uint32_t>{kNoInode, 0, 1, 1}));
    // one inode with two sizes: the store changed between the walks
    b.files[1].size = 4999;
    CHECK(scrub_group_inodes({&a, &b}, {ta_of, tb_of}, bb, &inodes, &inode_of) == VMIG_ESRCCHANGED);
    return 0;
}

static int escaping(const std::string& dir) {
    const std::vector<std::string> names = {"plain", "tab\there", "nl\nthere", "back\\slash", std::string("ctl\x01\x1f", 5),
                                            "\\x41", "utf8-\xc3\xa9", "sp ace", std::string("\x7f\xff", 2)};
    for (const auto& n : names) {
        const std::string e = scrub_escape(n);
        CHECK(e.find('\t') == std::string::npos && e.find('\n') == std::string::npos);
        for (unsigned char c : e) CHECK(c >= 0x20);
        std::string back;
        CHECK(scrub_unescape(e, &back) && back == n);
    }
    CHECK(scrub_escape(std::string("a\x01", 2)) == "a\\x01");
    std::string junk;
    CHECK(!scrub_unescape("bad\\", &junk) && !scrub_unescape("bad\\q", &junk) && !scrub_unescape("bad\\x4", &junk));
    // the report: sorted by version, path, block ("-" first), one line per finding
    std::vector<ScrubFinding> v(4);
    v[0].version = 1; v[0].kind = kScrubBlock; v[0].path = "b"; v[0].block = 3; v[0].has_hashes = true; v[0].got = 0xab; v[0].want = 0xcd;
    v[1].version = 0; v[1].kind = kScrubMissing; v[1].path = "z";
    v[2].version = 1; v[2].kind = kScrubUnreadable; v[2].path = "b";
    v[3].version = 0; v[3].kind = kScrubExtra; v[3].path = "tab\tname";
    scrub_sort(&v);
    const std::string p = dir + "/report.txt";
    CHECK(scrub_report_store(p, v, nullptr) == VMIG_OK);
    FILE* fp = fopen(p.c_str(), "rb");
    CHECK(fp);
    char buf[1024]; const size_t n = fread(buf, 1, sizeof buf, fp); fclose(fp);
    CHECK(std::string(buf, n) == "0\textra\ttab\\tname\t-\t-\t-\n0\tmissing\tz\t-\t-\t-\n1\tunreadable\tb\t-\t-\t-\n"
                                 "1\tblock\tb\t3\t00000000000000ab\t00000000000000cd\n");
    std::atomic<int> cancelled{1};
    const std::string q = dir + "/cancelled.txt";
    CHECK(scrub_report_store(q, v, &cancelled) == VMIG_ECANCELED);
    CHECK(access(q.c_str(), F_OK) != 0);
    return 0;
}

static int reader(const std::string& dir) {
    const std::string root = dir + "/root";
    mkdir(root.c_str(), 0755);
    const std::string good = root + "/good", bad = root + "/bad";
    std::vector<uint8_t> bytes(3 * 4096 + 5, 0x5a);
    for (const auto& p : {good, bad}) {
        FILE* f = fopen(p.c_str(), "wb"); CHECK(f);
        CHECK(fwrite(bytes.data(), 1, bytes.size(), f) == bytes.size()); fclose(f);
    }
    struct stat gs, bs;
    CHECK(stat(good.c_str(), &gs) == 0 && stat(bad.c_str(), &bs) == 0);
    std::vector<ScrubInode> inodes = {
        {(uint64_t)gs.st_dev, (uint64_t)gs.st_ino, bytes.size(), 0, 4, 0, "good"},
        {(uint64_t)bs.st_dev, (uint64_t)bs.st_ino, bytes.size(), 4, 4, 0, "bad"},
        {(uint64_t)gs.st_dev, (uint64_t)gs.st_ino + 999999, bytes.size(), 8, 4, 0, "good"},    // not the walked inode
    };
    const int rfd = open(root.c_str(), O_RDONLY | O_DIRECTORY);
    CHECK(rfd >= 0);
    ScrubReader r;
    r.root_fds = {rfd}; r.inodes = &inodes;
    r.init();
    const int wfd = open(bad.c_str(), O_WRONLY);                // every read of it fails (EBADF)
    CHECK(wfd >= 0);
    r.adopt(1, wfd, false);
    std::vector<uint8_t> slot(4096);
    for (uint32_t blk = 0; blk < 4; blk++) {
        const uint32_t len = blk < 3 ? 4096 : 5;
        CHECK(r.read(0, blk * 4096ull, len, slot.data()) == VMIG_OK);
        CHECK(slot[0] == 0x5a && slot[len - 1] == 0x5a);
        CHECK(r.read(1, blk * 4096ull, len, slot.data()) == VMIG_OK);       // success to the pipeline ...
        CHECK(r.unreadable(1));                                              // ... and the inode recorded as unreadable
    }
    CHECK(!r.unreadable(0));
    CHECK(r.why(1).find("pread bad") == 0);
    CHECK(fcntl(wfd, F_GETFD) == -1);                                        // closed after the inode's last block
    CHECK(r.read(2, 0, 4096, slot.data()) == VMIG_ESRCCHANGED);
    CHECK(!r.unreadable(2));
    r.close_all();
    close(rfd);
    return 0;
}

// A sparse inode of 2^32 + 9 MiB + 777 bytes whose words name their own offsets around 2^32 and in the tail
static int reader_large(const std::string& dir) {
    const uint64_t kBig = (1ull << 32) + (9ull << 20) + 777, k4G = 1ull << 32;
    const uint32_t bb = 4096;
    const std::string root = dir + "/bigroot", path = root + "/huge";
    mkdir(root.c_str(), 0755);
    const int wfd = open(path.c_str(), O_WRONLY | O_CREAT | O_TRUNC, 0600);
    CHECK(wfd >= 0 && ftruncate(wfd, (off_t)kBig) == 0);
    const uint64_t last_off = kBig / bb * bb;
    auto words = [](uint64_t off, size_t n) {
        std::vector<uint8_t> v(n);
        for (size_t i = 0; i < n; i++) { const uint64_t o = off + i, w = (o / 8) * 0x9E3779B97F4A7C15ull + 1; v[i] = (uint8_t)(w >> (8 * (o % 8))); }
        return v;
    };
    const std::vector<uint8_t> mid = words(k4G - 2 * bb, 4 * bb), tail = words(last_off, kBig - last_off);
    CHECK(pwrite(wfd, mid.data(), mid.size(), (off_t)(k4G - 2 * bb)) == (ssize_t)mid.size());
    CHECK(pwrite(wfd, tail.data(), tail.size(), (off_t)last_off) == (ssize_t)tail.size());
    CHECK(close(wfd) == 0);
    struct stat s;
    CHECK(stat(path.c_str(), &s) == 0 && (uint64_t)s.st_size == kBig);
    const uint64_t nb = (kBig + bb - 1) / bb;
    std::vector<ScrubInode> inodes = {{(uint64_t)s.st_dev, (uint64_t)s.st_ino, kBig, 0, nb, 0, "huge"}};
    const int rfd = open(root.c_str(), O_RDONLY | O_DIRECTORY);
    CHECK(rfd >= 0);
    ScrubReader r;
    r.root_fds = {rfd}; r.inodes = &inodes;
    r.init();
    std::vector<uint8_t> slot(bb);
    for (const uint64_t off : {k4G - 2 * bb, k4G - bb, k4G, k4G + bb}) {
        CHECK(r.read(0, off, bb, slot.data()) == VMIG_OK);
        CHECK(slot == words(off, bb));
    }
    CHECK(r.read(0, 0, bb, slot.data()) == VMIG_OK && slot == std::vector<uint8_t>(bb, 0));          // a hole: not 2^32's bytes
    CHECK(r.read(0, 3ull << 30, bb, slot.data()) == VMIG_OK && slot == std::vector<uint8_t>(bb, 0));
    CHECK(kBig - last_off == 777);
    CHECK(r.read(0, last_off, 777, slot.data()) == VMIG_OK);
    CHECK(std::equal(tail.begin(), tail.end(), slot.begin()));
    CHECK(!r.unreadable(0));
    CHECK(r.read(0, last_off, bb, slot.data()) == VMIG_ESRCCHANGED);                                   // a whole block there is past the end
    r.close_all();
    close(rfd);
    CHECK(unlink(path.c_str()) == 0);
    return 0;
}

int main(int argc, char** argv) {
    if (argc < 2) return 2;
    if (merge_and_group() || escaping(argv[1]) || reader(argv[1]) || reader_large(argv[1])) return 1;
    printf("scrub unit ok\n");
    return 0;
}
