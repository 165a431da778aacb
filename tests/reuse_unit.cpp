// reuse_unit.cpp -- CPU unit test of the content reuse of vmig_snapshot_tree (csrc/vmig_reuse.cpp) and of the copy with
// separate offsets it backfills with (copy_range_at, csrc/vmig_tree.cpp); compiled and run by
// tests/test_snapshot_moved_host.py.
//   * plan_backfill picks, per skipped block, the same-path base block, else the continuation of the previous block's
//     base run, else the first index entry; runs contiguous in both files are coalesced;
//   * a short last block only matches a base block of exactly its length;
//   * untrusted base files are not in the index;
//   * a file longer than 2^32 bytes: runs longer than 2^32 bytes, and source and destination offsets above 2^32;
//   * link_candidates: same path first, then table order; equal size and every hash;
//   * copy_range_at puts [in_off, +len) of the input at [out_off, +len) of the output and nothing else, through
//     copy_file_range and through the forced pread/pwrite fallback, and whole sectors into an O_DIRECT output.
//   usage: reuse_unit DIR [DIR2 ...]
#include "vmig_reuse.h"
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

static const uint32_t BB = 4096;

// a base table: files of the given sizes with the given block hashes, in this (bytewise-sorted) order
static BlockTable table(const std::vector<std::pair<uint64_t, std::vector<uint64_t>>>& files) {
    BlockTable t; t.block_bytes = BB;
    for (size_t i = 0; i < files.size(); i++) {
        t.files.push_back({"f" + std::to_string(i), files[i].first, t.hashes.size(), 100 + i, 1});
        t.hashes.insert(t.hashes.end(), files[i].second.begin(), files[i].second.end());
        t.index[t.files.back().rel] = i;
    }
    return t;
}

static bool run_is(const ReuseRun& u, uint32_t file, uint64_t src_off, uint64_t dst_off, uint64_t len) {
    if (u.file == file && u.src_off == src_off && u.dst_off == dst_off && u.len == len) return true;
    printf("run {%u, %llu, %llu, %llu} != {%u, %llu, %llu, %llu}\n", u.file, (unsigned long long)u.src_off, (unsigned long long)u.dst_off,
           (unsigned long long)u.len, file, (unsigned long long)src_off, (unsigned long long)dst_off, (unsigned long long)len);
    return false;
}

static int planning() {
    // f0: A B C (full blocks), f1: X A B C, f2: A B + short tail T (100 bytes), f3 (untrusted): D, f4: A B C again
    const BlockTable t = table({{3 * BB, {0xA, 0xB, 0xC}}, {4 * BB, {0x5, 0xA, 0xB, 0xC}}, {2 * BB + 100, {0xA, 0xB, 0x7}},
                                {BB, {0xD}}, {3 * BB, {0xA, 0xB, 0xC}}});
    BaseIndex idx;
    idx.build(t, {1, 1, 1, 0, 1});
    CHECK(!idx.empty() && idx.size() == 3 + 4 + 3 + 3);
    size_t n;
    const BaseIndex::Loc* l = idx.find(0xA, BB, &n);
    CHECK(l && n == 4 && l[0].file == 0 && l[0].block == 0 && l[1].file == 1 && l[1].block == 1 && l[2].file == 2 && l[3].file == 4);
    CHECK(!idx.contains(0xD, BB));                    // f3 is not trusted
    CHECK(idx.contains(0x7, 100) && !idx.contains(0x7, BB) && !idx.contains(0x7, 99));     // the key includes the length
    CHECK(idx.block_len(2, 2) == 100 && idx.block_len(2, 3) == 0);

    std::vector<ReuseRun> runs;
    // a file renamed from f1 (no same-path record): X A B C -> first entry of X, then continuations: one run
    {
        const uint64_t h[] = {0x5, 0xA, 0xB, 0xC}; const uint8_t sk[] = {1, 1, 1, 1};
        CHECK(plan_backfill(idx, -1, 4 * BB, BB, h, sk, "x", &runs) == VMIG_OK);
        CHECK(runs.size() == 1 && run_is(runs[0], 1, 0, 0, 4 * BB));
    }
    // A B C with f4 as its same path: the same path wins over f0 (the first entry)
    {
        const uint64_t h[] = {0xA, 0xB, 0xC}; const uint8_t sk[] = {1, 1, 1};
        CHECK(plan_backfill(idx, 4, 3 * BB, BB, h, sk, "x", &runs) == VMIG_OK);
        CHECK(runs.size() == 1 && run_is(runs[0], 4, 0, 0, 3 * BB));
        CHECK(plan_backfill(idx, -1, 3 * BB, BB, h, sk, "x", &runs) == VMIG_OK);
        CHECK(runs.size() == 1 && run_is(runs[0], 0, 0, 0, 3 * BB));
    }
    // first block cut off: B C (blocks moved to lower offsets) -> f0 blocks 1..2
    {
        const uint64_t h[] = {0xB, 0xC}; const uint8_t sk[] = {1, 1};
        CHECK(plan_backfill(idx, -1, 2 * BB, BB, h, sk, "x", &runs) == VMIG_OK);
        CHECK(runs.size() == 1 && run_is(runs[0], 0, BB, 0, 2 * BB));
    }
    // same path f2 (A B T) but the new file is X A B T': block 0 first entry (f1), blocks 1-2 continue in f1, T' written
    {
        const uint64_t h[] = {0x5, 0xA, 0xB, 0x99}; const uint8_t sk[] = {1, 1, 1, 0};
        CHECK(plan_backfill(idx, 2, 3 * BB + 10, BB, h, sk, "x", &runs) == VMIG_OK);
        CHECK(runs.size() == 1 && run_is(runs[0], 1, 0, 0, 3 * BB));
    }
    // a written block breaks the continuation: A [written] C -> f0 block 0, then C by its first entry (f0 block 2)
    {
        const uint64_t h[] = {0xA, 0x42, 0xC}; const uint8_t sk[] = {1, 0, 1};
        CHECK(plan_backfill(idx, -1, 3 * BB, BB, h, sk, "x", &runs) == VMIG_OK);
        CHECK(runs.size() == 2 && run_is(runs[0], 0, 0, 0, BB) && run_is(runs[1], 0, 2 * BB, 2 * BB, BB));
    }
    // a same-path block that does not match falls back to the continuation: same path f0, new file C C -> f0 block 2 (first
    // entry of C), then f0 block 3 does not exist, so block 1 takes C's first entry again: two runs, not coalesced
    {
        const uint64_t h[] = {0xC, 0xC}; const uint8_t sk[] = {1, 1};
        CHECK(plan_backfill(idx, 0, 2 * BB, BB, h, sk, "x", &runs) == VMIG_OK);
        CHECK(runs.size() == 2 && run_is(runs[0], 0, 2 * BB, 0, BB) && run_is(runs[1], 0, 2 * BB, BB, BB));
    }
    // a short last block: A B T (100 bytes) from f2, renamed; the run ends at the file's size
    {
        const uint64_t h[] = {0xA, 0xB, 0x7}; const uint8_t sk[] = {1, 1, 1};
        CHECK(plan_backfill(idx, -1, 2 * BB + 100, BB, h, sk, "x", &runs) == VMIG_OK);
        // A is f0's first entry, B continues in f0, T continues nowhere (f0 block 2 is C) -> f2 block 2
        CHECK(runs.size() == 2 && run_is(runs[0], 0, 0, 0, 2 * BB) && run_is(runs[1], 2, 2 * BB, 2 * BB, 100));
    }
    // a skipped block the base does not hold is an internal inconsistency, not a silent hole
    {
        const uint64_t h[] = {0xD}; const uint8_t sk[] = {1};
        CHECK(plan_backfill(idx, -1, BB, BB, h, sk, "lost", &runs) == VMIG_ECORRUPT);
        CHECK(std::string(last_error_cstr()).find("lost") != std::string::npos);
    }
    // link candidates: equal size and every hash; the same path first, then table order
    std::vector<uint32_t> c;
    {
        const uint64_t h[] = {0xA, 0xB, 0xC};
        link_candidates(idx, -1, 3 * BB, BB, h, &c, 16);
        CHECK(c == std::vector<uint32_t>({0, 4}));
        link_candidates(idx, 4, 3 * BB, BB, h, &c, 16);
        CHECK(c == std::vector<uint32_t>({4, 0}));
        link_candidates(idx, 2, 3 * BB, BB, h, &c, 16);       // the same path differs: not a candidate
        CHECK(c == std::vector<uint32_t>({0, 4}));
        link_candidates(idx, -1, 3 * BB, BB, h, &c, 1);
        CHECK(c == std::vector<uint32_t>({0}));
        link_candidates(idx, -1, 3 * BB - 1, BB, h, &c, 16);  // another size
        CHECK(c.empty());
        const uint64_t t2[] = {0xA, 0xB, 0x7};
        link_candidates(idx, -1, 2 * BB + 100, BB, t2, &c, 16);
        CHECK(c == std::vector<uint32_t>({2}));
    }
    return 0;
}

// A new file of 2^32 + 9 MiB + 777 bytes at 4 MiB blocks.  Base file 0 holds the same blocks at the same indices, base file 1
// holds them three blocks further on, behind three blocks of its own.
static int planning_large() {
    const uint32_t bb = 4u << 20;
    const uint64_t kBig = (1ull << 32) + (9ull << 20) + 777, k4G = 1ull << 32;
    const uint64_t nb = (kBig + bb - 1) / bb, last_len = kBig - (nb - 1) * bb;
    CHECK(nb == 1027 && last_len == (1u << 20) + 777);
    std::vector<uint64_t> h(nb);
    for (uint64_t r = 0; r < nb; r++) h[r] = 0x1000 + r;
    BlockTable t; t.block_bytes = bb;
    t.files.push_back({"huge.bin", kBig, 0, 100, 1});
    t.hashes = h;
    t.files.push_back({"moved.bin", kBig + 3ull * bb, nb, 101, 1});
    for (uint64_t x : {0x1, 0x2, 0x3}) t.hashes.push_back(x);
    t.hashes.insert(t.hashes.end(), h.begin(), h.end());
    t.index["huge.bin"] = 0; t.index["moved.bin"] = 1;
    BaseIndex both, moved;
    both.build(t, {1, 1});
    moved.build(t, {0, 1});
    CHECK(both.block_len(0, nb - 1) == last_len && both.block_len(1, nb + 2) == last_len && both.block_len(0, nb) == 0);
    CHECK(both.block_len(0, 1024) == bb && both.block_len(0, 1023) == bb);

    std::vector<ReuseRun> runs;
    std::vector<uint8_t> sk(nb, 1);
    // only the last block was written: one run of more than 2^32 bytes from the same path
    std::vector<uint64_t> nh = h;
    nh[nb - 1] = 0x99; sk[nb - 1] = 0;
    CHECK(plan_backfill(both, 0, kBig, bb, nh.data(), sk.data(), "huge.bin", &runs) == VMIG_OK);
    CHECK(runs.size() == 1 && run_is(runs[0], 0, 0, 0, kBig - last_len) && runs[0].len > k4G);
    // only the first block was written: the run starts at one block and ends at the file's size
    nh = h; sk.assign(nb, 1);
    nh[0] = 0x99; sk[0] = 0;
    CHECK(plan_backfill(both, 0, kBig, bb, nh.data(), sk.data(), "huge.bin", &runs) == VMIG_OK);
    CHECK(runs.size() == 1 && run_is(runs[0], 0, bb, bb, kBig - bb) && runs[0].dst_off + runs[0].len == kBig);
    // no same-path record; the block after the one that starts at 2^32 was written: the content is found in the other
    // file three blocks further on, and the second run has both offsets above 2^32
    nh = h; sk.assign(nb, 1);
    nh[1025] = 0x99; sk[1025] = 0;
    CHECK(plan_backfill(moved, -1, kBig, bb, nh.data(), sk.data(), "renamed.bin", &runs) == VMIG_OK);
    CHECK(runs.size() == 2 && run_is(runs[0], 1, 3ull * bb, 0, 1025ull * bb));
    CHECK(run_is(runs[1], 1, 1029ull * bb, 1026ull * bb, kBig - 1026ull * bb));
    CHECK(runs[1].src_off > k4G && runs[1].dst_off > k4G && runs[1].src_off != runs[1].dst_off && runs[0].len > k4G);
    // the whole file elsewhere is a link candidate only at its own size
    std::vector<uint32_t> c;
    link_candidates(both, -1, kBig, bb, h.data(), &c, 16);
    CHECK(c == std::vector<uint32_t>({0}));
    link_candidates(both, -1, kBig - k4G, bb, h.data(), &c, 16);       // the size a 32-bit length would see
    CHECK(c.empty());
    return 0;
}

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

static int copies(const std::string& dir) {
    const size_t size = (3u << 20) + 123;
    const std::vector<uint8_t> base = pattern(size, 1), old = pattern(size, 2);
    const std::string in = dir + "/base.bin";
    CHECK(put(in, base));
    for (int rw_only = 0; rw_only < 2; rw_only++) {
        const std::string out = dir + "/at" + std::to_string(rw_only) + ".bin";
        CHECK(put(out, old));
        const int ifd = open(in.c_str(), O_RDONLY), ofd = open(out.c_str(), O_WRONLY);
        CHECK(ifd >= 0 && ofd >= 0);
        // base [2 MiB, 3 MiB) to out [0, 1 MiB); base's short tail to out [1 MiB, +123); a range past base's end
        CHECK(copy_range_at(ifd, 2u << 20, ofd, 0, 1u << 20, false, rw_only != 0, in) == VMIG_OK);
        CHECK(copy_range_at(ifd, 3u << 20, ofd, 1u << 20, 123, false, rw_only != 0, in) == VMIG_OK);
        CHECK(copy_range_at(ifd, 3u << 20, ofd, 2u << 20, 200, false, rw_only != 0, in) == VMIG_ESRCCHANGED);
        close(ifd); close(ofd);
        std::vector<uint8_t> want = old;
        std::copy(base.begin() + (2u << 20), base.begin() + (3u << 20), want.begin());
        std::copy(base.begin() + (3u << 20), base.end(), want.begin() + (1u << 20));
        CHECK(get(out).size() == size);
        const std::vector<uint8_t> got = get(out);
        CHECK(std::equal(want.begin(), want.begin() + (1u << 20) + 123, got.begin()));
        CHECK(std::equal(want.begin() + (2u << 20) + 200, want.end(), got.begin() + (2u << 20) + 200));   // past the failed range: untouched
    }
    // O_DIRECT output: base [1 MiB, 3 MiB + 123) to [0, 2 MiB + 123), padded to whole sectors, then cut to size
    const std::string dout = dir + "/at_direct.bin";
    const int dfd = open(dout.c_str(), O_WRONLY | O_CREAT | O_TRUNC | O_DIRECT, 0600);
    if (dfd < 0) { printf("direct: refused by %s\n", dir.c_str()); return 0; }
    const int ifd = open(in.c_str(), O_RDONLY);
    CHECK(ifd >= 0);
    CHECK(copy_range_at(ifd, 1u << 20, dfd, 0, (2u << 20) + 123, true, false, in) == VMIG_OK);
    CHECK(ftruncate(dfd, (off_t)((2u << 20) + 123)) == 0);
    close(ifd); close(dfd);
    CHECK(get(dout) == std::vector<uint8_t>(base.begin() + (1u << 20), base.end()));
    printf("direct: ok in %s\n", dir.c_str());
    return 0;
}

int main(int argc, char** argv) {
    if (argc < 2) return 2;
    if (planning() || planning_large()) return 1;
    for (int i = 1; i < argc; i++) if (copies(argv[i])) return 1;
    printf("reuse unit ok\n");
    return 0;
}
