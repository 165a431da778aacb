// plan_unit.cpp -- CPU unit test of the plan of a tree call (csrc/vmig_plan.cpp; compiled and run by
// tests/test_plan_host.py), on real files with tables written by table_store:
//   - the block order is files in groups of 64, blocks round-robin across a group, for a migration's files (empty and
//     hard-linked paths left out) and for scrub-style spans;
//   - a destination file is patched in place only while it still is its prior record: a chmod or a same-size rewrite
//     makes it untrusted and counted; a second link, a missing file or a record without identity is neither;
//   - a base record that is no longer its file is counted for a same-path source file, one without identity is not;
//   - prior hashes come from the prior record or the base record, valid only where the block lengths agree;
//   - a cancel during the base check is VMIG_ECANCELED;
//   - a span longer than 2^32 bytes keeps 64-bit offsets: every block once, at r * block_bytes, the short last block last.
//   usage: plan_unit DIR
#include "vmig_plan.h"
#include "vmig_common.h"
#include <fcntl.h>
#include <unistd.h>
#include <sys/stat.h>
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <map>
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

static const uint32_t kBB = 4096;

static bool put(const std::string& p, uint64_t size, uint8_t fill) {
    const int fd = open(p.c_str(), O_WRONLY | O_CREAT | O_TRUNC, 0644);
    if (fd < 0) return false;
    std::vector<uint8_t> b(size, fill);
    const bool ok = size == 0 || pwrite(fd, b.data(), size, 0) == (ssize_t)size;
    return close(fd) == 0 && ok;
}

// The order the plan must produce, built the plain way: per group of 64, round r takes block r of every file that has one
struct Want { uint32_t file; uint64_t r; };
static std::vector<Want> round_robin(const std::vector<std::pair<uint32_t, uint64_t>>& files) {
    std::vector<Want> w;
    for (size_t g = 0; g < files.size(); g += 64) {
        const size_t g1 = std::min(files.size(), g + 64);
        for (uint64_t r = 0;; r++) {
            bool any = false;
            for (size_t i = g; i < g1; i++) if (r < files[i].second) { w.push_back({files[i].first, r}); any = true; }
            if (!any) break;
        }
    }
    return w;
}

static int block_order(const std::string& dir) {
    const std::string src = dir + "/order";
    CHECK(mkdir(src.c_str(), 0755) == 0);
    for (int i = 0; i < 130; i++) {
        char n[32]; snprintf(n, sizeof n, "/f%03d", i);
        const uint64_t size = i % 11 == 0 ? 0 : (uint64_t)(i * 2654435761u % (6 * kBB + 7));
        CHECK(put(src + n, size, (uint8_t)i));
        if (i % 17 == 3) { snprintf(n, sizeof n, "/f%03d", i); CHECK(link((src + n).c_str(), (src + n + "_link").c_str()) == 0); }
    }
    Manifest man;
    CHECK(walk_tree(src, kBB, false, &man) == VMIG_OK);
    TreePlan plan;
    CHECK(plan_tree(man, kBB, dir + "/none", nullptr, "", nullptr, nullptr, &plan) == VMIG_OK);
    std::vector<std::pair<uint32_t, uint64_t>> files;
    size_t links = 0, empty = 0;
    for (uint32_t f = 0; f < man.files.size(); f++) {
        const Entry& e = man.files[f];
        links += e.hardlink_of >= 0; empty += e.n_blocks == 0;
        if (e.hardlink_of >= 0) CHECK(!plan.files[(size_t)e.hardlink_of].solo);
        if (e.hardlink_of < 0 && e.n_blocks) files.push_back({f, e.n_blocks});
    }
    CHECK(man.files.size() == 138 && links == 8 && empty >= 12 && files.size() > 64);
    const std::vector<Want> w = round_robin(files);
    CHECK(plan.blocks.size() == w.size());
    for (size_t k = 0; k < w.size(); k++) {
        const BlockRef& b = plan.blocks[k];
        const Entry& e = man.files[w[k].file];
        CHECK(b.file == w[k].file && b.file_off == w[k].r * kBB && b.table_idx == e.first_block + w[k].r);
        CHECK(b.len == std::min<uint64_t>(kBB, e.size - b.file_off) && b.prior_valid == 0 && b.prior_hash == 0);
    }
    // scrub-style spans: inode indices, every span non-empty, first blocks packed in span order
    std::vector<BlockSpan> spans;
    std::vector<std::pair<uint32_t, uint64_t>> ids;
    uint64_t fb = 0;
    for (uint32_t u = 0; u < 150; u++) {
        const uint64_t size = 1 + (uint64_t)u * 40503u % (9 * kBB);
        const uint64_t nb = (size + kBB - 1) / kBB;
        spans.push_back({u, size, fb, nb});
        ids.push_back({u, nb});
        fb += nb;
    }
    std::vector<BlockRef> got;
    interleave_blocks(spans, kBB, &got);
    const std::vector<Want> ws = round_robin(ids);
    CHECK(got.size() == ws.size() && got.size() == fb);
    for (size_t k = 0; k < ws.size(); k++) {
        const BlockSpan& s = spans[ws[k].file];
        CHECK(got[k].file == s.file && got[k].file_off == ws[k].r * kBB && got[k].table_idx == s.first_block + ws[k].r);
        CHECK(got[k].len == std::min<uint64_t>(kBB, s.size - got[k].file_off));
    }
    return 0;
}

// One file of 2^32 + 9 MiB + 777 bytes among small ones, at 4 MiB blocks and at 1 MiB + 4096 (one block straddles 2^32)
static int large_spans() {
    const uint64_t kBig = (1ull << 32) + (9ull << 20) + 777;
    for (const uint32_t bb : {4u << 20, (1u << 20) + 4096}) {
        const uint64_t sizes[] = {3ull * bb + 5, kBig, 1, 2ull * bb};
        std::vector<BlockSpan> spans;
        std::vector<std::pair<uint32_t, uint64_t>> ids;
        uint64_t fb = 0;
        for (uint32_t u = 0; u < 4; u++) {
            const uint64_t nb = sizes[u] / bb + (sizes[u] % bb != 0);
            spans.push_back({u, sizes[u], fb, nb});
            ids.push_back({u, nb});
            fb += nb;
        }
        std::vector<BlockRef> got;
        interleave_blocks(spans, bb, &got);
        const std::vector<Want> w = round_robin(ids);
        CHECK(got.size() == w.size() && got.size() == fb);
        uint64_t next_r = 0, above = 0, straddle = 0, big_bytes = 0;       // of the big span
        for (size_t k = 0; k < w.size(); k++) {
            const BlockSpan& s = spans[w[k].file];
            const uint64_t off = w[k].r * (uint64_t)bb;
            const uint64_t len = w[k].r + 1 < s.n_blocks ? bb : s.size - off;
            CHECK(got[k].file == s.file && got[k].file_off == off && got[k].len == len && got[k].table_idx == s.first_block + w[k].r);
            if (s.file != 1) continue;
            CHECK(w[k].r == next_r++);                                      // in order, each exactly once
            above += off >= (1ull << 32);
            straddle += off < (1ull << 32) && off + len > (1ull << 32);
            big_bytes += len;
            if (w[k].r + 1 == s.n_blocks) CHECK(got[k].len == kBig % bb && got[k].file_off + got[k].len == kBig);
        }
        CHECK(next_r == spans[1].n_blocks && big_bytes == kBig);
        CHECK(above == spans[1].n_blocks - ((1ull << 32) + bb - 1) / bb && above >= 3);
        CHECK(straddle == ((1ull << 32) % bb != 0));
    }
    return 0;
}

// A table over the files of root, each record carrying the file's size, inode and ctime as lstat sees them (no identity
// for the names in no_id); block r of record i hashes to salt + 1000 * i + r.
static int write_table_of(const std::string& root, const std::vector<std::string>& names, const std::vector<std::string>& no_id,
                          uint64_t salt, const std::string& path) {
    BlockTable t; t.block_bytes = kBB;
    std::vector<std::string> sorted = names;
    std::sort(sorted.begin(), sorted.end());
    for (size_t i = 0; i < sorted.size(); i++) {
        const std::string& n = sorted[i];
        struct stat st;
        CHECK(lstat((root + "/" + n).c_str(), &st) == 0);
        TableFile f{n, (uint64_t)st.st_size, t.hashes.size(), (uint64_t)st.st_ino, ctime_ns(st)};
        if (std::find(no_id.begin(), no_id.end(), n) != no_id.end()) { f.ino = 0; f.ctime_ns = 0; }
        t.files.push_back(f);
        for (uint64_t r = 0; r < t.blocks_of(f); r++) t.hashes.push_back(salt + 1000 * i + r);
    }
    CHECK(table_store(path, t) == VMIG_OK);
    return 0;
}

static const Entry* find(const Manifest& m, const std::string& rel, uint32_t* f) {
    for (uint32_t i = 0; i < m.files.size(); i++) if (m.files[i].rel == rel) { *f = i; return &m.files[i]; }
    return nullptr;
}

// Every block of file rel: prior_valid as listed, and a valid prior hash is the record's (its table hash at block r)
static int check_prior(const TreePlan& plan, const Manifest& man, const BlockTable& t, const std::string& rel, const std::vector<int>& valid) {
    uint32_t f;
    const Entry* e = find(man, rel, &f);
    CHECK(e && e->n_blocks == valid.size());
    const TableFile& rec = t.files[t.index.at(rel)];
    size_t seen = 0;
    for (const BlockRef& b : plan.blocks) {
        if (b.file != f) continue;
        const uint64_t r = b.file_off / kBB;
        CHECK(b.prior_valid == valid[r]);
        CHECK(b.prior_hash == (valid[r] ? t.hashes[rec.first_block + r] : 0));
        seen++;
    }
    CHECK(seen == valid.size());
    return 0;
}

static int trust(const std::string& dir) {
    const std::string src = dir + "/src", dst = dir + "/dst", base = dir + "/base";
    for (const auto& d : {src, dst, base}) CHECK(mkdir(d.c_str(), 0755) == 0);
    // source: what the call migrates.  dst: the destination the prior table was written for.  base: a base snapshot.
    const std::map<std::string, uint64_t> src_sizes = {
        {"same", 2 * kBB + 100}, {"chmod", kBB}, {"rewrite", 3 * kBB}, {"linked", kBB}, {"missing", kBB}, {"fmt01", kBB},
        {"grew", 3 * kBB + 100}, {"short", 2 * kBB + 10}, {"snap", 2 * kBB + 5}, {"snap_chmod", kBB}, {"snap_fmt01", kBB}};
    for (const auto& kv : src_sizes) CHECK(put(src + "/" + kv.first, kv.second, 1));
    const std::vector<std::string> dnames = {"same", "chmod", "rewrite", "linked", "missing", "fmt01", "grew", "short"};
    const std::map<std::string, uint64_t> dst_sizes = {{"grew", 2 * kBB + 50}, {"short", 2 * kBB + 20}};
    for (const auto& n : dnames) CHECK(put(dst + "/" + n, dst_sizes.count(n) ? dst_sizes.at(n) : src_sizes.at(n), 2));
    CHECK(link((dst + "/linked").c_str(), (dst + "/linked.2").c_str()) == 0);
    const std::vector<std::string> bnames = {"snap", "snap_chmod", "snap_fmt01", "moved"};
    for (const auto& n : bnames) CHECK(put(base + "/" + n, n == "moved" ? 5 * kBB : src_sizes.at(n), 3));
    CHECK(write_table_of(dst, dnames, {"fmt01"}, 1u << 20, dir + "/prior.vmig") == 0);
    CHECK(write_table_of(base, bnames, {"snap_fmt01"}, 2u << 20, dir + "/base.vmig") == 0);
    usleep(50 * 1000);                                  // past the filesystem's timestamp granularity: ctimes move below
    CHECK(chmod((dst + "/chmod").c_str(), 0600) == 0);
    CHECK(put(dst + "/rewrite", 3 * kBB, 2));           // the same size and bytes, written again
    CHECK(unlink((dst + "/missing").c_str()) == 0);
    CHECK(chmod((base + "/snap_chmod").c_str(), 0600) == 0);

    Manifest man;
    CHECK(walk_tree(src, kBB, false, &man) == VMIG_OK);
    BlockTable prior, bt;
    CHECK(table_load(dir + "/prior.vmig", &prior) == VMIG_OK && table_load(dir + "/base.vmig", &bt) == VMIG_OK);

    // in-place trust against the prior table (a migration or restore with a prior table)
    TreePlan p;
    CHECK(plan_tree(man, kBB, dst, &prior, "", nullptr, nullptr, &p) == VMIG_OK);
    uint32_t f;
    for (const char* n : {"same", "grew", "short"}) { CHECK(find(man, n, &f) && p.files[f].prior_rec == &prior.files[prior.index.at(n)]); }
    for (const char* n : {"chmod", "rewrite", "linked", "missing", "fmt01"}) { CHECK(find(man, n, &f) && !p.files[f].prior_rec); }
    CHECK(p.files_untrusted == 2 && p.files_base_untrusted == 0 && !p.any_base && p.base_trusted.empty());
    CHECK(check_prior(p, man, prior, "same", {1, 1, 1}) == 0);            // equal sizes: the short last block too
    CHECK(check_prior(p, man, prior, "grew", {1, 1, 0, 0}) == 0);         // the record's block 2 is shorter, block 3 absent
    CHECK(check_prior(p, man, prior, "short", {1, 1, 0}) == 0);           // last blocks of 10 and 20 bytes
    CHECK(check_prior(p, man, prior, "chmod", {0}) == 0);

    // base trust (a snapshot): every base record is checked, a same-path one supplies prior hashes
    TreePlan s;
    CHECK(plan_tree(man, kBB, dst, nullptr, base, &bt, nullptr, &s) == VMIG_OK);
    CHECK((s.base_trusted == std::vector<uint8_t>{1, 1, 0, 0}));          // moved, snap, snap_chmod, snap_fmt01
    CHECK(find(man, "snap", &f) && s.files[f].base_rec == &bt.files[bt.index.at("snap")] && !s.files[f].prior_rec);
    CHECK(find(man, "snap_chmod", &f) && !s.files[f].base_rec);
    CHECK(find(man, "snap_fmt01", &f) && !s.files[f].base_rec);
    CHECK(s.files_base_untrusted == 1 && s.files_untrusted == 0 && s.any_base);
    CHECK(check_prior(s, man, bt, "snap", {1, 1, 1}) == 0);
    CHECK(check_prior(s, man, bt, "snap_chmod", {0}) == 0);

    // a cancel during the base check
    std::atomic<int> cancelled{1};
    TreePlan c;
    CHECK(plan_tree(man, kBB, dst, nullptr, base, &bt, &cancelled, &c) == VMIG_ECANCELED);
    CHECK(std::string(last_error_cstr()).find("base") != std::string::npos);
    return 0;
}

int main(int argc, char** argv) {
    if (argc < 2) return 2;
    if (block_order(argv[1]) || large_spans() || trust(argv[1])) return 1;
    printf("plan unit ok\n");
    return 0;
}
