// snapshot_layer_unit.cpp -- CPU unit test of the plan of vmig_snapshot_layer (csrc/vmig_plan.cpp with a layer table;
// compiled with g++ alone and run by tests/test_snapshot_layer_host.py), on real files:
//   - a trusted layer file's block is left out of the block list exactly when its record's (hash, length) is among the
//     trusted base files' blocks -- at its own path or any other, a short last block only against a block of its length;
//   - the remaining blocks keep interleave_blocks order and carry an expectation (the record's hash); untrusted files'
//     blocks carry none;
//   - a trusted file with no block to read is listed as unread and has no block in the list;
//   - a record that is no longer its file (ctime moved), a format-01 record, a hard-linked path and a table written for
//     another directory trust nothing;
//   - the counters: files / bytes trusted and read.
//   usage: snapshot_layer_unit DIR
#include "vmig_plan.h"
#include "vmig_common.h"
#include <fcntl.h>
#include <unistd.h>
#include <sys/stat.h>
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <set>
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

// A table of root's files rel -> hashes (sorted by rel), each record with the identity lstat shows now, except the
// paths in no_id (identity 0/0, as format 01 or a hard-linked path records it)
static bool table_of(const std::string& root, const std::map<std::string, std::vector<uint64_t>>& files, const std::set<std::string>& no_id,
                     BlockTable* t) {
    *t = BlockTable();
    t->block_bytes = kBB;
    for (const auto& kv : files) {
        struct stat st;
        if (lstat((root + "/" + kv.first).c_str(), &st) != 0) return false;
        TableFile f{kv.first, (uint64_t)st.st_size, t->hashes.size()};
        if (!no_id.count(kv.first)) { f.ino = st.st_ino; f.ctime_ns = ctime_ns(st); }
        if (t->blocks_of(f) != kv.second.size()) return false;
        t->index[f.rel] = t->files.size();
        t->files.push_back(f);
        t->hashes.insert(t->hashes.end(), kv.second.begin(), kv.second.end());
    }
    return true;
}

static bool find(const Manifest& m, const std::string& rel, uint32_t* f) {
    for (uint32_t i = 0; i < m.files.size(); i++) if (m.files[i].rel == rel) { *f = i; return true; }
    return false;
}

// (rel, block index) of every block in the plan's list, in list order
static std::vector<std::pair<std::string, uint64_t>> listed(const Manifest& m, const TreePlan& p) {
    std::vector<std::pair<std::string, uint64_t>> out;
    for (const BlockRef& b : p.blocks) out.push_back({m.files[b.file].rel, b.file_off / kBB});
    return out;
}

int main(int argc, char** argv) {
    if (argc < 2) return 2;
    const std::string dir = argv[1], src = dir + "/layer", dst = dir + "/dst", base = dir + "/base";
    for (const auto& d : {src, dst, base}) CHECK(mkdir(d.c_str(), 0755) == 0);
    CHECK(put(base + "/b_same", 3 * kBB, 1) && put(base + "/b_other", 2 * kBB, 2) && put(base + "/b_stale", kBB, 3));
    const std::map<std::string, std::vector<uint64_t>> bfiles = {{"b_other", {21, 22}}, {"b_same", {11, 12, 13}}, {"b_stale", {31}}};
    BlockTable bt;
    CHECK(table_of(base, bfiles, {}, &bt));
    const std::map<std::string, uint64_t> sizes = {
        {"b_same", 3 * kBB}, {"moved", 2 * kBB}, {"new", kBB + 5}, {"short", kBB + 10}, {"stale_base", kBB},
        {"untrusted", kBB}, {"fmt01", kBB}, {"hl", kBB}, {"empty", 0}};
    for (const auto& kv : sizes) CHECK(put(src + "/" + kv.first, kv.second, 9));
    CHECK(link((src + "/hl").c_str(), (src + "/hl2").c_str()) == 0);
    const std::map<std::string, std::vector<uint64_t>> lfiles = {
        {"b_same", {11, 12, 99}},        // blocks 0 and 1 at the same path in the base, block 2 nowhere
        {"moved", {21, 22}},             // every block in the base under another path: nothing to read
        {"new", {77, 13}},               // block 1 (5 bytes) has b_same's last hash but not its length
        {"short", {21, 22}},             // block 1 is 10 bytes: not the base's 4096-byte block with that hash
        {"stale_base", {31}},            // only in a base file that is no longer its record
        {"untrusted", {11}}, {"fmt01", {11}}, {"hl", {11}}, {"hl2", {11}}, {"empty", {}}};
    BlockTable lt;
    CHECK(table_of(src, lfiles, {"fmt01", "hl", "hl2"}, &lt));
    usleep(50 * 1000);                                  // past the filesystem's timestamp granularity: ctimes move below
    CHECK(chmod((src + "/untrusted").c_str(), 0600) == 0);
    CHECK(chmod((base + "/b_stale").c_str(), 0600) == 0);

    Manifest man;
    CHECK(walk_tree(src, kBB, false, &man) == VMIG_OK);
    TreePlan p;
    CHECK(plan_tree(man, kBB, dst, nullptr, base, &bt, nullptr, &p, src, &lt) == VMIG_OK);
    uint32_t f;
    for (const char* n : {"b_same", "moved", "new", "short", "stale_base"}) { CHECK(find(man, n, &f) && p.files[f].layer_rec == &lt.files[lt.index.at(n)]); }
    // a hard-linked path's record carries no identity
    for (const char* n : {"untrusted", "fmt01", "hl", "empty"}) { CHECK(find(man, n, &f) && !p.files[f].layer_rec); }
    CHECK(p.files_trusted == 5 && p.bytes_trusted == 3 * kBB + 2 * kBB + kBB + 5 + kBB + 10 + kBB);
    CHECK(find(man, "moved", &f) && p.unread == std::vector<uint32_t>{f});
    // what is read: b_same block 2, new (both), short block 1, stale_base, and the untrusted files in full
    std::vector<std::pair<std::string, uint64_t>> want;
    {
        TreePlan full;                                  // the same tree planned without the layer table: every block
        CHECK(plan_tree(man, kBB, dst, nullptr, base, &bt, nullptr, &full) == VMIG_OK);
        const std::set<std::pair<std::string, uint64_t>> skip = {{"b_same", 0}, {"b_same", 1}, {"moved", 0}, {"moved", 1}, {"short", 0}};
        for (const auto& b : listed(man, full)) if (!skip.count(b)) want.push_back(b);
    }
    CHECK(listed(man, p) == want);
    CHECK(p.files_read == 7 && p.bytes_read == kBB + (kBB + 5) + 10 + kBB + 3 * kBB);      // + untrusted, fmt01, hl
    for (const BlockRef& b : p.blocks) {
        const std::string& rel = man.files[b.file].rel;
        const bool trusted = p.files[b.file].layer_rec != nullptr;
        CHECK(p.expect[b.table_idx] == (trusted ? 1 : 0) && !p.skipped[b.table_idx]);
        if (trusted) CHECK(p.layer_hashes[b.table_idx] == lt.hashes[lt.files[lt.index.at(rel)].first_block + b.file_off / kBB]);
    }
    CHECK(find(man, "b_same", &f) && p.skipped[man.files[f].first_block] && p.skipped[man.files[f].first_block + 1] &&
          !p.skipped[man.files[f].first_block + 2]);
    CHECK(find(man, "moved", &f) && p.skipped[man.files[f].first_block] && p.layer_hashes[man.files[f].first_block + 1] == 22);
    // the same-path base block still supplies the positional prior hash of b_same's read block
    for (const BlockRef& b : p.blocks) if (man.files[b.file].rel == "b_same") CHECK(b.prior_valid && b.prior_hash == 13);

    // a table written for another directory (the base's own), or one without identities, trusts nothing
    BlockTable none;
    CHECK(table_of(src, lfiles, {"b_same", "moved", "new", "short", "stale_base", "untrusted", "fmt01", "hl", "hl2", "empty"}, &none));
    for (const BlockTable* t : {&bt, &none}) {
        TreePlan q;
        CHECK(plan_tree(man, kBB, dst, nullptr, base, &bt, nullptr, &q, src, t) == VMIG_OK);
        uint64_t primaries = 0;
        for (const Entry& e : man.files) if (e.hardlink_of < 0) primaries += e.size;
        CHECK(q.files_trusted == 0 && q.unread.empty() && q.bytes_read == primaries);
        TreePlan full;
        CHECK(plan_tree(man, kBB, dst, nullptr, base, &bt, nullptr, &full) == VMIG_OK);
        CHECK(listed(man, q) == listed(man, full));
        CHECK(std::count(q.expect.begin(), q.expect.end(), 1) == 0 && std::count(q.skipped.begin(), q.skipped.end(), 1) == 0);
    }
    printf("snapshot layer unit ok\n");
    return 0;
}
