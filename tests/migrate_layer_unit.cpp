// migrate_layer_unit.cpp -- CPU unit test of the plan of vmig_migrate_layer (csrc/vmig_plan.cpp with a source table and a
// prior table and no base; compiled with g++ alone and run by tests/test_migrate_layer_host.py), on real files:
//   - a trusted source file's block is left out of the block list exactly when its record's (hash, length) is the
//     destination's prior record's at the same index; a tail block whose length differs from the prior's is read;
//   - the remaining blocks keep interleave_blocks order and carry an expectation (the record's hash); untrusted files'
//     blocks carry none; a trusted file whose destination the prior table does not vouch for is read in full;
//   - a trusted file with no block to read is listed as unread and has no block in the list;
//   - a record whose inode, size or ctime is not the file's, a format-01 record, a hard-linked path and a table written
//     for another directory trust nothing;
//   - the counters: files / bytes trusted and read;
//   - the rule by which src_out_table records a file read while it may be written (live_identity_holds), on synthetic
//     stat values and clock readings.
//   usage: migrate_layer_unit DIR
#include "vmig_plan.h"
#include "vmig_common.h"
#include <fcntl.h>
#include <unistd.h>
#include <sys/stat.h>
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
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

static struct stat synth(uint64_t ino, uint64_t size, int64_t ctime, nlink_t nlink = 1) {
    struct stat st;
    memset(&st, 0, sizeof st);
    st.st_mode = S_IFREG | 0644; st.st_ino = ino; st.st_size = (off_t)size; st.st_nlink = nlink;
    st.st_ctim.tv_sec = ctime / 1000000000ll; st.st_ctim.tv_nsec = ctime % 1000000000ll;
    return st;
}

static int identity_rule() {
    const int64_t ct = 1700000000ll * 1000000000ll + 123456789;         // the file's ctime
    const struct stat before = synth(42, 10000, ct);
    CHECK(live_identity_holds(before, ct + 1, before));                // kept: older than the clock, nothing moved
    CHECK(live_identity_holds(before, ct + 4000000, synth(42, 10000, ct)));
    CHECK(!live_identity_holds(before, ct, before));                   // a ctime at the clock: a write in the same tick
    CHECK(!live_identity_holds(before, ct - 1, before));               // ... or past it
    CHECK(!live_identity_holds(before, 0, before));                    // no clock reading (the fstat failed)
    CHECK(!live_identity_holds(before, ct + 1, synth(43, 10000, ct)));        // the inode moved (replaced)
    CHECK(!live_identity_holds(before, ct + 1, synth(42, 10001, ct)));        // the size moved
    CHECK(!live_identity_holds(before, ct + 1, synth(42, 10000, ct + 1)));    // the ctime moved (written meanwhile)
    CHECK(!live_identity_holds(synth(42, 10000, ct, 2), ct + 1, synth(42, 10000, ct, 2)));   // a hard-linked inode
    struct stat dir = before;
    dir.st_mode = S_IFDIR | 0755;
    CHECK(!live_identity_holds(dir, ct + 1, dir));
    return 0;
}

int main(int argc, char** argv) {
    if (argc < 2) return 2;
    if (identity_rule()) return 1;
    const std::string dir = argv[1], src = dir + "/src", dst = dir + "/dst";
    for (const auto& d : {src, dst}) CHECK(mkdir(d.c_str(), 0755) == 0);
    const std::map<std::string, uint64_t> sizes = {
        {"same", 3 * kBB}, {"edit", 3 * kBB}, {"tail", kBB + 10}, {"grown", 2 * kBB}, {"nodst", 2 * kBB},
        {"ctime", kBB}, {"ino", kBB}, {"size", kBB + 5}, {"fmt01", kBB}, {"hl", kBB}, {"empty", 0}};
    for (const auto& kv : sizes) CHECK(put(src + "/" + kv.first, kv.second, 9));
    CHECK(link((src + "/hl").c_str(), (src + "/hl2").c_str()) == 0);
    // the destination as the previous pass left it, with its prior table
    const std::map<std::string, uint64_t> dsizes = {{"same", 3 * kBB}, {"edit", 3 * kBB}, {"tail", kBB + 20}, {"grown", kBB},
                                                    {"ctime", kBB}, {"ino", kBB}, {"size", kBB + 5}, {"fmt01", kBB}};
    for (const auto& kv : dsizes) CHECK(put(dst + "/" + kv.first, kv.second, 7));
    const std::map<std::string, std::vector<uint64_t>> pfiles = {
        {"edit", {1, 2, 3}}, {"fmt01", {4}}, {"grown", {5}}, {"ino", {4}}, {"same", {1, 2, 3}}, {"size", {6, 7}},
        {"tail", {5, 6}}, {"ctime", {4}}};
    BlockTable pt;
    CHECK(table_of(dst, pfiles, {}, &pt));
    const std::map<std::string, std::vector<uint64_t>> sfiles = {
        {"same", {1, 2, 3}},             // every block the prior's at the same index: nothing to read
        {"edit", {1, 99, 3}},            // block 1 differs
        {"tail", {5, 6}},                // block 1 is 10 bytes, the prior's 20: read although the hash is equal
        {"grown", {5, 8}},               // block 0 the prior's, block 1 past the prior's end
        {"nodst", {1, 2}},               // no destination record: read in full, each block checked
        {"ctime", {4}}, {"ino", {4}}, {"size", {6, 7}}, {"fmt01", {4}}, {"hl", {4}}, {"hl2", {4}}, {"empty", {}}};
    BlockTable st;
    CHECK(table_of(src, sfiles, {"fmt01", "hl", "hl2"}, &st));
    st.files[st.index.at("ino")].ino += 1000003;                     // a record of another inode
    st.files[st.index.at("size")].size += 1;                         // a record of another size (same block count)
    usleep(50 * 1000);                                  // past the filesystem's timestamp granularity: ctimes move below
    CHECK(chmod((src + "/ctime").c_str(), 0600) == 0);

    Manifest man;
    CHECK(walk_tree(src, kBB, false, &man) == VMIG_OK);
    TreePlan p;
    CHECK(plan_tree(man, kBB, dst, &pt, "", nullptr, nullptr, &p, src, &st) == VMIG_OK);
    uint32_t f;
    for (const char* n : {"same", "edit", "tail", "grown", "nodst"}) { CHECK(find(man, n, &f) && p.files[f].layer_rec == &st.files[st.index.at(n)]); }
    for (const char* n : {"ctime", "ino", "size", "fmt01", "hl", "hl2", "empty"}) { CHECK(find(man, n, &f) && !p.files[f].layer_rec); }
    for (const char* n : {"same", "edit", "tail", "grown", "ctime", "ino", "size", "fmt01"}) { CHECK(find(man, n, &f) && p.files[f].prior_rec); }
    CHECK(p.files_trusted == 5 && p.bytes_trusted == 3 * kBB + 3 * kBB + kBB + 10 + 2 * kBB + 2 * kBB);
    CHECK(find(man, "same", &f) && p.unread == std::vector<uint32_t>{f});
    std::vector<std::pair<std::string, uint64_t>> want;
    {
        TreePlan full;                                  // the same tree planned without the source table: every block
        CHECK(plan_tree(man, kBB, dst, &pt, "", nullptr, nullptr, &full) == VMIG_OK);
        const std::set<std::pair<std::string, uint64_t>> skip = {{"same", 0}, {"same", 1}, {"same", 2}, {"edit", 0}, {"edit", 2},
                                                                 {"tail", 0}, {"grown", 0}};
        for (const auto& b : listed(man, full)) if (!skip.count(b)) want.push_back(b);
        // the blocks read carry the same positional prior hash as without the source table
        for (const BlockRef& b : full.blocks)
            for (const BlockRef& c : p.blocks)
                if (b.table_idx == c.table_idx) CHECK(b.prior_valid == c.prior_valid && b.prior_hash == c.prior_hash);
    }
    CHECK(listed(man, p) == want);
    // read: edit block 1, tail block 1 (10 bytes), grown block 1, nodst in full; untrusted ctime, ino, size, fmt01, hl
    CHECK(p.files_read == 9 && p.bytes_read == kBB + 10 + kBB + 2 * kBB + kBB + kBB + (kBB + 5) + kBB + kBB);
    for (const BlockRef& b : p.blocks) {
        const std::string& rel = man.files[b.file].rel;
        const bool trusted = p.files[b.file].layer_rec != nullptr;
        CHECK(p.expect[b.table_idx] == (trusted ? 1 : 0) && !p.skipped[b.table_idx]);
        if (trusted) CHECK(p.layer_hashes[b.table_idx] == st.hashes[st.files[st.index.at(rel)].first_block + b.file_off / kBB]);
    }
    CHECK(find(man, "same", &f) && p.skipped[man.files[f].first_block] && p.skipped[man.files[f].first_block + 2] &&
          p.layer_hashes[man.files[f].first_block + 1] == 2);
    CHECK(find(man, "edit", &f) && p.skipped[man.files[f].first_block] && !p.skipped[man.files[f].first_block + 1]);
    CHECK(find(man, "tail", &f) && p.skipped[man.files[f].first_block] && !p.skipped[man.files[f].first_block + 1]);
    for (const BlockRef& b : p.blocks) if (man.files[b.file].rel == "tail") CHECK(!b.prior_valid);
    for (const BlockRef& b : p.blocks) if (man.files[b.file].rel == "edit") CHECK(b.prior_valid && b.prior_hash == 2);

    // without a prior table nothing is skipped: every trusted block is read and checked
    {
        TreePlan q;
        CHECK(plan_tree(man, kBB, dst, nullptr, "", nullptr, nullptr, &q, src, &st) == VMIG_OK);
        TreePlan full;
        CHECK(plan_tree(man, kBB, dst, nullptr, "", nullptr, nullptr, &full) == VMIG_OK);
        CHECK(q.files_trusted == 5 && q.unread.empty() && listed(man, q) == listed(man, full));
        CHECK(std::count(q.skipped.begin(), q.skipped.end(), 1) == 0);
        for (const BlockRef& b : q.blocks) CHECK(q.expect[b.table_idx] == (q.files[b.file].layer_rec ? 1 : 0));
    }
    // a table written for another directory (the destination's own), one without identities, or an empty one (no
    // src_table given) trusts nothing
    BlockTable none, empty;
    empty.block_bytes = kBB;
    CHECK(table_of(src, sfiles, {"same", "edit", "tail", "grown", "nodst", "ctime", "ino", "size", "fmt01", "hl", "hl2", "empty"}, &none));
    for (const BlockTable* t : {&pt, &none, &empty}) {
        TreePlan q;
        CHECK(plan_tree(man, kBB, dst, &pt, "", nullptr, nullptr, &q, src, t) == VMIG_OK);
        uint64_t primaries = 0;
        for (const Entry& e : man.files) if (e.hardlink_of < 0) primaries += e.size;
        CHECK(q.files_trusted == 0 && q.unread.empty() && q.bytes_read == primaries);
        TreePlan full;
        CHECK(plan_tree(man, kBB, dst, &pt, "", nullptr, nullptr, &full) == VMIG_OK);
        CHECK(listed(man, q) == listed(man, full));
        CHECK(std::count(q.expect.begin(), q.expect.end(), 1) == 0 && std::count(q.skipped.begin(), q.skipped.end(), 1) == 0);
    }
    printf("migrate layer unit ok\n");
    return 0;
}
