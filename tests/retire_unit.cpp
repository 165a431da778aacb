// retire_unit.cpp -- CPU unit test of the host side of vmig_retire_versions (csrc/vmig_retire.cpp; compiled and run by
// tests/test_retire_host.py):
//   - removal: the table goes first; files_freed / bytes_freed count an inode once, when its last link inside the
//     retired trees goes, and never an inode with a link outside them; a symlink to a directory outside is removed, not
//     followed; a missing version is not an error; a symlinked version is VMIG_ENOTDIR; a cancel stops the removal;
//   - selection: only a record of the same regular inode and size with another ctime is stale (another inode, another
//     size, no identity, a format-01 table, a missing path and an unchanged ctime are not);
//   - grouping and decision: one inode per (dev, ino) across versions; a record is re-stamped only when its blocks match,
//     its inode was readable and the ctime did not move after the walk;
//   - the table patch changes only the ino / ctime_ns bytes of the chosen records.
//   usage: retire_unit DIR
#include "vmig_retire.h"
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

static bool put(const std::string& p, size_t n, char c) {
    FILE* f = fopen(p.c_str(), "wb");
    if (!f) return false;
    std::string s(n, c);
    const bool ok = fwrite(s.data(), 1, n, f) == n;
    return fclose(f) == 0 && ok;
}
static bool exists(const std::string& p) { struct stat st; return lstat(p.c_str(), &st) == 0; }
static std::string slurp(const std::string& p) {
    std::string s; FILE* f = fopen(p.c_str(), "rb"); if (!f) return s;
    char b[4096]; size_t n; while ((n = fread(b, 1, sizeof b, f)) > 0) s.append(b, n);
    fclose(f); return s;
}

static int removal(const std::string& dir) {
    const std::string a = dir + "/a", b = dir + "/b", out = dir + "/outside", ta = dir + "/a.vmig";
    for (const auto& d : {a, a + "/sub", b, out, out + "/target"}) CHECK(mkdir(d.c_str(), 0755) == 0);
    CHECK(put(ta, 40, 't'));
    CHECK(put(a + "/only", 1000, 'o'));                     // freed with a
    CHECK(put(a + "/sub/deep", 300, 'd'));                  // freed with a
    CHECK(put(a + "/ab", 2000, 's'));                       // linked into b: freed once, with its last link
    CHECK(link((a + "/ab").c_str(), (b + "/ab").c_str()) == 0);
    CHECK(put(a + "/held", 5000, 'h'));                     // also linked outside: never freed
    CHECK(link((a + "/held").c_str(), (out + "/held").c_str()) == 0);
    CHECK(put(out + "/target/keep", 7, 'k'));
    CHECK(symlink((out + "/target").c_str(), (a + "/to_outside").c_str()) == 0);
    CHECK(put(b + "/own", 10, 'b'));
    RemoveCount n;
    CHECK(retire_remove(a, ta, &n, nullptr) == VMIG_OK);
    CHECK(!exists(a) && !exists(ta));
    CHECK(n.entries == 6);                                  // only, sub, sub/deep, ab, held, to_outside
    CHECK(n.files_freed == 2 && n.bytes_freed == 1300);
    CHECK(retire_remove(b, dir + "/b.vmig", &n, nullptr) == VMIG_OK);     // its table is already missing
    CHECK(!exists(b) && n.entries == 8 && n.files_freed == 4 && n.bytes_freed == 3310);
    CHECK(slurp(out + "/target/keep") == "kkkkkkk" && exists(out + "/held"));
    CHECK(retire_remove(a, ta, &n, nullptr) == VMIG_OK && n.entries == 8);   // a re-run finds nothing left
    // a version that is a symlink is not followed
    CHECK(symlink(out.c_str(), (dir + "/link").c_str()) == 0);
    CHECK(retire_remove(dir + "/link", dir + "/link.vmig", &n, nullptr) == VMIG_ENOTDIR);
    CHECK(exists(out + "/held") && exists(out + "/target/keep"));
    // a cancel: the table is gone, the tree stays, a re-run finishes
    const std::string c = dir + "/c", tc = dir + "/c.vmig";
    CHECK(mkdir(c.c_str(), 0755) == 0 && put(c + "/f", 1, 'f') && put(tc, 3, 't'));
    std::atomic<int> cancel{1};
    RemoveCount m;
    CHECK(retire_remove(c, tc, &m, &cancel) == VMIG_ECANCELED);
    CHECK(!exists(tc) && exists(c + "/f") && m.entries == 0);
    CHECK(retire_remove(c, tc, &m, nullptr) == VMIG_OK && !exists(c) && m.files_freed == 1);
    return 0;
}

static TableFile rec_of(const std::string& root, const std::string& rel) {
    struct stat st; stat((root + "/" + rel).c_str(), &st);
    return {rel, (uint64_t)st.st_size, 0, (uint64_t)st.st_ino, ctime_ns(st)};
}
static void lay_out(BlockTable* t) {
    uint64_t fb = 0;
    t->hashes.clear();
    for (auto& f : t->files) { f.first_block = fb; for (uint64_t r = 0; r < t->blocks_of(f); r++) t->hashes.push_back(0x1000 + fb + r); fb += t->blocks_of(f); }
}

static int selection(const std::string& dir) {
    const std::string v0 = dir + "/v0", v1 = dir + "/v1";
    CHECK(mkdir(v0.c_str(), 0755) == 0 && mkdir(v1.c_str(), 0755) == 0);
    for (const char* n : {"fresh", "missing", "no_id", "other_ino", "other_size", "stale", "unread", "moved", "wrong"}) CHECK(put(v0 + "/" + n, 9000, n[0]));
    const uint32_t bb = 4096;
    BlockTable t0; t0.block_bytes = bb;
    for (const char* n : {"fresh", "missing", "moved", "no_id", "other_ino", "other_size", "stale", "unread", "wrong"}) t0.files.push_back(rec_of(v0, n));
    t0.files[3].ino = 0; t0.files[3].ctime_ns = 0;          // no_id
    t0.files[4].ino += 1;                                  // other_ino
    t0.files[5].size += 1;                                 // other_size
    lay_out(&t0);
    // v1 names "stale" under another path: one inode, two records
    CHECK(link((v0 + "/stale").c_str(), (v1 + "/same").c_str()) == 0);
    BlockTable t1; t1.block_bytes = bb;
    t1.files.push_back(rec_of(v1, "same"));
    lay_out(&t1);
    unlink((v0 + "/missing").c_str());
    usleep(20000);
    for (const char* n : {"no_id", "other_ino", "other_size", "stale", "unread", "moved", "wrong"}) CHECK(chmod((v0 + "/" + n).c_str(), 0640) == 0);
    usleep(20000);
    CHECK(chmod((v1 + "/same").c_str(), 0600) == 0);        // t1's record moved too (the chmod above predates it)

    const int r0 = open(v0.c_str(), O_RDONLY | O_DIRECTORY), r1 = open(v1.c_str(), O_RDONLY | O_DIRECTORY);
    CHECK(r0 >= 0 && r1 >= 0);
    const std::vector<int> roots = {r0, r1};
    std::vector<const BlockTable*> tabs = {&t0, &t1};
    std::vector<StaleRecord> stale;
    CHECK(retire_find_stale(roots, tabs, &stale, nullptr) == VMIG_OK);
    std::vector<std::string> names;
    for (const auto& s : stale) names.push_back(tabs[s.version]->files[s.file].rel);
    CHECK((names == std::vector<std::string>{"moved", "stale", "unread", "wrong", "same"}));
    std::atomic<int> cancel{1};
    std::vector<StaleRecord> none;
    CHECK(retire_find_stale(roots, tabs, &none, &cancel) == VMIG_ECANCELED);

    // a format-01 table (no identities) has nothing stale
    const std::string p01 = dir + "/t01.vmig";
    {
        std::string raw("VMIGBT01", 8);
        const uint32_t b = bb, algo = 1, plen = 5; const uint64_t nf = 1, nb = 3, size = 9000, first = 0;
        raw.append((const char*)&b, 4); raw.append((const char*)&algo, 4); raw.append((const char*)&nf, 8); raw.append((const char*)&nb, 8);
        raw.append((const char*)&plen, 4); raw.append("stale"); raw.append((const char*)&size, 8); raw.append((const char*)&first, 8);
        raw.append(24, '\0');
        FILE* f = fopen(p01.c_str(), "wb"); CHECK(f && fwrite(raw.data(), 1, raw.size(), f) == raw.size()); fclose(f);
    }
    BlockTable t01;
    CHECK(table_load(p01, &t01) == VMIG_OK && t01.files.size() == 1 && t01.files[0].ino == 0);
    std::vector<const BlockTable*> tabs01 = {&t01};
    CHECK(retire_find_stale({r0}, tabs01, &none, nullptr) == VMIG_OK && none.empty());

    // grouping: "stale" and v1's "same" are one inode
    std::vector<ScrubInode> inodes;
    std::vector<uint32_t> inode_of;
    CHECK(retire_group(stale, tabs, bb, &inodes, &inode_of) == VMIG_OK);
    CHECK(inodes.size() == 4 && inode_of[1] == inode_of[4]);
    CHECK(inodes[inode_of[1]].rel == "stale" && inodes[inode_of[1]].version == 0 && inodes[inode_of[1]].n_blocks == 3);
    CHECK(inodes[0].first_block == 0 && inodes[1].first_block == 3 && inodes[3].first_block == 9);

    // decision: the read gave the table's hashes except for "wrong"; "unread" failed; "moved" changes after the walk
    std::vector<uint64_t> hashes(12);
    for (size_t r = 0; r < 4; r++) {
        const TableFile& rec = t0.files[stale[r].file];
        for (uint64_t b = 0; b < 3; b++) hashes[inodes[inode_of[r]].first_block + b] = t0.hashes[rec.first_block + b];
    }
    hashes[inodes[inode_of[3]].first_block + 2] ^= 1;      // "wrong": its last block differs
    std::vector<bool> unreadable(inodes.size(), false);
    unreadable[inode_of[2]] = true;
    CHECK(chmod((v0 + "/moved").c_str(), 0644) == 0);
    const std::vector<size_t> chosen = retire_decide(roots, tabs, stale, inodes, inode_of, hashes, unreadable);
    // only "stale" is re-stamped: v1's "same" is the same inode, but t1 records other hashes for it
    CHECK((chosen == std::vector<size_t>{1}));

    // the patch: only the identity bytes of the chosen record change
    const std::string pa = dir + "/t0.vmig", pb = dir + "/t0b.vmig";
    CHECK(table_store(pa, t0) == VMIG_OK);
    BlockTable t0b;
    CHECK(table_load(pa, &t0b) == VMIG_OK);
    CHECK(retire_patch(0, stale, chosen, inodes, inode_of, &t0b) == 1 && retire_patch(1, stale, chosen, inodes, inode_of, &t1) == 0);
    CHECK(t0b.files[6].ctime_ns == stale[1].ctime_ns && t0b.files[6].ino == t0.files[6].ino);
    CHECK(table_store(pb, t0b) == VMIG_OK);
    const std::string A = slurp(pa), B = slurp(pb);
    CHECK(A.size() == B.size());
    size_t off = 32;
    for (size_t i = 0; i < 6; i++) off += 4 + t0.files[i].rel.size() + 32;
    off += 4 + t0.files[6].rel.size() + 24;                 // stale's ctime_ns field
    for (size_t i = 0; i < A.size(); i++) CHECK((A[i] == B[i]) || (i >= off && i < off + 8));
    CHECK(A != B);
    close(r0); close(r1);
    return 0;
}

int main(int argc, char** argv) {
    if (argc != 2) { fprintf(stderr, "usage: retire_unit DIR\n"); return 2; }
    const std::string dir = argv[1];
    const std::string d1 = dir + "/removal", d2 = dir + "/selection";
    mkdir(d1.c_str(), 0755); mkdir(d2.c_str(), 0755);
    if (removal(d1) || selection(d2)) return 1;
    printf("retire unit ok\n");
    return 0;
}
