// rollback_unit.cpp -- CPU unit test of the host side of vmig_rollback_layer (csrc/vmig_rollback.cpp; compiled with g++
// alone and run by tests/test_rollback_host.py) over real trees walked by walk_tree:
//   - the action of every case: keep, patch (a changed block, layer longer, layer shorter, a last block of another length,
//     empty files on either side), rebuild (an inode shared with the snapshot, a link held outside the tree, hard-link
//     groups on either side) and create;
//   - the fetch list's order and table_idx, and the coalesced copy runs of rebuilt files;
//   - bytes_fetched against compare_merge's bytes_restore on the same inputs;
//   - the layer identity checks: a descriptor whose file was written, chmod'ed or replaced by a rename since the plan
//     is VMIG_ESRCCHANGED naming the path, an unchanged one passes; likewise the lstat re-check after the hash pass;
//   - the rebuild sequence over a layer hard-link group the snapshot holds as separate files (RebuildGuard).
//   usage: rollback_unit DIR
#include "vmig_rollback.h"
#include "vmig_common.h"
#include "vmig_table.h"
#include <fcntl.h>
#include <unistd.h>
#include <sys/stat.h>
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
static std::string g_dir;

// n bytes: block r filled with the byte seed + r
static void put(const std::string& p, size_t n, int seed) {
    std::string b(n, 0);
    for (size_t i = 0; i < n; i++) b[i] = (char)(seed + i / kBB);
    const int fd = open(p.c_str(), O_WRONLY | O_CREAT | O_TRUNC, 0644);
    if (fd < 0 || write(fd, b.data(), b.size()) != (ssize_t)b.size()) { perror(p.c_str()); exit(2); }
    close(fd);
}
static std::string fresh(const std::string& name) {
    const std::string d = g_dir + "/" + name;
    mkdir(d.c_str(), 0755);
    return d;
}
// a stand-in for K1: FNV-1a of each block's bytes, in the manifest's block order
static std::vector<uint64_t> hashes_of(const std::string& root, const Manifest& m) {
    std::vector<uint64_t> h(m.n_blocks);
    for (const Entry& e : m.files) {
        const int fd = open(pjoin(root, e.rel).c_str(), O_RDONLY);
        std::string b(kBB, 0);
        for (uint64_t r = 0; r < e.n_blocks; r++) {
            const ssize_t n = pread(fd, &b[0], kBB, (off_t)(r * kBB));
            uint64_t x = 1469598103934665603ull;
            for (ssize_t i = 0; i < n; i++) { x ^= (uint8_t)b[i]; x *= 1099511628211ull; }
            h[e.first_block + r] = x;
        }
        close(fd);
    }
    return h;
}
static std::vector<const uint64_t*> ptrs(const Manifest& m, const std::vector<uint64_t>& h) {
    std::vector<const uint64_t*> p;
    for (const Entry& e : m.files) p.push_back(e.n_blocks ? h.data() + e.first_block : nullptr);
    return p;
}
static const RollbackFile* file_at(const RollbackPlan& p, const Manifest& s, const std::string& rel) {
    for (const RollbackFile& f : p.files) if (s.files[f.snap].rel == rel) return &f;
    return nullptr;
}
static std::vector<uint64_t> fetched_blocks(const RollbackPlan& p, const RollbackFile* f) {
    std::vector<uint64_t> v;
    const uint32_t fi = (uint32_t)(f - p.files.data());
    for (const BlockRef& b : p.fetch) if (b.file == fi) v.push_back(b.file_off / kBB);
    return v;
}

struct Case {
    Manifest L, S;
    std::vector<uint64_t> lh, sh;
    ComparePlan cp;
    std::vector<LayerId> ids;
    RollbackPlan rp;
    CompareCounts cc;
};
static int plan_case(const std::string& Ld, const std::string& Sd, Case* c) {
    if (walk_tree(Ld, kBB, false, &c->L) || walk_tree(Sd, kBB, false, &c->S)) return 1;
    if (compare_plan(Ld, c->L, c->S, nullptr, kBB, &c->cp)) return 1;
    if (rollback_identify(Ld, c->L, c->cp, nullptr, &c->ids)) return 1;
    c->lh = hashes_of(Ld, c->L); c->sh = hashes_of(Sd, c->S);
    rollback_plan(c->L, c->S, c->sh, c->cp, ptrs(c->L, c->lh), c->ids, kBB, 0, &c->rp);
    std::vector<CompareFinding> findings;
    compare_merge(c->L, c->S, c->sh, ptrs(c->L, c->lh), kBB, false, true, &findings, &c->cc);
    return 0;
}

static int actions() {
    const std::string L = fresh("act_l"), S = fresh("act_s"), O = fresh("act_outside");
    put(S + "/same", 3 * kBB + 10, 1);        put(L + "/same", 3 * kBB + 10, 1);
    put(S + "/changed", 4 * kBB, 1);          put(L + "/changed", 4 * kBB, 1);
    { const int fd = open((L + "/changed").c_str(), O_WRONLY); if (pwrite(fd, "x", 1, kBB + 3) != 1) return 1; close(fd); }
    put(S + "/longer", 2 * kBB, 1);           put(L + "/longer", 3 * kBB + 5, 1);
    put(S + "/shorter", 3 * kBB + 7, 1);      put(L + "/shorter", kBB, 1);
    put(S + "/lastlen", 2 * kBB + 100, 1);    put(L + "/lastlen", 2 * kBB + 200, 1);
    put(S + "/empty_s", 0, 1);                put(L + "/empty_s", 2 * kBB, 1);
    put(S + "/empty_l", 2 * kBB + 1, 1);      put(L + "/empty_l", 0, 1);
    put(S + "/empty_both", 0, 1);             put(L + "/empty_both", 0, 1);
    put(S + "/gone", 2 * kBB, 1);
    mkdir((L + "/typed").c_str(), 0755);      put(S + "/typed", kBB, 1);    // (a pruning restore removes the directory first)
    put(S + "/shared", 3 * kBB, 1);           if (link((S + "/shared").c_str(), (L + "/shared").c_str())) return 1;
    put(S + "/outside", 3 * kBB, 1);          put(L + "/outside", 3 * kBB, 1);
    { const int fd = open((L + "/outside").c_str(), O_WRONLY); if (pwrite(fd, "y", 1, kBB) != 1) return 1; close(fd); }
    if (link((L + "/outside").c_str(), (O + "/x").c_str())) return 1;
    put(S + "/grp_a", 2 * kBB, 1);            put(L + "/grp_a", 2 * kBB, 1);  if (link((L + "/grp_a").c_str(), (L + "/grp_b").c_str())) return 1;
    put(S + "/grp_b", 2 * kBB, 1);
    put(S + "/sg_a", 2 * kBB, 1);             if (link((S + "/sg_a").c_str(), (S + "/sg_b").c_str())) return 1;
    put(L + "/sg_a", 2 * kBB, 1);             put(L + "/sg_b", 2 * kBB, 9);
    Case c;
    CHECK(plan_case(L, S, &c) == 0);
    const RollbackPlan& p = c.rp;
    struct Want { const char* rel; RollbackAction a; std::vector<uint64_t> fetch; };
    const std::vector<Want> want = {
        {"changed", kRbPatch, {1}}, {"empty_both", kRbKeep, {}}, {"empty_l", kRbPatch, {0, 1, 2}}, {"empty_s", kRbPatch, {}},
        {"gone", kRbCreate, {0, 1}}, {"grp_a", kRbRebuild, {}}, {"lastlen", kRbPatch, {2}}, {"longer", kRbPatch, {}},
        {"outside", kRbRebuild, {1}}, {"same", kRbKeep, {}}, {"sg_a", kRbRebuild, {}}, {"shared", kRbRebuild, {}},
        {"shorter", kRbPatch, {1, 2, 3}}, {"typed", kRbCreate, {0}}};
    for (const Want& w : want) {
        const RollbackFile* f = file_at(p, c.S, w.rel);
        if (!f || f->action != w.a || fetched_blocks(p, f) != w.fetch) {
            printf("FAIL %s: action %s, %zu blocks fetched\n", w.rel, f ? rollback_action_name(f->action) : "-", f ? fetched_blocks(p, f).size() : 0);
            return 1;
        }
    }
    CHECK(file_at(p, c.S, "grp_b") && file_at(p, c.S, "grp_b")->action == kRbRebuild);   // its layer path is in a group
    CHECK(!file_at(p, c.S, "sg_b"));                         // a secondary path is linked, never planned
    CHECK(p.files_kept == 2 && p.files_created == 2 && p.files_rebuilt == 5 && p.files_patched == 6);
    // fetch list: files in snapshot order, ascending offsets, table_idx the snapshot's global block index, lengths
    uint32_t last_file = 0; uint64_t last_off = 0; bool first = true;
    for (const BlockRef& b : p.fetch) {
        const Entry& s = c.S.files[p.files[b.file].snap];
        CHECK(first || b.file > last_file || (b.file == last_file && b.file_off > last_off));
        CHECK(b.table_idx == s.first_block + b.file_off / kBB && b.file_off % kBB == 0);
        CHECK(b.len == std::min<uint64_t>(kBB, s.size - b.file_off) && !b.prior_valid);
        first = false; last_file = b.file; last_off = b.file_off;
    }
    // copy runs: the shared file in one run, the outside-linked file around its fetched block, the groups whole
    std::map<std::string, std::vector<std::pair<uint64_t, uint64_t>>> runs;
    for (const CopyRun& u : p.runs) runs[c.S.files[p.files[u.file].snap].rel].push_back({u.off, u.len});
    CHECK((runs["shared"] == std::vector<std::pair<uint64_t, uint64_t>>{{0, 3 * kBB}}));
    CHECK((runs["outside"] == std::vector<std::pair<uint64_t, uint64_t>>{{0, kBB}, {2 * kBB, kBB}}));
    CHECK((runs["grp_a"] == std::vector<std::pair<uint64_t, uint64_t>>{{0, 2 * kBB}}));
    CHECK((runs["sg_a"] == std::vector<std::pair<uint64_t, uint64_t>>{{0, 2 * kBB}}));
    CHECK(p.bytes_copied == 3 * kBB + 2 * kBB + 2 * kBB + 2 * kBB + 2 * kBB);
    // bytes_fetched is compare's bytes_restore, less the snapshot group's second path (sg_b differs: 2 blocks)
    uint64_t bytes = 0;
    for (const BlockRef& b : p.fetch) bytes += b.len;
    CHECK(bytes == p.bytes_fetched && p.blocks_fetched == p.fetch.size());
    CHECK(p.bytes_fetched + 2 * kBB == c.cc.bytes_restore);
    // a non-root caller does not patch a file it cannot write: replaced instead
    RollbackPlan q;
    rollback_plan(c.L, c.S, c.sh, c.cp, ptrs(c.L, c.lh), c.ids, kBB, 4242, &q);
    CHECK(file_at(q, c.S, "changed")->action == kRbRebuild && q.bytes_fetched == p.bytes_fetched);
    return 0;
}

// bytes_fetched == bytes_restore where the snapshot has no hard-link group
static int restore_identity() {
    const std::string L = fresh("id_l"), S = fresh("id_s");
    for (int i = 0; i < 12; i++) {
        const std::string n = "/f" + std::to_string(i);
        put(S + n, (size_t)(i * 1500 + (i % 3) * kBB), i);
        if (i % 4) put(L + n, (size_t)(i * 1700 + (i % 2) * kBB), i + (i % 5 == 0));
    }
    Case c;
    CHECK(plan_case(L, S, &c) == 0);
    CHECK(c.rp.bytes_fetched == c.cc.bytes_restore && c.cc.bytes_restore > 0);
    return 0;
}

static int identity_checks() {
    const std::string D = fresh("ident");
    const std::string p = D + "/f";
    put(p, 2 * kBB, 3);
    struct stat st;
    CHECK(lstat(p.c_str(), &st) == 0);
    const LayerId id = layer_id_of(st);
    int fd = open(p.c_str(), O_RDWR);
    CHECK(rollback_check_fd(fd, id, p) == VMIG_OK);            // unchanged
    usleep(20000);                                            // past the filesystem clock's granularity
    CHECK(pwrite(fd, "z", 1, 5) == 1);                        // a write: same inode and size, the ctime moved
    CHECK(rollback_check_fd(fd, id, p) == VMIG_ESRCCHANGED && strstr(last_error_cstr(), p.c_str()));
    close(fd);
    put(p, 2 * kBB, 3);
    CHECK(lstat(p.c_str(), &st) == 0);
    const LayerId id2 = layer_id_of(st);
    usleep(20000);
    CHECK(chmod(p.c_str(), 0600) == 0);                       // a chmod
    fd = open(p.c_str(), O_RDONLY);
    CHECK(rollback_check_fd(fd, id2, p) == VMIG_ESRCCHANGED && strstr(last_error_cstr(), p.c_str()));
    close(fd);
    CHECK(lstat(p.c_str(), &st) == 0);
    const LayerId id3 = layer_id_of(st);
    put(D + "/g", 2 * kBB, 3);                                // a replacement by rename: another inode
    CHECK(rename((D + "/g").c_str(), p.c_str()) == 0);
    fd = open(p.c_str(), O_RDONLY);
    CHECK(rollback_check_fd(fd, id3, p) == VMIG_ESRCCHANGED && strstr(last_error_cstr(), p.c_str()));
    close(fd);
    CHECK(lstat(p.c_str(), &st) == 0);
    const LayerId id4 = layer_id_of(st);
    CHECK(truncate(p.c_str(), kBB) == 0);                     // a new size
    fd = open(p.c_str(), O_RDONLY);
    CHECK(rollback_check_fd(fd, id4, p) == VMIG_ESRCCHANGED);
    close(fd);

    // the lstat re-check after the hash pass
    const std::string L = fresh("re_l"), S = fresh("re_s");
    put(L + "/a", 2 * kBB, 1); put(S + "/a", 2 * kBB, 2);
    put(L + "/b", 2 * kBB, 1); put(S + "/b", 2 * kBB, 1);
    Manifest ml, ms;
    CHECK(walk_tree(L, kBB, false, &ml) == VMIG_OK && walk_tree(S, kBB, false, &ms) == VMIG_OK);
    ComparePlan cp;
    CHECK(compare_plan(L, ml, ms, nullptr, kBB, &cp) == VMIG_OK);
    std::vector<LayerId> ids;
    CHECK(rollback_identify(L, ml, cp, nullptr, &ids) == VMIG_OK && ids[0].set && ids[1].set);
    CHECK(rollback_recheck_paths(L, ml, ids) == VMIG_OK);
    usleep(20000);
    CHECK(chmod((L + "/b").c_str(), 0600) == 0);
    CHECK(rollback_recheck_paths(L, ml, ids) == VMIG_ESRCCHANGED && strstr(last_error_cstr(), "/b"));
    // a trusted file's identity is its record's
    BlockTable t; t.block_bytes = kBB;
    CHECK(lstat((L + "/a").c_str(), &st) == 0);
    t.files.push_back({"a", 2 * kBB, 0, (uint64_t)st.st_ino, ctime_ns(st)});
    t.files.push_back({"b", 2 * kBB, 2, 0, 0});
    t.hashes.assign(4, 0);
    t.index["a"] = 0; t.index["b"] = 1;
    CHECK(compare_plan(L, ml, ms, &t, kBB, &cp) == VMIG_OK && cp.source[0] == kCmpTrusted && cp.source[1] == kCmpRead);
    CHECK(rollback_identify(L, ml, cp, &t, &ids) == VMIG_OK && ids[0].ino == (uint64_t)st.st_ino && ids[0].ctime_ns == ctime_ns(st));
    return 0;
}

// The rebuild sequence prepare runs, in plan order: open the old inode, check it and clear its path (RebuildGuard),
// create the new file and copy the runs.  A layer hard-link group whose paths the snapshot holds as separate files is
// rebuilt path by path: the call's own unlink of the first path must not fail the second path's check, while a change
// made by anyone else still does.
static int run_rebuilds(const std::string& L, const Case& c, RebuildGuard* guard) {
    for (const RollbackFile& f : c.rp.files) {
        if (f.action != kRbRebuild) continue;
        const std::string p = pjoin(L, c.S.files[f.snap].rel);
        const int old = open(p.c_str(), (f.n_runs ? O_RDONLY : O_PATH) | O_NOFOLLOW);
        if (old < 0) return VMIG_EIO;
        int rc = guard->clear(old, c.ids[(size_t)f.layer], f.n_runs != 0, p);
        const int fd = rc ? -1 : open(p.c_str(), O_WRONLY | O_CREAT | O_EXCL, 0600);
        if (!rc && fd < 0) rc = VMIG_EIO;
        for (uint64_t k = 0; !rc && k < f.n_runs; k++) {
            const CopyRun& u = c.rp.runs[f.first_run + k];
            rc = copy_range_at(old, u.off, fd, u.off, u.len, false, false, p);
        }
        close(old);
        if (fd >= 0) close(fd);
        if (rc) return rc;
    }
    return VMIG_OK;
}

static std::string read_all(const std::string& p) {
    std::string b;
    const int fd = open(p.c_str(), O_RDONLY);
    char buf[8192];
    ssize_t n;
    while ((n = read(fd, buf, sizeof buf)) > 0) b.append(buf, (size_t)n);
    close(fd);
    return b;
}

static int rebuild_sequence() {
    // three layer paths of one inode, the snapshot's three separate files: all equal, one differing in block 1
    const std::string L = fresh("seq_l"), S = fresh("seq_s");
    put(S + "/x", 3 * kBB, 1); put(S + "/y", 3 * kBB, 1); put(S + "/z", 3 * kBB, 1);
    put(L + "/x", 3 * kBB, 1);
    CHECK(link((L + "/x").c_str(), (L + "/y").c_str()) == 0 && link((L + "/x").c_str(), (L + "/z").c_str()) == 0);
    put(S + "/w", 2 * kBB, 4); put(L + "/w", 0, 4);            // empty in the layer, in a group: nothing to copy
    CHECK(link((L + "/w").c_str(), (L + "/w2").c_str()) == 0);
    put(S + "/w2", 2 * kBB, 4);
    Case c;
    CHECK(plan_case(L, S, &c) == 0);
    for (const char* n : {"x", "y", "z", "w", "w2"}) CHECK(file_at(c.rp, c.S, n)->action == kRbRebuild);
    CHECK(file_at(c.rp, c.S, "w")->n_runs == 0 && file_at(c.rp, c.S, "x")->n_runs == 1);
    usleep(20000);                                            // past the filesystem clock's granularity
    RebuildGuard guard;
    CHECK(run_rebuilds(L, c, &guard) == VMIG_OK);
    struct stat a, b;
    for (const char* n : {"x", "y", "z"}) {
        CHECK(read_all(L + "/" + n) == read_all(S + "/x"));
        CHECK(lstat((L + "/" + n).c_str(), &a) == 0 && a.st_nlink == 1);
    }
    CHECK(lstat((L + "/x").c_str(), &a) == 0 && lstat((L + "/y").c_str(), &b) == 0 && a.st_ino != b.st_ino);

    // someone else's change to the group's inode after the plan still fails the check, also after an own unlink
    const std::string L2 = fresh("seq2_l"), S2 = fresh("seq2_s");
    put(S2 + "/x", 2 * kBB, 1); put(S2 + "/y", 2 * kBB, 1); put(S2 + "/z", 2 * kBB, 1);
    put(L2 + "/x", 2 * kBB, 1);
    CHECK(link((L2 + "/x").c_str(), (L2 + "/y").c_str()) == 0 && link((L2 + "/x").c_str(), (L2 + "/z").c_str()) == 0);
    Case c2;
    CHECK(plan_case(L2, S2, &c2) == 0);
    usleep(20000);
    CHECK(chmod((L2 + "/z").c_str(), 0600) == 0);               // before any path is cleared
    RebuildGuard g2;
    CHECK(run_rebuilds(L2, c2, &g2) == VMIG_ESRCCHANGED && strstr(last_error_cstr(), "/x"));
    const std::string L3 = fresh("seq3_l"), S3 = fresh("seq3_s");
    put(S3 + "/x", 2 * kBB, 1); put(S3 + "/y", 2 * kBB, 1);
    put(L3 + "/x", 2 * kBB, 1);
    CHECK(link((L3 + "/x").c_str(), (L3 + "/y").c_str()) == 0);
    Case c3;
    CHECK(plan_case(L3, S3, &c3) == 0);
    RebuildGuard g3;
    const RollbackFile* fx = file_at(c3.rp, c3.S, "x");
    int old = open((L3 + "/x").c_str(), O_RDONLY);
    CHECK(g3.clear(old, c3.ids[(size_t)fx->layer], true, L3 + "/x") == VMIG_OK);
    close(old);
    usleep(20000);
    CHECK(chmod((L3 + "/y").c_str(), 0600) == 0);               // after the own unlink
    const RollbackFile* fy = file_at(c3.rp, c3.S, "y");
    old = open((L3 + "/y").c_str(), O_RDONLY);
    CHECK(g3.clear(old, c3.ids[(size_t)fy->layer], true, L3 + "/y") == VMIG_ESRCCHANGED && strstr(last_error_cstr(), "/y"));
    close(old);
    return 0;
}

int main(int argc, char** argv)
{
    if (argc != 2) { fprintf(stderr, "usage: rollback_unit DIR\n"); return 2; }
    g_dir = argv[1];
    if (actions() || restore_identity() || identity_checks() || rebuild_sequence()) return 1;
    printf("rollback unit ok\n");
    return 0;
}
