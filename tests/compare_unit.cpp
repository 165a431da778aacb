// compare_unit.cpp -- CPU unit test of the host side of vmig_compare_snapshot (csrc/vmig_compare.cpp; compiled with g++
// alone and run by tests/test_compare_host.py) over real trees walked by walk_tree:
//   - the finding for every pair of entry kinds at one path, and the entries beneath a directory on one side only;
//   - sort order (path bytewise, then kind, then block) and the mtime precision rule;
//   - hard-link groups, including a link held outside the tree, which is no finding;
//   - the read plan: shared inode, trusted record, stale record, hard-linked paths without identity, layer-only files;
//   - bytes_restore.
//   usage: compare_unit DIR
#include "vmig_compare.h"
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

static const uint32_t kBB = 4096;
static std::string g_dir;

static void put(const std::string& p, size_t n, char c) {
    std::string b(n, c);
    const int fd = open(p.c_str(), O_WRONLY | O_CREAT | O_TRUNC, 0644);
    if (fd < 0 || write(fd, b.data(), b.size()) != (ssize_t)b.size()) { perror(p.c_str()); exit(2); }
    close(fd);
}
static void mtime(const std::string& p, time_t s, long ns) {
    struct timespec ts[2] = {{s, ns}, {s, ns}};
    if (utimensat(AT_FDCWD, p.c_str(), ts, AT_SYMLINK_NOFOLLOW) != 0) { perror(p.c_str()); exit(2); }
}
static void make(const std::string& p, char kind) {
    switch (kind) {
    case 'f': put(p, 100, 'k'); break;
    case 'd': mkdir(p.c_str(), 0755); put(p + "/child", 10, 'c'); break;
    case 'l': if (symlink("target", p.c_str())) perror(p.c_str()); break;
    case 'p': if (mkfifo(p.c_str(), 0644)) perror(p.c_str()); break;
    }
}
static std::string fresh(const std::string& name) {
    const std::string d = g_dir + "/" + name;
    mkdir(d.c_str(), 0755);
    return d;
}
// every path's and finding's times pinned, so that only what a case sets differs
static void pin_times(const std::string& root, const Manifest& m) {
    for (const auto* v : {&m.files, &m.symlinks, &m.specials, &m.dirs})
        for (const Entry& e : *v) mtime(pjoin(root, e.rel), 1000000, 0);
}
static int walk(const std::string& root, Manifest* m) { return walk_tree(root, kBB, false, m); }
// hashes where every block of a path hashes to the same thing in both trees unless `bump` names the file
static std::vector<uint64_t> hashes_of(const Manifest& m, const std::string& bump = "", uint64_t bump_block = 0) {
    std::vector<uint64_t> h(m.n_blocks);
    for (const Entry& e : m.files)
        for (uint64_t r = 0; r < e.n_blocks; r++) h[e.first_block + r] = 1000 * r + 7 + ((e.rel == bump && r == bump_block) ? 1 : 0);
    return h;
}
static std::vector<const uint64_t*> ptrs(const Manifest& m, const std::vector<uint64_t>& h) {
    std::vector<const uint64_t*> p;
    for (const Entry& e : m.files) p.push_back(h.data() + e.first_block);
    return p;
}
static const CompareFinding* find(const std::vector<CompareFinding>& v, CompareKind k, const std::string& path, int64_t block = -1) {
    for (const CompareFinding& f : v) if (f.kind == k && f.path == path && f.block == block) return &f;
    return nullptr;
}

static int kinds() {
    const std::string L = fresh("kinds_l"), S = fresh("kinds_s");
    const char ks[] = {'f', 'd', 'l', 'p'};
    for (char a : ks)
        for (char b : ks) {
            const std::string n = std::string("k_") + a + "_" + b;
            make(L + "/" + n, a); make(S + "/" + n, b);
        }
    make(L + "/only_l", 'd'); make(S + "/only_s", 'f');
    Manifest ml, ms;
    CHECK(walk(L, &ml) == VMIG_OK && walk(S, &ms) == VMIG_OK);
    pin_times(L, ml); pin_times(S, ms);
    CHECK(walk(L, &ml) == VMIG_OK && walk(S, &ms) == VMIG_OK);
    const std::vector<uint64_t> hl = hashes_of(ml), hs = hashes_of(ms);
    std::vector<CompareFinding> f;
    CompareCounts c;
    compare_merge(ml, ms, hs, ptrs(ml, hl), kBB, false, false, &f, &c);
    for (char a : ks)
        for (char b : ks) {
            const std::string n = std::string("k_") + a + "_" + b;
            if (a == b) { CHECK(!find(f, kCmpType, n)); continue; }
            const CompareFinding* t = find(f, kCmpType, n);
            CHECK(t && t->layer == std::string(1, a) && t->snap == std::string(1, b));
            if (a == 'd') CHECK(find(f, kCmpAdded, n + "/child"));
            if (b == 'd') CHECK(find(f, kCmpRemoved, n + "/child"));
        }
    CHECK(find(f, kCmpAdded, "only_l") && find(f, kCmpAdded, "only_l/child") && find(f, kCmpRemoved, "only_s"));
    // 12 type changes; added: only_l, its child, and the 3 children of k_d_*; removed likewise
    CHECK(c.paths_changed == 12 && c.paths_added == 2 + 3 && c.paths_removed == 1 + 3);
    CHECK(c.files_changed == 0 && c.blocks_changed == 0);
    // bytes_restore: every snapshot regular file the layer has no regular file for: k_{d,l,p}_f (100 each),
    // the children of k_{f,l,p}_d (10 each), only_s (100)
    CHECK(c.bytes_restore == 3 * 100 + 3 * 10 + 100);
    CHECK(f.size() == 12 + 5 + 4);
    return 0;
}

static int order_and_mtime() {
    const std::string L = fresh("ord_l"), S = fresh("ord_s");
    put(L + "/x", 3 * kBB, 'a'); put(S + "/x", 2 * kBB + 5, 'a');       // resized, blocks 1 and 2 (length) differ
    put(L + "/a-b", 10, 'a'); put(S + "/a-b", 10, 'a');                    // '-' sorts before '/'
    mkdir((L + "/a").c_str(), 0755); mkdir((S + "/a").c_str(), 0755);
    put(L + "/a/b", 10, 'a'); put(S + "/a/b", 10, 'a');
    const std::string sl = L + "/ln", ss = S + "/ln";
    if (symlink("one\ttwo", sl.c_str()) || symlink("three", ss.c_str())) return 1;
    Manifest ml, ms;
    CHECK(walk(L, &ml) == VMIG_OK && walk(S, &ms) == VMIG_OK);
    pin_times(L, ml); pin_times(S, ms);
    chmod((L + "/x").c_str(), 0600); chmod((S + "/x").c_str(), 0644);
    mtime(L + "/x", 2000000, 0);
    mtime(L + "/a-b", 1000000, 5);                                         // sub-second only
    mtime(L + "/a/b", 1000000, 0); mtime(S + "/a/b", 1000000, 0);
    CHECK(walk(L, &ml) == VMIG_OK && walk(S, &ms) == VMIG_OK);
    const std::vector<uint64_t> hl = hashes_of(ml, "x", 1), hs = hashes_of(ms);
    std::vector<CompareFinding> f;
    CompareCounts c;
    compare_merge(ml, ms, hs, ptrs(ml, hl), kBB, false, false, &f, &c);
    std::string got;
    for (const CompareFinding& x : f) got += compare_format(x);
    CHECK(got ==
          "target\tln\t-\tone\\ttwo\tthree\n"
          "resized\tx\t-\t12288\t8197\n"
          "block\tx\t1\t00000000000003f0\t00000000000003ef\n"
          "block\tx\t2\t00000000000007d7\t00000000000007d7\n"
          "mode\tx\t-\t0600\t0644\n"
          "mtime\tx\t-\t2000000\t1000000\n");
    CHECK(c.files_changed == 1 && c.blocks_changed == 2 && c.paths_changed == 2);
    CHECK(c.bytes_restore == kBB + 5);                                     // snapshot blocks 1 (4096) and 2 (5 bytes)
    compare_merge(ml, ms, hs, ptrs(ml, hl), kBB, true, false, &f, &c);
    got.clear();
    for (const CompareFinding& x : f) got += compare_format(x);
    CHECK(f.front().path == "a-b" && f.front().kind == kCmpMtime);
    CHECK(got.find("mtime\ta-b\t-\t1000000.000000005\t1000000.000000000\n") == 0);
    CHECK(got.find("mtime\tx\t-\t2000000.000000000\t1000000.000000000\n") != std::string::npos);
    CHECK(!find(f, kCmpMtime, "a/b") && !find(f, kCmpMtime, "."));
    compare_merge(ml, ms, hs, ptrs(ml, hl), kBB, true, true, &f, &c);      // VMIG_F_NO_METADATA
    CHECK(f.size() == 4 && !find(f, kCmpMode, "x") && !find(f, kCmpMtime, "x"));
    return 0;
}

static int hardlinks() {
    const std::string L = fresh("hl_l"), S = fresh("hl_s"), O = fresh("hl_outside");
    for (const std::string& r : {L, S}) for (const char* n : {"a", "b", "c", "d", "e"}) put(r + "/" + n, 100, 'h');
    // layer: {a, b} one inode, c alone; snapshot: a, b alone, {c, d} one inode; e linked outside the snapshot tree
    unlink((L + "/b").c_str()); if (link((L + "/a").c_str(), (L + "/b").c_str())) return 1;
    unlink((S + "/d").c_str()); if (link((S + "/c").c_str(), (S + "/d").c_str())) return 1;
    if (link((S + "/e").c_str(), (O + "/e").c_str())) return 1;
    Manifest ml, ms;
    CHECK(walk(L, &ml) == VMIG_OK && walk(S, &ms) == VMIG_OK);
    pin_times(L, ml); pin_times(S, ms);
    CHECK(walk(L, &ml) == VMIG_OK && walk(S, &ms) == VMIG_OK);
    const std::vector<uint64_t> hl = hashes_of(ml), hs = hashes_of(ms);
    std::vector<CompareFinding> f;
    CompareCounts c;
    compare_merge(ml, ms, hs, ptrs(ml, hl), kBB, false, false, &f, &c);
    std::string got;
    for (const CompareFinding& x : f) got += compare_format(x);
    CHECK(got ==
          "hardlink\ta\t-\ta\t-\n"
          "hardlink\tb\t-\ta\t-\n"
          "hardlink\tc\t-\t-\tc\n"
          "hardlink\td\t-\t-\tc\n");
    CHECK(c.paths_changed == 4 && c.bytes_restore == 0);
    return 0;
}

static int read_plan() {
    const std::string L = fresh("plan_l"), S = fresh("plan_s");
    for (const char* n : {"shared", "trusted", "stale", "h1", "h2", "empty_l", "grown"}) put(S + "/" + n, 2 * kBB, 's');
    put(S + "/empty_s", 0, 's');
    if (link((S + "/shared").c_str(), (L + "/shared").c_str())) return 1;
    put(L + "/trusted", 2 * kBB, 't'); put(L + "/stale", 2 * kBB, 't');
    put(L + "/h1", kBB + 1, 'h'); if (link((L + "/h1").c_str(), (L + "/h2").c_str())) return 1;
    put(L + "/empty_l", 0, 'e'); put(L + "/empty_s", 100, 'e'); put(L + "/grown", 3 * kBB, 'g'); put(L + "/only_l", 50, 'o');
    Manifest ml, ms;
    CHECK(walk(L, &ml) == VMIG_OK && walk(S, &ms) == VMIG_OK);
    // the layer's table: trusted is recorded as it is, stale with another ctime, h1/h2 without identity (hard links)
    BlockTable t; t.block_bytes = kBB;
    for (const Entry& e : ml.files) {
        struct stat st;
        CHECK(lstat(pjoin(L, e.rel).c_str(), &st) == 0);
        TableFile r{e.rel, e.size, t.hashes.size(), 0, 0};
        if (e.rel == "trusted" || e.rel == "stale") { r.ino = st.st_ino; r.ctime_ns = ctime_ns(st) + (e.rel == "stale" ? 1 : 0); }
        t.index[e.rel] = t.files.size();
        t.files.push_back(r);
        for (uint64_t b = 0; b < e.n_blocks; b++) t.hashes.push_back(5000 + b);
    }
    ComparePlan p;
    CHECK(compare_plan(L, ml, ms, &t, kBB, &p) == VMIG_OK);
    auto src = [&](const char* rel) {
        for (size_t i = 0; i < ml.files.size(); i++) if (ml.files[i].rel == rel) return (int)p.source[i];
        return -1;
    };
    CHECK(src("shared") == kCmpShared && src("trusted") == kCmpTrusted && src("stale") == kCmpRead);
    CHECK(src("h1") == kCmpRead && src("h2") == kCmpRead && src("grown") == kCmpRead);
    CHECK(src("empty_l") == kCmpNone && src("empty_s") == kCmpNone && src("only_l") == kCmpNone);
    CHECK(p.files_shared == 1 && p.files_trusted == 1);
    CHECK(p.inodes.size() == 3);                                  // stale, grown, and h1/h2 once
    CHECK(p.bytes_read == 2 * kBB + 3 * kBB + kBB + 1 && p.blocks_read == 2 + 3 + 2);
    // without the table, trusted is read too
    ComparePlan q;
    CHECK(compare_plan(L, ml, ms, nullptr, kBB, &q) == VMIG_OK && q.files_trusted == 0 && q.files_shared == 1 && q.inodes.size() == 4);
    // hashes: shared from the snapshot's table, trusted from the layer's, the rest from the read
    const std::vector<uint64_t> hs = hashes_of(ms);
    std::vector<uint64_t> rd(p.blocks_read, 7);
    const std::vector<const uint64_t*> lh = compare_layer_hashes(p, ml, ms, hs, &t, rd);
    for (size_t i = 0; i < ml.files.size(); i++) {
        const std::string& r = ml.files[i].rel;
        if (r == "shared") CHECK(lh[i] == hs.data() + ms.files[(size_t)p.snap_of[i]].first_block);
        else if (r == "trusted") CHECK(lh[i][0] == 5000 && lh[i][1] == 5001);
        else if (p.source[i] == kCmpRead) CHECK(lh[i][0] == 7);
        else CHECK(lh[i] == nullptr);
    }
    // bytes_restore: a read block hashes 7, which is the snapshot's block 0 (7 + 1000 r), so block 1 of stale, grown, h1
    // and h2 differs (4096 each); both of trusted's blocks differ (5000 + r); empty_l has no layer block (8192); shared
    // and grown's third layer block, past the snapshot's, bring back nothing
    std::vector<CompareFinding> f;
    CompareCounts c;
    compare_merge(ml, ms, hs, lh, kBB, false, true, &f, &c);
    CHECK(c.bytes_restore == 4 * kBB + 2 * kBB + 2 * kBB);
    CHECK(!find(f, kCmpBlock, "shared", 0) && find(f, kCmpBlock, "trusted", 0) && find(f, kCmpBlock, "h1", 1));
    CHECK(find(f, kCmpAdded, "only_l") && find(f, kCmpResized, "empty_l") && find(f, kCmpResized, "empty_s"));
    return 0;
}

int main(int argc, char** argv)
{
    if (argc != 2) { fprintf(stderr, "usage: compare_unit DIR\n"); return 2; }
    g_dir = argv[1];
    if (kinds() || order_and_mtime() || hardlinks() || read_plan()) return 1;
    printf("compare unit ok\n");
    return 0;
}
