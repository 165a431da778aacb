// select_unit.cpp -- CPU unit test of the host side of vmig_restore_paths (csrc/vmig_select.cpp; compiled and run by
// tests/test_restore_paths_host.py), on real files:
//   - the selection walk never lists or reads a sibling of a chosen path, nor a directory of a parent chain (their atime
//     stays put), and finds exactly the chosen entries and what lies beneath the chosen directories;
//   - a path whose parent chain is not a chain of real directories, or that VMIG_F_SKIP_HIDDEN_TOPDIRS hides, is not found;
//   - hard-link groups form inside the selection only;
//   - the table subset and its merge report missing, extra and resized paths inside the selection and ignore
//     mismatches outside it; its hashes are the table's;
//   - parent-chain preparation replaces a symlink, a file and a whiteout (or FIFO) with a directory, leaves the
//     symlink's target untouched, keeps an existing directory as it is, and records what it created;
//   - awkward names (tab, newline, non-UTF-8 bytes) survive.
//   usage: select_unit DIR
#include "vmig_select.h"
#include "vmig_scrub.h"
#include "vmig_common.h"
#include <fcntl.h>
#include <unistd.h>
#include <dirent.h>
#include <sys/stat.h>
#include <sys/sysmacros.h>
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

static bool put(const std::string& p, uint64_t size, uint8_t fill) {
    const int fd = open(p.c_str(), O_WRONLY | O_CREAT | O_TRUNC, 0644);
    if (fd < 0) return false;
    std::vector<uint8_t> b(size, fill);
    const bool ok = size == 0 || pwrite(fd, b.data(), size, 0) == (ssize_t)size;
    return close(fd) == 0 && ok;
}
static bool mkdirs(const std::string& p) {
    for (size_t s = p.find('/', 1); ; s = p.find('/', s + 1)) {
        const std::string q = s == std::string::npos ? p : p.substr(0, s);
        if (mkdir(q.c_str(), 0755) != 0 && errno != EEXIST) return false;
        if (s == std::string::npos) return true;
    }
}
// atime of 1 s, mtime kept: any read or listing moves it forward (relatime updates an atime older than the mtime)
static bool age(const std::string& p) {
    struct timespec ts[2] = {{1, 0}, {0, UTIME_OMIT}};
    return utimensat(AT_FDCWD, p.c_str(), ts, AT_SYMLINK_NOFOLLOW) == 0;
}
static bool aged(const std::string& p) { struct stat st; return lstat(p.c_str(), &st) == 0 && st.st_atim.tv_sec == 1; }
static const Entry* find(const std::vector<Entry>& v, const std::string& rel) {
    for (const Entry& e : v) if (e.rel == rel) return &e;
    return nullptr;
}

static int walk_reads_only_the_selection(const std::string& dir) {
    const std::string s = dir + "/walk";
    CHECK(mkdirs(s + "/a/chosen_dir/deep") && mkdirs(s + "/a/sibdir") && mkdirs(s + "/other") && mkdirs(s + "/.hid"));
    CHECK(put(s + "/a/chosen.bin", 3 * kBB + 5, 1) && put(s + "/a/sib.bin", 100, 2) && put(s + "/a/sibdir/x", 10, 3));
    CHECK(put(s + "/a/chosen_dir/f1", kBB, 4) && put(s + "/a/chosen_dir/deep/f2", 7, 5) && put(s + "/other/y", 9, 6));
    CHECK(put(s + "/.hid/h", 3, 7) && symlink("a", (s + "/lnkdir").c_str()) == 0 && symlink("t", (s + "/a/chosen_dir/ln").c_str()) == 0);
    for (const char* p : {"", "/a", "/a/sib.bin", "/a/sibdir", "/a/sibdir/x", "/other", "/other/y"}) CHECK(age(s + p));
    Selection sel;
    CHECK(select_walk(s, {"a/chosen.bin", "a/chosen_dir"}, kBB, false, &sel) == VMIG_OK);
    for (const char* p : {"", "/a", "/a/sib.bin", "/a/sibdir", "/a/sibdir/x", "/other", "/other/y"}) CHECK(aged(s + p));
    CHECK(sel.not_found.empty());
    CHECK(sel.man.dirs.size() == 3 && sel.man.dirs[0].rel == "." && sel.man.dirs[1].rel == "a/chosen_dir" && sel.man.dirs[2].rel == "a/chosen_dir/deep");
    CHECK(sel.man.files.size() == 3);
    CHECK(sel.man.files[0].rel == "a/chosen.bin" && sel.man.files[1].rel == "a/chosen_dir/deep/f2" && sel.man.files[2].rel == "a/chosen_dir/f1");
    CHECK(sel.man.files[0].first_block == 0 && sel.man.files[0].n_blocks == 4 && sel.man.files[1].first_block == 4 && sel.man.files[2].first_block == 5);
    CHECK(sel.man.n_blocks == 6 && sel.man.bytes_total == 3 * kBB + 5 + 7 + kBB);
    CHECK(sel.man.symlinks.size() == 1 && sel.man.symlinks[0].rel == "a/chosen_dir/ln" && sel.man.symlinks[0].target == "t");
    CHECK(sel.parents.size() == 1 && sel.parents[0].rel == "a" && sel.parents[0].type == kDir);
    CHECK(sel.chosen_dirs.size() == 1 && sel.chosen_dirs[0] == "a/chosen_dir");

    // not found: a missing entry, a file as a parent, a symlink as a parent, a hidden top directory when skipped
    CHECK(select_walk(s, {"a/nothere", "a/chosen.bin/x", "lnkdir/sib.bin", ".hid", ".hid/h", "other/y"}, kBB, true, &sel) == VMIG_OK);
    CHECK(sel.not_found.size() == 5 && sel.man.files.size() == 1 && sel.man.files[0].rel == "other/y");
    CHECK(select_walk(s, {".hid/h", "lnkdir"}, kBB, false, &sel) == VMIG_OK);
    CHECK(sel.not_found.empty() && sel.man.files.size() == 1 && sel.man.symlinks.size() == 1 && sel.man.symlinks[0].rel == "lnkdir");
    return 0;
}

static int hard_links_inside_the_selection(const std::string& dir) {
    const std::string s = dir + "/hl";
    CHECK(mkdirs(s + "/h") && mkdirs(s + "/q"));
    CHECK(put(s + "/h/p1", kBB + 1, 1) && link((s + "/h/p1").c_str(), (s + "/h/p2").c_str()) == 0 && link((s + "/h/p1").c_str(), (s + "/q/p3").c_str()) == 0);
    Selection sel;
    CHECK(select_walk(s, {"h"}, kBB, false, &sel) == VMIG_OK && sel.man.files.size() == 2);
    CHECK(sel.man.files[0].hardlink_of == -1 && sel.man.files[1].hardlink_of == 0);
    CHECK(select_walk(s, {"h/p2", "q/p3"}, kBB, false, &sel) == VMIG_OK && sel.man.files.size() == 2);
    CHECK(sel.man.files[0].rel == "h/p2" && sel.man.files[0].hardlink_of == -1 && sel.man.files[1].hardlink_of == 0);
    CHECK(select_walk(s, {"q/p3"}, kBB, false, &sel) == VMIG_OK && sel.man.files.size() == 1 && sel.man.files[0].hardlink_of == -1);
    // the block layout counts every path, linked or not, as walk_tree does
    CHECK(select_walk(s, {"h", "q"}, kBB, false, &sel) == VMIG_OK && sel.man.files.size() == 3 && sel.man.n_blocks == 6);
    CHECK(sel.man.files[2].rel == "q/p3" && sel.man.files[2].hardlink_of == 0 && sel.man.files[2].first_block == 4);
    return 0;
}

static TableFile rec(const std::string& rel, uint64_t size, uint64_t first) { TableFile f; f.rel = rel; f.size = size; f.first_block = first; return f; }

static int table_subset_merge(const std::string& dir) {
    const std::string s = dir + "/tab";
    CHECK(mkdirs(s + "/a/d") && mkdirs(s + "/a-b") && mkdirs(s + "/z"));
    CHECK(put(s + "/a/ok", 2 * kBB, 1) && put(s + "/a/d/resized", 10, 2) && put(s + "/a/d/extra", 11, 3) && put(s + "/a-b/f", 5, 4) && put(s + "/z/f", 6, 5));
    BlockTable t; t.block_bytes = kBB;
    // bytewise order: "a-b/f" < "a/..." < "z/..."; outside the selection "a-b/f" is resized and "z/gone" is missing
    std::vector<TableFile> f = {rec("a-b/f", 99, 0), rec("a/d/gone", 3, 1), rec("a/d/resized", 12, 2), rec("a/ok", 2 * kBB, 3),
                                rec("z/f", 6, 5), rec("z/gone", 1, 6)};
    t.files = f;
    for (uint64_t i = 0; i < 7; i++) t.hashes.push_back(0x1000 + i);
    for (size_t i = 0; i < t.files.size(); i++) t.index[t.files[i].rel] = i;
    Selection sel;
    CHECK(select_walk(s, {"a", "z/f"}, kBB, false, &sel) == VMIG_OK && sel.not_found.empty());
    BlockTable part;
    table_subset(t, sel.paths, &part);
    CHECK(part.files.size() == 4 && part.files[0].rel == "a/d/gone" && part.files[3].rel == "z/f");
    CHECK(part.hashes.size() == 5 && part.hashes[0] == 0x1001 && part.files[2].first_block == 2 && part.hashes[2] == 0x1003 &&
          part.hashes[4] == 0x1005 && part.index.at("z/f") == 3);
    std::vector<int64_t> tab_of;
    std::vector<ScrubFinding> diff;
    CHECK(scrub_merge_table(0, sel.man, part, &tab_of, &diff) == 3);
    CHECK(diff[0].kind == kScrubExtra && diff[0].path == "a/d/extra");
    CHECK(diff[1].kind == kScrubMissing && diff[1].path == "a/d/gone");
    CHECK(diff[2].kind == kScrubResized && diff[2].path == "a/d/resized");
    // "z/f" and "a/ok" match; nothing outside the selection was reported
    CHECK(select_walk(s, {"a/ok", "z/f"}, kBB, false, &sel) == VMIG_OK);
    table_subset(t, sel.paths, &part);
    std::vector<ScrubFinding> none;
    CHECK(scrub_merge_table(0, sel.man, part, &tab_of, &none) == 0 && tab_of[0] == 0 && tab_of[1] == 1);
    // "missing" vs "not in the snapshot": a record at or beneath the path
    table_subset(t, {"a/d/gone"}, &part); CHECK(part.files.size() == 1);
    table_subset(t, {"z"}, &part); CHECK(part.files.size() == 2);
    table_subset(t, {"a/d/nothere"}, &part); CHECK(part.files.empty());
    table_subset(t, {"a-"}, &part); CHECK(part.files.empty());
    return 0;
}

static int parent_chains(const std::string& dir, bool root) {
    const std::string s = dir + "/pc_snap", d = dir + "/pc_dst", out = dir + "/outside";
    for (const char* p : {"/l", "/f", "/w", "/keep/x", "/new/deeper"}) CHECK(mkdirs(s + p));
    for (const char* p : {"/l/e", "/f/e", "/w/e", "/keep/x/e", "/new/deeper/e"}) CHECK(put(s + p, 1, 1));
    CHECK(mkdirs(d + "/keep") && mkdirs(out) && put(out + "/victim", 4, 9));
    CHECK(chmod((d + "/keep").c_str(), 0750) == 0);
    CHECK(symlink(out.c_str(), (d + "/l").c_str()) == 0 && put(d + "/f", 3, 3));
    if (root) CHECK(mknod((d + "/w").c_str(), S_IFCHR | 0644, makedev(0, 0)) == 0);     // an overlay whiteout
    else CHECK(mkfifo((d + "/w").c_str(), 0644) == 0);
    Selection sel;
    CHECK(select_walk(s, {"f/e", "keep/x/e", "l/e", "new/deeper/e", "w/e"}, kBB, false, &sel) == VMIG_OK && sel.not_found.empty());
    CHECK(sel.parents.size() == 7);
    CHECK(prepare_parents(d, &sel) == VMIG_OK);
    for (const char* p : {"/l", "/f", "/w", "/keep", "/keep/x", "/new", "/new/deeper"}) {
        struct stat st;
        CHECK(lstat((d + p).c_str(), &st) == 0 && S_ISDIR(st.st_mode));
    }
    struct stat st;
    CHECK(lstat((d + "/keep").c_str(), &st) == 0 && (st.st_mode & 07777) == 0750);
    // the symlink's target is untouched: still one entry, its own bytes
    DIR* od = opendir(out.c_str());
    int n = 0;
    while (struct dirent* de = readdir(od)) n += de->d_name[0] != '.';
    closedir(od);
    CHECK(n == 1 && lstat((out + "/victim").c_str(), &st) == 0 && st.st_size == 4);
    // every directory it created, parents first, right after "."; "keep" existed and is not among them
    const std::vector<std::string> want = {".", "f", "keep/x", "l", "new", "new/deeper", "w"};
    CHECK(sel.man.dirs.size() == want.size());
    for (size_t i = 0; i < want.size(); i++) CHECK(sel.man.dirs[i].rel == want[i]);
    CHECK(!find(sel.man.dirs, "keep"));
    return 0;
}

static int awkward_names(const std::string& dir) {
    const std::string s = dir + "/awk";
    const std::string tab = "t\tab", nl = "new\nline", bad = "bad\xff\xfe" "byte";
    CHECK(mkdirs(s + "/" + tab) && put(s + "/" + tab + "/" + nl, 5, 1) && put(s + "/" + bad, 6, 2) && put(s + "/" + tab + "/sib", 1, 3));
    const std::string second = tab + "/" + nl;
    const char* raw[] = {second.c_str(), bad.c_str()};
    std::vector<std::string> paths;
    CHECK(select_check_paths(2, raw, &paths) == VMIG_OK && paths.size() == 2 && paths[0] == bad && paths[1] == second);
    Selection sel;
    CHECK(select_walk(s, paths, kBB, false, &sel) == VMIG_OK && sel.not_found.empty());
    CHECK(sel.man.files.size() == 2 && sel.man.files[0].rel == bad && sel.man.files[1].rel == second);
    CHECK(sel.parents.size() == 1 && sel.parents[0].rel == tab);
    BlockTable t; t.block_bytes = kBB;
    t.files = {rec(bad, 6, 0), rec(tab + "/" + nl, 5, 1), rec(tab + "/sib", 1, 2)};
    t.hashes = {1, 2, 3};
    for (size_t i = 0; i < t.files.size(); i++) t.index[t.files[i].rel] = i;
    BlockTable part;
    table_subset(t, paths, &part);
    CHECK(part.files.size() == 2 && part.hashes[1] == 2);
    std::vector<int64_t> tab_of;
    std::vector<ScrubFinding> diff;
    CHECK(scrub_merge_table(0, sel.man, part, &tab_of, &diff) == 0);
    return 0;
}

int main(int argc, char** argv) {
    if (argc != 2) { fprintf(stderr, "usage: select_unit DIR\n"); return 2; }
    const std::string dir = argv[1];
    if (walk_reads_only_the_selection(dir)) return 1;
    if (hard_links_inside_the_selection(dir)) return 1;
    if (table_subset_merge(dir)) return 1;
    if (parent_chains(dir, geteuid() == 0)) return 1;
    if (awkward_names(dir)) return 1;
    printf("select unit ok\n");
    return 0;
}
