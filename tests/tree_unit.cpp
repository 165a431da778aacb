// tree_unit.cpp -- CPU unit test of the source-side path safety in csrc/vmig_tree.cpp (compiled and run by
// tests/test_host.py).  The source layer may belong to a running tenant: open_beneath() must refuse symlinks and
// escapes, the walk must not descend through a symlinked directory, remove_source() must not leave the tree.  The file
// backends' shared descriptor code: ReadFds opens a slot once, runs the caller's hook before publishing, and closes it
// after its last counted read; open_for_write / cut_to_size / close_written on the destination side.
//   g++ -std=c++17 -I gpu-docker-api_b200/csrc tests/tree_unit.cpp gpu-docker-api_b200/csrc/vmig_tree.cpp -o tree_unit
#include "vmig_tree.h"
#include "vmig_common.h"
#include <fcntl.h>
#include <unistd.h>
#include <cstdio>
#include <cstdlib>
#include <atomic>
#include <thread>
#include <string>
#include <vector>
#include <sys/stat.h>

namespace vmig {   // the three error-channel functions normally provided by vmig_engine.cu
static thread_local std::string g_err;
void set_last_error(const char* fmt, ...) { char b[1024]; va_list ap; va_start(ap, fmt); vsnprintf(b, sizeof b, fmt, ap); va_end(ap); g_err = b; }
void set_last_error_str(const std::string& s) { g_err = s; }
const char* last_error_cstr() { return g_err.c_str(); }
long env_long(const char* name, long d) { const char* v = getenv(name); return v && *v ? atol(v) : d; }
}
using namespace vmig;

#define CHECK_VOID(c) do { if (!(c)) { printf("FAIL line %d: %s\n", __LINE__, #c); exit(1); } } while (0)
#define CHECK(c) do { if (!(c)) { printf("FAIL line %d: %s   [last error: %s]\n", __LINE__, #c, last_error_cstr()); return 1; } } while (0)
static void put(const std::string& p, const char* s) { FILE* f = fopen(p.c_str(), "w"); fputs(s, f); fclose(f); }
static std::string get(int fd) { char b[64] = {0}; ssize_t n = read(fd, b, 63); close(fd); return std::string(b, n > 0 ? (size_t)n : 0); }
static bool is_open(int fd) { return fcntl(fd, F_GETFD) != -1; }
static std::string pget(int fd) { char b[64] = {0}; ssize_t n = pread(fd, b, 63, 0); return std::string(b, n > 0 ? (size_t)n : 0); }

static int read_fds(const std::string& base) {
    const std::string root = base + "/rfd";
    CHECK(system(("mkdir -p " + root).c_str()) == 0);
    put(root + "/a", "alpha"); put(root + "/b", "bravo");
    const int rfd = open(root.c_str(), O_RDONLY | O_DIRECTORY);
    CHECK(rfd >= 0);
    auto accept = [](int*, const struct stat* st, bool) { return st ? VMIG_OK : VMIG_EIO; };
    {   // eight threads ask for one slot at once: one open, one hook call, one descriptor for all
        ReadFds t; t.init(1); t.add_reads(0, 8);
        std::atomic<int> hooks{0}, go{0};
        std::vector<int> got(8, -1);
        std::vector<std::thread> th;
        for (int i = 0; i < 8; i++)
            th.emplace_back([&, i] {
                while (!go.load()) {}
                t.get(0, rfd, "a", false, [&](int*, const struct stat*, bool) { hooks++; std::this_thread::sleep_for(std::chrono::milliseconds(20)); return VMIG_OK; }, &got[i]);
            });
        go = 1;
        for (auto& x : th) x.join();
        CHECK(hooks.load() == 1 && got[0] >= 0 && pget(got[0]) == "alpha");
        for (int fd : got) CHECK(fd == got[0]);
        CHECK(t.n_direct.load() == 0 && !t.direct(0));
    }
    {   // closed exactly after the last counted read, before_close first and only then
        ReadFds t; t.init(2); t.add_reads(1, 3);
        int fd = -1, before = 0;
        CHECK(t.get(1, rfd, "b", false, accept, &fd) == VMIG_OK && pget(fd) == "bravo");
        for (int r = 0; r < 3; r++) {
            CHECK(is_open(fd));
            t.read_done(1, [&](int c) { before++; CHECK_VOID(c == fd && is_open(c)); });
        }
        CHECK(before == 1 && !is_open(fd));
    }
    {   // a refusal closes the new descriptor and leaves the slot empty: the next get opens again
        ReadFds t; t.init(1); t.add_reads(0, 1);
        int seen = -1, fd = -1, hooks = 0;
        CHECK(t.get(0, rfd, "a", false, [&](int* f, const struct stat*, bool) { hooks++; seen = *f; return VMIG_ESRCCHANGED; }, &fd) == VMIG_ESRCCHANGED);
        CHECK(seen >= 0 && !is_open(seen) && fd == -1);
        CHECK(t.get(0, rfd, "a", false, [&](int*, const struct stat*, bool) { hooks++; return VMIG_OK; }, &fd) == VMIG_OK);
        CHECK(hooks == 2 && pget(fd) == "alpha");
        t.read_done(0);
        CHECK(!is_open(fd));
    }
    {   // a hook that replaces the descriptor has the replacement published, and later closed
        ReadFds t; t.init(1); t.add_reads(0, 2);
        int orig = -1, repl = -1, fd = -1;
        CHECK(t.get(0, rfd, "a", false, [&](int* f, const struct stat* st, bool) {
            struct stat bs;
            if (!st || stat((root + "/a").c_str(), &bs) != 0 || st->st_ino != bs.st_ino) return VMIG_EIO;    // st is the opened file's
            orig = *f; repl = open((root + "/b").c_str(), O_RDONLY); close(*f); *f = repl;
            return VMIG_OK;
        }, &fd) == VMIG_OK);
        CHECK(fd == repl && fd != orig && pget(fd) == "bravo");
        int again = -1;
        CHECK(t.get(0, rfd, "a", false, [](int*, const struct stat*, bool) { return VMIG_EIO; }, &again) == VMIG_OK && again == repl);
        t.read_done(0); CHECK(is_open(repl));
        t.read_done(0); CHECK(!is_open(repl));
    }
    {   // close_all closes what is still open (a failed pass), and the direct flag is what the open really got
        ReadFds t; t.init(3);
        for (size_t i = 0; i < 3; i++) t.add_reads(i, 5);
        int a = -1, b = -1;
        bool hook_direct = false;
        CHECK(t.get(0, rfd, "a", false, accept, &a) == VMIG_OK && !t.direct(0));
        CHECK(t.get(2, rfd, "b", true, [&](int*, const struct stat*, bool d) { hook_direct = d; return VMIG_OK; }, &b) == VMIG_OK);
        CHECK(t.direct(2) == hook_direct && t.direct(2) == ((fcntl(b, F_GETFL) & O_DIRECT) != 0) && t.n_direct.load() == (t.direct(2) ? 1u : 0u));
        t.close_all();
        CHECK(!is_open(a) && !is_open(b));
    }
    close(rfd);
    return 0;
}

static int dst_open(const std::string& base) {
    const std::string dir = base + "/dst";
    CHECK(system(("mkdir -p " + dir).c_str()) == 0);
    const std::string p = dir + "/new";
    bool direct = true;
    int fd = open_for_write(p, true, false, &direct);                  // create: a new 0600 file, no O_DIRECT unless asked
    struct stat st;
    CHECK(fd >= 0 && !direct && (fcntl(fd, F_GETFL) & O_DIRECT) == 0);
    CHECK(fstat(fd, &st) == 0 && (st.st_mode & 07777) == 0600 && st.st_size == 0);
    CHECK(pwrite(fd, "0123456789", 10, 0) == 10);
    CHECK(close_written(fd, VMIG_OK, p) == VMIG_OK);
    direct = true;
    CHECK(open_for_write(p, true, false, &direct) == -1 && errno == EEXIST && !direct);    // O_EXCL: an existing path is not taken
    CHECK(open_for_write(p, true, true, &direct) == -1 && errno == EEXIST && !direct);
    fd = open_for_write(p, false, false, &direct);                      // in place: no truncate
    CHECK(fd >= 0 && !direct && get(open(p.c_str(), O_RDONLY)) == "0123456789");
    CHECK(pwrite(fd, "ab", 2, 0) == 2);
    CHECK(cut_to_size(fd, 4, p) == VMIG_OK && fstat(fd, &st) == 0 && st.st_size == 4);
    CHECK(close_written(fd, VMIG_OK, p) == VMIG_OK);
    FILE* f = fopen(p.c_str(), "r"); char b[16] = {0}; CHECK(f && fread(b, 1, sizeof b, f) == 4); fclose(f);
    CHECK(std::string(b) == "ab23");
    CHECK(open_for_write(dir + "/missing", false, false, &direct) == -1 && errno == ENOENT);
    CHECK(symlink("new", (dir + "/sl").c_str()) == 0);
    CHECK(open_for_write(dir + "/sl", false, false, &direct) == -1);   // never through a symlink
    fd = open_for_write(dir + "/d", true, true, &direct);               // asked: reported as the descriptor really is
    CHECK(fd >= 0 && direct == ((fcntl(fd, F_GETFL) & O_DIRECT) != 0));
    CHECK(close_written(fd, VMIG_OK, dir + "/d") == VMIG_OK);
    // a failed close is the call's error only when it has none yet
    CHECK(close_written(fd, VMIG_OK, dir + "/d") == VMIG_EIO && std::string(last_error_cstr()).find("close " + dir + "/d") == 0);
    CHECK(close_written(fd, VMIG_ESRCCHANGED, dir + "/d") == VMIG_ESRCCHANGED);
    return 0;
}

int main(int argc, char** argv) {
    if (argc < 2) return 2;
    const std::string base = argv[1], root = base + "/root", outside = base + "/outside";
    if (read_fds(base) || dst_open(base)) return 1;
    CHECK(system(("mkdir -p " + root + "/a/b " + root + "/victim " + outside).c_str()) == 0);
    put(root + "/a/b/file", "inside"); put(root + "/victim/f", "inside2"); put(outside + "/f", "SECRET"); put(outside + "/secret", "SECRET");
    CHECK(symlink(outside.c_str(), (root + "/a/link").c_str()) == 0);
    CHECK(symlink("b/file", (root + "/a/sl").c_str()) == 0);
    const int rfd = open(root.c_str(), O_RDONLY | O_DIRECTORY);
    CHECK(rfd >= 0);
    int fd = -1;
    CHECK(open_beneath(rfd, "a/b/file", O_RDONLY, &fd) == VMIG_OK && get(fd) == "inside");
    CHECK(open_beneath(rfd, "a/link/secret", O_RDONLY, &fd) == VMIG_ESRCCHANGED);        // symlinked directory on the way
    CHECK(open_beneath(rfd, "a/sl", O_RDONLY, &fd) == VMIG_ESRCCHANGED);                 // symlink as the last component
    CHECK(open_beneath(rfd, "../outside/secret", O_RDONLY, &fd) != VMIG_OK);             // lexical escape
    CHECK(open_beneath(rfd, "/etc/passwd", O_RDONLY, &fd) == VMIG_EINVAL);               // absolute
    CHECK(open_beneath(rfd, "a/missing", O_RDONLY, &fd) == VMIG_ESRCCHANGED);            // vanished since the walk

    // the same through the component-wise fallback used on kernels without openat2
    CHECK(open_beneath_walk(rfd, "a/b/file", O_RDONLY, &fd) == VMIG_OK && get(fd) == "inside");
    CHECK(open_beneath_walk(rfd, "a/link/secret", O_RDONLY, &fd) == VMIG_ESRCCHANGED);
    CHECK(open_beneath_walk(rfd, "a/sl", O_RDONLY, &fd) == VMIG_ESRCCHANGED);
    CHECK(open_beneath_walk(rfd, "../outside/secret", O_RDONLY, &fd) == VMIG_EINVAL);
    CHECK(open_beneath_walk(rfd, "a/missing", O_RDONLY, &fd) == VMIG_ESRCCHANGED);

    Manifest m;
    CHECK(walk_tree(root, 4096, false, &m) == VMIG_OK);
    CHECK(m.files.size() == 2 && m.symlinks.size() == 2 && m.dirs.size() == 4);          // ".", a, a/b, victim; nothing from outside/
    for (auto& e : m.files) CHECK(e.rel == "a/b/file" || e.rel == "victim/f");

    // the tenant swaps victim/ for a symlink to outside/ after the walk: the file must not be reachable any more,
    // and a move's clean-up must not delete outside/f
    CHECK(rename((root + "/victim").c_str(), (root + "/victim.bak").c_str()) == 0);
    CHECK(symlink(outside.c_str(), (root + "/victim").c_str()) == 0);
    CHECK(open_beneath(rfd, "victim/f", O_RDONLY, &fd) == VMIG_ESRCCHANGED);
    CHECK(remove_source(root, m) != VMIG_OK);
    CHECK(access((outside + "/f").c_str(), F_OK) == 0);
    close(rfd);

    // ---- VMIG_F_PRUNE: prune_extras() removes exactly what the manifest does not list, by descriptor, never through a symlink
    {
        const std::string psrc = base + "/psrc", pdst = base + "/pdst";
        CHECK(system(("mkdir -p " + psrc + "/keep/sub " + pdst + "/keep/sub " + pdst + "/gone/deep " + pdst + "/keep/extra_dir").c_str()) == 0);
        put(psrc + "/keep/f", "1"); put(psrc + "/keep/sub/g", "2"); put(psrc + "/top", "3");
        CHECK(symlink("keep/f", (psrc + "/ln").c_str()) == 0);
        put(pdst + "/keep/f", "old"); put(pdst + "/keep/sub/g", "old"); put(pdst + "/top", "old"); CHECK(symlink("keep/f", (pdst + "/ln").c_str()) == 0);
        put(pdst + "/gone/deep/x", "x"); put(pdst + "/keep/stale", "s"); put(pdst + "/keep/extra_dir/y", "y");
        CHECK(symlink(outside.c_str(), (pdst + "/escape").c_str()) == 0);                 // an extra that points out of the tree
        CHECK(symlink(outside.c_str(), (pdst + "/gone/deep/esc2").c_str()) == 0);
        Manifest pm;
        CHECK(walk_tree(psrc, 4096, false, &pm) == VMIG_OK);
        uint64_t n = 0;
        CHECK(prune_extras(pdst, pm, true, &n) == VMIG_OK && n == 4);                     // dry run: gone/, keep/stale, keep/extra_dir/, escape
        CHECK(access((pdst + "/gone/deep/x").c_str(), F_OK) == 0);                        // ... and nothing was touched
        CHECK(prune_extras(pdst, pm, false, &n) == VMIG_OK);
        CHECK(n == 8);                          // gone/deep/{x,esc2}, gone/deep, gone, keep/stale, keep/extra_dir/y, keep/extra_dir, escape
        CHECK(access((pdst + "/gone").c_str(), F_OK) != 0 && access((pdst + "/keep/stale").c_str(), F_OK) != 0 && access((pdst + "/keep/extra_dir").c_str(), F_OK) != 0);
        struct stat lst; CHECK(lstat((pdst + "/escape").c_str(), &lst) != 0);
        CHECK(access((outside + "/f").c_str(), F_OK) == 0 && access((outside + "/secret").c_str(), F_OK) == 0);   // the symlinks were unlinked, not followed
        CHECK(access((pdst + "/keep/sub/g").c_str(), F_OK) == 0 && access((pdst + "/top").c_str(), F_OK) == 0 && lstat((pdst + "/ln").c_str(), &lst) == 0);
        CHECK(prune_extras(pdst, pm, true, &n) == VMIG_OK && n == 0);
        // an entry that changed TYPE since the destination was written is in the way and goes too: a file where the source
        // now has a directory, a directory (with content) where the source now has a file, a directory where it has a symlink
        CHECK(system(("mkdir -p " + psrc + "/flip_dir " + pdst + "/flip_file/inner " + pdst + "/ln2").c_str()) == 0);
        put(psrc + "/flip_file", "now a file"); put(pdst + "/flip_dir", "was a file"); put(pdst + "/flip_file/inner/z", "z");
        CHECK(symlink("top", (psrc + "/ln2").c_str()) == 0);
        CHECK(walk_tree(psrc, 4096, false, &pm) == VMIG_OK);
        CHECK(prune_extras(pdst, pm, false, &n) == VMIG_OK && n == 5);            // flip_dir (file), flip_file/{inner/z, inner}, flip_file, ln2 (dir)
        struct stat fst;
        CHECK(lstat((pdst + "/flip_dir").c_str(), &fst) != 0 && lstat((pdst + "/flip_file").c_str(), &fst) != 0 && lstat((pdst + "/ln2").c_str(), &fst) != 0);
        CHECK(make_dirs(pdst, pm) == VMIG_OK && lstat((pdst + "/flip_dir").c_str(), &fst) == 0 && S_ISDIR(fst.st_mode));
    }

    // ---- the walk is the same whether the root's sub-directories are taken by one thread or by eight
    {
        const std::string w = base + "/wide";
        CHECK(system(("mkdir -p " + w).c_str()) == 0);
        for (int d = 0; d < 11; d++) {
            const std::string dd = w + "/d" + std::to_string(d);
            CHECK(system(("mkdir -p " + dd + "/x/y").c_str()) == 0);
            for (int f = 0; f < 7; f++) put(dd + (f % 2 ? "/x/y/f" : "/f") + std::to_string(f), "data");
            CHECK(symlink("f0", (dd + "/sl").c_str()) == 0);
        }
        CHECK(link((w + "/d3/f0").c_str(), (w + "/d9/hard").c_str()) == 0);               // a hard-link pair across two sub-walks
        Manifest a, b;
        setenv("VMIG_WALK_THREADS", "1", 1); CHECK(walk_tree(w, 4096, false, &a) == VMIG_OK);
        setenv("VMIG_WALK_THREADS", "8", 1); CHECK(walk_tree(w, 4096, false, &b) == VMIG_OK);
        CHECK(a.dirs.size() == b.dirs.size() && a.files.size() == b.files.size() && a.symlinks.size() == b.symlinks.size() && a.files.size() == 78);
        for (size_t i = 0; i < a.dirs.size(); i++) CHECK(a.dirs[i].rel == b.dirs[i].rel);
        for (size_t i = 0; i < a.files.size(); i++) CHECK(a.files[i].rel == b.files[i].rel && a.files[i].hardlink_of == b.files[i].hardlink_of && a.files[i].first_block == b.files[i].first_block);
        for (size_t i = 0; i < a.symlinks.size(); i++) CHECK(a.symlinks[i].rel == b.symlinks[i].rel);
        int links = 0; for (auto& e : b.files) if (e.hardlink_of >= 0) { links++; CHECK(b.files[(size_t)e.hardlink_of].rel == "d3/f0" && e.rel == "d9/hard"); }
        CHECK(links == 1);
    }
    {
        // the metadata policy reads the umask without changing it: a thread watching the process umask while policies are
        // built never sees another value (a set-and-restore read showed 0 to calls running at the same time)
        const mode_t old = umask(027);
        std::atomic<bool> stop{false}; std::atomic<int> other{0};
        std::thread watch([&] {
            while (!stop.load()) {
                FILE* f = fopen("/proc/self/status", "r"); char line[256]; unsigned um = 027;
                while (f && fgets(line, sizeof line, f)) if (sscanf(line, "Umask: %o", &um) == 1) break;
                if (f) fclose(f);
                if (um != 027) other++;
            }
        });
        bool all = true;
        for (int i = 0; i < 20000; i++) all = all && default_meta_policy(0).umask_bits == 027;
        stop = true; watch.join();
        umask(old);
        CHECK(all && other.load() == 0);
    }
    printf("tree unit ok\n");
    return 0;
}
