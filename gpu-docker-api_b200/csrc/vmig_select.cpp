// vmig_select.cpp -- the host side of vmig_restore_paths (see vmig_select.h).
#include "vmig_select.h"
#include "vmig_common.h"

#include <fcntl.h>
#include <unistd.h>
#include <sys/stat.h>
#include <algorithm>
#include <iterator>
#include <map>
#include <unordered_set>

namespace vmig {

static std::vector<std::string> components(const std::string& p)
{
    std::vector<std::string> c;
    size_t pos = 0;
    for (;;) {
        const size_t slash = p.find('/', pos);
        c.push_back(p.substr(pos, slash == std::string::npos ? std::string::npos : slash - pos));
        if (slash == std::string::npos) return c;
        pos = slash + 1;
    }
}

int select_check_paths(uint32_t n, const char* const* paths, std::vector<std::string>* out)
{
    out->clear();
    if (n == 0) return fail(VMIG_EINVAL, "n_paths == 0: no path to restore");
    if (!paths) return fail(VMIG_EINVAL, "paths is NULL");
    std::map<std::string, uint32_t> index;
    for (uint32_t i = 0; i < n; i++) {
        if (!paths[i]) return fail(VMIG_EINVAL, "paths[%u] is NULL", i);
        const std::string p(paths[i]);
        if (p.empty()) return fail(VMIG_EINVAL, "paths[%u] is empty", i);
        if (p[0] == '/') return fail(VMIG_EINVAL, "paths[%u] '%s' is absolute: paths are relative to snap_dir", i, p.c_str());
        if (p.back() == '/') return fail(VMIG_EINVAL, "paths[%u] '%s' ends in '/'", i, p.c_str());
        for (const std::string& c : components(p))
            if (c.empty() || c == "." || c == "..")
                return fail(VMIG_EINVAL, "paths[%u] '%s' has an empty, '.' or '..' component", i, p.c_str());
        const auto ins = index.emplace(p, i);
        if (!ins.second) return fail(VMIG_EINVAL, "paths[%u] and paths[%u] are both '%s'", ins.first->second, i, p.c_str());
    }
    for (const auto& kv : index)
        for (size_t s = kv.first.find('/'); s != std::string::npos; s = kv.first.find('/', s + 1)) {
            const auto it = index.find(kv.first.substr(0, s));
            if (it != index.end())
                return fail(VMIG_EINVAL, "paths[%u] '%s' lies beneath paths[%u] '%s'", kv.second, kv.first.c_str(), it->second,
                            it->first.c_str());
        }
    for (const auto& kv : index) out->push_back(kv.first);        // std::map: bytewise order
    return VMIG_OK;
}

// One chosen path: its parent chain is lstat'ed and entered (never listed), the entry itself is added, and a directory's
// contents are walked by walk_tree.  *found = false when the snapshot's walk would not reach the path.
static int select_one(int rfd, const std::string& snap_root, const std::string& p, uint32_t block_bytes, bool skip_hidden_topdirs,
                      std::unordered_set<std::string>* parents_seen, Selection* out, bool* found, const std::atomic<int>* cancel)
{
    *found = false;
    const std::vector<std::string> comp = components(p);
    int cur = dup(rfd);
    if (cur < 0) return fail(VMIG_EIO, "dup: %s", errno_str(errno).c_str());
    std::string prefix;
    for (size_t i = 0; i + 1 < comp.size(); i++) {
        prefix = i ? prefix + "/" + comp[i] : comp[i];
        struct stat st;
        if (fstatat(cur, comp[i].c_str(), &st, AT_SYMLINK_NOFOLLOW) != 0) {
            const int e = errno; close(cur);
            return e == ENOENT ? VMIG_OK : fail(VMIG_EIO, "lstat %s/%s: %s", snap_root.c_str(), prefix.c_str(), errno_str(e).c_str());
        }
        if (!S_ISDIR(st.st_mode) || (skip_hidden_topdirs && i == 0 && comp[0][0] == '.')) { close(cur); return VMIG_OK; }
        if (parents_seen->insert(prefix).second) {
            Manifest one;
            manifest_add(cur, comp[i], prefix, st, block_bytes, &one);
            out->parents.push_back(one.dirs[0]);
        }
        const int nfd = openat(cur, comp[i].c_str(), O_RDONLY | O_DIRECTORY | O_NOFOLLOW | O_CLOEXEC);
        const int e = errno;
        close(cur);
        if (nfd < 0)
            return fail(e == ELOOP || e == ENOTDIR || e == ENOENT ? VMIG_ESRCCHANGED : VMIG_EIO, "open directory %s/%s: %s",
                        snap_root.c_str(), prefix.c_str(), errno_str(e).c_str());
        cur = nfd;
    }
    const std::string& name = comp.back();
    struct stat st;
    if (fstatat(cur, name.c_str(), &st, AT_SYMLINK_NOFOLLOW) != 0) {
        const int e = errno; close(cur);
        return e == ENOENT ? VMIG_OK : fail(VMIG_EIO, "lstat %s/%s: %s", snap_root.c_str(), p.c_str(), errno_str(e).c_str());
    }
    if (S_ISDIR(st.st_mode) && skip_hidden_topdirs && comp.size() == 1 && name[0] == '.') { close(cur); return VMIG_OK; }
    Manifest& m = out->man;
    int rc = manifest_add(cur, name, p, st, block_bytes, &m);
    close(cur);
    if (rc) return rc;
    *found = true;
    if (!S_ISDIR(st.st_mode)) return VMIG_OK;
    out->chosen_dirs.push_back(p);
    Manifest sub;
    rc = walk_tree(pjoin(snap_root, p), block_bytes, false, &sub, cancel);
    if (rc) return rc;
    auto move_under = [&](std::vector<Entry>& from, std::vector<Entry>& to, size_t first) {
        for (size_t i = first; i < from.size(); i++) { from[i].rel = p + "/" + from[i].rel; to.push_back(std::move(from[i])); }
    };
    move_under(sub.dirs, m.dirs, 1);               // sub.dirs[0] is the chosen directory itself, added above
    move_under(sub.files, m.files, 0);
    move_under(sub.symlinks, m.symlinks, 0);
    move_under(sub.specials, m.specials, 0);
    m.sockets_skipped += sub.sockets_skipped;
    return VMIG_OK;
}

int select_walk(const std::string& snap_root, const std::vector<std::string>& paths, uint32_t block_bytes,
                bool skip_hidden_topdirs, Selection* out, const std::atomic<int>* cancel)
{
    *out = Selection();
    out->paths = paths;
    struct stat rst;
    if (stat(snap_root.c_str(), &rst) != 0) return fail(VMIG_EIO, "stat %s: %s", snap_root.c_str(), errno_str(errno).c_str());
    if (!S_ISDIR(rst.st_mode)) return fail(VMIG_ENOTDIR, "%s is not a directory", snap_root.c_str());
    Entry root;
    root.rel = "."; root.type = kDir; root.mode = rst.st_mode; root.uid = rst.st_uid; root.gid = rst.st_gid;
    root.mtime = rst.st_mtim; root.atime = rst.st_atim;
    out->man.dirs.push_back(root);
    const int rfd = open(snap_root.c_str(), O_RDONLY | O_DIRECTORY | O_CLOEXEC);
    if (rfd < 0) return fail(VMIG_EIO, "open %s: %s", snap_root.c_str(), errno_str(errno).c_str());
    std::unordered_set<std::string> parents_seen;
    int rc = VMIG_OK;
    for (const std::string& p : paths) {
        if (cancel && cancel->load()) { rc = fail(VMIG_ECANCELED, "cancelled during the walk, before %s", p.c_str()); break; }
        bool found = false;
        rc = select_one(rfd, snap_root, p, block_bytes, skip_hidden_topdirs, &parents_seen, out, &found, cancel);
        if (rc) break;
        if (!found) out->not_found.push_back(p);
    }
    close(rfd);
    if (rc) return rc;
    // hard links are grouped inside the selection only: a path whose inode is also named outside it stands alone
    for (Entry& e : out->man.files) { e.hardlink_of = -1; e.target = inode_key(e.dev, e.ino); }
    finish_manifest(&out->man);
    return VMIG_OK;
}

void table_subset(const BlockTable& t, const std::vector<std::string>& paths, BlockTable* out)
{
    *out = BlockTable();
    out->block_bytes = t.block_bytes; out->algo = t.algo;
    auto at = [&](const std::string& rel) {
        return (size_t)(std::lower_bound(t.files.begin(), t.files.end(), rel, [](const TableFile& f, const std::string& r) { return f.rel < r; }) -
                        t.files.begin());
    };
    std::vector<size_t> keep;
    for (const std::string& p : paths) {
        const size_t i = at(p);
        if (i < t.files.size() && t.files[i].rel == p) keep.push_back(i);
        for (size_t j = at(p + "/"), end = at(p + "0"); j < end; j++) keep.push_back(j);     // '0' follows '/': all of p/...
    }
    std::sort(keep.begin(), keep.end());
    for (size_t i : keep) {
        TableFile f = t.files[i];
        const uint64_t nb = t.blocks_of(f);
        f.first_block = out->hashes.size();
        out->hashes.insert(out->hashes.end(), t.hashes.begin() + (ptrdiff_t)t.files[i].first_block,
                           t.hashes.begin() + (ptrdiff_t)(t.files[i].first_block + nb));
        out->index[f.rel] = out->files.size();
        out->files.push_back(std::move(f));
    }
}

int prepare_parents(const std::string& dst_root, Selection* sel, const std::atomic<int>* cancel)
{
    const int rfd = open(dst_root.c_str(), O_RDONLY | O_DIRECTORY | O_CLOEXEC);
    if (rfd < 0) return fail(VMIG_EIO, "open %s: %s", dst_root.c_str(), errno_str(errno).c_str());
    std::vector<Entry> created;
    int rc = VMIG_OK;
    for (const Entry& d : sel->parents) {          // parents first: each one's own parent is a real directory by now
        if (cancel && cancel->load()) { rc = fail(VMIG_ECANCELED, "cancelled before the destination directory %s", d.rel.c_str()); break; }
        const size_t slash = d.rel.rfind('/');
        const std::string parent = slash == std::string::npos ? "." : d.rel.substr(0, slash);
        const std::string name = slash == std::string::npos ? d.rel : d.rel.substr(slash + 1);
        int pfd = rfd;
        if (parent != "." && (rc = open_beneath(rfd, parent, O_RDONLY | O_DIRECTORY, &pfd))) break;
        struct stat st;
        const std::string p = pjoin(dst_root, d.rel);
        if (fstatat(pfd, name.c_str(), &st, AT_SYMLINK_NOFOLLOW) == 0) {
            if (!S_ISDIR(st.st_mode) && unlinkat(pfd, name.c_str(), 0) != 0 && errno != ENOENT)
                rc = fail(VMIG_EIO, "unlink %s (in the way of a directory): %s", p.c_str(), errno_str(errno).c_str());
            else if (S_ISDIR(st.st_mode)) { if (pfd != rfd) close(pfd); continue; }
        } else if (errno != ENOENT) {
            rc = fail(VMIG_EIO, "lstat %s: %s", p.c_str(), errno_str(errno).c_str());
        }
        if (!rc && mkdirat(pfd, name.c_str(), 0700) != 0) rc = fail(VMIG_EIO, "mkdir %s: %s", p.c_str(), errno_str(errno).c_str());
        if (pfd != rfd) close(pfd);
        if (rc) break;
        created.push_back(d);
    }
    close(rfd);
    if (rc) return rc;
    std::vector<Entry>& dirs = sel->man.dirs;
    dirs.insert(dirs.begin() + 1, std::make_move_iterator(created.begin()), std::make_move_iterator(created.end()));
    return VMIG_OK;
}

}  // namespace vmig
