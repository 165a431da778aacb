// vmig_retire.cpp -- the host side of vmig_retire_versions (see vmig_retire.h).
#include "vmig_retire.h"
#include "vmig_common.h"

#include <fcntl.h>
#include <unistd.h>
#include <sys/stat.h>

namespace vmig {

int retire_remove(const std::string& dir, const std::string& table, RemoveCount* n, const std::atomic<int>* cancel)
{
    if (unlink(table.c_str()) != 0 && errno != ENOENT) return fail(VMIG_EIO, "unlink %s: %s", table.c_str(), errno_str(errno).c_str());
    const size_t slash = dir.rfind('/');
    const std::string parent = slash == std::string::npos ? "." : slash == 0 ? "/" : dir.substr(0, slash);
    const std::string base = slash == std::string::npos ? dir : dir.substr(slash + 1);
    const int pfd = open(parent.c_str(), O_RDONLY | O_DIRECTORY | O_CLOEXEC);
    if (pfd < 0) return errno == ENOENT ? VMIG_OK : fail(VMIG_EIO, "open %s: %s", parent.c_str(), errno_str(errno).c_str());
    const int fd = openat(pfd, base.c_str(), O_RDONLY | O_DIRECTORY | O_NOFOLLOW | O_CLOEXEC);
    if (fd < 0) {
        const int e = errno;
        close(pfd);
        if (e == ENOENT) return VMIG_OK;
        if (e == ELOOP || e == ENOTDIR) return fail(VMIG_ENOTDIR, "%s is not a directory (a symlink is not followed)", dir.c_str());
        return fail(VMIG_EIO, "open %s: %s", dir.c_str(), errno_str(e).c_str());
    }
    int rc = remove_contents(fd, dir.c_str(), "retire", n, cancel);
    if (!rc && unlinkat(pfd, base.c_str(), AT_REMOVEDIR) != 0 && errno != ENOENT)
        rc = fail(VMIG_EIO, "rmdir %s: %s", dir.c_str(), errno_str(errno).c_str());
    close(pfd);
    return rc;
}

// the file at rel beneath root, not following any symlink; false when it cannot be opened
static bool stat_beneath(int root, const std::string& rel, struct stat* st)
{
    int fd;
    if (open_beneath(root, rel, O_PATH, &fd) != VMIG_OK) return false;
    const bool ok = fstat(fd, st) == 0;
    close(fd);
    return ok;
}

int retire_find_stale(const std::vector<int>& root_fds, const std::vector<const BlockTable*>& tabs,
                      std::vector<StaleRecord>* out, const std::atomic<int>* cancel)
{
    out->clear();
    size_t steps = 0;
    for (uint32_t v = 0; v < tabs.size(); v++) {
        const BlockTable& t = *tabs[v];
        for (uint32_t f = 0; f < t.files.size(); f++) {
            const TableFile& rec = t.files[f];
            if (rec.ino == 0) continue;
            if (cancel && steps++ % kMetaCheckEvery == 0 && cancel->load())
                return fail(VMIG_ECANCELED, "cancelled while checking the kept tables, before %s", rec.rel.c_str());
            struct stat st;
            if (!stat_beneath(root_fds[v], rec.rel, &st)) continue;
            if (S_ISREG(st.st_mode) && (uint64_t)st.st_ino == rec.ino && (uint64_t)st.st_size == rec.size && ctime_ns(st) != rec.ctime_ns)
                out->push_back({v, f, (uint64_t)st.st_dev, ctime_ns(st)});
        }
    }
    return VMIG_OK;
}

int retire_group(const std::vector<StaleRecord>& stale, const std::vector<const BlockTable*>& tabs, uint32_t block_bytes,
                 std::vector<ScrubInode>* inodes, std::vector<uint32_t>* inode_of)
{
    inodes->clear();
    inode_of->assign(stale.size(), kNoInode);
    InodeGroups groups{inodes, block_bytes, "retire"};
    for (size_t r = 0; r < stale.size(); r++) {
        const TableFile& rec = tabs[stale[r].version]->files[stale[r].file];
        const int rc = groups.add(stale[r].dev, rec.ino, rec.size, stale[r].version, rec.rel, &(*inode_of)[r]);
        if (rc) return rc;
    }
    return VMIG_OK;
}

std::vector<size_t> retire_decide(const std::vector<int>& root_fds, const std::vector<const BlockTable*>& tabs,
                                  const std::vector<StaleRecord>& stale, const std::vector<ScrubInode>& inodes,
                                  const std::vector<uint32_t>& inode_of, const std::vector<uint64_t>& hashes,
                                  const std::vector<bool>& unreadable)
{
    // the ctime of an inode before the read is what its first record saw; after the read it must still be that
    std::vector<int64_t> before(inodes.size(), 0);
    std::vector<bool> have(inodes.size(), false);
    for (size_t r = 0; r < stale.size(); r++)
        if (!have[inode_of[r]]) { have[inode_of[r]] = true; before[inode_of[r]] = stale[r].ctime_ns; }
    std::vector<int8_t> still(inodes.size(), -1);            // second fstat, once per inode: 1 unchanged, 0 moved
    auto unchanged = [&](uint32_t u) {
        if (still[u] < 0) {
            const ScrubInode& I = inodes[u];
            struct stat st;
            still[u] = stat_beneath(root_fds[I.version], I.rel, &st) && S_ISREG(st.st_mode) && (uint64_t)st.st_dev == I.dev &&
                       (uint64_t)st.st_ino == I.ino && (uint64_t)st.st_size == I.size && ctime_ns(st) == before[u];
        }
        return still[u] == 1;
    };
    std::vector<size_t> chosen;
    for (size_t r = 0; r < stale.size(); r++) {
        const uint32_t u = inode_of[r];
        if (unreadable[u] || stale[r].ctime_ns != before[u]) continue;
        const BlockTable& t = *tabs[stale[r].version];
        const TableFile& rec = t.files[stale[r].file];
        const ScrubInode& I = inodes[u];
        bool same = true;
        for (uint64_t b = 0; b < I.n_blocks && same; b++) same = hashes[I.first_block + b] == t.hashes[rec.first_block + b];
        if (same && unchanged(u)) chosen.push_back(r);
    }
    return chosen;
}

size_t retire_patch(uint32_t v, const std::vector<StaleRecord>& stale, const std::vector<size_t>& chosen,
                    const std::vector<ScrubInode>& inodes, const std::vector<uint32_t>& inode_of, BlockTable* t)
{
    size_t n = 0;
    for (size_t r : chosen) {
        if (stale[r].version != v) continue;
        TableFile& rec = t->files[stale[r].file];
        rec.ino = inodes[inode_of[r]].ino;
        rec.ctime_ns = stale[r].ctime_ns;
        n++;
    }
    return n;
}

}  // namespace vmig
