// vmig_tree.h -- source-tree manifest (walk) and destination metadata replay.
//
// What "the same result as the reference" means is fixed by what GNU tar restores when
// `(cd src; tar c .) | (cd dst; tar x)` runs as root (reference utils/copy.go:17-27): entry
// type, permission bits, uid/gid, mtime (whole seconds: tar's default gnu format), symlink
// targets, hard-link grouping inside the tree, char/block device numbers, FIFOs; sockets are
// skipped ("socket ignored"); xattrs/ACLs are dropped; existing destination entries are
// replaced, extras are kept.
#pragma once
#include <fcntl.h>
#include <stdint.h>
#include <atomic>
#include <memory>
#include <mutex>
#include <string>
#include <vector>
#include <sys/stat.h>
#include <sys/types.h>
#include <unistd.h>
#include "../../include/vmig.h"

namespace vmig {

// a manifest path under root ("." is the root itself)
inline std::string pjoin(const std::string& root, const std::string& rel) { return rel == "." ? root : root + "/" + rel; }

enum EntryType : uint8_t { kDir = 1, kFile, kSymlink, kSpecial /* chr, blk, fifo */ };

struct Entry {
    std::string rel;          // relative path, no leading "./"; "." for the root itself
    EntryType   type;
    mode_t      mode;         // full st_mode
    uid_t       uid;
    gid_t       gid;
    struct timespec mtime;
    struct timespec atime;
    uint64_t    size = 0;     // regular files
    dev_t       rdev = 0;     // specials
    std::string target;       // symlinks
    int64_t     hardlink_of = -1;   // files: index (in Manifest::files) of the first path to the same inode
    uint64_t    first_block = 0;    // files: index of this file's first hash in the block table
    uint64_t    n_blocks = 0;
    uint64_t    dev = 0, ino = 0;   // files: st_dev / st_ino as the walk saw them (vmig_scrub_store groups paths by inode)
};

struct Manifest {
    std::vector<Entry> dirs;      // parents before children; dirs[0] is "."
    std::vector<Entry> files;     // sorted bytewise by rel (block-table order)
    std::vector<Entry> symlinks;
    std::vector<Entry> specials;
    uint64_t bytes_total = 0;     // sum of regular-file sizes (hard-linked paths counted once per path)
    uint64_t n_blocks = 0;
    uint64_t sockets_skipped = 0;
};

// Open `rel` (a manifest path) beneath root_fd with `flags`, refusing every symlink on the way and every
// escape from the root (openat2 RESOLVE_BENEATH|RESOLVE_NO_SYMLINKS; a component-wise O_NOFOLLOW walk on
// kernels without it).  A path that stopped being plain since the walk fails with VMIG_ESRCCHANGED.
int open_beneath(int root_fd, const std::string& rel, int flags, int* out_fd);
int open_beneath_walk(int root_fd, const std::string& rel, int flags, int* out_fd);   // the fallback, exposed for tests/tree_unit.cpp

// The `cancel` arguments below: nullable; once *cancel is non-zero the function starts no new step (directory, metadata
// entry, prune entry, copy chunk) and returns VMIG_ECANCELED.
// Walk src_root.  skip_hidden_topdirs reproduces `mv /root/src/*` (reference utils/copy.go:116).
int walk_tree(const std::string& src_root, uint32_t block_bytes, bool skip_hidden_topdirs, Manifest* out,
              const std::atomic<int>* cancel = nullptr);
// The walk's entry for `name` in the open directory dfd, lstat'ed as st, appended to m under `rel` (a socket is only
// counted).  A regular file with more than one link carries its inode_key until finish_manifest groups it.
int manifest_add(int dfd, const std::string& name, const std::string& rel, const struct stat& st, uint32_t block_bytes, Manifest* m);
std::string inode_key(uint64_t dev, uint64_t ino);
// Sort m's files bytewise, resolve the inode keys to hardlink_of (the group's smallest path is its primary) and lay the
// blocks out in that order (first_block, n_blocks, bytes_total).
void finish_manifest(Manifest* m);

struct MetaPolicy {
    bool is_root;        // euid == 0: chown + exact modes (tar -p --same-owner defaults for root)
    mode_t umask_bits;   // applied when !is_root
    bool mtime_ns;       // VMIG_F_MTIME_NS
    bool no_metadata;    // VMIG_F_NO_METADATA
    bool keep_atime;     // move semantics (mv preserves atime too)
};
MetaPolicy default_meta_policy(uint32_t flags);

// Create every directory of the manifest under dst_root (parents first, traversable by us).
int make_dirs(const std::string& dst_root, const Manifest& m);
// Symlinks, specials, hard links and empty regular files; then directory metadata bottom-up.  Checks cancel every
// kMetaCheckEvery entries.
static constexpr size_t kMetaCheckEvery = 1024;
// Directory metadata is replayed for m.dirs[first_dir..] only (vmig_restore_paths leaves the destination root alone).
int replay_metadata(const std::string& dst_root, const Manifest& m, const MetaPolicy& pol,
                    uint64_t* n_symlinks, uint64_t* n_hardlinks, uint64_t* n_specials, const std::atomic<int>* cancel = nullptr,
                    size_t first_dir = 0);
// True if the open file already carries the owner/mode/mtime apply_file_meta would give it (then it is left alone: a
// diff pass that skips every block of a file must not move its ctime, the block table identifies files by it).
bool file_meta_matches(int fd, const Entry& e, const MetaPolicy& pol);
// Apply owner/mode/mtime to an open regular file (fd) or to a path (fd < 0).
int apply_file_meta(int fd, const std::string& path, const Entry& e, const MetaPolicy& pol);
// VMIG_F_MOVE_SRC: unlink migrated source entries, children before parents; the root stays.
int remove_source(const std::string& src_root, const Manifest& m);
// VMIG_F_PRUNE: remove every destination entry the manifest does not list (directories recursively); entries are
// handled by descriptor, symlinks are never followed.  dry_run only counts them (the verify pass uses that).
// scope (nullable): only what lies beneath these manifest directories is looked at (vmig_restore_paths).
int prune_extras(const std::string& dst_root, const Manifest& m, bool dry_run, uint64_t* n_extras,
                 const std::atomic<int>* cancel = nullptr, const std::vector<std::string>* scope = nullptr);
// What remove_contents removed: entries unlinked or rmdir'ed, and the regular files among them whose link count was 1
// just before the unlink (their space is freed unless a descriptor still holds them).
struct RemoveCount { uint64_t entries = 0, files_freed = 0, bytes_freed = 0; };
// Remove everything beneath the open directory fd (consumed; `name` and `what` only word the errors), children first,
// each entry by its parent's descriptor, never following a symlink.  The cancel check is per entry.  VMIG_F_PRUNE and
// vmig_retire_versions both remove trees this way.
int remove_contents(int fd, const char* name, const char* what, RemoveCount* n, const std::atomic<int>* cancel = nullptr);
// Remove whatever sits at path so that `what` (named in the error) can be created there: a non-directory or an EMPTY
// directory goes, as GNU tar replaces them; a non-empty directory is VMIG_EIO, as tar fails with "Cannot open: File
// exists".  ENOENT is fine.  Every non-directory the engine creates goes through this.
int clear_path(const std::string& path, const char* what);
// Copy bytes [off, off + len) of in_fd to the same offsets of out_fd (a snapshot file's unchanged blocks, taken from
// the base snapshot's file).  copy_file_range, which may share extents on filesystems that reflink; pread/pwrite where
// the kernel or filesystem refuses it (ENOSYS, EXDEV, EINVAL, EOPNOTSUPP) or rw_only is set.  out_direct: out_fd was
// opened O_DIRECT, off must be a multiple of 4096, and the bytes go out in whole sectors through an aligned buffer,
// zero-padded past off + len (the caller truncates the file to its size).  in_fd ending early is VMIG_ESRCCHANGED.
// The range is copied in chunks of kCopyChunk bytes; cancel is checked before each one.
static constexpr uint64_t kCopyChunk = 64ull << 20;
int copy_range(int in_fd, int out_fd, uint64_t off, uint64_t len, bool out_direct, bool rw_only, const std::string& what,
               const std::atomic<int>* cancel = nullptr);
// The same copy from [in_off, in_off + len) of in_fd to [out_off, out_off + len) of out_fd (a block that sits at another
// offset, or in another file, of the base snapshot).  out_direct: out_off must be a multiple of 4096.
int copy_range_at(int in_fd, uint64_t in_off, int out_fd, uint64_t out_off, uint64_t len, bool out_direct, bool rw_only,
                  const std::string& what, const std::atomic<int>* cancel = nullptr);

// The read descriptors of a file backend: one slot per file (or inode) of the call, opened by the first reader thread
// that needs it and closed after its last counted read.  The source may be a running tenant's layer: a file is opened
// with open_beneath (no symlink followed, the root never left), O_RDONLY | O_NONBLOCK so a FIFO swapped in cannot park
// a reader, and O_DIRECT first when asked (the filesystem may refuse it).  Per block a reader pays one acquire load in
// get and one fetch_sub in read_done.
class ReadFds {
public:
    std::atomic<uint64_t> n_direct{0};         // descriptors published that really were opened O_DIRECT

    void init(size_t n) { close_all(); n_ = n; slots_.reset(new Slot[n ? n : 1]); }     // n empty slots, no reads counted
    void add_reads(size_t i, uint64_t n) { slots_[i].reads_left.fetch_add(n, std::memory_order_relaxed); }
    bool direct(size_t i) const { return slots_[i].direct; }     // once get() has returned slot i's descriptor
    // *out: slot i's descriptor, opened if it is not yet (rel beneath root_fd).  A new descriptor is first given to
    // hook(int* fd, const struct stat* st, bool direct), st its fstat (nullptr when fstat failed; errno says why).  The
    // hook may replace *fd; a non-zero return is the call's code, and the table closes *fd and leaves the slot empty.
    template <class Hook> int get(size_t i, int root_fd, const std::string& rel, bool want_direct, Hook hook, int* out) {
        Slot& s = slots_[i];
        int fd = s.fd.load(std::memory_order_acquire);
        if (fd < 0) {
            std::lock_guard<std::mutex> lk(stripes_[i & 63]);
            fd = s.fd.load(std::memory_order_acquire);
            if (fd < 0) {
                int rc = want_direct ? open_beneath(root_fd, rel, O_RDONLY | O_NONBLOCK | O_DIRECT, &fd) : VMIG_EIO;
                const bool direct = rc == VMIG_OK;
                if (rc) rc = open_beneath(root_fd, rel, O_RDONLY | O_NONBLOCK, &fd);
                struct stat st;
                if (!rc && (rc = hook(&fd, fstat(fd, &st) == 0 ? &st : nullptr, direct))) close(fd);
                if (rc) return rc;
                s.direct = direct;
                if (direct) n_direct++;
                s.fd.store(fd, std::memory_order_release);
            }
        }
        *out = fd;
        return VMIG_OK;
    }
    // One counted read of slot i is done; after the last one the descriptor is closed, before_close(fd) first
    template <class BeforeClose> void read_done(size_t i, BeforeClose before_close) {
        if (slots_[i].reads_left.fetch_sub(1) != 1) return;
        const int fd = slots_[i].fd.exchange(-1);
        if (fd >= 0) { before_close(fd); close(fd); }
    }
    void read_done(size_t i) { read_done(i, [](int) {}); }
    void adopt(size_t i, int fd, bool direct) { slots_[i].direct = direct; slots_[i].fd.store(fd, std::memory_order_release); }
    void close_all() { for (size_t i = 0; i < n_; i++) { const int fd = slots_[i].fd.exchange(-1); if (fd >= 0) close(fd); } }
    ~ReadFds() { close_all(); }

private:
    struct Slot { std::atomic<int> fd{-1}; std::atomic<uint64_t> reads_left{0}; bool direct = false; };
    std::unique_ptr<Slot[]> slots_;
    size_t n_ = 0;
    std::mutex stripes_[64];
};

// Open path for writing, never through a symlink: in place, or as a new file (O_CREAT | O_EXCL, mode 0600).
// want_direct: O_DIRECT, and without it where the filesystem refuses it (EINVAL); *direct tells whether it held.
// Returns the descriptor, or -1 with errno.
int open_for_write(const std::string& path, bool create, bool want_direct, bool* direct);
// O_DIRECT writes whole sectors, so the last one of a file written that way is padded past the file's size: cut it back
// (ftruncate to size).  Also a patched file's resize.
int cut_to_size(int fd, uint64_t size, const std::string& path);
// Close a written file; its close error (deferred write-back) is the call's only when rc holds none yet.  Returns rc.
int close_written(int fd, int rc, const std::string& path);

}  // namespace vmig
