// vmig_rollback.h -- the host side of vmig_rollback_layer: roll a layer back to a version snapshot in place, reading from
// the snapshot only the blocks the layer does not already hold (DESIGN.md §6, "Rolling a layer back in place").
//
// The layer's block hashes come from vmig_compare_snapshot's read plan (compare_plan / compare_layer_hashes, unchanged).
// What is here is what the rollback does with them: one action per snapshot regular file, the sparse fetch list the block
// pipeline checks against the snapshot's table, the runs a rebuilt file copies from its old inode, the counters, and the
// identity check of a layer descriptor before anything is written into it or copied from it.  No CUDA header is needed
// (tests/rollback_unit.cpp builds it with g++ alone).
#pragma once
#include <stdint.h>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>
#include <sys/stat.h>
#include "vmig_compare.h"
#include "vmig_engine.h"
#include "vmig_tree.h"

namespace vmig {

enum RollbackAction : uint8_t { kRbKeep, kRbPatch, kRbRebuild, kRbCreate };
const char* rollback_action_name(RollbackAction a);

// What the plan trusted about a layer file: its inode, size and ctime (and link count, which decides whether it may be
// patched).  set == false: there is no layer regular file at the path.
struct LayerId {
    bool set = false;
    uint64_t ino = 0, size = 0, nlink = 0;
    int64_t ctime_ns = 0;
};
LayerId layer_id_of(const struct stat& st);

// The identity of every layer file a snapshot file's action may write into or copy from, per layer manifest file: a
// trusted file's is its record (compare_plan checked that the file still is it); any other's is an lstat taken now.
// Files the plan does not pair with a snapshot file are left unset.
int rollback_identify(const std::string& layer_root, const Manifest& layer, const ComparePlan& cp, const BlockTable* layer_tab,
                      std::vector<LayerId>* out);
// After the layer's hash pass: every identity taken before it must still be what an lstat shows, or the hashes the
// pass produced may describe other bytes (VMIG_ESRCCHANGED naming the path).
int rollback_recheck_paths(const std::string& layer_root, const Manifest& layer, const std::vector<LayerId>& ids);
// Before the first write into a patched file and before copying from a rebuilt file's old inode: fstat(fd) must show
// the inode, size and ctime the plan trusted (VMIG_ESRCCHANGED naming path otherwise).
int rollback_check_fd(int fd, const LayerId& id, const std::string& path);

// The replacement of a rebuilt file's path.  Its old inode may have other paths the same call rebuilds (a layer hard-link
// group whose paths the snapshot holds as separate files), and unlinking one path moves the inode's ctime.  The guard
// serialises the check and the clear of rebuilt paths and remembers the ctime each of the call's own unlinks left, so
// that only a change made by someone else fails the re-check.
class RebuildGuard {
public:
    // old_fd: the inode at path now (opened O_RDONLY when bytes are copied from it, O_PATH otherwise).  check: bytes are
    // copied from it, so it must be id -- with the ctime this call's own unlink of another of its paths left, if any --
    // else VMIG_ESRCCHANGED.  Then path is cleared (clear_path) and the inode's ctime after that unlink is remembered.
    int clear(int old_fd, const LayerId& id, bool check, const std::string& path);
private:
    std::mutex mu;
    std::unordered_map<uint64_t, int64_t> own_ctime;   // inode -> its ctime right after this call's last unlink of a path
};

// One snapshot regular file that is its hard-link group's primary (the other paths of a group are linked to it by the
// metadata replay, as in a restore).
struct RollbackFile {
    uint32_t snap = 0;                 // index in the snapshot manifest's files
    int64_t layer = -1;                // the layer's regular file at the same path, else -1
    RollbackAction action = kRbCreate;
    uint64_t n_fetch = 0;              // its blocks in the fetch list
    uint64_t first_run = 0, n_runs = 0;   // kRbRebuild: its copy runs
};

// A rebuilt file's bytes [off, off + len) copied from its old inode to the same offsets of the new one: consecutive
// blocks equal at the same index, coalesced.
struct CopyRun { uint32_t file; uint64_t off, len; };

struct RollbackPlan {
    std::vector<RollbackFile> files;   // in snapshot file order
    // The blocks to read from the snapshot, file by file in snapshot order, ascending offsets within a file.  BlockRef.file
    // is the index in files[]; table_idx the snapshot's global block index, so that the pipeline's expect is the
    // snapshot table's hashes as match_table returns them.
    std::vector<BlockRef> fetch;
    std::vector<CopyRun> runs;
    uint64_t files_kept = 0, files_patched = 0, files_rebuilt = 0, files_created = 0;
    uint64_t blocks_fetched = 0, bytes_fetched = 0, bytes_copied = 0;
};

// Per snapshot primary, the layer file at its path (if it is a regular file) is
//   patchable  its hashes, where the pair needs any, came from a trusted record or a read (not a shared inode), it has
//              one link (ids), it is writable by euid (root, or the owner with S_IWUSR: a read-only file is replaced, as
//              tar replaces it), and neither path is in a hard-link group;
//   keep       patchable, the same size, every (length, hash) equal;  patch  patchable, anything differs (a block past
//              the layer file's old end differs);  rebuild  there but not patchable: blocks equal at the same index are
//              copied from the old inode;  create  no regular file there: every block is fetched.
// snap_hashes: the snapshot table's hashes in the manifest's block order; layer_hashes: compare_layer_hashes'.
void rollback_plan(const Manifest& layer, const Manifest& snap, const std::vector<uint64_t>& snap_hashes, const ComparePlan& cp,
                   const std::vector<const uint64_t*>& layer_hashes, const std::vector<LayerId>& ids, uint32_t block_bytes,
                   uid_t euid, RollbackPlan* out);

}  // namespace vmig
