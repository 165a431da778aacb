// vmig_table.h -- per-(resource, version) block table: file manifest + one XXH64 per 4 MiB block.
// File format: include/vmig.h ("Block-table file").  No reference symbol exists for it (the
// reference has no hashing); its home is the per-version directory that
// internal/services/replicaset.go:681-704 (setToMergeMap) creates and
// internal/version/merge.go:16 (ContainerMergeMap) records.
#pragma once
#include <stdint.h>
#include <sys/stat.h>
#include <atomic>
#include <string>
#include <vector>
#include <unordered_map>

namespace vmig {

// ino / ctime_ns identify the on-disk file the hashes were taken FOR: the destination file the migration that
// wrote the table left behind (the source file for a VMIG_F_HASH_ONLY table).  0/0 = unknown (format 01, hard-linked
// paths).  The in-place diff path trusts a prior table for a destination file only while both still match
// (ctime cannot be set from user space: any out-of-band write, truncate, chmod or rename-over bumps it).
struct TableFile { std::string rel; uint64_t size; uint64_t first_block; uint64_t ino = 0; int64_t ctime_ns = 0; };

inline int64_t ctime_ns(const struct stat& st) { return (int64_t)st.st_ctim.tv_sec * 1000000000ll + st.st_ctim.tv_nsec; }
// st is the file rec was written for: a regular file with the recorded inode, size and ctime (rec.ino == 0: unknown)
inline bool is_recorded_file(const struct stat& st, const TableFile& rec) {
    return S_ISREG(st.st_mode) && rec.ino != 0 && (uint64_t)st.st_ino == rec.ino && (uint64_t)st.st_size == rec.size &&
           ctime_ns(st) == rec.ctime_ns;
}

struct BlockTable {
    uint32_t block_bytes = 0;
    uint32_t algo = 1;                       // 1 = XXH64, seed 0
    std::vector<TableFile> files;            // sorted bytewise by rel
    std::vector<uint64_t> hashes;
    std::unordered_map<std::string, size_t> index;   // rel -> files[] index (built by load)
    uint64_t bytes_total() const { uint64_t s = 0; for (auto& f : files) s += f.size; return s; }
    uint64_t blocks_of(const TableFile& f) const { return (f.size + block_bytes - 1) / block_bytes; }
};

int table_load(const std::string& path, BlockTable* out);
// Atomic: writes path.tmp.<pid>.<tid>, fsyncs, renames over path.  A non-zero *cancel (nullable) before the rename
// removes the .tmp and returns VMIG_ECANCELED: no table at all.
int table_store(const std::string& path, const BlockTable& t, const std::atomic<int>* cancel = nullptr);
// Called before table_store by every call that records identities.  A kernel without multigrain timestamps (Linux
// < 6.13) stamps ctime from CLOCK_REALTIME_COARSE, so a same-size write in the timer tick of a recorded ctime leaves
// inode, size and ctime as recorded, and is_recorded_file would vouch for stale hashes.  Returns once that clock is past
// the newest ctime t records: every later write then moves the ctime of any file it records.  At most one tick; a
// ctime more than a second ahead of the clock (another host's, on a network filesystem) is not waited for.
void wait_past_recorded_ctimes(const BlockTable& t);

}  // namespace vmig
