// vmig_retire.h -- the host side of vmig_retire_versions: remove old versions of a snapshot store, then re-verify and
// re-record the kept tables' records whose ctime the removal moved (DESIGN.md §6, "Retiring versions").
//
// Unlinking one hard link of an inode moves the inode's ctime, so removing a version leaves stale the kept tables'
// records of every file it shared with them.  The re-verify reads each such inode once through the block pipeline in
// hash-only mode, exactly as the scrub does (ScrubReader, unchanged); what is here is the plan around it: the removal
// with its counts, the selection and grouping of stale records, and the re-stamp decision with its table patch.  No
// CUDA header is needed (tests/retire_unit.cpp builds it with g++ alone).
#pragma once
#include <stdint.h>
#include <atomic>
#include <string>
#include <vector>
#include "vmig_scrub.h"
#include "vmig_table.h"
#include "vmig_tree.h"

namespace vmig {

// Remove one retired version: first its table (a half-removed version is never a base or a restore source again), then
// its tree with remove_contents, last the directory itself.  A missing table or directory is not an error; a dir that
// exists but is not a directory (a symlink included) is VMIG_ENOTDIR and is not followed.  n counts the entries beneath
// dir, not dir itself.
int retire_remove(const std::string& dir, const std::string& table, RemoveCount* n, const std::atomic<int>* cancel);

// A kept-table record whose file is still the recorded regular file (inode, size) but with another ctime.
struct StaleRecord { uint32_t version; uint32_t file; uint64_t dev; int64_t ctime_ns; };

// Every record with an identity (ino != 0) of every kept table tabs[k], opened beneath root_fds[k] (open_beneath, no
// symlink followed) and fstat'ed.  A record that cannot be opened, or is another inode, type or size, is not stale and
// is left alone.  Cancel checked every kMetaCheckEvery records.
int retire_find_stale(const std::vector<int>& root_fds, const std::vector<const BlockTable*>& tabs,
                      std::vector<StaleRecord>* out, const std::atomic<int>* cancel);

// Group stale records into the scrub's inodes by the scrub's rule (InodeGroups).  (*inode_of)[r] is record r's inode.
int retire_group(const std::vector<StaleRecord>& stale, const std::vector<const BlockTable*>& tabs, uint32_t block_bytes,
                 std::vector<ScrubInode>* inodes, std::vector<uint32_t>* inode_of);

// After the data pass (hashes[] in the inodes' block ranges; unreadable[u] from the reader): record r is re-stamped with
// the identity seen before the read when its inode was read, every block hash equals its table's, the record saw the
// same ctime as the inode's first record, and a second fstat of the inode (beneath its first record's root) shows the
// same inode, size and ctime.  Returns the re-stamped records' indices into stale.
std::vector<size_t> retire_decide(const std::vector<int>& root_fds, const std::vector<const BlockTable*>& tabs,
                                  const std::vector<StaleRecord>& stale, const std::vector<ScrubInode>& inodes,
                                  const std::vector<uint32_t>& inode_of, const std::vector<uint64_t>& hashes,
                                  const std::vector<bool>& unreadable);

// Set the identity of the chosen records of version v in t (only their ino / ctime_ns change); returns how many.
size_t retire_patch(uint32_t v, const std::vector<StaleRecord>& stale, const std::vector<size_t>& chosen,
                    const std::vector<ScrubInode>& inodes, const std::vector<uint32_t>& inode_of, BlockTable* t);

}  // namespace vmig
