// vmig_select.h -- the host side of vmig_restore_paths: which entries of a snapshot a partial restore takes, checked
// against which part of the snapshot's block table, and the destination's parent chains they are restored into.
//
// The per-byte work is the checked restore's (K1 with the expected-hash check, then the writer path); what is here is the
// plan around it.  No CUDA header is needed (tests/select_unit.cpp builds it with g++ alone).
#pragma once
#include <stdint.h>
#include <atomic>
#include <string>
#include <vector>
#include "vmig_table.h"
#include "vmig_tree.h"

namespace vmig {

// Check the caller's paths: each non-empty, relative, without an empty, "." or ".." component, not ending in '/', and no
// two equal or one beneath the other.  VMIG_EINVAL names the index and the path.  *out: the paths, sorted bytewise.
int select_check_paths(uint32_t n, const char* const* paths, std::vector<std::string>* out);

struct Selection {
    std::vector<std::string> paths;        // the chosen paths, sorted bytewise
    // The chosen entries and everything beneath the chosen directories, walked as walk_tree walks the snapshot, rel
    // relative to the snapshot root.  dirs[0] is "." (never created nor replayed: it stands for the destination root);
    // hard links are grouped inside the selection only.
    Manifest man;
    std::vector<Entry> parents;            // the snapshot's entry of every proper prefix of a chosen path, parents first
    std::vector<std::string> chosen_dirs;  // the chosen paths that are directories (the VMIG_F_PRUNE scope)
    std::vector<std::string> not_found;    // chosen paths the snapshot's walk would not find
};

// Walk the selection beneath snap_root.  A chosen path is found when every proper prefix is a real directory (lstat, no
// symlink followed) and the entry exists; skip_hidden_topdirs hides what walk_tree would skip.  Nothing but the chosen
// subtrees is listed or read; the parent chains are only lstat'ed and entered.  Paths that are not found are listed in
// out->not_found (the caller decides between "missing" and "not in the snapshot").
int select_walk(const std::string& snap_root, const std::vector<std::string>& paths, uint32_t block_bytes,
                bool skip_hidden_topdirs, Selection* out, const std::atomic<int>* cancel = nullptr);

// The records of t at a chosen path or beneath it, with their hashes, in table order (first_block rebased).  The table is
// sorted, so only those records are looked at.
void table_subset(const BlockTable& t, const std::vector<std::string>& paths, BlockTable* out);

// Make every proper prefix of every chosen path a real directory under dst_root: an existing directory is used as it is,
// a missing one is created (0700), anything else in the way -- symlink, file, special file, whiteout -- is removed (never
// followed) and replaced.  Each created prefix's snapshot entry (from sel->parents) is inserted into sel->man.dirs right
// after "." so that the metadata replay gives it the snapshot's owner, mode and mtime after its contents.
int prepare_parents(const std::string& dst_root, Selection* sel, const std::atomic<int>* cancel = nullptr);

}  // namespace vmig
