// vmig_compare.h -- the host side of vmig_compare_snapshot: every difference between a layer and a version snapshot,
// each regular file's blocks judged against the snapshot's table (DESIGN.md §6, "Comparing a layer with a version").
//
// The per-byte work is K1's, through the block pipeline in hash-only mode and the scrub's reader (ScrubReader,
// unchanged), exactly as vmig_scrub_store reads.  What is here is the plan around it: which layer files need their block
// hashes and where each takes them from (the snapshot's own inode, a trusted record of the layer's table, or a read of
// each distinct inode once), the merge of the two walks into findings, the hard-link group comparison, the arithmetic of
// bytes_restore, and the report's lines.  No CUDA header is needed (tests/compare_unit.cpp builds it with g++ alone).
#pragma once
#include <stdint.h>
#include <string>
#include <vector>
#include "vmig_scrub.h"
#include "vmig_table.h"
#include "vmig_tree.h"

namespace vmig {

// Report kinds, in the order the lines of one path are sorted in
enum CompareKind : uint8_t { kCmpAdded, kCmpRemoved, kCmpType, kCmpResized, kCmpBlock, kCmpTarget, kCmpRdev, kCmpHardlink,
                             kCmpMode, kCmpOwner, kCmpMtime };
const char* compare_kind_name(CompareKind k);

// One line of the report.  block < 0: "-".  layer / snap are printed as they are ("-" when the kind has no value).
struct CompareFinding {
    CompareKind kind = kCmpAdded;
    std::string path;
    int64_t block = -1;
    std::string layer = "-", snap = "-";
};

// Where a layer regular file's block hashes come from.  A file needs them only when it and the snapshot's regular file
// at the same path both have at least one block.
enum CompareSource : uint8_t { kCmpNone, kCmpShared, kCmpTrusted, kCmpRead };

struct ComparePlan {
    std::vector<int64_t> snap_of;           // per layer file: the snapshot's regular file at the same path, else -1
    std::vector<uint8_t> source;            // per layer file: CompareSource
    std::vector<int64_t> rec_of;            // per layer file: kCmpTrusted's layer-table record, else -1
    std::vector<ScrubInode> inodes;         // the distinct inodes of the kCmpRead files, in layer block order (version 0)
    std::vector<uint32_t> inode_of;         // per layer file: its inode, kNoInode where it is not read
    uint64_t files_shared = 0, files_trusted = 0, bytes_read = 0, blocks_read = 0;
};

// A layer file that needs hashes takes them from the first that applies:
//   kCmpShared   it is the snapshot path's own (st_dev, st_ino) with the same size: equal by construction;
//   kCmpTrusted  layer_tab (nullable) records the path, and the file at layer_root/rel (lstat'ed now, as plan_tree checks
//                a prior table) is still the walked inode and is that record (is_recorded_file);
//   kCmpRead     otherwise; the read files are grouped by inode (scrub_group_inodes), each inode read once.
// Two paths of one inode with different sizes: VMIG_ESRCCHANGED.
int compare_plan(const std::string& layer_root, const Manifest& layer, const Manifest& snap, const BlockTable* layer_tab,
                 uint32_t block_bytes, ComparePlan* out);

// After the data pass: each layer file's block hashes (nullptr where the plan needs none).  snap_hashes are the
// snapshot table's hashes in the snapshot manifest's block order (match_table); read_hashes the data pass's, in the
// plan's inode block order.
std::vector<const uint64_t*> compare_layer_hashes(const ComparePlan& p, const Manifest& layer, const Manifest& snap,
                                                  const std::vector<uint64_t>& snap_hashes, const BlockTable* layer_tab,
                                                  const std::vector<uint64_t>& read_hashes);

struct CompareCounts {
    uint64_t paths_added = 0, paths_removed = 0, paths_changed = 0, files_changed = 0, blocks_changed = 0, bytes_restore = 0;
};

// Every difference between the two walks (include/vmig.h, vmig_compare_snapshot), sorted (compare_sort), and the
// counters.  mtime_ns: VMIG_F_MTIME_NS; no_metadata: VMIG_F_NO_METADATA (mode, owner and mtime are not compared).
void compare_merge(const Manifest& layer, const Manifest& snap, const std::vector<uint64_t>& snap_hashes,
                   const std::vector<const uint64_t*>& layer_hashes, uint32_t block_bytes, bool mtime_ns, bool no_metadata,
                   std::vector<CompareFinding>* out, CompareCounts* counts);

// "<kind>\t<path>\t<block|->\t<layer>\t<snap>\n", the path escaped as in the scrub report (scrub_escape)
std::string compare_format(const CompareFinding& f);
// by path (bytewise), then kind (CompareKind order), then block
void compare_sort(std::vector<CompareFinding>* v);

}  // namespace vmig
