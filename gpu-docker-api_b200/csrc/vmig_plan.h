// vmig_plan.h -- the plan of a tree call (migrate, move, restore, snapshot): which destination files are patched in
// place, which base-snapshot files may supply blocks, and the block list in submission order.  No CUDA (tests/plan_unit.cpp).
#pragma once
#include <stdint.h>
#include <atomic>
#include <string>
#include <vector>
#include "vmig_engine.h"
#include "vmig_reuse.h"
#include "vmig_table.h"
#include "vmig_tree.h"

namespace vmig {

// The blocks of one file (or scrub inode): BlockRef.file = file, hashes [first_block, first_block + n_blocks)
struct BlockSpan { uint32_t file; uint64_t size, first_block, n_blocks; };

// Append the blocks of spans[]: files in groups of 64 (bounds open descriptors), blocks round-robin across a group so that
// many destination files are written at once (one tmpfs/xfs file takes writes one thread at a time: probe/hostio_probe.cu)
void interleave_blocks(const std::vector<BlockSpan>& spans, uint32_t block_bytes, std::vector<BlockRef>* out);

struct FilePlan {
    const TableFile* prior_rec = nullptr;   // patched in place: the destination file still is this prior-table record
    const TableFile* base_rec = nullptr;    // vmig_snapshot_tree: the same-path base file still is this record
    const TableFile* layer_rec = nullptr;   // vmig_snapshot_layer, vmig_migrate_layer: the source file still is this record
    bool solo = true;                       // no other source path is a hard link to this file
};

struct TreePlan {
    std::vector<FilePlan> files;            // per manifest file
    std::vector<uint8_t> base_trusted;      // per base-table file: it still is the file its record was written for
    bool any_base = false;                  // some file has a base_rec
    uint64_t files_untrusted = 0;           // vmig_stats.files_untrusted
    uint64_t files_base_untrusted = 0;      // vmig_snapshot_stats.files_base_untrusted
    BaseIndex bidx;                         // (XXH64, length) of every block of every trusted base file (base given)
    std::vector<BlockRef> blocks;           // interleave_blocks order; a block's prior hash is its prior_rec / base_rec one
    // layer table given (vmig_snapshot_layer, vmig_migrate_layer), per manifest block: a trusted file's block whose
    // record (hash, length) the base index holds, or the prior record holds at the same index, is not read (skipped) and
    // is not in blocks; its other blocks are, and must hash as recorded (expect)
    std::vector<uint64_t> layer_hashes;     // the record's hashes of trusted files' blocks, 0 elsewhere
    std::vector<uint8_t> skipped;           // 1: not read, the base or the destination holds its bytes
    std::vector<uint8_t> expect;            // 1: read, and K1 must return layer_hashes[] for it
    std::vector<uint32_t> unread;           // trusted files none of whose blocks is read
    uint64_t files_trusted = 0, bytes_trusted = 0;     // vmig_layer_snapshot_stats, vmig_layer_migrate_stats
    uint64_t files_read = 0, bytes_read = 0;
};

// prior (nullable): a destination file under dst_root is patched in place while it still is its record and has one link.
// base (nullable; only when base_root is on the destination's device): every record is checked once, as a source file
// may find its bytes in any base file.  Both tables are at block_bytes.  VMIG_ECANCELED once *cancel (nullable) is set,
// checked every kMetaCheckEvery base records.
// layer (nullable; vmig_snapshot_layer with a base, vmig_migrate_layer with a prior or neither): a source file under
// src_root is trusted while it is the walked inode and still is its record (is_recorded_file).  Of a trusted file only
// the blocks are read whose record (hash, length) is neither in the base index nor the prior record's at the same index
// (a destination file patched in place).  Untrusted files are planned as without it.
int plan_tree(const Manifest& man, uint32_t block_bytes, const std::string& dst_root, const BlockTable* prior,
              const std::string& base_root, const BlockTable* base, const std::atomic<int>* cancel, TreePlan* out,
              const std::string& src_root = std::string(), const BlockTable* layer = nullptr);

// vmig_migrate_layer's src_out_table, for a source file read while its tenant may be writing it: whether the hashes just
// taken may be recorded under the identity the file had before its first block was read.  before: the open descriptor's
// fstat before that read, clock_ns: CLOCK_REALTIME_COARSE read just before that fstat, after: the descriptor's fstat once
// the file's last block hash is back.  A regular file with one link whose ctime is strictly older than the clock, and
// whose inode, size and ctime did not move in between: any write after the first fstat stamps a ctime at or past the
// clock (with or without multigrain timestamps), so the record stops vouching for the file the moment it changes.
bool live_identity_holds(const struct stat& before, int64_t clock_ns, const struct stat& after);

}  // namespace vmig
