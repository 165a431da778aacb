// vmig_scrub.h -- the host side of vmig_scrub_store: check every version of a snapshot store against its block table,
// reading each inode the versions share once (DESIGN.md §6).
//
// The per-byte work is K1's, through the block pipeline in hash-only mode, exactly as a checked restore reads.  What is
// here is the plan around it: the table merge that lists every difference instead of stopping at the first, the grouping
// of all versions' regular files by (st_dev, st_ino), the reader that turns an unreadable inode into a finding instead
// of a call failure, and the report.  No CUDA header is needed (tests/scrub_unit.cpp builds it with g++ alone).
#pragma once
#include <stdint.h>
#include <atomic>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <utility>
#include <vector>
#include "vmig_engine.h"
#include "vmig_table.h"
#include "vmig_tree.h"

namespace vmig {

enum ScrubKind : uint8_t { kScrubMissing, kScrubExtra, kScrubResized, kScrubBlock, kScrubHardlink, kScrubUnreadable, kScrubTable, kScrubDir };
const char* scrub_kind_name(ScrubKind k);

// One line of the report.  block < 0: the finding is about the whole path ("-"); has_hashes: got / want are printed.
struct ScrubFinding {
    uint32_t version = 0;
    ScrubKind kind = kScrubBlock;
    std::string path;
    int64_t block = -1;
    bool has_hashes = false;
    uint64_t got = 0, want = 0;
};

// The merge of restore's plan-time check (the walked regular-file paths must be the table's, each with the table's
// size), recording every difference: a path only in the walk is `extra`, only in the table `missing`, in both with other
// sizes `resized`.  (*tab_of)[f] is the table index of manifest file f when both name it with one size, else -1.
// Returns the number of findings appended.
size_t scrub_merge_table(uint32_t version, const Manifest& man, const BlockTable& t, std::vector<int64_t>* tab_of,
                         std::vector<ScrubFinding>* out);

// One distinct inode of the store: read once, its blocks at [first_block, first_block + n_blocks) of the scrub's hash
// array.  (version, rel) is the first path that names it; it is opened there.
struct ScrubInode { uint64_t dev, ino, size, first_block, n_blocks; uint32_t version; std::string rel; };
static constexpr uint32_t kNoInode = 0xFFFFFFFFu;

// The grouping rule of every call that reads each distinct inode once: an inode is its (st_dev, st_ino), opened at the
// first path that names it, its block range laid out after those of the inodes seen before it.  A second size for one
// inode means the store changed between the walks: VMIG_ESRCCHANGED, "...during the <call>".
struct InodeGroups {
    std::vector<ScrubInode>* inodes;
    uint32_t block_bytes;
    const char* call;                          // "scrub", "retire"
    std::map<std::pair<uint64_t, uint64_t>, uint32_t> seen;
    uint64_t next_block = 0;
    // *u: the index in *inodes of the inode (dev, ino), which version's rel names with size bytes
    int add(uint64_t dev, uint64_t ino, uint64_t size, uint32_t version, const std::string& rel, uint32_t* u);
};

// Group the selected, non-empty regular files of every version (sel[v][f] >= 0: for the scrub, the table index of a file
// that matches its record; for vmig_compare_snapshot, a layer file to read; mans[v] may be null for a version that was
// not walked) by InodeGroups' rule, named "scrub".  (*inode_of)[v][f] is the inode's index, kNoInode where the path is
// not read.
int scrub_group_inodes(const std::vector<const Manifest*>& mans, const std::vector<std::vector<int64_t>>& sel,
                       uint32_t block_bytes, std::vector<ScrubInode>* inodes, std::vector<std::vector<uint32_t>>* inode_of);

// Report paths: '\' -> "\\", tab -> "\t", newline -> "\n", any other byte below 0x20 -> "\xHH" (two lower-case hex
// digits).  scrub_unescape is the inverse; false on a malformed escape.
std::string scrub_escape(const std::string& s);
bool scrub_unescape(const std::string& s, std::string* out);
// "<version>\t<kind>\t<path>\t<block|->\t<got|->\t<want|->\n", hashes as 16 lower-case hex digits
std::string scrub_format(const ScrubFinding& f);
// by version, then path (bytewise), then block ("-" first)
void scrub_sort(std::vector<ScrubFinding>* v);
// A report file (raw: its lines), written atomically like a block table: path.tmp.<pid>.<tid>, fsync, rename.  `what`
// names it in errors.  A non-zero *cancel before the rename removes the .tmp and returns VMIG_ECANCELED; any failure
// leaves no .tmp.  vmig_scrub_store and vmig_compare_snapshot write their reports through it.
int report_store(const std::string& path, const std::string& raw, const char* what, const std::atomic<int>* cancel);
// The scrub's findings, formatted, through report_store
int scrub_report_store(const std::string& path, const std::vector<ScrubFinding>& v, const std::atomic<int>* cancel);

// The scrub's source of block bytes.  An inode is opened lazily beneath the root of the version that names it first
// (open_beneath: no symlink followed), O_RDONLY, O_DIRECT when asked and the filesystem allows it.  An inode that is no
// longer the walked one (other dev/ino, not a regular file, other size, shorter than its blocks, or its path gone) is
// VMIG_ESRCCHANGED, a call failure as everywhere else.  Any other open or read error does NOT fail: the inode is marked
// unreadable, its remaining blocks are not read, and read() returns VMIG_OK so the pipeline's first-error latch stays
// clear.  Thread-safe; the descriptor is closed after the inode's last block.  It is the block pipeline's backend in
// hash-only mode: block b of inode u is BlockRef{file = u, table_idx = its index in the call's hash array}.
class ScrubReader : public BlockIO {
public:
    std::vector<int> root_fds;                 // per version; -1 for a version that is not read (not owned)
    const std::vector<ScrubInode>* inodes = nullptr;
    bool direct = false;                       // VMIG_F_DIRECT_IO
    uint32_t block_bytes = 4u << 20;           // numbers the blocks in block_name
    ReadFds fds;                               // one slot per inode; fds.n_direct: descriptors really opened O_DIRECT

    void init();                               // after inodes is set: one counted read per block
    int read(uint32_t u, uint64_t off, uint32_t len, uint8_t* dst);
    int read_block(const BlockRef& b, uint8_t* dst) override { return read(b.file, b.file_off, b.len, dst); }
    int write_block(const BlockRef&, const uint8_t*) override { return fail(VMIG_EINVAL, "a scrub writes nothing"); }
    uint32_t slot_align() override { return direct ? kSector : 512; }
    std::string block_name(const BlockRef& b) override;   // "<rel> (version N) block K"
    void adopt(uint32_t u, int fd, bool is_direct) { fds.adopt(u, fd, is_direct); }   // use this open descriptor for inode u (tests/scrub_unit.cpp)
    bool unreadable(uint32_t u) const { return st[u].bad.load(); }
    std::string why(uint32_t u);               // the error that made u unreadable
    void close_all() { fds.close_all(); }

private:
    struct State {
        std::atomic<bool> bad{false};
        std::string why;                       // under why_mu
    };
    std::unique_ptr<State[]> st;
    std::mutex why_mu;
    int open_inode(uint32_t u, int* out);
    void mark_bad(uint32_t u, const std::string& why);
};

}  // namespace vmig
