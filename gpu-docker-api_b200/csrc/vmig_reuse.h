// vmig_reuse.h -- where an incremental snapshot finds unchanged bytes in its base snapshot: by block content, wherever
// the base holds it, not only at the same path and offset (vmig_snapshot_tree, DESIGN.md §6).
//
// The index maps (XXH64, length) -> (base file, block) for every block of every trusted base file.  The length is part
// of the key: a short last block only matches a block of exactly its length, so every reuse copies one whole block.
// A lookup is one hash-map probe on the 8 bytes the hash-waiter already holds; there is no device-side index (a probe
// per changed 4 MiB block is not work worth a kernel launch).
#pragma once
#include <stdint.h>
#include <algorithm>
#include <string>
#include <unordered_map>
#include <vector>
#include "vmig_table.h"

namespace vmig {

class BaseIndex {
public:
    struct Loc { uint64_t hash; uint32_t len; uint32_t file; uint64_t block; };    // file: index in the base table
    const BlockTable* t = nullptr;
    // trusted[i] != 0: base file i still is what its record says (vmig_api.cu checks ino, ctime and size by lstat)
    void build(const BlockTable& table, const std::vector<uint8_t>& trusted);
    bool empty() const { return locs.empty(); }
    size_t size() const { return locs.size(); }
    // the base blocks with this key, in table order (file, then block); n == 0 when there is none
    const Loc* find(uint64_t hash, uint32_t len, size_t* n) const;
    bool contains(uint64_t hash, uint32_t len) const { size_t n; return find(hash, len, &n) != nullptr; }
    bool trusted(uint32_t file) const { return file < trust.size() && trust[file]; }
    uint32_t block_len(uint32_t file, uint64_t block) const;     // 0 past the file's end
    uint64_t hash_of(uint32_t file, uint64_t block) const { return t->hashes[t->files[file].first_block + block]; }

private:
    struct KeyHash { size_t operator()(const std::pair<uint64_t, uint32_t>& k) const { return (size_t)(k.first ^ (k.second * 0x9E3779B97F4A7C15ull)); } };
    std::vector<Loc> locs;                                        // sorted by (hash, len, file, block)
    std::unordered_map<std::pair<uint64_t, uint32_t>, uint32_t, KeyHash> first;   // key -> its first entry in locs
    std::vector<uint8_t> trust;
};

// (inline: vmig_plan.cpp cuts a snapshot's block list against the index and is built without this module)
inline void BaseIndex::build(const BlockTable& table, const std::vector<uint8_t>& trusted)
{
    t = &table; trust = trusted; locs.clear(); first.clear();
    for (uint32_t f = 0; f < table.files.size(); f++) {
        if (!trusted[f]) continue;
        const uint64_t nb = table.blocks_of(table.files[f]);
        for (uint64_t r = 0; r < nb; r++) locs.push_back({hash_of(f, r), block_len(f, r), f, r});
    }
    std::sort(locs.begin(), locs.end(), [](const Loc& a, const Loc& b) {
        if (a.hash != b.hash) return a.hash < b.hash;
        if (a.len != b.len) return a.len < b.len;
        return a.file != b.file ? a.file < b.file : a.block < b.block;
    });
    first.reserve(locs.size());
    for (uint32_t i = 0; i < locs.size(); i++) first.emplace(std::make_pair(locs[i].hash, locs[i].len), i);   // keeps the first
}

inline const BaseIndex::Loc* BaseIndex::find(uint64_t hash, uint32_t len, size_t* n) const
{
    *n = 0;
    auto it = first.find(std::make_pair(hash, len));
    if (it == first.end()) return nullptr;
    size_t j = it->second;
    while (j < locs.size() && locs[j].hash == hash && locs[j].len == len) j++;
    *n = j - it->second;
    return &locs[it->second];
}

inline uint32_t BaseIndex::block_len(uint32_t file, uint64_t block) const
{
    const TableFile& f = t->files[file];
    const uint64_t off = block * (uint64_t)t->block_bytes;
    return off < f.size ? (uint32_t)std::min<uint64_t>(t->block_bytes, f.size - off) : 0;
}

// One piece of a snapshot file's backfill: bytes [src_off, src_off + len) of base file `file` go to [dst_off, ...) of
// the new file.  Both offsets are multiples of block_bytes; len is whole blocks, except that a run ending in the file's
// short last block ends there.
struct ReuseRun { uint32_t file; uint64_t src_off; uint64_t dst_off; uint64_t len; };

// Plan the backfill of one new file of `size` bytes whose block hashes are hashes[0..n) and whose blocks with
// skipped[r] != 0 were not written from the staging ring.  Each such block takes its bytes from
//   1. block r of the same-path base file `same` (-1: none) when that block's key matches;
//   2. else the block that continues the previous block's base run (G, r' + 1) when its key matches;
//   3. else the first index entry with its key.
// Runs contiguous in the new file and in one base file are coalesced.  VMIG_ECORRUPT (naming `what`) if a skipped block
// has no source: the hash-waiter only skips blocks the index or the same-path record holds.
int plan_backfill(const BaseIndex& idx, int same, uint64_t size, uint32_t block_bytes, const uint64_t* hashes,
                  const uint8_t* skipped, const std::string& what, std::vector<ReuseRun>* out);

// Base files the new file could be a hard link to: trusted, `size` bytes, every block hash equal to hashes[] at the same
// index.  The same-path file first, then the others in table order; at most max_out of them, found among the first
// kLinkScan index entries of the file's first block (a block common to the whole base, an all-zero one say, must not
// make every file's finalization walk the base).
static constexpr size_t kLinkScan = 4096;
void link_candidates(const BaseIndex& idx, int same, uint64_t size, uint32_t block_bytes, const uint64_t* hashes,
                     std::vector<uint32_t>* out, size_t max_out);

}  // namespace vmig
