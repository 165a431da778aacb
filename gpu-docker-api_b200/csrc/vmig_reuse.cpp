// vmig_reuse.cpp -- the content index of a snapshot's base and the planning of what each new file takes from it
// (vmig_reuse.h).  Host code only: no CUDA, so tests/reuse_unit.cpp compiles it with g++.
#include "vmig_reuse.h"
#include "vmig_common.h"
#include <algorithm>

namespace vmig {

int plan_backfill(const BaseIndex& idx, int same, uint64_t size, uint32_t block_bytes, const uint64_t* hashes,
                  const uint8_t* skipped, const std::string& what, std::vector<ReuseRun>* out)
{
    out->clear();
    const uint64_t nb = (size + block_bytes - 1) / block_bytes;
    // the base block of this file's previous block (prev_file == UINT32_MAX: it came from the ring, or r == 0)
    uint32_t prev_file = UINT32_MAX; uint64_t prev_block = 0;
    for (uint64_t r = 0; r < nb; r++) {
        if (!skipped[r]) { prev_file = UINT32_MAX; continue; }
        const uint64_t off = r * (uint64_t)block_bytes;
        const uint32_t len = (uint32_t)std::min<uint64_t>(block_bytes, size - off);
        auto matches = [&](uint32_t g, uint64_t b) { return idx.trusted(g) && idx.block_len(g, b) == len && idx.hash_of(g, b) == hashes[r]; };
        uint32_t g; uint64_t b;
        if (same >= 0 && matches((uint32_t)same, r)) { g = (uint32_t)same; b = r; }
        else if (prev_file != UINT32_MAX && matches(prev_file, prev_block + 1)) { g = prev_file; b = prev_block + 1; }
        else {
            size_t n;
            const BaseIndex::Loc* l = idx.find(hashes[r], len, &n);
            if (!l) return fail(VMIG_ECORRUPT, "%s block %llu was skipped, but the base holds no block with its hash %016llx", what.c_str(),
                                (unsigned long long)r, (unsigned long long)hashes[r]);
            g = l->file; b = l->block;
        }
        const uint64_t src_off = b * (uint64_t)block_bytes;
        ReuseRun* last = out->empty() ? nullptr : &out->back();
        if (last && last->file == g && last->dst_off + last->len == off && last->src_off + last->len == src_off) last->len += len;
        else out->push_back({g, src_off, off, len});
        prev_file = g; prev_block = b;
    }
    return VMIG_OK;
}

void link_candidates(const BaseIndex& idx, int same, uint64_t size, uint32_t block_bytes, const uint64_t* hashes,
                     std::vector<uint32_t>* out, size_t max_out)
{
    out->clear();
    if (!size || !max_out) return;
    const uint64_t nb = (size + block_bytes - 1) / block_bytes;
    auto equal = [&](uint32_t g) {
        if (!idx.trusted(g) || idx.t->files[g].size != size) return false;
        for (uint64_t r = 0; r < nb; r++) if (idx.hash_of(g, r) != hashes[r]) return false;
        return true;
    };
    if (same >= 0 && equal((uint32_t)same)) out->push_back((uint32_t)same);
    size_t n;
    const BaseIndex::Loc* l = idx.find(hashes[0], (uint32_t)std::min<uint64_t>(block_bytes, size), &n);
    n = std::min(n, kLinkScan);
    for (size_t i = 0; i < n && out->size() < max_out; i++)       // entries of one key are in table order
        if (l[i].block == 0 && (int64_t)l[i].file != same && equal(l[i].file)) out->push_back(l[i].file);
}

}  // namespace vmig
