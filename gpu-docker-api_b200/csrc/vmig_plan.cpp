// vmig_plan.cpp -- the plan of a tree call (see vmig_plan.h).
#include "vmig_plan.h"
#include "vmig_common.h"

#include <algorithm>

namespace vmig {

void interleave_blocks(const std::vector<BlockSpan>& spans, uint32_t block_bytes, std::vector<BlockRef>* out)
{
    for (size_t g = 0; g < spans.size(); g += 64) {
        const size_t g1 = std::min(spans.size(), g + 64);
        uint64_t maxb = 0;
        for (size_t i = g; i < g1; i++) maxb = std::max(maxb, spans[i].n_blocks);
        for (uint64_t r = 0; r < maxb; r++)
            for (size_t i = g; i < g1; i++) {
                const BlockSpan& s = spans[i];
                if (r >= s.n_blocks) continue;
                BlockRef b; b.file = s.file; b.file_off = r * (uint64_t)block_bytes;
                b.len = (uint32_t)std::min<uint64_t>(block_bytes, s.size - b.file_off);
                b.table_idx = s.first_block + r; b.prior_hash = 0; b.prior_valid = 0;
                out->push_back(b);
            }
    }
}

int plan_tree(const Manifest& man, uint32_t block_bytes, const std::string& dst_root, const BlockTable* prior,
              const std::string& base_root, const BlockTable* base, const std::atomic<int>* cancel, TreePlan* out,
              const std::string& src_root, const BlockTable* layer)
{
    *out = TreePlan();
    out->files.resize(man.files.size());
    if (base) {
        // a base file's link count may exceed 1: base files are shared with older snapshots
        out->base_trusted.assign(base->files.size(), 0);
        for (size_t i = 0; i < base->files.size(); i++) {
            const TableFile& bf = base->files[i];
            if (i % kMetaCheckEvery == 0 && cancel && cancel->load()) return fail(VMIG_ECANCELED, "while checking the base's files");
            struct stat bs;
            out->base_trusted[i] = bf.ino != 0 && lstat(pjoin(base_root, bf.rel).c_str(), &bs) == 0 && is_recorded_file(bs, bf);
        }
        out->bidx.build(*base, out->base_trusted);
    }
    if (layer) {
        out->layer_hashes.assign(man.n_blocks, 0); out->skipped.assign(man.n_blocks, 0); out->expect.assign(man.n_blocks, 0);
    }
    for (const Entry& e : man.files) if (e.hardlink_of >= 0) out->files[(size_t)e.hardlink_of].solo = false;
    std::vector<BlockSpan> spans;
    for (uint32_t f = 0; f < man.files.size(); f++) {
        const Entry& e = man.files[f];
        if (e.hardlink_of >= 0 || e.n_blocks == 0) continue;
        FilePlan& p = out->files[f];
        if (base) {
            auto it = base->index.find(e.rel);
            if (it != base->index.end() && base->files[it->second].ino != 0) {
                if (out->base_trusted[it->second]) { p.base_rec = &base->files[it->second]; out->any_base = true; }
                else out->files_base_untrusted++;
            }
        }
        if (prior) {
            // any write, truncate, chmod or replacement since the table was written moved the file's ctime
            auto it = prior->index.find(e.rel);
            struct stat ds;
            if (it != prior->index.end() && prior->files[it->second].ino != 0 && lstat(pjoin(dst_root, e.rel).c_str(), &ds) == 0 &&
                S_ISREG(ds.st_mode) && ds.st_nlink == 1) {
                if (is_recorded_file(ds, prior->files[it->second])) p.prior_rec = &prior->files[it->second];
                else out->files_untrusted++;
            }
        }
        if (layer) {
            // the same skip the tree call makes after reading: a snapshot's, every block whose (hash, length) a trusted
            // base file holds, the same-path one included (base_rec is only set for a trusted base file); a migration's
            // (vmig_migrate_layer, no base), every block whose (hash, length) is the prior record's at the same index
            auto it = layer->index.find(e.rel);
            struct stat ls;
            if (it != layer->index.end() && lstat(pjoin(src_root, e.rel).c_str(), &ls) == 0 && (uint64_t)ls.st_ino == e.ino &&
                (uint64_t)ls.st_size == e.size && is_recorded_file(ls, layer->files[it->second])) {
                p.layer_rec = &layer->files[it->second];
                out->files_trusted++; out->bytes_trusted += e.size;
                uint64_t n_read = 0, b_read = 0;
                for (uint64_t r = 0; r < e.n_blocks; r++) {
                    const uint64_t h = layer->hashes[p.layer_rec->first_block + r];
                    const uint32_t len = (uint32_t)std::min<uint64_t>(block_bytes, e.size - r * block_bytes);
                    out->layer_hashes[e.first_block + r] = h;
                    const uint64_t off = r * (uint64_t)block_bytes;
                    const bool same_prior = p.prior_rec && off < p.prior_rec->size &&
                                            std::min<uint64_t>(block_bytes, p.prior_rec->size - off) == len &&
                                            prior->hashes[p.prior_rec->first_block + r] == h;
                    if (same_prior || out->bidx.contains(h, len)) out->skipped[e.first_block + r] = 1;
                    else { out->expect[e.first_block + r] = 1; n_read++; b_read += len; }
                }
                if (!n_read) { out->unread.push_back(f); continue; }
                out->files_read++; out->bytes_read += b_read;
                spans.push_back({f, e.size, e.first_block, e.n_blocks});
                continue;
            }
            out->files_read++; out->bytes_read += e.size;
        }
        spans.push_back({f, e.size, e.first_block, e.n_blocks});
    }
    out->blocks.reserve(man.n_blocks);
    interleave_blocks(spans, block_bytes, &out->blocks);
    if (layer) out->blocks.erase(std::remove_if(out->blocks.begin(), out->blocks.end(), [&](const BlockRef& b) { return out->skipped[b.table_idx] != 0; }),
                                 out->blocks.end());
    // the same rule for a file patched in place and for a snapshot file whose base is trusted
    for (BlockRef& b : out->blocks) {
        const FilePlan& p = out->files[b.file];
        const TableFile* rec = p.prior_rec ? p.prior_rec : p.base_rec;
        if (!rec) continue;
        const BlockTable& t = p.prior_rec ? *prior : *base;
        const uint64_t plen = b.file_off < rec->size ? std::min<uint64_t>(block_bytes, rec->size - b.file_off) : 0;
        if (plen == b.len) { b.prior_hash = t.hashes[rec->first_block + b.file_off / block_bytes]; b.prior_valid = 1; }
    }
    return VMIG_OK;
}

bool live_identity_holds(const struct stat& before, int64_t clock_ns, const struct stat& after)
{
    return S_ISREG(before.st_mode) && before.st_nlink == 1 && ctime_ns(before) < clock_ns &&
           after.st_ino == before.st_ino && after.st_size == before.st_size && ctime_ns(after) == ctime_ns(before);
}

}  // namespace vmig
