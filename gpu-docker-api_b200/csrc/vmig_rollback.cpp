// vmig_rollback.cpp -- the host side of vmig_rollback_layer (see vmig_rollback.h).
#include "vmig_rollback.h"
#include "vmig_common.h"
#include "vmig_table.h"

#include <algorithm>

namespace vmig {

const char* rollback_action_name(RollbackAction a)
{
    static const char* const names[] = {"keep", "patch", "rebuild", "create"};
    return a <= kRbCreate ? names[a] : "?";
}

LayerId layer_id_of(const struct stat& st)
{
    LayerId id;
    id.set = true; id.ino = (uint64_t)st.st_ino; id.size = (uint64_t)st.st_size; id.nlink = (uint64_t)st.st_nlink;
    id.ctime_ns = ctime_ns(st);
    return id;
}

int rollback_identify(const std::string& layer_root, const Manifest& layer, const ComparePlan& cp, const BlockTable* layer_tab,
                      std::vector<LayerId>* out)
{
    out->assign(layer.files.size(), LayerId());
    for (size_t i = 0; i < layer.files.size(); i++) {
        if (cp.snap_of[i] < 0) continue;
        const std::string p = pjoin(layer_root, layer.files[i].rel);
        struct stat st;
        if (lstat(p.c_str(), &st) != 0 || !S_ISREG(st.st_mode) || (uint64_t)st.st_ino != layer.files[i].ino)
            return fail(VMIG_ESRCCHANGED, "layer file %s changed since the walk", p.c_str());
        LayerId& id = (*out)[i];
        id = layer_id_of(st);
        if (cp.source[i] == kCmpTrusted) {          // the hashes are the record's: so is the identity they speak for
            const TableFile& r = layer_tab->files[(size_t)cp.rec_of[i]];
            id.ino = r.ino; id.size = r.size; id.ctime_ns = r.ctime_ns;
        }
    }
    return VMIG_OK;
}

int rollback_recheck_paths(const std::string& layer_root, const Manifest& layer, const std::vector<LayerId>& ids)
{
    for (size_t i = 0; i < layer.files.size(); i++) {
        if (!ids[i].set) continue;
        const std::string p = pjoin(layer_root, layer.files[i].rel);
        struct stat st;
        const LayerId& id = ids[i];
        if (lstat(p.c_str(), &st) != 0 || !S_ISREG(st.st_mode) || (uint64_t)st.st_ino != id.ino || (uint64_t)st.st_size != id.size ||
            ctime_ns(st) != id.ctime_ns)
            return fail(VMIG_ESRCCHANGED, "layer file %s changed while the layer was hashed", p.c_str());
    }
    return VMIG_OK;
}

int rollback_check_fd(int fd, const LayerId& id, const std::string& path)
{
    struct stat st;
    if (fstat(fd, &st) != 0 || !S_ISREG(st.st_mode) || (uint64_t)st.st_ino != id.ino || (uint64_t)st.st_size != id.size ||
        ctime_ns(st) != id.ctime_ns)
        return fail(VMIG_ESRCCHANGED, "layer file %s is no longer the file the rollback planned from (inode, size or ctime moved)",
                    path.c_str());
    return VMIG_OK;
}

int RebuildGuard::clear(int old_fd, const LayerId& id, bool check, const std::string& path)
{
    std::lock_guard<std::mutex> lk(mu);
    if (check) {
        LayerId want = id;
        auto it = own_ctime.find(id.ino);
        if (it != own_ctime.end()) want.ctime_ns = it->second;
        const int rc = rollback_check_fd(old_fd, want, path);
        if (rc) return rc;
    }
    const int rc = clear_path(path, "a regular file");      // tar replaces what is there
    if (rc) return rc;
    struct stat st;
    if (fstat(old_fd, &st) == 0 && st.st_nlink > 0) own_ctime[(uint64_t)st.st_ino] = ctime_ns(st);
    return VMIG_OK;
}

namespace {

// f is in an in-tree hard-link group: a secondary path, or the primary some other path links to
std::vector<uint8_t> grouped(const Manifest& m)
{
    std::vector<uint8_t> g(m.files.size(), 0);
    for (size_t f = 0; f < m.files.size(); f++)
        if (m.files[f].hardlink_of >= 0) { g[f] = 1; g[(size_t)m.files[f].hardlink_of] = 1; }
    return g;
}

}  // namespace

void rollback_plan(const Manifest& layer, const Manifest& snap, const std::vector<uint64_t>& snap_hashes, const ComparePlan& cp,
                   const std::vector<const uint64_t*>& layer_hashes, const std::vector<LayerId>& ids, uint32_t block_bytes,
                   uid_t euid, RollbackPlan* out)
{
    RollbackPlan& p = *out;
    p = RollbackPlan();
    std::vector<int64_t> layer_at(snap.files.size(), -1);
    for (size_t i = 0; i < layer.files.size(); i++) if (cp.snap_of[i] >= 0) layer_at[(size_t)cp.snap_of[i]] = (int64_t)i;
    const std::vector<uint8_t> lg = grouped(layer), sg = grouped(snap);
    for (uint32_t j = 0; j < snap.files.size(); j++) {
        const Entry& s = snap.files[j];
        if (s.hardlink_of >= 0) continue;
        RollbackFile rf;
        rf.snap = j; rf.layer = layer_at[j];
        const uint32_t fi = (uint32_t)p.files.size();
        const uint64_t* sh = snap_hashes.data() + s.first_block;
        const uint64_t* lh = nullptr;
        uint64_t l_blocks = 0, l_size = 0;
        bool in_place = false, writable = false;     // patchable == in_place && writable
        if (rf.layer >= 0) {
            const size_t l = (size_t)rf.layer;
            const Entry& e = layer.files[l];
            lh = layer_hashes[l]; l_blocks = e.n_blocks; l_size = e.size;
            in_place = cp.source[l] != kCmpShared && ids[l].set && ids[l].nlink == 1 && !lg[l] && !sg[j];
            writable = euid == 0 || (e.uid == euid && (e.mode & S_IWUSR));
        }
        // block r is equal when the layer holds it with the same (length, hash); everything else is fetched
        bool all_equal = rf.layer >= 0 && l_size == s.size;
        std::vector<CopyRun> runs;
        for (uint64_t r = 0; r < s.n_blocks; r++) {
            const uint64_t off = r * block_bytes;
            const uint32_t slen = (uint32_t)std::min<uint64_t>(block_bytes, s.size - off);
            const bool equal = lh && r < l_blocks && std::min<uint64_t>(block_bytes, l_size - off) == slen && lh[r] == sh[r];
            if (equal) {
                if (!runs.empty() && runs.back().off + runs.back().len == off) runs.back().len += slen;
                else runs.push_back({fi, off, slen});
                continue;
            }
            all_equal = false;
            BlockRef b;
            b.file = fi; b.len = slen; b.file_off = off; b.table_idx = s.first_block + r; b.prior_hash = 0; b.prior_valid = 0;
            p.fetch.push_back(b);
            rf.n_fetch++;
            p.blocks_fetched++; p.bytes_fetched += slen;
        }
        // a kept file is not written, so it need not be writable
        rf.action = rf.layer < 0 ? kRbCreate : in_place && all_equal ? kRbKeep : in_place && writable ? kRbPatch : kRbRebuild;
        switch (rf.action) {
        case kRbKeep: p.files_kept++; break;
        case kRbPatch: p.files_patched++; break;
        case kRbCreate: p.files_created++; break;
        case kRbRebuild:
            p.files_rebuilt++;
            rf.first_run = p.runs.size(); rf.n_runs = runs.size();
            for (const CopyRun& u : runs) { p.runs.push_back(u); p.bytes_copied += u.len; }
            break;
        }
        p.files.push_back(rf);
    }
}

}  // namespace vmig
