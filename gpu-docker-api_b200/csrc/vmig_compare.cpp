// vmig_compare.cpp -- the host side of vmig_compare_snapshot (see vmig_compare.h).
#include "vmig_compare.h"
#include "vmig_common.h"

#include <sys/stat.h>
#include <sys/sysmacros.h>
#include <algorithm>
#include <tuple>
#include <unordered_map>
#include <utility>

namespace vmig {

const char* compare_kind_name(CompareKind k)
{
    static const char* const names[] = {"added", "removed", "type", "resized", "block", "target", "rdev", "hardlink",
                                        "mode", "owner", "mtime"};
    return k <= kCmpMtime ? names[k] : "?";
}

int compare_plan(const std::string& layer_root, const Manifest& layer, const Manifest& snap, const BlockTable* layer_tab,
                 uint32_t block_bytes, ComparePlan* out)
{
    ComparePlan& p = *out;
    p = ComparePlan();
    const size_t n = layer.files.size();
    p.snap_of.assign(n, -1); p.source.assign(n, kCmpNone); p.rec_of.assign(n, -1);
    std::vector<std::vector<int64_t>> sel(1, std::vector<int64_t>(n, -1));
    for (size_t i = 0, j = 0; i < n; i++) {               // both file lists are sorted bytewise
        const Entry& e = layer.files[i];
        while (j < snap.files.size() && snap.files[j].rel < e.rel) j++;
        if (j == snap.files.size() || snap.files[j].rel != e.rel) continue;
        p.snap_of[i] = (int64_t)j;
        const Entry& s = snap.files[j];
        if (e.n_blocks == 0 || s.n_blocks == 0) continue;
        if (e.dev == s.dev && e.ino == s.ino && e.size == s.size) { p.source[i] = kCmpShared; p.files_shared++; continue; }
        if (layer_tab) {
            auto it = layer_tab->index.find(e.rel);
            if (it != layer_tab->index.end()) {
                struct stat st;                 // trusted only while it is still the inode the walk saw and the record's file
                if (lstat(pjoin(layer_root, e.rel).c_str(), &st) == 0 && (uint64_t)st.st_dev == e.dev && (uint64_t)st.st_ino == e.ino &&
                    (uint64_t)st.st_size == e.size &&
                    is_recorded_file(st, layer_tab->files[it->second])) {
                    p.source[i] = kCmpTrusted; p.rec_of[i] = (int64_t)it->second; p.files_trusted++;
                    continue;
                }
            }
        }
        p.source[i] = kCmpRead;
        sel[0][i] = 0;
    }
    std::vector<std::vector<uint32_t>> inode_of;
    const int rc = scrub_group_inodes({&layer}, sel, block_bytes, &p.inodes, &inode_of);
    if (rc) return rc;
    p.inode_of = std::move(inode_of[0]);
    for (const ScrubInode& I : p.inodes) { p.bytes_read += I.size; p.blocks_read += I.n_blocks; }
    return VMIG_OK;
}

std::vector<const uint64_t*> compare_layer_hashes(const ComparePlan& p, const Manifest& layer, const Manifest& snap,
                                                  const std::vector<uint64_t>& snap_hashes, const BlockTable* layer_tab,
                                                  const std::vector<uint64_t>& read_hashes)
{
    std::vector<const uint64_t*> h(layer.files.size(), nullptr);
    for (size_t i = 0; i < layer.files.size(); i++) {
        switch (p.source[i]) {
        case kCmpShared: h[i] = snap_hashes.data() + snap.files[(size_t)p.snap_of[i]].first_block; break;
        case kCmpTrusted: h[i] = layer_tab->hashes.data() + layer_tab->files[(size_t)p.rec_of[i]].first_block; break;
        case kCmpRead: h[i] = read_hashes.data() + p.inodes[p.inode_of[i]].first_block; break;
        default: break;
        }
    }
    return h;
}

namespace {

char type_letter(mode_t m)
{
    switch (m & S_IFMT) {
    case S_IFREG: return 'f';
    case S_IFDIR: return 'd';
    case S_IFLNK: return 'l';
    case S_IFCHR: return 'c';
    case S_IFBLK: return 'b';
    case S_IFIFO: return 'p';
    default: return '?';
    }
}

std::string hex16(uint64_t h) { char b[24]; snprintf(b, sizeof b, "%016llx", (unsigned long long)h); return b; }

std::string mtime_str(const struct timespec& t, bool ns)
{
    char b[48];
    if (ns) snprintf(b, sizeof b, "%lld.%09ld", (long long)t.tv_sec, (long)t.tv_nsec);
    else snprintf(b, sizeof b, "%lld", (long long)t.tv_sec);
    return b;
}

// One tree's entries in path order, and each regular file's in-tree hard-link group (its paths, sorted)
struct Side {
    const Manifest* m;
    std::vector<const Entry*> all;
    std::unordered_map<std::string, size_t> file_of;      // rel -> files[] index
    std::unordered_map<int64_t, std::vector<size_t>> groups;   // primary -> every member (primary first), only groups of >1
    explicit Side(const Manifest& man) : m(&man) {
        for (const auto* v : {&man.dirs, &man.files, &man.symlinks, &man.specials})
            for (const Entry& e : *v) all.push_back(&e);
        std::sort(all.begin(), all.end(), [](const Entry* a, const Entry* b) { return a->rel < b->rel; });
        for (size_t f = 0; f < man.files.size(); f++) {
            file_of.emplace(man.files[f].rel, f);
            const int64_t h = man.files[f].hardlink_of;
            if (h >= 0) {
                auto& g = groups[h];
                if (g.empty()) g.push_back((size_t)h);
                g.push_back(f);
            }
        }
    }
    // the paths of f's group; a file alone has only itself
    std::vector<std::string> group(size_t f) const {
        const int64_t h = m->files[f].hardlink_of >= 0 ? m->files[f].hardlink_of : (int64_t)f;
        auto it = groups.find(h);
        if (it == groups.end()) return {m->files[f].rel};
        std::vector<std::string> out;
        for (size_t x : it->second) out.push_back(m->files[x].rel);
        return out;
    }
};

}  // namespace

void compare_merge(const Manifest& layer, const Manifest& snap, const std::vector<uint64_t>& snap_hashes,
                   const std::vector<const uint64_t*>& layer_hashes, uint32_t block_bytes, bool mtime_ns, bool no_metadata,
                   std::vector<CompareFinding>* out, CompareCounts* counts)
{
    out->clear();
    CompareCounts c;
    const Side L(layer), S(snap);
    auto add = [&](CompareKind k, const std::string& rel, std::string lv = "-", std::string sv = "-", int64_t block = -1) {
        CompareFinding f; f.kind = k; f.path = rel; f.block = block; f.layer = std::move(lv); f.snap = std::move(sv);
        out->push_back(std::move(f));
    };
    size_t i = 0, j = 0;
    while (i < L.all.size() || j < S.all.size()) {
        if (j == S.all.size() || (i < L.all.size() && L.all[i]->rel < S.all[j]->rel)) { add(kCmpAdded, L.all[i]->rel); c.paths_added++; i++; continue; }
        if (i == L.all.size() || S.all[j]->rel < L.all[i]->rel) {
            const Entry& s = *S.all[j];
            add(kCmpRemoved, s.rel); c.paths_removed++;
            if (s.type == kFile) c.bytes_restore += s.size;
            j++;
            continue;
        }
        const Entry& l = *L.all[i++];
        const Entry& s = *S.all[j++];
        const size_t before = out->size();
        const mode_t lt = l.mode & S_IFMT, st = s.mode & S_IFMT;
        if (lt != st) {
            add(kCmpType, l.rel, std::string(1, type_letter(l.mode)), std::string(1, type_letter(s.mode)));
            if (s.type == kFile) c.bytes_restore += s.size;
        } else if (l.rel != ".") {
            if (lt == S_IFREG) {
                const size_t lf = L.file_of.at(l.rel), sf = S.file_of.at(s.rel);
                bool changed = false;
                if (l.size != s.size) { add(kCmpResized, l.rel, std::to_string(l.size), std::to_string(s.size)); changed = true; }
                const uint64_t* lh = layer_hashes[lf];
                const uint64_t* sh = snap_hashes.data() + s.first_block;
                for (uint64_t r = 0; r < s.n_blocks; r++) {
                    const uint64_t slen = std::min<uint64_t>(block_bytes, s.size - r * block_bytes);
                    bool differs = r >= l.n_blocks;
                    if (!differs) {
                        const uint64_t llen = std::min<uint64_t>(block_bytes, l.size - r * block_bytes);
                        differs = llen != slen || lh[r] != sh[r];
                        if (differs) { add(kCmpBlock, l.rel, hex16(lh[r]), hex16(sh[r]), (int64_t)r); c.blocks_changed++; changed = true; }
                    }
                    if (differs) c.bytes_restore += slen;
                }
                c.files_changed += changed;
                const std::vector<std::string> lg = L.group(lf), sg = S.group(sf);
                if (lg != sg)
                    add(kCmpHardlink, l.rel, lg.size() > 1 ? scrub_escape(lg[0]) : "-", sg.size() > 1 ? scrub_escape(sg[0]) : "-");
            } else if (lt == S_IFLNK) {
                if (l.target != s.target) add(kCmpTarget, l.rel, scrub_escape(l.target), scrub_escape(s.target));
            } else if (lt == S_IFCHR || lt == S_IFBLK) {
                if (l.rdev != s.rdev)
                    add(kCmpRdev, l.rel, std::to_string(major(l.rdev)) + ":" + std::to_string(minor(l.rdev)),
                        std::to_string(major(s.rdev)) + ":" + std::to_string(minor(s.rdev)));
            }
        }
        if (lt == st && !no_metadata) {
            char a[16], b[16];
            if ((l.mode & 07777) != (s.mode & 07777)) {
                snprintf(a, sizeof a, "%04o", (unsigned)(l.mode & 07777)); snprintf(b, sizeof b, "%04o", (unsigned)(s.mode & 07777));
                add(kCmpMode, l.rel, a, b);
            }
            if (l.uid != s.uid || l.gid != s.gid)
                add(kCmpOwner, l.rel, std::to_string(l.uid) + ":" + std::to_string(l.gid), std::to_string(s.uid) + ":" + std::to_string(s.gid));
            if (l.mtime.tv_sec != s.mtime.tv_sec || (mtime_ns && l.mtime.tv_nsec != s.mtime.tv_nsec))
                add(kCmpMtime, l.rel, mtime_str(l.mtime, mtime_ns), mtime_str(s.mtime, mtime_ns));
        }
        c.paths_changed += out->size() != before;
    }
    compare_sort(out);
    *counts = c;
}

std::string compare_format(const CompareFinding& f)
{
    std::string line = std::string(compare_kind_name(f.kind)) + "\t" + scrub_escape(f.path) + "\t";
    line += f.block >= 0 ? std::to_string(f.block) : "-";
    return line + "\t" + f.layer + "\t" + f.snap + "\n";
}

void compare_sort(std::vector<CompareFinding>* v)
{
    std::stable_sort(v->begin(), v->end(), [](const CompareFinding& a, const CompareFinding& b) {
        return std::tie(a.path, a.kind, a.block) < std::tie(b.path, b.kind, b.block);
    });
}

}  // namespace vmig
