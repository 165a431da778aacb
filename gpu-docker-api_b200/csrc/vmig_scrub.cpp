// vmig_scrub.cpp -- the host side of vmig_scrub_store (see vmig_scrub.h).
#include "vmig_scrub.h"
#include "vmig_common.h"

#include <fcntl.h>
#include <unistd.h>
#include <sys/stat.h>
#include <sys/syscall.h>
#include <algorithm>
#include <cctype>
#include <cstdlib>
#include <tuple>
#include <utility>

namespace vmig {

const char* scrub_kind_name(ScrubKind k)
{
    static const char* const names[] = {"missing", "extra", "resized", "block", "hardlink", "unreadable", "table", "dir"};
    return k <= kScrubDir ? names[k] : "?";
}

size_t scrub_merge_table(uint32_t version, const Manifest& man, const BlockTable& t, std::vector<int64_t>* tab_of,
                         std::vector<ScrubFinding>* out)
{
    tab_of->assign(man.files.size(), -1);
    size_t i = 0, j = 0, n = 0;
    auto add = [&](ScrubKind k, const std::string& rel) {
        ScrubFinding f; f.version = version; f.kind = k; f.path = rel;
        out->push_back(std::move(f)); n++;
    };
    while (i < man.files.size() || j < t.files.size()) {
        if (j == t.files.size() || (i < man.files.size() && man.files[i].rel < t.files[j].rel)) { add(kScrubExtra, man.files[i].rel); i++; continue; }
        if (i == man.files.size() || t.files[j].rel < man.files[i].rel) { add(kScrubMissing, t.files[j].rel); j++; continue; }
        if (man.files[i].size != t.files[j].size) add(kScrubResized, man.files[i].rel);
        else (*tab_of)[i] = (int64_t)j;
        i++; j++;
    }
    return n;
}

int InodeGroups::add(uint64_t dev, uint64_t ino, uint64_t size, uint32_t version, const std::string& rel, uint32_t* u)
{
    auto it = seen.find({dev, ino});
    if (it == seen.end()) {
        const uint64_t nb = (size + block_bytes - 1) / block_bytes;
        it = seen.emplace(std::make_pair(dev, ino), (uint32_t)inodes->size()).first;
        inodes->push_back({dev, ino, size, next_block, nb, version, rel});
        next_block += nb;
    } else if ((*inodes)[it->second].size != size) {
        const ScrubInode& I = (*inodes)[it->second];
        return fail(VMIG_ESRCCHANGED, "inode %llu is %llu bytes as version %u's %s and %llu bytes as version %u's %s: the store changed during the %s",
                    (unsigned long long)ino, (unsigned long long)I.size, I.version, I.rel.c_str(), (unsigned long long)size, version, rel.c_str(), call);
    }
    *u = it->second;
    return VMIG_OK;
}

int scrub_group_inodes(const std::vector<const Manifest*>& mans, const std::vector<std::vector<int64_t>>& sel,
                       uint32_t block_bytes, std::vector<ScrubInode>* inodes, std::vector<std::vector<uint32_t>>* inode_of)
{
    inodes->clear();
    inode_of->assign(mans.size(), {});
    InodeGroups groups{inodes, block_bytes, "scrub"};
    for (size_t v = 0; v < mans.size(); v++) {
        if (!mans[v]) continue;
        const Manifest& m = *mans[v];
        (*inode_of)[v].assign(m.files.size(), kNoInode);
        for (size_t f = 0; f < m.files.size() && f < sel[v].size(); f++) {
            const Entry& e = m.files[f];
            if (sel[v][f] < 0 || e.size == 0) continue;
            const int rc = groups.add(e.dev, e.ino, e.size, (uint32_t)v, e.rel, &(*inode_of)[v][f]);
            if (rc) return rc;
        }
    }
    return VMIG_OK;
}

std::string scrub_escape(const std::string& s)
{
    std::string o;
    o.reserve(s.size());
    for (unsigned char c : s) {
        if (c == '\\') o += "\\\\";
        else if (c == '\t') o += "\\t";
        else if (c == '\n') o += "\\n";
        else if (c < 0x20) { char b[8]; snprintf(b, sizeof b, "\\x%02x", c); o += b; }
        else o += (char)c;
    }
    return o;
}

bool scrub_unescape(const std::string& s, std::string* out)
{
    out->clear();
    for (size_t i = 0; i < s.size(); i++) {
        if (s[i] != '\\') { *out += s[i]; continue; }
        if (++i == s.size()) return false;
        if (s[i] == '\\') *out += '\\';
        else if (s[i] == 't') *out += '\t';
        else if (s[i] == 'n') *out += '\n';
        else if (s[i] == 'x' && i + 2 < s.size() && isxdigit((unsigned char)s[i + 1]) && isxdigit((unsigned char)s[i + 2])) {
            *out += (char)strtoul(s.substr(i + 1, 2).c_str(), nullptr, 16);
            i += 2;
        } else return false;
    }
    return true;
}

std::string scrub_format(const ScrubFinding& f)
{
    char b[96];
    std::string line = std::to_string(f.version) + "\t" + scrub_kind_name(f.kind) + "\t" + scrub_escape(f.path) + "\t";
    line += f.block >= 0 ? std::to_string(f.block) : "-";
    if (f.has_hashes) { snprintf(b, sizeof b, "\t%016llx\t%016llx\n", (unsigned long long)f.got, (unsigned long long)f.want); line += b; }
    else line += "\t-\t-\n";
    return line;
}

void scrub_sort(std::vector<ScrubFinding>* v)
{
    std::stable_sort(v->begin(), v->end(), [](const ScrubFinding& a, const ScrubFinding& b) {
        return std::tie(a.version, a.path, a.block) < std::tie(b.version, b.path, b.block);
    });
}

int report_store(const std::string& path, const std::string& raw, const char* what, const std::atomic<int>* cancel)
{
    if (cancel && cancel->load()) return fail(VMIG_ECANCELED, "cancelled before the %s %s was written", what, path.c_str());
    const std::string tmp = path + ".tmp." + std::to_string((long)getpid()) + "." + std::to_string((long)syscall(SYS_gettid));
    int fd = open(tmp.c_str(), O_WRONLY | O_CREAT | O_TRUNC | O_CLOEXEC, 0644);
    if (fd < 0) return fail(VMIG_EIO, "create %s: %s", tmp.c_str(), errno_str(errno).c_str());
    size_t put = 0;
    while (put < raw.size()) {
        ssize_t w = write(fd, raw.data() + put, raw.size() - put);
        if (w <= 0) { const int e = errno; close(fd); unlink(tmp.c_str()); return fail(VMIG_EIO, "write %s: %s", tmp.c_str(), errno_str(e).c_str()); }
        put += (size_t)w;
    }
    if (fsync(fd) != 0) { const int e = errno; close(fd); unlink(tmp.c_str()); return fail(VMIG_EIO, "fsync %s: %s", tmp.c_str(), errno_str(e).c_str()); }
    close(fd);
    if (cancel && cancel->load()) { unlink(tmp.c_str()); return fail(VMIG_ECANCELED, "cancelled before the %s %s was renamed into place", what, path.c_str()); }
    if (rename(tmp.c_str(), path.c_str()) != 0) { const int e = errno; unlink(tmp.c_str()); return fail(VMIG_EIO, "rename %s: %s", path.c_str(), errno_str(e).c_str()); }
    return VMIG_OK;
}

int scrub_report_store(const std::string& path, const std::vector<ScrubFinding>& v, const std::atomic<int>* cancel)
{
    std::string raw;
    for (const ScrubFinding& f : v) raw += scrub_format(f);
    return report_store(path, raw, "scrub report", cancel);
}

// ---------------------------------------------------------------------------------------------
void ScrubReader::init()
{
    const size_t n = inodes->size();
    st.reset(new State[n ? n : 1]);
    fds.init(n);
    for (size_t u = 0; u < n; u++) fds.add_reads(u, (*inodes)[u].n_blocks);
}

std::string ScrubReader::block_name(const BlockRef& b)
{
    const ScrubInode& I = (*inodes)[b.file];
    return I.rel + " (version " + std::to_string(I.version) + ") block " + std::to_string(b.file_off / block_bytes);
}

std::string ScrubReader::why(uint32_t u)
{
    std::lock_guard<std::mutex> lk(why_mu);
    return st[u].why;
}

void ScrubReader::mark_bad(uint32_t u, const std::string& why)
{
    std::lock_guard<std::mutex> lk(why_mu);
    if (!st[u].bad.load()) st[u].why = why;
    st[u].bad.store(true);
}

// VMIG_OK with *out; VMIG_ESRCCHANGED: not the walked inode any more; any other code: the inode cannot be opened
int ScrubReader::open_inode(uint32_t u, int* out)
{
    const ScrubInode& I = (*inodes)[u];
    return fds.get(u, root_fds[I.version], I.rel, direct, [&](int*, const struct stat* sb, bool) {
        if (!sb) return fail(VMIG_EIO, "fstat %s: %s", I.rel.c_str(), errno_str(errno).c_str());
        if (!S_ISREG(sb->st_mode) || (uint64_t)sb->st_dev != I.dev || (uint64_t)sb->st_ino != I.ino || (uint64_t)sb->st_size != I.size)
            return fail(VMIG_ESRCCHANGED, "%s (version %u) is no longer the %llu-byte regular file the walk saw: the store changed during the scrub",
                        I.rel.c_str(), I.version, (unsigned long long)I.size);
        return VMIG_OK;
    }, out);
}

int ScrubReader::read(uint32_t u, uint64_t off, uint32_t len, uint8_t* dst)
{
    if (st[u].bad.load()) { fds.read_done(u); return VMIG_OK; }    // the rest of an unreadable inode is not read
    int fd;
    int rc = open_inode(u, &fd);
    if (rc == VMIG_ESRCCHANGED) return rc;
    if (rc) { mark_bad(u, last_error_cstr()); fds.read_done(u); return VMIG_OK; }
    const ScrubInode& I = (*inodes)[u];
    // O_DIRECT: buffer, offset and length in whole sectors (the pipeline's slot layout leaves the room), as FileIO reads
    size_t got, at = 0;
    rc = xfer_block(fds.direct(u), true, len, &got, [&](size_t pos, size_t n) { at = pos; return pread(fd, dst + pos, n, (off_t)(off + pos)); });
    if (rc < 0) {
        char b[64]; snprintf(b, sizeof b, " at offset %llu: ", (unsigned long long)(off + at));
        mark_bad(u, "pread " + I.rel + b + errno_str(errno));
    } else if (rc > 0) {
        return fail(VMIG_ESRCCHANGED, "%s (version %u) shrank during the scrub (wanted %u bytes at %llu, got %zu)", I.rel.c_str(), I.version,
                    len, (unsigned long long)off, got);
    }
    fds.read_done(u);
    return VMIG_OK;
}

}  // namespace vmig
