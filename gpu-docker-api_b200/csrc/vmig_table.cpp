// vmig_table.cpp -- block-table (de)serialisation (see vmig_table.h, include/vmig.h).
#include "vmig_table.h"
#include "vmig_common.h"

#include <fcntl.h>
#include <unistd.h>
#include <sys/stat.h>
#include <sys/syscall.h>
#include <time.h>
#include <algorithm>

namespace vmig {

static const char kMagic1[8] = {'V', 'M', 'I', 'G', 'B', 'T', '0', '1'};   // no file identity
static const char kMagic[8]  = {'V', 'M', 'I', 'G', 'B', 'T', '0', '2'};   // + u64 ino, i64 ctime_ns per file

int table_load(const std::string& path, BlockTable* t)
{
    *t = BlockTable();
    int fd = open(path.c_str(), O_RDONLY | O_CLOEXEC);
    if (fd < 0) return fail(VMIG_ETABLE, "open table %s: %s", path.c_str(), errno_str(errno).c_str());
    struct stat st;
    if (fstat(fd, &st) != 0) { close(fd); return fail(VMIG_ETABLE, "fstat table %s", path.c_str()); }
    std::string raw((size_t)st.st_size, '\0');
    size_t got = 0;
    while (got < raw.size()) {
        ssize_t r = read(fd, &raw[got], raw.size() - got);
        if (r <= 0) { close(fd); return fail(VMIG_ETABLE, "short read on table %s", path.c_str()); }
        got += (size_t)r;
    }
    close(fd);
    if (raw.size() < 32 || (memcmp(raw.data(), kMagic, 8) != 0 && memcmp(raw.data(), kMagic1, 8) != 0)) return fail(VMIG_ETABLE, "%s: bad magic", path.c_str());
    const size_t rec = memcmp(raw.data(), kMagic, 8) == 0 ? 32 : 16;        // fixed bytes per file after the path
    uint64_t n_files, n_blocks;
    memcpy(&t->block_bytes, &raw[8], 4); memcpy(&t->algo, &raw[12], 4);
    memcpy(&n_files, &raw[16], 8); memcpy(&n_blocks, &raw[24], 8);
    if (t->algo != 1 || t->block_bytes == 0 || (t->block_bytes & 4095u)) return fail(VMIG_ETABLE, "%s: unsupported algo/block size", path.c_str());
    size_t off = 32;
    if (n_files > raw.size() / 20 + 1 || n_blocks > raw.size() / 8 + 1) return fail(VMIG_ETABLE, "%s: counts exceed file size", path.c_str());
    t->files.reserve((size_t)n_files);
    uint64_t expect_first = 0;
    for (uint64_t i = 0; i < n_files; i++) {
        if (off + 4 > raw.size()) return fail(VMIG_ETABLE, "%s: truncated manifest", path.c_str());
        uint32_t plen; memcpy(&plen, &raw[off], 4); off += 4;
        if (off + plen + rec > raw.size()) return fail(VMIG_ETABLE, "%s: truncated manifest", path.c_str());
        TableFile f; f.rel.assign(&raw[off], plen); off += plen;
        memcpy(&f.size, &raw[off], 8); memcpy(&f.first_block, &raw[off + 8], 8);
        if (rec == 32) { memcpy(&f.ino, &raw[off + 16], 8); memcpy(&f.ctime_ns, &raw[off + 24], 8); }
        off += rec;
        if (f.first_block != expect_first) return fail(VMIG_ETABLE, "%s: inconsistent first_block for %s", path.c_str(), f.rel.c_str());
        if (!t->files.empty() && !(t->files.back().rel < f.rel)) return fail(VMIG_ETABLE, "%s: manifest not sorted", path.c_str());
        expect_first += t->blocks_of(f);
        t->files.push_back(std::move(f));
    }
    if (expect_first != n_blocks || off + 8 * n_blocks != raw.size()) return fail(VMIG_ETABLE, "%s: block count mismatch", path.c_str());
    t->hashes.resize((size_t)n_blocks);
    if (n_blocks) memcpy(t->hashes.data(), &raw[off], 8 * (size_t)n_blocks);
    t->index.reserve(t->files.size() * 2);
    for (size_t i = 0; i < t->files.size(); i++) t->index.emplace(t->files[i].rel, i);
    return VMIG_OK;
}

int table_store(const std::string& path, const BlockTable& t, const std::atomic<int>* cancel)
{
    if (cancel && cancel->load()) return fail(VMIG_ECANCELED, "cancelled before the block table %s was written", path.c_str());
    std::string raw;
    size_t need = 32 + 8 * t.hashes.size();
    for (auto& f : t.files) need += 4 + f.rel.size() + 32;
    raw.reserve(need);
    raw.append(kMagic, 8);
    uint64_t n_files = t.files.size(), n_blocks = t.hashes.size();
    raw.append((const char*)&t.block_bytes, 4); raw.append((const char*)&t.algo, 4);
    raw.append((const char*)&n_files, 8); raw.append((const char*)&n_blocks, 8);
    for (auto& f : t.files) {
        uint32_t plen = (uint32_t)f.rel.size();
        raw.append((const char*)&plen, 4); raw.append(f.rel);
        raw.append((const char*)&f.size, 8); raw.append((const char*)&f.first_block, 8);
        raw.append((const char*)&f.ino, 8); raw.append((const char*)&f.ctime_ns, 8);
    }
    if (n_blocks) raw.append((const char*)t.hashes.data(), 8 * (size_t)n_blocks);

    const std::string tmp = path + ".tmp." + std::to_string((long)getpid()) + "." + std::to_string((long)syscall(SYS_gettid));
    int fd = open(tmp.c_str(), O_WRONLY | O_CREAT | O_TRUNC | O_CLOEXEC, 0644);
    if (fd < 0) return fail(VMIG_EIO, "create %s: %s", tmp.c_str(), errno_str(errno).c_str());
    size_t put = 0;
    while (put < raw.size()) {
        ssize_t w = write(fd, raw.data() + put, raw.size() - put);
        if (w <= 0) { close(fd); unlink(tmp.c_str()); return fail(VMIG_EIO, "write %s: %s", tmp.c_str(), errno_str(errno).c_str()); }
        put += (size_t)w;
    }
    if (fsync(fd) != 0) { close(fd); unlink(tmp.c_str()); return fail(VMIG_EIO, "fsync %s: %s", tmp.c_str(), errno_str(errno).c_str()); }
    close(fd);
    if (cancel && cancel->load()) { unlink(tmp.c_str()); return fail(VMIG_ECANCELED, "cancelled before the block table %s was renamed into place", path.c_str()); }
    if (rename(tmp.c_str(), path.c_str()) != 0) { unlink(tmp.c_str()); return fail(VMIG_EIO, "rename %s: %s", path.c_str(), errno_str(errno).c_str()); }
    return VMIG_OK;
}

void wait_past_recorded_ctimes(const BlockTable& t)
{
    int64_t newest = 0;
    for (auto& f : t.files) if (f.ino) newest = std::max(newest, f.ctime_ns);
    auto coarse = [] { struct timespec ts; clock_gettime(CLOCK_REALTIME_COARSE, &ts); return (int64_t)ts.tv_sec * 1000000000ll + ts.tv_nsec; };
    if (!newest || newest - coarse() > 1000000000ll) return;
    const uint64_t give_up = now_ns() + 1100000000ull;           // the realtime clock may be stepped back meanwhile
    while (coarse() <= newest && now_ns() < give_up) {
        const struct timespec nap = {0, 200000};
        nanosleep(&nap, nullptr);
    }
}

}  // namespace vmig
