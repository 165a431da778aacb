// vmig_api.cu -- the C ABI of libvmig (include/vmig.h): tree migration, buffer migration, direct
// block hashing, the HBM-resident batch, and the host-side helpers.
//
// Reference seam (SURVEY.md §8b): utils.CopyDir (utils/copy.go:21-27), moveVolumeData
// (utils/copy.go:74-128), utils.DirSize / utils.ToBytes (utils/file.go:13-48).
#include "vmig_engine.h"
#include "vmig_kernels.cuh"
#include "vmig_tree.h"
#include "vmig_table.h"
#include "vmig_cufile.h"
#include "vmig_reuse.h"
#include "vmig_scrub.h"
#include "vmig_compare.h"
#include "vmig_rollback.h"
#include "vmig_retire.h"
#include "vmig_plan.h"
#include "vmig_select.h"

#include <fcntl.h>
#include <unistd.h>
#include <sys/stat.h>
#include <algorithm>
#include <condition_variable>
#include <unordered_map>
#include <unordered_set>
#include <thread>
#include <cmath>

using namespace vmig;

void vmig::CallCtl::cancel()
{
    cancelled.store(1);
    {
        std::lock_guard<std::mutex> lk(mu);
        int none = 0;
        if (latch) latch->compare_exchange_strong(none, VMIG_ECANCELED);
    }
    ctx_wake_waiters();             // a call waiting for a staging pipe
}

namespace {

// ---------------------------------------------------------------------------------------------
// controls (vmig_ctl_*) and the calls in flight (vmig_shutdown cancels them and waits for them)
std::mutex g_ctl_mu;
std::unordered_map<uint32_t, std::shared_ptr<CallCtl>> g_ctls;
uint32_t g_ctl_next = 1;
std::mutex g_calls_mu;
std::condition_variable g_calls_cv;
std::unordered_set<CallCtl*> g_calls;

const char* phase_name(uint32_t p)
{
    static const char* const names[] = {"IDLE", "WALK", "DATA", "VERIFY", "META", "PRUNE", "TABLE", "UNLINK", "DONE"};
    return p <= VMIG_PHASE_DONE ? names[p] : "?";
}

// One data-path call: attached to the caller's control (vmig_opts.ctl) or to a private one, and counted as in flight.
class CallScope {
    std::shared_ptr<CallCtl> held;
public:
    CallCtl* ctl = nullptr;
    int attach(uint32_t id) {
        if (id) {
            std::lock_guard<std::mutex> lk(g_ctl_mu);
            auto it = g_ctls.find(id);
            if (it == g_ctls.end()) return fail(VMIG_EINVAL, "vmig_opts.ctl %u is not an open control", id);
            if (it->second->running.load()) return fail(VMIG_EINVAL, "control %u is already attached to a call in flight", id);
            held = it->second;
            held->running.store(1);
        } else {
            held = std::make_shared<CallCtl>();
            held->running.store(1);
        }
        ctl = held.get();
        ctl->phase.store(VMIG_PHASE_IDLE);
        for (auto* c : {&ctl->bytes_total, &ctl->blocks_total, &ctl->bytes_hashed, &ctl->blocks_hashed, &ctl->bytes_written, &ctl->bytes_verified})
            c->store(0);
        std::lock_guard<std::mutex> lk(g_calls_mu);
        g_calls.insert(ctl);
        return VMIG_OK;
    }
    const std::atomic<int>* cancel() const { return &ctl->cancelled; }
    void phase(uint32_t p) { ctl->phase.store(p); }
    // VMIG_ECANCELED: vmig_last_error() names the phase the call stopped in
    int finish(int rc) {
        if (rc == VMIG_OK) ctl->phase.store(VMIG_PHASE_DONE);
        if (rc == VMIG_ECANCELED) {
            const std::string why = last_error_cstr();
            fail(VMIG_ECANCELED, "cancelled in phase %s: %s", phase_name(ctl->phase.load()), why.c_str());
        }
        return rc;
    }
    ~CallScope() {
        if (!ctl) return;
        { std::lock_guard<std::mutex> lk(g_ctl_mu); ctl->running.store(0); }
        std::lock_guard<std::mutex> lk(g_calls_mu);
        g_calls.erase(ctl);
        g_calls_cv.notify_all();
    }
};

// body(call) as one data-path call attached to control id (0: a private one)
template <class Body>
int in_call(uint32_t id, Body body)
{
    CallScope call;
    const int rc = call.attach(id);
    if (rc) return rc;
    return call.finish(body(call));
}

// The block pipeline's first-error latch, reachable by CallCtl::cancel while run_blocks runs
struct LatchLink {
    CallCtl* c;
    LatchLink(CallCtl* ctl, std::atomic<int>* latch) : c(ctl) {
        std::lock_guard<std::mutex> lk(c->mu);
        c->latch = latch;
        int none = 0;
        if (c->cancelled.load()) latch->compare_exchange_strong(none, VMIG_ECANCELED);
    }
    ~LatchLink() { std::lock_guard<std::mutex> lk(c->mu); c->latch = nullptr; }
};

// ---------------------------------------------------------------------------------------------
// The identity a block table records for a file (vmig_table.h)
struct FileId { uint64_t ino = 0; int64_t ctime_ns = 0; };
FileId file_id(const struct stat& st) { return {(uint64_t)st.st_ino, ctime_ns(st)}; }

// A tree as a call leaves it in its destination: what the metadata, verify and table passes need of it
struct DstTree {
    const Manifest* m = nullptr;
    std::string dst_root;
    MetaPolicy pol;
    bool hash_only = false;
    bool direct = false;                 // VMIG_F_DIRECT_IO: O_DIRECT into / out of the pinned rings
    bool cufile = false;                 // VMIG_F_CUFILE: file <-> HBM slot through libcufile (GPUDirect Storage)
    uint32_t block_bytes = 4u << 20;
    std::vector<FileId> ids;             // per manifest file, the identity its table record carries; a writer sets only its file's
};

// file-backed BlockIO
class FileIO : public BlockIO, public DstTree {
public:
    // the call's mutable state of one file; what was decided about it before the data pass is in plan->files
    struct FS {
        std::atomic<int> dfd{-1};
        std::atomic<uint32_t> blocks_left{0};
        bool d_direct = false;                           // dfd was opened with O_DIRECT
        std::atomic<void*> s_cfh{nullptr}, d_cfh{nullptr};   // cuFile handles of the source descriptor / dfd (VMIG_F_CUFILE)
        std::atomic<bool> wrote{false};                  // at least one block of the file was written in this call
        std::atomic<bool> reused{false};                 // vmig_snapshot_tree: a changed block was found elsewhere in the base
        int lent_mode = -1;                              // >= 0: open_dst lent the file a write bit; its mode before that
        struct stat src_before;                          // record_src: the source's fstat before its first read, and the
        int64_t src_clock = 0;                           // CLOCK_REALTIME_COARSE reading taken just before that fstat
    };
    std::string src_root;
    int src_root_fd = -1;                // source files are opened beneath this descriptor, never by absolute path
    const TreePlan* plan = nullptr;
    ReadFds src;                         // source descriptors, per manifest file
    std::atomic<uint64_t> n_direct{0};   // destination descriptors that really were opened O_DIRECT (source: src.n_direct)
    uint32_t slot_align() override { return direct || cufile ? kSector : 512; }
    bool device_reads() override { return cufile; }
    bool device_writes() override { return cufile && !hash_only; }
    long corrupt_block = -1;             // VMIG_CORRUPT_BLOCK test hook: flip one bit of this block on its way to disk
    std::string block_name(const BlockRef& b) override {
        return m->files[b.file].rel + " block " + std::to_string(b.file_off / block_bytes);
    }
    std::unique_ptr<FS[]> fs;
    std::mutex stripes[64];
    // one FS per manifest file; a file's blocks in the plan's list count down to the close of its source and to its
    // finalization.  A file with blocks the plan already skipped (vmig_snapshot_layer) is finished from the base.
    void init_files(const Manifest& man, const TreePlan& p) {
        m = &man; plan = &p;
        fs.reset(new FS[man.files.size() ? man.files.size() : 1]);
        src.init(man.files.size());
        ids.assign(man.files.size(), FileId{});
        for (const BlockRef& b : p.blocks) { src.add_reads(b.file, 1); fs[b.file].blocks_left.fetch_add(1, std::memory_order_relaxed); }
        if (!p.skipped.empty()) {
            skipped = p.skipped;
            for (uint32_t f = 0; f < man.files.size(); f++)
                if (p.files[f].layer_rec && !p.bidx.empty())       // (vmig_migrate_layer's skipped blocks are the destination's)
                    for (uint64_t r = 0; r < man.files[f].n_blocks; r++) if (p.skipped[man.files[f].first_block + r]) { fs[f].reused.store(true); break; }
        }
    }

    // vmig_snapshot_tree: the base snapshot whose files supply the blocks K1 found unchanged, at the same path and offset
    // or anywhere else in the base (bidx: every block of every trusted base file, by hash and length)
    std::string base_root;
    const BaseIndex* bidx = nullptr;                       // the plan's index (TreePlan::bidx)
    const uint64_t* hashes = nullptr;                      // the call's block hashes (a file's are all there when it finalizes)
    std::vector<uint8_t> skipped;                          // per table block: 1 = not written, its bytes are in the base
    std::mutex link_mu;
    std::unordered_map<uint64_t, int64_t> linked_inos;     // base inode linked by this call -> its ctime after the link
    std::vector<uint32_t> linked_files;
    std::atomic<uint64_t> n_linked{0}, b_linked{0}, n_backfilled{0}, b_backfilled{0};
    const std::atomic<int>* cancel = nullptr;              // the call's cancel flag: checked per backfill chunk
    static constexpr size_t kLinkTries = 16;               // base files of equal content tried as a link target, per file
    bool done_on_writer(const BlockRef& b) override { return plan->files[b.file].base_rec != nullptr || fs[b.file].reused.load(); }
    bool reusable(const BlockRef& b, uint64_t hash) override {
        if (!bidx || !bidx->contains(hash, b.len)) return false;
        skipped[b.table_idx] = 1;
        fs[b.file].reused.store(true);
        return true;
    }

    // Open base file g and check that it still is the file its record describes: same inode, and the recorded ctime or
    // the one this call's own link to it left.  Anything else changed it, and the bytes it was to supply are gone.
    int open_base(uint32_t g, int* out, struct stat* bs) {
        const TableFile& bf = bidx->t->files[g];
        const std::string bp = pjoin(base_root, bf.rel);
        const int bfd = open(bp.c_str(), O_RDONLY | O_NOFOLLOW | O_CLOEXEC);
        bool same = bfd >= 0 && fstat(bfd, bs) == 0 && S_ISREG(bs->st_mode) && (uint64_t)bs->st_ino == bf.ino;
        if (same) {
            const int64_t ct = ctime_ns(*bs);
            std::lock_guard<std::mutex> lk(link_mu);     // a link in flight holds it from before linkat until linked_inos has its ctime
            auto it = linked_inos.find(bf.ino);
            same = ct == bf.ctime_ns || (it != linked_inos.end() && it->second == ct);
        }
        if (!same) {
            if (bfd >= 0) close(bfd);
            return fail(VMIG_ESRCCHANGED, "base file %s changed during the snapshot: the bytes of its unchanged blocks are gone", bp.c_str());
        }
        *out = bfd;
        return VMIG_OK;
    }

    // Last block of a file with blocks in the base passed: link the new path to a base file of the same content when
    // nothing was written and the link keeps the snapshot's hard-link structure and metadata equal to the source's
    // (the same-path file first, then the others in table order), else copy the skipped blocks from the base files that
    // hold them into the new file (block_done then finalizes it like any other).  Runs on a writer (done_on_writer).
    int finish_from_base(uint32_t f, bool* linked) {
        FS& s = fs[f];
        const Entry& e = m->files[f];
        bool any_skipped = false;
        for (uint64_t r = 0; r < e.n_blocks && !any_skipped; r++) any_skipped = skipped[e.first_block + r] != 0;
        if (!any_skipped) return VMIG_OK;
        const FilePlan& fp = plan->files[f];
        const int same = fp.base_rec ? (int)(fp.base_rec - bidx->t->files.data()) : -1;
        const uint64_t* h = hashes + e.first_block;
        const std::string p = pjoin(dst_root, e.rel);
        if (!s.wrote.load() && fp.solo) {
            std::vector<uint32_t> cands;
            link_candidates(*bidx, same, e.size, block_bytes, h, &cands, kLinkTries);
            for (uint32_t g : cands) {
                const TableFile& bf = bidx->t->files[g];
                { std::lock_guard<std::mutex> lk(link_mu); if (linked_inos.count(bf.ino)) continue; }
                int bfd; struct stat bs;
                int rc = open_base(g, &bfd, &bs);
                if (rc) return rc;
                if (!file_meta_matches(bfd, e, pol)) { close(bfd); continue; }
                std::lock_guard<std::mutex> lk(link_mu);
                if (linked_inos.count(bf.ino)) { close(bfd); continue; }
                const std::string bp = pjoin(base_root, bf.rel);
                rc = clear_path(p, "a regular file");
                if (!rc && linkat(AT_FDCWD, bp.c_str(), AT_FDCWD, p.c_str(), 0) != 0) rc = fail(VMIG_EIO, "link %s -> %s: %s", p.c_str(), bp.c_str(), errno_str(errno).c_str());
                struct stat ls;
                if (!rc && (lstat(p.c_str(), &ls) != 0 || ls.st_ino != bs.st_ino)) {      // the base path was replaced after the fstat
                    unlink(p.c_str());
                    rc = fail(VMIG_ESRCCHANGED, "base file %s was replaced during the snapshot", bp.c_str());
                }
                close(bfd);
                if (rc) return rc;
                linked_inos[bf.ino] = ctime_ns(ls);
                linked_files.push_back(f);
                n_linked++; b_linked += e.size;
                *linked = true;
                return VMIG_OK;
            }
        }
        std::vector<ReuseRun> runs;
        int rc = plan_backfill(*bidx, same, e.size, block_bytes, h, &skipped[e.first_block], e.rel, &runs);
        if (rc) return rc;
        int dfd; rc = open_dst(f, &dfd);
        std::unordered_map<uint32_t, int> bfds;              // base files this file takes bytes from, each checked once
        uint64_t bytes = 0;
        for (const ReuseRun& u : runs) {
            if (rc) break;
            auto it = bfds.find(u.file);
            if (it == bfds.end()) {
                int bfd; struct stat bs;
                rc = open_base(u.file, &bfd, &bs);
                if (rc) break;
                it = bfds.emplace(u.file, bfd).first;
            }
            rc = copy_range_at(it->second, u.src_off, dfd, u.dst_off, u.len, s.d_direct, false, pjoin(base_root, bidx->t->files[u.file].rel), cancel);
            bytes += u.len;
        }
        for (auto& kv : bfds) close(kv.second);
        if (rc) return rc;
        n_backfilled++; b_backfilled += bytes;
        return VMIG_OK;
    }

    // libcufile refuses descriptors whose open flags include O_NOFOLLOW / O_NONBLOCK ("unsupported file open flags"),
    // which is exactly how the safe opens below are made, and F_SETFL cannot clear O_NOFOLLOW.  The descriptor already
    // refers to the checked regular file, so it is re-opened through /proc/self/fd with plain flags and registered.
    // *fd is replaced by the new descriptor; on failure *fd (the old or the new one) is left for the caller to close.
    static int attach_cufile(int* fd, int flags, const char* what, void** handle) {
        char p[64]; snprintf(p, sizeof p, "/proc/self/fd/%d", *fd);
        const int nfd = open(p, flags | O_CLOEXEC);
        if (nfd < 0) return fail(VMIG_EIO, "reopen %s for cuFile: %s", what, errno_str(errno).c_str());
        close(*fd); *fd = nfd;
        return cufile_handle_open(nfd, handle);
    }
    // vmig_migrate_layer's src_out_table: the identity each source file may be recorded with (live_identity_holds).  A
    // listed file's descriptor is held open past its last read, until its last block's hash is back (note_source).
    bool record_src = false;
    std::vector<FileId> src_ids;                           // per manifest file; 0/0: the next call reads the file
    void hold_sources() {
        record_src = true;
        src_ids.assign(m->files.size(), FileId{});
        for (uint32_t f = 0; f < m->files.size(); f++) if (fs[f].blocks_left.load(std::memory_order_relaxed)) src.add_reads(f, 1);
    }
    void note_source(uint32_t f) {
        int fd;
        if (open_src(f, &fd) != VMIG_OK) return;           // (the held descriptor: nothing is opened here)
        struct stat after;
        if (plan->files[f].solo && fstat(fd, &after) == 0 && (uint64_t)after.st_size == m->files[f].size &&
            live_identity_holds(fs[f].src_before, fs[f].src_clock, after))
            src_ids[f] = file_id(after);
        read_done(f);
    }
    int open_src(uint32_t f, int* out) {
        const char* rel = m->files[f].rel.c_str();
        return src.get(f, src_root_fd, m->files[f].rel, direct, [&](int* fd, const struct stat* st, bool is_direct) {
            if (!st || !S_ISREG(st->st_mode)) return fail(VMIG_ESRCCHANGED, "%s is not a regular file any more", rel);
            if (hash_only && st->st_nlink == 1) ids[f] = file_id(*st);
            if (record_src) {                               // the clock first: a write after the fstat stamps a later ctime
                struct timespec ts;
                clock_gettime(CLOCK_REALTIME_COARSE, &ts);
                fs[f].src_clock = fstat(*fd, &fs[f].src_before) == 0 ? (int64_t)ts.tv_sec * 1000000000ll + ts.tv_nsec : 0;
            }
            if (!cufile) return VMIG_OK;
            void* h = nullptr;
            const int rc = attach_cufile(fd, O_RDONLY | (is_direct ? O_DIRECT : 0), rel, &h);
            if (!rc) fs[f].s_cfh.store(h, std::memory_order_release);
            return rc;
        }, out);
    }
    // one counted read of file f is done: after its last, the cuFile handle goes before the descriptor closes
    void read_done(uint32_t f) {
        src.read_done(f, [&](int) { void* h = fs[f].s_cfh.exchange(nullptr); if (h) cufile_handle_close(h); });
    }
    int open_dst(uint32_t f, int* out) {
        FS& s = fs[f];
        int fd = s.dfd.load(std::memory_order_acquire);
        if (fd < 0) {
            std::lock_guard<std::mutex> lk(stripes[f & 63]);
            fd = s.dfd.load(std::memory_order_acquire);
            if (fd < 0) {
                const std::string p = pjoin(dst_root, m->files[f].rel);
                const bool want_direct = direct && corrupt_block < 0;
                if (plan->files[f].prior_rec) {
                    fd = open_for_write(p, false, want_direct, &s.d_direct);
                    // an ordinary user's own read-only file (tar would replace it): made writable for the patch; its mode no
                    // longer matches the source's, so block_done puts the source's back whether a block was written or not
                    // (under VMIG_F_NO_METADATA the mode it had before the lend)
                    struct stat ws;
                    if (fd < 0 && errno == EACCES && lstat(p.c_str(), &ws) == 0 && S_ISREG(ws.st_mode) &&
                        chmod(p.c_str(), (ws.st_mode & 07777) | S_IWUSR) == 0) {
                        s.lent_mode = (int)(ws.st_mode & 07777);
                        fd = open_for_write(p, false, want_direct, &s.d_direct);
                    }
                } else {
                    int rc = clear_path(p, "a regular file");     // tar replaces what is there
                    if (rc) return rc;
                    fd = open_for_write(p, true, want_direct, &s.d_direct);
                }
                if (fd < 0) return fail(VMIG_EIO, "open %s for writing: %s", p.c_str(), errno_str(errno).c_str());
                if (s.d_direct) n_direct++;
                if (cufile && !hash_only) {
                    void* h = nullptr;
                    const int rc = attach_cufile(&fd, O_WRONLY | (s.d_direct ? O_DIRECT : 0), p.c_str(), &h);
                    if (rc) { close(fd); return rc; }
                    s.d_cfh.store(h, std::memory_order_release);
                }
                s.dfd.store(fd, std::memory_order_release);
            }
        }
        *out = fd; return VMIG_OK;
    }
    int read_block(const BlockRef& b, uint8_t* dst) override {
        int fd; int rc = open_src(b.file, &fd);
        if (rc) return rc;
        // O_DIRECT: the device DMAs straight into the pinned ring; the file's last block is short, the read past EOF simply
        // returns fewer bytes
        size_t got;
        rc = xfer_block(src.direct(b.file), true, b.len, &got, [&](size_t pos, size_t n) { return pread(fd, dst + pos, n, (off_t)(b.file_off + pos)); });
        if (rc < 0) return fail(VMIG_EIO, "pread %s: %s", m->files[b.file].rel.c_str(), errno_str(errno).c_str());
        if (rc) return shrank(b, got);
        read_done(b.file);
        return VMIG_OK;
    }
    int shrank(const BlockRef& b, size_t got) {
        return fail(VMIG_ESRCCHANGED, "%s shrank while being migrated (wanted %u bytes at %llu, got %zu)", m->files[b.file].rel.c_str(), b.len, (unsigned long long)b.file_off, got);
    }
    // GPUDirect Storage: file -> HBM slot
    int read_block_dev(const BlockRef& b, uint8_t* d_base, size_t d_off) override {
        int fd; int rc = open_src(b.file, &fd);
        if (rc) return rc;
        void* h = fs[b.file].s_cfh.load(std::memory_order_acquire);
        size_t got;
        rc = xfer_block(src.direct(b.file), false, b.len, &got, [&](size_t pos, size_t n) { return cufile_read(h, d_base, n, (off_t)(b.file_off + pos), (off_t)(d_off + pos)); });
        if (rc < 0) return rc;
        if (rc) return shrank(b, got);
        read_done(b.file);
        return VMIG_OK;
    }
    // GPUDirect Storage: HBM slot -> file (surviving blocks only)
    int write_block_dev(const BlockRef& b, const uint8_t* d_base, size_t d_off) override {
        int fd; int rc = open_dst(b.file, &fd);
        if (rc) return rc;
        FS& s = fs[b.file];
        s.wrote.store(true, std::memory_order_relaxed);
        void* h = s.d_cfh.load(std::memory_order_acquire);
        size_t put;
        rc = xfer_block(s.d_direct, false, b.len, &put, [&](size_t pos, size_t n) { return cufile_write(h, d_base, n, (off_t)(b.file_off + pos), (off_t)(d_off + pos)); });
        if (rc < 0) return rc;
        if (rc) return fail(VMIG_EIO, "cuFileWrite %s: wrote 0 bytes", m->files[b.file].rel.c_str());
        return VMIG_OK;
    }
    int write_block(const BlockRef& b, const uint8_t* src) override {
        int fd; int rc = open_dst(b.file, &fd);
        if (rc) return rc;
        fs[b.file].wrote.store(true, std::memory_order_relaxed);
        if (corrupt_block >= 0 && (uint64_t)corrupt_block == b.table_idx && b.len) {
            const uint8_t bad = src[0] ^ 1u;           // what VMIG_F_VERIFY exists to catch
            if (pwrite(fd, &bad, 1, (off_t)b.file_off) != 1) return fail(VMIG_EIO, "pwrite (fault hook)");
            if (b.len == 1) return VMIG_OK;
            size_t put1 = 1;
            while (put1 < b.len) { ssize_t w = pwrite(fd, src + put1, b.len - put1, (off_t)(b.file_off + put1)); if (w <= 0) return fail(VMIG_EIO, "pwrite (fault hook)"); put1 += (size_t)w; }
            return VMIG_OK;
        }
        // O_DIRECT: whole sectors out of the pinned ring; a short last block is written padded (whatever follows it in the
        // slot) and block_done() cuts the file back to its size
        size_t put;
        rc = xfer_block(fs[b.file].d_direct, true, b.len, &put, [&](size_t pos, size_t n) { return pwrite(fd, src + pos, n, (off_t)(b.file_off + pos)); });
        if (rc < 0) return fail(VMIG_EIO, "pwrite %s: %s", m->files[b.file].rel.c_str(), errno_str(errno).c_str());
        if (rc) return fail(VMIG_EIO, "pwrite %s: wrote 0 bytes", m->files[b.file].rel.c_str());
        return VMIG_OK;
    }
    int block_done(const BlockRef& b, bool written) override {
        FS& s = fs[b.file];
        const FilePlan& fp = plan->files[b.file];
        if (!written && fp.base_rec) skipped[b.table_idx] = 1;          // (a reused block was marked by reusable())
        if (s.blocks_left.fetch_sub(1) != 1) return VMIG_OK;
        if (hash_only) return VMIG_OK;
        if (record_src) note_source(b.file);
        return finish_file(b.file);
    }
    // The file's last block passed (or none is read: the layer calls' unread files): link or backfill from the base,
    // else cut and apply metadata, and take the identity the table records
    int finish_file(uint32_t f) {
        FS& s = fs[f];
        const FilePlan& fp = plan->files[f];
        const Entry& e = m->files[f];
        if (fp.base_rec || s.reused.load()) {
            bool linked = false;
            int rc = finish_from_base(f, &linked);
            if (rc || linked) return rc;
        }
        int fd; int rc = open_dst(f, &fd);      // also covers "every block was skipped"
        if (rc) return rc;
        const std::string p = pjoin(dst_root, e.rel);
        const bool inplace = fp.prior_rec != nullptr;
        // O_DIRECT writes whole sectors: cut the padding of the last one.  A file patched in place that took no write has
        // none, and a truncate would move its mtime and ctime and so the identity its table records
        const bool padded = s.d_direct && (e.size & (kSector - 1)) && (s.wrote.load() || !inplace);
        if ((inplace && fp.prior_rec->size != e.size) || padded) rc = cut_to_size(fd, e.size, p);
        // a patched-in-place file none of whose blocks changed and whose metadata is already right is not touched at all:
        // its ctime -- by which the block table knows it -- stays what the table recorded
        const bool untouched = inplace && !s.wrote.load() && fp.prior_rec->size == e.size && file_meta_matches(fd, e, pol);
        if (!rc && !untouched) rc = apply_file_meta(fd, p, e, pol);
        if (!rc && pol.no_metadata && s.lent_mode >= 0 && fchmod(fd, (mode_t)s.lent_mode) != 0)
            rc = fail(VMIG_EIO, "fchmod %s (mode lent for the patch): %s", p.c_str(), errno_str(errno).c_str());
        struct stat fst;                            // nothing touches the file after this point: its ctime is final
        if (!rc && fstat(fd, &fst) == 0) ids[f] = file_id(fst);
        { void* h = s.d_cfh.exchange(nullptr); if (h) cufile_handle_close(h); }
        rc = close_written(fd, rc, p);
        s.dfd.store(-1);
        return rc;
    }
    int open_root() {
        src_root_fd = open(src_root.c_str(), O_RDONLY | O_DIRECTORY | O_CLOEXEC);
        if (src_root_fd < 0) return fail(VMIG_EIO, "open %s: %s", src_root.c_str(), errno_str(errno).c_str());
        return VMIG_OK;
    }
    ~FileIO() {
        for (size_t i = 0; m && i < m->files.size(); i++) {     // what a failed data pass left open (src closes its own after)
            void* h = fs[i].s_cfh.exchange(nullptr); if (h) cufile_handle_close(h);
            h = fs[i].d_cfh.exchange(nullptr); if (h) cufile_handle_close(h);
            const int d = fs[i].dfd.exchange(-1); if (d >= 0) close(d);
        }
        if (src_root_fd >= 0) close(src_root_fd);
    }
};

// ---------------------------------------------------------------------------------------------
// memory-backed BlockIO (vmig_migrate_buffer, vmig_hash_blocks)
class MemIO : public BlockIO {
public:
    const uint8_t* src = nullptr; uint8_t* dst = nullptr;
    bool src_pinned = false, dst_pinned = false;
    int read_block(const BlockRef& b, uint8_t* d) override { if (b.len) memcpy(d, src + b.file_off, b.len); return VMIG_OK; }
    int write_block(const BlockRef& b, const uint8_t* s) override { if (b.len) memcpy(dst + b.file_off, s, b.len); return VMIG_OK; }
    uint32_t write_key(const BlockRef& b) override { return (uint32_t)b.table_idx; }
    const uint8_t* pinned_src(const BlockRef& b) override { return src_pinned ? src + b.file_off : nullptr; }
    uint8_t* pinned_dst(const BlockRef& b) override { return dst_pinned ? dst + b.file_off : nullptr; }
};

bool is_pinned(const void* p) {
    if (!p) return false;
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeHost;
}

// ---------------------------------------------------------------------------------------------
// run a block list over the selected GPUs: n_gpus x lanes_per_gpu lanes, whole files per lane (LPT by bytes);
// contiguous byte-balanced ranges only when there are fewer than two files per lane
// ctl: the call's control; a cancel sets this pipeline's first-error latch.  verify: progress goes to bytes_verified.
int run_blocks(const std::vector<BlockRef>& blocks, BlockIO* io, bool has_prior, bool hash_only, const vmig_opts& o,
               uint64_t* hashes, vmig_stats* st, CallCtl* ctl, bool verify, const BlockExpect* expect = nullptr)
{
    std::vector<DeviceInfo> devs;
    int rc = ctx_select(o.gpu_mask, &devs);
    if (rc) return rc;
    if (blocks.empty()) { st->gpus_used = 0; return VMIG_OK; }
    // lanes: one per GPU of the mask, times lanes_per_gpu (lane i runs on GPU i % n_gpus); the split below
    // does not care whether two lanes share a device
    uint32_t lpg = o.lanes_per_gpu ? o.lanes_per_gpu : (uint32_t)std::max<long>(1, env_long("VMIG_LANES_PER_GPU", 1));
    if (lpg > 16) lpg = 16;
    const size_t n_gpus = devs.size();
    size_t lanes = std::min(n_gpus * lpg, blocks.size());
    std::vector<DeviceInfo> lane_devs(lanes);
    for (size_t i = 0; i < lanes; i++) lane_devs[i] = devs[i % n_gpus];
    uint64_t total = 0;
    for (auto& b : blocks) total += std::max<uint32_t>(b.len, 4096);
    std::vector<std::vector<BlockRef>> share(lanes);
    if (lanes == 1) {
        share[0] = blocks;
    } else {
        // Prefer giving each GPU whole files (write keys): two lanes writing one destination file
        // would queue on its inode lock.  Longest-processing-time packing of the keys by bytes; the
        // interleaved block order is kept inside every lane.  With fewer keys than GPUs (one huge
        // file) the list is cut into contiguous byte-balanced ranges instead.
        std::unordered_map<uint32_t, uint64_t> key_bytes;
        for (auto& b : blocks) key_bytes[io->write_key(b)] += std::max<uint32_t>(b.len, 4096);
        if (key_bytes.size() >= 2 * lanes) {
            std::vector<std::pair<uint64_t, uint32_t>> keys;
            for (auto& kv : key_bytes) keys.push_back({kv.second, kv.first});
            std::sort(keys.begin(), keys.end(), [](auto& a, auto& b) { return a.first != b.first ? a.first > b.first : a.second < b.second; });
            std::vector<uint64_t> load(lanes, 0);
            std::unordered_map<uint32_t, uint32_t> key_lane;
            for (auto& k : keys) {
                size_t best = 0;
                for (size_t l = 1; l < lanes; l++) if (load[l] < load[best]) best = l;
                load[best] += k.first; key_lane[k.second] = (uint32_t)best;
            }
            for (auto& b : blocks) share[key_lane[io->write_key(b)]].push_back(b);
        } else {
            uint64_t acc = 0; size_t lane = 0;
            for (auto& b : blocks) {
                share[lane].push_back(b);
                acc += std::max<uint32_t>(b.len, 4096);
                if (lane + 1 < lanes && acc >= total * (lane + 1) / lanes) lane++;
            }
        }
    }
    std::atomic<int> err{0}; std::string err_msg; std::mutex err_mu;
    LatchLink link(ctl, &err);
    std::vector<Pipe*> pipes;
    rc = ctx_acquire_pipes(lane_devs, &pipes, &ctl->cancelled);
    if (rc) return rc;
    LaneProgress prog;
    if (verify) prog.hashed_bytes = &ctl->bytes_verified;
    else { prog.hashed_bytes = &ctl->bytes_hashed; prog.hashed_blocks = &ctl->blocks_hashed; prog.written = &ctl->bytes_written; }
    uint32_t readers, writers;       // sized AFTER the pipes are checked out: the count of lanes in flight includes this call's
    {
        std::unordered_map<uint32_t, int> seen;                  // blocks are interleaved across <= 64 files
        for (size_t i = 0; i < blocks.size() && i < 256; i++) seen[io->write_key(blocks[i])] = 1;
        // "many files" is a property of what ONE lane sees: 100 x 1 GiB over 8 lanes is 12 large files per lane
        io_threads_default(&readers, &writers, o.io_threads, lanes, std::min(n_gpus, lanes), seen.size() / lanes >= 32, has_prior, hash_only);
    }
    std::vector<LaneStats> ls(lanes);
    std::vector<std::thread> th;
    for (size_t i = 0; i < lanes; i++)
        th.emplace_back([&, i] {
            run_lane(pipes[i], share[i], io, has_prior, hash_only, readers, writers, o.streams_per_gpu, expect, hashes, &ls[i], &err, &err_msg,
                     &err_mu, prog);
        });
    for (auto& t : th) t.join();
    for (size_t i = 0; i < lanes; i++) ctx_release_pipe(pipes[i]);
    for (auto& l : ls) {
        st->bytes_h2d += l.bytes_h2d; st->bytes_d2h += l.bytes_d2h; st->bytes_written += l.bytes_written;
        st->blocks_skipped += l.blocks_skipped; st->kernel_launches += l.kernel_launches; st->ms_kernel += l.ms_kernel;
    }
    st->gpus_used = (uint32_t)std::min(n_gpus, lanes);
    st->lanes_used = (uint32_t)lanes;          // lanes the block list was sharded over
    if (err.load() == VMIG_ECANCELED && err_msg.empty()) return fail(VMIG_ECANCELED, "the block pipeline issued no new work after the cancel");
    if (err.load()) { set_last_error_str(err_msg); return err.load(); }
    return VMIG_OK;
}

// Restore, plan time: the walked tree must be the one the snapshot's table describes -- the same regular-file paths
// (hard-linked ones included) with the same sizes.  ino/ctime_ns are not compared: a snapshot copied elsewhere keeps
// its bytes, not its inodes.  The first difference in merge order fails the call.  On success expect[] holds the
// table's hashes in the manifest's block order.
int match_table(const Manifest& man, const BlockTable& t, std::vector<uint64_t>* expect)
{
    std::vector<int64_t> tab_of;
    std::vector<ScrubFinding> diff;
    if (scrub_merge_table(0, man, t, &tab_of, &diff)) {
        const ScrubFinding& d = diff[0];
        const char* p = d.path.c_str();
        if (d.kind == kScrubExtra) return fail(VMIG_ECORRUPT, "%s is in the snapshot but not in its block table (extra)", p);
        if (d.kind == kScrubMissing) return fail(VMIG_ECORRUPT, "%s is in the block table but not in the snapshot (missing)", p);
        const Entry& e = *std::lower_bound(man.files.begin(), man.files.end(), d.path, [](const Entry& a, const std::string& rel) { return a.rel < rel; });
        return fail(VMIG_ECORRUPT, "%s is %llu bytes in the snapshot, %llu in its block table (resized)", p, (unsigned long long)e.size,
                    (unsigned long long)t.files[t.index.at(d.path)].size);
    }
    expect->assign(man.n_blocks, 0);
    for (size_t f = 0; f < man.files.size(); f++) {
        const Entry& e = man.files[f];
        std::copy_n(t.hashes.begin() + (ptrdiff_t)t.files[(size_t)tab_of[f]].first_block, e.n_blocks, expect->begin() + (ptrdiff_t)e.first_block);
    }
    return VMIG_OK;
}

vmig_opts norm_opts(const vmig_opts* in) {
    vmig_opts o; memset(&o, 0, sizeof o);
    if (in) o = *in;
    if (!o.block_bytes) o.block_bytes = 4u << 20;
    if (env_long("VMIG_DIRECT_IO", 0) == 1) o.flags |= VMIG_F_DIRECT_IO;
    if (env_long("VMIG_CUFILE", 0) == 1) o.flags |= VMIG_F_CUFILE;
    return o;
}

int load_table(const char* path, const char* what, uint32_t block_bytes, BlockTable* t)
{
    const int rc = table_load(path, t);
    if (rc) return rc;
    if (t->block_bytes != block_bytes) return fail(VMIG_ETABLE, "%s table block size %u != %u", what, t->block_bytes, block_bytes);
    return VMIG_OK;
}

int check_block_bytes(const vmig_opts& o)
{
    if (o.block_bytes & 4095u) return fail(VMIG_EINVAL, "block_bytes %u is not a multiple of 4096", o.block_bytes);
    if (o.block_bytes > pipe_slot_bytes()) return fail(VMIG_EINVAL, "block_bytes %u exceeds the staging slot (%u)", o.block_bytes, pipe_slot_bytes());
    return VMIG_OK;
}

// What the passes of a tree call consume (tree_passes).  Every table is loaded by the call before the passes start;
// a null table is none.
struct TreeCall {
    std::string src, dst;
    const Manifest* man = nullptr;
    std::vector<uint64_t> expect;           // a checked restore: the snapshot table's hashes in the manifest's block order
    const BlockTable* prior = nullptr;      // a destination file that still is its record is patched in place
    const BlockTable* base = nullptr;       // the snapshots: unchanged files and blocks come from the base
    std::string base_dir;                   //   (FileIO::finish_from_base), when base_dir is on the destination's device
    const BlockTable* layer = nullptr;      // the layer calls: the source's own table (an empty one trusts nothing)
    // vmig_restore_paths: the parent chains are made real directories before the plan looks at the destination, the
    // prune and its verify stay beneath the chosen directories, the destination root's metadata ("." here stands for
    // it) is not replayed, and no table is written
    Selection* sel = nullptr;
    const char* out_table = nullptr;
    const char* src_out_table = nullptr;    // vmig_migrate_layer: out_table with the source files' identities
    bool refresh_ids = false;               // the snapshots: record the identities the call's own links moved
    vmig_snapshot_stats* snap_out = nullptr;                // the call-specific stats (nullable)
    vmig_layer_snapshot_stats* layer_snap_out = nullptr;
    vmig_layer_migrate_stats* layer_mig_out = nullptr;
};

// After the data pass: hard-linked paths take their primary's hashes, empty regular files are created, then the rest of
// the tree's metadata is replayed (vmig_tree.h replay_metadata).
// make_empty == false: the caller has already put every empty regular file in place (vmig_rollback_layer keeps one
// that is already right).
int meta_pass(CallScope& call, DstTree& t, const std::vector<uint64_t>& expect, std::vector<uint64_t>* hashes, vmig_stats* st,
              size_t first_dir, bool make_empty = true)
{
    const Manifest& man = *t.m;
    const std::atomic<int>* cancel = call.cancel();
    std::vector<uint64_t>& h = *hashes;
    if (cancel->load()) return fail(VMIG_ECANCELED, "after the data pass, before any metadata step");
    for (auto& e : man.files)                      // hard-linked paths share their primary's hashes
        if (e.hardlink_of >= 0) {
            const Entry& p = man.files[(size_t)e.hardlink_of];
            for (uint64_t r = 0; r < e.n_blocks; r++) {
                h[e.first_block + r] = h[p.first_block + r];
                // restore: the table hashed this path on its own; it must describe the bytes its primary now holds
                // (checked before replay_metadata creates any link)
                if (!expect.empty() && expect[e.first_block + r] != h[e.first_block + r])
                    return fail(VMIG_ECORRUPT, "%s block %llu (a hard link to %s) hashes %016llx, its block table says %016llx",
                                e.rel.c_str(), (unsigned long long)r, p.rel.c_str(), (unsigned long long)h[e.first_block + r],
                                (unsigned long long)expect[e.first_block + r]);
            }
        }
    if (t.hash_only) return VMIG_OK;
    size_t steps = 0;
    for (auto& e : man.files) {                    // empty regular files carry no blocks
        if (e.hardlink_of >= 0 || e.n_blocks || !make_empty) continue;
        if (steps++ % kMetaCheckEvery == 0 && cancel->load()) return fail(VMIG_ECANCELED, "before creating %s", e.rel.c_str());
        const std::string p = pjoin(t.dst_root, e.rel);
        int rc = clear_path(p, "an empty regular file"); if (rc) return rc;
        int fd = open(p.c_str(), O_WRONLY | O_CREAT | O_EXCL | O_CLOEXEC | O_NOFOLLOW, 0600);
        if (fd < 0) return fail(VMIG_EIO, "create %s: %s", p.c_str(), errno_str(errno).c_str());
        rc = apply_file_meta(fd, p, e, t.pol);
        struct stat fst;
        if (!rc && fstat(fd, &fst) == 0) t.ids[&e - &man.files[0]] = file_id(fst);
        close(fd);
        if (rc) return rc;
    }
    return replay_metadata(t.dst_root, man, t.pol, &st->symlinks, &st->hardlinks, &st->specials, cancel, first_dir);
}

// The manifest files that carry blocks (a hard-link group's first path): what VMIG_F_VERIFY re-reads, except
// vmig_snapshot_layer's linked files
std::vector<uint32_t> data_files(const Manifest& man)
{
    std::vector<uint32_t> out;
    for (uint32_t f = 0; f < man.files.size(); f++) if (man.files[f].hardlink_of < 0 && man.files[f].n_blocks) out.push_back(f);
    return out;
}

// VMIG_F_VERIFY: read the given destination files back through the same GPU path (hash only) and compare block tables
int verify_pass(CallScope& call, const vmig_opts& o, const DstTree& t, const std::vector<uint64_t>& hashes, vmig_stats* st,
                const std::vector<std::string>* prune_scope, const std::vector<uint32_t>& files)
{
    const Manifest& man = *t.m;
    FileIO vio;
    vio.src_root = t.dst_root; vio.dst_root = t.dst_root; vio.pol = t.pol; vio.hash_only = true;
    vio.direct = t.direct;           // O_DIRECT re-read: what is verified is what the device holds, not the page cache
    vio.cufile = t.cufile;
    TreePlan blank;                  // nothing patched in place or taken from a base: every block is read back
    blank.files.resize(man.files.size());
    {
        std::vector<BlockSpan> spans;
        for (uint32_t f : files) spans.push_back({f, man.files[f].size, man.files[f].first_block, man.files[f].n_blocks});
        interleave_blocks(spans, o.block_bytes, &blank.blocks);
    }
    vio.init_files(man, blank);
    int rc = vio.open_root(); if (rc) return rc;
    const std::vector<BlockRef>& vblocks = blank.blocks;
    std::vector<uint64_t> vh(man.n_blocks, 0);
    vmig_stats vst; memset(&vst, 0, sizeof vst);
    rc = run_blocks(vblocks, &vio, false, true, o, vh.data(), &vst, call.ctl, true);
    if (rc) return rc;
    st->kernel_launches += vst.kernel_launches; st->ms_kernel += vst.ms_kernel; st->bytes_h2d += vst.bytes_h2d;
    for (auto& b : vblocks)
        if (vh[b.table_idx] != hashes[b.table_idx])
            return fail(VMIG_EVERIFY, "verify: %s block %llu hashes %016llx in the destination, %016llx in the source",
                        man.files[b.file].rel.c_str(), (unsigned long long)(b.file_off / o.block_bytes),
                        (unsigned long long)vh[b.table_idx], (unsigned long long)hashes[b.table_idx]);
    if (o.flags & VMIG_F_PRUNE) {               // the destination's entry set must now equal the source's
        uint64_t extras = 0;
        rc = prune_extras(t.dst_root, man, true, &extras, call.cancel(), prune_scope); if (rc) return rc;
        if (extras) return fail(VMIG_EVERIFY, "verify: %llu destination entries are not in the source after pruning", (unsigned long long)extras);
    }
    return VMIG_OK;
}

// Record the identity the given files have now, each by an lstat of its destination path: for those whose ctime moved
// after their writer recorded it.  Nothing later in the call touches these inodes.
int record_ids(DstTree& t, const std::vector<uint32_t>& files)
{
    for (uint32_t f : files) {
        const std::string p = pjoin(t.dst_root, t.m->files[f].rel);
        struct stat ls;
        if (lstat(p.c_str(), &ls) != 0) return fail(VMIG_EIO, "lstat %s: %s", p.c_str(), errno_str(errno).c_str());
        t.ids[f] = file_id(ls);
    }
    return VMIG_OK;
}

// The table records each file as the call leaves it
int write_table(const DstTree& t, const char* out_path, const std::vector<uint64_t>& hashes, const std::atomic<int>* cancel)
{
    const Manifest& man = *t.m;
    if (!out_path || !*out_path) return VMIG_OK;
    BlockTable tab; tab.block_bytes = t.block_bytes; tab.algo = 1;
    tab.files.reserve(man.files.size());
    for (uint32_t f = 0; f < man.files.size(); f++) {
        const Entry& e = man.files[f];
        const bool own = e.hardlink_of < 0 && (e.n_blocks || !t.hash_only);      // hard-linked paths are never patched in place
        tab.files.push_back({e.rel, e.size, e.first_block, own ? t.ids[f].ino : 0, own ? t.ids[f].ctime_ns : 0});
    }
    tab.hashes = hashes;
    wait_past_recorded_ctimes(tab);
    return table_store(out_path, tab, cancel);
}

// VMIG_F_MOVE_SRC: the old volume's data is about to be unlinked, so deferred write-back errors (ENOSPC / EIO on delayed
// allocation, network filesystems) must surface first: a no-op on tmpfs, one flush on a disk.  A cancelled call leaves
// no table, also when the cancel comes after the table was renamed into place.
int finish_move(CallScope& call, const std::string& src, const std::string& dst, const Manifest& man, const char* out_path)
{
    auto cancelled = [&](const char* when) {
        if (out_path && *out_path) unlink(out_path);
        return fail(VMIG_ECANCELED, "%s (source left in place)", when);
    };
    if (call.cancel()->load()) return cancelled("before the destination was flushed");
    int dfd = open(dst.c_str(), O_RDONLY | O_DIRECTORY | O_CLOEXEC);
    if (dfd < 0) return fail(VMIG_EIO, "open %s: %s", dst.c_str(), errno_str(errno).c_str());
    const int sr = syncfs(dfd); const int se = errno;
    close(dfd);
    if (sr != 0) return fail(VMIG_EIO, "syncfs %s: %s (source left in place)", dst.c_str(), errno_str(se).c_str());
    if (call.cancel()->load()) return cancelled("before the first unlink");
    // the point of no return: a half-unlinked source is worse than a finished move, so a cancel is no longer honoured
    call.phase(VMIG_PHASE_UNLINK);
    return remove_source(src, man);
}

// a is root or lies beneath it (both real paths)
bool path_inside(const std::string& a, const std::string& root)
{
    return a == root || (a.size() > root.size() && a.compare(0, root.size(), root) == 0 && (root == "/" || a[root.size()] == '/'));
}

// The layer calls: the trusted source files none of whose blocks is read are linked or backfilled from the base
// (vmig_snapshot_layer) or left as the prior record they are (vmig_migrate_layer), then finished, as their last block's
// writer finishes a file that was read; spread over as many threads as a lane has writers
int finish_unread(CallScope& call, const vmig_opts& o, FileIO& io, const std::vector<uint32_t>& files)
{
    if (files.empty()) return VMIG_OK;
    uint32_t readers, writers;
    io_threads_default(&readers, &writers, o.io_threads, 1, 1, files.size() >= 32, true, false);
    const size_t n_threads = std::min<size_t>(files.size(), std::max<uint32_t>(writers, 1));
    std::atomic<size_t> next{0};
    std::atomic<int> err{0};
    std::string err_msg; std::mutex err_mu;
    auto work = [&] {
        for (size_t i = next++; i < files.size() && !err.load(); i = next++) {
            const uint32_t f = files[i];
            const int rc = call.cancel()->load() ? fail(VMIG_ECANCELED, "before the unread file %s was finished", io.m->files[f].rel.c_str())
                                                 : io.finish_file(f);
            int none = 0;
            if (rc && err.compare_exchange_strong(none, rc)) { std::lock_guard<std::mutex> lk(err_mu); err_msg = last_error_cstr(); }
        }
    };
    std::vector<std::thread> th;
    for (size_t t = 1; t < n_threads; t++) th.emplace_back(work);
    work();
    for (auto& t : th) t.join();
    if (err.load()) set_last_error_str(err_msg);
    return err.load();
}

// The layer calls, after the data pass: every trusted source file must still be its record, or the hashes the call took
// from the record may not be the bytes the source holds
int recheck_trusted(const std::string& src, const Manifest& man, const TreePlan& plan)
{
    for (uint32_t f = 0; f < man.files.size(); f++) {
        const TableFile* rec = plan.files[f].layer_rec;
        if (!rec) continue;
        struct stat ls;
        if (lstat(pjoin(src, man.files[f].rel).c_str(), &ls) != 0 || !is_recorded_file(ls, *rec))
            return fail(VMIG_ESRCCHANGED, "source file %s changed during the call: it is no longer the file its table record "
                        "vouched for", man.files[f].rel.c_str());
    }
    return VMIG_OK;
}

// The passes of a tree call after its manifest is walked and checked and its tables are loaded: plan, (prune), data,
// metadata, (verify), table, (move).  st arrives with the walk's and the table loads' times.
int tree_passes(CallScope& call, const TreeCall& c, const vmig_opts& o, vmig_stats& st, uint64_t t_begin, vmig_stats* stats_out)
{
    const std::string& src = c.src;
    const std::string& dst = c.dst;
    const Manifest& man = *c.man;
    const BlockTable* layer = c.layer;
    Selection* sel = c.sel;
    const std::atomic<int>* cancel = call.cancel();
    const bool hash_only = (o.flags & VMIG_F_HASH_ONLY) != 0;
    int rc;
    uint64_t t0 = now_ns();
    // a hard link cannot cross devices, and a base on another filesystem shares nothing with the snapshot
    struct stat bst, dst_st;
    const bool has_base = c.base && stat(c.base_dir.c_str(), &bst) == 0 && stat(dst.c_str(), &dst_st) == 0 && bst.st_dev == dst_st.st_dev;
    if (sel) {
        if (cancel->load()) return fail(VMIG_ECANCELED, "before the destination's parent directories were made");
        rc = prepare_parents(dst, sel, cancel);
        if (rc) return rc;
    }
    FileIO io;
    io.src_root = src; io.dst_root = dst; io.pol = default_meta_policy(o.flags); io.hash_only = hash_only;
    io.block_bytes = o.block_bytes;
    io.corrupt_block = env_long("VMIG_CORRUPT_BLOCK", -1);
    io.direct = (o.flags & VMIG_F_DIRECT_IO) != 0;
    io.cufile = (o.flags & VMIG_F_CUFILE) != 0;
    io.cancel = cancel;
    if (io.cufile) { rc = cufile_open(); if (rc) return rc; }
    rc = io.open_root(); if (rc) return rc;
    TreePlan plan;
    rc = plan_tree(man, o.block_bytes, dst, c.prior, has_base ? c.base_dir : "", has_base ? c.base : nullptr, cancel, &plan, src, layer);
    if (rc) return rc;
    st.files_untrusted = plan.files_untrusted;
    io.init_files(man, plan);
    const bool src_out = c.src_out_table && *c.src_out_table;
    if (src_out) {
        io.hold_sources();
        for (uint32_t f : plan.unread)                     // a trusted unread file keeps its record's identity
            if (plan.files[f].solo) io.src_ids[f] = {plan.files[f].layer_rec->ino, plan.files[f].layer_rec->ctime_ns};
    }
    // a trusted layer file's hashes are its record's: the unread blocks keep them, K1 must return them for the rest
    std::vector<uint64_t> hashes = layer ? plan.layer_hashes : std::vector<uint64_t>(man.n_blocks, 0);
    if (has_base) { io.base_root = c.base_dir; io.bidx = &plan.bidx; io.hashes = hashes.data(); }
    // skip mode whenever the base can supply a block, also when no source path has a same-path record (a layer whose
    // files were all moved): without it the submitter streams every block back with its hash (DESIGN.md §3)
    const bool skip_mode = c.prior || plan.any_base || !plan.bidx.empty();
    if ((plan.any_base || !plan.bidx.empty()) && io.skipped.empty()) io.skipped.assign(man.n_blocks, 0);
    if (layer) { call.ctl->bytes_total.store(plan.bytes_read); call.ctl->blocks_total.store(plan.blocks.size()); }
    st.ns_plan += now_ns() - t0;
    const std::vector<std::string>* prune_scope = sel ? &sel->chosen_dirs : nullptr;

    // VMIG_F_PRUNE runs first: what it removes is by definition not in the source, a directory sitting where the source
    // now has a file (or the reverse) is out of the way before anything is created, and the directory mtimes restored
    // at the end are not disturbed by unlinks
    if ((o.flags & VMIG_F_PRUNE) && !hash_only) {
        call.phase(VMIG_PHASE_PRUNE);
        rc = prune_extras(dst, man, false, &st.pruned, cancel, prune_scope);
        if (rc) return rc;
    }
    call.phase(VMIG_PHASE_DATA);
    if (cancel->load()) return fail(VMIG_ECANCELED, "before the destination's directories were made");
    if (!hash_only) { rc = make_dirs(dst, man); if (rc) return rc; }

    t0 = now_ns();
    BlockExpect bexp;
    if (!c.expect.empty()) bexp.hashes = c.expect.data();
    if (layer) { bexp.hashes = plan.layer_hashes.data(); bexp.valid = plan.expect.data(); bexp.code = VMIG_ESRCCHANGED; }
    if (layer) rc = finish_unread(call, o, io, plan.unread);
    if (!rc) rc = run_blocks(plan.blocks, &io, skip_mode, hash_only, o, hashes.data(), &st, call.ctl, false, bexp.hashes ? &bexp : nullptr);
    if (!rc && layer) rc = recheck_trusted(src, man, plan);
    st.ns_data = now_ns() - t0;
    if (rc) return rc;

    t0 = now_ns();
    call.phase(VMIG_PHASE_META);
    rc = meta_pass(call, io, c.expect, &hashes, &st, sel ? 1 : 0);
    if (rc) return rc;
    st.ns_meta = now_ns() - t0;

    uint64_t n_verified = 0, b_verified = 0;
    if ((o.flags & VMIG_F_VERIFY) && !hash_only) {
        call.phase(VMIG_PHASE_VERIFY);
        std::vector<uint32_t> files = data_files(man);
        if (layer) {
            // a layer call does not re-read what it linked (the base table already vouches for it) nor what it left alone
            // (it still is its prior record).  vmig_snapshot_layer has no prior and vmig_migrate_layer no base, so in each
            // call only one of the two tests can remove a file.
            std::unordered_set<uint32_t> linked(io.linked_files.begin(), io.linked_files.end());
            files.erase(std::remove_if(files.begin(), files.end(), [&](uint32_t f) {
                const TableFile* pr = plan.files[f].prior_rec;
                return linked.count(f) != 0 || (pr && !io.fs[f].wrote.load() && pr->size == man.files[f].size);
            }), files.end());
        }
        for (uint32_t f : files) { n_verified++; b_verified += man.files[f].size; }
        rc = verify_pass(call, o, io, hashes, &st, prune_scope, files);
        if (rc) return rc;
    }

    if (!sel) {
        t0 = now_ns();
        call.phase(VMIG_PHASE_TABLE);
        if (c.refresh_ids) {
            // a snapshot's table must let the next increment trust it: a linked path's ctime moved with this call's link to
            // the base inode, and a hard-linked file's with replay_metadata's link, both after block_done recorded it
            std::vector<uint32_t> moved = io.linked_files;
            for (uint32_t f = 0; f < man.files.size(); f++) if (!plan.files[f].solo && man.files[f].n_blocks) moved.push_back(f);
            rc = record_ids(io, moved);
        }
        if (!rc && src_out) {
            // the source's table first, under the cancel; once it is in place the call commits, and a failure to store
            // out_table takes it away again
            DstTree sv = static_cast<const DstTree&>(io);
            sv.ids = io.src_ids;
            rc = write_table(sv, c.src_out_table, hashes, cancel);
            if (!rc && (rc = write_table(io, c.out_table, hashes, nullptr))) unlink(c.src_out_table);
        } else if (!rc) {
            rc = write_table(io, c.out_table, hashes, cancel);
        }
        if (rc) return rc;
        st.ns_table = now_ns() - t0;
    }

    if ((o.flags & VMIG_F_MOVE_SRC) && !hash_only) {
        rc = finish_move(call, src, dst, man, c.out_table);
        if (rc) return rc;
    }

    st.files_direct = io.src.n_direct.load() + io.n_direct.load();
    st.bytes_total = man.bytes_total; st.blocks_total = man.n_blocks;
    if (layer) { st.bytes_total = call.ctl->bytes_total.load(); st.blocks_total = call.ctl->blocks_total.load(); }
    st.files = man.files.size(); st.dirs = man.dirs.size() - (sel ? 1 : 0);
    st.ns_total = now_ns() - t_begin;
    if (stats_out) *stats_out = st;
    if (c.snap_out) {
        vmig_snapshot_stats ss; memset(&ss, 0, sizeof ss);
        ss.files_base_untrusted = plan.files_base_untrusted;
        ss.files_linked = io.n_linked.load(); ss.bytes_linked = io.b_linked.load();
        ss.files_backfilled = io.n_backfilled.load(); ss.bytes_backfilled = io.b_backfilled.load();
        *c.snap_out = ss;
    }
    if (c.layer_snap_out) {
        vmig_layer_snapshot_stats ls; memset(&ls, 0, sizeof ls);
        ls.files_linked = io.n_linked.load(); ls.bytes_linked = io.b_linked.load();
        ls.files_backfilled = io.n_backfilled.load(); ls.bytes_backfilled = io.b_backfilled.load();
        ls.files_base_untrusted = plan.files_base_untrusted;
        ls.files_trusted = plan.files_trusted; ls.bytes_trusted = plan.bytes_trusted;
        ls.files_read = plan.files_read; ls.bytes_read = plan.bytes_read;
        *c.layer_snap_out = ls;
    }
    if (c.layer_mig_out) {
        vmig_layer_migrate_stats ms; memset(&ms, 0, sizeof ms);
        ms.files_trusted = plan.files_trusted; ms.bytes_trusted = plan.bytes_trusted;
        ms.files_read = plan.files_read; ms.bytes_read = plan.bytes_read;
        ms.files_unread = plan.unread.size();
        ms.files_verified = n_verified; ms.bytes_verified = b_verified;
        if (src_out)
            for (const FileId& id : io.src_ids) (id.ino ? ms.src_recorded : ms.src_unrecorded)++;
        *c.layer_mig_out = ms;
    }
    return VMIG_OK;
}

// A table a call names (path NULL or empty: none), loaded at the call's block size into *t
struct NamedTable { const char* path; const char* what; BlockTable* t; };

// The refusals of a call after its arguments, in this order: a cancelled control, a directory that is missing or not a
// directory, a table that does not load, no GPU.  No CPU fallback: the GPU is there before anything is touched.
int start_checks(CallScope& call, const vmig_opts& o, std::initializer_list<const char*> dirs, const std::vector<NamedTable>& tables)
{
    if (call.cancel()->load()) return fail(VMIG_ECANCELED, "the control was cancelled before the call started");
    for (const char* d : dirs) {
        struct stat sb;
        if (stat(d, &sb) != 0 || !S_ISDIR(sb.st_mode)) return fail(VMIG_ENOTDIR, "%s is missing or not a directory", d);
    }
    for (const NamedTable& n : tables)
        if (n.path && *n.path) { const int rc = load_table(n.path, n.what, o.block_bytes, n.t); if (rc) return rc; }
    std::vector<DeviceInfo> devs;
    return ctx_select(o.gpu_mask, &devs);
}

// The tree calls' refusals after the arguments, in this order: a directory that cannot be stat'ed (VMIG_EIO) or is
// not a directory (NULL: not checked), then start_checks' cancel and GPU
int tree_start_checks(CallScope& call, const vmig_opts& o, std::initializer_list<const char*> dirs)
{
    for (const char* d : dirs) {
        struct stat sb;
        if (!d) continue;
        if (stat(d, &sb) != 0) return fail(VMIG_EIO, "stat %s: %s", d, errno_str(errno).c_str());
        if (!S_ISDIR(sb.st_mode)) return fail(VMIG_ENOTDIR, "%s is not a directory", d);
    }
    return start_checks(call, o, {}, {});
}

// vmig_migrate_tree, vmig_restore_tree, vmig_snapshot_tree, vmig_copy_dir and vmig_move_dir: the refusals after the
// arguments, the walk, then the tables the call names, loaded into c in this order: snap_path (vmig_restore_tree:
// src_dir must be the tree that table describes, checked before anything touches the destination), prior_path (not
// under VMIG_F_HASH_ONLY), base_table.  c arrives with the rest: out_table, and a snapshot's base_dir, identity
// refresh and stats.
int migrate_tree_body(CallScope& call, TreeCall c, const char* src_dir, const char* dst_dir, const char* prior_path,
                      const char* snap_path, const char* base_table, const vmig_opts& o, vmig_stats* stats_out)
{
    vmig_stats st; memset(&st, 0, sizeof st);
    const uint64_t t_begin = now_ns();
    if (!src_dir || !*src_dir) return fail(VMIG_EINVAL, "src_dir is NULL/empty");
    const bool hash_only = (o.flags & VMIG_F_HASH_ONLY) != 0;
    if (!hash_only && (!dst_dir || !*dst_dir)) return fail(VMIG_EINVAL, "dst_dir is NULL/empty");
    int rc = check_block_bytes(o);
    if (!rc) rc = tree_start_checks(call, o, {src_dir, hash_only ? nullptr : dst_dir});
    if (rc) return rc;
    c.src = src_dir; c.dst = dst_dir ? dst_dir : "";

    Manifest man;
    uint64_t t0 = now_ns();
    call.phase(VMIG_PHASE_WALK);
    rc = walk_tree(c.src, o.block_bytes, (o.flags & VMIG_F_SKIP_HIDDEN_TOPDIRS) != 0, &man, call.cancel());
    if (rc) return rc;
    st.ns_walk = now_ns() - t0;
    call.ctl->bytes_total.store(man.bytes_total); call.ctl->blocks_total.store(man.n_blocks);
    c.man = &man;

    t0 = now_ns();
    BlockTable snap, prior, base;
    if (snap_path) {
        rc = load_table(snap_path, "snapshot", o.block_bytes, &snap);
        if (!rc) rc = match_table(man, snap, &c.expect);
    }
    if (!rc && prior_path && *prior_path && !hash_only) { rc = load_table(prior_path, "prior", o.block_bytes, &prior); c.prior = &prior; }
    if (!rc && base_table) { rc = load_table(base_table, "base", o.block_bytes, &base); c.base = &base; }
    if (rc) return rc;
    st.ns_plan = now_ns() - t0;
    return tree_passes(call, c, o, st, t_begin, stats_out);
}

// vmig_restore_paths: the chosen entries of a snapshot, checked against the part of its table they cover (DESIGN.md §6)
int restore_paths_body(CallScope& call, const char* snap_dir, const char* snap_table, const char* dst_dir,
                       const std::vector<std::string>& paths, const char* prior_path, const vmig_opts& o, vmig_stats* stats_out)
{
    const std::atomic<int>* cancel = call.cancel();
    vmig_stats st; memset(&st, 0, sizeof st);
    const uint64_t t_begin = now_ns();
    int rc = tree_start_checks(call, o, {snap_dir, dst_dir});
    if (rc) return rc;
    TreeCall c;
    c.src = snap_dir; c.dst = dst_dir;

    uint64_t t0 = now_ns();
    call.phase(VMIG_PHASE_WALK);
    Selection sel;
    rc = select_walk(c.src, paths, o.block_bytes, (o.flags & VMIG_F_SKIP_HIDDEN_TOPDIRS) != 0, &sel, cancel);
    if (rc) return rc;
    st.ns_walk = now_ns() - t0;
    call.ctl->bytes_total.store(sel.man.bytes_total); call.ctl->blocks_total.store(sel.man.n_blocks);
    c.man = &sel.man; c.sel = &sel;

    t0 = now_ns();
    BlockTable snap;
    rc = load_table(snap_table, "snapshot", o.block_bytes, &snap);
    if (rc) return rc;
    for (const std::string& p : sel.not_found) {
        BlockTable under;
        table_subset(snap, {p}, &under);
        if (!under.files.empty())
            return fail(VMIG_ECORRUPT, "%s is in the block table but not in the snapshot (missing)", under.files[0].rel.c_str());
        return fail(VMIG_EINVAL, "%s is not in the snapshot", p.c_str());
    }
    BlockTable part, prior;                          // records outside the selection are not looked at
    table_subset(snap, sel.paths, &part);
    rc = match_table(sel.man, part, &c.expect);
    if (!rc && prior_path && *prior_path) { rc = load_table(prior_path, "prior", o.block_bytes, &prior); c.prior = &prior; }
    if (rc) return rc;
    st.ns_plan = now_ns() - t0;
    return tree_passes(call, c, o, st, t_begin, stats_out);
}

// The real path of p; empty when it does not resolve (errno says why)
std::string real_path(const char* p)
{
    char* r = realpath(p, nullptr);
    const std::string s = r ? r : "";
    free(r);
    return s;
}

// Refuses real paths ra and rb (named a and b, a first in the message) that are the same directory or where one lies
// inside the other.  An empty one, a path that does not resolve, is left to the call's own checks.
int check_apart(const char* a, const std::string& ra, const char* b, const std::string& rb)
{
    if (ra.empty() || rb.empty() || !(path_inside(ra, rb) || path_inside(rb, ra))) return VMIG_OK;
    return fail(VMIG_EINVAL, "%s %s and %s %s are the same directory or one is inside the other", a, ra.c_str(), b, rb.c_str());
}

int migrate_tree_impl(const TreeCall& c, const char* src_dir, const char* dst_dir, const char* prior_path, const char* snap_path,
                      const char* base_table, const vmig_opts* opts_in, vmig_stats* stats_out)
{
    const vmig_opts o = norm_opts(opts_in);
    return in_call(o.ctl, [&](CallScope& call) {
        return migrate_tree_body(call, c, src_dir, dst_dir, prior_path, snap_path, base_table, o, stats_out);
    });
}

// vmig_snapshot_tree: a base directory equal to the destination, or either one inside the other, is refused -- a
// link or backfill would read what the same call is writing.  A directory that does not resolve is refused too: a
// missing base must not become a full snapshot.
int check_snapshot_paths(const char* dst_dir, const char* base_dir)
{
    const std::string ds = real_path(dst_dir);
    if (ds.empty()) return fail(VMIG_EIO, "realpath %s: %s", dst_dir, errno_str(errno).c_str());
    const std::string bs = real_path(base_dir);
    if (bs.empty()) return fail(VMIG_EIO, "realpath %s: %s", base_dir, errno_str(errno).c_str());
    return check_apart("base_dir", bs, "dst_dir", ds);
}

// ---------------------------------------------------------------------------------------------
// vmig_scrub_store, vmig_retire_versions and vmig_compare_snapshot read each distinct inode once (ScrubInode, vmig_scrub.h)

// The root directories of a call's versions, opened as the call needs them and closed with the holder
struct VersionRoots {
    std::vector<int> fds;                            // -1: not opened
    explicit VersionRoots(size_t n) : fds(n, -1) {}
    VersionRoots(const VersionRoots&) = delete;
    ~VersionRoots() { for (int fd : fds) if (fd >= 0) close(fd); }
    int open(size_t v, const char* dir) {
        fds[v] = ::open(dir, O_RDONLY | O_DIRECTORY | O_CLOEXEC);
        return fds[v] >= 0 ? VMIG_OK : fail(VMIG_ESRCCHANGED, "open %s: %s", dir, errno_str(errno).c_str());
    }
};

// The data pass over inodes: every block through *reader (each inode opened beneath roots[its version]) in a migration's
// block order, hashed by K1 in hash-only mode into *hashes at the inodes' block ranges.  What an unreadable inode means
// is the caller's (reader->unreadable).  Sets the call's progress totals and st's data-pass fields.
int inode_pass(CallScope& call, const vmig_opts& o, const std::vector<int>& roots, const std::vector<ScrubInode>& inodes,
               ScrubReader* reader, std::vector<uint64_t>* hashes, vmig_stats* st)
{
    const uint64_t t0 = now_ns();
    uint64_t bytes = 0, n_blocks = 0;
    for (const ScrubInode& I : inodes) { bytes += I.size; n_blocks += I.n_blocks; }
    call.ctl->bytes_total.store(bytes); call.ctl->blocks_total.store(n_blocks);
    reader->root_fds = roots; reader->inodes = &inodes; reader->direct = (o.flags & VMIG_F_DIRECT_IO) != 0;
    reader->block_bytes = o.block_bytes;
    reader->init();
    std::vector<BlockSpan> spans;
    for (uint32_t u = 0; u < inodes.size(); u++) spans.push_back({u, inodes[u].size, inodes[u].first_block, inodes[u].n_blocks});
    std::vector<BlockRef> blocks; blocks.reserve(n_blocks);
    interleave_blocks(spans, o.block_bytes, &blocks);
    call.phase(VMIG_PHASE_DATA);
    if (call.cancel()->load()) return fail(VMIG_ECANCELED, "before the data pass");
    hashes->assign(n_blocks, 0);
    const int rc = run_blocks(blocks, reader, false, true, o, hashes->data(), st, call.ctl, false);
    reader->close_all();
    st->ns_data = now_ns() - t0;
    st->files_direct = reader->fds.n_direct.load();
    st->bytes_total = bytes; st->blocks_total = n_blocks; st->files = inodes.size();
    return rc;
}

int scrub_body(CallScope& call, uint32_t n, const char* const* dirs, const char* const* tables, const char* report_path,
               int32_t* verdicts_out, const vmig_opts& o, vmig_stats* stats_out, vmig_scrub_stats* ss_out)
{
    const std::atomic<int>* cancel = call.cancel();
    vmig_stats st; memset(&st, 0, sizeof st);
    vmig_scrub_stats ss; memset(&ss, 0, sizeof ss);
    const uint64_t t_begin = now_ns();
    int rc = start_checks(call, o, {}, {});
    if (rc) return rc;

    // ---- walk every version, load its table, merge the two (every difference recorded)
    call.phase(VMIG_PHASE_WALK);
    uint64_t t0 = now_ns();
    std::vector<Manifest> man(n);
    std::vector<BlockTable> tab(n);
    std::vector<const Manifest*> walked(n, nullptr);
    std::vector<std::vector<int64_t>> tab_of(n);
    std::vector<int32_t> verdict(n, VMIG_OK);
    std::vector<ScrubFinding> findings;
    auto whole = [&](uint32_t v, ScrubKind k, const char* path) {
        ScrubFinding f; f.version = v; f.kind = k; f.path = path; findings.push_back(f);
    };
    for (uint32_t v = 0; v < n; v++) {
        struct stat sb;
        if (stat(dirs[v], &sb) != 0 || !S_ISDIR(sb.st_mode)) { verdict[v] = VMIG_ENOTDIR; whole(v, kScrubDir, "."); continue; }
        rc = walk_tree(dirs[v], o.block_bytes, (o.flags & VMIG_F_SKIP_HIDDEN_TOPDIRS) != 0, &man[v], cancel);
        if (rc == VMIG_ECANCELED || rc == VMIG_ESRCCHANGED || rc == VMIG_ENOMEM) return rc;
        if (rc) { verdict[v] = VMIG_ECORRUPT; whole(v, kScrubUnreadable, "."); continue; }      // a directory that cannot be read
        ss.bytes_referenced += man[v].bytes_total;
        if (table_load(tables[v], &tab[v]) != VMIG_OK || tab[v].block_bytes != o.block_bytes) { verdict[v] = VMIG_ETABLE; whole(v, kScrubTable, "."); continue; }
        if (scrub_merge_table(v, man[v], tab[v], &tab_of[v], &findings)) verdict[v] = VMIG_ECORRUPT;
        walked[v] = &man[v];
    }
    st.ns_walk = now_ns() - t0;

    // ---- the distinct inodes, and the roots they are opened beneath
    t0 = now_ns();
    std::vector<ScrubInode> inodes;
    std::vector<std::vector<uint32_t>> inode_of;
    rc = scrub_group_inodes(walked, tab_of, o.block_bytes, &inodes, &inode_of);
    if (rc) return rc;
    VersionRoots roots(n);
    for (const ScrubInode& I : inodes)
        if (roots.fds[I.version] < 0 && (rc = roots.open(I.version, dirs[I.version]))) return rc;
    st.ns_plan = now_ns() - t0;

    // ---- the data pass: K1 over every distinct block, once
    ScrubReader reader;
    std::vector<uint64_t> hashes;
    rc = inode_pass(call, o, roots.fds, inodes, &reader, &hashes, &st);
    if (rc) return rc;
    ss.bytes_unique = st.bytes_total;

    // ---- compare every table record with the hashes of the inode it names
    t0 = now_ns();
    std::unordered_set<uint64_t> bad_blocks;
    for (uint32_t v = 0; v < n; v++) {
        if (!walked[v]) continue;
        const Manifest& m = man[v];
        for (size_t f = 0; f < m.files.size(); f++) {
            const uint32_t u = inode_of[v][f];
            if (u == kNoInode) continue;
            const Entry& e = m.files[f];
            const ScrubInode& I = inodes[u];
            if (reader.unreadable(u)) { verdict[v] = VMIG_ECORRUPT; whole(v, kScrubUnreadable, e.rel.c_str()); continue; }
            const TableFile& tf = tab[v].files[(size_t)tab_of[v][f]];
            for (uint64_t r = 0; r < e.n_blocks; r++) {
                const uint64_t got = hashes[I.first_block + r], want = tab[v].hashes[tf.first_block + r];
                if (got == want) continue;
                ScrubFinding x; x.version = v; x.kind = e.hardlink_of >= 0 ? kScrubHardlink : kScrubBlock; x.path = e.rel;
                x.block = (int64_t)r; x.has_hashes = true; x.got = got; x.want = want;
                findings.push_back(x);
                bad_blocks.insert(I.first_block + r);
                verdict[v] = VMIG_ECORRUPT;
            }
        }
    }
    for (uint32_t u = 0; u < inodes.size(); u++) ss.files_unreadable += reader.unreadable(u);
    scrub_sort(&findings);
    for (size_t i = 0; i < findings.size(); i++) {
        const ScrubFinding& f = findings[i];
        if (f.kind == kScrubTable || f.kind == kScrubDir || (f.kind == kScrubUnreadable && f.path == ".")) continue;
        if (i && findings[i - 1].version == f.version && findings[i - 1].path == f.path) continue;   // sorted: one count per path
        ss.files_damaged++;
    }
    ss.versions = n; ss.blocks_damaged = bad_blocks.size();
    for (int32_t x : verdict) ss.versions_damaged += x != VMIG_OK;
    if (report_path && *report_path) {
        rc = scrub_report_store(report_path, findings, cancel);
        if (rc) return rc;
    }
    st.ns_table = now_ns() - t0;
    st.ns_total = now_ns() - t_begin;
    if (verdicts_out) std::copy(verdict.begin(), verdict.end(), verdicts_out);
    if (stats_out) *stats_out = st;
    if (ss_out) *ss_out = ss;
    return VMIG_OK;
}

// ---------------------------------------------------------------------------------------------
// vmig_retire_versions: the removal and the re-stamp plan are vmig_retire.cpp's; the re-verify is inode_pass over
// the stale records' inodes
// The real path of p without following its last component (it may be a symlink, or missing): realpath of the parent
// plus the name.  A parent that does not exist leaves p as given (nothing can be removed beneath it).
int real_parent_path(const char* p, std::string* out)
{
    std::string s(p);
    while (s.size() > 1 && s.back() == '/') s.pop_back();
    const size_t slash = s.rfind('/');
    const std::string parent = slash == std::string::npos ? "." : slash == 0 ? "/" : s.substr(0, slash);
    const std::string base = slash == std::string::npos ? s : s.substr(slash + 1);
    if (base.empty() || base == "." || base == ".." || base == "/") return fail(VMIG_EINVAL, "%s names no directory entry", p);
    char* r = realpath(parent.c_str(), nullptr);
    if (!r) {
        if (errno != ENOENT) return fail(VMIG_EIO, "realpath %s: %s", parent.c_str(), errno_str(errno).c_str());
        *out = s;
        return VMIG_OK;
    }
    *out = std::string(r) + (strcmp(r, "/") ? "/" : "") + base;
    free(r);
    return VMIG_OK;
}

struct RetireArgs {
    std::vector<std::string> retire_dirs, retire_tables, keep_dirs, keep_tables;   // real paths
};

// the refusals that touch nothing, before the call is attached
int check_retire_args(uint32_t n_retire, const char* const* retire_dirs, const char* const* retire_tables, uint32_t n_keep,
                      const char* const* keep_dirs, const char* const* keep_tables, RetireArgs* a)
{
    for (uint32_t i = 0; i < n_retire; i++) {
        std::string d, t;
        int rc = real_parent_path(retire_dirs[i], &d);
        if (!rc) rc = real_parent_path(retire_tables[i], &t);
        if (rc) return rc;
        struct stat st;
        if (lstat(d.c_str(), &st) == 0 && !S_ISDIR(st.st_mode))
            return fail(VMIG_ENOTDIR, "retired version %s is not a directory (a symlink is not followed)", retire_dirs[i]);
        a->retire_dirs.push_back(d); a->retire_tables.push_back(t);
    }
    for (uint32_t i = 0; i < n_keep; i++) {
        char* r = realpath(keep_dirs[i], nullptr);
        struct stat st;
        if (!r || stat(r, &st) != 0 || !S_ISDIR(st.st_mode)) { free(r); return fail(VMIG_ENOTDIR, "kept version %s is not a directory", keep_dirs[i]); }
        a->keep_dirs.push_back(r);
        free(r);
        std::string t;
        const int rc = real_parent_path(keep_tables[i], &t);
        if (rc) return rc;
        a->keep_tables.push_back(t);
    }
    std::vector<std::string> all(a->retire_dirs);
    all.insert(all.end(), a->keep_dirs.begin(), a->keep_dirs.end());
    for (size_t i = 0; i < all.size(); i++)
        for (size_t j = i + 1; j < all.size(); j++)
            if (path_inside(all[i], all[j]) || path_inside(all[j], all[i]))
                return fail(VMIG_EINVAL, "%s and %s are the same directory or one is inside the other", all[i].c_str(), all[j].c_str());
    for (const std::string& t : a->retire_tables)
        for (size_t k = 0; k < n_keep; k++)
            if (t == a->keep_tables[k] || path_inside(t, a->keep_dirs[k]))
                return fail(VMIG_EINVAL, "retired table %s is kept version %s's table or lies inside it", t.c_str(), a->keep_dirs[k].c_str());
    for (const std::string& t : a->keep_tables)
        for (const std::string& d : a->retire_dirs)
            if (path_inside(t, d)) return fail(VMIG_EINVAL, "kept table %s lies inside retired version %s", t.c_str(), d.c_str());
    return VMIG_OK;
}

int retire_body(CallScope& call, const RetireArgs& a, const vmig_opts& o, vmig_stats* stats_out, vmig_retire_stats* rs_out)
{
    const std::atomic<int>* cancel = call.cancel();
    vmig_stats st; memset(&st, 0, sizeof st);
    vmig_retire_stats rs; memset(&rs, 0, sizeof rs);
    const uint64_t t_begin = now_ns();
    const size_t n_keep = a.keep_dirs.size();
    std::vector<BlockTable> tab(n_keep);
    std::vector<NamedTable> kept;
    for (size_t k = 0; k < n_keep; k++) kept.push_back({a.keep_tables[k].c_str(), "kept", &tab[k]});
    int rc = start_checks(call, o, {}, kept);
    if (rc) return rc;

    // ---- remove the retired versions, table first
    call.phase(VMIG_PHASE_UNLINK);
    uint64_t t0 = now_ns();
    RemoveCount removed;
    for (size_t i = 0; i < a.retire_dirs.size(); i++) {
        rc = retire_remove(a.retire_dirs[i], a.retire_tables[i], &removed, cancel);
        if (rc) return rc;
        rs.versions_retired++;
    }
    rs.entries_removed = removed.entries; rs.files_freed = removed.files_freed; rs.bytes_freed = removed.bytes_freed;

    // ---- the kept records whose ctime moved, grouped by inode
    call.phase(VMIG_PHASE_WALK);
    VersionRoots roots(n_keep);
    for (size_t k = 0; k < n_keep; k++)
        if ((rc = roots.open(k, a.keep_dirs[k].c_str()))) return rc;
    std::vector<const BlockTable*> tabs;
    for (const BlockTable& t : tab) tabs.push_back(&t);
    std::vector<StaleRecord> stale;
    std::vector<ScrubInode> inodes;
    std::vector<uint32_t> inode_of;
    rc = retire_find_stale(roots.fds, tabs, &stale, cancel);
    if (!rc) rc = retire_group(stale, tabs, o.block_bytes, &inodes, &inode_of);
    if (rc) return rc;
    st.ns_walk = now_ns() - t0;
    rs.records_stale = stale.size();

    // ---- re-verify each stale inode once: K1 in hash-only mode, compared on the host
    ScrubReader reader;
    std::vector<uint64_t> hashes;
    rc = inode_pass(call, o, roots.fds, inodes, &reader, &hashes, &st);
    if (rc) return rc;
    rs.bytes_rehashed = st.bytes_total;
    std::vector<bool> unreadable(inodes.size());
    for (uint32_t u = 0; u < inodes.size(); u++) unreadable[u] = reader.unreadable(u);
    const std::vector<size_t> chosen = retire_decide(roots.fds, tabs, stale, inodes, inode_of, hashes, unreadable);
    rs.records_restamped = chosen.size();

    // ---- rewrite each kept table that gained a verified identity
    call.phase(VMIG_PHASE_TABLE);
    t0 = now_ns();
    for (uint32_t k = 0; k < n_keep; k++) {
        if (!retire_patch(k, stale, chosen, inodes, inode_of, &tab[k])) continue;
        wait_past_recorded_ctimes(tab[k]);
        rc = table_store(a.keep_tables[k], tab[k], cancel);
        if (rc) return rc;
        rs.tables_rewritten++;
    }
    st.ns_table = now_ns() - t0;
    st.ns_total = now_ns() - t_begin;
    if (stats_out) *stats_out = st;
    if (rs_out) *rs_out = rs;
    return VMIG_OK;
}

// ---------------------------------------------------------------------------------------------
// The layer side of vmig_compare_snapshot and vmig_rollback_layer: the layer's walk, where each layer file takes its block
// hashes from (compare_plan: a shared inode, a trusted record of the layer's table, or a read), and the data pass over the
// files that need reading, each distinct inode once through inode_pass (one root: the layer, as version 0)
struct LayerSide {
    Manifest man;
    ComparePlan plan;
    VersionRoots roots{1};
    std::vector<uint64_t> read_hashes;
    std::vector<const uint64_t*> hashes;     // per layer file (compare_layer_hashes)
};

int layer_plan(const char* layer_dir, const Manifest& snap, const BlockTable* ltab, const vmig_opts& o, const std::atomic<int>* cancel,
               LayerSide* L, vmig_stats* st)
{
    uint64_t t0 = now_ns();
    int rc = walk_tree(layer_dir, o.block_bytes, (o.flags & VMIG_F_SKIP_HIDDEN_TOPDIRS) != 0, &L->man, cancel);
    if (rc) return rc;
    st->ns_walk += now_ns() - t0;
    t0 = now_ns();
    rc = compare_plan(layer_dir, L->man, snap, ltab, o.block_bytes, &L->plan);
    if (!rc && !L->plan.inodes.empty()) rc = L->roots.open(0, layer_dir);
    st->ns_plan += now_ns() - t0;
    return rc;
}

// K1 over every block of the distinct layer inodes that need reading, once; then every layer file's hashes
int layer_hash_pass(CallScope& call, const vmig_opts& o, const Manifest& snap, const std::vector<uint64_t>& snap_hashes,
                    const BlockTable* ltab, LayerSide* L, vmig_stats* st)
{
    ScrubReader reader;
    const int rc = inode_pass(call, o, L->roots.fds, L->plan.inodes, &reader, &L->read_hashes, st);
    if (rc) return rc;
    for (uint32_t u = 0; u < L->plan.inodes.size(); u++)
        if (reader.unreadable(u)) return fail(VMIG_EIO, "layer file %s: %s", L->plan.inodes[u].rel.c_str(), reader.why(u).c_str());
    L->hashes = compare_layer_hashes(L->plan, L->man, snap, snap_hashes, ltab, L->read_hashes);
    return VMIG_OK;
}

// The snapshot's walk, which must be the tree its table describes: its manifest and the table's hashes in its block order
int walk_snapshot(CallScope& call, const char* snap_dir, const BlockTable& snap_tab, const vmig_opts& o, Manifest* snap,
                  std::vector<uint64_t>* snap_hashes, vmig_stats* st)
{
    call.phase(VMIG_PHASE_WALK);
    const uint64_t t0 = now_ns();
    int rc = walk_tree(snap_dir, o.block_bytes, (o.flags & VMIG_F_SKIP_HIDDEN_TOPDIRS) != 0, snap, call.cancel());
    if (!rc) rc = match_table(*snap, snap_tab, snap_hashes);
    if (rc) return rc;
    st->ns_walk = now_ns() - t0;
    return VMIG_OK;
}

// vmig_compare_snapshot: the plan, the merge and the report are vmig_compare.cpp's
int compare_body(CallScope& call, const char* layer_dir, const char* layer_table, const char* snap_dir, const char* snap_table,
                 const char* report_path, const vmig_opts& o, vmig_stats* stats_out, vmig_compare_stats* cs_out)
{
    const std::atomic<int>* cancel = call.cancel();
    vmig_stats st; memset(&st, 0, sizeof st);
    vmig_compare_stats cs; memset(&cs, 0, sizeof cs);
    const uint64_t t_begin = now_ns();
    BlockTable snap_tab, layer_tab;
    int rc = start_checks(call, o, {layer_dir, snap_dir}, {{snap_table, "snapshot", &snap_tab}, {layer_table, "layer", &layer_tab}});
    if (rc) return rc;
    const BlockTable* ltab = layer_table && *layer_table ? &layer_tab : nullptr;

    // ---- walk both trees; which layer files are read
    Manifest snap;
    std::vector<uint64_t> snap_hashes;
    rc = walk_snapshot(call, snap_dir, snap_tab, o, &snap, &snap_hashes, &st);
    if (rc) return rc;
    LayerSide L;
    rc = layer_plan(layer_dir, snap, ltab, o, cancel, &L, &st);
    if (!rc) rc = layer_hash_pass(call, o, snap, snap_hashes, ltab, &L, &st);
    if (rc) return rc;

    // ---- the findings, compared on the host (8 bytes per block), and the report
    const uint64_t t0 = now_ns();
    std::vector<CompareFinding> findings;
    CompareCounts c;
    compare_merge(L.man, snap, snap_hashes, L.hashes, o.block_bytes, (o.flags & VMIG_F_MTIME_NS) != 0,
                  (o.flags & VMIG_F_NO_METADATA) != 0, &findings, &c);
    if (report_path && *report_path) {
        std::string raw;
        for (const CompareFinding& f : findings) raw += compare_format(f);
        rc = report_store(report_path, raw, "compare report", cancel);
        if (rc) return rc;
    }
    st.ns_table = now_ns() - t0;
    cs.paths_added = c.paths_added; cs.paths_removed = c.paths_removed; cs.paths_changed = c.paths_changed;
    cs.files_changed = c.files_changed; cs.blocks_changed = c.blocks_changed; cs.bytes_restore = c.bytes_restore;
    cs.files_read = L.plan.inodes.size(); cs.bytes_read = L.plan.bytes_read;
    cs.files_trusted = L.plan.files_trusted; cs.files_shared = L.plan.files_shared;
    st.ns_total = now_ns() - t_begin;
    if (stats_out) *stats_out = st;
    if (cs_out) *cs_out = cs;
    return VMIG_OK;
}

// ---------------------------------------------------------------------------------------------
// vmig_rollback_layer: the actions, the fetch list and the copy runs are vmig_rollback.cpp's.  The snapshot blocks the
// layer lacks are read beneath the snapshot's root and written into the layer file each action names, made ready when its
// first block is written (RollbackIO::prepare); the rest of the tree is a pruning restore's (prune_extras, meta_pass,
// verify_pass, write_table over the snapshot's manifest).
class RollbackIO : public BlockIO {
public:
    const Manifest* snap = nullptr;
    const RollbackPlan* plan = nullptr;
    const std::vector<LayerId>* ids = nullptr;      // per layer file (rollback_identify)
    std::string layer_root;
    int snap_fd = -1;                               // snapshot files are opened beneath it (not owned)
    bool direct = false;                            // VMIG_F_DIRECT_IO
    uint32_t block_bytes = 4u << 20;
    const std::atomic<int>* cancel = nullptr;       // checked per copy chunk of a rebuilt file
    ReadFds src;                                    // per plan file: its snapshot file
    std::atomic<uint64_t> n_direct{0}, b_copied{0};      // layer descriptors opened O_DIRECT; bytes copied from old inodes
    RebuildGuard rebuild_guard;                          // the call's own unlinks of rebuilt paths

    void init() {
        fs.reset(new FS[plan->files.size() ? plan->files.size() : 1]);
        src.init(plan->files.size());
        for (size_t i = 0; i < plan->files.size(); i++) { src.add_reads(i, plan->files[i].n_fetch); fs[i].blocks_left.store(plan->files[i].n_fetch); }
    }
    uint32_t slot_align() override { return direct ? kSector : 512; }
    std::string block_name(const BlockRef& b) override {
        return snap->files[plan->files[b.file].snap].rel + " block " + std::to_string(b.file_off / block_bytes);
    }

    // Make file i of the plan ready to take its fetched blocks: a patched file opened in place (no O_TRUNC), checked and
    // set to the snapshot's size; a rebuilt one replaced by a new inode that first takes the equal blocks from the old
    // one; a created one made new.  *out: the descriptor to write into.
    int prepare(uint32_t i, int* out) {
        const RollbackFile& rf = plan->files[i];
        const Entry& s = snap->files[rf.snap];
        const std::string p = pjoin(layer_root, s.rel);
        FS& f = fs[i];
        int fd = -1, rc = VMIG_OK;
        if (rf.action == kRbPatch) {
            fd = open_for_write(p, false, direct, &f.d_direct);
            if (fd < 0) return fail(VMIG_EIO, "open %s for writing: %s", p.c_str(), errno_str(errno).c_str());
            const LayerId& id = (*ids)[(size_t)rf.layer];
            rc = rollback_check_fd(fd, id, p);
            if (!rc && id.size != s.size) rc = cut_to_size(fd, s.size, p);
        } else {
            int old = -1;
            if (rf.action == kRbRebuild) {
                // read only when bytes are copied from it: an unreadable file with nothing to give is just replaced
                const int oflags = rf.n_runs ? O_RDONLY | O_NONBLOCK : O_PATH;
                old = open(p.c_str(), oflags | O_CLOEXEC | O_NOFOLLOW);
                if (old < 0) return fail(errno == ENOENT ? VMIG_ESRCCHANGED : VMIG_EIO, "open %s: %s", p.c_str(), errno_str(errno).c_str());
                rc = rebuild_guard.clear(old, (*ids)[(size_t)rf.layer], rf.n_runs != 0, p);
            } else {
                rc = clear_path(p, "a regular file");           // tar replaces what is there
            }
            if (!rc && (fd = open_for_write(p, true, direct, &f.d_direct)) < 0) rc = fail(VMIG_EIO, "create %s: %s", p.c_str(), errno_str(errno).c_str());
            for (uint64_t k = 0; !rc && k < rf.n_runs; k++) {
                const CopyRun& u = plan->runs[rf.first_run + k];
                rc = copy_range_at(old, u.off, fd, u.off, u.len, f.d_direct, false, p, cancel);
                if (!rc) b_copied += u.len;
            }
            if (old >= 0) close(old);
        }
        if (rc) { if (fd >= 0) close(fd); return rc; }
        if (f.d_direct) n_direct++;
        *out = fd;
        return VMIG_OK;
    }
    // O_DIRECT writes whole sectors: cut the padding of the last one
    int finish(uint32_t i, int fd) {
        const Entry& s = snap->files[plan->files[i].snap];
        const std::string p = pjoin(layer_root, s.rel);
        return close_written(fd, fs[i].d_direct && (s.size & (kSector - 1)) ? cut_to_size(fd, s.size, p) : VMIG_OK, p);
    }

    int read_block(const BlockRef& b, uint8_t* dst) override {
        const Entry& s = snap->files[plan->files[b.file].snap];
        int fd;
        int rc = src.get(b.file, snap_fd, s.rel, direct, [&](int*, const struct stat* st, bool) {
            if (!st || !S_ISREG(st->st_mode) || (uint64_t)st->st_size != s.size)
                return fail(VMIG_ESRCCHANGED, "snapshot file %s is not the walked file any more", s.rel.c_str());
            return VMIG_OK;
        }, &fd);
        if (rc) return rc;
        size_t got;
        rc = xfer_block(src.direct(b.file), true, b.len, &got, [&](size_t pos, size_t n) { return pread(fd, dst + pos, n, (off_t)(b.file_off + pos)); });
        if (rc < 0) return fail(VMIG_EIO, "pread %s: %s", s.rel.c_str(), errno_str(errno).c_str());
        if (rc) return fail(VMIG_ESRCCHANGED, "snapshot file %s shrank (wanted %u bytes at %llu, got %zu)", s.rel.c_str(), b.len, (unsigned long long)b.file_off, got);
        src.read_done(b.file);
        return VMIG_OK;
    }
    int write_block(const BlockRef& b, const uint8_t* src) override {
        FS& f = fs[b.file];
        int fd = f.dfd.load(std::memory_order_acquire);
        if (fd < 0) {
            // a file with few fetched siblings may have its blocks cut across lanes (run_blocks): the first writer to
            // get here makes it ready, the others wait for that and write into the same descriptor
            std::lock_guard<std::mutex> lk(f.open_mu);
            fd = f.dfd.load(std::memory_order_acquire);
            if (fd < 0) {
                const int rc = prepare(b.file, &fd);
                if (rc) return rc;
                f.dfd.store(fd, std::memory_order_release);
            }
        }
        size_t put;
        const int rc = xfer_block(f.d_direct, true, b.len, &put, [&](size_t pos, size_t n) { return pwrite(fd, src + pos, n, (off_t)(b.file_off + pos)); });
        const std::string& rel = snap->files[plan->files[b.file].snap].rel;
        if (rc < 0) return fail(VMIG_EIO, "pwrite %s/%s: %s", layer_root.c_str(), rel.c_str(), errno_str(errno).c_str());
        if (rc) return fail(VMIG_EIO, "pwrite %s/%s: wrote 0 bytes", layer_root.c_str(), rel.c_str());
        return VMIG_OK;
    }
    int block_done(const BlockRef& b, bool) override {
        if (fs[b.file].blocks_left.fetch_sub(1) != 1) return VMIG_OK;
        const int fd = fs[b.file].dfd.exchange(-1);
        return fd >= 0 ? finish(b.file, fd) : VMIG_OK;
    }
    ~RollbackIO() {                                 // what a failed pass left open (src closes its own)
        for (size_t i = 0; fs && i < plan->files.size(); i++) { const int d = fs[i].dfd.exchange(-1); if (d >= 0) close(d); }
    }

private:
    struct FS { std::atomic<int> dfd{-1}; std::atomic<uint64_t> blocks_left{0}; bool d_direct = false; std::mutex open_mu; };
    std::unique_ptr<FS[]> fs;
};

int rollback_body(CallScope& call, const char* layer_dir, const char* layer_table, const char* snap_dir, const char* snap_table,
                  const char* out_table, const vmig_opts& o, vmig_stats* stats_out, vmig_rollback_stats* rs_out)
{
    const std::atomic<int>* cancel = call.cancel();
    vmig_stats st; memset(&st, 0, sizeof st);
    const uint64_t t_begin = now_ns();
    BlockTable snap_tab, layer_tab;
    int rc = start_checks(call, o, {layer_dir, snap_dir}, {{snap_table, "snapshot", &snap_tab}, {layer_table, "layer", &layer_tab}});
    if (rc) return rc;
    const BlockTable* ltab = layer_table && *layer_table ? &layer_tab : nullptr;
    const std::string layer(layer_dir);

    // ---- the snapshot's walk, before the layer is touched
    Manifest snap;
    std::vector<uint64_t> snap_hashes;
    rc = walk_snapshot(call, snap_dir, snap_tab, o, &snap, &snap_hashes, &st);
    if (rc) return rc;

    // ---- what the snapshot does not list goes first, as in a pruning restore; the layer is walked as it then stands
    call.phase(VMIG_PHASE_PRUNE);
    rc = prune_extras(layer, snap, false, &st.pruned, cancel);
    if (rc) return rc;

    // ---- the layer's hashes (compare's read plan), each identity they speak for taken before the read and after it
    call.phase(VMIG_PHASE_DATA);
    LayerSide L;
    std::vector<LayerId> ids;
    rc = layer_plan(layer_dir, snap, ltab, o, cancel, &L, &st);
    if (!rc) rc = rollback_identify(layer, L.man, L.plan, ltab, &ids);
    if (!rc) rc = layer_hash_pass(call, o, snap, snap_hashes, ltab, &L, &st);
    if (!rc) rc = rollback_recheck_paths(layer, L.man, ids);
    if (rc) return rc;
    const uint64_t hashed_bytes = st.bytes_total, hashed_blocks = st.blocks_total;

    // ---- the plan: one action per snapshot file, the sparse fetch list, the copy runs
    uint64_t t0 = now_ns();
    RollbackPlan rp;
    rollback_plan(L.man, snap, snap_hashes, L.plan, L.hashes, ids, o.block_bytes, geteuid(), &rp);
    call.ctl->bytes_total.store(hashed_bytes + rp.bytes_fetched); call.ctl->blocks_total.store(hashed_blocks + rp.blocks_fetched);
    st.ns_plan += now_ns() - t0;

    // ---- the fetch pass: every block the layer lacks, checked by K1 against the snapshot's table before it is written
    t0 = now_ns();
    if (cancel->load()) return fail(VMIG_ECANCELED, "before the layer's directories were made");
    rc = make_dirs(layer, snap);
    if (rc) return rc;
    RollbackIO rio;
    rio.snap = &snap; rio.plan = &rp; rio.ids = &ids; rio.layer_root = layer; rio.direct = (o.flags & VMIG_F_DIRECT_IO) != 0;
    rio.block_bytes = o.block_bytes; rio.cancel = cancel;
    rio.init();
    VersionRoots sroot(1);
    if (!rp.fetch.empty() && (rc = sroot.open(0, snap_dir))) return rc;
    rio.snap_fd = sroot.fds[0];
    for (uint32_t i = 0; i < rp.files.size(); i++) {        // files that take no block from the snapshot
        const RollbackFile& rf = rp.files[i];
        if (rf.n_fetch || rf.action == kRbKeep) continue;
        if (cancel->load()) return fail(VMIG_ECANCELED, "before %s was made ready", snap.files[rf.snap].rel.c_str());
        int fd;
        rc = rio.prepare(i, &fd);
        if (!rc) rc = rio.finish(i, fd);
        if (rc) return rc;
    }
    std::vector<uint64_t> fetched(snap.n_blocks, 0);
    BlockExpect fetch_expect; fetch_expect.hashes = snap_hashes.data();
    rc = run_blocks(rp.fetch, &rio, false, false, o, fetched.data(), &st, call.ctl, false, &fetch_expect);
    st.ns_data += now_ns() - t0;
    if (rc) return rc;

    // ---- metadata: each regular file's where it differs, then the restore's replay; the layer now holds the table's bytes
    t0 = now_ns();
    call.phase(VMIG_PHASE_META);
    DstTree tree;
    tree.m = &snap; tree.dst_root = layer; tree.pol = default_meta_policy(o.flags); tree.block_bytes = o.block_bytes;
    tree.direct = (o.flags & VMIG_F_DIRECT_IO) != 0;
    tree.ids.resize(snap.files.size());
    for (size_t i = 0; i < rp.files.size(); i++) {
        if (i % kMetaCheckEvery == 0 && cancel->load()) return fail(VMIG_ECANCELED, "before the metadata of %s", snap.files[rp.files[i].snap].rel.c_str());
        const Entry& e = snap.files[rp.files[i].snap];
        const std::string p = pjoin(layer, e.rel);
        const int fd = open(p.c_str(), O_RDONLY | O_CLOEXEC | O_NOFOLLOW | O_NONBLOCK);
        if (fd < 0 && errno != EACCES) return fail(VMIG_EIO, "open %s: %s", p.c_str(), errno_str(errno).c_str());
        if (fd < 0) rc = apply_file_meta(-1, p, e, tree.pol);        // an ordinary user's unreadable file: by path
        else rc = file_meta_matches(fd, e, tree.pol) ? VMIG_OK : apply_file_meta(fd, p, e, tree.pol);     // a kept file's ctime stays
        if (fd >= 0) close(fd);
        if (rc) return rc;
    }
    std::vector<uint64_t> hashes(snap_hashes);
    rc = meta_pass(call, tree, snap_hashes, &hashes, &st, 0, false);
    if (rc) return rc;
    st.ns_meta = now_ns() - t0;

    vmig_opts vo = o;
    vo.flags |= VMIG_F_PRUNE;                        // the verify's entry-set check is the pruning restore's
    if (o.flags & VMIG_F_VERIFY) {
        call.phase(VMIG_PHASE_VERIFY);
        rc = verify_pass(call, vo, tree, hashes, &st, nullptr, data_files(snap));
        if (rc) return rc;
    }

    // ---- the table: the snapshot's hashes, and each layer file's identity as the call leaves it
    t0 = now_ns();
    call.phase(VMIG_PHASE_TABLE);
    std::vector<uint32_t> own;
    for (uint32_t f = 0; f < snap.files.size(); f++) if (snap.files[f].hardlink_of < 0) own.push_back(f);
    rc = record_ids(tree, own);
    if (!rc) rc = write_table(tree, out_table, hashes, cancel);
    if (rc) return rc;
    st.ns_table = now_ns() - t0;

    st.files_direct += rio.src.n_direct.load() + rio.n_direct.load();
    st.bytes_total = hashed_bytes + rp.bytes_fetched; st.blocks_total = hashed_blocks + rp.blocks_fetched;
    st.files = snap.files.size(); st.dirs = snap.dirs.size();
    st.ns_total = now_ns() - t_begin;
    if (stats_out) *stats_out = st;
    if (rs_out) {
        vmig_rollback_stats rs; memset(&rs, 0, sizeof rs);
        rs.files_kept = rp.files_kept; rs.files_patched = rp.files_patched; rs.files_rebuilt = rp.files_rebuilt;
        rs.files_created = rp.files_created; rs.blocks_fetched = rp.blocks_fetched; rs.bytes_fetched = rp.bytes_fetched;
        rs.files_trusted = L.plan.files_trusted; rs.files_read = L.plan.inodes.size(); rs.bytes_read = L.plan.bytes_read;
        rs.bytes_copied = rio.b_copied.load();
        *rs_out = rs;
    }
    return VMIG_OK;
}

// The layer calls after their refusals: the source's walk, then the tree passes with the source's table
int layer_tree_passes(CallScope& call, TreeCall& c, const vmig_opts& o, vmig_stats& st, uint64_t t_begin, vmig_stats* stats_out)
{
    Manifest man;
    const uint64_t t0 = now_ns();
    call.phase(VMIG_PHASE_WALK);
    const int rc = walk_tree(c.src, o.block_bytes, (o.flags & VMIG_F_SKIP_HIDDEN_TOPDIRS) != 0, &man, call.cancel());
    if (rc) return rc;
    st.ns_walk = now_ns() - t0;
    c.man = &man;
    return tree_passes(call, c, o, st, t_begin, stats_out);
}

// vmig_snapshot_layer: the snapshot's passes with the layer table
int snapshot_layer_body(CallScope& call, const char* layer_dir, const char* layer_table, const char* dst_dir, const char* base_dir,
                        const char* base_table, const char* out_table, const vmig_opts& o, vmig_stats* stats_out,
                        vmig_layer_snapshot_stats* ls_out)
{
    vmig_stats st; memset(&st, 0, sizeof st);
    const uint64_t t_begin = now_ns();
    BlockTable base, layer;
    const int rc = start_checks(call, o, {layer_dir, dst_dir, base_dir}, {{base_table, "base", &base}, {layer_table, "layer", &layer}});
    if (rc) return rc;
    TreeCall c;
    c.src = layer_dir; c.dst = dst_dir; c.base = &base; c.base_dir = base_dir; c.layer = &layer;
    c.out_table = out_table; c.refresh_ids = true; c.layer_snap_out = ls_out;
    return layer_tree_passes(call, c, o, st, t_begin, stats_out);
}

// vmig_migrate_layer: the migration's passes with the source's table
int migrate_layer_body(CallScope& call, const char* src_dir, const char* src_table, const char* dst_dir, const char* prior_table,
                       const char* out_table, const char* src_out_table, const vmig_opts& o, vmig_stats* stats_out,
                       vmig_layer_migrate_stats* lm_out)
{
    vmig_stats st; memset(&st, 0, sizeof st);
    const uint64_t t_begin = now_ns();
    BlockTable src_tab, prior;
    src_tab.block_bytes = o.block_bytes;             // no src_table: an empty table, which trusts nothing
    const int rc = start_checks(call, o, {src_dir, dst_dir}, {{src_table, "source", &src_tab}, {prior_table, "prior", &prior}});
    if (rc) return rc;
    TreeCall c;
    c.src = src_dir; c.dst = dst_dir; c.layer = &src_tab; c.prior = prior_table && *prior_table ? &prior : nullptr;
    c.out_table = out_table; c.src_out_table = src_out_table; c.layer_mig_out = lm_out;
    return layer_tree_passes(call, c, o, st, t_begin, stats_out);
}

}  // namespace

// =============================================================================================
extern "C" {

int vmig_init(uint32_t gpu_mask) { return ctx_init(gpu_mask); }
void vmig_shutdown(void)
{
    {
        // calls in flight hold pipes and cuFile handles: cancel them and wait until they have returned
        std::unique_lock<std::mutex> lk(g_calls_mu);
        while (!g_calls.empty()) {
            for (CallCtl* c : g_calls) c->cancel();
            g_calls_cv.wait(lk);
        }
    }
    ctx_shutdown(); cufile_shutdown();
}

int vmig_ctl_open(uint32_t* id)
{
    if (!id) return fail(VMIG_EINVAL, "null id pointer");
    std::lock_guard<std::mutex> lk(g_ctl_mu);
    if (g_ctl_next == 0) return fail(VMIG_ENOMEM, "control ids exhausted (they are never reused within a process)");
    *id = g_ctl_next++;
    g_ctls.emplace(*id, std::make_shared<CallCtl>());
    return VMIG_OK;
}
int vmig_ctl_cancel(uint32_t id)
{
    std::shared_ptr<CallCtl> c;
    {
        std::lock_guard<std::mutex> lk(g_ctl_mu);
        auto it = g_ctls.find(id);
        if (it == g_ctls.end()) return fail(VMIG_EINVAL, "control %u is not open", id);
        c = it->second;
    }
    c->cancel();
    return VMIG_OK;
}
int vmig_ctl_progress(uint32_t id, vmig_progress* out)
{
    if (!out) return fail(VMIG_EINVAL, "null progress pointer");
    std::shared_ptr<CallCtl> c;
    {
        std::lock_guard<std::mutex> lk(g_ctl_mu);
        auto it = g_ctls.find(id);
        if (it == g_ctls.end()) return fail(VMIG_EINVAL, "control %u is not open", id);
        c = it->second;
    }
    memset(out, 0, sizeof *out);
    out->phase = c->phase.load(); out->running = c->running.load();
    const auto r = std::memory_order_relaxed;
    out->bytes_total = c->bytes_total.load(r); out->blocks_total = c->blocks_total.load(r);
    out->bytes_hashed = c->bytes_hashed.load(r); out->blocks_hashed = c->blocks_hashed.load(r);
    out->bytes_written = c->bytes_written.load(r); out->bytes_verified = c->bytes_verified.load(r);
    return VMIG_OK;
}
int vmig_ctl_close(uint32_t id)
{
    std::lock_guard<std::mutex> lk(g_ctl_mu);
    auto it = g_ctls.find(id);
    if (it == g_ctls.end()) return fail(VMIG_EINVAL, "control %u is not open", id);
    if (it->second->running.load()) return fail(VMIG_EINVAL, "control %u is attached to a call in flight", id);
    g_ctls.erase(it);
    return VMIG_OK;
}
int vmig_device_count(void) { return ctx_device_count(); }
const char* vmig_last_error(void) { return last_error_cstr(); }
const char* vmig_version(void) { return "libvmig 0.2 (abi 2, sm_90a)"; }
const char* vmig_strerror(int code)
{
    switch (code) {
    case VMIG_OK: return "ok";
    case VMIG_EINVAL: return "invalid argument";
    case VMIG_ENOGPU: return "no usable sm_90 GPU (no CPU fallback)";
    case VMIG_ECUDA: return "CUDA error";
    case VMIG_EIO: return "I/O error";
    case VMIG_ENOMEM: return "out of memory";
    case VMIG_ETABLE: return "bad block table";
    case VMIG_EFAULT: return "injected fault";
    case VMIG_ENOTDIR: return "not a directory";
    case VMIG_ESRCCHANGED: return "source changed during migration";
    case VMIG_EVERIFY: return "destination does not verify against the source";
    case VMIG_ECORRUPT: return "source tree does not match its block table";
    case VMIG_ECANCELED: return "call cancelled";
    default: return "unknown vmig error";
    }
}

int vmig_migrate_tree(const char* src_dir, const char* dst_dir, const char* prior_table, const char* out_table,
                      const vmig_opts* opts, vmig_stats* stats)
{
    TreeCall c;
    c.out_table = out_table;
    return migrate_tree_impl(c, src_dir, dst_dir, prior_table, nullptr, nullptr, opts, stats);
}
int vmig_restore_tree(const char* snap_dir, const char* snap_table, const char* dst_dir, const char* prior_table,
                      const char* out_table, const vmig_opts* opts, vmig_stats* stats)
{
    if (!snap_table || !*snap_table) return fail(VMIG_EINVAL, "snap_table is NULL/empty: a snapshot is only restored against its block table");
    if (opts && (opts->flags & VMIG_F_MOVE_SRC)) return fail(VMIG_EINVAL, "VMIG_F_MOVE_SRC: a restore never consumes the snapshot");
    TreeCall c;
    c.out_table = out_table;
    return migrate_tree_impl(c, snap_dir, dst_dir, prior_table, snap_table, nullptr, opts, stats);
}
int vmig_restore_paths(const char* snap_dir, const char* snap_table, const char* dst_dir, uint32_t n_paths,
                       const char* const* paths, const char* prior_table, const vmig_opts* opts, vmig_stats* stats)
{
    std::vector<std::string> sorted;
    int rc = select_check_paths(n_paths, paths, &sorted);
    if (rc) return rc;
    if (!snap_table || !*snap_table) return fail(VMIG_EINVAL, "snap_table is NULL/empty: a snapshot is only restored against its block table");
    if (!snap_dir || !*snap_dir) return fail(VMIG_EINVAL, "snap_dir is NULL/empty");
    if (!dst_dir || !*dst_dir) return fail(VMIG_EINVAL, "dst_dir is NULL/empty");
    const vmig_opts o = norm_opts(opts);                     // VMIG_CUFILE=1 in the environment is refused too
    if (o.flags & VMIG_F_MOVE_SRC) return fail(VMIG_EINVAL, "VMIG_F_MOVE_SRC: a restore never consumes the snapshot");
    if (o.flags & VMIG_F_HASH_ONLY) return fail(VMIG_EINVAL, "VMIG_F_HASH_ONLY: a partial restore writes its destination (vmig_scrub_store checks a version)");
    if (o.flags & VMIG_F_CUFILE) return fail(VMIG_EINVAL, "VMIG_F_CUFILE: not supported for a partial restore");
    rc = check_block_bytes(o);
    if (!rc) rc = check_apart("snap_dir", real_path(snap_dir), "dst_dir", real_path(dst_dir));
    if (rc) return rc;
    return in_call(o.ctl, [&](CallScope& call) { return restore_paths_body(call, snap_dir, snap_table, dst_dir, sorted, prior_table, o, stats); });
}
int vmig_snapshot_tree(const char* src_dir, const char* dst_dir, const char* base_dir, const char* base_table,
                       const char* out_table, const vmig_opts* opts, vmig_stats* stats, vmig_snapshot_stats* snap_stats)
{
    const bool has_dir = base_dir && *base_dir, has_table = base_table && *base_table;
    if (has_dir != has_table) return fail(VMIG_EINVAL, "base_dir and base_table go together: one of them is NULL/empty");
    if (!out_table || !*out_table) return fail(VMIG_EINVAL, "out_table is NULL/empty: a snapshot is only restored against its block table");
    const uint32_t flags = norm_opts(opts).flags;          // VMIG_CUFILE=1 in the environment is refused too
    if (flags & VMIG_F_MOVE_SRC) return fail(VMIG_EINVAL, "VMIG_F_MOVE_SRC: a snapshot never consumes its source");
    if (flags & VMIG_F_HASH_ONLY) return fail(VMIG_EINVAL, "VMIG_F_HASH_ONLY: a snapshot writes its destination");
    if (flags & VMIG_F_CUFILE) return fail(VMIG_EINVAL, "VMIG_F_CUFILE: not supported for snapshots (a backfilled file would mix cuFile and buffered writes)");
    if (!dst_dir || !*dst_dir) return fail(VMIG_EINVAL, "dst_dir is NULL/empty");
    if (has_dir) { const int rc = check_snapshot_paths(dst_dir, base_dir); if (rc) return rc; }
    if (snap_stats) memset(snap_stats, 0, sizeof *snap_stats);
    TreeCall c;                                            // no base: a full snapshot
    c.out_table = out_table; c.base_dir = has_dir ? base_dir : ""; c.refresh_ids = true; c.snap_out = snap_stats;
    return migrate_tree_impl(c, src_dir, dst_dir, nullptr, nullptr, has_table ? base_table : nullptr, opts, stats);
}
int vmig_snapshot_layer(const char* layer_dir, const char* layer_table, const char* dst_dir, const char* base_dir,
                        const char* base_table, const char* out_table, const vmig_opts* opts, vmig_stats* stats,
                        vmig_layer_snapshot_stats* ls_stats)
{
    const char* const names[] = {"layer_dir", "layer_table", "dst_dir", "base_dir", "base_table", "out_table"};
    const char* const paths[] = {layer_dir, layer_table, dst_dir, base_dir, base_table, out_table};
    for (int i = 0; i < 6; i++)
        if (!paths[i] || !*paths[i])
            return fail(VMIG_EINVAL, "%s is NULL/empty: a layer snapshot takes the layer's table and a base (without them vmig_snapshot_tree is the call)", names[i]);
    const vmig_opts o = norm_opts(opts);                     // VMIG_CUFILE=1 in the environment is refused too
    const uint32_t allowed = VMIG_F_VERIFY | VMIG_F_PRUNE | VMIG_F_DIRECT_IO | VMIG_F_MTIME_NS | VMIG_F_NO_METADATA | VMIG_F_SKIP_HIDDEN_TOPDIRS;
    if (o.flags & ~allowed)
        return fail(VMIG_EINVAL, "flags 0x%x: a layer snapshot takes only VMIG_F_VERIFY, VMIG_F_PRUNE, VMIG_F_DIRECT_IO, VMIG_F_MTIME_NS, "
                    "VMIG_F_NO_METADATA and VMIG_F_SKIP_HIDDEN_TOPDIRS", o.flags & ~allowed);
    int rc = check_block_bytes(o);
    const std::string rd = real_path(dst_dir), rb = real_path(base_dir), rl = real_path(layer_dir);
    if (!rc) rc = check_apart("dst_dir", rd, "base_dir", rb);
    if (!rc) rc = check_apart("dst_dir", rd, "layer_dir", rl);
    if (!rc) rc = check_apart("base_dir", rb, "layer_dir", rl);
    if (rc) return rc;
    std::string ro, rt;
    rc = real_parent_path(out_table, &ro);
    if (!rc) rc = real_parent_path(base_table, &rt);
    if (rc) return rc;
    if (ro == rt || (!rb.empty() && path_inside(ro, rb)) || (!rl.empty() && path_inside(ro, rl)))
        return fail(VMIG_EINVAL, "out_table %s is the base's table or lies inside base_dir or layer_dir: neither is ever written", out_table);
    if (ls_stats) memset(ls_stats, 0, sizeof *ls_stats);
    return in_call(o.ctl, [&](CallScope& call) {
        return snapshot_layer_body(call, layer_dir, layer_table, dst_dir, base_dir, base_table, out_table, o, stats, ls_stats);
    });
}
int vmig_migrate_layer(const char* src_dir, const char* src_table, const char* dst_dir, const char* prior_table,
                       const char* out_table, const char* src_out_table, const vmig_opts* opts, vmig_stats* stats,
                       vmig_layer_migrate_stats* lm_stats)
{
    if (!src_dir || !*src_dir) return fail(VMIG_EINVAL, "src_dir is NULL/empty");
    if (!dst_dir || !*dst_dir) return fail(VMIG_EINVAL, "dst_dir is NULL/empty");
    const vmig_opts o = norm_opts(opts);                     // VMIG_CUFILE=1 in the environment is refused too
    const uint32_t allowed = VMIG_F_VERIFY | VMIG_F_PRUNE | VMIG_F_DIRECT_IO | VMIG_F_MTIME_NS | VMIG_F_NO_METADATA | VMIG_F_SKIP_HIDDEN_TOPDIRS;
    if (o.flags & ~allowed)
        return fail(VMIG_EINVAL, "flags 0x%x: a layer migration takes only VMIG_F_VERIFY, VMIG_F_PRUNE, VMIG_F_DIRECT_IO, VMIG_F_MTIME_NS, "
                    "VMIG_F_NO_METADATA and VMIG_F_SKIP_HIDDEN_TOPDIRS", o.flags & ~allowed);
    int rc = check_block_bytes(o);
    const std::string rs = real_path(src_dir), rd = real_path(dst_dir);
    if (!rc) rc = check_apart("src_dir", rs, "dst_dir", rd);
    if (rc) return rc;
    const bool has_out = out_table && *out_table, has_src_out = src_out_table && *src_out_table;
    std::string ro, rso;
    if (has_out && (rc = real_parent_path(out_table, &ro))) return rc;
    if (has_src_out && (rc = real_parent_path(src_out_table, &rso))) return rc;
    if (has_out && has_src_out && ro == rso)
        return fail(VMIG_EINVAL, "out_table and src_out_table are the same file %s: one table records the destination, the other the source", ro.c_str());
    if (!rs.empty() && ((has_out && path_inside(ro, rs)) || (has_src_out && path_inside(rso, rs))))
        return fail(VMIG_EINVAL, "out_table or src_out_table lies inside src_dir %s: the source is never written", rs.c_str());
    if (has_src_out && !rd.empty() && path_inside(rso, rd))
        return fail(VMIG_EINVAL, "src_out_table %s lies inside dst_dir %s: it would be part of the tree it describes the source of", rso.c_str(), rd.c_str());
    if (lm_stats) memset(lm_stats, 0, sizeof *lm_stats);
    return in_call(o.ctl, [&](CallScope& call) {
        return migrate_layer_body(call, src_dir, src_table, dst_dir, prior_table, out_table, src_out_table, o, stats, lm_stats);
    });
}
int vmig_scrub_store(uint32_t n, const char* const* snap_dirs, const char* const* snap_tables, const char* report_path,
                     int32_t* verdicts, const vmig_opts* opts, vmig_stats* stats, vmig_scrub_stats* scrub_stats)
{
    if (n == 0) return fail(VMIG_EINVAL, "n == 0: no version to scrub");
    if (!snap_dirs || !snap_tables) return fail(VMIG_EINVAL, "snap_dirs / snap_tables is NULL");
    for (uint32_t i = 0; i < n; i++)
        if (!snap_dirs[i] || !*snap_dirs[i] || !snap_tables[i] || !*snap_tables[i]) return fail(VMIG_EINVAL, "version %u: snap_dir or snap_table is NULL/empty", i);
    const vmig_opts o = norm_opts(opts);                     // VMIG_CUFILE=1 in the environment is refused too
    const uint32_t allowed = VMIG_F_DIRECT_IO | VMIG_F_SKIP_HIDDEN_TOPDIRS;
    if (o.flags & ~allowed) return fail(VMIG_EINVAL, "flags 0x%x: a scrub takes only VMIG_F_DIRECT_IO and VMIG_F_SKIP_HIDDEN_TOPDIRS", o.flags & ~allowed);
    int rc = check_block_bytes(o);
    if (rc) return rc;
    return in_call(o.ctl, [&](CallScope& call) { return scrub_body(call, n, snap_dirs, snap_tables, report_path, verdicts, o, stats, scrub_stats); });
}
int vmig_retire_versions(uint32_t n_retire, const char* const* retire_dirs, const char* const* retire_tables,
                         uint32_t n_keep, const char* const* keep_dirs, const char* const* keep_tables,
                         const vmig_opts* opts, vmig_stats* stats, vmig_retire_stats* retire_stats)
{
    if (n_retire + (uint64_t)n_keep == 0) return fail(VMIG_EINVAL, "n_retire + n_keep == 0: no version to retire or keep");
    if ((n_retire && (!retire_dirs || !retire_tables)) || (n_keep && (!keep_dirs || !keep_tables)))
        return fail(VMIG_EINVAL, "retire_dirs / retire_tables / keep_dirs / keep_tables is NULL");
    for (uint32_t i = 0; i < n_retire; i++)
        if (!retire_dirs[i] || !*retire_dirs[i] || !retire_tables[i] || !*retire_tables[i]) return fail(VMIG_EINVAL, "retired version %u: dir or table is NULL/empty", i);
    for (uint32_t i = 0; i < n_keep; i++)
        if (!keep_dirs[i] || !*keep_dirs[i] || !keep_tables[i] || !*keep_tables[i]) return fail(VMIG_EINVAL, "kept version %u: dir or table is NULL/empty", i);
    const vmig_opts o = norm_opts(opts);                     // VMIG_CUFILE=1 in the environment is refused too
    const uint32_t allowed = VMIG_F_DIRECT_IO | VMIG_F_SKIP_HIDDEN_TOPDIRS;
    if (o.flags & ~allowed) return fail(VMIG_EINVAL, "flags 0x%x: a retire takes only VMIG_F_DIRECT_IO and VMIG_F_SKIP_HIDDEN_TOPDIRS", o.flags & ~allowed);
    int rc = check_block_bytes(o);
    if (rc) return rc;
    RetireArgs a;
    rc = check_retire_args(n_retire, retire_dirs, retire_tables, n_keep, keep_dirs, keep_tables, &a);
    if (rc) return rc;
    return in_call(o.ctl, [&](CallScope& call) { return retire_body(call, a, o, stats, retire_stats); });
}
int vmig_compare_snapshot(const char* layer_dir, const char* layer_table, const char* snap_dir, const char* snap_table,
                          const char* report_path, const vmig_opts* opts, vmig_stats* stats, vmig_compare_stats* cmp_stats)
{
    if (!layer_dir || !*layer_dir) return fail(VMIG_EINVAL, "layer_dir is NULL/empty");
    if (!snap_dir || !*snap_dir) return fail(VMIG_EINVAL, "snap_dir is NULL/empty");
    if (!snap_table || !*snap_table) return fail(VMIG_EINVAL, "snap_table is NULL/empty: a layer is only compared with a snapshot through its block table");
    const vmig_opts o = norm_opts(opts);                     // VMIG_CUFILE=1 in the environment is refused too
    const uint32_t allowed = VMIG_F_DIRECT_IO | VMIG_F_SKIP_HIDDEN_TOPDIRS | VMIG_F_MTIME_NS | VMIG_F_NO_METADATA;
    if (o.flags & ~allowed)
        return fail(VMIG_EINVAL, "flags 0x%x: a compare takes only VMIG_F_DIRECT_IO, VMIG_F_SKIP_HIDDEN_TOPDIRS, VMIG_F_MTIME_NS and VMIG_F_NO_METADATA", o.flags & ~allowed);
    int rc = check_block_bytes(o);
    if (rc) return rc;
    return in_call(o.ctl, [&](CallScope& call) {
        return compare_body(call, layer_dir, layer_table, snap_dir, snap_table, report_path, o, stats, cmp_stats);
    });
}
int vmig_rollback_layer(const char* layer_dir, const char* layer_table, const char* snap_dir, const char* snap_table,
                        const char* out_table, const vmig_opts* opts, vmig_stats* stats, vmig_rollback_stats* rb_stats)
{
    if (!layer_dir || !*layer_dir) return fail(VMIG_EINVAL, "layer_dir is NULL/empty");
    if (!snap_dir || !*snap_dir) return fail(VMIG_EINVAL, "snap_dir is NULL/empty");
    if (!snap_table || !*snap_table) return fail(VMIG_EINVAL, "snap_table is NULL/empty: a layer is only rolled back to a snapshot through its block table");
    const vmig_opts o = norm_opts(opts);                     // VMIG_CUFILE=1 in the environment is refused too
    const uint32_t allowed = VMIG_F_DIRECT_IO | VMIG_F_SKIP_HIDDEN_TOPDIRS | VMIG_F_MTIME_NS | VMIG_F_NO_METADATA | VMIG_F_VERIFY | VMIG_F_PRUNE;
    if (o.flags & ~allowed)
        return fail(VMIG_EINVAL, "flags 0x%x: a rollback takes only VMIG_F_DIRECT_IO, VMIG_F_SKIP_HIDDEN_TOPDIRS, VMIG_F_MTIME_NS, "
                    "VMIG_F_NO_METADATA, VMIG_F_VERIFY and VMIG_F_PRUNE", o.flags & ~allowed);
    int rc = check_block_bytes(o);
    const std::string rs = real_path(snap_dir);
    if (!rc) rc = check_apart("layer_dir", real_path(layer_dir), "snap_dir", rs);
    if (rc) return rc;
    if (out_table && *out_table) {
        std::string ro, rt;
        rc = real_parent_path(out_table, &ro);
        if (!rc) rc = real_parent_path(snap_table, &rt);
        if (rc) return rc;
        if (ro == rt || (!rs.empty() && path_inside(ro, rs)))
            return fail(VMIG_EINVAL, "out_table %s is the snapshot's table or lies inside snap_dir: the store is never written", out_table);
    }
    return in_call(o.ctl, [&](CallScope& call) {
        return rollback_body(call, layer_dir, layer_table, snap_dir, snap_table, out_table, o, stats, rb_stats);
    });
}
int vmig_copy_dir(const char* src_dir, const char* dst_dir) { return migrate_tree_impl({}, src_dir, dst_dir, nullptr, nullptr, nullptr, nullptr, nullptr); }
int vmig_move_dir(const char* src_dir, const char* dst_dir)
{
    // a move destroys the only other copy: the destination is re-read through the GPU and must hash like the
    // source (VMIG_F_VERIFY) and is flushed (syncfs) before anything is unlinked
    vmig_opts o; memset(&o, 0, sizeof o); o.flags = VMIG_F_MOVE_SRC | VMIG_F_VERIFY;
    return migrate_tree_impl({}, src_dir, dst_dir, nullptr, nullptr, nullptr, &o, nullptr);
}

int vmig_thread_plan(uint32_t lanes, uint32_t n_gpus, uint32_t flags, int has_prior, uint32_t* readers, uint32_t* writers)
{
    if (!readers || !writers || !lanes || !n_gpus) return fail(VMIG_EINVAL, "bad thread-plan arguments");
    return io_threads_default(readers, writers, 0, lanes, std::min<size_t>(n_gpus, lanes), false, has_prior != 0, (flags & VMIG_F_HASH_ONLY) != 0);
}

int vmig_host_alloc(void** p, uint64_t nbytes)
{
    if (!p) return fail(VMIG_EINVAL, "null out pointer");
    std::vector<DeviceInfo> devs; int rc = ctx_select(0, &devs); if (rc) return rc;
    cudaError_t e = cudaHostAlloc(p, nbytes ? nbytes : 1, cudaHostAllocPortable);
    if (e != cudaSuccess) { cudaGetLastError(); return fail(VMIG_ENOMEM, "cudaHostAlloc(%llu): %s", (unsigned long long)nbytes, cudaGetErrorString(e)); }
    return VMIG_OK;
}
void vmig_host_free(void* p) { if (p) cudaFreeHost(p); }

int vmig_migrate_buffer(const void* src, void* dst, uint64_t nbytes, const uint64_t* prior_hashes, const uint8_t* prior_valid,
                        uint64_t* out_hashes, const vmig_opts* opts, vmig_stats* stats)
{
    vmig_stats st; memset(&st, 0, sizeof st);
    const uint64_t t0 = now_ns();
    vmig_opts o = norm_opts(opts);
    const bool hash_only = (o.flags & VMIG_F_HASH_ONLY) != 0;
    if (!src || (!dst && !hash_only)) return fail(VMIG_EINVAL, "null buffer");
    int rc = check_block_bytes(o); if (rc) return rc;
    CallScope call;
    rc = call.attach(o.ctl); if (rc) return rc;
    if (call.cancel()->load()) return call.finish(fail(VMIG_ECANCELED, "the control was cancelled before the call started"));
    std::vector<DeviceInfo> devs; rc = ctx_select(o.gpu_mask, &devs); if (rc) return rc;
    const uint64_t nb = (nbytes + o.block_bytes - 1) / o.block_bytes;
    call.ctl->bytes_total.store(nbytes); call.ctl->blocks_total.store(nb);
    call.phase(VMIG_PHASE_DATA);
    std::vector<BlockRef> blocks(nb);
    const bool has_prior = prior_hashes != nullptr && prior_valid != nullptr;
    for (uint64_t i = 0; i < nb; i++) {
        BlockRef& b = blocks[i];
        b.file = 0; b.file_off = i * o.block_bytes; b.len = (uint32_t)std::min<uint64_t>(o.block_bytes, nbytes - b.file_off);
        b.table_idx = i; b.prior_hash = has_prior ? prior_hashes[i] : 0; b.prior_valid = has_prior ? prior_valid[i] : 0;
    }
    MemIO io; io.src = (const uint8_t*)src; io.dst = (uint8_t*)dst;
    io.src_pinned = is_pinned(src); io.dst_pinned = !hash_only && is_pinned(dst);
    std::vector<uint64_t> hashes(nb);
    rc = run_blocks(blocks, &io, has_prior, hash_only, o, hashes.data(), &st, call.ctl, false);
    if (rc) return call.finish(rc);
    if (out_hashes && nb) memcpy(out_hashes, hashes.data(), nb * 8);
    st.bytes_total = nbytes; st.blocks_total = nb; st.ns_total = st.ns_data = now_ns() - t0;
    if (stats) *stats = st;
    return call.finish(VMIG_OK);
}

int vmig_hash_blocks(int gpu, const void* host_buf, const uint64_t* offs, const uint32_t* lens, uint64_t n,
                     uint64_t* out_hashes, double* kernel_ms)
{
    if (n && (!offs || !lens || !out_hashes)) return fail(VMIG_EINVAL, "null array");
    if (gpu < 0 || gpu > 31) return fail(VMIG_EINVAL, "bad gpu index %d", gpu);
    vmig_opts o; memset(&o, 0, sizeof o); o.gpu_mask = 1u << gpu; o.block_bytes = 4u << 20; o.flags = VMIG_F_HASH_ONLY;
    std::vector<DeviceInfo> devs; int rc = ctx_select(o.gpu_mask, &devs); if (rc) return rc;
    std::vector<BlockRef> blocks(n);
    for (uint64_t i = 0; i < n; i++) {
        if (lens[i] && !host_buf) return fail(VMIG_EINVAL, "null host_buf");
        blocks[i].file = 0; blocks[i].file_off = offs[i]; blocks[i].len = lens[i]; blocks[i].table_idx = i;
        blocks[i].prior_hash = 0; blocks[i].prior_valid = 0;
    }
    MemIO io; io.src = (const uint8_t*)host_buf; io.dst = nullptr;   // staged: arbitrary offsets become 512-B aligned in HBM
    vmig_stats st; memset(&st, 0, sizeof st);
    CallScope call;                  // not cancellable by the caller; vmig_shutdown still waits for it
    rc = call.attach(0); if (rc) return rc;
    call.phase(VMIG_PHASE_DATA);
    rc = call.finish(run_blocks(blocks, &io, false, true, o, out_hashes, &st, call.ctl, false));
    if (kernel_ms) *kernel_ms = st.ms_kernel;
    return rc;
}

// ---------------------------------------------------------------------------------------------
// host<->HBM link probe
#define CU_API(call) do { cudaError_t e__ = (call); if (e__ != cudaSuccess) { cudaGetLastError(); return fail(e__ == cudaErrorMemoryAllocation ? VMIG_ENOMEM : VMIG_ECUDA, "%s: %s", #call, cudaGetErrorString(e__)); } } while (0)

static int link_probe_here(int gpu, uint64_t bytes, double* gbs)
{
    const size_t piece = 32u << 20, ring = 8;           // 8 x 32 MiB per direction: larger than any host cache
    CU_API(cudaSetDevice(gpu));
    uint8_t *h_a = nullptr, *h_b = nullptr, *d_a = nullptr, *d_b = nullptr;
    cudaStream_t s0 = nullptr, s1 = nullptr; cudaEvent_t e[4] = {nullptr, nullptr, nullptr, nullptr};
    auto cleanup = [&] {
        if (h_a) cudaFreeHost(h_a); if (h_b) cudaFreeHost(h_b); if (d_a) cudaFree(d_a); if (d_b) cudaFree(d_b);
        if (s0) cudaStreamDestroy(s0); if (s1) cudaStreamDestroy(s1);
        for (auto& x : e) if (x) cudaEventDestroy(x);
    };
    auto run = [&]() -> int {
        CU_API(cudaHostAlloc((void**)&h_a, piece * ring, cudaHostAllocPortable)); memset(h_a, 1, piece * ring);
        CU_API(cudaHostAlloc((void**)&h_b, piece * ring, cudaHostAllocPortable)); memset(h_b, 2, piece * ring);
        CU_API(cudaMalloc((void**)&d_a, piece * ring)); CU_API(cudaMalloc((void**)&d_b, piece * ring));
        CU_API(cudaMemset(d_b, 3, piece * ring));
        CU_API(cudaStreamCreateWithFlags(&s0, cudaStreamNonBlocking)); CU_API(cudaStreamCreateWithFlags(&s1, cudaStreamNonBlocking));
        for (auto& x : e) CU_API(cudaEventCreate(&x));
        const uint64_t n = std::max<uint64_t>(1, bytes / piece);
        auto pass = [&](bool up, bool down, double* up_gbs, double* down_gbs) -> int {
            for (int rep = 0; rep < 2; rep++) {          // rep 0 warms up
                if (up) CU_API(cudaEventRecord(e[0], s0));
                if (down) CU_API(cudaEventRecord(e[2], s1));
                for (uint64_t i = 0; i < n; i++) {
                    const size_t o = (size_t)(i % ring) * piece;
                    if (up) CU_API(cudaMemcpyAsync(d_a + o, h_a + o, piece, cudaMemcpyHostToDevice, s0));
                    if (down) CU_API(cudaMemcpyAsync(h_b + o, d_b + o, piece, cudaMemcpyDeviceToHost, s1));
                }
                if (up) CU_API(cudaEventRecord(e[1], s0));
                if (down) CU_API(cudaEventRecord(e[3], s1));
                CU_API(cudaStreamSynchronize(s0)); CU_API(cudaStreamSynchronize(s1));
            }
            float ms = 0;
            if (up) { CU_API(cudaEventElapsedTime(&ms, e[0], e[1])); *up_gbs = (double)(n * piece) / (ms * 1e-3) / 1e9; }
            if (down) { CU_API(cudaEventElapsedTime(&ms, e[2], e[3])); *down_gbs = (double)(n * piece) / (ms * 1e-3) / 1e9; }
            return VMIG_OK;
        };
        double dummy = 0;
        int rc = pass(true, false, &gbs[0], &dummy); if (rc) return rc;
        rc = pass(false, true, &dummy, &gbs[1]); if (rc) return rc;
        return pass(true, true, &gbs[2], &gbs[3]);
    };
    const int rc = run();
    const std::string keep = rc ? last_error_cstr() : "";
    cleanup();
    if (rc) set_last_error_str(keep);
    return rc;
}

int vmig_link_probe(int gpu, uint64_t bytes, double gbs[4])
{
    if (!gbs || gpu < 0 || gpu > 31) return fail(VMIG_EINVAL, "bad link-probe arguments");
    std::vector<DeviceInfo> devs; int rc = ctx_select(1u << gpu, &devs); if (rc) return rc;
    gbs[0] = gbs[1] = gbs[2] = gbs[3] = 0;
    // allocate and first-touch the pinned buffers on the GPU's NUMA node, like the staging rings
    std::string msg;
    std::thread t([&] {
        if (!devs[0].cpus.empty()) {
            cpu_set_t set; CPU_ZERO(&set);
            for (int c : devs[0].cpus) if (c < CPU_SETSIZE) CPU_SET(c, &set);
            sched_setaffinity(0, sizeof set, &set);
        }
        rc = link_probe_here(gpu, bytes ? bytes : (4ull << 30), gbs);
        if (rc) msg = last_error_cstr();
    });
    t.join();
    if (rc) set_last_error_str(msg);
    return rc;
}

// ---------------------------------------------------------------------------------------------
// HBM-resident batch.  Every call puts its copies and memsets on the handle's (non-blocking) stream and synchronises it
// before it returns: the caller's buffer may go right after, and a pass issued next is ordered after them.
struct vmig_resident {
    int dev; int sm_count; uint64_t n; uint32_t block_bytes;
    uint8_t* d_data; uint64_t* d_offs; uint32_t* d_lens; uint64_t* d_hashes; uint64_t* d_prior; uint8_t* d_valid;
    uint8_t* d_changed; uint32_t* d_survivors; uint32_t* d_nsurv; uint32_t* d_counter; uint64_t* d_scratch;
    bool has_prior; cudaStream_t stream; cudaEvent_t e0, e1, e2, e3;
};


void vmig_resident_close(vmig_resident* r);

static int resident_alloc(vmig_resident* r, uint64_t n_blocks, uint32_t block_bytes)
{
    CU_API(cudaSetDevice(r->dev));
    CU_API(cudaMalloc((void**)&r->d_data, n_blocks * (uint64_t)block_bytes + kTailPad));
    CU_API(cudaMalloc((void**)&r->d_offs, n_blocks * 8)); CU_API(cudaMalloc((void**)&r->d_lens, n_blocks * 4));
    CU_API(cudaMalloc((void**)&r->d_hashes, n_blocks * 8)); CU_API(cudaMalloc((void**)&r->d_prior, n_blocks * 8));
    CU_API(cudaMalloc((void**)&r->d_valid, n_blocks)); CU_API(cudaMalloc((void**)&r->d_changed, n_blocks));
    CU_API(cudaMalloc((void**)&r->d_survivors, n_blocks * 4)); CU_API(cudaMalloc((void**)&r->d_nsurv, 256));
    CU_API(cudaMalloc((void**)&r->d_counter, 256)); CU_API(cudaMalloc((void**)&r->d_scratch, n_blocks * 8));
    CU_API(cudaStreamCreateWithFlags(&r->stream, cudaStreamNonBlocking));
    CU_API(cudaEventCreate(&r->e0)); CU_API(cudaEventCreate(&r->e1)); CU_API(cudaEventCreate(&r->e2)); CU_API(cudaEventCreate(&r->e3));
    std::vector<uint64_t> offs(n_blocks); std::vector<uint32_t> lens(n_blocks, block_bytes);
    for (uint64_t i = 0; i < n_blocks; i++) offs[i] = i * (uint64_t)block_bytes;
    CU_API(cudaMemcpyAsync(r->d_offs, offs.data(), n_blocks * 8, cudaMemcpyHostToDevice, r->stream));
    CU_API(cudaMemcpyAsync(r->d_lens, lens.data(), n_blocks * 4, cudaMemcpyHostToDevice, r->stream));
    CU_API(cudaMemsetAsync(r->d_valid, 0, n_blocks, r->stream)); CU_API(cudaMemsetAsync(r->d_prior, 0, n_blocks * 8, r->stream));
    CU_API(cudaMemsetAsync(r->d_data + n_blocks * (uint64_t)block_bytes, 0, kTailPad, r->stream));
    CU_API(cudaStreamSynchronize(r->stream));        // offs / lens are locals
    return VMIG_OK;
}

int vmig_resident_open(int gpu, uint64_t n_blocks, uint32_t block_bytes, vmig_resident** out)
{
    if (!out || !n_blocks || !block_bytes || (block_bytes & 511u) || n_blocks > 0x7FFFFFFFull) return fail(VMIG_EINVAL, "bad resident geometry");
    if (gpu < 0 || gpu > 31) return fail(VMIG_EINVAL, "bad gpu index %d", gpu);
    std::vector<DeviceInfo> devs; int rc = ctx_select(1u << gpu, &devs); if (rc) return rc;
    vmig_resident* r = new vmig_resident(); memset(r, 0, sizeof *r);
    r->dev = gpu; r->sm_count = devs[0].sm_count; r->n = n_blocks; r->block_bytes = block_bytes;
    rc = resident_alloc(r, n_blocks, block_bytes);
    if (rc) {                                   // e.g. the batch does not fit in HBM: give back what was taken
        const std::string keep = last_error_cstr();
        vmig_resident_close(r);
        set_last_error_str(keep);
        return rc;
    }
    *out = r;
    return VMIG_OK;
}
void vmig_resident_close(vmig_resident* r)
{
    if (!r) return;
    cudaSetDevice(r->dev);
    if (r->stream) cudaStreamSynchronize(r->stream);
    cudaFree(r->d_data); cudaFree(r->d_offs); cudaFree(r->d_lens); cudaFree(r->d_hashes); cudaFree(r->d_prior); cudaFree(r->d_valid);
    cudaFree(r->d_changed); cudaFree(r->d_survivors); cudaFree(r->d_nsurv); cudaFree(r->d_counter); cudaFree(r->d_scratch);
    if (r->stream) cudaStreamDestroy(r->stream);
    if (r->e0) cudaEventDestroy(r->e0); if (r->e1) cudaEventDestroy(r->e1); if (r->e2) cudaEventDestroy(r->e2); if (r->e3) cudaEventDestroy(r->e3);
    delete r;
}
int vmig_resident_fill(vmig_resident* r, uint64_t seed)
{
    if (!r) return fail(VMIG_EINVAL, "null handle");
    CU_API(cudaSetDevice(r->dev));
    CU_API(launch_splitmix_fill(r->d_data, r->n * (uint64_t)r->block_bytes, seed, r->sm_count, r->stream));
    std::vector<uint32_t> lens(r->n, r->block_bytes);
    CU_API(cudaMemcpyAsync(r->d_lens, lens.data(), r->n * 4, cudaMemcpyHostToDevice, r->stream));
    CU_API(cudaStreamSynchronize(r->stream));
    return VMIG_OK;
}
int vmig_resident_set_len(vmig_resident* r, uint64_t block, uint32_t len)
{
    if (!r || block >= r->n || len > r->block_bytes) return fail(VMIG_EINVAL, "bad block/len");
    CU_API(cudaSetDevice(r->dev));
    CU_API(cudaMemcpyAsync(r->d_lens + block, &len, 4, cudaMemcpyHostToDevice, r->stream));
    CU_API(cudaStreamSynchronize(r->stream));
    return VMIG_OK;
}
int vmig_resident_upload(vmig_resident* r, uint64_t block, const void* host, uint32_t len)
{
    if (!r || block >= r->n || len > r->block_bytes || (len && !host)) return fail(VMIG_EINVAL, "bad block/len");
    CU_API(cudaSetDevice(r->dev));
    if (len) CU_API(cudaMemcpyAsync(r->d_data + block * (uint64_t)r->block_bytes, host, len, cudaMemcpyHostToDevice, r->stream));
    CU_API(cudaMemcpyAsync(r->d_lens + block, &len, 4, cudaMemcpyHostToDevice, r->stream));
    CU_API(cudaStreamSynchronize(r->stream));
    return VMIG_OK;
}
int vmig_resident_download(vmig_resident* r, uint64_t block, void* host, uint32_t len)
{
    if (!r || block >= r->n || len > r->block_bytes || !host) return fail(VMIG_EINVAL, "bad block/len");
    CU_API(cudaSetDevice(r->dev));
    CU_API(cudaMemcpyAsync(host, r->d_data + block * (uint64_t)r->block_bytes, len, cudaMemcpyDeviceToHost, r->stream));
    CU_API(cudaStreamSynchronize(r->stream));
    return VMIG_OK;
}
int vmig_resident_flip(vmig_resident* r, const uint64_t* blocks, uint64_t n)
{
    if (!r || (n && !blocks) || n > r->n) return fail(VMIG_EINVAL, "bad flip list");
    for (uint64_t i = 0; i < n; i++) if (blocks[i] >= r->n) return fail(VMIG_EINVAL, "flip index out of range");
    CU_API(cudaSetDevice(r->dev));
    if (n) {
        CU_API(cudaMemcpyAsync(r->d_scratch, blocks, n * 8, cudaMemcpyHostToDevice, r->stream));
        CU_API(launch_flip_first8(r->d_data, r->d_offs, r->d_scratch, n, r->stream));
        CU_API(cudaStreamSynchronize(r->stream));
    }
    return VMIG_OK;
}
int vmig_resident_set_prior(vmig_resident* r, const uint64_t* hashes, const uint8_t* valid)
{
    if (!r) return fail(VMIG_EINVAL, "null handle");
    CU_API(cudaSetDevice(r->dev));
    r->has_prior = hashes != nullptr && valid != nullptr;
    if (r->has_prior) {
        CU_API(cudaMemcpyAsync(r->d_prior, hashes, r->n * 8, cudaMemcpyHostToDevice, r->stream));
        CU_API(cudaMemcpyAsync(r->d_valid, valid, r->n, cudaMemcpyHostToDevice, r->stream));
    } else {
        CU_API(cudaMemsetAsync(r->d_valid, 0, r->n, r->stream));
    }
    CU_API(cudaStreamSynchronize(r->stream));
    return VMIG_OK;
}
int vmig_resident_pass(vmig_resident* r, uint32_t iters, double* ms_hash_last, double* ms_total)
{
    if (!r || !iters) return fail(VMIG_EINVAL, "bad arguments");
    CU_API(cudaSetDevice(r->dev));
    HashLaunch a;
    a.base = r->d_data; a.offs = r->d_offs; a.lens = r->d_lens; a.n = (uint32_t)r->n; a.hashes = r->d_hashes;
    a.prior = r->d_prior; a.prior_valid = r->d_valid; a.changed = r->d_changed; a.work_counter = r->d_counter;
    CU_API(cudaEventRecord(r->e0, r->stream));
    for (uint32_t it = 0; it < iters; it++) {
        if (it + 1 == iters) CU_API(cudaEventRecord(r->e1, r->stream));
        CU_API(launch_xxh64_blocks(a, r->sm_count, r->stream));
        if (it + 1 == iters) CU_API(cudaEventRecord(r->e2, r->stream));
        CU_API(launch_diff_select(r->d_changed, (uint32_t)r->n, r->d_survivors, r->d_nsurv, r->stream));
    }
    CU_API(cudaEventRecord(r->e3, r->stream));
    CU_API(cudaStreamSynchronize(r->stream));
    float a_ms = 0, b_ms = 0;
    CU_API(cudaEventElapsedTime(&a_ms, r->e1, r->e2));
    CU_API(cudaEventElapsedTime(&b_ms, r->e0, r->e3));
    if (ms_hash_last) *ms_hash_last = a_ms;
    if (ms_total) *ms_total = b_ms;
    return VMIG_OK;
}
int vmig_resident_results(vmig_resident* r, uint64_t* hashes, uint32_t* survivors, uint64_t* n_survivors)
{
    if (!r) return fail(VMIG_EINVAL, "null handle");
    CU_API(cudaSetDevice(r->dev));
    if (hashes) CU_API(cudaMemcpyAsync(hashes, r->d_hashes, r->n * 8, cudaMemcpyDeviceToHost, r->stream));
    uint32_t ns = 0;
    CU_API(cudaMemcpyAsync(&ns, r->d_nsurv, 4, cudaMemcpyDeviceToHost, r->stream));
    CU_API(cudaStreamSynchronize(r->stream));
    if (n_survivors) *n_survivors = ns;
    if (survivors && ns) {
        CU_API(cudaMemcpyAsync(survivors, r->d_survivors, (size_t)ns * 4, cudaMemcpyDeviceToHost, r->stream));
        CU_API(cudaStreamSynchronize(r->stream));
    }
    return VMIG_OK;
}

}  // extern "C"
