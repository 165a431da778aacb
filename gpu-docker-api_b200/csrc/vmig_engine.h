// vmig_engine.h -- per-GPU streaming pipeline of libvmig (internal interface).
//
//   source blocks --(reader threads: pread / memcpy)--> pinned IN slot
//       --cudaMemcpyAsync H2D (slot's side stream)--> HBM slot
//       --xxh64_blocks kernel (+ compare with prior table)--> hashes, changed flags
//       --cudaMemcpyAsync D2H of the surviving blocks--> pinned OUT slot
//       --(writer threads: pwrite / memcpy)--> destination
//
// One Pipe owns kSlots such slot triples on one GPU; a lane (one GPU's share of one call) checks
// a Pipe out of the process-wide pool, runs its block list through it and returns it.
#pragma once
#include <stdint.h>
#include <atomic>
#include <memory>
#include <mutex>
#include <string>
#include <vector>
#include "vmig_common.h"

namespace vmig {

struct BlockRef {
    uint32_t file;         // backend-defined (index of the file in the manifest; 0 for buffers)
    uint32_t len;          // bytes in this block (<= block_bytes; 0 allowed)
    uint64_t file_off;     // byte offset inside the file / buffer
    uint64_t table_idx;    // where this block's hash goes in the call-wide hash array
    uint64_t prior_hash;   // prior version's hash of the same block ...
    uint8_t  prior_valid;  // ... if 1
};

// Where block bytes come from and go to.  Implementations must be thread-safe.
class BlockIO {
public:
    virtual ~BlockIO() {}
    virtual int  read_block(const BlockRef& b, uint8_t* dst) = 0;
    virtual int  write_block(const BlockRef& b, const uint8_t* src) = 0;
    // called exactly once per block when it needs nothing more (written == false: skipped)
    virtual int  block_done(const BlockRef&, bool /*written*/) { return VMIG_OK; }
    // true: block_done of this block, if skipped, may do file-sized work (vmig_snapshot_tree links or backfills the file
    // when its last block passes); it then runs on a writer thread under the block's write key, not on the d2h-waiter
    virtual bool done_on_writer(const BlockRef&) { return false; }
    // skip mode (has_prior): asked in the hash-waiter, before any D2H, for each block K1 found changed against its prior
    // hash.  true: the backend has these bytes elsewhere (vmig_snapshot_tree: a base block with the same hash and
    // length); the block is then skipped like an unchanged one -- no D2H, no write, block_done(b, false)
    virtual bool reusable(const BlockRef&, uint64_t /*hash*/) { return false; }
    // writes with the same key are issued by one writer thread, in order (a file takes writes from one
    // thread at a time anyway); backends without such a constraint spread the keys
    virtual uint32_t write_key(const BlockRef& b) { return b.file; }
    // staging layout: every block starts at a multiple of this inside a slot (>= 512, a power of two).  O_DIRECT
    // file I/O needs logical-sector alignment of buffer, offset and length: 4096.
    virtual uint32_t slot_align() { return 512; }
    // GPUDirect-Storage style backends move bytes between the file and the HBM slot themselves (no pinned ring, no
    // cudaMemcpyAsync): read_block_dev fills d_base + d_off, write_block_dev drains it.  Called on reader / writer threads.
    virtual bool device_reads()  { return false; }
    virtual bool device_writes() { return false; }
    virtual int  read_block_dev(const BlockRef&, uint8_t* /*d_base*/, size_t /*d_off*/) { return VMIG_EINVAL; }
    virtual int  write_block_dev(const BlockRef&, const uint8_t* /*d_base*/, size_t /*d_off*/) { return VMIG_EINVAL; }
    // non-null: page-locked memory the DMA engines can use directly (no staging copy)
    virtual const uint8_t* pinned_src(const BlockRef&) { return nullptr; }
    virtual uint8_t*       pinned_dst(const BlockRef&) { return nullptr; }
    // how error messages name a block
    virtual std::string block_name(const BlockRef& b) { return "block at offset " + std::to_string(b.file_off); }
};

// The hashes blocks must have (nullable in run_lane): hashes[b.table_idx], for every block or, with a mask, for the blocks
// with valid[b.table_idx] != 0.  A block that hashes otherwise fails the call with `code` before any block of its batch
// is written: VMIG_ECORRUPT when the table speaks for the source (a checked restore), VMIG_ESRCCHANGED when it speaks for
// a file that may have been written since (vmig_snapshot_layer).
struct BlockExpect {
    const uint64_t* hashes = nullptr;
    const uint8_t* valid = nullptr;
    int code = VMIG_ECORRUPT;
};

struct LaneStats {
    uint64_t bytes_h2d = 0, bytes_d2h = 0, bytes_written = 0, blocks_skipped = 0, kernel_launches = 0;
    double   ms_kernel = 0;
};

// Cancellation and progress of one call (include/vmig.h, vmig_ctl_*).  Every data-path call has one, a caller's
// control (vmig_opts.ctl) or a private one, so that vmig_shutdown can cancel whatever is in flight.
struct CallCtl {
    std::atomic<int> cancelled{0};
    std::atomic<uint32_t> phase{VMIG_PHASE_IDLE}, running{0};
    std::atomic<uint64_t> bytes_total{0}, blocks_total{0}, bytes_hashed{0}, blocks_hashed{0}, bytes_written{0}, bytes_verified{0};
    std::mutex mu;
    std::atomic<int>* latch = nullptr;    // first-error latch of the block pipeline in progress (under mu)
    void cancel();                        // vmig_api.cu
};

// Where run_lane reports progress (relaxed adds: once per batch in the hash-waiter, once per write task)
struct LaneProgress {
    std::atomic<uint64_t>* hashed_bytes = nullptr;
    std::atomic<uint64_t>* hashed_blocks = nullptr;
    std::atomic<uint64_t>* written = nullptr;
};

struct DeviceInfo {
    int dev = -1;
    int sm_count = 0;
    std::vector<int> cpus;     // NUMA-local CPUs of the GPU (empty: no affinity)
};

class Pipe;   // defined in vmig_engine.cu

// ---- process-wide context -------------------------------------------------------------------
int  ctx_init(uint32_t gpu_mask);
void ctx_shutdown();
int  ctx_device_count();
// devices selected by `mask` (0 = all initialised); error if none
int  ctx_select(uint32_t mask, std::vector<DeviceInfo>* out);
int  ctx_acquire_pipe(const DeviceInfo& d, Pipe** out);
// one Pipe per lane, all reserved atomically (a device may repeat: lanes_per_gpu).  While it waits for pipes other calls
// hold, a non-zero *cancel makes it return VMIG_ECANCELED with nothing reserved (the canceller calls ctx_wake_waiters).
int  ctx_acquire_pipes(const std::vector<DeviceInfo>& lane_devs, std::vector<Pipe*>* out, const std::atomic<int>* cancel = nullptr);
void ctx_wake_waiters();
void ctx_release_pipe(Pipe* p);
uint32_t pipe_slot_bytes();
int  io_threads_default(uint32_t* readers, uint32_t* writers, uint32_t requested, size_t lanes, size_t n_gpus, bool many_files,
                        bool has_prior, bool hash_only);

// Run blocks[] through one GPU.  hashes_out[b.table_idx] receives every block's hash.
//   hash_only : no D2H of data, no writes (block_done(b,false) is still called).
//   expect    : nullable; the hash block b must have (BlockExpect).  Checked before any block of its batch is written
//               (skipped ones included).
//   err       : call-wide first-error latch shared by all lanes (0 = fine); a cancel sets it from outside.
int run_lane(Pipe* pipe, const std::vector<BlockRef>& blocks, BlockIO* io, bool has_prior, bool hash_only,
             uint32_t readers, uint32_t writers, uint32_t max_slots, const BlockExpect* expect, uint64_t* hashes_out,
             LaneStats* stats, std::atomic<int>* err, std::string* err_msg, std::mutex* err_mu, LaneProgress prog = LaneProgress());

}  // namespace vmig
