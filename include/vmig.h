/*
 * vmig.h -- C ABI of libvmig, the H100-native volume-migration engine.
 *
 * Drop-in boundary for the ONE data-parallel path of XShengTech/gpu-docker-api: the bulk copy
 * of a container's system-disk diff layer (ReplicaSet Patch / Rollback / Restart) and of a
 * Docker-volume data disk (Volume resize).  The reference has no plugin/FFI interface; the
 * seam is three package-level Go functions in package utils (SURVEY.md §8b):
 *
 *   utils.CopyDir(src, dest string) error                         reference utils/copy.go:21-27
 *   utils.CopyOldMergedToNewContainerMerged(old, new string) error reference utils/copy.go:31-46
 *   utils.CopyOldMountPointToContainerMountPoint(old, new) error   reference utils/copy.go:58-63
 *     (-> moveVolumeData, reference utils/copy.go:74-128)
 *
 * called from internal/services/replicaset.go:333,421,831 and internal/services/volume.go:150.
 * A cgo shim (INTEGRATION.md) re-implements those three functions on top of the entry points
 * below; nothing else in the reference changes.
 *
 * Conventions (what a cgo binding needs):
 *   - every function returns 0 (VMIG_OK) or a negative VMIG_E* code; vmig_last_error() gives a
 *     thread-local human-readable message for the calling thread's last failure;
 *   - all pointers are borrowed for the duration of the call only (no Go memory is retained);
 *   - no callbacks into the caller; every entry point is re-entrant and thread-safe (the
 *     reference calls the copy from concurrent gin goroutines with no locking, SURVEY.md F9);
 *   - there is NO CPU fallback: without a usable sm_90 device the data-path calls fail with
 *     VMIG_ENOGPU.
 *
 * Data path of one migration (DESIGN.md):  source file blocks (4 MiB, file-aligned) -> pinned
 * host slot -> cudaMemcpyAsync H2D on a side stream -> xxh64_blocks kernel (canonical XXH64,
 * seed 0, one hash per block) -> compare with the prior version's block table -> surviving
 * blocks cudaMemcpyAsync D2H into the destination pinned slot -> destination file.
 */
#ifndef VMIG_H
#define VMIG_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VMIG_ABI_VERSION 2     /* 2: vmig_opts.lanes_per_gpu, vmig_stats.lanes_used/.pruned, VMIG_F_PRUNE, table format 02 */

/* ---- error codes ------------------------------------------------------------------------ */
#define VMIG_OK          0
#define VMIG_EINVAL     (-1)   /* bad argument (NULL path, unaligned device offset, ...)        */
#define VMIG_ENOGPU     (-2)   /* no CUDA driver / no sm_90 device in the mask: no CPU fallback  */
#define VMIG_ECUDA      (-3)   /* a CUDA runtime call or kernel failed                          */
#define VMIG_EIO        (-4)   /* open/read/write/metadata syscall failed, or short read/write   */
#define VMIG_ENOMEM     (-5)   /* host or device allocation failed                              */
#define VMIG_ETABLE     (-6)   /* malformed / incompatible block-table file                     */
#define VMIG_EFAULT     (-7)   /* injected fault (VMIG_FAIL_BLOCK test hook)                    */
#define VMIG_ENOTDIR    (-8)   /* src or dst is not a directory (reference utils/file.go:50-59)  */
#define VMIG_ESRCCHANGED (-9)  /* a source file shrank while it was being read                  */
#define VMIG_EVERIFY    (-10)  /* VMIG_F_VERIFY: a destination block does not hash like its source */
#define VMIG_ECORRUPT   (-11)  /* vmig_restore_tree: the source tree is not the one its block table describes */
#define VMIG_ECANCELED  (-12)  /* the call's control was cancelled (vmig_ctl_cancel, vmig_shutdown) */

/* ---- lifecycle --------------------------------------------------------------------------- */
/* Idempotent, thread-safe.  gpu_mask bit i selects CUDA device i; 0 = all visible devices.
 * Creates the per-GPU contexts lazily (streams, pinned staging rings, HBM slots).  Hook:
 * reference cmd/gpu-docker-api/main.go:53-97 (Init); optional -- every call inits on demand. */
int  vmig_init(uint32_t gpu_mask);
/* Frees every pooled resource.  Hook: reference cmd/gpu-docker-api/main.go:139-154 (Stop).  Calls still in flight are
 * cancelled first (they return VMIG_ECANCELED) and shutdown waits for them to return before it frees anything. */
void vmig_shutdown(void);
int  vmig_device_count(void);                 /* usable sm_90 devices, or VMIG_ENOGPU           */
const char* vmig_strerror(int code);
const char* vmig_last_error(void);            /* thread-local detail of the last failure         */
const char* vmig_version(void);

/* ---- options / statistics ------------------------------------------------------------------ */
#define VMIG_F_MOVE_SRC          0x01u  /* unlink source entries after the copy succeeded and the destination
                                           was flushed (syncfs): the `mv` of moveVolumeData (reference
                                           utils/copy.go:116).  Combine with VMIG_F_VERIFY (vmig_move_dir
                                           does) to also re-hash the destination before unlinking           */
#define VMIG_F_SKIP_HIDDEN_TOPDIRS 0x02u /* reproduce `mv /root/src/ *`: top-level hidden DIRECTORIES
                                           are left behind (reference utils/copy.go:116)           */
#define VMIG_F_MTIME_NS          0x04u  /* keep nanosecond mtimes (mv does; GNU tar's default archive
                                           format keeps whole seconds only -> default off)         */
#define VMIG_F_NO_METADATA       0x08u  /* data only: no chown/chmod/utimens.  Directories that already exist and
                                           regular files patched in place keep their owner and mode (a read-only
                                           file an ordinary user's diff pass patches gets its own mode back), and
                                           their mtime unless the call writes into them.  Whatever the call
                                           creates -- every other file, every special file and symlink, missing
                                           directories -- is owned by the caller, has the mtime of its creation and
                                           the creation mode less the process umask: regular files and specials
                                           0600, directories 0700                                            */
#define VMIG_F_HASH_ONLY         0x10u  /* build the block table of src; dst is not touched        */
#define VMIG_F_VERIFY            0x20u  /* after the copy, re-read the DESTINATION through the GPU and
                                           require its block hashes to equal the source's; with
                                           VMIG_F_MOVE_SRC the source is only unlinked if they do    */

#define VMIG_F_PRUNE             0x40u  /* after the copy, remove every destination entry the source does not
                                           have (files, symlinks, specials, whole directories).  tar never does
                                           (default off); the final, paused pass of a hand-off needs it: a file
                                           the tenant deleted or renamed since the live pass must not reappear
                                           in the new container.  With VMIG_F_VERIFY the destination's entry set
                                           is then re-walked and must equal the source's                       */

#define VMIG_F_DIRECT_IO         0x80u  /* disk-backed trees (the documented deployment keeps the Docker root on
                                           xfs/LVM: reference docs/volume/volume-size-scale-en.md:5-21): source
                                           files are read with O_DIRECT straight INTO the pinned staging ring and
                                           destination files written with O_DIRECT straight OUT of it -- the NVMe
                                           DMAs to/from the same page-locked memory the GPU's copy engines use, and
                                           the page cache (two CPU copies per byte) is bypassed.  Falls back to
                                           buffered I/O per file where the filesystem refuses O_DIRECT.  Env
                                           VMIG_DIRECT_IO=1 sets it for every call.                              */
#define VMIG_F_CUFILE            0x100u /* GPUDirect Storage: source blocks are read with cuFileRead straight into the
                                           HBM slot (no IN ring, no H2D copy) and surviving blocks written with
                                           cuFileWrite straight out of it (no D2H copy, no OUT ring).  libcufile is
                                           dlopen()ed: VMIG_EINVAL if it cannot be loaded or its driver cannot be
                                           opened, VMIG_EIO with libcufile's own reason if it refuses a descriptor
                                           (inside containers it needs a udev-visible block device: DESIGN.md §10).
                                           Without the nvidia-fs kernel module the call fails with VMIG_EINVAL
                                           before libcufile is entered (its compatibility mode is not used).
                                           Env VMIG_CUFILE=1.                                                      */

typedef struct vmig_opts {
    uint32_t gpu_mask;         /* 0 = every initialised GPU; blocks are sharded across the set   */
    uint32_t block_bytes;      /* 0 -> 4 MiB (4194304); must be a multiple of 4096               */
    uint32_t streams_per_gpu;  /* side streams = staging slots in flight PER LANE (each lane has its own pipe of
                                  VMIG_SLOTS slots, 16 by default); 0 or more than the pipe has -> all of them     */
    uint32_t flags;            /* VMIG_F_*                                                       */
    uint32_t io_threads;       /* host copy threads PER LANE: n >= 2 -> exactly n, r = (n+1)*2/5 readers and n - r
                                  writers; 1 -> one reader and one writer; 0 -> the per-box budget divided among
                                  the lanes in flight (vmig_thread_plan)                                          */
    uint32_t lanes_per_gpu;    /* 0/1 -> one lane (staging-ring set + thread pipeline) per GPU of the
                                  mask; k -> k lanes per GPU, the block list is sharded over
                                  n_gpus*k lanes exactly as it is over n_gpus*k GPUs (more host
                                  copy parallelism per link; also how the multi-GPU split is
                                  exercised on a 1-GPU box).  Env VMIG_LANES_PER_GPU overrides 0. */
    uint32_t ctl;              /* 0 = no control; else an id from vmig_ctl_open: the call can be cancelled and
                                  reports its progress through it (see "Cancellation and progress")             */
    uint32_t reserved;
} vmig_opts;

typedef struct vmig_stats {
    uint64_t bytes_total;      /* N: sum of regular-file sizes migrated                          */
    uint64_t bytes_h2d;        /* bytes DMA'd host->HBM                                          */
    uint64_t bytes_d2h;        /* bytes DMA'd HBM->host (surviving blocks)                       */
    uint64_t bytes_written;    /* bytes written to destination files                             */
    uint64_t blocks_total;
    uint64_t blocks_skipped;   /* unchanged vs prior table: no D2H, no write                     */
    uint64_t files, dirs, symlinks, hardlinks, specials;
    uint64_t kernel_launches;  /* xxh64_blocks + diff_select launches                            */
    uint64_t ns_total, ns_walk, ns_plan, ns_data, ns_meta, ns_table;
    double   ms_kernel;        /* sum of CUDA-event time of the hash kernels                     */
    uint32_t gpus_used;
    uint32_t lanes_used;       /* lanes the block list was sharded over (gpus_used * lanes_per_gpu) */
    uint64_t pruned;           /* VMIG_F_PRUNE: destination entries removed                      */
    uint64_t files_untrusted;  /* prior table given, but the destination file is no longer the one it was
                                  written for (inode/ctime/size): copied in full, not patched    */
    uint64_t files_direct;     /* VMIG_F_DIRECT_IO / VMIG_F_CUFILE: descriptors (source + destination) the
                                  filesystem really let us open with O_DIRECT                    */
} vmig_stats;

/* ---- the hot path -------------------------------------------------------------------------- */
/* Migrate directory tree src_dir/. into the existing directory dst_dir (semantics of
 * `(cd src; tar c .) | (cd dst; tar x)` run as root: reference utils/copy.go:17-27 -- file
 * bytes, mode, uid, gid, mtime, symlinks, hard links, device nodes and FIFOs are reproduced;
 * xattrs are not; existing destination entries are overwritten, extras are never pruned).
 *   prior_table : nullable path of the block table describing what dst ALREADY holds (the prior
 *                 version).  Blocks whose XXH64 equals the prior entry are neither copied back
 *                 from HBM nor written (diff-skip) -- per file, and only while the destination file
 *                 still is the one the table was written for (see "Block-table file").
 *   out_table   : nullable path; receives the block table of src (tmp + rename, after all data
 *                 writes completed).
 * Blocking; re-entrant; returns 0 or -VMIG_E*.  On error the destination may be partially
 * written (the reference does no cleanup either: SURVEY.md §8b) but the call never reports
 * success after a short read/write or a CUDA error. */
int vmig_migrate_tree(const char* src_dir, const char* dst_dir,
                      const char* prior_table, const char* out_table,
                      const vmig_opts* opts /*nullable*/, vmig_stats* stats /*nullable*/);

/* Restore a snapshot (a tree a migration wrote together with snap_table, its block table) into dst_dir: exactly
 * vmig_migrate_tree(snap_dir, dst_dir, prior_table, out_table, opts, stats), except that snap_dir must still be the
 * tree snap_table describes.  A restore store that puts back whatever happens to be on disk -- a snapshot that
 * failed part way, was edited, or rotted -- is refused instead:
 *   - snap_table is required (NULL/empty: VMIG_EINVAL); it is loaded like prior_table (formats 01 and 02, algo 1)
 *     and its block_bytes must equal the call's (VMIG_ETABLE).  VMIG_F_MOVE_SRC: VMIG_EINVAL.
 *   - before the destination is touched (before VMIG_F_PRUNE, before any directory is made or block read): the
 *     walked regular-file paths, hard-linked ones included, must be the table's paths, each with the table's size.
 *     The table's ino/ctime_ns are not used (a copied snapshot keeps its bytes, not its inodes).
 *   - every block's XXH64, computed on the GPU as it passes, must equal the table's; a block that does not is never
 *     written, also where prior_table says the destination already holds it.  A hard-linked path's table hashes
 *     must equal what its primary hashed, checked before any link is created.
 * The first difference fails the call with VMIG_ECORRUPT; vmig_last_error() names the path and says whether it is
 * missing, extra or resized, or names the block and both hashes.  Directories, symlinks, specials and metadata are
 * not in the table and are not checked.  As always on failure, no out_table is written and the destination may
 * be partially written (never with a block that failed the check).
 * With VMIG_F_HASH_ONLY, dst_dir may be NULL: the snapshot is only checked against its table and no destination is
 * touched (pass out_table = NULL to write nothing at all).
 * The walk flags (VMIG_F_SKIP_HIDDEN_TOPDIRS) must be those the snapshot's table was written with. */
int vmig_restore_tree(const char* snap_dir, const char* snap_table, const char* dst_dir,
                      const char* prior_table, const char* out_table,
                      const vmig_opts* opts /*nullable*/, vmig_stats* stats /*nullable*/);

/* Restore chosen entries of a snapshot (snap_dir with its block table snap_table) into dst_dir, each regular file with
 * the guarantees vmig_restore_tree gives, and nothing in dst_dir outside those entries and their parent directories.
 *   - paths[0..n_paths) are bytes relative to snap_dir, naming entries exactly as the table does.  VMIG_EINVAL, before
 *     the GPU check and with nothing touched: n_paths == 0, a NULL array or entry, a path that is empty, absolute, has
 *     an empty, "." or ".." component or ends in '/', two paths equal or one beneath the other (vmig_last_error() names
 *     the index and the path); snap_table NULL/empty; snap_dir and dst_dir the same directory or one inside the other
 *     (real paths); VMIG_F_MOVE_SRC, VMIG_F_HASH_ONLY or VMIG_F_CUFILE; a bad block_bytes.  A control cancelled before
 *     the call is VMIG_ECANCELED; then comes VMIG_ENOGPU.
 *   - A path is found when every proper prefix is a real directory under snap_dir (no symlink followed) and the entry
 *     exists; it may be of any kind.  Not found: VMIG_ECORRUPT when the table has a record at or beneath it (missing),
 *     else VMIG_EINVAL (not in the snapshot).  The selection -- the chosen entries and everything beneath the chosen
 *     directories -- is walked as walk_tree walks (order, block layout, VMIG_F_SKIP_HIDDEN_TOPDIRS) and only it is read;
 *     hard links are grouped inside the selection only (a path whose inode is also named outside it is restored as a
 *     file of its own).
 *   - Before dst_dir is touched, the table records at a chosen path or beneath a chosen directory must be exactly the
 *     selection's regular-file paths with the table's sizes (VMIG_ECORRUPT: missing, extra or resized, as restore says
 *     it).  Every block's XXH64 is checked on the GPU against the table as it passes and a block that fails is never
 *     written; a hard-linked path's hashes are checked before any link is made.  Records outside the selection are not
 *     looked at: a snapshot damaged elsewhere restores its intact part.
 *   - dst_dir must exist (VMIG_EIO / VMIG_ENOTDIR).  No destination symlink is ever followed.  Each proper prefix of a
 *     chosen path is made a real directory: an existing one is used as it is (owner and mode unchanged); a missing one,
 *     or anything else in the way (symlink, file, special file, overlay whiteout, removed), becomes a directory with the
 *     snapshot's owner, mode and mtime, applied after its contents.  The chosen entries and everything beneath them are
 *     replaced exactly as vmig_restore_tree replaces them.  Nothing else in dst_dir is created, removed or modified; only
 *     a parent directory's mtime moves, as any create in it moves it.
 *   - VMIG_F_PRUNE removes, by descriptor, destination entries beneath each chosen directory that the snapshot's
 *     subtree does not have, never anything elsewhere; with VMIG_F_VERIFY the chosen directories' entry sets are then
 *     re-walked and must equal the snapshot's.  VMIG_F_VERIFY, VMIG_F_DIRECT_IO, VMIG_F_MTIME_NS, VMIG_F_NO_METADATA,
 *     VMIG_F_SKIP_HIDDEN_TOPDIRS, lanes_per_gpu, gpu_mask and ctl act as in a restore.
 *   - prior_table (nullable): the destination's own table, used as vmig_migrate_tree uses it (a file still its record
 *     is patched in place; one whose blocks and metadata are unchanged is left alone).  No out table is written: the
 *     records of the files this call rewrote go stale by the usual trust rule, and the next diff pass copies them in full.
 * Phases WALK, (PRUNE), DATA, META, (VERIFY), DONE; bytes_total / blocks_total and stats are the selection's (dirs
 * counts the selection's directories and the parents the call created).  On failure or cancel the destination may be
 * partly written inside the selection and its parent chains, never with a block that failed a check; snap_dir and
 * both tables are never modified. */
int vmig_restore_paths(const char* snap_dir, const char* snap_table, const char* dst_dir,
                       uint32_t n_paths, const char* const* paths,
                       const char* prior_table /*nullable*/,
                       const vmig_opts* opts /*nullable*/, vmig_stats* stats /*nullable*/);

/* Incremental version snapshot: what vmig_snapshot_tree took from the base snapshot instead of the GPU's staging ring. */
typedef struct vmig_snapshot_stats {
    uint64_t files_linked;          /* regular files that are a hard link to the base snapshot's file: no data written */
    uint64_t bytes_linked;
    uint64_t files_backfilled;      /* new files whose unchanged blocks were copied from the base file, not the ring */
    uint64_t bytes_backfilled;
    uint64_t files_base_untrusted;  /* base table names the path but the base file is no longer the one it recorded */
    uint64_t reserved[3];
} vmig_snapshot_stats;

/* Write a version snapshot of src_dir into dst_dir (a new, empty directory, or a partial earlier attempt with
 * VMIG_F_PRUNE) and its block table into out_table, sharing what did not change with the previous snapshot:
 * base_dir, written together with base_table by an earlier vmig_snapshot_tree / vmig_migrate_tree.
 *   - base_dir == base_table == NULL: a full snapshot, the copy vmig_migrate_tree(src_dir, dst_dir, NULL, out_table,
 *     opts, stats) makes.  Only one of them given: VMIG_EINVAL.  out_table NULL/empty: VMIG_EINVAL (a snapshot is restored against it).
 *   - VMIG_F_MOVE_SRC, VMIG_F_HASH_ONLY and VMIG_F_CUFILE: VMIG_EINVAL.  So is a base_dir that is dst_dir, or lies
 *     inside it, or contains it (compared by real path).  VMIG_F_VERIFY, VMIG_F_PRUNE, VMIG_F_DIRECT_IO,
 *     lanes_per_gpu and gpu_mask act as in a migration.
 *   - base_table loads like a prior table (formats 01 and 02); its block_bytes must equal the call's (VMIG_ETABLE).
 * A base file is trusted when dst_dir and base_dir are on one device, the base table records it with an inode, and it
 * is still that regular file with that inode, ctime and size (its link count may exceed 1: base files are shared with
 * older snapshots).  Unchanged content is found in the trusted base files by block, wherever it sits there:
 *   - a source file whose path a trusted base file has is compared on the GPU with that file's hashes, block by block,
 *     exactly as the in-place diff path compares with a prior table;
 *   - every other block -- a changed one, or one of a file the base holds under another path -- is looked up by its
 *     (XXH64, length) among all blocks of all trusted base files.
 * A block found either way is neither copied back from HBM nor written.  When the file's last block has passed:
 *   - link: the new path becomes a hard link to a base file if no block was written, the base file has the source
 *     file's size and every block hash at the same index, the source file has no hard-link partner in src_dir, no
 *     other path of this call was linked to that base inode, and the base inode already carries the owner, mode and
 *     mtime the copy would get.  The same-path base file is tried first, then the others in table order, so a file
 *     moved or renamed with its mtime kept is linked.  A linked inode's metadata is never changed (that would change
 *     older snapshots too);
 *   - backfill: otherwise the file is written new: changed blocks from the ring, the others copied from the base --
 *     the same-path block when it matches, else the block that continues the previous block's base run, else the
 *     first base block with that hash and length -- in runs contiguous in one base file (copy_file_range, or
 *     pread/pwrite where that is refused), then its metadata applied.  Matches are whole blocks at block offsets.
 * Before it links or copies from a base file the call re-checks its inode and ctime (the ctime it recorded, or the one
 * this call's own link to it left); a base file that changed during the call fails it with VMIG_ESRCCHANGED naming the
 * path (a retry copies that file in full).  A reused block trusts (XXH64, length) equality as the positional skip does:
 * with n changed source blocks and m base blocks, a chance collision has probability at most n*m/2^64 (about 5e-8 for
 * 1e6 x 1e6); VMIG_F_VERIFY re-reads linked and backfilled files.  Files none of whose blocks the base holds are copied
 * as by vmig_migrate_tree; where the base table named the path but the file is not trusted, files_base_untrusted counts
 * it.
 * Empty files are never linked.  out_table records the inode and ctime of every file as this call leaves it, linked
 * and hard-linked files included (vmig_migrate_tree records a hard-linked file before its links are made), so that the
 * next snapshot can use each one as a base.
 * Linking moves the base inode's ctime, so the base table's own record of that file goes stale: a later snapshot
 * against that same base copies the file in full, and vmig_restore_tree does not read identities at all.
 * snap_stats (nullable) receives the counters above; stats as for vmig_migrate_tree (bytes_written counts ring
 * writes only). */
int vmig_snapshot_tree(const char* src_dir, const char* dst_dir,
                       const char* base_dir /*nullable*/, const char* base_table /*nullable*/,
                       const char* out_table, const vmig_opts* opts /*nullable*/,
                       vmig_stats* stats /*nullable*/, vmig_snapshot_stats* snap_stats /*nullable*/);

/* Scrub of a snapshot store: what vmig_scrub_store read and found. */
typedef struct vmig_scrub_stats {
    uint64_t versions, versions_damaged;   /* versions whose verdict is not VMIG_OK                                  */
    uint64_t bytes_referenced;             /* sum of regular-file sizes over all versions' walks (per path)          */
    uint64_t bytes_unique;                 /* bytes of distinct inodes read and hashed: what the scrub cost          */
    uint64_t files_damaged;                /* (version, path) pairs with at least one finding                        */
    uint64_t blocks_damaged;               /* (inode, block) pairs whose hash differs from some table naming it      */
    uint64_t files_unreadable;             /* distinct inodes that failed to read (every naming version damaged)     */
    uint64_t reserved[4];
} vmig_scrub_stats;

/* Check the n versions of a snapshot store -- snap_dirs[i] written together with its block table snap_tables[i] by
 * vmig_snapshot_tree -- in one pass that reads each distinct inode once, however many versions hard-link it.  Nothing
 * is written under any snap_dir and no table is touched: inode ctimes stay as they were, so the identities the next
 * incremental snapshot trusts stay valid.
 *   - verdicts[i] (nullable; n entries, written on success) is what vmig_restore_tree(snap_dirs[i], snap_tables[i],
 *     NULL, NULL, NULL, {VMIG_F_HASH_ONLY}) returns for that version, with two differences: a snapshot directory that
 *     is missing or not a directory is VMIG_ENOTDIR (restore: VMIG_EIO when missing), and a file that cannot be read
 *     (or a directory of the version that cannot be walked) is VMIG_ECORRUPT (restore: VMIG_EIO):
 *       VMIG_OK        the version matches its table;
 *       VMIG_ECORRUPT  a path is missing, extra or resized, a block's XXH64 differs from the table's, a hard-linked
 *                      path's table hashes differ from what its primary holds, or a file could not be read;
 *       VMIG_ETABLE    the table is missing, cannot be loaded, or its block_bytes differs from the call's;
 *       VMIG_ENOTDIR   the snapshot directory is missing or is not a directory.
 *   - A damaged version is a result, not a failure: the call returns VMIG_OK when it ran to the end.  It fails with
 *     VMIG_EINVAL (n == 0, a NULL array or entry, flags other than VMIG_F_DIRECT_IO | VMIG_F_SKIP_HIDDEN_TOPDIRS, bad
 *     block_bytes), VMIG_ENOGPU (checked before anything is read), VMIG_ECANCELED, VMIG_ECUDA, VMIG_ENOMEM,
 *     VMIG_ESRCCHANGED (an inode is no longer the one the walk saw -- other inode, type or size, or shorter than its
 *     blocks: the store was modified during the scrub) or VMIG_EIO (writing the report).  A failed call writes no
 *     verdicts and leaves report_path as it was, with no .tmp beside it.
 *   - Plan: every version is walked as restore walks it, its table merged against the walk (every difference recorded),
 *     and the matched regular files of all versions grouped by (st_dev, st_ino).  Each distinct inode is read once
 *     through the block pipeline in hash-only mode -- lanes, GPUs and VMIG_F_DIRECT_IO as in a checked restore; with
 *     VMIG_F_DIRECT_IO what is checked is what the device holds -- and each block hash is then compared on the host with
 *     every table record that names that inode.  An inode that fails to open or read is not a call failure: it is
 *     reported `unreadable` for every version that names it, and its remaining blocks are not read.
 *   - report_path (nullable): one line per finding, sorted by version, then path (bytewise), then block:
 *       <version index>\t<kind>\t<path>\t<block|->\t<got|->\t<want|->\n
 *     kind: missing, extra, resized, block (a primary path's block), hardlink (a hard-linked path's block), unreadable,
 *     table, dir (the last two with path "."); got / want: 16 lower-case hex digits (block and hardlink only).  In paths
 *     '\' is "\\", tab "\t", newline "\n" and any other byte below 0x20 "\xHH".  Written like a table: tmp, fsync,
 *     rename; an empty file when nothing was found.
 *   - Control: vmig_opts.ctl as for the tree calls; phases WALK, DATA, DONE; bytes_total is bytes_unique and
 *     bytes_hashed counts unique bytes.  stats (nullable): the vmig_stats of the data pass (bytes_h2d == bytes_unique,
 *     bytes_total / blocks_total / files: the distinct inodes).
 * Directories, symlinks, specials and metadata are not in the tables and are not checked, as for restore.  The walk flag
 * VMIG_F_SKIP_HIDDEN_TOPDIRS must be the one the snapshots were taken with. */
int vmig_scrub_store(uint32_t n, const char* const* snap_dirs, const char* const* snap_tables,
                     const char* report_path /*nullable*/, int32_t* verdicts /*n, nullable*/,
                     const vmig_opts* opts /*nullable*/, vmig_stats* stats /*nullable*/,
                     vmig_scrub_stats* scrub_stats /*nullable*/);

/* Retirement of old versions of a snapshot store: what vmig_retire_versions removed and re-recorded. */
typedef struct vmig_retire_stats {
    uint64_t versions_retired;             /* retired snapshot directories gone at the end (already missing counts)   */
    uint64_t entries_removed;              /* directory entries this call unlinked or rmdir'ed under them             */
    uint64_t files_freed, bytes_freed;     /* regular files whose link count was 1 when this call unlinked them        */
    uint64_t records_stale;                /* kept-table records found stale after the removal                        */
    uint64_t records_restamped;            /* of those: re-verified on the GPU and re-recorded                        */
    uint64_t bytes_rehashed;               /* distinct inodes read through the GPU to do so                           */
    uint64_t tables_rewritten;
    uint64_t reserved[4];
} vmig_retire_stats;

/* Remove the n_retire versions retire_dirs[i] (with their tables retire_tables[i]) of a snapshot store, and keep the
 * n_keep versions keep_dirs[i] / keep_tables[i] usable as bases for the next incremental snapshot.
 * Unlinking one hard link of an inode moves the inode's ctime, so removing a version by hand (rm -rf) leaves stale the
 * kept tables' records of nearly every file it shared with them: the next vmig_snapshot_tree no longer trusts them and
 * copies those files in full.  This call removes the versions, then re-verifies exactly the records whose identity went
 * stale and re-records them.
 *   - Refusals that touch nothing: VMIG_EINVAL for n_retire + n_keep == 0, a NULL array or entry, flags other than
 *     VMIG_F_DIRECT_IO | VMIG_F_SKIP_HIDDEN_TOPDIRS, bad block_bytes, any two directories of the call that are the same
 *     or one inside the other (compared by real path), a retired table that is a kept table or lies inside a kept
 *     directory, and a kept table that lies inside a retired directory.  VMIG_ENOTDIR: a retired directory that exists
 *     but is not a directory (a symlink included: it is never followed), or a kept directory that is missing or not a
 *     directory.  A control cancelled before the call starts: VMIG_ECANCELED.  VMIG_ETABLE: a kept table that does not
 *     load (formats 01 and 02) or whose block_bytes differs from the call's.  VMIG_ENOGPU, checked after the tables.
 *   - Removal (phase UNLINK), one retired version at a time: first its table is unlinked, so a half-removed version is
 *     never a base or a restore source again; then its tree, children first, each entry by its parent's descriptor,
 *     never following a symlink (as VMIG_F_PRUNE removes); last the directory itself.  A missing table or directory is
 *     not an error, so re-running a call that failed part way finishes the job.  files_freed / bytes_freed count the
 *     regular files whose st_nlink was 1 just before this call unlinked them: a link held anywhere else keeps its
 *     inode and is not counted.
 *   - Stale records (phase WALK): every record of every kept table that carries an identity (ino != 0) is opened
 *     beneath its version's directory (no symlink followed) and fstat'ed.  It is stale when the file is still a regular
 *     file with the recorded inode and size but another ctime.  The rule does not depend on what this call unlinked: it
 *     also covers a re-run after a failed or cancelled call, and records earlier snapshots' links had already left
 *     stale.  Records of another inode or size, format-01 records and records without an identity are left alone.
 *   - Re-verify (phase DATA): the stale records are grouped by (st_dev, st_ino) and each distinct inode is read once
 *     through the block pipeline in hash-only mode, as vmig_scrub_store reads (lanes, GPUs and VMIG_F_DIRECT_IO as
 *     there).  Then each inode is fstat'ed again.  A record is re-stamped with the identity seen before the read only
 *     when every one of its blocks hashes as its table says and the ctime did not move during the read.  Any other
 *     stale record stays exactly as it was (a mismatch, an unreadable inode, a ctime that moved): untrusted, which is
 *     the state rm -rf leaves.  An inode that is no longer the one planned (other inode, type or size, or shorter than
 *     its blocks) fails the call with VMIG_ESRCCHANGED.
 *   - Tables (phase TABLE): each kept table with at least one re-stamped record is rewritten atomically (tmp, fsync,
 *     rename).  Only the ino / ctime_ns fields of re-stamped records change; every other byte is identical.  No other
 *     table is touched.
 *   - Failure and cancel: a cancel is honoured in every phase (per removed entry, in the data pass, before each table
 *     rename).  After any failure each kept table is byte-identical to what it was or already fully rewritten, never
 *     half written, and never carries an identity that was not verified; a retired version is intact, gone, or half
 *     removed with its table already gone.  The call never writes into a kept version's tree: nothing there moves
 *     except the ctimes its own unlinks move.
 *   - Control: phases UNLINK, WALK, DATA, TABLE, DONE; bytes_total is the stale bytes to re-hash.  stats (nullable):
 *     the vmig_stats of the data pass.  retire_stats (nullable): the counters above, written on success.
 * A snapshot that uses a kept version as its base must not run concurrently with a retire of the same store: if one
 * does, it fails with VMIG_ESRCCHANGED or copies more than it needed to, but it is never wrong. */
int vmig_retire_versions(uint32_t n_retire, const char* const* retire_dirs, const char* const* retire_tables,
                         uint32_t n_keep, const char* const* keep_dirs, const char* const* keep_tables,
                         const vmig_opts* opts /*nullable*/, vmig_stats* stats /*nullable*/,
                         vmig_retire_stats* retire_stats /*nullable*/);

/* Comparison of a layer with a version snapshot: what vmig_compare_snapshot found and read. */
typedef struct vmig_compare_stats {
    uint64_t paths_added, paths_removed;   /* entries only in the layer / only in the snapshot (each path beneath counts) */
    uint64_t paths_changed;                /* paths in both trees with at least one finding                            */
    uint64_t files_changed;                /* regular file in both trees with a `resized` or `block` finding          */
    uint64_t blocks_changed;               /* `block` findings                                                          */
    uint64_t bytes_restore;                /* snapshot bytes a rollback must bring back (rule below)                   */
    uint64_t files_read, bytes_read;       /* distinct layer inodes hashed through the GPU                              */
    uint64_t files_trusted;                /* layer paths whose hashes came from layer_table, not from a read           */
    uint64_t files_shared;                 /* layer paths that are the snapshot path's own inode: not read              */
    uint64_t reserved[4];
} vmig_compare_stats;

/* List every difference between the layer layer_dir and the version snapshot snap_dir (written with its block table
 * snap_table by vmig_snapshot_tree): everything vmig_restore_tree(snap_dir, snap_table, layer_dir, ..., VMIG_F_PRUNE |
 * flags) would change -- entry type, permission bits, owner, mtime, symlink target, device numbers, hard-link grouping
 * inside the tree and regular-file contents.  It previews a checked rollback.  Nothing is written anywhere except
 * report_path, and no inode's ctime moves (in either tree or table), so every identity the next incremental snapshot
 * or diff pass trusts stays valid.
 *   - Refusals, in this order, each before anything is read or written: VMIG_EINVAL (layer_dir, snap_dir or snap_table
 *     NULL or empty; flags other than VMIG_F_DIRECT_IO | VMIG_F_SKIP_HIDDEN_TOPDIRS | VMIG_F_MTIME_NS |
 *     VMIG_F_NO_METADATA; bad block_bytes); a control cancelled before the call: VMIG_ECANCELED; VMIG_ENOTDIR (either
 *     directory missing or not a directory); VMIG_ETABLE (either table does not load -- formats 01 and 02 -- or its
 *     block_bytes differs from the call's); VMIG_ENOGPU (no CPU fallback, even when no layer file needs reading).
 *   - Snapshot side: snap_dir is walked for metadata only and must match snap_table in paths and sizes, as a restore
 *     requires at plan time; otherwise VMIG_ECORRUPT with the restore's message, and no report.  None of its file data
 *     is read: its regular-file contents are taken to be its table's hashes.  A snapshot whose bytes rotted without a
 *     change in size compares as its table says; finding that is vmig_scrub_store's job.
 *   - Layer side: layer_dir is walked as a migration's source (no symlink followed).  A layer regular file needs its
 *     block hashes when it and the snapshot's regular file at the same path both have at least one block, and takes
 *     them from the first of these that applies:
 *       shared   the layer path is the snapshot path's own inode (same st_dev, st_ino and size), as versions of one
 *                incremental store share inodes: equal by construction, not read (files_shared);
 *       trusted  layer_table (nullable) records the path and the file is still that record's inode, size and ctime --
 *                the in-place diff path's trust rule: not read (files_trusted);
 *       read     otherwise: each distinct inode read once through the block pipeline in hash-only mode, lanes, GPUs and
 *                VMIG_F_DIRECT_IO as in vmig_scrub_store (files_read, bytes_read).  An inode that is no longer the walked
 *                one (other inode, type or size, or shorter than its blocks) is VMIG_ESRCCHANGED; one that cannot be
 *                opened or read is VMIG_EIO.
 *     Files only in the layer are never read.  The block comparison is one 8-byte compare per block on the host.
 *   - Both walks take the call's VMIG_F_SKIP_HIDDEN_TOPDIRS.  Sockets are skipped, as everywhere in the engine; xattrs
 *     are not compared, as the engine drops them.
 *   - report_path (nullable): one line per finding, sorted by path (bytewise), then kind in the order below, then block:
 *       <kind>\t<path>\t<block|->\t<layer|->\t<snap|->\n
 *     added     the path is only in the layer (every entry beneath an added directory is listed too)        - / -
 *     removed   the path is only in the snapshot (likewise)                                                - / -
 *     type      both have the path, as different S_IFMT                                one letter each of f d l c b p
 *     resized   regular in both, different sizes                                                   decimal sizes
 *     block     regular in both; block r is below both block counts and its (length, XXH64) differs   16 hex digits
 *     target    symlink in both, different targets                                               escaped targets
 *     rdev      char or block device in both, different device numbers                                major:minor
 *     hardlink  regular in both; the set of other paths of the same tree sharing its inode differs (a link held
 *               outside a tree does not count)          the group's smallest path in each tree, "-" when alone
 *     mode      same type in both, different permission bits (07777)                          four octal digits
 *     owner     same type in both, different uid or gid                                                 uid:gid
 *     mtime     same type in both, different mtime: whole seconds (tar's precision, and what a default snapshot
 *               keeps), nanoseconds with VMIG_F_MTIME_NS                                   sec or sec.nnnnnnnnn
 *     With VMIG_F_NO_METADATA mode, owner and mtime are not compared.  The root is path "." and takes only mode,
 *     owner and mtime findings.  Paths and targets are escaped as in the vmig_scrub_store report.  Written like a
 *     table: tmp, fsync, rename; an empty file when there is no difference.  A failed or cancelled call leaves
 *     report_path as it was, with no .tmp beside it.
 *   - bytes_restore, summed over the snapshot's regular-file paths (each path of a hard-link group once): where the
 *     layer has a regular file at the path, the snapshot lengths of the blocks past the layer file's last block or
 *     whose (length, hash) differs; otherwise the snapshot file's whole size.  It is the content a rollback has to
 *     bring back: vmig_rollback_layer reads exactly this from the snapshot (its bytes_fetched), less what this sum
 *     counts for the second and later paths of a snapshot hard-link group, which the rollback links to the group's
 *     first path instead of reading them.  vmig_restore_tree reads the whole snapshot.
 *   - Control: vmig_opts.ctl as for the tree calls; phases WALK, DATA, DONE; a cancel is honoured per directory of the
 *     walks, in the block pipeline and before the report is renamed into place.  bytes_total / blocks_total are the
 *     bytes and blocks to be read.  stats (nullable): the vmig_stats of the data pass (bytes_h2d == bytes_read, 0 when
 *     nothing needs reading).  cmp_stats (nullable): the counters above, written on success. */
int vmig_compare_snapshot(const char* layer_dir, const char* layer_table /*nullable*/,
                          const char* snap_dir, const char* snap_table,
                          const char* report_path /*nullable*/,
                          const vmig_opts* opts /*nullable*/, vmig_stats* stats /*nullable*/,
                          vmig_compare_stats* cmp_stats /*nullable*/);

/* An in-place rollback of a layer to a version snapshot: what vmig_rollback_layer did and read. */
typedef struct vmig_rollback_stats {
    uint64_t files_kept;            /* regular files whose size and every block already were the snapshot's: not written   */
    uint64_t files_patched;         /* written in place: only the differing blocks, then cut or grown to the snapshot's size */
    uint64_t files_rebuilt;         /* replaced by a new inode: blocks the old inode held copied from it, the rest fetched  */
    uint64_t files_created;         /* no usable regular file at the path: fetched from the snapshot in full                */
    uint64_t blocks_fetched, bytes_fetched;   /* snapshot blocks read and checked on the GPU                                */
    uint64_t files_trusted;         /* layer files whose hashes came from layer_table                                       */
    uint64_t files_read, bytes_read;          /* distinct layer inodes hashed on the GPU                                    */
    uint64_t bytes_copied;          /* rebuilt files' bytes copied from their old inode (copy_file_range)                   */
    uint64_t reserved[4];
} vmig_rollback_stats;

/* Roll the layer layer_dir back to the version snapshot snap_dir (written with its block table snap_table by
 * vmig_snapshot_tree) in place, reading from the snapshot only the blocks the layer does not already hold.  Its cost is
 * the difference between the layer and the version -- the layer bytes that have to be hashed (none that layer_table
 * still vouches for) plus vmig_compare_snapshot's bytes_restore -- where vmig_restore_tree reads the whole version.
 *   - Result: on success layer_dir is what vmig_restore_tree(snap_dir, snap_table, layer_dir, NULL, out_table,
 *     flags | VMIG_F_PRUNE) leaves: entries, types, contents, permission bits, owners, mtimes (whole seconds, or ns with
 *     VMIG_F_MTIME_NS), symlink targets, device numbers and in-tree hard-link grouping.  The call always prunes;
 *     VMIG_F_PRUNE is accepted and changes nothing.
 *   - Refusals, in this order, each before anything is read or written: VMIG_EINVAL (layer_dir, snap_dir or snap_table
 *     NULL or empty; flags other than VMIG_F_DIRECT_IO | VMIG_F_SKIP_HIDDEN_TOPDIRS | VMIG_F_MTIME_NS |
 *     VMIG_F_NO_METADATA | VMIG_F_VERIFY | VMIG_F_PRUNE; bad block_bytes; layer_dir and snap_dir the same directory or
 *     one inside the other, by real path; out_table equal to snap_table or inside snap_dir -- out_table == layer_table
 *     is allowed, it is how a hand-off's table is carried forward); a control cancelled before the call:
 *     VMIG_ECANCELED; VMIG_ENOTDIR (either directory missing or not a directory); VMIG_ETABLE (either table does not
 *     load, or its block_bytes differs from the call's); VMIG_ENOGPU (no CPU fallback, even when nothing needs reading).
 *   - Snapshot side: snap_dir is walked for metadata and must match snap_table in paths and sizes before the layer is
 *     touched (VMIG_ECORRUPT with the restore's message otherwise).  Then the layer is pruned as a pruning restore
 *     prunes it, and walked.
 *   - Layer hashes: exactly vmig_compare_snapshot's sources -- the snapshot path's own inode (shared), a record of
 *     layer_table the file still is (trusted), or one hash-only read per distinct inode through the GPU (files_read,
 *     bytes_read).  The identity each speaks for (a trusted file's record; otherwise an lstat taken before the read)
 *     must still be what an lstat shows after the read, or the call fails with VMIG_ESRCCHANGED.
 *   - One action per snapshot regular file (a hard-link group's first path; the others are linked to it afterwards):
 *       keep     the layer file at the path is patchable, has the same size and every (length, XXH64) equal: nothing is
 *                read or written; its metadata is replayed only where it differs, so its ctime and identity stay;
 *       patch    patchable and something differs: the file is set to the snapshot's size, then the differing blocks --
 *                and every block past the layer file's old end -- are fetched and written in place.  Patchable: a
 *                regular file whose hashes came from a trusted record or a read (not a shared inode), with one link,
 *                writable by the caller (root, or the owner with S_IWUSR: a read-only file is replaced, as tar replaces
 *                it), and neither path is in a hard-link group;
 *       rebuild  a regular file that is not patchable (an inode shared with the snapshot -- a restore never lets a layer
 *                share an inode with the store --, a link held outside the tree, a hard-link group): the old inode is
 *                opened, the path replaced by a new file, the blocks equal at the same index copied from the old inode
 *                in coalesced runs (copy_file_range), the rest fetched (the old inode is opened for reading only when
 *                something is copied from it);
 *       create   no regular file at the path: every block is fetched.
 *     The match is positional (same path, same block index), as vmig_compare_snapshot's.
 *   - Before the first write into a patched file and before copying from a rebuilt file's old inode, the open
 *     descriptor's inode, size and ctime must be the ones the plan trusted, else VMIG_ESRCCHANGED naming the path.  The
 *     call's own unlink of another path of a rebuilt inode (a layer hard-link group the snapshot holds as separate
 *     files) moves its ctime too; that change, and only that, is allowed for.  The
 *     layer must not be in use (as for vmig_restore_paths).
 *   - What is checked: every fetched block is hashed by K1 against snap_table, as a restore checks it, and a mismatch is
 *     VMIG_ECORRUPT before any block of its batch is written.  Snapshot blocks that are not fetched are not read: the
 *     layer already holds bytes with the table's hash.  A rotted snapshot block the layer does not need therefore
 *     neither fails the call nor reaches the layer; finding it is vmig_scrub_store's job.
 *   - The store is only read: nothing is written under snap_dir.  After success no layer regular file shares an inode
 *     with a snapshot file.  Replacing a layer path that was a hard link to a snapshot inode unlinks it, which moves
 *     that inode's ctime as every unlink does (its table record then no longer vouches for it, so the next snapshot
 *     based on that version re-reads it); no other snapshot inode's ctime moves.
 *   - VMIG_F_VERIFY: every regular file of the layer is re-read through the GPU and must hash as snap_table says, then
 *     the layer's entry set must be the snapshot's (the pruning restore's check).
 *   - out_table (nullable): the restore's out table -- snap_table's paths, sizes and hashes, and the identities of the
 *     layer files as the call leaves them.  Handed back as layer_table it vouches for every file.
 *   - Control: vmig_opts.ctl as for the tree calls; phases WALK, PRUNE, DATA (the layer's hash pass, then the fetch
 *     pass), META, (VERIFY), TABLE, DONE.  bytes_total / blocks_total are the layer bytes to hash plus the snapshot
 *     bytes to fetch.  A cancel is honoured per directory of the walks, per entry of the prune, in both block
 *     pipeline passes, per <= 64 MiB chunk of a rebuilt file's copy, per <= 1024 metadata entries and before the table
 *     is renamed into place.  A failed or cancelled call leaves what a failed restore leaves: no out_table and no .tmp,
 *     both tables and the snapshot untouched, the layer possibly partly written but never with a block that failed a
 *     check; a file patched part way carries a moved ctime, so the next pass copies it in full.
 *   - stats (nullable): the vmig_stats of both passes (bytes_h2d == bytes_read + bytes_fetched, plus the re-read with
 *     VMIG_F_VERIFY).  rb_stats (nullable): the counters above, written on success.  On the same layer state with the
 *     same layer_table, files_read and bytes_read equal vmig_compare_snapshot's, and bytes_fetched equals its
 *     bytes_restore less the second and later paths of snapshot hard-link groups.  One exception to the first: the
 *     prune runs before the layer's trust is taken, so a file layer_table vouches for whose extra hard link the prune
 *     removes has a moved ctime and is read, where a compare of the state before the call trusts it. */
int vmig_rollback_layer(const char* layer_dir, const char* layer_table /*nullable*/,
                        const char* snap_dir, const char* snap_table, const char* out_table /*nullable*/,
                        const vmig_opts* opts /*nullable*/, vmig_stats* stats /*nullable*/,
                        vmig_rollback_stats* rb_stats /*nullable*/);

/* A version snapshot taken through the layer's own block table: what vmig_snapshot_layer took from the base and read. */
typedef struct vmig_layer_snapshot_stats {
    uint64_t files_linked, bytes_linked;          /* as vmig_snapshot_stats                                              */
    uint64_t files_backfilled, bytes_backfilled;
    uint64_t files_base_untrusted;
    uint64_t files_trusted, bytes_trusted;        /* layer files whose hashes came from layer_table                      */
    uint64_t files_read, bytes_read;              /* layer files with >= 1 block read; layer bytes read (H2D)            */
    uint64_t reserved[4];
} vmig_layer_snapshot_stats;

/* Write the version snapshot of the layer layer_dir that vmig_snapshot_tree(layer_dir, dst_dir, base_dir, base_table,
 * out_table, ...) writes, reading from the layer only the blocks the base does not already hold.  layer_table is the
 * block table written for the layer's files (vmig_migrate_tree into the layer, or vmig_rollback_layer's out_table); the
 * hashes of a file it still vouches for are taken from it instead of from a read.  Its cost is what changed in the
 * layer since that table was written, where vmig_snapshot_tree reads the whole layer.
 *   - Result: compared with the snapshot vmig_snapshot_tree writes with the same arguments and flags, these are equal:
 *     the tree (entry kinds, contents, permission bits, owners, mtimes, symlink targets, device numbers, in-tree
 *     hard-link grouping); which paths are hard links to which base inode; the bytes backfilled; and out_table's paths,
 *     sizes and hashes.  Inode identities differ only where a file is a new inode.  Why: the blocks vmig_snapshot_tree
 *     does not write are exactly those whose (XXH64, length) is among the blocks of the trusted base files (a same-path
 *     match is one of them, since only a trusted base file is compared by path), so taking the hashes from a record
 *     that still describes the file yields the same skipped blocks, and so the same links and backfills, without a read.
 *   - Layer side: a layer regular file is trusted when layer_table records it with an inode and it is still the walked
 *     regular file with that record's inode, size and ctime (the in-place diff path's rule).  Format-01 tables,
 *     hard-linked paths (no identity) and a table written for another directory trust nothing.  Of a trusted file, a
 *     block whose recorded (XXH64, length) a trusted base file holds is not read; every other block is read through the
 *     block pipeline and K1's hash must equal the record's before its batch is written, else VMIG_ESRCCHANGED naming the
 *     path and block.  A trusted file with no block to read is linked or backfilled from the base without entering the
 *     pipeline.  An untrusted file is read and handled exactly as vmig_snapshot_tree handles it.  After the data pass
 *     every trusted file must still be its record (lstat), else VMIG_ESRCCHANGED.  Nothing under layer_dir is written
 *     and no layer ctime moves.  The layer must not be in use, as for vmig_rollback_layer.
 *   - VMIG_F_VERIFY re-reads every snapshot file this call wrote from the ring or backfilled, and not the files it
 *     linked -- the one place where this call deliberately differs from vmig_snapshot_tree.  A linked path's hashes in
 *     out_table are the base table's record of that same inode, so the new table claims nothing the base table did not;
 *     re-reading them would put the whole layer back into the call's cost.  Rot in shared inodes is vmig_scrub_store's
 *     job, as it is for the snapshot blocks vmig_compare_snapshot and vmig_rollback_layer do not read.
 *   - Refusals, in this order, each before anything is read or written: VMIG_EINVAL (any of the six paths NULL or
 *     empty; flags other than VMIG_F_VERIFY | VMIG_F_PRUNE | VMIG_F_DIRECT_IO | VMIG_F_MTIME_NS | VMIG_F_NO_METADATA |
 *     VMIG_F_SKIP_HIDDEN_TOPDIRS; bad block_bytes; two of dst_dir, base_dir and layer_dir the same directory or one
 *     inside the other, by real path; out_table equal to base_table, or inside base_dir or layer_dir -- out_table ==
 *     layer_table is allowed, it is one blocks.vmig in the hand-off layout); a control cancelled before the call:
 *     VMIG_ECANCELED; VMIG_ENOTDIR (any of the three directories missing or not a directory); VMIG_ETABLE (either table
 *     does not load, or its block_bytes differs from the call's); VMIG_ENOGPU (no CPU fallback, even when nothing needs
 *     reading).
 *   - Control: vmig_opts.ctl as for the tree calls; phases WALK, (PRUNE), DATA, META, (VERIFY), TABLE, DONE.
 *     bytes_total / blocks_total are the layer bytes and blocks to read.  A cancel is honoured where vmig_snapshot_tree
 *     honours it and per file of the unread trusted files.  A failed or cancelled call leaves what a failed snapshot
 *     leaves: no out_table and no .tmp, both input tables untouched, the layer untouched.
 *   - stats (nullable): as for vmig_snapshot_tree, with bytes_total / blocks_total as above; without VMIG_F_VERIFY,
 *     bytes_h2d == ls_stats.bytes_read.  ls_stats (nullable): the counters above, written on success; the first five
 *     are vmig_snapshot_stats' and equal what vmig_snapshot_tree counts. */
int vmig_snapshot_layer(const char* layer_dir, const char* layer_table,
                        const char* dst_dir, const char* base_dir, const char* base_table,
                        const char* out_table, const vmig_opts* opts /*nullable*/, vmig_stats* stats /*nullable*/,
                        vmig_layer_snapshot_stats* ls_stats /*nullable*/);

/* A migration through the source's own block table: what vmig_migrate_layer trusted, read, verified and recorded. */
typedef struct vmig_layer_migrate_stats {
    uint64_t files_trusted, bytes_trusted;        /* source files whose hashes came from src_table                       */
    uint64_t files_read, bytes_read;              /* source files with >= 1 block read; source bytes read (H2D)          */
    uint64_t files_unread;                        /* trusted files with nothing to read: every block is the prior's      */
    uint64_t files_verified, bytes_verified;      /* VMIG_F_VERIFY: destination files re-read, and their bytes           */
    uint64_t src_recorded, src_unrecorded;        /* src_out_table records with / without an identity                    */
    uint64_t reserved[4];
} vmig_layer_migrate_stats;

/* Migrate src_dir into dst_dir as vmig_migrate_tree(src_dir, dst_dir, prior_table, out_table, ...) does, reading from
 * the source only the blocks the destination does not already hold.  src_table is a block table written for the
 * source's files (src_out_table of an earlier call of this function, typically the hand-off's live pass); the hashes of
 * a file it still vouches for are taken from it instead of from a read.  The paused pass of a hand-off then costs what
 * the tenant changed since the live pass, where vmig_migrate_tree reads the whole layer and VMIG_F_VERIFY re-reads all
 * of the destination.
 *   - Result: with truthful records, dst_dir, out_table's paths, sizes and hashes, and bytes_written equal what
 *     vmig_migrate_tree leaves with the same prior_table and flags (prune, metadata, hard links and kind changes
 *     included).  Why: a block that is not read is one whose source record (XXH64, length) equals the prior record's at
 *     the same index of a destination file the prior table still vouches for; K1 would return that hash, and
 *     vmig_migrate_tree would skip that block too.
 *   - Source side: a source regular file is trusted when src_table records it with an inode, an lstat still shows the
 *     walked inode and size, and it still is its record (inode, size, ctime: the in-place diff path's rule).  Format-01
 *     tables, hard-linked paths and a table written for another directory trust nothing.  Of a trusted file whose
 *     destination prior_table trusts, a block whose recorded (XXH64, length) equals the prior record's at the same index
 *     is neither read nor written; every other block of a trusted file is read and K1 must return the record's hash
 *     before its batch is written, else VMIG_ESRCCHANGED naming the path and block.  A trusted file with nothing to read
 *     is finished (size, metadata) without entering the pipeline.  An untrusted file is handled exactly as
 *     vmig_migrate_tree handles it.  After the data pass every trusted file must still be its record (lstat), else
 *     VMIG_ESRCCHANGED.  Nothing under src_dir is written.
 *   - src_out_table (nullable): out_table's paths, sizes and hashes with the SOURCE files' identities, for the next call
 *     to trust.  The source may be written while it is read, so a read file's identity is recorded only when its fstat
 *     before the first block was read shows a ctime strictly older than a CLOCK_REALTIME_COARSE reading taken just
 *     before that fstat, and an fstat once its last block's hash is back shows the same inode, size and ctime; else the
 *     record carries 0/0 and the next call reads the file (not an error).  A trusted unread file carries its src_table
 *     record forward; hard-linked paths carry 0/0.  The rule is the ctime rule of every table: a write that moves no
 *     ctime (a shared-mmap store on a filesystem that does not stamp it) is invisible to it.
 *   - VMIG_F_VERIFY re-reads every destination file this call created or replaced, wrote a block into, or resized, and
 *     not the files it left alone: those still are their prior record, whose hashes the earlier pass computed (and, in
 *     the hand-off, verified).  This is the one deliberate difference from vmig_migrate_tree.  With VMIG_F_PRUNE the
 *     entry-set check runs as in a migration.
 *   - Refusals, in this order, each before anything is read or written: VMIG_EINVAL (src_dir or dst_dir NULL or empty;
 *     flags other than VMIG_F_VERIFY | VMIG_F_PRUNE | VMIG_F_DIRECT_IO | VMIG_F_MTIME_NS | VMIG_F_NO_METADATA |
 *     VMIG_F_SKIP_HIDDEN_TOPDIRS; bad block_bytes; src_dir and dst_dir the same directory or one inside the other, by
 *     real path; out_table equal to src_out_table; either output table inside src_dir; src_out_table inside dst_dir);
 *     a control cancelled before the call: VMIG_ECANCELED; VMIG_ENOTDIR (either directory missing or not a directory);
 *     VMIG_ETABLE (src_table or prior_table given and does not load, or its block_bytes differs from the call's);
 *     VMIG_ENOGPU (no CPU fallback, even when nothing needs reading).
 *   - Control: vmig_opts.ctl as for the tree calls; phases WALK, (PRUNE), DATA, META, (VERIFY), TABLE, DONE.
 *     bytes_total / blocks_total are the source bytes and blocks to read.  A cancel is honoured where vmig_migrate_tree
 *     honours it and per unread trusted file.  A failed or cancelled call leaves no new out_table or src_out_table and no
 *     .tmp of either; src_table and prior_table are left byte-identical.
 *   - stats (nullable): as for vmig_migrate_tree, with bytes_total / blocks_total as above; without VMIG_F_VERIFY,
 *     bytes_h2d == lm_stats.bytes_read.  lm_stats (nullable): the counters above, written on success. */
int vmig_migrate_layer(const char* src_dir, const char* src_table /*nullable*/,
                       const char* dst_dir, const char* prior_table /*nullable*/,
                       const char* out_table /*nullable*/, const char* src_out_table /*nullable*/,
                       const vmig_opts* opts /*nullable*/, vmig_stats* stats /*nullable*/,
                       vmig_layer_migrate_stats* lm_stats /*nullable*/);

/* utils.CopyDir(src, dest) (reference utils/copy.go:21-27) == vmig_migrate_tree with defaults. */
int vmig_copy_dir(const char* src_dir, const char* dst_dir);

/* moveVolumeData(src, dest) on resolved host paths (reference utils/copy.go:74-128): copy, re-read the
 * destination through the GPU and require it to hash like the source (VMIG_F_VERIFY), syncfs the destination,
 * and only then unlink the source entries; nanosecond mtimes; synchronous, exit status checked.
 * Divergence from `mv`: sockets are skipped and stay in the source (tar skips them too; a listening socket's
 * inode means nothing in another volume). */
int vmig_move_dir(const char* src_dir, const char* dst_dir);

/* Host buffer -> host buffer through the same pipeline (H2D, hash, diff, D2H of survivors).
 * n_blocks = ceil(nbytes / block_bytes).  prior_hashes/prior_valid nullable (all blocks survive);
 * out_hashes nullable.  dst regions of skipped blocks are left untouched.  Buffers allocated by
 * vmig_host_alloc (or cudaHostRegister'ed by the caller) are DMA'd directly. */
int vmig_migrate_buffer(const void* src, void* dst, uint64_t nbytes,
                        const uint64_t* prior_hashes, const uint8_t* prior_valid,
                        uint64_t* out_hashes, const vmig_opts* opts, vmig_stats* stats);
int  vmig_host_alloc(void** p, uint64_t nbytes);   /* pinned host memory                        */
void vmig_host_free(void* p);

/* ---- cancellation and progress ------------------------------------------------------------------
 * A control is a numeric id (cgo passes it in vmig_opts.ctl without any pointer rules).  It serves the entry points
 * that take vmig_opts: vmig_migrate_tree, vmig_restore_tree, vmig_restore_paths, vmig_snapshot_tree, vmig_scrub_store, vmig_retire_versions, vmig_compare_snapshot, vmig_rollback_layer, vmig_snapshot_layer, vmig_migrate_layer and vmig_migrate_buffer (a caller that
 * wants to cancel a copy or a move calls vmig_migrate_tree with the flags vmig_copy_dir / vmig_move_dir use).  One
 * control serves one call at a time: attaching it to a second concurrent call fails with VMIG_EINVAL.  The engine has
 * no deadline of its own; a deadline is the caller's timer calling vmig_ctl_cancel.
 *   - A control cancelled before the call starts: the call returns VMIG_ECANCELED right after argument validation,
 *     before the GPU check and before the destination, the tables or the base are touched.  A cancel is never undone.
 *   - After a cancel no new work is issued: no read, H2D copy, kernel launch, D2H copy, write, link, backfill chunk or
 *     metadata step starts.  Work already issued finishes (at most one read or write task per copy thread -- <= 1 MiB
 *     or 64 blocks -- plus what is enqueued on the slot streams), then the call returns VMIG_ECANCELED and
 *     vmig_last_error() names the phase it stopped in.  A cancel latches like any other first error: a real error that
 *     happened first keeps its own code.  Outside the block pipeline the call checks the control per directory of the
 *     walk, while it waits for a staging pipe, per <= 64 MiB chunk of a snapshot's backfill, per <= 1024 metadata
 *     entries, per entry of VMIG_F_PRUNE, in the VMIG_F_VERIFY re-read, and before the table is renamed into place.
 *   - A cancelled call gives the guarantees of any failed call: no out_table (and no .tmp of it); prior_table,
 *     snap_table and base_table untouched; the base snapshot's contents, modes and mtimes unchanged (inode ctimes may
 *     move, as a snapshot's links always move them); the destination possibly partly written, never with a block that
 *     failed a check; a file patched in place part way no longer matches its table's identity, so the next pass
 *     copies it in full.  Every lane thread is joined, the slot streams are synchronised, the pipes are back in the
 *     pool, no descriptor is left open, and the next call succeeds.
 *   - VMIG_F_MOVE_SRC: a cancel is honoured up to the first unlink of the source (phase VMIG_PHASE_UNLINK).  From then
 *     on the move runs to completion and returns VMIG_OK: the source is either intact or the move is complete.
 *   - Progress: the counters never decrease during a call and start from zero each time the control is attached.
 *     After a successful call bytes_total, blocks_total and bytes_written equal vmig_stats' fields of the same name,
 *     and bytes_hashed + bytes_verified equals vmig_stats.bytes_h2d.  The phases of a tree call follow the order
 *     WALK, (PRUNE), DATA, META, (VERIFY), TABLE, (UNLINK), DONE; a call that fails keeps the phase it stopped in. */
#define VMIG_PHASE_IDLE    0u   /* attached to no call yet                                                  */
#define VMIG_PHASE_WALK    1u   /* reading the source tree's metadata                                       */
#define VMIG_PHASE_DATA    2u   /* the block pipeline (read, hash, diff, write; a snapshot's backfill)     */
#define VMIG_PHASE_VERIFY  3u   /* VMIG_F_VERIFY: re-reading the destination through the GPU                */
#define VMIG_PHASE_META    4u   /* empty files, symlinks, specials, hard links, directory metadata          */
#define VMIG_PHASE_PRUNE   5u   /* VMIG_F_PRUNE: removing destination entries the source does not have      */
#define VMIG_PHASE_TABLE   6u   /* writing out_table                                                        */
#define VMIG_PHASE_UNLINK  7u   /* VMIG_F_MOVE_SRC: unlinking the source; a cancel is no longer honoured.
                                   vmig_retire_versions: removing retired versions; a cancel is honoured   */
#define VMIG_PHASE_DONE    8u   /* the call returned VMIG_OK                                                */

typedef struct vmig_progress {
    uint32_t phase;            /* VMIG_PHASE_*                                                              */
    uint32_t running;          /* 1 while a call is attached                                               */
    uint64_t bytes_total, blocks_total;      /* known once the walk is done                                */
    uint64_t bytes_hashed, blocks_hashed;    /* data pass: blocks whose hash is back from the GPU          */
    uint64_t bytes_written;                  /* ring writes so far (the count of vmig_stats.bytes_written) */
    uint64_t bytes_verified;                 /* VMIG_F_VERIFY re-read                                      */
    uint64_t reserved[4];
} vmig_progress;

int vmig_ctl_open(uint32_t* id);                        /* a new control id; ids are never reused within a process */
int vmig_ctl_cancel(uint32_t id);                       /* any thread, any time, idempotent; unknown/closed id: VMIG_EINVAL */
int vmig_ctl_progress(uint32_t id, vmig_progress* out); /* any thread, while a call runs or afterwards              */
int vmig_ctl_close(uint32_t id);                        /* VMIG_EINVAL while a call is still attached              */

/* K1 direct: canonical XXH64(seed 0) of n blocks (host_buf + offs[i], lens[i]); the blocks are
 * staged to HBM at 16-byte-aligned offsets and hashed by the xxh64_blocks kernel.  kernel_ms
 * (nullable) receives the CUDA-event time of the kernel alone. */
int vmig_hash_blocks(int gpu, const void* host_buf, const uint64_t* offs, const uint32_t* lens,
                     uint64_t n, uint64_t* out_hashes, double* kernel_ms);

/* ---- HBM-resident batch (the "block-hash GB/s" metric: inputs already in HBM) --------------- */
typedef struct vmig_resident vmig_resident;
/* n_blocks slots of block_bytes each in one device allocation (+ hash/prior/survivor arrays). */
int  vmig_resident_open(int gpu, uint64_t n_blocks, uint32_t block_bytes, vmig_resident** out);
void vmig_resident_close(vmig_resident* r);
/* Device-side generator: 8-byte word w of block b = SplitMix64 stream `seed` at word index
 * b*(block_bytes/8)+w (the generator of BASELINE.md §3; restated in oracle/).  All lens reset
 * to block_bytes. */
int  vmig_resident_fill(vmig_resident* r, uint64_t seed);
int  vmig_resident_set_len(vmig_resident* r, uint64_t block, uint32_t len);
int  vmig_resident_upload(vmig_resident* r, uint64_t block, const void* host, uint32_t len);
int  vmig_resident_download(vmig_resident* r, uint64_t block, void* host, uint32_t len);
/* XOR the first 8 bytes of each listed block with ~0 (BASELINE.md §3 config 4's mutation). */
int  vmig_resident_flip(vmig_resident* r, const uint64_t* blocks, uint64_t n);
/* prior table for diff_select: hashes (nullable = none valid) + per-block validity bytes. */
int  vmig_resident_set_prior(vmig_resident* r, const uint64_t* hashes, const uint8_t* valid);
/* One pass = xxh64_blocks over all blocks + diff_select (ordered compaction of changed block
 * indices).  Repeats `iters` times back to back; ms_hash / ms_total are CUDA-event times of the
 * LAST iteration's hash kernel / of all iterations together (on the launching stream). */
int  vmig_resident_pass(vmig_resident* r, uint32_t iters, double* ms_hash_last, double* ms_total);
int  vmig_resident_results(vmig_resident* r, uint64_t* hashes /*n_blocks, nullable*/,
                           uint32_t* survivors /*n_blocks cap, nullable*/, uint64_t* n_survivors);

/* ---- host<->HBM link probe (the e2e roofline denominator; BASELINE.md §4) ----------------------------------
 * Pinned-memory cudaMemcpyAsync sweep on GPU `gpu`: `bytes` per direction in 32 MiB pieces out of a NUMA-local
 * page-locked buffer, timed with CUDA events.  gbs[0] = H2D alone, gbs[1] = D2H alone, gbs[2] / gbs[3] = H2D / D2H
 * while both directions run at once (two streams) -- the state the copy-back path of a migration is in.
 * GB/s = 1e9 bytes per second. */
int vmig_link_probe(int gpu, uint64_t bytes, double gbs[4]);

/* What the engine would use on THIS box right now: host reader / writer threads PER LANE for a call of `lanes` lanes on
 * `n_gpus` GPUs (plain copy; has_prior = 1: diff path; flags & VMIG_F_HASH_ONLY: hash-only), given the per-box budget
 * (20 copy threads for one GPU, 13 per GPU beyond, capped by the CPUs), the lanes other calls of this process have in
 * flight, and VMIG_READERS / VMIG_WRITERS / VMIG_IO_SHARE.  No GPU needed; for operators and tests. */
int vmig_thread_plan(uint32_t lanes, uint32_t n_gpus, uint32_t flags, int has_prior, uint32_t* readers, uint32_t* writers);

/* ---- block table + host-side helpers (no GPU needed) ---------------------------------------- */
/* Block-table file, little-endian:
 *   char[8] "VMIGBT02"; u32 block_bytes; u32 algo (1 = XXH64 seed 0); u64 n_files; u64 n_blocks;
 *   n_files x { u32 path_len; char path[path_len] (relative, no leading ./); u64 size;
 *               u64 first_block; u64 ino; i64 ctime_ns } sorted bytewise by path;
 *   u64 hashes[n_blocks].
 * A file of `size` bytes owns ceil(size/block_bytes) consecutive hashes (0 for an empty file).
 * ino/ctime_ns identify the on-disk file the table speaks FOR: the destination file as the migration that wrote
 * the table left it (the source file for a VMIG_F_HASH_ONLY table); 0/0 = unknown.  A later call that is handed
 * the table as prior_table patches a destination file in place -- skipping blocks whose hash matches -- only
 * while the file's inode, ctime and size still equal the record; otherwise (failed or partial earlier pass,
 * out-of-band write, a table that belongs to another directory) that file is copied in full.  Format "VMIGBT01"
 * (no ino/ctime_ns fields) is still read; its files are never patched in place.
 * Home in the reference: merges/<rs>/<rs>-<version>/ (internal/services/replicaset.go:681-704,
 * internal/version/merge.go:16). */
typedef struct vmig_table_info {
    uint32_t block_bytes, algo;
    uint64_t n_files, n_blocks, bytes_total;
} vmig_table_info;
int vmig_table_info_read(const char* path, vmig_table_info* out);
/* Copies up to cap hashes of the table into out; returns VMIG_OK. */
int vmig_table_hashes(const char* path, uint64_t* out, uint64_t cap);
/* Walk src_dir exactly as vmig_migrate_tree would (same ordering, block layout, hard-link grouping,
 * VMIG_F_SKIP_HIDDEN_TOPDIRS) and return the totals in *stats (bytes_total, blocks_total, files, dirs,
 * symlinks, hardlinks, specials); if out_table is non-NULL also write the manifest as a block table
 * whose hashes are all zero.  No GPU involved: this is the single metadata pass that can replace the
 * separate DirSize walk of PatchVolumeSize's shrink check (reference internal/services/volume.go:126-140,
 * SURVEY.md §8f N3). */
int vmig_manifest(const char* src_dir, uint32_t flags, uint32_t block_bytes,
                  const char* out_table /*nullable*/, vmig_stats* stats /*nullable*/);
/* utils.DirSize (reference utils/file.go:13-22): sum of non-directory sizes under dir. */
int vmig_dir_size(const char* dir, int64_t* bytes, uint64_t* n_files);
/* utils.ToBytes (reference utils/file.go:24-48): "20GB" -> 21474836480; 1024-based; KB/MB/GB/TB. */
int vmig_to_bytes(const char* s, int64_t* out);
/* Deterministic synthetic tree (BASELINE.md §3): n_files files of file_bytes each named
 * f%05d.bin under dir, bytes = SplitMix64 stream seeded seed ^ fnv1a64(relative path). */
int vmig_datagen_files(const char* dir, uint64_t seed, uint32_t n_files, uint64_t file_bytes,
                       uint32_t threads);

#ifdef __cplusplus
}
#endif
#endif /* VMIG_H */
