//go:build vmig

package utils

/*
#cgo LDFLAGS: -lvmig -lstdc++ -lpthread -ldl -lrt
#include <stdlib.h>
#include <vmig.h>
*/
import "C"

import (
	"context"
	"fmt"
	"runtime"
	"unsafe"

	"github.com/ngaut/log"
	"github.com/pkg/errors"
)

// vmigErr turns a return code into an error.  vmig_last_error() is thread-local and is read by a SEPARATE cgo call:
// between two cgo calls the Go scheduler may move the goroutine to another OS thread, so every caller below brackets
// "call + vmigErr" with runtime.LockOSThread()/UnlockOSThread() (lockedCall).
func vmigErr(rc C.int, what string) error {
	if rc == 0 {
		return nil
	}
	return errors.Errorf("%s: %s (%d): %s", what, C.GoString(C.vmig_strerror(rc)), int(rc),
		C.GoString(C.vmig_last_error()))
}

// lockedCall runs f (one libvmig call) and fetches its error text on the same OS thread.
func lockedCall(what string, f func() C.int) error {
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	return vmigErr(f(), what)
}

// CopyDir replaces `sh -c "(cd src; tar c .) | (cd dest; tar x)"` (utils/copy.go:17-27).
func CopyDir(src, dest string) error {
	cs, cd := C.CString(src), C.CString(dest)
	defer C.free(unsafe.Pointer(cs))
	defer C.free(unsafe.Pointer(cd))
	return errors.Wrapf(lockedCall("vmig_copy_dir", func() C.int { return C.vmig_copy_dir(cs, cd) }),
		"vmig copy failed, src:%s, dest: %s", src, dest)
}

// CopyDirDiff is CopyDir with the block tables the diff-skip path needs. prior/out are paths
// under the per-version directory setToMergeMap already creates
// (internal/services/replicaset.go:681-704): merges/<rs>/<rs>-<v>/blocks.vmig.
func CopyDirDiff(src, dest, priorTable, outTable string) error {
	return CopyDirDiffContext(context.Background(), src, dest, priorTable, outTable)
}

// CopyDirDiffContext is CopyDirDiff that stops when ctx is done: the engine issues no new work, returns
// VMIG_ECANCELED, and the error wraps ctx.Err().  As after any failure, outTable is not written.
func CopyDirDiffContext(ctx context.Context, src, dest, priorTable, outTable string) error {
	return copyDirDiff(ctx, src, dest, priorTable, outTable, 0)
}

// CopyDirDiffVerified additionally re-reads the destination through the GPU and compares block tables
// (VMIG_F_VERIFY), and removes every destination entry the source no longer has (VMIG_F_PRUNE: a file the tenant
// deleted or renamed since an earlier pass must not reappear), before it reports success: for the pass after which
// the old container is deleted, and for rollbacks onto a seeded layer.
func CopyDirDiffVerified(src, dest, priorTable, outTable string) error {
	return CopyDirDiffVerifiedContext(context.Background(), src, dest, priorTable, outTable)
}

// CopyDirDiffVerifiedContext is CopyDirDiffVerified that stops when ctx is done (see CopyDirDiffContext).
func CopyDirDiffVerifiedContext(ctx context.Context, src, dest, priorTable, outTable string) error {
	return copyDirDiff(ctx, src, dest, priorTable, outTable, C.VMIG_F_VERIFY|C.VMIG_F_PRUNE)
}

// SnapshotDirVerified writes a version snapshot: the copy is re-read through the GPU (VMIG_F_VERIFY) before
// outTable is written, so the table describes what really landed in dest.
func SnapshotDirVerified(src, dest, outTable string) error {
	return SnapshotDirVerifiedContext(context.Background(), src, dest, outTable)
}

// SnapshotDirVerifiedContext is SnapshotDirVerified that stops when ctx is done (see CopyDirDiffContext).
func SnapshotDirVerifiedContext(ctx context.Context, src, dest, outTable string) error {
	return copyDirDiff(ctx, src, dest, "", outTable, C.VMIG_F_VERIFY)
}

// RestoreDirDiffVerified is CopyDirDiffVerified from a snapshot that must still be the tree its own block table
// snapTable describes (vmig_restore_tree): same paths and sizes before dest is touched, every block's hash as it
// passes.  A snapshot without its table (one that failed part way) or one changed since fails with VMIG_ECORRUPT /
// VMIG_ETABLE instead of being restored.
func RestoreDirDiffVerified(snap, snapTable, dest, priorTable, outTable string) error {
	return RestoreDirDiffVerifiedContext(context.Background(), snap, snapTable, dest, priorTable, outTable)
}

// RestoreDirDiffVerifiedContext is RestoreDirDiffVerified that stops when ctx is done (see CopyDirDiffContext);
// the snapshot and its table are untouched either way.
func RestoreDirDiffVerifiedContext(ctx context.Context, snap, snapTable, dest, priorTable, outTable string) error {
	ct := C.CString(snapTable)
	defer C.free(unsafe.Pointer(ct))
	return runDiff(ctx, "vmig_restore_tree", snap, dest, priorTable, outTable, C.VMIG_F_VERIFY|C.VMIG_F_PRUNE,
		func(cs, cd, cp, co *C.char, o *C.vmig_opts, st *C.vmig_stats, _ *C.vmig_snapshot_stats) C.int {
			return C.vmig_restore_tree(cs, ct, cd, cp, co, o, st)
		})
}

// RestorePathsVerified puts the chosen paths (relative to snap, named as snapTable names them) of a snapshot back into
// dest and touches nothing else there but their parent directories (vmig_restore_paths): each regular file is checked
// against snapTable as RestoreDirDiffVerified checks it, the result is re-read through the GPU (VMIG_F_VERIFY), and
// VMIG_F_PRUNE removes extras beneath the chosen directories only.  priorTable is dest's own table (files still as it
// recorded them are patched block by block); no table is written.
func RestorePathsVerified(snap, snapTable, dest, priorTable string, paths []string) error {
	return RestorePathsVerifiedContext(context.Background(), snap, snapTable, dest, priorTable, paths)
}

// RestorePathsVerifiedContext is RestorePathsVerified that stops when ctx is done (see CopyDirDiffContext); the
// snapshot, its table and priorTable are untouched either way.
func RestorePathsVerifiedContext(ctx context.Context, snap, snapTable, dest, priorTable string, paths []string) error {
	n := len(paths)
	if n == 0 {
		return errors.Errorf("RestorePathsVerified: no path to restore")
	}
	ptrSize := C.size_t(unsafe.Sizeof((*C.char)(nil)))
	cpaths := (*[1 << 28]*C.char)(C.malloc(C.size_t(n) * ptrSize))[:n:n] // C memory: cgo forbids Go pointers to Go pointers
	defer C.free(unsafe.Pointer(&cpaths[0]))
	for i := 0; i < n; i++ {
		cpaths[i] = C.CString(paths[i])
		defer C.free(unsafe.Pointer(cpaths[i]))
	}
	ct := C.CString(snapTable)
	defer C.free(unsafe.Pointer(ct))
	return runDiff(ctx, "vmig_restore_paths", snap, dest, priorTable, "", C.VMIG_F_VERIFY|C.VMIG_F_PRUNE,
		func(cs, cd, cp, _ *C.char, o *C.vmig_opts, st *C.vmig_stats, _ *C.vmig_snapshot_stats) C.int {
			return C.vmig_restore_paths(cs, ct, cd, C.uint32_t(n), &cpaths[0], cp, o, st)
		})
}

// SnapshotDirIncrementalVerified is SnapshotDirVerified that shares what did not change with the previous snapshot
// baseDir, taken with baseTable (vmig_snapshot_tree): an unchanged file becomes a hard link to the base's, also when it
// was renamed or moved since, and a changed or copied file takes every block the base holds from the base file that
// holds it, found by block hash.  The re-read (VMIG_F_VERIFY) covers linked files too, so a base
// that rotted without moving its ctime is caught when the snapshot is taken.
func SnapshotDirIncrementalVerified(src, dest, baseDir, baseTable, outTable string) error {
	return SnapshotDirIncrementalVerifiedContext(context.Background(), src, dest, baseDir, baseTable, outTable)
}

// SnapshotDirIncrementalVerifiedContext is SnapshotDirIncrementalVerified that stops when ctx is done (see
// CopyDirDiffContext); the base snapshot's contents, modes and mtimes are unchanged either way.
func SnapshotDirIncrementalVerifiedContext(ctx context.Context, src, dest, baseDir, baseTable, outTable string) error {
	cb, ct := C.CString(baseDir), C.CString(baseTable)
	defer C.free(unsafe.Pointer(cb))
	defer C.free(unsafe.Pointer(ct))
	return runDiff(ctx, "vmig_snapshot_tree", src, dest, "", outTable, C.VMIG_F_VERIFY,
		func(cs, cd, _, co *C.char, o *C.vmig_opts, st *C.vmig_stats, ss *C.vmig_snapshot_stats) C.int {
			return C.vmig_snapshot_tree(cs, cd, cb, ct, co, o, st, ss)
		})
}

// SnapshotDirFromLayerVerified is SnapshotDirIncrementalVerified with the layer's own block table layerTable
// (vmig_snapshot_layer): of a file the table still vouches for, only the blocks the base does not hold are read.  The
// snapshot, its links and its table are the ones SnapshotDirIncrementalVerified writes.  The re-read (VMIG_F_VERIFY)
// covers what was written or backfilled, not what was linked: a linked file's hashes are the base table's own record,
// and rot in shared inodes is ScrubSnapshots' job.  outTable may be layerTable.
func SnapshotDirFromLayerVerified(src, dest, baseDir, baseTable, outTable, layerTable string) error {
	return SnapshotDirFromLayerVerifiedContext(context.Background(), src, dest, baseDir, baseTable, outTable, layerTable)
}

// SnapshotDirFromLayerVerifiedContext is SnapshotDirFromLayerVerified that stops when ctx is done (see
// CopyDirDiffContext); the layer, both tables and the base snapshot's contents are unchanged either way.
func SnapshotDirFromLayerVerifiedContext(ctx context.Context, src, dest, baseDir, baseTable, outTable, layerTable string) error {
	cb, ct, cl := C.CString(baseDir), C.CString(baseTable), C.CString(layerTable)
	defer C.free(unsafe.Pointer(cb))
	defer C.free(unsafe.Pointer(ct))
	defer C.free(unsafe.Pointer(cl))
	return runDiff(ctx, "vmig_snapshot_layer", src, dest, "", outTable, C.VMIG_F_VERIFY,
		func(cs, cd, _, co *C.char, o *C.vmig_opts, st *C.vmig_stats, _ *C.vmig_snapshot_stats) C.int {
			var ls C.vmig_layer_snapshot_stats
			return C.vmig_snapshot_layer(cs, cl, cd, cb, ct, co, o, st, &ls)
		})
}

// CopyDirFromLayerVerified is CopyDirDiffVerified through the source's own block table srcTable (vmig_migrate_layer):
// of a source file srcTable still vouches for, only the blocks that differ from dest's priorTable record at the same
// index are read, and the re-read (VMIG_F_VERIFY) covers only the destination files the call created, wrote into or
// resized.  dest and outTable are what CopyDirDiffVerified leaves.  srcOutTable (may be "") receives outTable's hashes
// with the source files' identities, for the next call's srcTable; a file written while it was read is recorded without
// one.  prune false: no VMIG_F_PRUNE (the hand-off's live pass).  srcTable and priorTable may be "".
func CopyDirFromLayerVerified(src, srcTable, dest, priorTable, outTable, srcOutTable string, prune bool) error {
	return CopyDirFromLayerVerifiedContext(context.Background(), src, srcTable, dest, priorTable, outTable, srcOutTable, prune)
}

// CopyDirFromLayerVerifiedContext is CopyDirFromLayerVerified that stops when ctx is done (see CopyDirDiffContext);
// the source, srcTable and priorTable are untouched either way, and neither outTable nor srcOutTable is written.
func CopyDirFromLayerVerifiedContext(ctx context.Context, src, srcTable, dest, priorTable, outTable, srcOutTable string, prune bool) error {
	var ct, cso *C.char
	if srcTable != "" {
		ct = C.CString(srcTable)
		defer C.free(unsafe.Pointer(ct))
	}
	if srcOutTable != "" {
		cso = C.CString(srcOutTable)
		defer C.free(unsafe.Pointer(cso))
	}
	flags := C.uint32_t(C.VMIG_F_VERIFY)
	if prune {
		flags |= C.VMIG_F_PRUNE
	}
	return runDiff(ctx, "vmig_migrate_layer", src, dest, priorTable, outTable, flags,
		func(cs, cd, cp, co *C.char, o *C.vmig_opts, st *C.vmig_stats, _ *C.vmig_snapshot_stats) C.int {
			var ms C.vmig_layer_migrate_stats
			return C.vmig_migrate_layer(cs, ct, cd, cp, co, cso, o, st, &ms)
		})
}

// ScrubSnapshots checks every snapshot snapDirs[i] against its block table snapTables[i] in one pass that reads each
// inode the snapshots share once (vmig_scrub_store), and writes every finding to report.  verdicts[i] is the VMIG_*
// code a hash-only restore of that snapshot would return (VMIG_OK, VMIG_ECORRUPT, VMIG_ETABLE, VMIG_ENOTDIR); a
// damaged snapshot is a verdict, not an error.  Nothing is written under any snapshot.
func ScrubSnapshots(snapDirs, snapTables []string, report string) ([]int, error) {
	return ScrubSnapshotsContext(context.Background(), snapDirs, snapTables, report)
}

// ScrubSnapshotsContext is ScrubSnapshots that stops when ctx is done (see CopyDirDiffContext); no report is written then.
func ScrubSnapshotsContext(ctx context.Context, snapDirs, snapTables []string, report string) ([]int, error) {
	n := len(snapDirs)
	if n == 0 || len(snapTables) != n {
		return nil, errors.Errorf("ScrubSnapshots: %d directories, %d tables", n, len(snapTables))
	}
	ptrSize := C.size_t(unsafe.Sizeof((*C.char)(nil)))
	cdirs := (*[1 << 28]*C.char)(C.malloc(C.size_t(n) * ptrSize))[:n:n] // C memory: cgo forbids Go pointers to Go pointers
	ctabs := (*[1 << 28]*C.char)(C.malloc(C.size_t(n) * ptrSize))[:n:n]
	defer C.free(unsafe.Pointer(&cdirs[0]))
	defer C.free(unsafe.Pointer(&ctabs[0]))
	for i := 0; i < n; i++ {
		cdirs[i], ctabs[i] = C.CString(snapDirs[i]), C.CString(snapTables[i])
		defer C.free(unsafe.Pointer(cdirs[i]))
		defer C.free(unsafe.Pointer(ctabs[i]))
	}
	var cr *C.char
	if report != "" {
		cr = C.CString(report)
		defer C.free(unsafe.Pointer(cr))
	}
	verdicts := make([]C.int32_t, n)
	var st C.vmig_stats
	var ss C.vmig_scrub_stats
	var o C.vmig_opts
	var id C.uint32_t
	if err := lockedCall("vmig_ctl_open", func() C.int { return C.vmig_ctl_open(&id) }); err != nil {
		return nil, err
	}
	defer C.vmig_ctl_close(id)
	stop := context.AfterFunc(ctx, func() { C.vmig_ctl_cancel(id) })
	defer stop()
	o.ctl = id
	var rc C.int
	err := lockedCall("vmig_scrub_store", func() C.int {
		rc = C.vmig_scrub_store(C.uint32_t(n), &cdirs[0], &ctabs[0], cr, &verdicts[0], &o, &st, &ss)
		return rc
	})
	if rc == C.VMIG_ECANCELED && ctx.Err() != nil {
		return nil, fmt.Errorf("%w: %v", ctx.Err(), err)
	}
	if err != nil {
		return nil, err
	}
	log.Infof("vmig: scrubbed %d snapshots, %d damaged: %d bytes read for %d referenced, %d paths and %d blocks damaged, %d files unreadable",
		uint64(ss.versions), uint64(ss.versions_damaged), uint64(ss.bytes_unique), uint64(ss.bytes_referenced),
		uint64(ss.files_damaged), uint64(ss.blocks_damaged), uint64(ss.files_unreadable))
	out := make([]int, n)
	for i, v := range verdicts {
		out[i] = int(v)
	}
	return out, nil
}

// CompareStats is what CompareWithSnapshot found and read (vmig_compare_stats).
type CompareStats struct {
	PathsAdded, PathsRemoved, PathsChanged, FilesChanged, BlocksChanged uint64
	BytesRestore                                                         uint64 // snapshot bytes a rollback must bring back
	FilesRead, BytesRead, FilesTrusted, FilesShared                      uint64
}

// CompareWithSnapshot lists every difference between the layer and the snapshot snapDir (checked against snapTable)
// in report: everything a rollback of the layer to that snapshot would change (vmig_compare_snapshot).  Nothing else is
// written and no ctime moves.  layerTable ("" for none) is a table of the layer whose records still vouch for their
// files; those files are not read.  The snapshot's file data is never read: its table stands for it.
func CompareWithSnapshot(layer, layerTable, snapDir, snapTable, report string) (CompareStats, error) {
	return CompareWithSnapshotContext(context.Background(), layer, layerTable, snapDir, snapTable, report)
}

// CompareWithSnapshotContext is CompareWithSnapshot that stops when ctx is done (see CopyDirDiffContext); no report is
// written then.
func CompareWithSnapshotContext(ctx context.Context, layer, layerTable, snapDir, snapTable, report string) (CompareStats, error) {
	cl, cs, ct := C.CString(layer), C.CString(snapDir), C.CString(snapTable)
	defer C.free(unsafe.Pointer(cl))
	defer C.free(unsafe.Pointer(cs))
	defer C.free(unsafe.Pointer(ct))
	var clt, cr *C.char
	if layerTable != "" {
		clt = C.CString(layerTable)
		defer C.free(unsafe.Pointer(clt))
	}
	if report != "" {
		cr = C.CString(report)
		defer C.free(unsafe.Pointer(cr))
	}
	var st C.vmig_stats
	var cmp C.vmig_compare_stats
	var o C.vmig_opts
	var id C.uint32_t
	if err := lockedCall("vmig_ctl_open", func() C.int { return C.vmig_ctl_open(&id) }); err != nil {
		return CompareStats{}, err
	}
	defer C.vmig_ctl_close(id)
	stop := context.AfterFunc(ctx, func() { C.vmig_ctl_cancel(id) })
	defer stop()
	o.ctl = id
	var rc C.int
	err := lockedCall("vmig_compare_snapshot", func() C.int {
		rc = C.vmig_compare_snapshot(cl, clt, cs, ct, cr, &o, &st, &cmp)
		return rc
	})
	if rc == C.VMIG_ECANCELED && ctx.Err() != nil {
		return CompareStats{}, fmt.Errorf("%w: %v", ctx.Err(), err)
	}
	if err != nil {
		return CompareStats{}, err
	}
	out := CompareStats{uint64(cmp.paths_added), uint64(cmp.paths_removed), uint64(cmp.paths_changed), uint64(cmp.files_changed),
		uint64(cmp.blocks_changed), uint64(cmp.bytes_restore), uint64(cmp.files_read), uint64(cmp.bytes_read),
		uint64(cmp.files_trusted), uint64(cmp.files_shared)}
	log.Infof("vmig: compared %s with %s: %d added, %d removed, %d changed, %d bytes to restore; %d bytes read, %d files trusted, %d shared",
		layer, snapDir, out.PathsAdded, out.PathsRemoved, out.PathsChanged, out.BytesRestore, out.BytesRead, out.FilesTrusted, out.FilesShared)
	return out, nil
}

// RollbackStats is what RollbackLayer did and read (vmig_rollback_stats).
type RollbackStats struct {
	FilesKept, FilesPatched, FilesRebuilt, FilesCreated uint64
	BlocksFetched, BytesFetched                         uint64 // snapshot blocks read and checked on the GPU
	FilesTrusted, FilesRead, BytesRead                  uint64
	BytesCopied                                         uint64 // rebuilt files' bytes copied from their old inode
}

// RollbackLayer rolls the layer back to the snapshot snapDir (checked against snapTable) in place
// (vmig_rollback_layer): afterwards it is what a verified, pruning restore of the snapshot into it leaves, but only the
// snapshot blocks the layer does not already hold are read.  layerTable ("" for none) is a table of the layer whose
// records still vouch for their files; outTable ("" for none) receives the layer's new table and may be layerTable.
func RollbackLayer(layer, layerTable, snapDir, snapTable, outTable string) (RollbackStats, error) {
	return RollbackLayerContext(context.Background(), layer, layerTable, snapDir, snapTable, outTable)
}

// RollbackLayerContext is RollbackLayer that stops when ctx is done (see CopyDirDiffContext); no out table is written
// then, and the layer may be partly rolled back (never with a block that failed its check).
func RollbackLayerContext(ctx context.Context, layer, layerTable, snapDir, snapTable, outTable string) (RollbackStats, error) {
	cl, cs, ct := C.CString(layer), C.CString(snapDir), C.CString(snapTable)
	defer C.free(unsafe.Pointer(cl))
	defer C.free(unsafe.Pointer(cs))
	defer C.free(unsafe.Pointer(ct))
	var clt, co *C.char
	if layerTable != "" {
		clt = C.CString(layerTable)
		defer C.free(unsafe.Pointer(clt))
	}
	if outTable != "" {
		co = C.CString(outTable)
		defer C.free(unsafe.Pointer(co))
	}
	var st C.vmig_stats
	var rb C.vmig_rollback_stats
	var o C.vmig_opts
	o.flags = C.VMIG_F_VERIFY
	var id C.uint32_t
	if err := lockedCall("vmig_ctl_open", func() C.int { return C.vmig_ctl_open(&id) }); err != nil {
		return RollbackStats{}, err
	}
	defer C.vmig_ctl_close(id)
	stop := context.AfterFunc(ctx, func() { C.vmig_ctl_cancel(id) })
	defer stop()
	o.ctl = id
	var rc C.int
	err := lockedCall("vmig_rollback_layer", func() C.int {
		rc = C.vmig_rollback_layer(cl, clt, cs, ct, co, &o, &st, &rb)
		return rc
	})
	if rc == C.VMIG_ECANCELED && ctx.Err() != nil {
		return RollbackStats{}, fmt.Errorf("%w: %v", ctx.Err(), err)
	}
	if err != nil {
		return RollbackStats{}, err
	}
	out := RollbackStats{uint64(rb.files_kept), uint64(rb.files_patched), uint64(rb.files_rebuilt), uint64(rb.files_created),
		uint64(rb.blocks_fetched), uint64(rb.bytes_fetched), uint64(rb.files_trusted), uint64(rb.files_read), uint64(rb.bytes_read),
		uint64(rb.bytes_copied)}
	log.Infof("vmig: rolled %s back to %s: %d kept, %d patched, %d rebuilt, %d created; %d bytes fetched, %d read, %d copied",
		layer, snapDir, out.FilesKept, out.FilesPatched, out.FilesRebuilt, out.FilesCreated, out.BytesFetched, out.BytesRead, out.BytesCopied)
	return out, nil
}

// RetireSnapshots removes the snapshots retireDirs[i] with their tables retireTables[i] and keeps keepDirs[i] /
// keepTables[i] usable as bases (vmig_retire_versions): each retired table goes first, then its tree, never following
// a symlink; then the kept tables' records whose ctime the removal moved are re-verified on the GPU and re-recorded.
// Nothing is written under a kept snapshot.  A snapshot based on a kept one must not run at the same time.
func RetireSnapshots(retireDirs, retireTables, keepDirs, keepTables []string) error {
	return RetireSnapshotsContext(context.Background(), retireDirs, retireTables, keepDirs, keepTables)
}

// RetireSnapshotsContext is RetireSnapshots that stops when ctx is done (see CopyDirDiffContext).  A retired snapshot is
// then intact, gone, or half removed without its table; each kept table is as it was or fully rewritten.
func RetireSnapshotsContext(ctx context.Context, retireDirs, retireTables, keepDirs, keepTables []string) error {
	nr, nk := len(retireDirs), len(keepDirs)
	if nr+nk == 0 || len(retireTables) != nr || len(keepTables) != nk {
		return errors.Errorf("RetireSnapshots: %d/%d retired directories/tables, %d/%d kept", nr, len(retireTables), nk, len(keepTables))
	}
	ptrSize := C.size_t(unsafe.Sizeof((*C.char)(nil)))
	carr := func(v []string) **C.char { // C memory: cgo forbids Go pointers to Go pointers
		if len(v) == 0 {
			return nil
		}
		a := (*[1 << 28]*C.char)(C.malloc(C.size_t(len(v)) * ptrSize))[:len(v):len(v)]
		for i, s := range v {
			a[i] = C.CString(s)
		}
		return &a[0]
	}
	cfree := func(p **C.char, n int) {
		if p == nil {
			return
		}
		a := (*[1 << 28]*C.char)(unsafe.Pointer(p))[:n:n]
		for i := range a {
			C.free(unsafe.Pointer(a[i]))
		}
		C.free(unsafe.Pointer(p))
	}
	crd, crt, ckd, ckt := carr(retireDirs), carr(retireTables), carr(keepDirs), carr(keepTables)
	defer cfree(crd, nr)
	defer cfree(crt, nr)
	defer cfree(ckd, nk)
	defer cfree(ckt, nk)
	var st C.vmig_stats
	var rs C.vmig_retire_stats
	var o C.vmig_opts
	var id C.uint32_t
	if err := lockedCall("vmig_ctl_open", func() C.int { return C.vmig_ctl_open(&id) }); err != nil {
		return err
	}
	defer C.vmig_ctl_close(id)
	stop := context.AfterFunc(ctx, func() { C.vmig_ctl_cancel(id) })
	defer stop()
	o.ctl = id
	var rc C.int
	err := lockedCall("vmig_retire_versions", func() C.int {
		rc = C.vmig_retire_versions(C.uint32_t(nr), crd, crt, C.uint32_t(nk), ckd, ckt, &o, &st, &rs)
		return rc
	})
	if rc == C.VMIG_ECANCELED && ctx.Err() != nil {
		return fmt.Errorf("%w: %v", ctx.Err(), err)
	}
	if err != nil {
		return err
	}
	log.Infof("vmig: retired %d snapshots (%d entries, %d bytes freed); %d kept records stale, %d re-stamped after re-hashing %d bytes, %d tables rewritten",
		uint64(rs.versions_retired), uint64(rs.entries_removed), uint64(rs.bytes_freed), uint64(rs.records_stale),
		uint64(rs.records_restamped), uint64(rs.bytes_rehashed), uint64(rs.tables_rewritten))
	return nil
}

func copyDirDiff(ctx context.Context, src, dest, priorTable, outTable string, flags C.uint32_t) error {
	return runDiff(ctx, "vmig_migrate_tree", src, dest, priorTable, outTable, flags,
		func(cs, cd, cp, co *C.char, o *C.vmig_opts, st *C.vmig_stats, _ *C.vmig_snapshot_stats) C.int {
			return C.vmig_migrate_tree(cs, cd, cp, co, o, st)
		})
}

// runDiff makes one engine call under a control of its own: context.AfterFunc cancels it when ctx is done (a
// deadline is ctx's timer; the engine has none), and VMIG_ECANCELED comes back as an error that wraps ctx.Err().
func runDiff(ctx context.Context, what, src, dest, priorTable, outTable string, flags C.uint32_t,
	call func(cs, cd, cp, co *C.char, o *C.vmig_opts, st *C.vmig_stats, ss *C.vmig_snapshot_stats) C.int) error {
	cs, cd := C.CString(src), C.CString(dest)
	defer C.free(unsafe.Pointer(cs))
	defer C.free(unsafe.Pointer(cd))
	var cp, co *C.char
	if priorTable != "" {
		cp = C.CString(priorTable)
		defer C.free(unsafe.Pointer(cp))
	}
	if outTable != "" {
		co = C.CString(outTable)
		defer C.free(unsafe.Pointer(co))
	}
	var st C.vmig_stats
	var ss C.vmig_snapshot_stats // filled by vmig_snapshot_tree only
	var o C.vmig_opts            // zero value = defaults (all GPUs, 4 MiB blocks)
	o.flags = flags
	var id C.uint32_t
	if err := lockedCall("vmig_ctl_open", func() C.int { return C.vmig_ctl_open(&id) }); err != nil {
		return err
	}
	defer C.vmig_ctl_close(id) // runs after stop(): the call has returned, nothing is attached any more
	stop := context.AfterFunc(ctx, func() { C.vmig_ctl_cancel(id) })
	defer stop()
	o.ctl = id
	var rc C.int
	err := lockedCall(what, func() C.int { rc = call(cs, cd, cp, co, &o, &st, &ss); return rc })
	if rc == C.VMIG_ECANCELED && ctx.Err() != nil {
		return fmt.Errorf("%w: %v", ctx.Err(), err)
	}
	if err == nil {
		log.Infof("vmig: %d bytes, %d/%d blocks skipped, %d files copied in full (stale table), %d pruned, "+
			"%d files linked to the base snapshot (%d bytes), %d backfilled from it (%d bytes), %d base files stale, %.2f GiB/s",
			uint64(st.bytes_total), uint64(st.blocks_skipped), uint64(st.blocks_total), uint64(st.files_untrusted),
			uint64(st.pruned), uint64(ss.files_linked), uint64(ss.bytes_linked), uint64(ss.files_backfilled),
			uint64(ss.bytes_backfilled), uint64(ss.files_base_untrusted), float64(st.bytes_total)/float64(st.ns_total)*1e9/(1<<30))
	}
	return err
}

// CopyOldMergedToNewContainerMerged (utils/copy.go:31-46): unchanged except for the callee.
// GetContainerMergedLayer (Docker ContainerInspect -> UpperDir, utils/copy.go:48-54) stays in Go.

// CopyOldMountPointToContainerMountPoint replaces moveVolumeData's helper container + `mv`
// (utils/copy.go:74-128): resolve both volume names with GetVolumeMountPoint (utils/copy.go:65-72,
// kept) and move on the host paths, synchronously, with the status checked.
func CopyOldMountPointToContainerMountPoint(oldVolume, newVolume string) error {
	src, err := GetVolumeMountPoint(oldVolume)
	if err != nil {
		return errors.WithMessage(err, "GetVolumeMountPoint failed")
	}
	dst, err := GetVolumeMountPoint(newVolume)
	if err != nil {
		return errors.WithMessage(err, "GetVolumeMountPoint failed")
	}
	cs, cd := C.CString(src), C.CString(dst)
	defer C.free(unsafe.Pointer(cs))
	defer C.free(unsafe.Pointer(cd))
	return errors.WithMessage(lockedCall("vmig_move_dir", func() C.int { return C.vmig_move_dir(cs, cd) }), "moveData failed")
}
