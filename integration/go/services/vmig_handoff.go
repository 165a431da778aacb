//go:build vmig

// vmig_handoff.go -- Go wiring for the "next" rows N1-N3 of SURVEY.md section 8f, on top of the cgo shim in
// utils/copy_vmig.go.  New file: nothing in it exists in the reference; the comments name the reference lines a
// maintainer changes to call it.  NOT COMPILED in this repository's image (no Go toolchain); the engine calls it
// makes are the ones tests/test_gpu.py exercises through the Python mirror gpu-docker-api_b200/handoff.py, which is
// kept line for line with this file (tests/test_gpu.py::test_handoff_*).
package services

/*
#cgo LDFLAGS: -lvmig -lstdc++ -lpthread -ldl -lrt
#include <stdlib.h>
#include <string.h>
#include <vmig.h>
*/
import "C"

import (
	"context"
	stderrors "errors"
	"os"
	"path/filepath"
	"runtime"
	"sort"
	"strconv"
	"strings"
	"time"
	"unsafe"

	"github.com/ngaut/log"
	"github.com/pkg/errors"

	vmap "github.com/mayooot/gpu-docker-api/internal/version"
	"github.com/mayooot/gpu-docker-api/utils"
)

// versionDir is where a ReplicaSet version keeps its artefacts; same rule as setToMergeMap
// (internal/services/replicaset.go:689-692): <cwd>/merges/<rs>/<rs>-<v>.  The snapshot of the diff layer goes
// to <dir>/diff, its block table to <dir>/blocks.vmig.
func versionDir(ctrVersionName string) string {
	cwd, _ := os.Getwd()
	return filepath.Join(cwd, "merges", strings.Split(ctrVersionName, "-")[0], ctrVersionName)
}

func snapshotPaths(ctrVersionName string) (data, table string) {
	d := versionDir(ctrVersionName)
	return filepath.Join(d, "diff"), filepath.Join(d, "blocks.vmig")
}

// N1 -- SnapshotVersion is the body the commented-out block of setToMergeMap (replicaset.go:684-701) was
// meant to have: keep the layer of <rs>-<v> and the XXH64 table of its 4 MiB blocks before the container is
// deleted.  Call it from setToMergeMap in place of the commented utils.CopyDir; ContainerMergeMap keeps
// pointing at versionDir.
func SnapshotVersion(ctrVersionName string) error {
	upper, err := utils.GetContainerMergedLayer(ctrVersionName)
	if err != nil {
		return errors.WithMessagef(err, "utils.GetContainerMergedLayer failed, container: %s", ctrVersionName)
	}
	data, table := snapshotPaths(ctrVersionName)
	if err := os.MkdirAll(data, 0755); err != nil {
		return errors.Wrapf(err, "mkdir %s", data)
	}
	return errors.WithMessagef(utils.SnapshotDirVerified(upper, data, table), "snapshot of %s failed", ctrVersionName)
}

// baseVersion returns the newest earlier version <rs>-<k> (k < v) whose directory holds both diff/ and blocks.vmig.
func baseVersion(ctrVersionName string) (string, bool) {
	rs := strings.Split(ctrVersionName, "-")[0]
	v, err := strconv.Atoi(ctrVersionName[strings.LastIndex(ctrVersionName, "-")+1:])
	if err != nil {
		return "", false
	}
	entries, _ := os.ReadDir(filepath.Dir(versionDir(ctrVersionName)))
	best := -1
	for _, e := range entries {
		k, err := strconv.Atoi(strings.TrimPrefix(e.Name(), rs+"-"))
		if !strings.HasPrefix(e.Name(), rs+"-") || err != nil || k <= best || k >= v {
			continue
		}
		d := filepath.Join(filepath.Dir(versionDir(ctrVersionName)), e.Name())
		if st, err := os.Stat(filepath.Join(d, "diff")); err != nil || !st.IsDir() {
			continue
		}
		if st, err := os.Stat(filepath.Join(d, "blocks.vmig")); err != nil || !st.Mode().IsRegular() {
			continue
		}
		best = k
	}
	if best < 0 {
		return "", false
	}
	return rs + "-" + strconv.Itoa(best), true
}

// N1 -- SnapshotVersionIncremental is what setToMergeMap calls: SnapshotVersion that shares unchanged files and blocks
// with the newest earlier snapshot of the ReplicaSet (a full SnapshotDirVerified when there is none).  That version's
// blocks.vmig may have been written last by HandoffCopy for the container's layer, not for diff/ (a snapshot of it that
// failed part way): the identities it records then name no file under diff/, the engine trusts none of them, and the
// result is a plain verified copy.
func SnapshotVersionIncremental(ctrVersionName string) error {
	upper, err := utils.GetContainerMergedLayer(ctrVersionName)
	if err != nil {
		return errors.WithMessagef(err, "utils.GetContainerMergedLayer failed, container: %s", ctrVersionName)
	}
	data, table := snapshotPaths(ctrVersionName)
	if err := os.MkdirAll(data, 0755); err != nil {
		return errors.Wrapf(err, "mkdir %s", data)
	}
	base, ok := baseVersion(ctrVersionName)
	if !ok {
		return errors.WithMessagef(utils.SnapshotDirVerified(upper, data, table), "snapshot of %s failed", ctrVersionName)
	}
	baseData, baseTable := snapshotPaths(base)
	return errors.WithMessagef(utils.SnapshotDirIncrementalVerified(upper, data, baseData, baseTable, table),
		"snapshot of %s against %s failed", ctrVersionName, base)
}

// N1 -- SnapshotVersionFromLayer is the snapshot SnapshotVersionIncremental writes, at the cost of what the tenant
// changed since the hand-off.  While the version's directory has no diff/ yet, its blocks.vmig is the table HandoffCopy
// (or RollbackInPlace) wrote for the running layer: it is the layer's table, and the snapshot's table replaces it (the
// rule of CompareWithVersion).  Without that table or an earlier snapshot it is SnapshotVersionIncremental.
func SnapshotVersionFromLayer(ctrVersionName string) error {
	data, table := snapshotPaths(ctrVersionName)
	base, ok := baseVersion(ctrVersionName)
	_, dataErr := os.Stat(data)
	tableInfo, tableErr := os.Stat(table)
	if dataErr == nil || tableErr != nil || !tableInfo.Mode().IsRegular() || !ok {
		return SnapshotVersionIncremental(ctrVersionName)
	}
	upper, err := utils.GetContainerMergedLayer(ctrVersionName)
	if err != nil {
		return errors.WithMessagef(err, "utils.GetContainerMergedLayer failed, container: %s", ctrVersionName)
	}
	if err := os.MkdirAll(data, 0755); err != nil {
		return errors.Wrapf(err, "mkdir %s", data)
	}
	baseData, baseTable := snapshotPaths(base)
	return errors.WithMessagef(utils.SnapshotDirFromLayerVerified(upper, data, baseData, baseTable, table, table),
		"snapshot of %s from its layer against %s failed", ctrVersionName, base)
}

// N1 -- ScrubReplicaSet checks every snapshot of the ReplicaSet against its block table in one pass that reads each
// inode the versions share once.  The versions are the merges/<rs>/<rs>-<k> that hold diff/ (the rule of baseVersion;
// a missing blocks.vmig is that version's VMIG_ETABLE).  It returns each version's verdict by name and the report,
// merges/<rs>/scrub.txt, which lists every damaged path and block.
func ScrubReplicaSet(rs string) (map[string]int, string, error) {
	names := snapshotVersions(rs)
	report := filepath.Join(filepath.Dir(versionDir(rs+"-0")), "scrub.txt")
	if len(names) == 0 {
		return map[string]int{}, "", nil
	}
	dirs, tables := make([]string, len(names)), make([]string, len(names))
	for i, name := range names {
		dirs[i], tables[i] = snapshotPaths(name)
	}
	verdicts, err := utils.ScrubSnapshots(dirs, tables, report)
	if err != nil {
		return nil, "", errors.WithMessagef(err, "scrub of %s failed", rs)
	}
	out := make(map[string]int, len(names))
	for i, name := range names {
		out[name] = verdicts[i]
	}
	return out, report, nil
}

// snapshotVersions lists the snapshot versions of the ReplicaSet, oldest first: every merges/<rs>/<rs>-<k> that holds
// diff/ (with or without blocks.vmig).  A version directory without diff/ holds only the running container's table
// (HandoffCopy).
func snapshotVersions(rs string) []string {
	parent := filepath.Dir(versionDir(rs + "-0"))
	entries, _ := os.ReadDir(parent)
	type version struct {
		k    int
		name string
	}
	var found []version
	for _, e := range entries {
		k, err := strconv.Atoi(strings.TrimPrefix(e.Name(), rs+"-"))
		if !strings.HasPrefix(e.Name(), rs+"-") || err != nil || k < 0 {
			continue
		}
		if st, err := os.Stat(filepath.Join(parent, e.Name(), "diff")); err != nil || !st.IsDir() {
			continue
		}
		found = append(found, version{k, e.Name()})
	}
	sort.Slice(found, func(i, j int) bool { return found[i].k < found[j].k })
	names := make([]string, len(found))
	for i, v := range found {
		names[i] = v.name
	}
	return names
}

// N1 -- RetireVersions keeps the newest `keep` snapshots of the ReplicaSet and removes the older ones
// (utils.RetireSnapshots), then removes each emptied merges/<rs>/<rs>-<k> and drops it from ContainerMergeMap.  Unlike
// rm -rf, the kept versions' tables stay trusted: the records whose ctime the removal moved are re-verified on the GPU
// and re-recorded, so the next SnapshotVersionIncremental still links every unchanged file.  A version directory
// without diff/ is never touched.  It returns the retired and the kept version names.
func RetireVersions(rs string, keep int) (retired, kept []string, err error) {
	if keep < 1 {
		return nil, nil, errors.Errorf("RetireVersions: keep must be at least 1, not %d", keep)
	}
	names := snapshotVersions(rs)
	if len(names) == 0 {
		return nil, nil, nil
	}
	cut := len(names) - keep
	if cut < 0 {
		cut = 0
	}
	retired, kept = names[:cut], names[cut:]
	var rdirs, rtables, kdirs, ktables []string
	for _, name := range retired {
		d, t := snapshotPaths(name)
		rdirs, rtables = append(rdirs, d), append(rtables, t)
	}
	for _, name := range kept {
		d, t := snapshotPaths(name)
		kdirs, ktables = append(kdirs, d), append(ktables, t)
	}
	if err := utils.RetireSnapshots(rdirs, rtables, kdirs, ktables); err != nil {
		return nil, nil, errors.WithMessagef(err, "retire of %s failed", rs)
	}
	for _, name := range retired {
		_ = os.Remove(versionDir(name)) // something else lives there too: the directory stays
		k, _ := strconv.ParseInt(name[strings.LastIndex(name, "-")+1:], 10, 64)
		vmap.ContainerMergeMap.Remove(k)
	}
	return retired, kept, nil
}

// N1 -- RollbackFromSnapshot fills newContainer's layer with version `target` of the ReplicaSet.  The new
// layer was just created from the image, so it is seeded with a plain copy of the snapshot; when the caller
// has first put the CURRENT version there (seedTable = that version's blocks.vmig, e.g. after a failed
// roll-forward), only the blocks that differ between the two versions travel.  The snapshot must still match the
// block table it was taken with: one without its table (a SnapshotVersion that failed part way) or one changed
// since fails the rollback instead of being restored.  Replaces the CopyDir of RollbackContainer (replicaset.go:421).
func RollbackFromSnapshot(targetCtrVersionName, newContainer, seedTable string) error {
	data, table := snapshotPaths(targetCtrVersionName)
	upper, err := utils.GetContainerMergedLayer(newContainer)
	if err != nil {
		return errors.WithMessagef(err, "utils.GetContainerMergedLayer failed, container: %s", newContainer)
	}
	_, newTable := snapshotPaths(newContainer)
	if err := os.MkdirAll(filepath.Dir(newTable), 0755); err != nil {
		return errors.Wrapf(err, "mkdir %s", filepath.Dir(newTable))
	}
	// verified + pruned: a seed table that no longer describes the layer is detected per file by the engine (inode/ctime
	// recorded in the table) and that file is copied in full; the re-hash of the destination is the backstop
	return errors.WithMessagef(utils.RestoreDirDiffVerified(data, table, upper, seedTable, newTable), "rollback to %s failed", targetCtrVersionName)
}

// N1 -- RestorePathsFromSnapshot puts the chosen paths of version `target` back into container's layer and leaves
// everything else in it as it is: a tenant who deleted or overwrote one file or directory gets it back without the
// whole-layer Rollback throwing away what they did since.  Each restored file is checked against the snapshot's block
// table (utils.RestorePathsVerified).
//   - The container must not be running: the upper dir of a mounted overlay must not change under it.
//   - The intended flow is Patch-like: HandoffCopy(old, new), then RestorePathsFromSnapshot(target, new, paths,
//     <new's blocks.vmig>), then start new.  seedTable is that table: files still as it recorded them are patched block
//     by block.  No table is written; the seed's records of the files this call rewrote go stale and the next diff
//     pass copies those in full.
//   - No REST route is added; the control plane stays as it is.
func RestorePathsFromSnapshot(targetCtrVersionName, container string, paths []string, seedTable string) error {
	data, table := snapshotPaths(targetCtrVersionName)
	upper, err := utils.GetContainerMergedLayer(container)
	if err != nil {
		return errors.WithMessagef(err, "utils.GetContainerMergedLayer failed, container: %s", container)
	}
	return errors.WithMessagef(utils.RestorePathsVerified(data, table, upper, seedTable, paths), "restore of %d paths from %s failed", len(paths), targetCtrVersionName)
}

// N1 -- CompareWithVersion lists in report every difference between container's layer and version `target`: what
// RollbackFromSnapshot would change, and the paths RestorePathsFromSnapshot could be given.  The snapshot's table stands
// for its data, which is not read; nothing is written but the report.  When the container's own version directory has no
// diff/, its blocks.vmig is the table HandoffCopy wrote for the running layer: files still as it recorded them are not
// read, so "what changed since the hand-off" costs only the files the tenant touched.
//   - No REST route is added; the control plane stays as it is.
func CompareWithVersion(targetCtrVersionName, container, report string) (utils.CompareStats, error) {
	data, table := snapshotPaths(targetCtrVersionName)
	upper, err := utils.GetContainerMergedLayer(container)
	if err != nil {
		return utils.CompareStats{}, errors.WithMessagef(err, "utils.GetContainerMergedLayer failed, container: %s", container)
	}
	ownData, ownTable := snapshotPaths(container)
	layerTable := ""
	if _, err := os.Stat(ownData); os.IsNotExist(err) {
		if _, err := os.Stat(ownTable); err == nil {
			layerTable = ownTable
		}
	}
	st, err := utils.CompareWithSnapshot(upper, layerTable, data, table, report)
	return st, errors.WithMessagef(err, "compare of %s with %s failed", container, targetCtrVersionName)
}

// N1 -- RollbackInPlace rolls the stopped container's layer back to version `target` in place: afterwards it is what
// RollbackFromSnapshot would leave, but only the snapshot blocks the layer does not already hold are read, so a rollback
// costs what differs, not the size of the version.  When the container's own version directory has no diff/, its
// blocks.vmig is the table HandoffCopy wrote for the layer: it is the layer's table (files still as it recorded them
// are not read) and is rewritten for the rolled-back layer.  Otherwise no table is written.
//   - The container must not be running: the upper dir of a mounted overlay must not change under it.
//   - No REST route is added; the control plane stays as it is.
func RollbackInPlace(targetCtrVersionName, container string) (utils.RollbackStats, error) {
	data, table := snapshotPaths(targetCtrVersionName)
	upper, err := utils.GetContainerMergedLayer(container)
	if err != nil {
		return utils.RollbackStats{}, errors.WithMessagef(err, "utils.GetContainerMergedLayer failed, container: %s", container)
	}
	ownData, ownTable := snapshotPaths(container)
	layerTable := ""
	if _, err := os.Stat(ownData); os.IsNotExist(err) {
		if _, err := os.Stat(ownTable); err == nil {
			layerTable = ownTable
		}
	}
	st, err := utils.RollbackLayer(upper, layerTable, data, table, layerTable)
	return st, errors.WithMessagef(err, "rollback of %s to %s failed", container, targetCtrVersionName)
}

// N2 -- HandoffCopy replaces utils.CopyOldMergedToNewContainerMerged in PatchContainer (replicaset.go:333):
// the old container keeps running during pass 1 (the bulk of the bytes), is paused for pass 2, which re-reads
// the source and moves only the blocks whose hash changed in between, and stays paused until the caller has
// started the new container and deleted the old one.  Any engine error resumes the old container and is
// returned BEFORE DeleteContainerForUpdate (replicaset.go:350) can run -- the reference ignores the tar pipe's
// exit status (utils/copy.go:23).  pause/resume are rs.PauseContainer (replicaset.go:641) and its inverse.
// pauseBudget (0 = no limit) bounds how long the old container stays paused: when pass 2 has not finished by then
// it is cancelled, the old container is resumed and ErrPauseBudgetExceeded is returned; the new layer then has no
// table.  ctx (the request's) cancels pass 1, which aborts the hand-off: the fallback to one paused pass is for a live
// source that changed under the reader, not for a caller who gave up.  Once the tenant is paused the hand-off ends by
// finishing or by its budget.
func HandoffCopy(ctx context.Context, oldContainer, newContainer string, pauseBudget time.Duration, pause, resume func(name string) error) error {
	src, err := utils.GetContainerMergedLayer(oldContainer)
	if err != nil {
		return errors.WithMessagef(err, "utils.GetContainerMergedLayer failed, container: %s", oldContainer)
	}
	dst, err := utils.GetContainerMergedLayer(newContainer)
	if err != nil {
		return errors.WithMessagef(err, "utils.GetContainerMergedLayer failed, container: %s", newContainer)
	}
	_, table := snapshotPaths(newContainer)
	if err := os.MkdirAll(filepath.Dir(table), 0755); err != nil {
		return errors.Wrapf(err, "mkdir %s", filepath.Dir(table))
	}
	pass1 := table + ".pass1"
	defer os.Remove(pass1)
	// pass 1, live: a file that shrinks under the reader fails with VMIG_ESRCCHANGED, a directory swapped for a
	// symlink is never followed (DESIGN.md, source-side path safety); both are retried once, paused.
	if err := utils.CopyDirDiffContext(ctx, src, dst, "", pass1); err != nil {
		if ctx.Err() != nil {
			return errors.WithMessage(err, "hand-off cancelled during the live pass; old container untouched")
		}
		log.Warnf("vmig: live pass of %s failed (%v); falling back to one paused pass", oldContainer, err)
		pass1 = ""
	}
	if err := pause(oldContainer); err != nil {
		return errors.WithMessage(err, "pause before the final pass failed")
	}
	budget, cancel := context.Background(), context.CancelFunc(func() {})
	if pauseBudget > 0 {
		budget, cancel = context.WithTimeout(context.Background(), pauseBudget)
	}
	defer cancel()
	if err := utils.CopyDirDiffVerifiedContext(budget, src, dst, pass1, table); err != nil {
		_ = resume(oldContainer)
		if errors.Is(err, context.DeadlineExceeded) {
			log.Warnf("vmig: final pass of %s exceeded its pause budget of %v; old container resumed", oldContainer, pauseBudget)
			return errors.WithMessagef(ErrPauseBudgetExceeded, "%v", err)
		}
		return errors.WithMessage(err, "final pass failed; old container resumed, nothing deleted")
	}
	return nil
}

// N2 -- HandoffCopyFromLayer is HandoffCopy whose paused pass costs what the tenant changed during the live pass, not
// two reads of the layer.  Pass 1 (live) is verified and also leaves a table of the SOURCE's files (<table>.pass1src; a
// file written while it was read is recorded without an identity).  Pass 2 (paused) trusts that table: a source file
// still as it recorded it is not read where the destination still is pass 1's record (<table>.pass1), and only what
// pass 2 wrote is re-read.  Pause budget, resume-on-error and ctx as in HandoffCopy; a failed live pass falls back to
// HandoffCopy's single paused pass.  Both .pass1 tables are removed at the end.
func HandoffCopyFromLayer(ctx context.Context, oldContainer, newContainer string, pauseBudget time.Duration, pause, resume func(name string) error) error {
	src, err := utils.GetContainerMergedLayer(oldContainer)
	if err != nil {
		return errors.WithMessagef(err, "utils.GetContainerMergedLayer failed, container: %s", oldContainer)
	}
	dst, err := utils.GetContainerMergedLayer(newContainer)
	if err != nil {
		return errors.WithMessagef(err, "utils.GetContainerMergedLayer failed, container: %s", newContainer)
	}
	_, table := snapshotPaths(newContainer)
	if err := os.MkdirAll(filepath.Dir(table), 0755); err != nil {
		return errors.Wrapf(err, "mkdir %s", filepath.Dir(table))
	}
	pass1, pass1src := table+".pass1", table+".pass1src"
	defer os.Remove(pass1)
	defer os.Remove(pass1src)
	fallback := false
	if err := utils.CopyDirFromLayerVerifiedContext(ctx, src, "", dst, "", pass1, pass1src, false); err != nil {
		if ctx.Err() != nil {
			return errors.WithMessage(err, "hand-off cancelled during the live pass; old container untouched")
		}
		log.Warnf("vmig: live pass of %s failed (%v); falling back to one paused pass", oldContainer, err)
		fallback = true
	}
	if err := pause(oldContainer); err != nil {
		return errors.WithMessage(err, "pause before the final pass failed")
	}
	budget, cancel := context.Background(), context.CancelFunc(func() {})
	if pauseBudget > 0 {
		budget, cancel = context.WithTimeout(context.Background(), pauseBudget)
	}
	defer cancel()
	if fallback {
		err = utils.CopyDirDiffVerifiedContext(budget, src, dst, "", table)
	} else {
		err = utils.CopyDirFromLayerVerifiedContext(budget, src, pass1src, dst, pass1, table, "", true)
	}
	if err != nil {
		_ = resume(oldContainer)
		if errors.Is(err, context.DeadlineExceeded) {
			log.Warnf("vmig: final pass of %s exceeded its pause budget of %v; old container resumed", oldContainer, pauseBudget)
			return errors.WithMessagef(ErrPauseBudgetExceeded, "%v", err)
		}
		return errors.WithMessage(err, "final pass failed; old container resumed, nothing deleted")
	}
	return nil
}

// ErrPauseBudgetExceeded: HandoffCopy's final pass did not finish within its pause budget; the old container was
// resumed and nothing was deleted.  Test with errors.Is.
var ErrPauseBudgetExceeded = stderrors.New("vmig: final pass exceeded the pause budget")

// N3 -- UsedBytes replaces utils.DirSize in PatchVolumeSize's shrink check (volume.go:126-140): the engine's
// metadata walk (no GPU work) returns the same sum of regular-file sizes; with a non-empty tablePath it also
// leaves the manifest the coming migration can reuse.
func UsedBytes(volVersionName string) (int64, error) {
	mountpoint, err := utils.GetVolumeMountPoint(volVersionName)
	if err != nil {
		return 0, errors.WithMessage(err, "utils.GetVolumeMountPoint failed")
	}
	cs := C.CString(mountpoint)
	defer C.free(unsafe.Pointer(cs))
	var st C.vmig_stats
	runtime.LockOSThread() // vmig_last_error() is thread-local: keep the call and the error fetch on one OS thread
	defer runtime.UnlockOSThread()
	if rc := C.vmig_manifest(cs, 0, 0, nil, &st); rc != 0 {
		return 0, errors.Errorf("vmig_manifest(%s): %s: %s", mountpoint, C.GoString(C.vmig_strerror(rc)), C.GoString(C.vmig_last_error()))
	}
	return int64(st.bytes_total), nil
}
