"""Python mirror of integration/go/services/vmig_handoff.go -- the "next" rows N1-N3 of SURVEY.md §8f.

The Go toolchain is absent in this image, so the hand-off logic a maintainer would add to
internal/services (snapshot per version, rollback from a snapshot, two-pass live hand-off) is kept here
line for line with the Go text, on top of the same C-ABI calls, so that the SEQUENCE is testable
(tests/test_gpu.py::test_handoff_*).  Names and layout follow the reference:

    merges/<rs>/<rs>-<v>/            setToMergeMap, internal/services/replicaset.go:681-704
    merges/<rs>/<rs>-<v>/diff        the snapshot of the version's UpperDir (the commented-out CopyDir there)
    merges/<rs>/<rs>-<v>/blocks.vmig its block table (new)

Docker lookups stay injected (set_resolver), pause/resume are callables (rs.PauseContainer,
internal/services/replicaset.go:641, and its inverse).
"""
from __future__ import annotations

import logging
import os
from pathlib import Path
from typing import Callable, Optional

import threading

from . import (F_PRUNE, F_VERIFY, VMIG_ECANCELED, Ctl, GetContainerMergedLayer, GetVolumeMountPoint, VmigError,
               compare_snapshot, manifest, migrate_layer, migrate_tree, restore_paths, restore_tree, retire_versions,
               rollback_layer, scrub_store, snapshot_layer, snapshot_tree)

log = logging.getLogger("vmig.handoff")
_root: dict = {"cwd": None}


def set_merges_root(path) -> None:
    """The control plane uses its working directory (os.Getwd, replicaset.go:689); tests point it elsewhere."""
    _root["cwd"] = None if path is None else Path(path)


def versionDir(ctrVersionName: str) -> Path:
    """<cwd>/merges/<rs>/<rs>-<v> -- same rule as setToMergeMap (replicaset.go:689-692)."""
    cwd = _root["cwd"] or Path(os.getcwd())
    return cwd / "merges" / ctrVersionName.split("-")[0] / ctrVersionName


def snapshotPaths(ctrVersionName: str):
    d = versionDir(ctrVersionName)
    return d / "diff", d / "blocks.vmig"


def CopyDirDiff(src, dest, priorTable: Optional[os.PathLike], outTable: Optional[os.PathLike], flags: int = 0,
                ctl: Optional[Ctl] = None) -> dict:
    """utils.CopyDirDiff of the cgo shim: CopyDir with the block tables of the diff-skip path.  ctl: the mirror of the
    shim's ...Context variants (a cancelled control raises VmigError(VMIG_ECANCELED))."""
    return migrate_tree(src, dest, priorTable or None, outTable or None, flags=flags, ctl=ctl)


def CopyDirDiffVerified(src, dest, priorTable, outTable, ctl: Optional[Ctl] = None) -> dict:
    """The pass after which the old container is deleted: the destination is re-read through the GPU and must hash
    like the source (VMIG_F_VERIFY), and holds nothing the source does not (VMIG_F_PRUNE)."""
    return CopyDirDiff(src, dest, priorTable, outTable, F_VERIFY | F_PRUNE, ctl)


def CopyDirFromLayerVerified(src, srcTable, dest, priorTable, outTable, srcOutTable, prune: bool = True,
                             ctl: Optional[Ctl] = None) -> dict:
    """utils.CopyDirFromLayerVerified of the cgo shim: CopyDirDiffVerified through the source's own block table
    (vmig_migrate_layer).  Of a source file srcTable still vouches for, only the blocks that differ from the destination's
    priorTable record are read; the re-read covers only the destination files the call created, wrote into or resized.
    srcOutTable receives the table the next call trusts as srcTable.  prune False: no F_PRUNE (the hand-off's live
    pass).  ctl: the mirror of the shim's ...Context variant."""
    return migrate_layer(src, srcTable or None, dest, priorTable or None, outTable or None, srcOutTable or None,
                         flags=F_VERIFY | (F_PRUNE if prune else 0), ctl=ctl)


def SnapshotDirVerified(src, dest, outTable) -> dict:
    """utils.SnapshotDirVerified of the cgo shim: a snapshot is re-read through the GPU (VMIG_F_VERIFY) before its
    table is written, so the table describes what really landed in `dest`."""
    return CopyDirDiff(src, dest, None, outTable, F_VERIFY)


def SnapshotDirIncrementalVerified(src, dest, baseDir, baseTable, outTable) -> dict:
    """utils.SnapshotDirIncrementalVerified of the cgo shim: SnapshotDirVerified that shares what did not change with
    the previous snapshot baseDir (vmig_snapshot_tree).  The re-read covers linked files too, so a base that rotted
    without moving its ctime is caught when the snapshot is taken."""
    return snapshot_tree(src, dest, baseDir, baseTable, outTable, flags=F_VERIFY)


def RestoreDirDiffVerified(snap, snapTable, dest, priorTable, outTable) -> dict:
    """utils.RestoreDirDiffVerified of the cgo shim: CopyDirDiffVerified from a snapshot that must still match its own
    block table (vmig_restore_tree); a partial, edited or rotted snapshot fails with VMIG_ECORRUPT."""
    return restore_tree(snap, snapTable, dest, priorTable or None, outTable or None, flags=F_VERIFY | F_PRUNE)


def RestorePathsVerified(snap, snapTable, dest, priorTable, paths, ctl: Optional[Ctl] = None) -> dict:
    """utils.RestorePathsVerified of the cgo shim: the chosen paths of a snapshot (vmig_restore_paths), each regular file
    checked against the snapshot's table, verified, and pruned beneath the chosen directories only.  No table is written."""
    return restore_paths(snap, snapTable, dest, paths, priorTable or None, flags=F_VERIFY | F_PRUNE, ctl=ctl)


def SnapshotVersion(ctrVersionName: str) -> dict:
    """N1: keep the layer of <rs>-<v> and the XXH64 table of its 4 MiB blocks before the container is deleted."""
    upper = GetContainerMergedLayer(ctrVersionName)
    data, table = snapshotPaths(ctrVersionName)
    data.mkdir(parents=True, exist_ok=True)
    return SnapshotDirVerified(upper, data, table)


def baseVersion(ctrVersionName: str) -> Optional[str]:
    """The newest earlier version <rs>-<k> (k < v) whose directory holds both diff/ and blocks.vmig, or None."""
    rs, v = ctrVersionName.split("-")[0], int(ctrVersionName.rsplit("-", 1)[1])
    best = -1
    parent = versionDir(ctrVersionName).parent
    for d in (parent.iterdir() if parent.is_dir() else ()):
        k = d.name[len(rs) + 1:]
        if not d.name.startswith(rs + "-") or not k.isdigit() or not best < int(k) < v:
            continue
        if (d / "diff").is_dir() and (d / "blocks.vmig").is_file():
            best = int(k)
    return None if best < 0 else f"{rs}-{best}"


def SnapshotVersionIncremental(ctrVersionName: str) -> dict:
    """N1, as setToMergeMap calls it: SnapshotVersion that shares unchanged files and blocks with the newest earlier
    snapshot of the ReplicaSet, wherever that snapshot holds them (a file renamed or moved since is still shared), and
    a full SnapshotDirVerified when there is none.  That version's blocks.vmig may have
    been written last by HandoffCopy for the container's layer, not for diff/ (a snapshot of it that failed part
    way): the identities it records then name no file under diff/, the engine trusts none of them, and the result is
    a plain verified copy."""
    upper = GetContainerMergedLayer(ctrVersionName)
    data, table = snapshotPaths(ctrVersionName)
    data.mkdir(parents=True, exist_ok=True)
    base = baseVersion(ctrVersionName)
    if base is None:
        return SnapshotDirVerified(upper, data, table)
    baseData, baseTable = snapshotPaths(base)
    return SnapshotDirIncrementalVerified(upper, data, baseData, baseTable, table)


def SnapshotDirFromLayerVerified(src, dest, baseDir, baseTable, outTable, layerTable) -> dict:
    """utils.SnapshotDirFromLayerVerified of the cgo shim: SnapshotDirIncrementalVerified with the layer's own block table
    (vmig_snapshot_layer): of a file the table still vouches for only the blocks the base lacks are read.  The re-read
    covers what was written or backfilled; linked files are the base table's own record and are left to the scrub."""
    return snapshot_layer(src, dest, baseDir, baseTable, outTable, layerTable, flags=F_VERIFY)


def SnapshotVersionFromLayer(ctrVersionName: str) -> dict:
    """N1: the snapshot SnapshotVersionIncremental writes, at the cost of what the tenant changed since the hand-off.  When
    the version's directory has no diff/ yet, its blocks.vmig is the table HandoffCopy (or RollbackInPlace) wrote for the
    running layer: it is the layer's table, and the snapshot's table replaces it (the rule of CompareWithVersion).  Without
    that table or an earlier snapshot to share with, it is SnapshotVersionIncremental."""
    data, table = snapshotPaths(ctrVersionName)
    base = baseVersion(ctrVersionName)
    if data.exists() or not table.is_file() or base is None:
        return SnapshotVersionIncremental(ctrVersionName)
    upper = GetContainerMergedLayer(ctrVersionName)
    data.mkdir(parents=True, exist_ok=True)
    baseData, baseTable = snapshotPaths(base)
    return SnapshotDirFromLayerVerified(upper, data, baseData, baseTable, table, table)


def ScrubReplicaSet(rs: str) -> dict:
    """N1: check every snapshot of the ReplicaSet against its block table in one pass (vmig_scrub_store) that reads each
    inode the versions share once.  The versions are the merges/<rs>/<rs>-<k> that hold diff/ (the rule of baseVersion;
    a missing blocks.vmig is that version's VMIG_ETABLE).  Returns {"verdicts": {version name: VMIG_* verdict},
    "report": merges/<rs>/scrub.txt}, the report listing every damaged path and block."""
    names = snapshotVersions(rs)
    report = versionDir(rs + "-0").parent / "scrub.txt"
    if not names:
        return {"verdicts": {}, "report": None}
    out = scrub_store([snapshotPaths(name) for name in names], report)
    return {"verdicts": dict(zip(names, out["verdicts"])), "report": report}


def snapshotVersions(rs: str) -> list:
    """The snapshot versions of the ReplicaSet, oldest first: every merges/<rs>/<rs>-<k> that holds diff/ (with or
    without blocks.vmig).  A version directory without diff/ holds only the running container's table (HandoffCopy)."""
    parent = versionDir(rs + "-0").parent
    found = []
    for d in (parent.iterdir() if parent.is_dir() else ()):
        k = d.name[len(rs) + 1:]
        if not d.name.startswith(rs + "-") or not k.isdigit():
            continue
        if (d / "diff").is_dir():
            found.append((int(k), d.name))
    found.sort()
    return [name for _, name in found]


def RetireVersions(rs: str, keep: int) -> dict:
    """N1: keep the newest `keep` snapshots of the ReplicaSet and remove the older ones (vmig_retire_versions), then remove
    each emptied merges/<rs>/<rs>-<k>.  Unlike rm -rf, the kept versions' tables stay trusted: the records whose ctime
    the removal moved are re-verified on the GPU and re-recorded, so the next SnapshotVersionIncremental still links
    every unchanged file.  A version directory without diff/ is never touched.  Returns {"retired": [version names],
    "kept": [version names]} plus the counters of retire_versions."""
    if keep < 1:
        raise ValueError(f"keep must be at least 1, not {keep}")
    names = snapshotVersions(rs)
    if not names:
        return {"retired": [], "kept": []}
    retired, kept = names[:-keep], names[-keep:]
    out = retire_versions([snapshotPaths(name) for name in retired], [snapshotPaths(name) for name in kept])
    for name in retired:
        try:
            versionDir(name).rmdir()
        except OSError:             # something else lives there too: the directory stays
            pass
    return {"retired": retired, "kept": kept, **out}


def RollbackFromSnapshot(targetCtrVersionName: str, newContainer: str, seedTable=None) -> dict:
    """N1: fill newContainer's layer with version `target`.  seedTable = the table written FOR newContainer's layer by
    whatever put its present content there; only blocks that differ then travel.  A seed table that no longer
    describes the layer (failed earlier pass, out-of-band change) is detected per file by the engine and that file is
    copied in full; the result is verified either way.  The snapshot itself must still match the table it was taken
    with: one without its table (a snapshot that failed part way) or one that changed since fails the rollback."""
    data, table = snapshotPaths(targetCtrVersionName)
    upper = GetContainerMergedLayer(newContainer)
    _, newTable = snapshotPaths(newContainer)
    newTable.parent.mkdir(parents=True, exist_ok=True)
    return RestoreDirDiffVerified(data, table, upper, seedTable, newTable)


def RestorePathsFromSnapshot(targetCtrVersionName: str, container: str, paths: list, seedTable=None) -> dict:
    """N1: put the chosen paths of version `target` back into `container`'s layer and leave everything else in it as it
    is: a tenant who deleted or overwrote one file or directory gets it back without the whole-layer Rollback throwing
    away what they did since.  Each restored file is checked against the snapshot's block table (RestorePathsVerified).
      - The container must not be running: the upper dir of a mounted overlay must not change under it.
      - The intended flow is Patch-like: HandoffCopy(old, new), then RestorePathsFromSnapshot(target, new, paths,
        <new's blocks.vmig>), then start new.  seedTable is that table: files still as it recorded them are patched block
        by block.  No table is written; the seed's records of the files this call rewrote go stale and the next diff
        pass copies those in full.
      - No REST route is added; the control plane stays as it is."""
    data, table = snapshotPaths(targetCtrVersionName)
    upper = GetContainerMergedLayer(container)
    return RestorePathsVerified(data, table, upper, seedTable, paths)


def CompareWithVersion(targetCtrVersionName: str, container: str, report) -> dict:
    """N1: list in `report` every difference between `container`'s layer and version `target`: what RollbackFromSnapshot
    would change, and the paths RestorePathsFromSnapshot could be given.  The snapshot's table stands for its data, which
    is not read; nothing is written but the report.  When the container's own version directory has no diff/, its
    blocks.vmig is the table HandoffCopy wrote for the running layer: files still as it recorded them are not read, so
    "what changed since the hand-off" costs only the files the tenant touched.
      - No REST route is added; the control plane stays as it is."""
    data, table = snapshotPaths(targetCtrVersionName)
    upper = GetContainerMergedLayer(container)
    ownData, ownTable = snapshotPaths(container)
    layerTable = None
    if not ownData.exists():
        if ownTable.exists():
            layerTable = ownTable
    return compare_snapshot(upper, data, table, report, layerTable)


def RollbackInPlace(targetCtrVersionName: str, container: str) -> dict:
    """N1: roll the stopped container's layer back to version `target` in place: afterwards it is what
    RollbackFromSnapshot would leave, but only the snapshot blocks the layer does not already hold are read, so a
    rollback costs what differs, not the size of the version.  When the container's own version directory has no diff/,
    its blocks.vmig is the table HandoffCopy wrote for the layer: it is the layer's table (files still as it recorded them
    are not read) and is rewritten for the rolled-back layer.  Otherwise no table is written.
      - The container must not be running: the upper dir of a mounted overlay must not change under it.
      - No REST route is added; the control plane stays as it is."""
    data, table = snapshotPaths(targetCtrVersionName)
    upper = GetContainerMergedLayer(container)
    ownData, ownTable = snapshotPaths(container)
    layerTable = None
    if not ownData.exists():
        if ownTable.exists():
            layerTable = ownTable
    return rollback_layer(upper, data, table, layerTable, layerTable, flags=F_VERIFY)


def HandoffCopy(oldContainer: str, newContainer: str, pause: Callable[[str], None], resume: Callable[[str], None],
                pauseBudget: float = 0.0, ctl: Optional[Ctl] = None) -> dict:
    """N2: replaces utils.CopyOldMergedToNewContainerMerged in PatchContainer (replicaset.go:333).  The old container
    keeps running during pass 1 (the bulk of the bytes), is paused for pass 2, which re-reads the source and moves
    only the blocks whose hash changed in between, prunes what the tenant deleted meanwhile, verifies, and leaves the
    old container paused for the caller to delete.  Any engine error resumes the old container and is raised.
    pauseBudget (seconds, 0 = no limit) bounds how long the old container stays paused: pass 2 is cancelled when it
    runs out, the old container is resumed, and a VmigError(VMIG_ECANCELED) with pause_budget_exceeded = True is
    raised; the new layer then has no table.  ctl (the Go version's ctx) cancels pass 1: the hand-off is aborted, the
    paused-pass fallback is only for a live source that changed under the reader."""
    src = GetContainerMergedLayer(oldContainer)
    dst = GetContainerMergedLayer(newContainer)
    _, table = snapshotPaths(newContainer)
    table.parent.mkdir(parents=True, exist_ok=True)
    pass1: Optional[Path] = Path(str(table) + ".pass1")
    out = {"pass1": None, "pass1_error": None}
    try:
        try:
            out["pass1"] = CopyDirDiff(src, dst, None, pass1, ctl=ctl)
        except VmigError as e:      # live source: a file that shrinks under the reader, a directory swapped for a symlink
            if e.code == VMIG_ECANCELED:
                raise
            log.warning("vmig: live pass of %s failed (%s); falling back to one paused pass", oldContainer, e)
            out["pass1_error"] = e.code
            pass1 = None
        pause(oldContainer)
        # once the tenant is paused the hand-off ends by finishing or by its budget, whatever happens to the request
        with Ctl() as budget:
            expired = threading.Event()

            def expire():
                expired.set()
                budget.cancel()
            timer = threading.Timer(pauseBudget, expire) if pauseBudget > 0 else None
            if timer is not None:
                timer.start()
            try:
                out["pass2"] = CopyDirDiffVerified(src, dst, pass1, table, ctl=budget)
            except VmigError as e:
                resume(oldContainer)
                if e.code == VMIG_ECANCELED and expired.is_set():
                    e.pause_budget_exceeded = True
                    log.warning("vmig: final pass of %s exceeded its pause budget of %.3f s; old container resumed",
                                oldContainer, pauseBudget)
                raise
            finally:
                if timer is not None:
                    timer.cancel()
                    timer.join()
        return out
    finally:
        if pass1 is not None and pass1.exists():
            pass1.unlink()


def HandoffCopyFromLayer(oldContainer: str, newContainer: str, pause: Callable[[str], None],
                         resume: Callable[[str], None], pauseBudget: float = 0.0, ctl: Optional[Ctl] = None) -> dict:
    """N2: HandoffCopy whose paused pass costs what the tenant changed during the live pass, not two reads of the layer.
    Pass 1 (live) is verified and also leaves a table of the SOURCE's files (<table>.pass1src; a file written while it
    was read is recorded without an identity).  Pass 2 (paused) trusts that table: a source file still as it recorded
    it is not read where the destination still is pass 1's record (<table>.pass1), and only what pass 2 wrote is
    re-read.  Pause budget, resume-on-error and ctl as in HandoffCopy; a failed live pass falls back to HandoffCopy's
    single paused pass.  Both .pass1 tables are removed at the end."""
    src = GetContainerMergedLayer(oldContainer)
    dst = GetContainerMergedLayer(newContainer)
    _, table = snapshotPaths(newContainer)
    table.parent.mkdir(parents=True, exist_ok=True)
    pass1, pass1src = Path(str(table) + ".pass1"), Path(str(table) + ".pass1src")
    out = {"pass1": None, "pass1_error": None}
    try:
        fallback = False
        try:
            out["pass1"] = CopyDirFromLayerVerified(src, None, dst, None, pass1, pass1src, prune=False, ctl=ctl)
        except VmigError as e:      # live source: a file that shrinks under the reader, a directory swapped for a symlink
            if e.code == VMIG_ECANCELED:
                raise
            log.warning("vmig: live pass of %s failed (%s); falling back to one paused pass", oldContainer, e)
            out["pass1_error"] = e.code
            fallback = True
        pause(oldContainer)
        with Ctl() as budget:
            expired = threading.Event()

            def expire():
                expired.set()
                budget.cancel()
            timer = threading.Timer(pauseBudget, expire) if pauseBudget > 0 else None
            if timer is not None:
                timer.start()
            try:
                if fallback:
                    out["pass2"] = CopyDirDiffVerified(src, dst, None, table, ctl=budget)
                else:
                    out["pass2"] = CopyDirFromLayerVerified(src, pass1src, dst, pass1, table, None, ctl=budget)
            except VmigError as e:
                resume(oldContainer)
                if e.code == VMIG_ECANCELED and expired.is_set():
                    e.pause_budget_exceeded = True
                    log.warning("vmig: final pass of %s exceeded its pause budget of %.3f s; old container resumed",
                                oldContainer, pauseBudget)
                raise
            finally:
                if timer is not None:
                    timer.cancel()
                    timer.join()
        return out
    finally:
        for p in (pass1, pass1src):
            if p.exists():
                p.unlink()


def UsedBytes(volVersionName: str) -> int:
    """N3: replaces utils.DirSize in PatchVolumeSize's shrink check (volume.go:126-140)."""
    return manifest(GetVolumeMountPoint(volVersionName))["bytes_total"]
