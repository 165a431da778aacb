"""gpu-docker-api_b200 -- host-side mirror of the reference's copy interface over libvmig.

The reference (XShengTech/gpu-docker-api, Go) exposes the bulk-copy path as three package-level
functions in ``utils`` (SURVEY.md §8b).  The Go toolchain is absent in this image, so the mirror
that tests and the bench drive is this ctypes binding; the cgo shim a maintainer would add is in
INTEGRATION.md.  Names, argument meaning and error behaviour follow the reference:

    CopyDir(src, dest)                                   utils/copy.go:21-27
    CopyOldMergedToNewContainerMerged(old, new)          utils/copy.go:31-46
    GetContainerMergedLayer(name)                        utils/copy.go:48-54
    CopyOldMountPointToContainerMountPoint(old, new)     utils/copy.go:58-63  (moveVolumeData :74-128)
    GetVolumeMountPoint(name)                            utils/copy.go:65-72
    DirSize(path) / ToBytes("20GB")                      utils/file.go:13-48

Go returns ``error``; here a failure raises :class:`VmigError` (``.code`` is the VMIG_E* value,
the message is libvmig's thread-local detail).  Docker lookups (container -> overlay2 UpperDir,
volume -> Mountpoint) stay in the control plane: they are injected through :func:`set_resolver`.

This package never imports ``oracle/`` and has no CPU fallback: if ``libvmig.so`` is missing the
import fails, and without an sm_90 GPU (H100) every data-path call raises VmigError(VMIG_ENOGPU).
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path
from typing import Callable, Optional

import numpy as np

_HERE = Path(__file__).resolve().parent
LIB_PATH = _HERE / "libvmig.so"

VMIG_OK, VMIG_EINVAL, VMIG_ENOGPU, VMIG_ECUDA, VMIG_EIO = 0, -1, -2, -3, -4
VMIG_ENOMEM, VMIG_ETABLE, VMIG_EFAULT, VMIG_ENOTDIR, VMIG_ESRCCHANGED, VMIG_EVERIFY = -5, -6, -7, -8, -9, -10
VMIG_ECORRUPT, VMIG_ECANCELED = -11, -12
PHASES = ("IDLE", "WALK", "DATA", "VERIFY", "META", "PRUNE", "TABLE", "UNLINK", "DONE")     # VMIG_PHASE_* by value
F_MOVE_SRC, F_SKIP_HIDDEN_TOPDIRS, F_MTIME_NS, F_NO_METADATA, F_HASH_ONLY, F_VERIFY = 0x01, 0x02, 0x04, 0x08, 0x10, 0x20
F_PRUNE, F_DIRECT_IO, F_CUFILE = 0x40, 0x80, 0x100
BLOCK_BYTES = 4 << 20
MOVE_DIR_FLAGS = F_MOVE_SRC | F_VERIFY          # what vmig_move_dir passes (include/vmig.h)

EXPORTS = [
    "vmig_init", "vmig_shutdown", "vmig_device_count", "vmig_strerror", "vmig_last_error", "vmig_version",
    "vmig_migrate_tree", "vmig_restore_tree", "vmig_snapshot_tree", "vmig_copy_dir", "vmig_move_dir", "vmig_migrate_buffer", "vmig_host_alloc",
    "vmig_host_free", "vmig_hash_blocks", "vmig_resident_open", "vmig_resident_close", "vmig_resident_fill",
    "vmig_resident_set_len", "vmig_resident_upload", "vmig_resident_download", "vmig_resident_flip",
    "vmig_resident_set_prior", "vmig_resident_pass", "vmig_resident_results", "vmig_table_info_read",
    "vmig_table_hashes", "vmig_dir_size", "vmig_to_bytes", "vmig_datagen_files", "vmig_manifest", "vmig_link_probe", "vmig_thread_plan",
    "vmig_ctl_open", "vmig_ctl_cancel", "vmig_ctl_progress", "vmig_ctl_close", "vmig_scrub_store",
    "vmig_retire_versions", "vmig_restore_paths", "vmig_compare_snapshot", "vmig_rollback_layer",
    "vmig_snapshot_layer", "vmig_migrate_layer",
]
SCRUB_KINDS = ("missing", "extra", "resized", "block", "hardlink", "unreadable", "table", "dir")
COMPARE_KINDS = ("added", "removed", "type", "resized", "block", "target", "rdev", "hardlink", "mode", "owner", "mtime")


class Opts(C.Structure):
    """vmig_opts (include/vmig.h).  io_threads and streams_per_gpu apply PER LANE: every one of the n_gpus *
    lanes_per_gpu lanes runs io_threads copy threads (n >= 2: (n+1)*2//5 readers, the rest writers; 1: one of each;
    0: the per-box budget divided among the lanes in flight) and keeps up to streams_per_gpu of its pipe's staging
    slots in flight (0, or more than the pipe has: all of them)."""
    _fields_ = [("gpu_mask", C.c_uint32), ("block_bytes", C.c_uint32), ("streams_per_gpu", C.c_uint32),
                ("flags", C.c_uint32), ("io_threads", C.c_uint32), ("lanes_per_gpu", C.c_uint32),
                ("ctl", C.c_uint32), ("reserved", C.c_uint32)]


class Progress(C.Structure):
    _fields_ = [("phase", C.c_uint32), ("running", C.c_uint32)] + [(n, C.c_uint64) for n in (
        "bytes_total", "blocks_total", "bytes_hashed", "blocks_hashed", "bytes_written", "bytes_verified")] + \
        [("reserved", C.c_uint64 * 4)]


class Stats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in (
        "bytes_total", "bytes_h2d", "bytes_d2h", "bytes_written", "blocks_total", "blocks_skipped", "files", "dirs",
        "symlinks", "hardlinks", "specials", "kernel_launches", "ns_total", "ns_walk", "ns_plan", "ns_data",
        "ns_meta", "ns_table")] + [("ms_kernel", C.c_double), ("gpus_used", C.c_uint32), ("lanes_used", C.c_uint32), ("pruned", C.c_uint64),
                                                    ("files_untrusted", C.c_uint64), ("files_direct", C.c_uint64)]

    def as_dict(self) -> dict:
        return {n: getattr(self, n) for n, _ in self._fields_ if n != "reserved"}


class SnapshotStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("files_linked", "bytes_linked", "files_backfilled", "bytes_backfilled",
                                          "files_base_untrusted")] + [("reserved", C.c_uint64 * 3)]

    def as_dict(self) -> dict:
        return {n: getattr(self, n) for n, _ in self._fields_ if n != "reserved"}


class ScrubStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("versions", "versions_damaged", "bytes_referenced", "bytes_unique", "files_damaged",
                                          "blocks_damaged", "files_unreadable")] + [("reserved", C.c_uint64 * 4)]

    def as_dict(self) -> dict:
        return {n: getattr(self, n) for n, _ in self._fields_ if n != "reserved"}


class RetireStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("versions_retired", "entries_removed", "files_freed", "bytes_freed", "records_stale",
                                          "records_restamped", "bytes_rehashed", "tables_rewritten")] + [("reserved", C.c_uint64 * 4)]

    def as_dict(self) -> dict:
        return {n: getattr(self, n) for n, _ in self._fields_ if n != "reserved"}


class CompareStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("paths_added", "paths_removed", "paths_changed", "files_changed", "blocks_changed",
                                          "bytes_restore", "files_read", "bytes_read", "files_trusted", "files_shared")] + \
        [("reserved", C.c_uint64 * 4)]

    def as_dict(self) -> dict:
        return {n: getattr(self, n) for n, _ in self._fields_ if n != "reserved"}


class RollbackStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("files_kept", "files_patched", "files_rebuilt", "files_created", "blocks_fetched",
                                          "bytes_fetched", "files_trusted", "files_read", "bytes_read", "bytes_copied")] + \
        [("reserved", C.c_uint64 * 4)]

    def as_dict(self) -> dict:
        return {n: getattr(self, n) for n, _ in self._fields_ if n != "reserved"}


class LayerSnapshotStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("files_linked", "bytes_linked", "files_backfilled", "bytes_backfilled",
                                          "files_base_untrusted", "files_trusted", "bytes_trusted", "files_read",
                                          "bytes_read")] + [("reserved", C.c_uint64 * 4)]

    def as_dict(self) -> dict:
        return {n: getattr(self, n) for n, _ in self._fields_ if n != "reserved"}


class LayerMigrateStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("files_trusted", "bytes_trusted", "files_read", "bytes_read", "files_unread",
                                          "files_verified", "bytes_verified", "src_recorded", "src_unrecorded")] + \
        [("reserved", C.c_uint64 * 4)]

    def as_dict(self) -> dict:
        return {n: getattr(self, n) for n, _ in self._fields_ if n != "reserved"}


class TableInfo(C.Structure):
    _fields_ = [("block_bytes", C.c_uint32), ("algo", C.c_uint32), ("n_files", C.c_uint64),
                ("n_blocks", C.c_uint64), ("bytes_total", C.c_uint64)]


class VmigError(RuntimeError):
    def __init__(self, code: int, what: str):
        self.code = code
        super().__init__(f"{what}: {strerror(code)} ({code}): {last_error()}")


if not LIB_PATH.exists():
    raise ImportError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                      "(make -C gpu-docker-api_b200/csrc). There is no CPU fallback.")
_lib = C.CDLL(str(LIB_PATH))
_u64p, _u32p, _u8p = C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), C.POINTER(C.c_uint8)
_sig = {
    "vmig_init": (C.c_int, [C.c_uint32]), "vmig_shutdown": (None, []), "vmig_device_count": (C.c_int, []),
    "vmig_strerror": (C.c_char_p, [C.c_int]), "vmig_last_error": (C.c_char_p, []), "vmig_version": (C.c_char_p, []),
    "vmig_migrate_tree": (C.c_int, [C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.POINTER(Opts), C.POINTER(Stats)]),
    "vmig_restore_tree": (C.c_int, [C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.POINTER(Opts),
                                    C.POINTER(Stats)]),
    "vmig_snapshot_tree": (C.c_int, [C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.POINTER(Opts),
                                     C.POINTER(Stats), C.POINTER(SnapshotStats)]),
    "vmig_copy_dir": (C.c_int, [C.c_char_p, C.c_char_p]), "vmig_move_dir": (C.c_int, [C.c_char_p, C.c_char_p]),
    "vmig_migrate_buffer": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.POINTER(Opts), C.POINTER(Stats)]),
    "vmig_host_alloc": (C.c_int, [C.POINTER(C.c_void_p), C.c_uint64]), "vmig_host_free": (None, [C.c_void_p]),
    "vmig_hash_blocks": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p,
                                   C.POINTER(C.c_double)]),
    "vmig_resident_open": (C.c_int, [C.c_int, C.c_uint64, C.c_uint32, C.POINTER(C.c_void_p)]),
    "vmig_resident_close": (None, [C.c_void_p]), "vmig_resident_fill": (C.c_int, [C.c_void_p, C.c_uint64]),
    "vmig_resident_set_len": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint32]),
    "vmig_resident_upload": (C.c_int, [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32]),
    "vmig_resident_download": (C.c_int, [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32]),
    "vmig_resident_flip": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64]),
    "vmig_resident_set_prior": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "vmig_resident_pass": (C.c_int, [C.c_void_p, C.c_uint32, C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "vmig_resident_results": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]),
    "vmig_table_info_read": (C.c_int, [C.c_char_p, C.POINTER(TableInfo)]),
    "vmig_table_hashes": (C.c_int, [C.c_char_p, C.c_void_p, C.c_uint64]),
    "vmig_dir_size": (C.c_int, [C.c_char_p, C.POINTER(C.c_int64), C.POINTER(C.c_uint64)]),
    "vmig_to_bytes": (C.c_int, [C.c_char_p, C.POINTER(C.c_int64)]),
    "vmig_datagen_files": (C.c_int, [C.c_char_p, C.c_uint64, C.c_uint32, C.c_uint64, C.c_uint32]),
    "vmig_manifest": (C.c_int, [C.c_char_p, C.c_uint32, C.c_uint32, C.c_char_p, C.POINTER(Stats)]),
    "vmig_link_probe": (C.c_int, [C.c_int, C.c_uint64, C.POINTER(C.c_double)]),
    "vmig_thread_plan": (C.c_int, [C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]),
    "vmig_ctl_open": (C.c_int, [C.POINTER(C.c_uint32)]), "vmig_ctl_cancel": (C.c_int, [C.c_uint32]),
    "vmig_ctl_progress": (C.c_int, [C.c_uint32, C.POINTER(Progress)]), "vmig_ctl_close": (C.c_int, [C.c_uint32]),
    "vmig_scrub_store": (C.c_int, [C.c_uint32, C.POINTER(C.c_char_p), C.POINTER(C.c_char_p), C.c_char_p, C.POINTER(C.c_int32),
                                   C.POINTER(Opts), C.POINTER(Stats), C.POINTER(ScrubStats)]),
    "vmig_retire_versions": (C.c_int, [C.c_uint32, C.POINTER(C.c_char_p), C.POINTER(C.c_char_p), C.c_uint32, C.POINTER(C.c_char_p),
                                       C.POINTER(C.c_char_p), C.POINTER(Opts), C.POINTER(Stats), C.POINTER(RetireStats)]),
    "vmig_restore_paths": (C.c_int, [C.c_char_p, C.c_char_p, C.c_char_p, C.c_uint32, C.POINTER(C.c_char_p), C.c_char_p,
                                     C.POINTER(Opts), C.POINTER(Stats)]),
    "vmig_compare_snapshot": (C.c_int, [C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.POINTER(Opts),
                                        C.POINTER(Stats), C.POINTER(CompareStats)]),
    "vmig_rollback_layer": (C.c_int, [C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.POINTER(Opts),
                                      C.POINTER(Stats), C.POINTER(RollbackStats)]),
    "vmig_snapshot_layer": (C.c_int, [C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p,
                                      C.POINTER(Opts), C.POINTER(Stats), C.POINTER(LayerSnapshotStats)]),
    "vmig_migrate_layer": (C.c_int, [C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p,
                                     C.POINTER(Opts), C.POINTER(Stats), C.POINTER(LayerMigrateStats)]),
}
for _n, (_r, _a) in _sig.items():
    _f = getattr(_lib, _n)
    _f.restype, _f.argtypes = _r, _a


def lib() -> C.CDLL:
    return _lib


def strerror(code: int) -> str:
    return _lib.vmig_strerror(code).decode()


def last_error() -> str:
    return _lib.vmig_last_error().decode(errors="replace")


def version() -> str:
    return _lib.vmig_version().decode()


def _check(rc: int, what: str) -> None:
    if rc != 0:
        raise VmigError(rc, what)


def init(gpu_mask: int = 0) -> None:
    _check(_lib.vmig_init(gpu_mask), "vmig_init")


def shutdown() -> None:
    _lib.vmig_shutdown()


def device_count() -> int:
    n = _lib.vmig_device_count()
    if n < 0:
        raise VmigError(n, "vmig_device_count")
    return n


def _b(p) -> Optional[bytes]:
    return None if p is None else os.fsencode(p)


class Ctl:
    """A call control (vmig_ctl_*): pass it as ``ctl=`` to migrate_tree, restore_tree, restore_paths, snapshot_tree,
    scrub_store, retire_versions, compare_snapshot, rollback_layer, snapshot_layer, migrate_layer or migrate_buffer,
    then cancel() from any thread (the call raises VmigError(VMIG_ECANCELED)) or read progress() while it runs.  ctypes
    releases the GIL during the call.  One control serves one call at a time; a deadline is a threading.Timer."""

    def __init__(self):
        i = C.c_uint32(0)
        _check(_lib.vmig_ctl_open(C.byref(i)), "vmig_ctl_open")
        self.id = i.value

    def cancel(self) -> None:
        _check(_lib.vmig_ctl_cancel(self.id), "vmig_ctl_cancel")

    def progress(self) -> dict:
        p = Progress()
        _check(_lib.vmig_ctl_progress(self.id, C.byref(p)), "vmig_ctl_progress")
        d = {n: getattr(p, n) for n, _ in p._fields_ if n != "reserved"}
        d["phase_name"] = PHASES[d["phase"]] if d["phase"] < len(PHASES) else "?"
        return d

    def close(self) -> None:
        if self.id:
            _check(_lib.vmig_ctl_close(self.id), "vmig_ctl_close")
            self.id = 0

    def __enter__(self) -> "Ctl":
        return self

    def __exit__(self, *exc) -> None:
        self.close()


def _ctl_id(ctl: Optional[Ctl]) -> int:
    return 0 if ctl is None else ctl.id


# ------------------------------------------------------------------------------------------------
# the reference's interface
_resolver: dict = {"container": None, "volume": None}


def set_resolver(container_upperdir: Optional[Callable[[str], str]] = None,
                 volume_mountpoint: Optional[Callable[[str], str]] = None) -> None:
    """Inject the Docker lookups the control plane owns (ContainerInspect -> GraphDriver.Data
    ["UpperDir"], VolumeInspect -> Mountpoint: reference utils/copy.go:48-54, 65-72)."""
    _resolver["container"], _resolver["volume"] = container_upperdir, volume_mountpoint


def GetContainerMergedLayer(name: str) -> str:
    """reference utils/copy.go:48-54 -- the overlay2 UpperDir (despite the name)."""
    if _resolver["container"] is None:
        raise VmigError(VMIG_EINVAL, f"docker.ContainerInspect failed, name: {name} (no resolver injected)")
    p = _resolver["container"](name)
    if not p:
        raise VmigError(VMIG_EINVAL, f"docker.ContainerInspect failed, name: {name}")
    return p


def GetVolumeMountPoint(name: str) -> str:
    """reference utils/copy.go:65-72."""
    if _resolver["volume"] is None:
        raise VmigError(VMIG_EINVAL, f"docker.VolumeInspect failed, name: {name} (no resolver injected)")
    p = _resolver["volume"](name)
    if not p:
        raise VmigError(VMIG_EINVAL, f"docker.VolumeInspect failed, name: {name}")
    return p


def CopyDir(src: str, dest: str) -> None:
    """reference utils.CopyDir (utils/copy.go:21-27): `(cd src; tar c .) | (cd dest; tar x)`."""
    _check(_lib.vmig_copy_dir(_b(src), _b(dest)), f"CopyDir failed, src:{src}, dest: {dest}")


def CopyOldMergedToNewContainerMerged(oldContainer: str, newContainer: str) -> None:
    """reference utils/copy.go:31-46 (called at services/replicaset.go:333,421,831)."""
    CopyDir(GetContainerMergedLayer(oldContainer), GetContainerMergedLayer(newContainer))


def CopyOldMountPointToContainerMountPoint(oldVolume: str, newVolume: str) -> None:
    """reference utils/copy.go:58-63 -> moveVolumeData (:74-128), called at services/volume.go:150.
    Move semantics, synchronous, status checked (the reference neither waits nor checks)."""
    src, dst = GetVolumeMountPoint(oldVolume), GetVolumeMountPoint(newVolume)
    _check(_lib.vmig_move_dir(_b(src), _b(dst)), f"moveData failed, src:{src}, dest: {dst}")


def DirSize(path: str) -> int:
    """reference utils/file.go:13-22."""
    out = C.c_int64(0)
    _check(_lib.vmig_dir_size(_b(path), C.byref(out), None), "DirSize")
    return out.value


def ToBytes(origin: str) -> int:
    """reference utils/file.go:24-48."""
    out = C.c_int64(0)
    _check(_lib.vmig_to_bytes(origin.encode(), C.byref(out)), "ToBytes")
    return out.value


# ------------------------------------------------------------------------------------------------
# engine entry points
def migrate_tree(src, dst, prior_table=None, out_table=None, *, gpu_mask: int = 0, flags: int = 0,
                 block_bytes: int = 0, io_threads: int = 0, streams_per_gpu: int = 0, lanes_per_gpu: int = 0,
                 ctl: Optional[Ctl] = None) -> dict:
    o = Opts(gpu_mask=gpu_mask, block_bytes=block_bytes, flags=flags, io_threads=io_threads,
             streams_per_gpu=streams_per_gpu, lanes_per_gpu=lanes_per_gpu, ctl=_ctl_id(ctl))
    st = Stats()
    _check(_lib.vmig_migrate_tree(_b(src), _b(dst), _b(prior_table), _b(out_table), C.byref(o), C.byref(st)),
           f"vmig_migrate_tree({src} -> {dst})")
    return st.as_dict()


def restore_tree(snap, snap_table, dst, prior_table=None, out_table=None, *, gpu_mask: int = 0, flags: int = 0,
                 block_bytes: int = 0, io_threads: int = 0, streams_per_gpu: int = 0, lanes_per_gpu: int = 0,
                 ctl: Optional[Ctl] = None) -> dict:
    """migrate_tree(snap, dst, ...) that first requires `snap` to still be the tree `snap_table` describes (same
    paths and sizes, every block's hash): VMIG_ECORRUPT otherwise.  flags=F_HASH_ONLY with dst=None only checks."""
    o = Opts(gpu_mask=gpu_mask, block_bytes=block_bytes, flags=flags, io_threads=io_threads,
             streams_per_gpu=streams_per_gpu, lanes_per_gpu=lanes_per_gpu, ctl=_ctl_id(ctl))
    st = Stats()
    _check(_lib.vmig_restore_tree(_b(snap), _b(snap_table), _b(dst), _b(prior_table), _b(out_table), C.byref(o),
                                  C.byref(st)), f"vmig_restore_tree({snap} -> {dst})")
    return st.as_dict()


def restore_paths(snap, snap_table, dst, paths, prior_table=None, *, flags: int = 0, gpu_mask: int = 0,
                  lanes_per_gpu: int = 0, block_bytes: int = 0, io_threads: int = 0, streams_per_gpu: int = 0,
                  ctl: Optional[Ctl] = None) -> dict:
    """Restore the chosen entries `paths` (str or bytes, relative to `snap`, named as the table names them) of a snapshot
    into `dst`, each regular file checked against `snap_table` as restore_tree checks it; nothing in `dst` outside those
    entries and their parent directories is touched.  prior_table: `dst`'s own table (unchanged blocks are not written);
    no table is written.  Returns the migrate_tree counters of the selection."""
    paths = list(paths)
    arr = (C.c_char_p * max(len(paths), 1))(*[_b(p) for p in paths])
    o = Opts(gpu_mask=gpu_mask, block_bytes=block_bytes, flags=flags, lanes_per_gpu=lanes_per_gpu, io_threads=io_threads,
             streams_per_gpu=streams_per_gpu, ctl=_ctl_id(ctl))
    st = Stats()
    _check(_lib.vmig_restore_paths(_b(snap), _b(snap_table), _b(dst), len(paths), arr, _b(prior_table), C.byref(o),
                                   C.byref(st)), f"vmig_restore_paths({snap} -> {dst}, {len(paths)} paths)")
    return st.as_dict()


def snapshot_tree(src, dst, base=None, base_table=None, out_table=None, *, flags: int = 0, gpu_mask: int = 0,
                  block_bytes: int = 0, io_threads: int = 0, streams_per_gpu: int = 0, lanes_per_gpu: int = 0,
                  ctl: Optional[Ctl] = None) -> dict:
    """Snapshot `src` into `dst` with its block table `out_table` (required), sharing what did not change with the
    previous snapshot `base` (taken with `base_table`): unchanged files become hard links to the base's, changed files
    take their unchanged blocks from the base file.  Without a base it is migrate_tree(src, dst, None, out_table).
    Returns the migrate_tree counters plus files_linked, bytes_linked, files_backfilled, bytes_backfilled and
    files_base_untrusted."""
    o = Opts(gpu_mask=gpu_mask, block_bytes=block_bytes, flags=flags, io_threads=io_threads,
             streams_per_gpu=streams_per_gpu, lanes_per_gpu=lanes_per_gpu, ctl=_ctl_id(ctl))
    st, ss = Stats(), SnapshotStats()
    _check(_lib.vmig_snapshot_tree(_b(src), _b(dst), _b(base), _b(base_table), _b(out_table), C.byref(o), C.byref(st),
                                   C.byref(ss)), f"vmig_snapshot_tree({src} -> {dst}, base {base})")
    return {**st.as_dict(), **ss.as_dict()}


def snapshot_layer(layer, dst, base, base_table, out_table, layer_table, *, flags: int = 0, gpu_mask: int = 0,
                   block_bytes: int = 0, io_threads: int = 0, streams_per_gpu: int = 0, lanes_per_gpu: int = 0,
                   ctl: Optional[Ctl] = None) -> dict:
    """The snapshot snapshot_tree(layer, dst, base, base_table, out_table) writes, with the layer's hashes taken from
    `layer_table` (the table written for the layer's files) wherever it still vouches for a file: of such a file only the
    blocks the base does not hold are read.  F_VERIFY re-reads what was written or backfilled, not what was linked.
    out_table may be layer_table.  Returns the migrate_tree counters plus the vmig_layer_snapshot_stats fields."""
    o = Opts(gpu_mask=gpu_mask, block_bytes=block_bytes, flags=flags, io_threads=io_threads,
             streams_per_gpu=streams_per_gpu, lanes_per_gpu=lanes_per_gpu, ctl=_ctl_id(ctl))
    st, ls = Stats(), LayerSnapshotStats()
    _check(_lib.vmig_snapshot_layer(_b(layer), _b(layer_table), _b(dst), _b(base), _b(base_table), _b(out_table), C.byref(o),
                                    C.byref(st), C.byref(ls)), f"vmig_snapshot_layer({layer} -> {dst}, base {base})")
    return {**st.as_dict(), **ls.as_dict()}


def migrate_layer(src, src_table, dst, prior_table=None, out_table=None, src_out_table=None, *, flags: int = 0,
                  gpu_mask: int = 0, block_bytes: int = 0, io_threads: int = 0, streams_per_gpu: int = 0,
                  lanes_per_gpu: int = 0, ctl: Optional[Ctl] = None) -> dict:
    """What migrate_tree(src, dst, prior_table, out_table) leaves, with the source's hashes taken from `src_table` (a table
    written for the source's files, None: none) wherever it still vouches for a file: of such a file only the blocks that
    differ from the prior record at the same index are read.  src_out_table: the same table with the source's identities,
    for the next call's src_table; a file written while it was read is recorded without one.  F_VERIFY re-reads only the
    destination files the call created, wrote into or resized.  Returns the migrate_tree counters plus the
    vmig_layer_migrate_stats fields."""
    o = Opts(gpu_mask=gpu_mask, block_bytes=block_bytes, flags=flags, io_threads=io_threads,
             streams_per_gpu=streams_per_gpu, lanes_per_gpu=lanes_per_gpu, ctl=_ctl_id(ctl))
    st, ms = Stats(), LayerMigrateStats()
    _check(_lib.vmig_migrate_layer(_b(src), _b(src_table), _b(dst), _b(prior_table), _b(out_table), _b(src_out_table),
                                   C.byref(o), C.byref(st), C.byref(ms)), f"vmig_migrate_layer({src} -> {dst})")
    return {**st.as_dict(), **ms.as_dict()}


def unescape_report_path(s: str) -> bytes:
    """The inverse of the report's path escaping (include/vmig.h, vmig_scrub_store): "\\\\", "\\t", "\\n", "\\xHH"."""
    raw, out, i = os.fsencode(s), bytearray(), 0
    while i < len(raw):
        c = raw[i]
        if c != 0x5C:
            out.append(c)
            i += 1
            continue
        e = raw[i + 1:i + 2]
        if e == b"\\":
            out.append(0x5C)
        elif e == b"t":
            out.append(0x09)
        elif e == b"n":
            out.append(0x0A)
        elif e == b"x":
            out.append(int(raw[i + 2:i + 4], 16))
            i += 2
        else:
            raise ValueError(f"bad escape in report path {s!r}")
        i += 2
    return bytes(out)


def parse_scrub_report(path) -> list:
    """The findings of a vmig_scrub_store report: dicts with version, kind, path (str, os.fsdecode of the raw name),
    block, got and want (None where the report has "-")."""
    out = []
    with open(path, "rb") as f:
        for line in f.read().split(b"\n"):
            if not line:
                continue
            v, kind, p, blk, got, want = os.fsdecode(line).split("\t")
            out.append({"version": int(v), "kind": kind, "path": os.fsdecode(unescape_report_path(p)),
                        "block": None if blk == "-" else int(blk), "got": None if got == "-" else int(got, 16),
                        "want": None if want == "-" else int(want, 16)})
    return out


def scrub_store(pairs, report=None, *, flags: int = 0, gpu_mask: int = 0, lanes_per_gpu: int = 0, block_bytes: int = 0,
                ctl: Optional[Ctl] = None) -> dict:
    """Check every version of a snapshot store, pairs = [(snap_dir, snap_table), ...], in one pass that reads each shared
    inode once.  Returns {"verdicts": [VMIG_* per version], "findings": [...], "stats": the data pass's counters} plus
    the vmig_scrub_stats fields.  A damaged version is a verdict, not an exception.  report: where the report file is
    written (the findings are parsed from it); None: a temporary file that is removed afterwards."""
    import tempfile
    pairs = list(pairs)
    n = len(pairs)
    dirs = (C.c_char_p * max(n, 1))(*[_b(d) for d, _ in pairs])
    tabs = (C.c_char_p * max(n, 1))(*[_b(t) for _, t in pairs])
    verdicts = (C.c_int32 * max(n, 1))()
    o = Opts(gpu_mask=gpu_mask, block_bytes=block_bytes, flags=flags, lanes_per_gpu=lanes_per_gpu, ctl=_ctl_id(ctl))
    st, ss = Stats(), ScrubStats()
    tmpdir = tempfile.mkdtemp(prefix="vmig_scrub_") if report is None else None
    rpath = Path(tmpdir) / "scrub.txt" if tmpdir else Path(report)
    try:
        _check(_lib.vmig_scrub_store(n, dirs, tabs, _b(rpath), verdicts, C.byref(o), C.byref(st), C.byref(ss)),
               f"vmig_scrub_store({n} versions)")
        findings = parse_scrub_report(rpath)
    finally:
        if tmpdir:
            import shutil
            shutil.rmtree(tmpdir, ignore_errors=True)
    return {"verdicts": list(verdicts[:n]), "findings": findings, "stats": st.as_dict(), **ss.as_dict()}


def retire_versions(retire_pairs, keep_pairs, *, flags: int = 0, gpu_mask: int = 0, lanes_per_gpu: int = 0,
                    block_bytes: int = 0, ctl: Optional[Ctl] = None) -> dict:
    """Remove the versions retire_pairs = [(snap_dir, snap_table), ...] of a snapshot store, then re-verify on the GPU and
    re-record the records of the kept versions keep_pairs whose ctime the removal moved, so that the next incremental
    snapshot still trusts them.  Returns the vmig_retire_stats fields plus the data pass's counters ("stats")."""
    retire_pairs, keep_pairs = list(retire_pairs), list(keep_pairs)

    def arr(pairs, i):
        return (C.c_char_p * max(len(pairs), 1))(*[_b(p[i]) for p in pairs])
    o = Opts(gpu_mask=gpu_mask, block_bytes=block_bytes, flags=flags, lanes_per_gpu=lanes_per_gpu, ctl=_ctl_id(ctl))
    st, rs = Stats(), RetireStats()
    _check(_lib.vmig_retire_versions(len(retire_pairs), arr(retire_pairs, 0), arr(retire_pairs, 1), len(keep_pairs),
                                     arr(keep_pairs, 0), arr(keep_pairs, 1), C.byref(o), C.byref(st), C.byref(rs)),
           f"vmig_retire_versions({len(retire_pairs)} retired, {len(keep_pairs)} kept)")
    return {"stats": st.as_dict(), **rs.as_dict()}


def parse_compare_report(path) -> list:
    """The findings of a vmig_compare_snapshot report: dicts with kind, path (str, os.fsdecode of the raw name), block
    (None for "-"), layer and snap (the report's fields as str, None for "-"; the paths of `target` and `hardlink` are
    unescaped like path)."""
    out = []
    with open(path, "rb") as f:
        for line in f.read().split(b"\n"):
            if not line:
                continue
            kind, p, blk, lv, sv = os.fsdecode(line).split("\t")

            def field(v):
                if v == "-":
                    return None
                return os.fsdecode(unescape_report_path(v)) if kind in ("target", "hardlink") else v
            out.append({"kind": kind, "path": os.fsdecode(unescape_report_path(p)), "block": None if blk == "-" else int(blk),
                        "layer": field(lv), "snap": field(sv)})
    return out


def compare_snapshot(layer, snap, snap_table, report=None, layer_table=None, *, flags: int = 0, gpu_mask: int = 0,
                     lanes_per_gpu: int = 0, block_bytes: int = 0, ctl: Optional[Ctl] = None) -> dict:
    """List every difference between the layer `layer` and the version snapshot `snap` (checked against `snap_table`):
    what restore_tree(snap, snap_table, layer, flags=F_PRUNE | flags) would change.  Writes nothing but `report` (one
    line per finding, parse_compare_report reads it).  layer_table: a table of `layer` whose records still vouch for
    their files (those are not read).  Returns the vmig_compare_stats fields plus the data pass's counters ("stats")."""
    o = Opts(gpu_mask=gpu_mask, block_bytes=block_bytes, flags=flags, lanes_per_gpu=lanes_per_gpu, ctl=_ctl_id(ctl))
    st, cs = Stats(), CompareStats()
    _check(_lib.vmig_compare_snapshot(_b(layer), _b(layer_table), _b(snap), _b(snap_table), _b(report), C.byref(o),
                                      C.byref(st), C.byref(cs)), f"vmig_compare_snapshot({layer} vs {snap})")
    return {"stats": st.as_dict(), **cs.as_dict()}


def rollback_layer(layer, snap, snap_table, out_table=None, layer_table=None, *, flags: int = 0, gpu_mask: int = 0,
                   lanes_per_gpu: int = 0, block_bytes: int = 0, io_threads: int = 0, streams_per_gpu: int = 0,
                   ctl: Optional[Ctl] = None) -> dict:
    """Roll the layer `layer` back to the version snapshot `snap` (checked against `snap_table`) in place: afterwards it is
    what restore_tree(snap, snap_table, layer, flags=F_PRUNE | flags) leaves, but only the snapshot blocks the layer does
    not already hold are read.  layer_table: a table of `layer` whose records still vouch for their files (those are not
    read); out_table may be the same path.  Returns the vmig_rollback_stats fields plus the counters of both data passes
    ("stats")."""
    o = Opts(gpu_mask=gpu_mask, block_bytes=block_bytes, flags=flags, lanes_per_gpu=lanes_per_gpu, io_threads=io_threads,
             streams_per_gpu=streams_per_gpu, ctl=_ctl_id(ctl))
    st, rs = Stats(), RollbackStats()
    _check(_lib.vmig_rollback_layer(_b(layer), _b(layer_table), _b(snap), _b(snap_table), _b(out_table), C.byref(o),
                                    C.byref(st), C.byref(rs)), f"vmig_rollback_layer({layer} to {snap})")
    return {"stats": st.as_dict(), **rs.as_dict()}


def hash_tree(src, out_table, *, gpu_mask: int = 0, block_bytes: int = 0) -> dict:
    """Block table of a tree without copying it (VMIG_F_HASH_ONLY)."""
    return migrate_tree(src, None, None, out_table, gpu_mask=gpu_mask, flags=F_HASH_ONLY, block_bytes=block_bytes)


def hash_blocks(buf: np.ndarray, offs, lens, gpu: int = 0):
    """K1 direct: returns (hashes u64[n], kernel_ms)."""
    buf = np.ascontiguousarray(buf, dtype=np.uint8)
    offs = np.ascontiguousarray(offs, dtype=np.uint64)
    lens = np.ascontiguousarray(lens, dtype=np.uint32)
    out = np.zeros(len(offs), dtype=np.uint64)
    ms = C.c_double(0)
    _check(_lib.vmig_hash_blocks(gpu, buf.ctypes.data if buf.size else None, offs.ctypes.data, lens.ctypes.data,
                                 len(offs), out.ctypes.data, C.byref(ms)), "vmig_hash_blocks")
    return out, ms.value


class PinnedBuffer:
    """Page-locked host memory from vmig_host_alloc, exposed as a numpy uint8 array."""

    def __init__(self, nbytes: int):
        p = C.c_void_p()
        _check(_lib.vmig_host_alloc(C.byref(p), nbytes), "vmig_host_alloc")
        self.ptr, self.nbytes = p.value, nbytes
        self.array = np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(self.ptr))

    def free(self):
        if self.ptr:
            self.array = None
            _lib.vmig_host_free(self.ptr)
            self.ptr = None


def migrate_buffer(src: np.ndarray, dst: Optional[np.ndarray], prior_hashes=None, prior_valid=None, *,
                   gpu_mask: int = 0, flags: int = 0, block_bytes: int = 0, io_threads: int = 0, streams_per_gpu: int = 0,
                   lanes_per_gpu: int = 0, ctl: Optional[Ctl] = None):
    """Host buffer -> host buffer through H2D / hash / diff / D2H.  Returns (hashes, stats)."""
    bb = block_bytes or BLOCK_BYTES
    n = src.size
    nb = (n + bb - 1) // bb
    out = np.zeros(nb, dtype=np.uint64)
    ph = None if prior_hashes is None else np.ascontiguousarray(prior_hashes, dtype=np.uint64)
    pv = None if prior_valid is None else np.ascontiguousarray(prior_valid, dtype=np.uint8)
    o = Opts(gpu_mask=gpu_mask, block_bytes=block_bytes, flags=flags, io_threads=io_threads, streams_per_gpu=streams_per_gpu,
             lanes_per_gpu=lanes_per_gpu, ctl=_ctl_id(ctl))
    st = Stats()
    _check(_lib.vmig_migrate_buffer(src.ctypes.data, None if dst is None else dst.ctypes.data, n,
                                    None if ph is None else ph.ctypes.data, None if pv is None else pv.ctypes.data,
                                    out.ctypes.data, C.byref(o), C.byref(st)), "vmig_migrate_buffer")
    return out, st.as_dict()


class Resident:
    """HBM-resident batch of equally sized block slots (the "block-hash GB/s" metric)."""

    def __init__(self, n_blocks: int, block_bytes: int = BLOCK_BYTES, gpu: int = 0):
        h = C.c_void_p()
        _check(_lib.vmig_resident_open(gpu, n_blocks, block_bytes, C.byref(h)), "vmig_resident_open")
        self.h, self.n, self.block_bytes = h, n_blocks, block_bytes

    def close(self):
        if self.h:
            _lib.vmig_resident_close(self.h)
            self.h = None

    def fill(self, seed: int):
        _check(_lib.vmig_resident_fill(self.h, seed & ((1 << 64) - 1)), "vmig_resident_fill")

    def set_len(self, block: int, length: int):
        _check(_lib.vmig_resident_set_len(self.h, block, length), "vmig_resident_set_len")

    def upload(self, block: int, data: np.ndarray):
        data = np.ascontiguousarray(data, dtype=np.uint8)
        _check(_lib.vmig_resident_upload(self.h, block, data.ctypes.data if data.size else None, data.size),
               "vmig_resident_upload")

    def download(self, block: int, length: int) -> np.ndarray:
        out = np.empty(length, dtype=np.uint8)
        _check(_lib.vmig_resident_download(self.h, block, out.ctypes.data, length), "vmig_resident_download")
        return out

    def flip(self, blocks):
        b = np.ascontiguousarray(blocks, dtype=np.uint64)
        _check(_lib.vmig_resident_flip(self.h, b.ctypes.data if b.size else None, b.size), "vmig_resident_flip")

    def set_prior(self, hashes=None, valid=None):
        if hashes is None:
            _check(_lib.vmig_resident_set_prior(self.h, None, None), "vmig_resident_set_prior")
            return
        h = np.ascontiguousarray(hashes, dtype=np.uint64)
        v = np.ascontiguousarray(valid, dtype=np.uint8)
        assert h.size == self.n and v.size == self.n
        _check(_lib.vmig_resident_set_prior(self.h, h.ctypes.data, v.ctypes.data), "vmig_resident_set_prior")

    def run(self, iters: int = 1):
        """Returns (ms of the last hash kernel, ms of all iterations) by CUDA events."""
        a, b = C.c_double(0), C.c_double(0)
        _check(_lib.vmig_resident_pass(self.h, iters, C.byref(a), C.byref(b)), "vmig_resident_pass")
        return a.value, b.value

    def results(self):
        hashes = np.empty(self.n, dtype=np.uint64)
        surv = np.empty(self.n, dtype=np.uint32)
        ns = C.c_uint64(0)
        _check(_lib.vmig_resident_results(self.h, hashes.ctypes.data, surv.ctypes.data, C.byref(ns)),
               "vmig_resident_results")
        return hashes, surv[:ns.value].copy()


def link_probe(gpu: int = 0, nbytes: int = 4 << 30) -> dict:
    """Pinned cudaMemcpyAsync sweep: GB/s host->HBM, HBM->host, and both at once (the e2e roofline denominators)."""
    g = (C.c_double * 4)()
    _check(_lib.vmig_link_probe(gpu, nbytes, g), "vmig_link_probe")
    return {"h2d_GBps": g[0], "d2h_GBps": g[1], "duplex_h2d_GBps": g[2], "duplex_d2h_GBps": g[3]}


def thread_plan(lanes: int = 1, n_gpus: int = 1, *, flags: int = 0, has_prior: bool = False):
    """(readers, writers) per lane the engine would use on this box for such a call (no GPU needed)."""
    r, w = C.c_uint32(0), C.c_uint32(0)
    _check(_lib.vmig_thread_plan(lanes, n_gpus, flags, int(has_prior), C.byref(r), C.byref(w)), "vmig_thread_plan")
    return r.value, w.value


def manifest(src, out_table=None, *, flags: int = 0, block_bytes: int = 0) -> dict:
    """The engine's metadata pass alone (no GPU): totals, and optionally the manifest as a zero-hash table."""
    st = Stats()
    _check(_lib.vmig_manifest(_b(src), flags, block_bytes, _b(out_table), C.byref(st)), f"vmig_manifest({src})")
    return st.as_dict()


def table_info(path) -> dict:
    t = TableInfo()
    _check(_lib.vmig_table_info_read(_b(path), C.byref(t)), "vmig_table_info_read")
    return {n: getattr(t, n) for n, _ in t._fields_}


def table_hashes(path) -> np.ndarray:
    n = table_info(path)["n_blocks"]
    out = np.empty(n, dtype=np.uint64)
    _check(_lib.vmig_table_hashes(_b(path), out.ctypes.data if n else None, n), "vmig_table_hashes")
    return out


def datagen_files(dirpath, seed: int, n_files: int, file_bytes: int, threads: int = 16) -> None:
    _check(_lib.vmig_datagen_files(_b(dirpath), seed & ((1 << 64) - 1), n_files, file_bytes, threads),
           "vmig_datagen_files")
