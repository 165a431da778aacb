"""vmig_snapshot_tree without a GPU: argument checks before the destination is touched, no CPU fallback, the C layout
of vmig_snapshot_stats, and the host-side copy that backfills a snapshot file from its base."""
import ctypes
import os
import subprocess
import tempfile
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


def _no_gpu(vm):
    try:
        vm.device_count()
        return False
    except vm.VmigError:
        return True


def _layer(base: Path):
    """src with one file, an earlier snapshot v1 with its table (a zero-hash manifest table), an empty v2."""
    src, v1, v2 = base / "src", base / "v1", base / "v2"
    for d in (src, v1, v2):
        d.mkdir()
    (src / "f").write_bytes(b"payload")
    (v1 / "f").write_bytes(b"payload")
    return src, v1, base / "v1.vmig", v2


def _refused(vm, code, call, needle=None):
    with pytest.raises(vm.VmigError) as ei:
        call()
    assert ei.value.code == code, ei.value
    if needle:
        assert needle in str(ei.value), str(ei.value)


def test_snapshot_argument_errors_leave_the_destination_untouched(vm, shm_tmp):
    src, v1, t1, v2 = _layer(shm_tmp)
    vm.manifest(v1, t1)
    out = shm_tmp / "v2.vmig"
    E = vm.VMIG_EINVAL
    _refused(vm, E, lambda: vm.snapshot_tree(src, v2, v1, None, out), "base_table")
    _refused(vm, E, lambda: vm.snapshot_tree(src, v2, None, t1, out), "base_dir")
    _refused(vm, E, lambda: vm.snapshot_tree(src, v2, v1, t1, None), "out_table")
    _refused(vm, E, lambda: vm.snapshot_tree(src, v2, None, None, ""), "out_table")
    for flag, needle in ((vm.F_MOVE_SRC, "VMIG_F_MOVE_SRC"), (vm.F_HASH_ONLY, "VMIG_F_HASH_ONLY"), (vm.F_CUFILE, "VMIG_F_CUFILE")):
        _refused(vm, E, lambda: vm.snapshot_tree(src, v2, v1, t1, out, flags=flag), needle)
        _refused(vm, E, lambda: vm.snapshot_tree(src, v2, None, None, out, flags=flag), needle)
    _refused(vm, E, lambda: vm.snapshot_tree(src, v1, v1, t1, out), "inside")                       # base == dst
    (v1 / "next").mkdir()
    _refused(vm, E, lambda: vm.snapshot_tree(src, v1 / "next", v1, t1, out), "inside")              # dst inside base
    _refused(vm, E, lambda: vm.snapshot_tree(src, shm_tmp, v1, t1, out), "inside")                  # base inside dst
    os.symlink(v1, shm_tmp / "v1_alias")
    _refused(vm, E, lambda: vm.snapshot_tree(src, shm_tmp / "v1_alias", v1, t1, out), "inside")     # by real path
    assert os.listdir(v2) == [] and not out.exists()
    assert sorted(os.listdir(v1)) == ["f", "next"] and os.listdir(v1 / "next") == []


def test_snapshot_has_no_cpu_fallback(vm, shm_tmp):
    if not _no_gpu(vm):
        pytest.skip("a GPU is present; tests/test_snapshot.py covers the data path")
    src, v1, t1, v2 = _layer(shm_tmp)
    vm.manifest(v1, t1)
    for base, table in ((None, None), (v1, t1)):
        with pytest.raises(vm.VmigError) as ei:
            vm.snapshot_tree(src, v2, base, table, shm_tmp / "v2.vmig")
        assert ei.value.code == vm.VMIG_ENOGPU, ei.value
    assert os.listdir(v2) == [] and not (shm_tmp / "v2.vmig").exists()


def test_snapshot_stats_layout_matches_header(vm):
    exe_dir = Path(tempfile.mkdtemp(prefix="vmig_snaplayout_"))         # /dev/shm may be mounted noexec
    exe = exe_dir / "snapshot_layout"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", str(ROOT / "include"), str(ROOT / "tests" / "snapshot_layout.c"),
                    "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    S = vm.SnapshotStats
    assert out[1] == f"{ctypes.sizeof(S)}:" + ",".join(str(getattr(S, n).offset) for n in (
        "files_linked", "bytes_linked", "files_backfilled", "bytes_backfilled", "files_base_untrusted", "reserved"))
    assert ctypes.sizeof(S) == 64 and out[2] == "abi=2"


def test_backfill_copy_unit(shm_tmp, tmp_path):
    """copy_range (csrc/vmig_tree.cpp) alone: copy_file_range and the forced pread/pwrite fallback copy exactly the
    requested range; an O_DIRECT destination takes whole sectors where the filesystem allows O_DIRECT."""
    exe = tmp_path / "backfill_unit"
    csrc = ROOT / "gpu-docker-api_b200" / "csrc"
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-pthread", "-I", str(csrc), str(ROOT / "tests" / "backfill_unit.cpp"),
                    str(csrc / "vmig_tree.cpp"), "-o", str(exe)], check=True)
    disk = tmp_path / "disk"
    disk.mkdir()
    r = subprocess.run([str(exe), str(shm_tmp), str(disk)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "backfill unit ok" in r.stdout, r.stdout + r.stderr
