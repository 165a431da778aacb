"""vmig_restore_tree without a GPU: argument checks, the new error code, and no CPU fallback."""
import os

import pytest


def _no_gpu(vm):
    try:
        vm.device_count()
        return False
    except vm.VmigError:
        return True


def test_strerror_of_ecorrupt(vm):
    assert vm.VMIG_ECORRUPT == -11
    assert vm.strerror(vm.VMIG_ECORRUPT) == "source tree does not match its block table"


def test_restore_requires_its_table(vm, shm_tmp):
    snap, dst = shm_tmp / "snap", shm_tmp / "dst"
    snap.mkdir(), dst.mkdir()
    (snap / "f").write_bytes(b"payload")
    for table in (None, ""):
        with pytest.raises(vm.VmigError) as ei:
            vm.restore_tree(snap, table, dst)
        assert ei.value.code == vm.VMIG_EINVAL, ei.value
        assert "snap_table" in str(ei.value)
    assert os.listdir(dst) == []


def test_restore_never_moves_the_snapshot(vm, shm_tmp):
    snap, dst = shm_tmp / "snap", shm_tmp / "dst"
    snap.mkdir(), dst.mkdir()
    (snap / "f").write_bytes(b"payload")
    vm.manifest(snap, shm_tmp / "t.vmig")
    with pytest.raises(vm.VmigError) as ei:
        vm.restore_tree(snap, shm_tmp / "t.vmig", dst, flags=vm.F_MOVE_SRC)
    assert ei.value.code == vm.VMIG_EINVAL, ei.value
    assert (snap / "f").read_bytes() == b"payload" and os.listdir(dst) == []


def test_restore_has_no_cpu_fallback(vm, shm_tmp):
    if not _no_gpu(vm):
        pytest.skip("a GPU is present; tests/test_restore.py covers the data path")
    snap, dst = shm_tmp / "snap", shm_tmp / "dst"
    snap.mkdir(), dst.mkdir()
    (snap / "f").write_bytes(b"payload")
    vm.manifest(snap, shm_tmp / "t.vmig")        # a well-formed table: only the missing GPU can fail the call
    for call in (lambda: vm.restore_tree(snap, shm_tmp / "t.vmig", dst),
                 lambda: vm.restore_tree(snap, shm_tmp / "t.vmig", None, flags=vm.F_HASH_ONLY)):
        with pytest.raises(vm.VmigError) as ei:
            call()
        assert ei.value.code == vm.VMIG_ENOGPU, ei.value
    assert os.listdir(dst) == []
