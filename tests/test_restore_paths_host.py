"""vmig_restore_paths without a GPU: every argument refusal touches nothing and names what it refuses, a pre-cancelled
control comes before the GPU check, valid arguments fail only for want of a GPU, and the host side of the call
(selection walk, table subset, parent chains) as a unit program (tests/select_unit.cpp)."""
import ctypes
import os
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


def _no_gpu(vm):
    try:
        vm.device_count()
        return False
    except vm.VmigError:
        return True


def _state(root: Path) -> dict:
    out = {}
    for dirpath, dirnames, filenames in os.walk(root):
        for n in [""] + dirnames + filenames:
            p = os.path.join(dirpath, n) if n else dirpath
            st = os.lstat(p)
            body = Path(p).read_bytes() if os.path.isfile(p) and not os.path.islink(p) else None
            out[os.path.relpath(p, root)] = (st.st_mode, st.st_uid, st.st_mtime_ns, body)
    return out


@pytest.fixture()
def store(vm, shm_tmp):
    snap, dst = shm_tmp / "snap", shm_tmp / "dst"
    (snap / "sub" / "deep").mkdir(parents=True)
    (snap / "a.bin").write_bytes(b"a" * 5000)
    (snap / "sub" / "deep" / "f").write_bytes(b"f" * 70)
    vm.manifest(snap, shm_tmp / "t.vmig")          # a well-formed table
    (dst / "sub").mkdir(parents=True)
    (dst / "a.bin").write_bytes(b"old")
    os.symlink("a.bin", dst / "lnk")
    for p in (dst / "a.bin", dst / "sub", dst):
        os.utime(p, ns=(1_500_000_000_000_000_000, 1_500_000_000_000_000_000))
    return snap, shm_tmp / "t.vmig", dst


BAD_PATHS = [
    ([], "n_paths == 0"),
    ([""], "paths[0] is empty"),
    (["/a.bin"], "paths[0] '/a.bin' is absolute"),
    (["sub//deep"], "paths[0] 'sub//deep'"),
    (["./a.bin"], "paths[0] './a.bin'"),
    (["sub/../a.bin"], "paths[0] 'sub/../a.bin'"),
    (["sub/."], "paths[0] 'sub/.'"),
    (["sub/"], "paths[0] 'sub/' ends in '/'"),
    (["a.bin", "sub", "a.bin"], "paths[0] and paths[2] are both 'a.bin'"),
    (["sub/deep/f", "sub"], "paths[0] 'sub/deep/f' lies beneath paths[1] 'sub'"),
    ([b"sub/deep", b"sub"], "paths[0] 'sub/deep' lies beneath paths[1] 'sub'"),
]


@pytest.mark.parametrize("paths,needle", BAD_PATHS)
def test_bad_paths_touch_nothing(vm, store, paths, needle):
    snap, table, dst = store
    before = _state(dst), _state(snap)
    with pytest.raises(vm.VmigError) as ei:
        vm.restore_paths(snap, table, dst, paths)
    assert ei.value.code == vm.VMIG_EINVAL, ei.value
    assert needle in str(ei.value)
    assert (_state(dst), _state(snap)) == before


def test_null_array_and_entry(vm, store):
    snap, table, dst = store
    before = _state(dst)
    lib = vm.lib()
    for n, arr, needle in ((1, None, "paths is NULL"), (2, (ctypes.c_char_p * 2)(b"a.bin", None), "paths[1] is NULL")):
        rc = lib.vmig_restore_paths(os.fsencode(snap), os.fsencode(table), os.fsencode(dst), n, arr, None, None, None)
        assert rc == vm.VMIG_EINVAL and needle in vm.last_error()
    assert _state(dst) == before


def test_other_refusals_touch_nothing(vm, store, shm_tmp):
    snap, table, dst = store
    (dst / "inner").mkdir()
    os.utime(dst, ns=(1_500_000_000_000_000_000, 1_500_000_000_000_000_000))
    before = _state(dst)
    calls = [
        (lambda: vm.restore_paths(snap, None, dst, ["a.bin"]), "snap_table"),
        (lambda: vm.restore_paths(snap, "", dst, ["a.bin"]), "snap_table"),
        (lambda: vm.restore_paths(snap, table, snap, ["a.bin"]), "same directory or one is inside the other"),
        (lambda: vm.restore_paths(snap, table, snap / "sub", ["a.bin"]), "same directory or one is inside the other"),
        (lambda: vm.restore_paths(dst / "inner", table, dst, ["a.bin"]), "same directory or one is inside the other"),
        (lambda: vm.restore_paths(snap, table, dst, ["a.bin"], flags=vm.F_MOVE_SRC), "VMIG_F_MOVE_SRC"),
        (lambda: vm.restore_paths(snap, table, dst, ["a.bin"], flags=vm.F_HASH_ONLY), "VMIG_F_HASH_ONLY"),
        (lambda: vm.restore_paths(snap, table, dst, ["a.bin"], flags=vm.F_CUFILE), "VMIG_F_CUFILE"),
        (lambda: vm.restore_paths(snap, table, dst, ["a.bin"], block_bytes=1000), "block_bytes 1000"),
    ]
    for call, needle in calls:
        with pytest.raises(vm.VmigError) as ei:
            call()
        assert ei.value.code == vm.VMIG_EINVAL, ei.value
        assert needle in str(ei.value)
    assert _state(dst) == before
    assert (snap / "a.bin").read_bytes() == b"a" * 5000


def test_missing_destination(vm, store, shm_tmp):
    snap, table, _ = store
    with pytest.raises(vm.VmigError) as ei:
        vm.restore_paths(snap, table, shm_tmp / "nowhere", ["a.bin"])
    assert ei.value.code == vm.VMIG_EIO, ei.value
    (shm_tmp / "plain").write_bytes(b"x")
    with pytest.raises(vm.VmigError) as ei:
        vm.restore_paths(snap, table, shm_tmp / "plain", ["a.bin"])
    assert ei.value.code == vm.VMIG_ENOTDIR, ei.value


def test_cancelled_control_comes_before_the_gpu_check(vm, store):
    snap, table, dst = store
    before = _state(dst)
    with vm.Ctl() as ctl:
        ctl.cancel()
        with pytest.raises(vm.VmigError) as ei:
            vm.restore_paths(snap, table, dst, ["a.bin", "sub"], ctl=ctl)
        assert ei.value.code == vm.VMIG_ECANCELED, ei.value
    assert _state(dst) == before


def test_restore_paths_has_no_cpu_fallback(vm, store):
    if not _no_gpu(vm):
        pytest.skip("a GPU is present; tests/test_restore_paths.py covers the data path")
    snap, table, dst = store
    before = _state(dst)
    for paths in (["a.bin"], ["sub"], ["sub/deep/f", "a.bin"], ["not/in/the/snapshot"]):
        with pytest.raises(vm.VmigError) as ei:
            vm.restore_paths(snap, table, dst, paths, flags=vm.F_VERIFY | vm.F_PRUNE)
        assert ei.value.code == vm.VMIG_ENOGPU, ei.value
    assert _state(dst) == before


def test_selection_unit(shm_tmp, tmp_path):
    exe = tmp_path / "select_unit"
    csrc = ROOT / "gpu-docker-api_b200" / "csrc"
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-pthread", "-I", str(csrc), str(ROOT / "tests" / "select_unit.cpp"),
                    str(csrc / "vmig_select.cpp"), str(csrc / "vmig_tree.cpp"), str(csrc / "vmig_table.cpp"),
                    str(csrc / "vmig_scrub.cpp"), "-o", str(exe)], check=True)
    r = subprocess.run([str(exe), str(shm_tmp)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "select unit ok" in r.stdout, r.stdout + r.stderr
