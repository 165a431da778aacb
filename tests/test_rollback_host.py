"""vmig_rollback_layer without a GPU: the C layout of vmig_rollback_stats, every refusal in its order with nothing
touched, a pre-cancelled control, no CPU fallback, and the host side of the rollback (actions, fetch list, copy runs,
bytes_fetched, the layer identity checks) as a unit program built with g++ alone."""
import ctypes
import os
import shutil
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


def _trees(vm, root: Path):
    """A layer and a snapshot with their (zero-hash) tables; only the missing GPU or the arguments can fail a rollback."""
    layer, snap = root / "layer", root / "snap"
    for d, n in ((layer, 5000), (snap, 6000)):
        (d / "sub").mkdir(parents=True)
        (d / "a").write_bytes(b"x" * n)
        (d / "sub" / "b").write_bytes(b"y" * 70)
    vm.manifest(snap, root / "snap.vmig")
    vm.manifest(layer, root / "layer.vmig")
    return layer, snap, root / "snap.vmig", root / "layer.vmig"


def _state(root: Path):
    """Every entry under root with its identity and, for regular files, its bytes."""
    out = {}
    for dp, dns, fns in os.walk(root):
        for n in dns + fns:
            p = os.path.join(dp, n)
            s = os.lstat(p)
            data = open(p, "rb").read() if os.path.isfile(p) and not os.path.islink(p) else None
            out[p] = (s.st_ino, s.st_nlink, s.st_mode, s.st_size, s.st_mtime_ns, s.st_ctime_ns, data)
    return out


def _refused(vm, code, out, *args, **kw):
    with pytest.raises(vm.VmigError) as ei:
        vm.rollback_layer(*args, **kw)
    assert ei.value.code == code, (args, kw, ei.value)
    assert not out.exists() and not any(n.startswith(out.name) for n in os.listdir(out.parent))
    return ei.value


def test_rollback_stats_layout_matches_header(vm):
    exe_dir = Path(tempfile.mkdtemp(prefix="vmig_rblayout_"))           # /dev/shm may be mounted noexec
    try:
        exe = exe_dir / "rollback_layout"
        subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", str(ROOT / "include"), str(ROOT / "tests" / "rollback_layout.c"),
                        "-o", str(exe)], check=True)
        out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    finally:
        shutil.rmtree(exe_dir, ignore_errors=True)
    S = vm.RollbackStats
    assert out[1] == f"{ctypes.sizeof(S)}:" + ",".join(str(getattr(S, n).offset) for n in (
        "files_kept", "files_patched", "files_rebuilt", "files_created", "blocks_fetched", "bytes_fetched", "files_trusted",
        "files_read", "bytes_read", "bytes_copied", "reserved"))
    assert ctypes.sizeof(S) == 112 and out[2] == "abi=2"
    assert "vmig_rollback_layer" in vm.EXPORTS and hasattr(vm.lib(), "vmig_rollback_layer")


def test_rollback_refusals_in_order(vm, shm_tmp):
    layer, snap, st, lt = _trees(vm, shm_tmp)
    out = shm_tmp / "out.vmig"
    missing = shm_tmp / "nowhere"
    bad_table = shm_tmp / "bad.vmig"
    bad_table.write_bytes(b"not a table")
    (snap / "inner").mkdir()
    before = _state(shm_tmp)
    # 1. VMIG_EINVAL, ahead of a cancelled control, a missing directory and a bad table
    for a in ((None, snap, st), ("", snap, st), (layer, None, st), (layer, "", st), (layer, snap, None), (layer, snap, "")):
        _refused(vm, vm.VMIG_EINVAL, out, *a, out)
    with vm.Ctl() as c:
        c.cancel()
        for flags in (vm.F_HASH_ONLY, vm.F_MOVE_SRC, vm.F_CUFILE, 0x8000):
            _refused(vm, vm.VMIG_EINVAL, out, missing, snap, bad_table, out, flags=flags, ctl=c)
        _refused(vm, vm.VMIG_EINVAL, out, missing, snap, bad_table, out, block_bytes=4097, ctl=c)
        for la, sn in ((layer, layer), (layer, layer / "sub"), (snap / "inner", snap)):     # the same tree, or one inside
            e = _refused(vm, vm.VMIG_EINVAL, out, la, sn, bad_table, out, ctl=c)
            assert "one is inside the other" in str(e)
        for o in (st, snap / "inner" / "t.vmig", snap / "t.vmig"):                  # the snapshot's table, or inside it
            e = _refused(vm, vm.VMIG_EINVAL, out, layer, snap, st, o, ctl=c)
            assert "snap_dir" in str(e)
        # 2. a control cancelled before the call, ahead of a missing directory
        e = _refused(vm, vm.VMIG_ECANCELED, out, missing, snap, bad_table, out, ctl=c)
        assert "before the call started" in str(e)
        assert c.progress()["running"] == 0
    # 3. VMIG_ENOTDIR for either directory, ahead of a bad table
    _refused(vm, vm.VMIG_ENOTDIR, out, missing, snap, bad_table, out)
    _refused(vm, vm.VMIG_ENOTDIR, out, layer / "a", snap, st, out)
    _refused(vm, vm.VMIG_ENOTDIR, out, layer, missing, bad_table, out)
    _refused(vm, vm.VMIG_ENOTDIR, out, layer, snap / "a", st, out, lt)
    # 4. VMIG_ETABLE: either table, ahead of the GPU check
    _refused(vm, vm.VMIG_ETABLE, out, layer, snap, bad_table, out)
    _refused(vm, vm.VMIG_ETABLE, out, layer, snap, missing, out)
    _refused(vm, vm.VMIG_ETABLE, out, layer, snap, st, out, bad_table)
    _refused(vm, vm.VMIG_ETABLE, out, layer, snap, st, out, block_bytes=65536)          # the tables are at 4 MiB
    assert _state(shm_tmp) == before


def test_rollback_precancelled_returns_ecanceled(vm, shm_tmp):
    layer, snap, st, lt = _trees(vm, shm_tmp)
    before = _state(shm_tmp)
    with vm.Ctl() as c:
        c.cancel()
        with pytest.raises(vm.VmigError) as ei:
            vm.rollback_layer(layer, snap, st, lt, lt, ctl=c)          # out_table == layer_table is allowed
        assert ei.value.code == vm.VMIG_ECANCELED and "before the call started" in str(ei.value)
        p = c.progress()
        assert p["running"] == 0 and p["bytes_hashed"] == 0
    assert _state(shm_tmp) == before


def test_rollback_has_no_cpu_fallback(vm, shm_tmp):
    if not _no_gpu(vm):
        pytest.skip("a GPU is present; tests/test_rollback.py covers the data path")
    layer, snap, st, lt = _trees(vm, shm_tmp)
    before = _state(shm_tmp)
    rs = vm.RollbackStats()
    rs.files_kept = 77
    for table in (None, lt):
        rc = vm.lib().vmig_rollback_layer(os.fsencode(layer), None if table is None else os.fsencode(table), os.fsencode(snap),
                                          os.fsencode(st), os.fsencode(shm_tmp / "out.vmig"), None, None, ctypes.byref(rs))
        assert rc == vm.VMIG_ENOGPU
    assert rs.files_kept == 77
    assert _state(shm_tmp) == before


def test_rollback_host_side_unit(tmp_path):
    """csrc/vmig_rollback.cpp with the compare's, the scrub's and the walk's modules alone (no GPU, no CUDA)."""
    exe_dir = Path(tempfile.mkdtemp(prefix="vmig_rbunit_"))             # /dev/shm may be mounted noexec
    try:
        exe = exe_dir / "rollback_unit"
        csrc = ROOT / "gpu-docker-api_b200" / "csrc"
        subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-pthread", "-I", str(csrc), str(ROOT / "tests" / "rollback_unit.cpp"),
                        str(csrc / "vmig_rollback.cpp"), str(csrc / "vmig_compare.cpp"), str(csrc / "vmig_scrub.cpp"),
                        str(csrc / "vmig_tree.cpp"), "-o", str(exe)], check=True)
        work = tmp_path / "work"
        work.mkdir()
        r = subprocess.run([str(exe), str(work)], capture_output=True, text=True, timeout=120)
        assert r.returncode == 0 and "rollback unit ok" in r.stdout, r.stdout + r.stderr
    finally:
        shutil.rmtree(exe_dir, ignore_errors=True)
