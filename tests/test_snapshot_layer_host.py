"""vmig_snapshot_layer without a GPU: the C layout of vmig_layer_snapshot_stats, every refusal in its order with nothing
touched, a pre-cancelled control, no CPU fallback, and the plan of the call (which layer blocks are read, which trusted
files need no read, what trusts nothing) as a unit program built with g++ alone."""
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
    """A layer, a destination and a base with their (zero-hash) tables; only the missing GPU or the arguments can fail."""
    layer, dst, base = root / "layer", root / "dst", root / "base"
    for d, n in ((layer, 5000), (base, 6000)):
        (d / "sub").mkdir(parents=True)
        (d / "a").write_bytes(b"x" * n)
        (d / "sub" / "b").write_bytes(b"y" * 70)
    dst.mkdir()
    vm.manifest(base, root / "base.vmig")
    vm.manifest(layer, root / "layer.vmig")
    return layer, dst, base, root / "base.vmig", root / "layer.vmig"


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


def _refused(vm, code, out, layer, dst, base, bt, o, lt, **kw):
    with pytest.raises(vm.VmigError) as ei:
        vm.snapshot_layer(layer, dst, base, bt, o, lt, **kw)
    assert ei.value.code == code, (layer, dst, base, bt, o, lt, kw, ei.value)
    assert not out.exists() and not any(n.startswith(out.name) for n in os.listdir(out.parent))
    return ei.value


def test_layer_snapshot_stats_layout_matches_header(vm):
    exe_dir = Path(tempfile.mkdtemp(prefix="vmig_lslayout_"))           # /dev/shm may be mounted noexec
    try:
        exe = exe_dir / "snapshot_layer_layout"
        subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", str(ROOT / "include"),
                        str(ROOT / "tests" / "snapshot_layer_layout.c"), "-o", str(exe)], check=True)
        out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    finally:
        shutil.rmtree(exe_dir, ignore_errors=True)
    S = vm.LayerSnapshotStats
    assert out[1] == f"{ctypes.sizeof(S)}:" + ",".join(str(getattr(S, n).offset) for n in (
        "files_linked", "bytes_linked", "files_backfilled", "bytes_backfilled", "files_base_untrusted", "files_trusted",
        "bytes_trusted", "files_read", "bytes_read", "reserved"))
    assert ctypes.sizeof(S) == 104 and out[2] == "abi=2"
    assert "vmig_snapshot_layer" in vm.EXPORTS and hasattr(vm.lib(), "vmig_snapshot_layer")


def test_snapshot_layer_refusals_in_order(vm, shm_tmp):
    layer, dst, base, bt, lt = _trees(vm, shm_tmp)
    out = shm_tmp / "out.vmig"
    missing = shm_tmp / "nowhere"
    bad = shm_tmp / "bad.vmig"
    bad.write_bytes(b"not a table")
    (base / "inner").mkdir()
    (layer / "inner").mkdir()
    (dst / "x").mkdir()
    before = _state(shm_tmp)
    good = [layer, dst, base, bt, out, lt]
    # 1. VMIG_EINVAL, ahead of a cancelled control, a missing directory and a bad table: each of the six paths
    for i in range(6):
        for v in (None, ""):
            a = list(good)
            a[i] = v
            e = _refused(vm, vm.VMIG_EINVAL, out, *a)
            assert "NULL/empty" in str(e)
    with vm.Ctl() as c:
        c.cancel()
        args = (missing, missing, missing, bad, out, bad)
        for flags in (vm.F_HASH_ONLY, vm.F_MOVE_SRC, vm.F_CUFILE, 0x8000):
            _refused(vm, vm.VMIG_EINVAL, out, *args, flags=flags, ctl=c)
        _refused(vm, vm.VMIG_EINVAL, out, *args, block_bytes=4097, ctl=c)
        for la, d, b in ((layer, dst, dst), (layer, dst, dst / "x"), (layer, base / "inner", base),       # dst / base
                         (layer, layer, base), (layer, layer / "inner", base), (dst / "x", dst, base),    # dst / layer
                         (layer, dst, layer), (layer / "inner", dst, layer), (base / "inner", dst, base)):  # base / layer
            e = _refused(vm, vm.VMIG_EINVAL, out, la, d, b, bad, out, bad, ctl=c)
            assert "one is inside the other" in str(e)
        for o in (bt, base / "t.vmig", base / "inner" / "t.vmig", layer / "t.vmig", layer / "inner" / "t.vmig"):
            e = _refused(vm, vm.VMIG_EINVAL, out, layer, dst, base, bt, o, lt, ctl=c)
            assert "out_table" in str(e)
        # 2. a control cancelled before the call, ahead of a missing directory; out_table == layer_table is allowed
        e = _refused(vm, vm.VMIG_ECANCELED, out, missing, dst, base, bad, out, bad, ctl=c)
        assert "before the call started" in str(e)
        with pytest.raises(vm.VmigError) as ei:
            vm.snapshot_layer(layer, dst, base, bt, lt, lt, ctl=c)
        assert ei.value.code == vm.VMIG_ECANCELED
        assert c.progress()["running"] == 0 and c.progress()["bytes_hashed"] == 0
    # 3. VMIG_ENOTDIR for any of the three directories, ahead of a bad table
    _refused(vm, vm.VMIG_ENOTDIR, out, missing, dst, base, bad, out, bad)
    _refused(vm, vm.VMIG_ENOTDIR, out, layer / "a", dst, base, bt, out, lt)
    _refused(vm, vm.VMIG_ENOTDIR, out, layer, missing, base, bad, out, bad)
    _refused(vm, vm.VMIG_ENOTDIR, out, layer, dst, missing, bad, out, bad)
    _refused(vm, vm.VMIG_ENOTDIR, out, layer, dst, base / "a", bt, out, lt)
    # 4. VMIG_ETABLE: either table, ahead of the GPU check
    _refused(vm, vm.VMIG_ETABLE, out, layer, dst, base, bad, out, lt)
    _refused(vm, vm.VMIG_ETABLE, out, layer, dst, base, missing, out, lt)
    _refused(vm, vm.VMIG_ETABLE, out, layer, dst, base, bt, out, bad)
    _refused(vm, vm.VMIG_ETABLE, out, layer, dst, base, bt, out, missing)
    _refused(vm, vm.VMIG_ETABLE, out, layer, dst, base, bt, out, lt, block_bytes=65536)        # the tables are at 4 MiB
    assert _state(shm_tmp) == before


def test_snapshot_layer_has_no_cpu_fallback(vm, shm_tmp):
    if not _no_gpu(vm):
        pytest.skip("a GPU is present; tests/test_snapshot_layer.py covers the data path")
    layer, dst, base, bt, lt = _trees(vm, shm_tmp)
    before = _state(shm_tmp)
    ls = vm.LayerSnapshotStats()
    ls.files_read = 77
    for o in (shm_tmp / "out.vmig", lt):
        rc = vm.lib().vmig_snapshot_layer(*(os.fsencode(p) for p in (layer, lt, dst, base, bt, o)), None, None, ctypes.byref(ls))
        assert rc == vm.VMIG_ENOGPU
    assert ls.files_read == 0                       # cleared before the call, written again only on success
    assert _state(shm_tmp) == before


def test_snapshot_layer_plan_unit(tmp_path):
    """The plan with a layer table: csrc/vmig_plan.cpp with the walk's and the table's modules alone (no GPU, no CUDA)."""
    exe_dir = Path(tempfile.mkdtemp(prefix="vmig_slunit_"))             # /dev/shm may be mounted noexec
    try:
        exe = exe_dir / "snapshot_layer_unit"
        csrc = ROOT / "gpu-docker-api_b200" / "csrc"
        subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-pthread", "-I", str(csrc),
                        str(ROOT / "tests" / "snapshot_layer_unit.cpp"), str(csrc / "vmig_plan.cpp"), str(csrc / "vmig_tree.cpp"),
                        str(csrc / "vmig_table.cpp"), "-o", str(exe)], check=True)
        work = tmp_path / "work"
        work.mkdir()
        r = subprocess.run([str(exe), str(work)], capture_output=True, text=True, timeout=120)
        assert r.returncode == 0 and "snapshot layer unit ok" in r.stdout, r.stdout + r.stderr
    finally:
        shutil.rmtree(exe_dir, ignore_errors=True)
