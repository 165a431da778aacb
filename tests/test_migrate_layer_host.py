"""vmig_migrate_layer without a GPU: the C layout of vmig_layer_migrate_stats, every refusal in its order with nothing
touched, a pre-cancelled control, no CPU fallback, and the plan of the call (which source blocks are read, which trusted
files need no read, what trusts nothing) and its identity-recording rule as a unit program built with g++ alone."""
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
    """A source, a destination and their (zero-hash) tables; only the missing GPU or the arguments can fail."""
    src, dst = root / "src", root / "dst"
    for d, n in ((src, 5000), (dst, 6000)):
        (d / "sub").mkdir(parents=True)
        (d / "a").write_bytes(b"x" * n)
        (d / "sub" / "b").write_bytes(b"y" * 70)
    vm.manifest(src, root / "src.vmig")
    vm.manifest(dst, root / "prior.vmig")
    return src, dst, root / "src.vmig", root / "prior.vmig"


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


def _refused(vm, code, outs, src, st, dst, pt, o, so, **kw):
    with pytest.raises(vm.VmigError) as ei:
        vm.migrate_layer(src, st, dst, pt, o, so, **kw)
    assert ei.value.code == code, (src, st, dst, pt, o, so, kw, ei.value)
    for out in outs:
        assert not out.exists() and not any(n.startswith(out.name) for n in os.listdir(out.parent))
    return ei.value


def test_layer_migrate_stats_layout_matches_header(vm):
    exe_dir = Path(tempfile.mkdtemp(prefix="vmig_lmlayout_"))           # /dev/shm may be mounted noexec
    try:
        exe = exe_dir / "migrate_layer_layout"
        subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", str(ROOT / "include"),
                        str(ROOT / "tests" / "migrate_layer_layout.c"), "-o", str(exe)], check=True)
        out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    finally:
        shutil.rmtree(exe_dir, ignore_errors=True)
    S = vm.LayerMigrateStats
    assert out[1] == f"{ctypes.sizeof(S)}:" + ",".join(str(getattr(S, n).offset) for n in (
        "files_trusted", "bytes_trusted", "files_read", "bytes_read", "files_unread", "files_verified", "bytes_verified",
        "src_recorded", "src_unrecorded", "reserved"))
    assert ctypes.sizeof(S) == 104 and out[2] == "abi=2"
    assert "vmig_migrate_layer" in vm.EXPORTS and hasattr(vm.lib(), "vmig_migrate_layer")


def test_migrate_layer_refusals_in_order(vm, shm_tmp):
    src, dst, st, pt = _trees(vm, shm_tmp)
    tabs = shm_tmp / "tabs"
    tabs.mkdir()
    out, so = tabs / "out.vmig", tabs / "src_out.vmig"
    outs = (out, so)
    missing = shm_tmp / "nowhere"
    bad = shm_tmp / "bad.vmig"
    bad.write_bytes(b"not a table")
    (src / "inner").mkdir()
    (dst / "x").mkdir()
    before = _state(shm_tmp)
    # 1. VMIG_EINVAL, ahead of a cancelled control, a missing directory and a bad table
    for s_, d_ in ((None, dst), ("", dst), (src, None), (src, "")):
        e = _refused(vm, vm.VMIG_EINVAL, outs, s_, st, d_, pt, out, so)
        assert "NULL/empty" in str(e)
    with vm.Ctl() as c:
        c.cancel()
        for flags in (vm.F_HASH_ONLY, vm.F_MOVE_SRC, vm.F_CUFILE, 0x8000):
            _refused(vm, vm.VMIG_EINVAL, outs, missing, bad, missing, bad, out, so, flags=flags, ctl=c)
        _refused(vm, vm.VMIG_EINVAL, outs, missing, bad, missing, bad, out, so, block_bytes=4097, ctl=c)
        for s_, d_ in ((src, src), (src, src / "inner"), (dst / "x", dst)):
            e = _refused(vm, vm.VMIG_EINVAL, outs, s_, bad, d_, bad, out, so, ctl=c)
            assert "one is inside the other" in str(e)
        e = _refused(vm, vm.VMIG_EINVAL, outs, src, bad, dst, bad, out, tabs / "." / "out.vmig", ctl=c)
        assert "same file" in str(e)
        for o, s_o in ((src / "t.vmig", so), (src / "inner" / "t.vmig", None), (out, src / "t.vmig"), (None, src / "inner" / "t.vmig")):
            e = _refused(vm, vm.VMIG_EINVAL, outs, src, bad, dst, bad, o, s_o, ctl=c)
            assert "inside src_dir" in str(e)
        for s_o in (dst / "t.vmig", dst / "x" / "t.vmig"):
            e = _refused(vm, vm.VMIG_EINVAL, outs, src, bad, dst, bad, out, s_o, ctl=c)
            assert "inside dst_dir" in str(e)
        # 2. a control cancelled before the call, ahead of a missing directory and a bad table
        e = _refused(vm, vm.VMIG_ECANCELED, outs, missing, bad, missing, bad, out, so, ctl=c)
        assert "before the call started" in str(e)
        _refused(vm, vm.VMIG_ECANCELED, outs, src, None, dst, None, None, None, ctl=c)
        assert c.progress()["running"] == 0 and c.progress()["bytes_hashed"] == 0
    # 3. VMIG_ENOTDIR for either directory, ahead of a bad table
    _refused(vm, vm.VMIG_ENOTDIR, outs, missing, bad, dst, bad, out, so)
    _refused(vm, vm.VMIG_ENOTDIR, outs, src / "a", st, dst, pt, out, so)
    _refused(vm, vm.VMIG_ENOTDIR, outs, src, bad, missing, bad, out, so)
    _refused(vm, vm.VMIG_ENOTDIR, outs, src, st, dst / "a", pt, out, so)
    # 4. VMIG_ETABLE: either input table, ahead of the GPU check
    _refused(vm, vm.VMIG_ETABLE, outs, src, bad, dst, pt, out, so)
    _refused(vm, vm.VMIG_ETABLE, outs, src, missing, dst, None, out, so)
    _refused(vm, vm.VMIG_ETABLE, outs, src, st, dst, bad, out, so)
    _refused(vm, vm.VMIG_ETABLE, outs, src, None, dst, missing, out, so)
    _refused(vm, vm.VMIG_ETABLE, outs, src, st, dst, None, out, so, block_bytes=65536)       # the tables are at 4 MiB
    _refused(vm, vm.VMIG_ETABLE, outs, src, None, dst, pt, out, so, block_bytes=65536)
    assert _state(shm_tmp) == before


def test_migrate_layer_has_no_cpu_fallback(vm, shm_tmp):
    if not _no_gpu(vm):
        pytest.skip("a GPU is present; tests/test_migrate_layer.py covers the data path")
    src, dst, st, pt = _trees(vm, shm_tmp)
    tabs = shm_tmp / "tabs"
    tabs.mkdir()
    before = _state(shm_tmp)
    ms = vm.LayerMigrateStats()
    ms.files_read = 77
    for args in ((src, st, dst, pt, tabs / "out.vmig", tabs / "src_out.vmig"), (src, None, dst, None, None, None)):
        rc = vm.lib().vmig_migrate_layer(*(None if p is None else os.fsencode(p) for p in args), None, None, ctypes.byref(ms))
        assert rc == vm.VMIG_ENOGPU
    assert ms.files_read == 0                       # cleared before the call, written again only on success
    assert _state(shm_tmp) == before


def test_migrate_layer_plan_unit(tmp_path):
    """The plan with a source table and a prior table: csrc/vmig_plan.cpp with the walk's and the table's modules alone
    (no GPU, no CUDA)."""
    exe_dir = Path(tempfile.mkdtemp(prefix="vmig_mlunit_"))             # /dev/shm may be mounted noexec
    try:
        exe = exe_dir / "migrate_layer_unit"
        csrc = ROOT / "gpu-docker-api_b200" / "csrc"
        subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-pthread", "-I", str(csrc),
                        str(ROOT / "tests" / "migrate_layer_unit.cpp"), str(csrc / "vmig_plan.cpp"), str(csrc / "vmig_tree.cpp"),
                        str(csrc / "vmig_table.cpp"), "-o", str(exe)], check=True)
        work = tmp_path / "work"
        work.mkdir()
        r = subprocess.run([str(exe), str(work)], capture_output=True, text=True, timeout=120)
        assert r.returncode == 0 and "migrate layer unit ok" in r.stdout, r.stdout + r.stderr
    finally:
        shutil.rmtree(exe_dir, ignore_errors=True)
