"""vmig_compare_snapshot without a GPU: the C layout of vmig_compare_stats, every refusal in its order, a pre-cancelled
control, no CPU fallback, the report parser on awkward names, and the host side of the compare (merge, hard-link
groups, read plan, bytes_restore) as a unit program built with g++ alone."""
import ctypes
import os
import shutil
import subprocess
import tempfile
from pathlib import Path

import pytest

import _layer_model as lm

ROOT = Path(__file__).resolve().parent.parent


def _no_gpu(vm):
    try:
        vm.device_count()
        return False
    except vm.VmigError:
        return True


def _trees(vm, root: Path):
    """A layer and a snapshot with its (zero-hash) table; only the missing GPU or the arguments can fail a compare."""
    layer, snap = root / "layer", root / "snap"
    for d, n in ((layer, 5000), (snap, 6000)):
        (d / "sub").mkdir(parents=True)
        (d / "a").write_bytes(b"x" * n)
        (d / "sub" / "b").write_bytes(b"y" * 70)
    vm.manifest(snap, root / "snap.vmig")
    vm.manifest(layer, root / "layer.vmig")
    return layer, snap, root / "snap.vmig", root / "layer.vmig"


def _state(root: Path):
    out = {}
    for dp, dns, fns in os.walk(root):
        for n in dns + fns:
            p = os.path.join(dp, n)
            s = os.lstat(p)
            out[p] = (s.st_ino, s.st_nlink, s.st_mode, s.st_size, s.st_mtime_ns, s.st_ctime_ns)
    return out


def _refused(vm, code, report, *args, **kw):
    with pytest.raises(vm.VmigError) as ei:
        vm.compare_snapshot(*args, report, **kw)
    assert ei.value.code == code, (args, kw, ei.value)
    assert not report.exists() and not any(n.startswith(report.name) for n in os.listdir(report.parent))
    return ei.value


def test_compare_stats_layout_matches_header(vm):
    exe_dir = Path(tempfile.mkdtemp(prefix="vmig_cmplayout_"))          # /dev/shm may be mounted noexec
    try:
        exe = exe_dir / "compare_layout"
        subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", str(ROOT / "include"), str(ROOT / "tests" / "compare_layout.c"),
                        "-o", str(exe)], check=True)
        out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    finally:
        shutil.rmtree(exe_dir, ignore_errors=True)
    S = vm.CompareStats
    assert out[1] == f"{ctypes.sizeof(S)}:" + ",".join(str(getattr(S, n).offset) for n in (
        "paths_added", "paths_removed", "paths_changed", "files_changed", "blocks_changed", "bytes_restore", "files_read",
        "bytes_read", "files_trusted", "files_shared", "reserved"))
    assert ctypes.sizeof(S) == 112 and out[2] == "abi=2"
    assert "vmig_compare_snapshot" in vm.EXPORTS and hasattr(vm.lib(), "vmig_compare_snapshot")


def test_compare_refusals_in_order(vm, shm_tmp):
    layer, snap, st, lt = _trees(vm, shm_tmp)
    report = shm_tmp / "cmp.txt"
    missing = shm_tmp / "nowhere"
    bad_table = shm_tmp / "bad.vmig"
    bad_table.write_bytes(b"not a table")
    before = _state(shm_tmp)
    # 1. VMIG_EINVAL, ahead of a cancelled control, a missing directory and a bad table
    for a in ((None, snap, st), ("", snap, st), (layer, None, st), (layer, "", st), (layer, snap, None), (layer, snap, "")):
        _refused(vm, vm.VMIG_EINVAL, report, *a)
    with vm.Ctl() as c:
        c.cancel()
        for flags in (vm.F_HASH_ONLY, vm.F_VERIFY, vm.F_PRUNE, vm.F_MOVE_SRC, vm.F_CUFILE, 0x8000):
            _refused(vm, vm.VMIG_EINVAL, report, missing, snap, bad_table, flags=flags, ctl=c)
        _refused(vm, vm.VMIG_EINVAL, report, missing, snap, bad_table, block_bytes=4097, ctl=c)
        # 2. a control cancelled before the call, ahead of a missing directory
        e = _refused(vm, vm.VMIG_ECANCELED, report, missing, snap, bad_table, ctl=c)
        assert "before the call started" in str(e)
        assert c.progress()["running"] == 0
    # 3. VMIG_ENOTDIR for either directory, ahead of a bad table
    _refused(vm, vm.VMIG_ENOTDIR, report, missing, snap, bad_table)
    _refused(vm, vm.VMIG_ENOTDIR, report, layer / "a", snap, st)
    _refused(vm, vm.VMIG_ENOTDIR, report, layer, missing, bad_table)
    _refused(vm, vm.VMIG_ENOTDIR, report, layer, snap / "a", st, lt)
    # 4. VMIG_ETABLE: either table, ahead of the GPU check
    _refused(vm, vm.VMIG_ETABLE, report, layer, snap, bad_table)
    _refused(vm, vm.VMIG_ETABLE, report, layer, snap, missing)
    _refused(vm, vm.VMIG_ETABLE, report, layer, snap, st, bad_table)
    _refused(vm, vm.VMIG_ETABLE, report, layer, snap, st, block_bytes=65536)       # the tables are at 4 MiB
    assert _state(shm_tmp) == before


def test_compare_precancelled_returns_ecanceled(vm, shm_tmp):
    layer, snap, st, lt = _trees(vm, shm_tmp)
    before = _state(shm_tmp)
    report = shm_tmp / "cmp.txt"
    with vm.Ctl() as c:
        c.cancel()
        with pytest.raises(vm.VmigError) as ei:
            vm.compare_snapshot(layer, snap, st, report, lt, ctl=c)
        assert ei.value.code == vm.VMIG_ECANCELED and "before the call started" in str(ei.value)
        p = c.progress()
        assert p["running"] == 0 and p["bytes_hashed"] == 0
    assert not any(n.startswith("cmp.txt") for n in os.listdir(shm_tmp)) and _state(shm_tmp) == before


def test_compare_has_no_cpu_fallback(vm, shm_tmp):
    if not _no_gpu(vm):
        pytest.skip("a GPU is present; tests/test_compare.py covers the data path")
    layer, snap, st, lt = _trees(vm, shm_tmp)
    before = _state(shm_tmp)
    report = shm_tmp / "cmp.txt"
    cs = vm.CompareStats()
    cs.paths_added = 77
    for table in (None, lt):
        rc = vm.lib().vmig_compare_snapshot(os.fsencode(layer), None if table is None else os.fsencode(table), os.fsencode(snap),
                                            os.fsencode(st), os.fsencode(report), None, None, ctypes.byref(cs))
        assert rc == vm.VMIG_ENOGPU
    assert cs.paths_added == 77
    assert not any(n.startswith("cmp.txt") for n in os.listdir(shm_tmp)) and _state(shm_tmp) == before


def _escape(raw: bytes) -> bytes:
    """The report's path escaping, restated (include/vmig.h)."""
    out = bytearray()
    for c in raw:
        out += {0x5C: b"\\\\", 0x09: b"\\t", 0x0A: b"\\n"}.get(c, b"\\x%02x" % c if c < 0x20 else bytes([c]))
    return bytes(out)


def test_parse_compare_report_round_trips_awkward_names(vm, tmp_path):
    names = [lm.awkward(i) for i in range(len(lm.NAME_POOL))] + ["ctl\x01\x1fchar", "back\\slash"]
    lines, want = [], []
    for i, n in enumerate(names):
        e = _escape(os.fsencode(n))
        lines.append(b"block\t" + e + b"\t%d\t%016x\t%016x\n" % (i, i + 1, 0xFFFFFFFFFFFFFFFF - i))
        want.append({"kind": "block", "path": n, "block": i, "layer": f"{i + 1:016x}", "snap": f"{0xFFFFFFFFFFFFFFFF - i:016x}"})
        lines.append(b"target\t" + e + b"\t-\t" + e + b"\t-\n")
        want.append({"kind": "target", "path": n, "block": None, "layer": n, "snap": None})
        lines.append(b"hardlink\t" + e + b"\t-\t-\t" + e + b"\n")
        want.append({"kind": "hardlink", "path": n, "block": None, "layer": None, "snap": n})
    lines.append(b"added\t.dot/x\t-\t-\t-\n")
    want.append({"kind": "added", "path": ".dot/x", "block": None, "layer": None, "snap": None})
    report = tmp_path / "cmp.txt"
    report.write_bytes(b"".join(lines))
    assert vm.parse_compare_report(report) == want
    report.write_bytes(b"")
    assert vm.parse_compare_report(report) == []


def test_compare_host_side_unit(tmp_path):
    """csrc/vmig_compare.cpp with the scrub's and the walk's modules alone (no GPU, no CUDA): findings for every kind
    change, sort order and mtime precision, hard-link groups, the read plan and bytes_restore."""
    exe_dir = Path(tempfile.mkdtemp(prefix="vmig_cmpunit_"))            # /dev/shm may be mounted noexec
    try:
        exe = exe_dir / "compare_unit"
        csrc = ROOT / "gpu-docker-api_b200" / "csrc"
        subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-pthread", "-I", str(csrc), str(ROOT / "tests" / "compare_unit.cpp"),
                        str(csrc / "vmig_compare.cpp"), str(csrc / "vmig_scrub.cpp"), str(csrc / "vmig_tree.cpp"), "-o", str(exe)],
                       check=True)
        work = tmp_path / "work"
        work.mkdir()
        r = subprocess.run([str(exe), str(work)], capture_output=True, text=True, timeout=120)
        assert r.returncode == 0 and "compare unit ok" in r.stdout, r.stdout + r.stderr
    finally:
        shutil.rmtree(exe_dir, ignore_errors=True)
