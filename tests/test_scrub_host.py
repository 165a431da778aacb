"""vmig_scrub_store without a GPU: the C layout of vmig_scrub_stats, argument checks, a pre-cancelled control, no CPU
fallback, and the host side of the scrub (merge, inode grouping, report, reader) as a unit program."""
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


def _store(vm, root: Path):
    """Two versions and their (zero-hash) tables; only the missing GPU or the arguments can fail a scrub of them."""
    pairs = []
    for k in (1, 2):
        d = root / f"rs-{k}" / "diff"
        (d / "sub").mkdir(parents=True)
        (d / "a").write_bytes(b"x" * 5000)
        (d / "sub" / "b").write_bytes(b"y" * (70 + k))
        vm.manifest(d, root / f"rs-{k}" / "blocks.vmig")
        pairs.append((d, root / f"rs-{k}" / "blocks.vmig"))
    return pairs


def _snapshot_state(root: Path):
    out = {}
    for dp, dns, fns in os.walk(root):
        for n in dns + fns:
            p = os.path.join(dp, n)
            s = os.lstat(p)
            out[p] = (s.st_ino, s.st_nlink, s.st_mode, s.st_size, s.st_mtime_ns, s.st_ctime_ns)
    return out


def test_scrub_stats_layout_matches_header(vm):
    exe_dir = Path(tempfile.mkdtemp(prefix="vmig_scrublayout_"))         # /dev/shm may be mounted noexec
    try:
        exe = exe_dir / "scrub_layout"
        subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", str(ROOT / "include"), str(ROOT / "tests" / "scrub_layout.c"),
                        "-o", str(exe)], check=True)
        out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    finally:
        shutil.rmtree(exe_dir, ignore_errors=True)
    S = vm.ScrubStats
    assert out[1] == f"{ctypes.sizeof(S)}:" + ",".join(str(getattr(S, n).offset) for n in (
        "versions", "versions_damaged", "bytes_referenced", "bytes_unique", "files_damaged", "blocks_damaged",
        "files_unreadable", "reserved"))
    assert ctypes.sizeof(S) == 88 and out[2] == "abi=2"
    assert "vmig_scrub_store" in vm.EXPORTS and hasattr(vm.lib(), "vmig_scrub_store")


def test_scrub_refuses_bad_arguments(vm, shm_tmp):
    pairs = _store(vm, shm_tmp)
    before = _snapshot_state(shm_tmp)
    report = shm_tmp / "scrub.txt"
    for flags in (vm.F_HASH_ONLY, vm.F_VERIFY, vm.F_PRUNE, vm.F_MOVE_SRC, vm.F_CUFILE, vm.F_MTIME_NS, 0x8000):
        with pytest.raises(vm.VmigError) as ei:
            vm.scrub_store(pairs, report, flags=flags)
        assert ei.value.code == vm.VMIG_EINVAL, (flags, ei.value)
    with pytest.raises(vm.VmigError) as ei:
        vm.scrub_store([], report)
    assert ei.value.code == vm.VMIG_EINVAL and "n == 0" in str(ei.value)
    with pytest.raises(vm.VmigError) as ei:
        vm.scrub_store(pairs, report, block_bytes=4097)
    assert ei.value.code == vm.VMIG_EINVAL
    lib = vm.lib()
    assert lib.vmig_scrub_store(2, None, None, None, None, None, None, None) == vm.VMIG_EINVAL
    assert not report.exists() and _snapshot_state(shm_tmp) == before


def test_scrub_precancelled_returns_ecanceled(vm, shm_tmp):
    pairs = _store(vm, shm_tmp)
    before = _snapshot_state(shm_tmp)
    report = shm_tmp / "scrub.txt"
    with vm.Ctl() as c:
        c.cancel()
        with pytest.raises(vm.VmigError) as ei:
            vm.scrub_store(pairs, report, ctl=c)
        assert ei.value.code == vm.VMIG_ECANCELED and "before the call started" in str(ei.value)
        p = c.progress()
        assert p["running"] == 0 and p["bytes_hashed"] == 0
    assert not report.exists() and not any(n.startswith("scrub.txt") for n in os.listdir(shm_tmp))
    assert _snapshot_state(shm_tmp) == before


def test_scrub_has_no_cpu_fallback(vm, shm_tmp):
    if not _no_gpu(vm):
        pytest.skip("a GPU is present; tests/test_scrub.py covers the data path")
    pairs = _store(vm, shm_tmp)
    before = _snapshot_state(shm_tmp)
    tables = [t.read_bytes() for _, t in pairs]
    report = shm_tmp / "scrub.txt"
    verdicts = (ctypes.c_int32 * 2)(7, 7)
    dirs = (ctypes.c_char_p * 2)(*[os.fsencode(d) for d, _ in pairs])
    tabs = (ctypes.c_char_p * 2)(*[os.fsencode(t) for _, t in pairs])
    rc = vm.lib().vmig_scrub_store(2, dirs, tabs, os.fsencode(report), verdicts, None, None, None)
    assert rc == vm.VMIG_ENOGPU
    assert list(verdicts) == [7, 7] and not report.exists()
    assert not any(n.startswith("scrub.txt") for n in os.listdir(shm_tmp))
    assert _snapshot_state(shm_tmp) == before and [t.read_bytes() for _, t in pairs] == tables


def test_report_path_unescape(vm):
    assert vm.unescape_report_path("a\\tb\\nc\\\\d\\x01e") == b"a\tb\nc\\d\x01e"
    with pytest.raises(ValueError):
        vm.unescape_report_path("bad\\q")


def test_scrub_host_side_unit(tmp_path):
    """csrc/vmig_scrub.cpp alone (no GPU, no CUDA): the multi-difference merge, the inode grouping, report escaping and
    ordering, and the reader that turns a failing descriptor into an `unreadable` finding."""
    exe = tmp_path / "scrub_unit"
    csrc = ROOT / "gpu-docker-api_b200" / "csrc"
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-pthread", "-I", str(csrc), str(ROOT / "tests" / "scrub_unit.cpp"),
                    str(csrc / "vmig_scrub.cpp"), str(csrc / "vmig_tree.cpp"), "-o", str(exe)], check=True)
    work = tmp_path / "work"
    work.mkdir()
    r = subprocess.run([str(exe), str(work)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "scrub unit ok" in r.stdout, r.stdout + r.stderr
