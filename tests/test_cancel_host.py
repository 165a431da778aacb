"""Call controls (vmig_ctl_*) without a GPU: the C layout of vmig_progress and vmig_opts.ctl, id bookkeeping, a control
that is cancelled before its call starts, and the cancel checkpoints of the host-side steps (unit program)."""
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


def test_progress_and_opts_layout_match_header(vm):
    exe_dir = Path(tempfile.mkdtemp(prefix="vmig_proglayout_"))         # /dev/shm may be mounted noexec
    exe = exe_dir / "progress_layout"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", str(ROOT / "include"), str(ROOT / "tests" / "progress_layout.c"),
                    "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    shutil.rmtree(exe_dir, ignore_errors=True)
    P, O = vm.Progress, vm.Opts
    assert out[1] == f"{ctypes.sizeof(P)}:" + ",".join(str(getattr(P, n).offset) for n in (
        "phase", "running", "bytes_total", "blocks_total", "bytes_hashed", "blocks_hashed", "bytes_written", "bytes_verified", "reserved"))
    assert out[3] == f"{ctypes.sizeof(O)}:{O.ctl.offset},{O.reserved.offset}"
    assert O.ctl.offset == 24 and ctypes.sizeof(O) == 32 and ctypes.sizeof(P) == 88
    assert out[4] == "abi=2" and out[5] == f"ecanceled={vm.VMIG_ECANCELED}" and vm.VMIG_ECANCELED == -12
    assert out[6] == "phases=" + ",".join(str(i) for i in range(len(vm.PHASES)))


def test_control_ids_are_distinct_and_never_reused(vm):
    ids = []
    for _ in range(5):
        c = vm.Ctl()
        ids.append(c.id)
        c.close()
    with vm.Ctl() as a, vm.Ctl() as b:
        ids += [a.id, b.id]
    assert len(set(ids)) == len(ids) and 0 not in ids


def test_unknown_or_closed_control_is_refused(vm):
    c = vm.Ctl()
    cid = c.id
    c.close()
    lib = vm.lib()
    p = vm.Progress()
    for bad in (cid, 0, 0xFFFFFFFF):
        assert lib.vmig_ctl_cancel(bad) == vm.VMIG_EINVAL
        assert lib.vmig_ctl_progress(bad, ctypes.byref(p)) == vm.VMIG_EINVAL
        assert lib.vmig_ctl_close(bad) == vm.VMIG_EINVAL


def test_fresh_control_is_idle_with_zero_counters(vm):
    with vm.Ctl() as c:
        p = c.progress()
        assert p.pop("phase_name") == "IDLE"
        assert set(p.values()) == {0}, p
        c.cancel()
        c.cancel()                          # idempotent
        assert c.progress()["running"] == 0


def test_unknown_control_in_opts_is_refused_before_the_destination(vm, shm_tmp):
    src, dst = shm_tmp / "s", shm_tmp / "d"
    src.mkdir(), dst.mkdir()
    (src / "a").write_bytes(b"x" * 5000)
    c = vm.Ctl()
    closed = c.id
    c.close()
    for bad in (closed, 0xFFFFFF00):
        o = vm.Opts(ctl=bad)
        rc = vm.lib().vmig_migrate_tree(os.fsencode(src), os.fsencode(dst), None, os.fsencode(shm_tmp / "t.vmig"), ctypes.byref(o), None)
        assert rc == vm.VMIG_EINVAL and "not an open control" in vm.last_error()
    assert os.listdir(dst) == [] and not (shm_tmp / "t.vmig").exists()


def test_precancelled_control_returns_ecanceled_not_enogpu(vm, shm_tmp):
    if not _no_gpu(vm):
        pytest.skip("a GPU is present; tests/test_cancel.py covers the data path")
    src, dst, snap = shm_tmp / "s", shm_tmp / "d", shm_tmp / "snap"
    (src / "sub").mkdir(parents=True), dst.mkdir(), snap.mkdir()
    (src / "a").write_bytes(b"x" * 5000), (src / "sub" / "b").write_bytes(b"y" * 70)
    vm.manifest(src, shm_tmp / "snap.vmig")
    import numpy as np
    buf = np.arange(4096, dtype=np.uint8)
    out = np.zeros_like(buf)
    with vm.Ctl() as c:
        c.cancel()
        calls = [
            lambda: vm.migrate_tree(src, dst, None, shm_tmp / "t.vmig", ctl=c),
            lambda: vm.migrate_tree(src, dst, None, shm_tmp / "t.vmig", flags=vm.MOVE_DIR_FLAGS, ctl=c),
            lambda: vm.restore_tree(src, shm_tmp / "snap.vmig", dst, None, shm_tmp / "t.vmig", ctl=c),
            lambda: vm.snapshot_tree(src, snap, None, None, shm_tmp / "t.vmig", ctl=c),
            lambda: vm.migrate_buffer(buf, out, ctl=c),
        ]
        for call in calls:
            with pytest.raises(vm.VmigError) as ei:
                call()
            assert ei.value.code == vm.VMIG_ECANCELED, ei.value
            assert "before the call started" in str(ei.value)
            p = c.progress()
            assert p["running"] == 0 and p["phase_name"] == "IDLE"
    assert os.listdir(dst) == [] and os.listdir(snap) == [] and not (shm_tmp / "t.vmig").exists()
    assert not any(n.startswith("t.vmig") for n in os.listdir(shm_tmp))
    assert (src / "a").read_bytes() == b"x" * 5000 and (out == 0).all()
    with pytest.raises(vm.VmigError) as ei:                            # without the control: no CPU fallback, as before
        vm.migrate_tree(src, dst, None, shm_tmp / "t.vmig")
    assert ei.value.code == vm.VMIG_ENOGPU


def test_cancel_checkpoints_unit(tmp_path, shm_tmp):
    """copy_range (a snapshot's backfill from its base) stops at a 64 MiB chunk boundary once the latch is set; the walk,
    prune, metadata replay and the table write start nothing after it (csrc/vmig_tree.cpp, csrc/vmig_table.cpp)."""
    exe = tmp_path / "cancel_unit"
    csrc = ROOT / "gpu-docker-api_b200" / "csrc"
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-pthread", "-I", str(csrc), str(ROOT / "tests" / "cancel_unit.cpp"),
                    str(csrc / "vmig_tree.cpp"), str(csrc / "vmig_table.cpp"), "-o", str(exe)], check=True)
    work = shm_tmp if shutil.disk_usage(shm_tmp).free > (1 << 30) else tmp_path / "work"
    work.mkdir(exist_ok=True)
    r = subprocess.run([str(exe), str(work)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "cancel unit ok" in r.stdout, r.stdout + r.stderr
