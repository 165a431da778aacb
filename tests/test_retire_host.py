"""vmig_retire_versions without a GPU: the C layout of vmig_retire_stats, the refusals that touch nothing, a pre-cancelled
control, no CPU fallback, and the host side of the retire (removal counts, stale-record selection, re-stamp decision,
table patch) as a unit program."""
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


def _store(vm, root: Path, n: int = 4):
    """n versions root/rs-k/diff with (zero-hash) tables root/rs-k/blocks.vmig, the file `a` shared by all of them."""
    pairs = []
    for k in range(1, n + 1):
        d = root / f"rs-{k}" / "diff"
        (d / "sub").mkdir(parents=True)
        if k == 1:
            (d / "a").write_bytes(b"x" * 5000)
        else:
            os.link(pairs[0][0] / "a", d / "a")
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
            body = Path(p).read_bytes() if os.path.isfile(p) and not os.path.islink(p) else None
            out[p] = (s.st_ino, s.st_nlink, s.st_mode, s.st_size, s.st_mtime_ns, s.st_ctime_ns, body)
    return out


def test_retire_stats_layout_matches_header(vm):
    exe_dir = Path(tempfile.mkdtemp(prefix="vmig_retirelayout_"))         # /dev/shm may be mounted noexec
    try:
        exe = exe_dir / "retire_layout"
        subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", str(ROOT / "include"), str(ROOT / "tests" / "retire_layout.c"),
                        "-o", str(exe)], check=True)
        out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    finally:
        shutil.rmtree(exe_dir, ignore_errors=True)
    S = vm.RetireStats
    assert out[1] == f"{ctypes.sizeof(S)}:" + ",".join(str(getattr(S, n).offset) for n in (
        "versions_retired", "entries_removed", "files_freed", "bytes_freed", "records_stale", "records_restamped",
        "bytes_rehashed", "tables_rewritten", "reserved"))
    assert ctypes.sizeof(S) == 96 and out[2] == "abi=2"
    assert "vmig_retire_versions" in vm.EXPORTS and hasattr(vm.lib(), "vmig_retire_versions")


def _refused(vm, code, *args, **kw):
    with pytest.raises(vm.VmigError) as ei:
        vm.retire_versions(*args, **kw)
    assert ei.value.code == code, ei.value
    return ei.value


def test_retire_refusals_touch_nothing(vm, shm_tmp):
    store = shm_tmp / "store"
    pairs = _store(vm, store)
    outside = shm_tmp / "outside"
    outside.mkdir()
    (outside / "f").write_bytes(b"keep")
    os.symlink(pairs[2][0], store / "link_to_kept")
    other_bb = store / "other_bb.vmig"
    vm.manifest(pairs[3][0], other_bb, block_bytes=1 << 20)
    (store / "junk.vmig").write_bytes(b"VMIGBT02" + bytes(10))
    before = _snapshot_state(shm_tmp)
    old, kept = pairs[:2], pairs[2:]
    for flags in (vm.F_HASH_ONLY, vm.F_VERIFY, vm.F_PRUNE, vm.F_MOVE_SRC, vm.F_CUFILE, vm.F_MTIME_NS, 0x8000):
        _refused(vm, vm.VMIG_EINVAL, old, kept, flags=flags)
    assert "n_retire + n_keep == 0" in str(_refused(vm, vm.VMIG_EINVAL, [], []))
    _refused(vm, vm.VMIG_EINVAL, old, kept, block_bytes=4097)
    lib = vm.lib()
    assert lib.vmig_retire_versions(2, None, None, 0, None, None, None, None, None) == vm.VMIG_EINVAL
    # the same directory twice, or one inside another, compared by real path
    _refused(vm, vm.VMIG_EINVAL, [pairs[0]], [pairs[0]])
    _refused(vm, vm.VMIG_EINVAL, [pairs[0], pairs[0]], kept)
    _refused(vm, vm.VMIG_EINVAL, [(pairs[2][0] / "sub", store / "x.vmig")], kept)
    _refused(vm, vm.VMIG_EINVAL, [(store, store / "x.vmig")], kept)
    _refused(vm, vm.VMIG_EINVAL, old, [pairs[2], (str(pairs[2][0]) + "/../diff", pairs[3][1])])
    # a retired table that is a kept one, a kept table inside a retired directory
    _refused(vm, vm.VMIG_EINVAL, [(pairs[0][0], pairs[2][1])], kept)
    _refused(vm, vm.VMIG_EINVAL, old, [(pairs[2][0], pairs[0][0] / "sub" / "b")])
    # a retired directory that is a symlink (to a kept one): never followed; a kept directory that is missing
    _refused(vm, vm.VMIG_ENOTDIR, [(store / "link_to_kept", store / "l.vmig")], kept)
    _refused(vm, vm.VMIG_ENOTDIR, [(pairs[0][0] / "a", store / "l.vmig")], kept)
    _refused(vm, vm.VMIG_ENOTDIR, old, [(store / "nowhere", pairs[2][1])])
    # a kept table that does not load, or at another block size
    _refused(vm, vm.VMIG_ETABLE, old, [(pairs[2][0], store / "absent.vmig")])
    _refused(vm, vm.VMIG_ETABLE, old, [(pairs[3][0], other_bb)])
    _refused(vm, vm.VMIG_ETABLE, old, [(pairs[3][0], store / "junk.vmig")])
    assert _snapshot_state(shm_tmp) == before


def test_retire_precancelled_returns_ecanceled(vm, shm_tmp):
    pairs = _store(vm, shm_tmp)
    before = _snapshot_state(shm_tmp)
    with vm.Ctl() as c:
        c.cancel()
        e = _refused(vm, vm.VMIG_ECANCELED, pairs[:2], pairs[2:], ctl=c)
        assert "before the call started" in str(e)
        p = c.progress()
        assert p["running"] == 0 and p["bytes_hashed"] == 0
    assert _snapshot_state(shm_tmp) == before


def test_retire_has_no_cpu_fallback(vm, shm_tmp):
    if not _no_gpu(vm):
        pytest.skip("a GPU is present; tests/test_retire.py covers the data path")
    pairs = _store(vm, shm_tmp)
    before = _snapshot_state(shm_tmp)
    rs = vm.RetireStats()
    rs.versions_retired = 7
    dirs = (ctypes.c_char_p * 2)(*[os.fsencode(d) for d, _ in pairs[:2]])
    tabs = (ctypes.c_char_p * 2)(*[os.fsencode(t) for _, t in pairs[:2]])
    kdirs = (ctypes.c_char_p * 2)(*[os.fsencode(d) for d, _ in pairs[2:]])
    ktabs = (ctypes.c_char_p * 2)(*[os.fsencode(t) for _, t in pairs[2:]])
    rc = vm.lib().vmig_retire_versions(2, dirs, tabs, 2, kdirs, ktabs, None, None, ctypes.byref(rs))
    assert rc == vm.VMIG_ENOGPU and rs.versions_retired == 7
    assert _snapshot_state(shm_tmp) == before


def test_retire_versions_keep_must_be_positive(vm, shm_tmp):
    import importlib
    ho = importlib.import_module(vm.__name__ + ".handoff")
    ho.set_merges_root(shm_tmp)
    try:
        for keep in (0, -1):
            with pytest.raises(ValueError):
                ho.RetireVersions("rs", keep)
        assert ho.RetireVersions("rs", 1) == {"retired": [], "kept": []}      # no store yet: nothing to do
    finally:
        ho.set_merges_root(None)


def test_retire_host_side_unit(tmp_path):
    """csrc/vmig_retire.cpp alone (no GPU, no CUDA): removal counts with hard links across two retired trees and one
    outside them, stale-record selection, grouping, the re-stamp decision and the table patch."""
    exe = tmp_path / "retire_unit"
    csrc = ROOT / "gpu-docker-api_b200" / "csrc"
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-pthread", "-I", str(csrc), str(ROOT / "tests" / "retire_unit.cpp"),
                    *[str(csrc / f) for f in ("vmig_retire.cpp", "vmig_scrub.cpp", "vmig_tree.cpp", "vmig_table.cpp")],
                    "-o", str(exe)], check=True)
    work = tmp_path / "work"
    work.mkdir()
    r = subprocess.run([str(exe), str(work)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "retire unit ok" in r.stdout, r.stdout + r.stderr
